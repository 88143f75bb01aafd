/* ndt_layout_probe.c -- TEST-ONLY: prints sizeof / offsetof of the C-ABI structs the pipelines' NDT settings changed, one
 * "name value" per line, for tests/test_ndt_pipeline_cpu.py to compare with the ctypes mirrors in locus_b200/api.py. */
#include <stddef.h>
#include <stdio.h>

#include "../include/locus_b200.h"

#define SZ(T) printf("%s %zu\n", #T, sizeof(T))
#define OFF(T, f) printf("%s.%s %zu\n", #T, #f, offsetof(T, f))

int main(void) {
  SZ(lb_ndt_params); SZ(lb_ndt_result);
  SZ(lb_odometry_result);
  OFF(lb_odometry_result, ticket); OFF(lb_odometry_result, status); OFF(lb_odometry_result, has_pose);
  OFF(lb_odometry_result, n_filtered); OFF(lb_odometry_result, gicp); OFF(lb_odometry_result, error);
  OFF(lb_odometry_result, ndt);
  SZ(lb_locus_params);
  OFF(lb_locus_params, odometry); OFF(lb_locus_params, localization); OFF(lb_locus_params, odometry_thresholds);
  OFF(lb_locus_params, localization_thresholds); OFF(lb_locus_params, translation_threshold_kf);
  OFF(lb_locus_params, rotation_threshold_kf); OFF(lb_locus_params, add_keyframes); OFF(lb_locus_params, refresh_every);
  OFF(lb_locus_params, msw); OFF(lb_locus_params, window_half_size); OFF(lb_locus_params, prior_map);
  OFF(lb_locus_params, initial_pose); OFF(lb_locus_params, front_end); OFF(lb_locus_params, icp_covariance);
  OFF(lb_locus_params, odometry_method); OFF(lb_locus_params, localization_method); OFF(lb_locus_params, odometry_ndt);
  OFF(lb_locus_params, localization_ndt);
  SZ(lb_locus_result);
  OFF(lb_locus_result, ticket); OFF(lb_locus_result, status); OFF(lb_locus_result, error); OFF(lb_locus_result, n_filtered);
  OFF(lb_locus_result, has_odometry); OFF(lb_locus_result, odometry); OFF(lb_locus_result, odometry_accepted);
  OFF(lb_locus_result, has_localization); OFF(lb_locus_result, localization); OFF(lb_locus_result, correction_accepted);
  OFF(lb_locus_result, odometry_pose); OFF(lb_locus_result, incremental); OFF(lb_locus_result, pose);
  OFF(lb_locus_result, keyframe); OFF(lb_locus_result, n_inserted); OFF(lb_locus_result, n_removed);
  OFF(lb_locus_result, map_size); OFF(lb_locus_result, leaf_size); OFF(lb_locus_result, has_icp_covariance);
  OFF(lb_locus_result, icp_covariance); OFF(lb_locus_result, condition_number); OFF(lb_locus_result, icp_covariance_flags);
  OFF(lb_locus_result, odometry_ndt); OFF(lb_locus_result, localization_ndt);
  return 0;
}
