// lo_pose_harness.cpp -- TEST-ONLY C entry points over locus_b200/csrc/lo_pose.h, built by tests/test_locus_cpu.py with
// the library's host flags (-ffp-contract=off) so that oracle/locus_oracle.py can be compared with it bit for bit.
#include "../locus_b200/csrc/lo_pose.h"

extern "C" {
void lp_update(const double* a, const double* b, double* out) { lo::to_mat(lo::update(lo::from_mat(a), lo::from_mat(b)), out); }
void lp_delta(const double* a, const double* b, double* out) { lo::to_mat(lo::delta(lo::from_mat(a), lo::from_mat(b)), out); }
void lp_from_float(const float* a, double* out) { lo::to_mat(lo::from_mat(a), out); }
void lp_to_float(const double* a, float* out) { lo::to_mat(lo::from_mat(a), out); }
void lp_euler(const double* a, double* rpy) { lo::euler_zyx(lo::from_mat(a), rpy); }
double lp_euler_norm(const double* a) { return lo::euler_norm(lo::from_mat(a)); }
double lp_translation_norm(const double* a) { return lo::translation_norm(lo::from_mat(a)); }
double lp_quat_w(const double* a) { return lo::quat_w(lo::from_mat(a)); }
double lp_keyframe_angle(const double* a) { return lo::keyframe_angle(lo::from_mat(a)); }
int lp_passes(const double* a, int enabled, double max_t, double max_r) { return lo::passes(lo::from_mat(a), enabled, max_t, max_r); }
int lp_is_keyframe(const double* a, double t_kf, double r_kf) { return lo::is_keyframe(lo::from_mat(a), t_kf, r_kf); }
}
