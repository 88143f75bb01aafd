"""CPU restatement of lb_locus's front end -- TEST AND BENCHMARK INFRASTRUCTURE ONLY.

What LOCUS runs around its lidar callback in the shipped configuration, in plain sequential Python, for the tests and
tools/bench_locus.py to drive the pre-existing blocking calls with:

  adaptive_leaf(state, n, points_to_process)
      Locus::ApplyAdaptiveInputVoxelization (locus/src/Locus.cc:780-810), one filtered scan of n points at a time:
          d = clamp(leaf * (double(n) / double(points_to_process)), 0.01, 5.0)
          if |leaf - d| > 0.01 or counter % 20 == 0:  leaf = d, counter = 0   (the new leaf is published)
          counter += 1
      leaf starts at the VoxelGrid's leaf (double_param.value = 0.25 in Locus.cc:39, what the shipped launch sets), the
      counter at 0 (Locus.h:302).  The VoxelGrid applies float(leaf) on every axis (custom_voxel_grid.cc:62-73) to the
      next scan.  A scan whose VoxelGrid failed is a callback that never ran: nothing changes.

  SubmapNormalsOracle
      oracle/submap_oracle.py's map with a normal per point: the winning point of a voxel keeps its normal, points
      inserted without one get NaN, crops keep points and normals paired, and covariances from normals are
      C = I - (1 - eps) n n' in double of the float normal (hd.h cov_from_normal; CalculateCovarianceFromNormals is
      external to the reference, so this arithmetic is unpinned).

  FrontEndChain
      oracle/locus_oracle.py's LocusChain plus the leaf bookkeeping of the callback.  With `icp_covariance` enabled it
      also keeps what stage L hands to lb_gicp_icp_covariance and what it reports: `normal_rotation` (the float32
      rotation of P^-1 for the scan being localized, P the align's guess, inverted as lo_pose.h inverts it) and
      `published_condition_number(r)` (the last condition number computed; a D-NaN fallback keeps the previous one).
"""
import numpy as np

from oracle import locus_oracle as LO
from oracle import submap_oracle as SO

# the shipped configuration (locus.launch:177-181 NormalComputation k = 20; lo_settings.yaml:84-85; both registrations
# with covariances from normals: point_cloud_odometry parameters.yaml:27, point_cloud_localization parameters.yaml:41,45)
NO_RECOMPUTE = dict(recompute_source_covariance=0, recompute_target_covariance=0)
SHIPPED = dict(front_end=dict(normals_k=20, adaptive_voxelization=1, points_to_process=3000),
               odometry=dict(NO_RECOMPUTE), localization=dict(NO_RECOMPUTE))


class LeafState:
    def __init__(self, leaf):
        self.leaf = float(leaf)      # double_param.value
        self.counter = 0             # counter_voxel_


def adaptive_leaf(state, n, points_to_process):
    """one callback's update of `state` (a LeafState) after a filtered scan of n points; returns whether the leaf was
    published (the VoxelGrid's next leaf is float(state.leaf) either way)"""
    d = state.leaf * (float(n) / float(points_to_process))
    if d < 0.01:
        d = 0.01
    if d > 5.0:
        d = 5.0
    change = abs(state.leaf - d) > 0.01 or state.counter % 20 == 0
    if change:
        state.leaf = d
        state.counter = 0
    state.counter += 1
    return change


def cov_from_normals(normals, eps):
    """(n, 3, 3) float64: I - (1 - eps) n n', the operation order of hd.h cov_from_normal"""
    n = np.asarray(normals, np.float32).astype(np.float64)
    s = 1.0 - eps
    out = np.empty((len(n), 3, 3))
    for r in range(3):
        for c in range(3):
            i, j = min(r, c), max(r, c)           # the upper triangle, mirrored
            out[:, r, c] = (1.0 if r == c else 0.0) - (s * n[:, i]) * n[:, j]
    return out


class SubmapNormalsOracle(SO.SubmapOracle):
    def __init__(self, resolution):
        super().__init__(resolution)
        self.nrm = np.zeros((0, 3), dtype=np.float32)

    def insert(self, points, normals=None):
        """oracle/submap_oracle.py's insert, with the winning points' normals (NaN without normals)"""
        p = np.ascontiguousarray(points, dtype=np.float32)[:, :3]
        vox = self._voxels(np.where(np.isfinite(p), p, 0))
        added = []
        for i in range(len(p)):
            if not np.isfinite(p[i]).all():
                continue
            key = (int(vox[i, 0]), int(vox[i, 1]), int(vox[i, 2]))
            if key in self.occ:
                continue
            self.occ.add(key)
            added.append(i)
        if added:
            self.pts = np.concatenate([self.pts, p[added]])
            nn = (np.asarray(normals, np.float32)[:, :3][added] if normals is not None
                  else np.full((len(added), 3), np.nan, np.float32))
            self.nrm = np.concatenate([self.nrm, nn])
        return p[added]

    def crop(self, center, half):
        c = np.asarray(center, dtype=np.float32); h = np.float32(half)
        mn, mx = (c - h).astype(np.float32), (c + h).astype(np.float32)
        keep = ~(((self.pts < mn).any(axis=1)) | ((self.pts > mx).any(axis=1)))
        self.nrm = np.ascontiguousarray(self.nrm[keep])
        return super().crop(center, half)

    def normal_covariances(self, eps=1e-3):
        return cov_from_normals(self.nrm, eps)


class FrontEndChain(LO.LocusChain):
    """LocusChain plus the leaf bookkeeping: filtered(n) after every scan whose VoxelGrid succeeded"""

    def __init__(self, params, leaf0):
        super().__init__(params)
        self.leaf = LeafState(leaf0)
        self.next_leaf = np.float32(leaf0)
        self.normal_rotation = None
        self.condition_number = float("nan")      # nothing computed yet

    def filtered(self, n):
        """the VoxelGrid kept n points with leaf self.next_leaf; returns that leaf and updates it for the next scan"""
        used = self.next_leaf
        if self.p.front_end.adaptive_voxelization:
            if adaptive_leaf(self.leaf, n, self.p.front_end.points_to_process):
                self.next_leaf = np.float32(self.leaf.leaf)
        return used

    def _localize(self, I, rec, localize, insert, crop):
        # stage L's normal rotation for this scan: float32 of inverse(P).R, P = update(L, I)
        P = LO.update(self.L, I)
        self.normal_rotation = np.array(LO.inverse(P).R, dtype=np.float64).reshape(3, 3).astype(np.float32)
        return super()._localize(I, rec, localize, insert, crop)

    def published_condition_number(self, result=None):
        """the condition number lb_locus_result reports after a scan; result: the scan's lb_gicp_icp_covariance output
        (a dict with condition_number and flags) or None when the scan was not localized"""
        if result is not None and not (result["flags"] & 2):      # LB_ICPCOV_D_NAN keeps the previous value
            self.condition_number = result["condition_number"]
        return self.condition_number
