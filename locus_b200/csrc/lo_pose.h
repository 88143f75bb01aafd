// lo_pose.h -- the pose bookkeeping of LOCUS's lidar callback (host, double precision), as lb_locus_* runs it.
//
// The reference does this with geometry_utils (gu::Transform3, gu::PoseUpdate, gu::PoseDelta, Rot3::ToEulerZYX), which is
// not vendored in the reference tree.  Its definitions are restated here and are UNPINNED: the operations are the ones
// the reference's callers name, the rounding order is this header's choice:
//   * every three-term sum (matrix products, norms, the trace) is a + (b + c), the order of Eigen 3's unrolled
//     reduction of a fixed-size 3-vector;
//   * PoseUpdate(a, b): R = Ra Rb, t = ta + Ra tb;
//   * PoseDelta(a, b) = a^-1 b, with a^-1 = (Ra^-1, -(Ra^-1 ta)) and Ra^-1 the matrix inverse (adjugate / determinant)
//     rather than geometry_utils' transpose.  The localization correction U = P^-1 F (P the prediction, F the align's
//     float32 pose) is composed back into L, so L_k = P P^-1 F: with the transpose, P P^T != I by the float32 rounding
//     F carries, that error is fed back into L and grows about threefold per scan; with the inverse L_k ~ F and the
//     error stays that of one float32 pose;
//   * ToEulerZYX: roll = atan2(R21, R22), pitch = asin(-R20), yaw = atan2(R10, R00) (the extraction of gicp.hpp:235-241);
//     the thresholds use its Euclidean norm;
//   * the keyframe angle is 2 acos(q.w) with q = Eigen's Quaterniond(Matrix3d), restated below with both branches
//     (in the trace <= 0 branch w can be negative).
// Compiled with -ffp-contract=off (no fused multiply-add), so oracle/locus_oracle.py, which does the same operations
// on Python floats, gives the same bits.  Values outside a function's domain give NaN, which fails every threshold test.
#pragma once
#include <cmath>

namespace lo {

struct Pose {
  double R[9];   // row-major rotation
  double t[3];
};

inline double sum3(double a, double b, double c) { return a + (b + c); }

inline Pose identity() {
  Pose p;
  for (int i = 0; i < 9; i++) p.R[i] = (i % 4 == 0) ? 1.0 : 0.0;
  p.t[0] = p.t[1] = p.t[2] = 0.0;
  return p;
}

// row-major 4x4 (float or double) -> pose; the bottom row is ignored
template <typename T>
inline Pose from_mat(const T* m) {
  Pose p;
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) p.R[3 * r + c] = (double)m[4 * r + c];
    p.t[r] = (double)m[4 * r + 3];
  }
  return p;
}

template <typename T>
inline void to_mat(const Pose& p, T* m) {
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++) m[4 * r + c] = (T)p.R[3 * r + c];
    m[4 * r + 3] = (T)p.t[r];
  }
  m[12] = m[13] = m[14] = (T)0; m[15] = (T)1;
}

inline Pose update(const Pose& a, const Pose& b) {
  Pose o;
  for (int r = 0; r < 3; r++) {
    for (int c = 0; c < 3; c++)
      o.R[3 * r + c] = sum3(a.R[3 * r] * b.R[c], a.R[3 * r + 1] * b.R[3 + c], a.R[3 * r + 2] * b.R[6 + c]);
    o.t[r] = a.t[r] + sum3(a.R[3 * r] * b.t[0], a.R[3 * r + 1] * b.t[1], a.R[3 * r + 2] * b.t[2]);
  }
  return o;
}

inline Pose inverse(const Pose& a) {
  const double* m = a.R;
  // cofactors, row by row; the inverse is the transposed cofactor matrix over the determinant
  const double c[9] = {m[4] * m[8] - m[5] * m[7], m[5] * m[6] - m[3] * m[8], m[3] * m[7] - m[4] * m[6],
                       m[2] * m[7] - m[1] * m[8], m[0] * m[8] - m[2] * m[6], m[1] * m[6] - m[0] * m[7],
                       m[1] * m[5] - m[2] * m[4], m[2] * m[3] - m[0] * m[5], m[0] * m[4] - m[1] * m[3]};
  const double det = sum3(m[0] * c[0], m[1] * c[1], m[2] * c[2]);
  Pose o;
  for (int r = 0; r < 3; r++)
    for (int k = 0; k < 3; k++) o.R[3 * r + k] = c[3 * k + r] / det;
  for (int r = 0; r < 3; r++) o.t[r] = -sum3(o.R[3 * r] * a.t[0], o.R[3 * r + 1] * a.t[1], o.R[3 * r + 2] * a.t[2]);
  return o;
}

inline Pose delta(const Pose& a, const Pose& b) { return update(inverse(a), b); }

inline double translation_norm(const Pose& p) { return std::sqrt(sum3(p.t[0] * p.t[0], p.t[1] * p.t[1], p.t[2] * p.t[2])); }

inline void euler_zyx(const Pose& p, double* rpy) {
  rpy[0] = std::atan2(p.R[7], p.R[8]);
  rpy[1] = std::asin(-p.R[6]);
  rpy[2] = std::atan2(p.R[3], p.R[0]);
}

inline double euler_norm(const Pose& p) {
  double e[3];
  euler_zyx(p, e);
  return std::sqrt(sum3(e[0] * e[0], e[1] * e[1], e[2] * e[2]));
}

// w of Eigen's Quaterniond(const Matrix3d&) (Eigen/src/Geometry/Quaternion.h, quaternionbase_assign_impl)
inline double quat_w(const Pose& p) {
  const double* m = p.R;
  double t = sum3(m[0], m[4], m[8]);
  if (t > 0.0) return 0.5 * std::sqrt(t + 1.0);
  int i = 0;
  if (m[4] > m[0]) i = 1;
  if (m[8] > m[3 * i + i]) i = 2;
  const int j = (i + 1) % 3, k = (j + 1) % 3;
  t = std::sqrt(m[3 * i + i] - m[3 * j + j] - m[3 * k + k] + 1.0);
  t = 0.5 / t;
  return (m[3 * k + j] - m[3 * j + k]) * t;
}

inline double keyframe_angle(const Pose& p) { return std::fabs(2.0 * std::acos(quat_w(p))); }

// the transform_thresholding test of PointCloudOdometry.cc:305-307 and PointCloudLocalization.cc:369-371
inline bool passes(const Pose& p, int enabled, double max_translation, double max_rotation) {
  return !enabled || (translation_norm(p) <= max_translation && euler_norm(p) <= max_rotation);
}

// the keyframe test of Locus.cc:514-524 (delta = PoseDelta(last keyframe, current pose))
inline bool is_keyframe(const Pose& delta_kf, double t_kf, double r_kf) {
  return translation_norm(delta_kf) > t_kf || keyframe_angle(delta_kf) > r_kf;
}

}  // namespace lo
