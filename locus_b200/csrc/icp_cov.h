// icp_cov.h -- the 6x6 part of LOCUS's point-to-plane ICP covariance (host, double precision), as
// lb_gicp_icp_covariance runs it after the GPU has accumulated Ap.
//
// PointCloudLocalization::ComputePoint2PlaneICPCovariance (point_cloud_localization/src/PointCloudLocalization.cc:469-541),
// steps 5-9 of the semantics in include/locus_b200.h, restated as written:
//   5. cov = 0.05 * 0.05 * Ap.inverse()                                                               (:487)
//   6. ldlt = cov.ldlt(); D has a NaN -> cov = max * I, return before the SVD (condition number kept)  (:491-502)
//   7. D_i <= 0 -> 1e-12, D_i > max -> max; if either happened cov = L * diag(D) * L^T               (:504-517)
//      AS WRITTEN: Eigen's LDLT pivots (P^T L D L^T P = cov), and the reference rebuilds without P, so the clamped
//      covariance is the symmetrically permuted P cov P^T.  This is not "fixed" here.
//   8. cov has a NaN -> max on the diagonal, 0 elsewhere                                               (:519-525)
//   9. condition number = s0 / s5 of JacobiSVD(cov)                                                    (:528-538)
//
// Eigen is not vendored in the reference tree (LOCUS builds against the system Eigen, 3.3.7 on ROS noetic).  The
// readings below are therefore UNPINNED, like the other Eigen readings in DESIGN.md section 2:
//   * inverse(): partial-pivot LU (PartialPivLU, unblocked for 6x6): pivot = largest |a_ik| in column k, first index on
//     ties, a comparison with NaN is false; a zero pivot leaves its column unscaled; then the identity is solved by
//     forward (unit lower) and back (upper) substitution per column, each dot product summed in ascending index.  A
//     zero pivot divides by zero there: a singular Ap gives inf / NaN, as in Eigen.  Eigen's PartialPivLU::inverse
//     solves the identity through its blocked triangular-solve kernel, whose update order may differ from these
//     dot products in the last bits.
//   * ldlt(): Eigen's ldlt_inplace<Lower>: reads the lower triangle; pivot = largest |remaining diagonal|, first index
//     on ties (a NaN never wins a comparison); the row / column swap as Eigen performs it on the lower triangle;
//     mat(k,k) -= sum_j mat(k,j) * (D_j mat(k,j)); column k below the pivot -= sum_j mat(i,j) * (D_j mat(k,j)), then
//     divided by the pivot when the pivot is non-zero (a zero pivot leaves the column as it is).  Sums ascend in j.
//     A first pivot that is zero or NaN ends the factorisation at once (Eigen's early return for an all-zero diagonal).
//   * L * diag(D) * L^T: (L D)(i,m) = L(i,m) D(m), then sum over m ascending.
//   * JacobiSVD: the matrix is divided by its largest |entry| (a non-finite one makes the SVD invalid: condition number
//     NaN here; whether Eigen 3.3.7 already returns early on a non-finite input is itself unpinned), then Eigen's
//     cyclic two-sided Jacobi sweeps (real_2x2_jacobi_svd + makeJacobi, p = 1..5, q < p, threshold
//     max(DBL_MIN, 2 eps max|diag|)) until no off-diagonal pair exceeds the threshold; singular values = |diag| * scale.
//     The condition number is max / min of them (= s0 / s5 after Eigen's descending sort).
// Compiled with -ffp-contract=off (no fused multiply-add); oracle/icp_cov_oracle.py restates the same operations on
// Python floats and gives the same bits.
#pragma once
#include <cfloat>
#include <cmath>

namespace icpcov {

enum { CLAMPED = 1, D_NAN = 2, COV_NAN = 4 };   // LB_ICPCOV_* of include/locus_b200.h

struct Result {
  double cov[36];
  double condition_number;   // NaN when step 6 returned early (the caller keeps its previous value)
  int flags;
};

// 5: Ainv = inverse(A) through PartialPivLU
inline void lu_inverse(const double* A, double* out) {
  double lu[36];
  for (int i = 0; i < 36; i++) lu[i] = A[i];
  int perm[6] = {0, 1, 2, 3, 4, 5};
  for (int k = 0; k < 6; k++) {
    int p = k;
    double best = std::fabs(lu[6 * k + k]);
    for (int i = k + 1; i < 6; i++) {
      const double v = std::fabs(lu[6 * i + k]);
      if (v > best) { best = v; p = i; }
    }
    if (best != 0.0) {
      if (p != k) {
        for (int c = 0; c < 6; c++) { const double t = lu[6 * k + c]; lu[6 * k + c] = lu[6 * p + c]; lu[6 * p + c] = t; }
        const int t = perm[k]; perm[k] = perm[p]; perm[p] = t;
      }
      for (int i = k + 1; i < 6; i++) lu[6 * i + k] = lu[6 * i + k] / lu[6 * k + k];
    }
    for (int i = k + 1; i < 6; i++)
      for (int c = k + 1; c < 6; c++) lu[6 * i + c] = lu[6 * i + c] - lu[6 * i + k] * lu[6 * k + c];
  }
  for (int col = 0; col < 6; col++) {
    double x[6];
    for (int i = 0; i < 6; i++) x[i] = perm[i] == col ? 1.0 : 0.0;     // P * identity
    for (int i = 0; i < 6; i++) {
      double s = 0.0;
      for (int j = 0; j < i; j++) s = s + lu[6 * i + j] * x[j];
      x[i] = x[i] - s;
    }
    for (int i = 5; i >= 0; i--) {
      double s = 0.0;
      for (int j = i + 1; j < 6; j++) s = s + lu[6 * i + j] * x[j];
      x[i] = (x[i] - s) / lu[6 * i + i];
    }
    for (int i = 0; i < 6; i++) out[6 * i + col] = x[i];
  }
}

// 6: Eigen's LDLT of the lower triangle of m (in place); D = diagonal, L = unit lower part
inline void ldlt(double* m, double* D) {
  for (int k = 0; k < 6; k++) {
    int b = k;
    double best = std::fabs(m[6 * k + k]);
    for (int i = k + 1; i < 6; i++) {
      const double v = std::fabs(m[6 * i + i]);
      if (v > best) { best = v; b = i; }
    }
    if (b != k) {
      for (int j = 0; j < k; j++) { const double t = m[6 * k + j]; m[6 * k + j] = m[6 * b + j]; m[6 * b + j] = t; }
      for (int i = b + 1; i < 6; i++) { const double t = m[6 * i + k]; m[6 * i + k] = m[6 * i + b]; m[6 * i + b] = t; }
      { const double t = m[6 * k + k]; m[6 * k + k] = m[6 * b + b]; m[6 * b + b] = t; }
      for (int i = k + 1; i < b; i++) { const double t = m[6 * i + k]; m[6 * i + k] = m[6 * b + i]; m[6 * b + i] = t; }
    }
    double tmp[6];
    if (k > 0) {
      for (int j = 0; j < k; j++) tmp[j] = m[6 * j + j] * m[6 * k + j];
      double s = 0.0;
      for (int j = 0; j < k; j++) s = s + m[6 * k + j] * tmp[j];
      m[6 * k + k] = m[6 * k + k] - s;
      for (int i = k + 1; i < 6; i++) {
        double r = 0.0;
        for (int j = 0; j < k; j++) r = r + m[6 * i + j] * tmp[j];
        m[6 * i + k] = m[6 * i + k] - r;
      }
    }
    const double akk = m[6 * k + k];
    if (k == 0 && !(std::fabs(akk) > 0.0)) break;   // the whole diagonal is zero (or the first pivot NaN): Eigen stops here
    if (std::fabs(akk) > 0.0)
      for (int i = k + 1; i < 6; i++) m[6 * i + k] = m[6 * i + k] / akk;
  }
  for (int i = 0; i < 6; i++) D[i] = m[6 * i + i];
}

// Eigen's JacobiRotation (c, s)
struct Rot { double c, s; };

// JacobiRotation::makeJacobi(x, y, z)
inline Rot make_jacobi(double x, double y, double z) {
  const double deno = 2.0 * std::fabs(y);
  if (deno < DBL_MIN) return Rot{1.0, 0.0};
  const double tau = (x - z) / deno;
  const double w = std::sqrt(tau * tau + 1.0);
  const double t = tau > 0.0 ? 1.0 / (tau + w) : 1.0 / (tau - w);
  const double sign_t = t > 0.0 ? 1.0 : -1.0;
  const double n = 1.0 / std::sqrt(t * t + 1.0);
  return Rot{n, -sign_t * (y / std::fabs(y)) * std::fabs(t) * n};
}

// rows p, q of m <- J (apply_rotation_in_the_plane)
inline void rot_left(double* m, int p, int q, Rot j) {
  for (int i = 0; i < 6; i++) {
    const double x = m[6 * p + i], y = m[6 * q + i];
    m[6 * p + i] = j.c * x + j.s * y;
    m[6 * q + i] = -j.s * x + j.c * y;
  }
}

// columns p, q of m <- m J (applyOnTheRight: the rotation in the plane with J^T = (c, -s))
inline void rot_right(double* m, int p, int q, Rot j) {
  for (int i = 0; i < 6; i++) {
    const double x = m[6 * i + p], y = m[6 * i + q];
    m[6 * i + p] = j.c * x + -j.s * y;
    m[6 * i + q] = j.s * x + j.c * y;
  }
}

// 9: max / min singular value (Eigen's JacobiSVD without U / V); NaN when a coefficient is not finite
inline double condition_number(const double* A) {
  double scale = 0.0;
  bool finite = true;
  for (int i = 0; i < 36; i++) {
    if (!std::isfinite(A[i])) finite = false;
    const double v = std::fabs(A[i]);
    if (v > scale) scale = v;
  }
  if (!finite) return NAN;
  if (scale == 0.0) scale = 1.0;
  double w[36];
  for (int i = 0; i < 36; i++) w[i] = A[i] / scale;
  const double precision = 2.0 * DBL_EPSILON;
  double max_diag = 0.0;
  for (int i = 0; i < 6; i++) { const double v = std::fabs(w[6 * i + i]); if (v > max_diag) max_diag = v; }
  bool finished = false;
  while (!finished) {
    finished = true;
    for (int p = 1; p < 6; p++)
      for (int q = 0; q < p; q++) {
        const double threshold = std::fmax(DBL_MIN, precision * max_diag);
        if (std::fabs(w[6 * p + q]) > threshold || std::fabs(w[6 * q + p]) > threshold) {
          finished = false;
          // real_2x2_jacobi_svd on the (p, q) block
          double m00 = w[6 * p + p], m01 = w[6 * p + q], m10 = w[6 * q + p], m11 = w[6 * q + q];
          const double t = m00 + m11, d = m10 - m01;
          Rot r1;
          if (std::fabs(d) < DBL_MIN) {
            r1 = Rot{1.0, 0.0};
          } else {
            const double u = t / d;
            const double tmp = std::sqrt(1.0 + u * u);
            r1 = Rot{u / tmp, 1.0 / tmp};
          }
          const double a00 = r1.c * m00 + r1.s * m10, a01 = r1.c * m01 + r1.s * m11;
          const double a11 = -r1.s * m01 + r1.c * m11;
          m00 = a00; m01 = a01; m11 = a11;
          const Rot jr = make_jacobi(m00, m01, m11);
          // j_left = r1 * jr^T, Eigen's JacobiRotation product with jr^T = (c, -s)
          const Rot jl{r1.c * jr.c - r1.s * -jr.s, r1.c * -jr.s + r1.s * jr.c};
          rot_left(w, p, q, jl);
          rot_right(w, p, q, jr);
          max_diag = std::fmax(max_diag, std::fmax(std::fabs(w[6 * p + p]), std::fabs(w[6 * q + q])));
        }
      }
  }
  double smax = 0.0, smin = INFINITY;
  for (int i = 0; i < 6; i++) {
    const double s = std::fabs(w[6 * i + i]) * scale;
    if (s > smax) smax = s;
    if (s < smin) smin = s;
  }
  return smax / smin;
}

// steps 5-9 for Ap (36 doubles, row-major) and icp_max_covariance `max_cov`
inline Result compute(const double* Ap, double max_cov) {
  Result r;
  r.flags = 0;
  double inv[36];
  lu_inverse(Ap, inv);
  for (int i = 0; i < 36; i++) r.cov[i] = 0.05 * 0.05 * inv[i];
  double m[36], D[6];
  for (int i = 0; i < 36; i++) m[i] = r.cov[i];
  ldlt(m, D);
  bool d_nan = false;
  for (int i = 0; i < 6; i++) d_nan = d_nan || std::isnan(D[i]);
  if (d_nan) {
    for (int i = 0; i < 36; i++) r.cov[i] = (i % 7 == 0) ? max_cov : 0.0;
    r.condition_number = NAN;
    r.flags = D_NAN;
    return r;
  }
  bool recompute = false;
  for (int i = 0; i < 6; i++) {
    if (D[i] <= 0.0) { D[i] = 1e-12; recompute = true; }
    if (D[i] > max_cov) { D[i] = max_cov; recompute = true; }
  }
  if (recompute) {
    r.flags |= CLAMPED;
    double LD[36];
    for (int i = 0; i < 6; i++)
      for (int c = 0; c < 6; c++) LD[6 * i + c] = (c < i ? m[6 * i + c] : c == i ? 1.0 : 0.0) * D[c];
    for (int i = 0; i < 6; i++)
      for (int j = 0; j < 6; j++) {
        double s = 0.0;
        for (int c = 0; c < 6; c++) s = s + LD[6 * i + c] * (c < j ? m[6 * j + c] : c == j ? 1.0 : 0.0);
        r.cov[6 * i + j] = s;
      }
  }
  bool c_nan = false;
  for (int i = 0; i < 36; i++) c_nan = c_nan || std::isnan(r.cov[i]);
  if (c_nan) {
    for (int i = 0; i < 36; i++) r.cov[i] = (i % 7 == 0) ? max_cov : 0.0;
    r.flags |= COV_NAN;
  }
  r.condition_number = condition_number(r.cov);
  return r;
}

}  // namespace icpcov
