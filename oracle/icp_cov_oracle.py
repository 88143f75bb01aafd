"""Independent restatement of LOCUS's point-to-plane ICP covariance (PointCloudLocalization.cc:325-336, 398-421,
469-541, 723-750) for the tests of lb_gicp_icp_covariance.

Steps 1-4 (per point): the float32 transform of transformPointCloudWithNormals, the kd-tree's exact 1-NN (ties to the
lowest index), normalizePCloud (og_normalize_pcloud) and the Ap sum of the PointCloudF overload (og_compute_ap).
Steps 5-9 (6x6): partial-pivot LU inverse, Eigen's pivoting LDLT of the lower triangle, the clamp and the reference's
L D L^T rebuild without the permutation, the NaN fallbacks, and Eigen's two-sided Jacobi SVD -- written here as plain
loops over Python floats (IEEE doubles, no fused multiply-add), in the operation order DESIGN.md 4i and
locus_b200/csrc/icp_cov.h state.  It does not call that header.
"""
import math
import sys

import numpy as np

from oracle import oracle as O

CLAMPED, D_NAN, COV_NAN = 1, 2, 4
_DBL_MIN = sys.float_info.min
_EPS = sys.float_info.epsilon


def lu_inverse(A):
    """Eigen's Ap.inverse() for 6x6: PartialPivLU, then the identity solved column by column."""
    n = 6
    lu = [[float(A[i][j]) for j in range(n)] for i in range(n)]
    perm = list(range(n))
    for k in range(n):
        p, best = k, abs(lu[k][k])
        for i in range(k + 1, n):
            if abs(lu[i][k]) > best:
                p, best = i, abs(lu[i][k])
        if best != 0.0:
            if p != k:
                lu[k], lu[p] = lu[p], lu[k]
                perm[k], perm[p] = perm[p], perm[k]
            for i in range(k + 1, n):
                lu[i][k] = lu[i][k] / lu[k][k]
        for i in range(k + 1, n):
            for c in range(k + 1, n):
                lu[i][c] = lu[i][c] - lu[i][k] * lu[k][c]
    out = [[0.0] * n for _ in range(n)]
    for col in range(n):
        x = [1.0 if perm[i] == col else 0.0 for i in range(n)]
        for i in range(n):
            s = 0.0
            for j in range(i):
                s = s + lu[i][j] * x[j]
            x[i] = x[i] - s
        for i in range(n - 1, -1, -1):
            s = 0.0
            for j in range(i + 1, n):
                s = s + lu[i][j] * x[j]
            den = lu[i][i]
            num = x[i] - s
            x[i] = _div(num, den)
        for i in range(n):
            out[i][col] = x[i]
    return out


def _div(a, b):
    """IEEE double division (Python raises on a zero divisor)."""
    if b != 0.0 or math.isnan(a) or math.isnan(b):
        if math.isnan(a) or math.isnan(b):
            return math.nan
        return a / b
    if a == 0.0:
        return math.nan
    neg = (math.copysign(1.0, a) < 0) != (math.copysign(1.0, b) < 0)
    return -math.inf if neg else math.inf


def ldlt(M):
    """Eigen's LDLT<Lower> in place on a copy: returns (m, D); L = unit lower part of m."""
    n = 6
    m = [[float(M[i][j]) for j in range(n)] for i in range(n)]
    for k in range(n):
        b, best = k, abs(m[k][k])
        for i in range(k + 1, n):
            if abs(m[i][i]) > best:
                b, best = i, abs(m[i][i])
        if b != k:
            for j in range(k):
                m[k][j], m[b][j] = m[b][j], m[k][j]
            for i in range(b + 1, n):
                m[i][k], m[i][b] = m[i][b], m[i][k]
            m[k][k], m[b][b] = m[b][b], m[k][k]
            for i in range(k + 1, b):
                m[i][k], m[b][i] = m[b][i], m[i][k]
        if k > 0:
            tmp = [m[j][j] * m[k][j] for j in range(k)]
            s = 0.0
            for j in range(k):
                s = s + m[k][j] * tmp[j]
            m[k][k] = m[k][k] - s
            for i in range(k + 1, n):
                r = 0.0
                for j in range(k):
                    r = r + m[i][j] * tmp[j]
                m[i][k] = m[i][k] - r
        akk = m[k][k]
        if k == 0 and not abs(akk) > 0.0:
            break
        if abs(akk) > 0.0:
            for i in range(k + 1, n):
                m[i][k] = m[i][k] / akk
    return m, [m[i][i] for i in range(n)]


def _make_jacobi(x, y, z):
    deno = 2.0 * abs(y)
    if deno < _DBL_MIN:
        return 1.0, 0.0
    tau = (x - z) / deno
    w = math.sqrt(tau * tau + 1.0)
    t = 1.0 / (tau + w) if tau > 0.0 else 1.0 / (tau - w)
    sign_t = 1.0 if t > 0.0 else -1.0
    nn = 1.0 / math.sqrt(t * t + 1.0)
    return nn, -sign_t * (y / abs(y)) * abs(t) * nn


def condition_number(A):
    """max / min singular value of Eigen's JacobiSVD; NaN for a non-finite matrix."""
    n = 6
    vals = [float(A[i][j]) for i in range(n) for j in range(n)]
    if not all(math.isfinite(v) for v in vals):
        return math.nan
    scale = max(abs(v) for v in vals)
    if scale == 0.0:
        scale = 1.0
    w = [[float(A[i][j]) / scale for j in range(n)] for i in range(n)]
    max_diag = max(abs(w[i][i]) for i in range(n))
    finished = False
    while not finished:
        finished = True
        for p in range(1, n):
            for q in range(p):
                threshold = max(_DBL_MIN, 2.0 * _EPS * max_diag)
                if abs(w[p][q]) > threshold or abs(w[q][p]) > threshold:
                    finished = False
                    m00, m01, m10, m11 = w[p][p], w[p][q], w[q][p], w[q][q]
                    t, d = m00 + m11, m10 - m01
                    if abs(d) < _DBL_MIN:
                        c1, s1 = 1.0, 0.0
                    else:
                        u = t / d
                        tmp = math.sqrt(1.0 + u * u)
                        c1, s1 = u / tmp, 1.0 / tmp
                    a00 = c1 * m00 + s1 * m10
                    a01 = c1 * m01 + s1 * m11
                    a11 = -s1 * m01 + c1 * m11
                    cr, sr = _make_jacobi(a00, a01, a11)
                    cl, sl = c1 * cr - s1 * -sr, c1 * -sr + s1 * cr
                    for i in range(n):          # rows p, q <- J_left
                        x, y = w[p][i], w[q][i]
                        w[p][i] = cl * x + sl * y
                        w[q][i] = -sl * x + cl * y
                    for i in range(n):          # columns p, q <- J_right
                        x, y = w[i][p], w[i][q]
                        w[i][p] = cr * x + -sr * y
                        w[i][q] = sr * x + cr * y
                    max_diag = max(max_diag, max(abs(w[p][p]), abs(w[q][q])))
    sv = [abs(w[i][i]) * scale for i in range(n)]
    return _div(max(sv), min(sv))


def covariance(Ap, max_cov):
    """Steps 5-9: (cov 6x6 float64, condition number (NaN after the D-NaN return), flags)."""
    Ap = np.asarray(Ap, dtype=np.float64).reshape(6, 6)
    inv = lu_inverse(Ap.tolist())
    cov = [[0.05 * 0.05 * inv[i][j] for j in range(6)] for i in range(6)]
    fallback = [[max_cov if i == j else 0.0 for j in range(6)] for i in range(6)]
    m, D = ldlt(cov)
    if any(math.isnan(d) for d in D):
        return np.array(fallback), math.nan, D_NAN
    flags, recompute = 0, False
    for i in range(6):
        if D[i] <= 0.0:
            D[i] = 1e-12
            recompute = True
        if D[i] > max_cov:
            D[i] = max_cov
            recompute = True
    if recompute:
        flags |= CLAMPED
        L = [[m[i][c] if c < i else (1.0 if c == i else 0.0) for c in range(6)] for i in range(6)]
        LD = [[L[i][c] * D[c] for c in range(6)] for i in range(6)]
        cov = [[0.0] * 6 for _ in range(6)]
        for i in range(6):
            for j in range(6):
                s = 0.0
                for c in range(6):
                    s = s + LD[i][c] * L[j][c]
                cov[i][j] = s
    if any(math.isnan(v) for row in cov for v in row):
        cov = fallback
        flags |= COV_NAN
    return np.array(cov), condition_number(cov), flags


def transform(xyz, T):
    """pcl::transformPointCloud in float32: p0 + (p1 + (p2 + t))."""
    q = np.asarray(xyz, dtype=np.float32).reshape(-1, 3)
    T = np.asarray(T, dtype=np.float32).reshape(4, 4)
    out = np.empty_like(q)
    for r in range(3):
        out[:, r] = T[r, 0] * q[:, 0] + (T[r, 1] * q[:, 1] + (T[r, 2] * q[:, 2] + T[r, 3]))
    return out


def rotate_normals(nrm, R):
    """the normal rotation of transformPointCloudWithNormals in float32: r0 x + (r1 y + r2 z)."""
    v = np.asarray(nrm, dtype=np.float32).reshape(-1, 3)
    R = np.asarray(R, dtype=np.float32).reshape(3, 3)
    out = np.empty_like(v)
    for r in range(3):
        out[:, r] = R[r, 0] * v[:, 0] + (R[r, 1] * v[:, 1] + R[r, 2] * v[:, 2])
    return out


def icp_covariance(query, target, target_normals, T=None, correspondences=None, normal_rotation=None, max_cov=0.01,
                   tree=None):
    """Steps 1-9 for a query cloud against a target with normals (NaN rows = no normal).  Returns a dict like
    GicpB200.icpCovariance plus `correspondences`.  tree: an O.KdTree of `target` built beforehand (the reference
    searches the registration's own target tree)."""
    q = np.ascontiguousarray(query, dtype=np.float32).reshape(-1, 3)
    tgt = np.ascontiguousarray(target, dtype=np.float32).reshape(-1, 3)
    if correspondences is None:
        corr, _ = (tree or O.KdTree(tgt)).nn_batch(transform(q, T))
    else:
        corr = np.asarray(correspondences, dtype=np.int32)
    nrm = np.asarray(target_normals, dtype=np.float32).reshape(-1, 3)
    if normal_rotation is not None:
        nrm = rotate_normals(nrm, normal_rotation)
    a = O.normalize_pcloud(q)
    Ap = O.compute_ap(a, nrm, corr)
    used = int((~np.isnan(a).any(1) & ~np.isnan(nrm[corr]).any(1)).sum())
    cov, cond, flags = covariance(Ap, max_cov)
    return {"Ap": Ap, "covariance": cov, "condition_number": cond, "flags": flags, "n_query": q.shape[0],
            "n_used": used, "correspondences": corr}
