"""Pure-Python restatement of lb_locus's pose bookkeeping (locus_b200/csrc/lo_pose.h) and of the per-scan logic of
its localization stage (Locus.cc:462-543 as the chain runs it), for the tests.

Every value is a Python float (an IEEE double) and every operation is the one lo_pose.h performs, in the same order, so
the results are bit-equal to the C++ compiled with -ffp-contract=off.  The math functions are libm's (math.atan2,
math.asin, math.acos, math.sqrt); where the C functions return NaN outside their domain, the helpers below do too.

The registration and map calls are injected (LocusChain.scan's callbacks), so the same logic checks the GPU chain
against blocking GicpB200 / SubmapB200 calls and the host pipeline against fake stages."""
import math

import numpy as np

NAN = float("nan")


def sum3(a, b, c):
    return a + (b + c)


def _sqrt(x):
    return math.sqrt(x) if x >= 0.0 else NAN        # NaN compares false, as in C


def _asin(x):
    return math.asin(x) if -1.0 <= x <= 1.0 else NAN


def _acos(x):
    return math.acos(x) if -1.0 <= x <= 1.0 else NAN


class Pose:
    __slots__ = ("R", "t")

    def __init__(self, R, t):
        self.R = list(R)        # row-major 3x3
        self.t = list(t)


def identity():
    return Pose([1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0], [0.0, 0.0, 0.0])


def from_mat(m):
    """row-major 4x4 (any sequence of floats, float32 values widened exactly) -> Pose"""
    m = [float(x) for x in np.asarray(m).reshape(16)]
    return Pose([m[4 * r + c] for r in range(3) for c in range(3)], [m[3], m[7], m[11]])


def to_mat(p, dtype=np.float64):
    m = np.zeros(16, dtype=dtype)
    for r in range(3):
        for c in range(3):
            m[4 * r + c] = p.R[3 * r + c]
        m[4 * r + 3] = p.t[r]
    m[15] = 1.0
    return m


def update(a, b):
    R = [sum3(a.R[3 * r] * b.R[c], a.R[3 * r + 1] * b.R[3 + c], a.R[3 * r + 2] * b.R[6 + c]) for r in range(3) for c in range(3)]
    t = [a.t[r] + sum3(a.R[3 * r] * b.t[0], a.R[3 * r + 1] * b.t[1], a.R[3 * r + 2] * b.t[2]) for r in range(3)]
    return Pose(R, t)


def inverse(a):
    """matrix inverse of the rotation (adjugate / determinant), not the transpose: see lo_pose.h"""
    m = a.R
    c = [m[4] * m[8] - m[5] * m[7], m[5] * m[6] - m[3] * m[8], m[3] * m[7] - m[4] * m[6],
         m[2] * m[7] - m[1] * m[8], m[0] * m[8] - m[2] * m[6], m[1] * m[6] - m[0] * m[7],
         m[1] * m[5] - m[2] * m[4], m[2] * m[3] - m[0] * m[5], m[0] * m[4] - m[1] * m[3]]
    det = sum3(m[0] * c[0], m[1] * c[1], m[2] * c[2])
    R = [_div(c[3 * k + r], det) for r in range(3) for k in range(3)]
    t = [-sum3(R[3 * r] * a.t[0], R[3 * r + 1] * a.t[1], R[3 * r + 2] * a.t[2]) for r in range(3)]
    return Pose(R, t)


def _div(x, y):
    if y != 0.0:
        return x / y
    return NAN if x == 0.0 or x != x else math.copysign(math.inf, x) * math.copysign(1.0, y)


def delta(a, b):
    return update(inverse(a), b)


def translation_norm(p):
    return _sqrt(sum3(p.t[0] * p.t[0], p.t[1] * p.t[1], p.t[2] * p.t[2]))


def euler_zyx(p):
    return (math.atan2(p.R[7], p.R[8]), _asin(-p.R[6]), math.atan2(p.R[3], p.R[0]))


def euler_norm(p):
    e = euler_zyx(p)
    return _sqrt(sum3(e[0] * e[0], e[1] * e[1], e[2] * e[2]))


def quat_w(p):
    """w of Eigen's Quaterniond(Matrix3d), both branches"""
    m = p.R
    t = sum3(m[0], m[4], m[8])
    if t > 0.0:
        return 0.5 * _sqrt(t + 1.0)
    i = 0
    if m[4] > m[0]:
        i = 1
    if m[8] > m[3 * i + i]:
        i = 2
    j = (i + 1) % 3
    k = (j + 1) % 3
    t = _sqrt(m[3 * i + i] - m[3 * j + j] - m[3 * k + k] + 1.0)
    t = 0.5 / t if t != 0.0 else math.copysign(math.inf, t)
    return (m[3 * k + j] - m[3 * j + k]) * t


def keyframe_angle(p):
    return abs(2.0 * _acos(quat_w(p)))


def passes(p, enabled, max_translation, max_rotation):
    return (not enabled) or (translation_norm(p) <= max_translation and euler_norm(p) <= max_rotation)


def is_keyframe(d, t_kf, r_kf):
    return translation_norm(d) > t_kf or keyframe_angle(d) > r_kf


def f32(p):
    """float(P): the 4x4 float32 a pose is handed to the GPU as"""
    return to_mat(p, np.float32).reshape(4, 4)


class LocusChain:
    """The localization stage of lb_locus, one scan at a time.  `params` has the fields of lb_locus_params (a
    LocusParams or any object with those attributes)."""

    def __init__(self, params):
        self.p = params
        self.started = False
        self.O = identity()
        self.L = from_mat(list(params.initial_pose))
        self.KF = self.L
        self.counter = 0

    def scan(self, ok, odometry_T, localize, insert, crop):
        """ok: the voxel and odometry stages succeeded with a non-empty scan.  odometry_T: the odometry align's
        final_transformation (float32 4x4) or None when the scan has no odometry target.  localize(guess f32 4x4) ->
        final f32 4x4, or None
        when the align failed; insert(T f32 4x4) -> points added; crop(centre f32 (3,), half_size) -> points removed.
        Returns the record lb_locus_result reports."""
        rec = dict(odometry_accepted=0, has_localization=0, correction_accepted=0, keyframe=0, n_inserted=0, n_removed=0)
        I = identity()
        if ok:
            if odometry_T is not None:
                I = from_mat(odometry_T)
                th = self.p.odometry_thresholds
                rec["odometry_accepted"] = int(passes(I, th.enabled, th.max_translation, th.max_rotation))
                if rec["odometry_accepted"]:
                    self.O = update(self.O, I)
            if not self.started:
                self.started = True
                if self.p.prior_map:
                    self._localize(I, rec, localize, insert, crop)
                else:
                    rec["keyframe"] = 1
                    rec["n_inserted"] = insert(f32(self.L))
            else:
                self._localize(I, rec, localize, insert, crop)
        rec.update(O=to_mat(self.O), I=to_mat(I), L=to_mat(self.L))
        return rec

    def _localize(self, I, rec, localize, insert, crop):
        P = update(self.L, I)
        F = localize(f32(P))
        if F is None:                # the align failed: L and the keyframe state stay as they were
            return
        rec["has_localization"] = 1
        U = delta(P, from_mat(F))
        th = self.p.localization_thresholds
        rec["correction_accepted"] = int(passes(U, th.enabled, th.max_translation, th.max_rotation))
        self.L = update(self.L, update(I, U) if rec["correction_accepted"] else I)
        if not self.p.add_keyframes or not is_keyframe(delta(self.KF, self.L), self.p.translation_threshold_kf,
                                                       self.p.rotation_threshold_kf):
            return
        rec["keyframe"] = 1
        rec["n_inserted"] = insert(f32(self.L))
        self.counter += 1
        if self.counter == self.p.refresh_every:
            self.counter = 0
            if self.p.msw:
                rec["n_removed"] = crop(np.array(self.L.t, dtype=np.float32), self.p.window_half_size)
        self.KF = self.L
