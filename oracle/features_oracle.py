"""ctypes bindings of the feature-extraction oracle (oracle/features_oracle.c), built into its own library
oracle/_build/libfeatures_oracle.so with the flags of oracle/Makefile.

TEST INFRASTRUCTURE ONLY: imported by tests/ and tools/bench_features.py -- never by locus_b200/.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libfeatures_oracle.so")
_SRCS = ["features_oracle.c"]
# oracle/Makefile's CFLAGS: float32 arithmetic must not fuse (-ffp-contract=off), as in the reference's x86-64 build
_CFLAGS = ["-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-std=gnu11"]

# PointCloudFilter.h:79-96
DEFAULTS = dict(n_rings=16, lower_deg=-15.0, upper_deg=15.0, scan_period=0.1, curvature_region=5, n_feature_regions=6,
                max_corner_sharp=2, max_corner_less_sharp=20, max_surface_flat=4, curvature_threshold=0.1,
                less_flat_leaf=0.2)
COUNT_NAMES = ("n_arranged", "n_sharp", "n_less_sharp", "n_flat", "n_less_flat", "n_out")


class Params(C.Structure):
    _fields_ = [("n_rings", C.c_int), ("lower_deg", C.c_float), ("upper_deg", C.c_float), ("scan_period", C.c_float),
                ("curvature_region", C.c_int), ("n_feature_regions", C.c_int), ("max_corner_sharp", C.c_int),
                ("max_corner_less_sharp", C.c_int), ("max_surface_flat", C.c_int), ("curvature_threshold", C.c_float),
                ("less_flat_leaf", C.c_float)]


def params(**kw):
    d = dict(DEFAULTS)
    for k in kw:
        if k not in d:
            raise TypeError("unknown feature parameter %r" % k)
    d.update(kw)
    return d


def build(force=False):
    deps = _SRCS + ["features_oracle.py"]
    if not force and os.path.exists(_SO):
        mt = os.path.getmtime(_SO)
        if all(os.path.getmtime(os.path.join(_HERE, s)) <= mt for s in deps):
            return _SO
    os.makedirs(os.path.dirname(_SO), exist_ok=True)
    cc = os.environ.get("ORACLE_CC", "gcc")
    subprocess.check_call([cc] + _CFLAGS + ["-shared", "-o", _SO] + [os.path.join(_HERE, s) for s in _SRCS] + ["-lm"])
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_SO)
        L.of_extract_features.restype = C.c_int
        L.of_extract_features.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.POINTER(Params), C.c_void_p, C.c_size_t,
                                          C.c_void_p]
        _lib = L
    return _lib


def extract_features(xyz, **kw):
    """xyz: (n, >=3) float32 (x, y, z in the first three columns).  Returns (out (m, 4) float32, counts dict)."""
    a = np.ascontiguousarray(xyz, dtype=np.float32)
    assert a.ndim == 2 and a.shape[1] >= 3
    n = a.shape[0]
    P = Params(**params(**kw))
    cap = 2 * n + 1
    out = np.zeros((cap, 4), np.float32)
    cnt = np.zeros(6, np.uint64)
    s = lib().of_extract_features(a.ctypes.data_as(C.c_void_p), n, a.shape[1], C.byref(P), out.ctypes.data_as(C.c_void_p),
                                  cap, cnt.ctypes.data_as(C.c_void_p))
    if s == -1:
        raise ValueError("of_extract_features: empty input")
    assert s == 0, s
    counts = dict(zip(COUNT_NAMES, (int(c) for c in cnt)))
    return out[: counts["n_out"]].copy(), counts
