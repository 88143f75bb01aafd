"""ctypes bindings of the outlier-filter oracle (oracle/outlier_oracle.c on oracle/kdtree.c), built into its own
library oracle/_build/liboutlier_oracle.so with the flags of oracle/Makefile.

TEST INFRASTRUCTURE ONLY: imported by tests/ and tools/bench_outliers.py -- never by locus_b200/.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "liboutlier_oracle.so")
_SRCS = ["kdtree.c", "outlier_oracle.c"]
# oracle/Makefile's CFLAGS: float32 arithmetic must not fuse (-ffp-contract=off), as in the reference's x86-64 build
_CFLAGS = ["-O2", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wno-misleading-indentation",
           "-std=gnu11"]


def build(force=False):
    deps = _SRCS + ["lb_oracle.h", "outlier_oracle.py"]
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
        vp = C.c_void_p
        L.og_statistical_outlier_removal.restype = C.c_int
        L.og_statistical_outlier_removal.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, vp, vp, vp]
        L.og_sor_threshold.restype = C.c_int
        L.og_sor_threshold.argtypes = [vp, C.c_int, C.c_double, C.c_int, vp, vp]
        L.og_radius_outlier_removal.restype = C.c_int
        L.og_radius_outlier_removal.argtypes = [vp, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int, C.c_int, vp]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _as_cloud(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    assert a.ndim == 2 and a.shape[1] >= 3
    return a


def statistical_outlier_removal(pts, mean_k=10, std_mul=1.0, negative=False):
    """pcl::StatisticalOutlierRemoval.  pts: (n, >=3) float32.
    Returns (kept int32 ascending, mean_dist (n,) float32, stats3 = [mean, stddev, threshold] float64)."""
    p = _as_cloud(pts)
    n = p.shape[0]
    kept = np.zeros(max(n, 1), np.int32); md = np.zeros(n, np.float32); st = np.zeros(3)
    m = lib().og_statistical_outlier_removal(_p(p), n, p.shape[1], int(mean_k), float(std_mul), int(bool(negative)), _p(kept),
                                             _p(md), _p(st))
    if m < 0:
        raise ValueError("og_statistical_outlier_removal: need 1 <= mean_k and n >= mean_k + 1")
    return kept[:m], md, st


def sor_threshold(distances, std_mul=1.0, negative=False):
    """the statistics + flag pass of StatisticalOutlierRemoval on given per-point distances: (kept, stats3)"""
    d = np.ascontiguousarray(distances, dtype=np.float32)
    kept = np.zeros(max(len(d), 1), np.int32); st = np.zeros(3)
    m = lib().og_sor_threshold(_p(d), len(d), float(std_mul), int(bool(negative)), _p(kept), _p(st))
    return kept[:m], st


def radius_outlier_removal(pts, radius, min_neighbors, dense=True, negative=False):
    """pcl::RadiusOutlierRemoval, PCL's is_dense branch (k-NN form) or its radius-search branch.
    Returns the kept indices, int32 ascending."""
    p = _as_cloud(pts)
    n = p.shape[0]
    kept = np.zeros(max(n, 1), np.int32)
    m = lib().og_radius_outlier_removal(_p(p), n, p.shape[1], float(radius), int(min_neighbors), int(bool(dense)),
                                        int(bool(negative)), _p(kept))
    if m < 0:
        raise ValueError("og_radius_outlier_removal: need radius > 0 and min_neighbors >= 0")
    return kept[:m]
