"""locus_b200 -- H100 (sm_90a) GICP scan matcher + VoxelGrid front-end for LOCUS.

The product is the C-ABI shared library `liblocus_b200.so` (hand-written CUDA
for sm_90a, see include/locus_b200.h).  This Python package is only the
host-side mirror of the reference's C++ interface used by the tests and
bench.py (the reference's own toolchain -- ROS/PCL C++ -- is absent here; the
C++ mirror a LOCUS maintainer would compile lives in locus_b200/host/).

There is NO CPU fallback: importing works without a GPU (so the symbol table
can be checked), but creating a handle without a CUDA device raises.
"""
from .api import (  # noqa: F401
    LocusB200Error, lib, lib_path, build, GicpB200, VoxelGridB200, SubmapB200, OdometryB200, OdometryResult, NdtB200, NdtParams, NdtResult, NDT_KDTREE, NDT_DIRECT26, NDT_DIRECT7, NDT_DIRECT1, GicpParams, GicpResult,
    LB_MEM_HOST, LB_MEM_DEVICE, LB_OPT_BFGS, LB_OPT_GAUSS_NEWTON, LB_EXEC_PERSISTENT, LB_EXEC_HOST_DRIVEN, LB_EXEC_PERSISTENT_CLUSTER, LB_EXEC_STREAM_ORDERED,
    device_count, xyzi_fields, LocusB200, LocusParams, LocusResult, locus_params,
)
