"""Every shape of the GICP solve against the oracle, in every execution, with BFGS and Gauss-Newton.

The align picks its objective code from the source points each CTA owns (lb_gicp_align, gicp.cu): grid_for gives
grid = clamp(ceil(n_src / ppc), 8, SMs) CTAs (ppc = align_points_per_cta, 0 = 512), CTA c owns the contiguous chunk
[c * chunk, (c + 1) * chunk) with chunk = ceil(n_src / grid), and

    chunk        stream-ordered                   persistent                    host-driven
    <= 512       loop_solve_kernel<4, 256>,       align_persistent_kernel<4>    objective_kernel<13 / 28>,
                 correspondences in registers                                   read from global memory
    513..1024    loop_solve_kernel<8, 160>,       align_persistent_kernel<8>    same
                 correspondences in shared memory
    > 1024       <8, 160>, read back from L2      <8>, same                     same

The cluster execution is its own kernel up to 16 x 2816 source points and the persistent kernel above that.

Per case (ppc, n_src): the shape is restated here and the kernels that ran are read back from torch.profiler, so a
change of the boundaries fails instead of quietly testing another shape; host-driven, persistent and stream-ordered
agree bit for bit (same lane -> point mapping and reduction shape at every chunk size); the pose is within 1e-4 m /
1e-4 rad of the oracle with the same iteration, correspondence and inner-iteration counts, and the same number of
objective evaluations as the serial CPU build of the same driver (tests/hd_harness.cpp, held here to the oracle's
pose bits and counts on every input).  The oracle's own evaluation count is not comparable: it counts the
reference's separate f, df and fdf calls, which the library's driver serves from one fused pass (bfgs.h).
The inputs are seeded so that the oracle's own result does not move when only the association of its sums changes
(set_sum_chunk, and the order of the source points): on such inputs the counts are a sharp check of f and grad f,
and a kernel that drops, doubles or scrambles terms of the sums changes them.  The last test runs the odometry
pipeline's shape (1024 points per CTA) on consecutive pairs of a lidar stream against the oracle, which the pipeline
tests (GPU against blocking GPU calls) cannot do."""
import collections
import ctypes as C
import time

import numpy as np
import pytest

import fixtures as F
from test_gicp_gpu import NTHREADS, _assert_pose_parity, _mk

pytestmark = pytest.mark.gpu

PERSISTENT, HOST, CLUSTER, STREAM = 0, 1, 2, 3       # lb_execution
BFGS, GN = 0, 1                                      # lb_optimizer
AL_PPC, AL_ACC, AL_MAXCTA = 512, 128, 160            # gicp_kernels.cuh
CLUSTER_MAX_N = 16 * 2816                            # align_cluster.cuh: CL_SIZE x CL_CAP
REGS, SMEM, L2 = "registers", "shared memory", "L2"
CHUNKS = (64, 256, 1024, 4096, 16384)                # the re-associations of _assert_pose_parity
RESULT_FIELDS = ("converged", "iterations", "n_correspondences", "delta", "n_objective_evals", "n_inner_iterations")

Shape = collections.namedtuple("Shape", "grid chunk spans row stream persistent")


def shape(ppc, n_src, sms):
    """grid_for and the chunk rule of lb_gicp_align restated: CTAs, points per CTA, each CTA's [begin, end), and the
    objective path and kernel instantiations that chunk selects"""
    p = max(ppc if ppc > 0 else AL_PPC, AL_ACC)
    grid = min(max(-(-n_src // p), 8), sms, AL_MAXCTA)
    chunk = -(-n_src // grid)
    spans = [(min(n_src, c * chunk), min(n_src, min(n_src, c * chunk) + chunk)) for c in range(grid)]
    row = REGS if chunk <= AL_PPC else SMEM if chunk <= 2 * AL_PPC else L2
    ppl = 4 if row == REGS else 8
    stream = "loop_solve_kernel<4, 256>" if row == REGS else "loop_solve_kernel<8, 160>"
    return Shape(grid, chunk, spans, row, stream, "align_persistent_kernel<%d>" % ppl)


# (id, ppc, n_src or n_src(SMs), expected row, what else the shape must show, data seed).  The seeds are inputs on
# which the oracle's pose and counts are unchanged under the five set_sum_chunk re-associations and under
# permutations of the source.
Case = collections.namedtuple("Case", "id ppc n row expect seed")
CASES = [
    Case("floor8_registers", 0, 3000, REGS, dict(grid=8, chunk=375), 1),
    Case("standard", 0, 9000, REGS, dict(grid=18, chunk=500), 1),
    Case("min_ppc", 128, 30000, REGS, dict(grid="sms"), 1),
    Case("floor8_shared", 1024, 6000, SMEM, dict(grid=8, chunk=750), 1),
    Case("c2_worker", 1024, 30000, SMEM, dict(grid=30, chunk=1000), 1),
    Case("l2_2048", 2048, 20000, L2, dict(grid=10, chunk=2000), 1),
    Case("l2_4096", 4096, 40000, L2, dict(grid=10, chunk=4000), 1),
    Case("switch_to_shared", 0, lambda s: 512 * s + 1, SMEM, dict(grid="sms", chunk=513), 1),
    Case("switch_to_l2", 0, lambda s: 1024 * s + 1, L2, dict(grid="sms", chunk=1025), 1),
    Case("tiny4", 0, 4, REGS, dict(grid=8, empty=True), 1),
    Case("tiny5", 0, 5, REGS, dict(grid=8, empty=True), 1),
    Case("tiny9", 0, 9, REGS, dict(grid=8, empty=True), 1),
    Case("tiny37", 0, 37, REGS, dict(grid=8, last=2), 2),
    Case("tiny127", 0, 127, REGS, dict(grid=8, last=15), 2),
    Case("tiny129", 0, 129, REGS, dict(grid=8, last=10), 1),
    Case("single_point_tail", 0, 57, REGS, dict(grid=8, chunk=8, last=1), 1),
]


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def clouds(n, seed):
    """(source, target, oracle parameters).  Target: surface points of a room; source: another sample of the same
    room seen from a pose a few cm / mrad off, with about 3 % outliers that no target point is near (unmatched points
    take the zero-padded branch of every objective path).  Tiny sources: target points plus noise, k = n below 20."""
    rng = np.random.default_rng(1000 + seed)
    Tg = F.se3([0.15, -0.08, 0.04], [0.008, -0.012, 0.02])
    if n < 1000:
        tgt = F.random_scene(6000, 50 + seed)
        pick = tgt[rng.choice(len(tgt), n, replace=False)].astype(np.float64) + rng.normal(0, 0.005, (n, 3))
        Ts = F.se3([0.03, -0.02, 0.01], [0.002, -0.003, 0.004])
        src = ((pick - Ts[:3, 3]) @ Ts[:3, :3]).astype(np.float32)
        if n > 20:
            src[n // 2] = np.float32([60.0, 60.0, 60.0])
        return src, tgt, dict(transformation_epsilon=1e-4, corr_dist_threshold=0.5, max_iterations=30,
                              k_correspondences=min(20, n))
    src = (F.random_scene(n, seed).astype(np.float64) @ Tg[:3, :3].T + Tg[:3, 3]).astype(np.float32)
    out = rng.choice(n, n // 32, replace=False)
    src[out] = rng.uniform(-60, 60, (len(out), 3)).astype(np.float32) + np.float32([0, 0, 40])
    tgt = F.random_scene(max(n, 6000), 50 + seed)
    return src, tgt, dict(transformation_epsilon=1e-3, corr_dist_threshold=1.0, max_iterations=50)


def _kernels(run):
    """names of the CUDA kernels `run` launched"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = run()
    return out, {e.name for e in prof.events()}


def _bits(T):
    return np.asarray(T, np.float32).view(np.uint32)


def _fields(res):
    return tuple(getattr(res, f) for f in RESULT_FIELDS)


def _serial(harness, tag, src, tgt, prm, r):
    """The driver of bfgs.h built for the CPU with a serial backend (the oracle's summation order): its fused-pass
    count of objective evaluations.  Its pose bits, iteration, correspondence and inner-iteration counts must be the
    oracle's, which ties that count to the oracle on this very input."""
    src = np.ascontiguousarray(src, np.float32); tgt = np.ascontiguousarray(tgt, np.float32)
    T = np.zeros(16, np.float32); info = np.zeros(5, np.int32); d = np.zeros(1)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    harness.hh_align(p(src), len(src), p(tgt), len(tgt), 0.5, 0.5, prm.k_correspondences, prm.gicp_epsilon,
                     prm.rotation_epsilon, prm.transformation_epsilon, prm.corr_dist_threshold, prm.max_iterations,
                     prm.max_inner_iterations, prm.optimizer, None, p(T), p(info), p(d))
    assert np.array_equal(_bits(T.reshape(4, 4)), _bits(r["T"])), tag
    assert list(info[[0, 1, 2, 4]]) == [r["iterations"], int(r["converged"]), r["n_corr"], r["n_inner"]], (tag, info)
    return int(info[3])


def _counts_parity(oracle, tag, r, rerun, res, serial_evals, tally):
    """With the pose within the bar, the inner-iteration count must equal the oracle's and the objective-evaluation
    count the serial driver's -- except on an input whose oracle counts themselves change under the five
    re-associations of _assert_pose_parity, which is asserted and counted, never assumed"""
    want = (r["n_evals"], r["n_inner"])
    if (res.n_objective_evals, res.n_inner_iterations) == (serial_evals, r["n_inner"]):
        return
    moved = []
    for chunk in CHUNKS:
        oracle.set_sum_chunk(chunk)
        try:
            o = rerun()
        finally:
            oracle.set_sum_chunk(0)
        moved.append((o["n_evals"], o["n_inner"]) != want)
    assert any(moved), (tag, "evals / inner iterations", (res.n_objective_evals, res.n_inner_iterations), "serial driver",
                        (serial_evals, r["n_inner"]), "although the oracle's counts do not depend on the association of its sums on this input")
    tally.verdicts["counts_reference_not_reproducible"] += 1


def _parity(oracle, tag, r, rerun, T, res, serial_evals, tally):
    verdict = _assert_pose_parity(oracle, tag, r, rerun, T, res)
    tally.verdicts[verdict] += 1
    if verdict == "within_bar":
        _counts_parity(oracle, tag, r, rerun, res, serial_evals, tally)
    return verdict


class Tally:
    """verdicts of the oracle comparisons, and the time spent in the oracle"""

    def __init__(self):
        self.verdicts = collections.Counter()
        self.oracle_s = 0.0
        self.t0 = time.perf_counter()

    def timed(self, fn):
        def run():
            t = time.perf_counter()
            try:
                return fn()
            finally:
                self.oracle_s += time.perf_counter() - t
        return run


@pytest.fixture(scope="module")
def tally(request):
    t = Tally()
    yield t
    tr = request.config.pluginmanager.get_plugin("terminalreporter")
    if tr is not None and t.verdicts:
        tr.write_line("test_gicp_shapes_gpu: %.0f s, %.0f s of it in the oracle; comparisons: %s" % (
            time.perf_counter() - t.t0, t.oracle_s, ", ".join("%s %d" % kv for kv in sorted(t.verdicts.items()))))


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_solve_shape_vs_oracle_and_executions(oracle, harness, tally, case):
    sms = _sms()
    n = case.n(sms) if callable(case.n) else case.n
    sh = shape(case.ppc, n, sms)
    ex = case.expect
    assert sh.row == case.row, (case.id, sh.grid, sh.chunk)
    assert sh.grid == (sms if ex["grid"] == "sms" else ex["grid"]), (case.id, sh.grid)
    if "chunk" in ex:
        assert sh.chunk == ex["chunk"], (case.id, sh.chunk)
    if "last" in ex:
        assert sh.spans[-1][1] - sh.spans[-1][0] == ex["last"], (case.id, sh.spans[-1])
    assert any(b == e for b, e in sh.spans) == ex.get("empty", False), case.id
    src, tgt, kw = clouds(n, case.seed)
    assert src.shape[0] == n
    for opt in (BFGS, GN):
        tag = "%s n=%d ppc=%d %s" % (case.id, n, case.ppc, ("BFGS", "GN")[opt])
        prm = oracle.default_params(num_threads=NTHREADS, optimizer=opt, **kw)
        rerun = tally.timed(lambda: oracle.gicp_align(src, tgt, prm))
        r = rerun()
        assert r["status"] == 0 and r["n_corr"] >= 4, (tag, r["status"], r["n_corr"])

        def run():
            out = {}
            for e in (HOST, PERSISTENT, STREAM, CLUSTER):
                g = _mk(prm, e, opt)
                g.setCorrespondenceRandomness(kw.get("k_correspondences", 20))
                g.setAlignPointsPerCta(case.ppc)
                g.setInputSource(src); g.setInputTarget(tgt)
                res = g.align()
                out[e] = (g.getFinalTransformation(), res)
                g.close()
            return out
        out, names = _kernels(run)

        # the instantiations this shape selects ran, and the ones it does not select did not
        def ran(k):
            return any(k in s for s in names)
        other = shape(0, 1 if sh.row != REGS else 2 * AL_PPC * 8, 8)      # a shape of the other register width
        objective = "objective_kernel<%d>" % (13 if opt == BFGS else 28)
        assert ran(sh.stream) and not ran(other.stream), (tag, sorted(s for s in names if "_kernel<" in s))
        assert ran(sh.persistent) and not ran(other.persistent), (tag, sorted(s for s in names if "_kernel<" in s))
        assert ran(objective) and not ran("objective_kernel<%d>" % (28 if opt == BFGS else 13)), tag
        assert ran("align_cluster_kernel") == (n <= CLUSTER_MAX_N), tag

        # host-driven, persistent and stream-ordered: same bits, same counts
        T0, r0 = out[HOST]
        for e in (PERSISTENT, STREAM):
            T, res = out[e]
            assert np.array_equal(_bits(T), _bits(T0)) and _fields(res) == _fields(r0), (tag, e, _fields(res), _fields(r0))
        # the cluster kernel sums other partials (within 1e-6); above its capacity the request runs the persistent kernel
        Tc, rc = out[CLUSTER]
        if n <= CLUSTER_MAX_N:
            dt, dr = F.pose_delta(T0, Tc)
            assert dt <= 1e-6 and dr <= 1e-6, (tag, "cluster", dt, dr)
        else:
            assert np.array_equal(_bits(Tc), _bits(out[PERSISTENT][0])) and _fields(rc) == _fields(out[PERSISTENT][1]), tag

        _parity(oracle, tag, r, rerun, T0, r0, _serial(harness, tag, src, tgt, prm, r), tally)


def test_odometry_pipeline_shape_on_lidar_pairs_vs_oracle(oracle, harness, tally):
    """The odometry pipeline's registration settings (lb_locus_default_params().odometry: 1024 points per CTA, the
    shared-memory solve) on 6 consecutive scan pairs of a c2 lidar stream filtered at the c2 leaf, through blocking
    calls, against the oracle.  The pipeline tests then carry this to lb_odometry and lb_locus, whose results they
    hold bit-equal to such calls."""
    import locus_b200
    from tools import gen_lidar as G
    P = locus_b200.locus_params().odometry
    assert P.align_points_per_cta == 1024 and P.execution == STREAM
    _, _, blobs = G.stream(2, 7)
    vg = locus_b200.VoxelGridB200(); vg.setLeafSize(0.1088)
    vg.setFilterFieldName("z"); vg.setFilterLimits(-100, 100)
    f = [np.ascontiguousarray(vg.filter(b, 32, locus_b200.xyzi_fields())).view(np.float32).reshape(-1, 8)[:, :3].copy()
         for b in blobs]
    g = locus_b200.GicpB200()
    C.memmove(C.byref(g._p), C.byref(P), C.sizeof(P))
    g._apply()
    prm = oracle.default_params(k_correspondences=P.k_correspondences, gicp_epsilon=P.gicp_epsilon,
                                rotation_epsilon=P.rotation_epsilon, transformation_epsilon=P.transformation_epsilon,
                                corr_dist_threshold=P.max_correspondence_distance, max_iterations=P.max_iterations,
                                max_inner_iterations=P.max_optimizer_iterations, num_threads=NTHREADS)
    sms = _sms()
    verdicts = []
    for i in range(1, 7):
        src, tgt = f[i], f[i - 1]
        assert shape(1024, len(src), sms).row == SMEM, len(src)
        g.setInputSource(src); g.setInputTarget(tgt)
        res, names = _kernels(g.align)
        assert any("loop_solve_kernel<8, 160>" in s for s in names), i
        rerun = tally.timed(lambda: oracle.gicp_align(src, tgt, prm))
        r = rerun()
        tag = "c2 pair %d" % i
        verdicts.append(_parity(oracle, tag, r, rerun, g.getFinalTransformation(), res,
                                _serial(harness, tag, src, tgt, prm, r), tally))
    assert "within_bar" in verdicts, verdicts
