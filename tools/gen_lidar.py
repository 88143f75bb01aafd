"""Synthetic 64-beam lidar stream for the BASELINE.json configs (SURVEY.md section 8d).

Analytic scene: axis-aligned room 40 x 30 x 6 m + 12 boxes + 8 vertical
cylinders (positions from np.random.default_rng(seed)); HDL-64E-like sensor:
`beams` elevations linearly spaced in [-24.8 deg, +2.0 deg], `az` azimuth steps
-> beams*az rays per scan (64*2048 = 131072).  Range noise N(0, 0.02 m), 1 %
drop-outs -> NaN (exercises the finite check of the voxel filter).

Output layout = pcl::PointXYZI as it leaves the BodyFilter nodelet
(point_cloud_filter/src/body_filter.cc:36-39): point_step 32 bytes,
x@0 y@4 z@8 (float32), intensity@16 (float32), the rest padding.
"""
import numpy as np

POINT_STEP = 32
X_OFF, Y_OFF, Z_OFF, I_OFF = 0, 4, 8, 16
FLOAT_FIELDS = (0, 4, 8, 16)

ROOM_MIN = np.array([-20.0, -15.0, -1.5])
ROOM_MAX = np.array([20.0, 15.0, 4.5])


def make_scene(seed):
    rng = np.random.default_rng(seed)
    boxes = []
    for _ in range(12):
        c = np.array([rng.uniform(-17, 17), rng.uniform(-12, 12), 0.0])
        h = np.array([rng.uniform(0.4, 2.0), rng.uniform(0.4, 2.0), rng.uniform(0.5, 2.5)])
        lo = np.array([c[0] - h[0], c[1] - h[1], ROOM_MIN[2]])
        hi = np.array([c[0] + h[0], c[1] + h[1], ROOM_MIN[2] + 2 * h[2]])
        boxes.append((lo, hi))
    cyls = []
    for _ in range(8):
        cyls.append((rng.uniform(-17, 17), rng.uniform(-12, 12), rng.uniform(0.2, 0.8)))
    return {"boxes": boxes, "cyls": cyls, "seed": seed}


def _rot(rpy):
    r, p, y = rpy
    cr, sr, cp, sp, cy, sy = np.cos(r), np.sin(r), np.cos(p), np.sin(p), np.cos(y), np.sin(y)
    Rz = np.array([[cy, -sy, 0], [sy, cy, 0], [0, 0, 1.0]])
    Ry = np.array([[cp, 0, sp], [0, 1, 0], [-sp, 0, cp]])
    Rx = np.array([[1, 0, 0], [0, cr, -sr], [0, sr, cr]])
    return Rz @ Ry @ Rx


def pose_matrix(t, rpy):
    T = np.eye(4)
    T[:3, :3] = _rot(rpy)
    T[:3, 3] = t
    return T


def trajectory(seed, n, t_step=0.3, r_step_deg=2.0):
    """World poses of the sensor: random walk, ego-motion per frame t~U(-t_step,t_step) per
    axis, rpy~U(-r_step,r_step) (inside the 1.0 m / 1.0 rad gates of the callers)."""
    rng = np.random.default_rng(seed + 1000)
    T = np.eye(4)
    poses = [T.copy()]
    for _ in range(n - 1):
        for _try in range(100):
            dt = rng.uniform(-t_step, t_step, 3)
            dt[2] *= 0.2
            dr = np.deg2rad(rng.uniform(-r_step_deg, r_step_deg, 3))
            Tn = T @ pose_matrix(dt, dr)
            p = Tn[:3, 3]
            # stay well inside the room and near-level
            if (abs(p[0]) < 8 and abs(p[1]) < 6 and abs(p[2]) < 0.8 and abs(Tn[2, 2]) > 0.95):
                break
        T = Tn
        poses.append(T.copy())
    return poses


def _ray_dirs(beams, az, elev_deg=(-24.8, 2.0)):
    el = np.deg2rad(np.linspace(elev_deg[0], elev_deg[1], beams))
    a = np.linspace(0, 2 * np.pi, az, endpoint=False)
    ce, se = np.cos(el)[:, None], np.sin(el)[:, None]
    d = np.stack([ce * np.cos(a)[None, :], ce * np.sin(a)[None, :], se * np.ones_like(a)[None, :]], axis=-1)
    return d.reshape(-1, 3)


def _cast(scene, o, d):
    """o: (3,), d: (n,3) unit. returns range t (n,), inf if nothing hit."""
    n = d.shape[0]
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / d
        # room interior: exit distance
        t1 = (ROOM_MIN - o) * inv
        t2 = (ROOM_MAX - o) * inv
        texit = np.min(np.maximum(t1, t2), axis=1)
        t = texit.copy()
        for lo, hi in scene["boxes"]:
            a = (lo - o) * inv
            b = (hi - o) * inv
            tn = np.max(np.minimum(a, b), axis=1)
            tf = np.min(np.maximum(a, b), axis=1)
            hit = (tn <= tf) & (tn > 0.05)
            t = np.where(hit & (tn < t), tn, t)
        for cx, cy, r in scene["cyls"]:
            ox, oy = o[0] - cx, o[1] - cy
            A = d[:, 0] ** 2 + d[:, 1] ** 2
            B = 2 * (ox * d[:, 0] + oy * d[:, 1])
            Cc = ox * ox + oy * oy - r * r
            disc = B * B - 4 * A * Cc
            ok = (disc > 0) & (A > 1e-12)
            sq = np.sqrt(np.where(ok, disc, 0))
            tc = np.where(ok, (-B - sq) / (2 * A), np.inf)
            hit = ok & (tc > 0.05) & (tc < t)
            t = np.where(hit, tc, t)
    return t


def scan(scene, pose, seed, beams=64, az=2048, noise=0.02, dropout=0.01, elev_deg=(-24.8, 2.0)):
    """One scan in the SENSOR frame.  returns uint8 blob (n*32,), n = beams*az.  elev_deg: the beams' elevation span
    (a VLP-16 sweep: beams=16, az=1800, elev_deg=(-15.0, 15.0))."""
    rng = np.random.default_rng(seed)
    d_s = _ray_dirs(beams, az, elev_deg)
    R = pose[:3, :3]
    o = pose[:3, 3]
    d_w = d_s @ R.T
    t = _cast(scene, o, d_w)
    t = t + rng.normal(0, noise, t.shape)
    drop = rng.random(t.shape) < dropout
    t = np.where(drop | ~np.isfinite(t) | (t > 120.0), np.nan, t)
    p = (d_s * t[:, None]).astype(np.float32)
    inten = (100.0 / (1.0 + np.nan_to_num(t))).astype(np.float32)
    n = p.shape[0]
    blob = np.zeros((n, POINT_STEP // 4), dtype=np.float32)
    blob[:, 0:3] = p
    blob[:, 3] = 1.0
    blob[:, 4] = inten
    return blob.view(np.uint8).reshape(-1)


def blob_xyz(blob, point_step=POINT_STEP):
    a = np.ascontiguousarray(blob).view(np.uint8).reshape(-1, point_step)
    return a[:, :12].copy().view(np.float32).reshape(-1, 3)


WORKERS = 1      # processes used to ray-cast the scans of a stream (bench.py raises it; the scans do not depend on it)


def _scan_job(a):
    scene, pose, seed, beams, az = a
    return scan(scene, pose, seed, beams, az)


def _world_job(a):
    scene, T, seed, beams, az = a
    p = blob_xyz(scan(scene, T, seed, beams, az))
    p = p[np.isfinite(p).all(axis=1)]
    return (p.astype(np.float64) @ T[:3, :3].T + T[:3, 3]).astype(np.float32)


def _map_jobs(fn, jobs):
    if WORKERS > 1 and len(jobs) > 1:
        import multiprocessing as mp
        with mp.get_context("fork").Pool(min(WORKERS, len(jobs))) as pool:      # fork: call before CUDA is initialised
            return pool.map(fn, jobs)
    return [fn(j) for j in jobs]


def stream(seed, n_scans, beams=64, az=2048):
    """(scene, poses, [blob...]) for a stream of n_scans."""
    scene = make_scene(seed)
    poses = trajectory(seed, n_scans)
    blobs = _map_jobs(_scan_job, [(scene, poses[i], seed * 7919 + i, beams, az) for i in range(n_scans)])
    return scene, poses, blobs


def world_points(scene, poses, seed, beams=64, az=2048):
    """Union of posed scans in the world frame (finite points only), float32 (n,3)."""
    return np.concatenate(_map_jobs(_world_job, [(scene, T, seed * 104729 + i, beams, az) for i, T in enumerate(poses)]))


if __name__ == "__main__":
    import argparse
    import time
    ap = argparse.ArgumentParser()
    ap.add_argument("--seed", type=int, default=2)
    ap.add_argument("--scans", type=int, default=2)
    a = ap.parse_args()
    t0 = time.time()
    scene, poses, blobs = stream(a.seed, a.scans)
    p = blob_xyz(blobs[0])
    fin = np.isfinite(p).all(axis=1)
    print("scans", len(blobs), "pts/scan", p.shape[0], "finite", int(fin.sum()),
          "bbox", p[fin].min(0), p[fin].max(0), "gen s/scan", (time.time() - t0) / a.scans)


# ------------------------------------------------------------------------------------------ C3 / C4 / C5 workloads
# sensor -> base_link mounts of the three lidars point_cloud_merger concatenates (PointCloudMerger.cc:150-178)
LIDAR_MOUNTS = (pose_matrix([0.3, 0.0, 0.4], [0.0, 0.0, 0.0]),
                pose_matrix([-0.2, 0.25, 0.3], [0.0, 0.05, 2.1]),
                pose_matrix([-0.2, -0.25, 0.3], [0.0, 0.05, -2.1]))


def merged_scan(seed, beams=64, az=2048):
    """One sweep of the three lidars in base_link, concatenated in merger order, finite points only: float32 (n, 3),
    n ~ 3 * 0.99 * beams * az (~390 k at 64 x 2048) -- the full-resolution cloud the merger's radius filter sees."""
    return world_points(make_scene(seed), LIDAR_MOUNTS, seed, beams, az)


def _merged_job(a):
    scene, P, seed, beams, az = a
    return [scan(scene, P @ M, seed * 3 + i, beams, az) for i, M in enumerate(LIDAR_MOUNTS)]


def merged_stream(seed, n_scans, beams=64, az=2048):
    """A robot with the three lidars of LIDAR_MOUNTS driving the trajectory of stream(seed, n_scans): per scan k the
    three SENSOR-frame blobs of the mounts at base pose P_k (scan(scene, P_k @ M_i, ...)), in merger order.  Returns
    (scene, base poses P_k (the ground truth), [[blob_a, blob_b, blob_c] per scan], mounts as float32 4x4 sensor ->
    base_link)."""
    scene = make_scene(seed)
    poses = trajectory(seed, n_scans)
    scans = _map_jobs(_merged_job, [(scene, poses[k], seed * 7919 + k, beams, az) for k in range(n_scans)])
    return scene, poses, scans, [M.astype(np.float32) for M in LIDAR_MOUNTS]


def perturbed_prior(T, seed, t=0.05, r_deg=0.4):
    """the odometry estimate handed to scan-to-submap registration as its guess: the true pose off by a few
    centimetres / tenths of a degree (PointCloudLocalization.cc:181-200 pre-transforms the query with it)"""
    rng = np.random.default_rng(seed)
    d = pose_matrix(rng.uniform(-t, t, 3), np.deg2rad(rng.uniform(-r_deg, r_deg, 3)))
    return (T @ d).astype(np.float32)


def submap_cloud(scene, seed, n_scans=40, beams=64, az=2048):
    """raw material of a rolling submap (SURVEY 8d, C3): the union of n_scans posed scans of `scene` in the world
    frame, float32 (n, 3).  The map poses wander further than the ego-motion of the registered stream so that the
    submap covers the room from several viewpoints."""
    poses = trajectory(seed + 50, n_scans, t_step=1.5, r_step_deg=20.0)
    return world_points(scene, poses, seed + 50, beams, az)


def xyz_blob(xyz):
    """(n, 3) float32 -> the 32-byte point layout of this module (intensity 0)"""
    b = np.zeros((len(xyz), POINT_STEP // 4), dtype=np.float32)
    b[:, :3] = xyz
    b[:, 3] = 1.0
    return b.view(np.uint8).reshape(-1)


def voxel_merge_to(xyz, n_target, voxel_fn, lo=0.005, hi=0.5, rounds=16, seed=0):
    """voxel-merge a point union down to exactly n_target points: leaf by bisection (voxel_fn(blob, leaf) -> (m, 32)
    uint8 filtered blob; the GPU filter in bench.py, the oracle's in the tests) so that slightly more than n_target
    voxels remain, then a seeded random subset of exactly n_target, kept in voxel order.  returns (xyz (n_target, 3), leaf)"""
    blob = xyz_blob(xyz)
    best = None
    for _ in range(rounds):
        mid = 0.5 * (lo + hi)
        out = voxel_fn(blob, mid)
        if out.shape[0] >= n_target:
            lo, best = mid, (out, mid)
        else:
            hi = mid
    if best is None:
        raise ValueError("voxel_merge_to: the union holds fewer than %d voxels at leaf %g" % (n_target, lo))
    out, leaf = best
    pts = np.ascontiguousarray(out).view(np.float32).reshape(-1, POINT_STEP // 4)[:, :3]
    keep = np.sort(np.random.default_rng(seed).choice(len(pts), n_target, replace=False))
    return np.ascontiguousarray(pts[keep]), float(np.float32(leaf))


def subsample_to(xyz, n_target, seed=0):
    """seeded random subset of exactly n_target points, input order kept (the C5 map: the room cannot hold 10 M distinct
    PCL voxels without overflowing VoxelGrid's int32 leaf index, so the dense map is a subsample, not a voxel merge)"""
    if len(xyz) < n_target:
        raise ValueError("subsample_to: the union holds %d points, fewer than %d" % (len(xyz), n_target))
    keep = np.sort(np.random.default_rng(seed).choice(len(xyz), n_target, replace=False))
    return np.ascontiguousarray(xyz[keep])


def c3_workload(seed, n_scans, voxel_fn, n_map_scans=40, n_submap=500_000, beams=64, az=2048, merge="voxel"):
    """BASELINE configs[2] (SURVEY 8d, C3): a stream of n_scans raw scans of one scene, the rolling submap of the same
    scene (voxel-merged union of n_map_scans posed scans, exactly n_submap points, world frame) and the prior each scan
    is registered with.  voxel_fn(blob, leaf) -> filtered (m, 32) uint8 blob (the GPU filter or the oracle's: they
    agree bit for bit, so both give the same submap)."""
    scene, poses, blobs = stream(seed, n_scans, beams, az)
    world = submap_cloud(scene, seed, n_map_scans, beams, az)
    sub, leaf = (subsample_to(world, n_submap), 0.0) if merge == "subsample" else voxel_merge_to(world, n_submap, voxel_fn)
    guesses = [perturbed_prior(poses[i], 100 + i) for i in range(n_scans)]
    return {"scene": scene, "poses": poses, "blobs": blobs, "submap": sub, "submap_leaf": leaf, "guesses": guesses,
            "union_points": int(len(world))}
