"""Seeded synthetic workloads of the shapes BASELINE.json names (SURVEY.md section 8d).

No dataset or checkpoint is reachable offline, so every benchmark / parity input is generated
here; seed = sample id so the CPU oracle and the GPU path consume identical arrays.

KITTI-shaped: N=20480 points, H=160, W=512, intrinsics of KITTI odometry P2 after the
loader's crop/scale (data/kitti_pc_img_pose_loader.py:329-349, kitti/options.py:23-28).
Oxford-shaped: H=384, W=640 (data/oxford_pc_img_pose_loader.py:221-259).
"""
import math

import numpy as np

KITTI = dict(H=160, W=512, K=np.array([[353.5, 0.0, 250.5], [0.0, 353.5, 66.5], [0.0, 0.0, 1.0]]), rmax=80.0)
OXFORD = dict(H=384, W=640, K=np.array([[482.4145, 0.0, 321.894], [0.0, 482.4145, 194.204], [0.0, 0.0, 1.0]]),
              rmax=50.0)
T_LB = (-5.0, -0.1, -10.0)     # registration_lsq.py:340
T_UB = (5.0, 0.1, 10.0)


def ry_matrix(a):
    c, s = math.cos(a), math.sin(a)
    return np.array([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]])


def inside_mask(points, P, K, H, W):
    """GT in-frustum rule (models/multimodal_classifier.py:143-148, registration_lsq.py:67-84)."""
    q = P[:3, :3] @ points.astype(np.float64) + P[:3, 3:4]
    with np.errstate(divide="ignore", invalid="ignore"):
        u = K[0, 0] * q[0] / q[2] + K[0, 2]
        v = K[1, 1] * q[1] / q[2] + K[1, 2]
    return (u >= 0) & (u <= W - 1) & (v >= 0) & (v <= H - 1) & (q[2] > 0.1)


def make_sample(seed, n_points=20480, shape="kitti", flip=0.05):
    """One (cloud, predicted labels, intrinsics, GT pose) sample.  points are float32."""
    cfg = KITTI if shape == "kitti" else OXFORD
    rng = np.random.default_rng(seed)
    r = rng.uniform(2.0, cfg["rmax"], n_points)
    az = rng.uniform(-math.pi, math.pi, n_points)
    y = rng.uniform(-2.5, 1.7, n_points)
    points = np.stack([r * np.sin(az), y, r * np.cos(az)]).astype(np.float32)
    ry = rng.uniform(-math.pi, math.pi)
    t = np.array([rng.uniform(-3, 3), 0.0, rng.uniform(-8, 8)])
    P = np.eye(4)
    P[:3, :3] = ry_matrix(ry)
    P[:3, 3] = t
    gt = inside_mask(points, P, cfg["K"], cfg["H"], cfg["W"]).astype(np.int32)
    flips = rng.uniform(size=n_points) < flip
    pred = np.where(flips, 1 - gt, gt).astype(np.int32)
    return dict(points=points, pred=pred, gt=gt, K=cfg["K"].copy(), P_gt=P, H=cfg["H"], W=cfg["W"],
                ry_gt=ry, t_gt=t)


def make_fine_labels(sample, scale=1 / 32.0, noise=0.3, seed=0):
    """Fine predictions of a make_sample() frame: the fine-label rule of visualize_and_save_data.py:137-139 (cell
    floor(u * scale) + floor(v * scale) * round(W * scale) of the GT projection), with a seeded fraction `noise` of the
    points moved to a uniformly random cell.  Points behind the camera get cell 0.  Returns int32 [N]."""
    P, K = sample["P_gt"], sample["K"]
    q = P[:3, :3] @ sample["points"].astype(np.float64) + P[:3, 3:4]
    with np.errstate(divide="ignore", invalid="ignore"):
        u = K[0, 0] * q[0] / q[2] + K[0, 2]
        v = K[1, 1] * q[1] / q[2] + K[1, 2]
    Wf, Hf = int(round(sample["W"] * scale)), int(round(sample["H"] * scale))
    ok = (q[2] > 0.1) & np.isfinite(u) & np.isfinite(v)
    cell = np.zeros(u.shape, dtype=np.int64)
    cell[ok] = np.floor(u[ok] * scale).astype(np.int64) + np.floor(v[ok] * scale).astype(np.int64) * Wf
    rng = np.random.default_rng(seed + 0xF1E)
    moved = rng.uniform(size=cell.shape) < noise
    cell = np.where(moved, rng.integers(0, Wf * Hf, cell.shape), cell)
    return np.clip(cell, -2**31, 2**31 - 1).astype(np.int32)


def make_inits(seed, init_y_angle, n_inits=60, ry_sigma=10.0 * math.pi / 180.0, t_amp=10.0):
    """The multi-start inits of registration_lsq.py:163-164, materialised:
    ry_i = init_y_angle + N(0, sigma), t_i = (0, 0, U(-amp, amp)).  Returns (ry[I], t[I,3])."""
    rng = np.random.default_rng(seed + 0x5EED)
    ry = init_y_angle + rng.normal(0.0, ry_sigma, n_inits)
    t = np.zeros((n_inits, 3))
    t[:, 2] = rng.uniform(-t_amp, t_amp, n_inits)
    return ry, t


def _ray_boxes(o, d, lo, hi):
    """Nearest positive hit distance of rays o + t d (d [R,3]) with axis-aligned boxes (lo, hi [B,3]); inf = none."""
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / d
        best = np.full(d.shape[0], np.inf)
        for b in range(lo.shape[0]):
            t1 = (lo[b] - o) * inv
            t2 = (hi[b] - o) * inv
            tmin = np.nanmax(np.minimum(t1, t2), axis=1)
            tmax = np.nanmin(np.maximum(t1, t2), axis=1)
            hit = (tmax >= np.maximum(tmin, 0.0)) & (tmin > 0.0)
            best = np.where(hit & (tmin < best), tmin, best)
    return best


def make_icp_frame(seed, shape="oxford", n_rings=32, n_azimuth=640, ground=1.7, max_depth=80.0):
    """One seeded monodepth + ICP frame (the inputs of evaluation/icp/registration_icp.py:196-218), ray-cast from a
    scene of a ground plane (y = `ground`, y points down as in make_sample), a closed ring of 24 buildings 27-37 m from
    the LiDAR and 20 small boxes inside it:

      src  [3, n_rings * n_azimuth] float32  a 360 deg LiDAR pattern (elevations 15 deg up to 10 deg down)
      tgt  [3, H * W] float64  the depth map of the ground-truth camera with an unknown global scale and smooth
           multiplicative noise, back-projected through K^-1 in save_depth_map.py:84-102's order (index y * W + x)

    Returns dict(src, tgt, depth [H,W], K, H, W, P_gt (LiDAR -> camera, Ry and (tx, 0, tz) like make_sample), scale
    (the factor the depth map was multiplied by))."""
    cfg = KITTI if shape == "kitti" else OXFORD
    H, W, K = cfg["H"], cfg["W"], cfg["K"].copy()
    rng = np.random.default_rng(seed + 0x1C9)
    ry = rng.uniform(-math.pi, math.pi)
    t = np.array([rng.uniform(-3, 3), 0.0, rng.uniform(-6, 6)])
    P = np.eye(4)
    P[:3, :3] = ry_matrix(ry)
    P[:3, 3] = t
    cam = -P[:3, :3].T @ t                      # camera centre in the LiDAR frame
    lo, hi = [], []
    for k in range(24):                         # buildings: 10 m squares on a 32 m circle overlap, so the ring is closed
        a = 2 * math.pi * k / 24 + rng.uniform(-0.05, 0.05)
        r = 32.0 + rng.uniform(-2, 2)
        h = rng.uniform(8.0, 15.0)
        c = np.array([r * math.sin(a), 0.0, r * math.cos(a)])
        lo.append([c[0] - 5, ground - h, c[2] - 5])
        hi.append([c[0] + 5, ground + 1.0, c[2] + 5])
    while len(lo) < 44:                         # cars / kiosks, kept clear of the LiDAR and the camera
        half = rng.uniform(0.75, 2.25, 2)
        h = rng.uniform(1.0, 2.5)
        a, r = rng.uniform(-math.pi, math.pi), rng.uniform(5.0, 22.0)
        c = np.array([r * math.sin(a), 0.0, r * math.cos(a)])
        clear = 3.0 + float(np.hypot(*half))
        if np.hypot(c[0], c[2]) < clear or np.hypot(c[0] - cam[0], c[2] - cam[2]) < clear:
            continue
        lo.append([c[0] - half[0], ground - h, c[2] - half[1]])
        hi.append([c[0] + half[0], ground + 1.0, c[2] + half[1]])
    lo, hi = np.array(lo), np.array(hi)

    def cast(o, d):
        tb = _ray_boxes(o, d, lo, hi)
        with np.errstate(divide="ignore", invalid="ignore"):
            tg = np.where(d[:, 1] > 1e-9, (ground - o[1]) / d[:, 1], np.inf)
        return np.minimum(tb, np.where(tg > 0, tg, np.inf))

    el = np.deg2rad(np.linspace(-15.0, 10.0, n_rings))
    az = np.linspace(-math.pi, math.pi, n_azimuth, endpoint=False)
    e, a = np.meshgrid(el, az, indexing="ij")
    d = np.stack([np.cos(e) * np.sin(a), np.sin(e), np.cos(e) * np.cos(a)], -1).reshape(-1, 3)
    rl = cast(np.zeros(3), d)
    rl = np.where(np.isfinite(rl), rl, max_depth)
    src = (d * rl[:, None]).T.astype(np.float32)

    xv, yv = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    pix = np.stack([xv, yv, np.ones_like(xv)], -1).reshape(-1, 3)
    dcam = pix @ np.linalg.inv(K).T                            # z = 1: the hit distance is the depth
    depth = cast(cam, dcam @ P[:3, :3])                        # rows of dcam @ R = R^T dcam
    depth = np.minimum(np.where(np.isfinite(depth), depth, max_depth), max_depth).reshape(H, W)
    scale = rng.uniform(0.5, 2.0)
    ph = rng.uniform(0, 2 * math.pi, 4)
    noise = 1.0 + 0.02 * (np.sin(xv / W * 2 * math.pi + ph[0]) * np.cos(yv / H * math.pi + ph[1])
                          + 0.5 * np.sin(xv / W * 5 * math.pi + ph[2] + yv / H * 3 * math.pi) * math.cos(ph[3]))
    depth = depth * noise * scale
    tgt = np.linalg.inv(K) @ (pix * depth.reshape(-1, 1)).T
    return dict(src=src, tgt=tgt, depth=depth, K=K, H=H, W=W, P_gt=P, scale=scale)


def make_lidar_scan(seed, n_rings=64, n_azimuth=2048, noise=0.01, ground=-1.73, max_range=80.0):
    """One seeded HDL-64-shaped scan in Velodyne axes (x forward, y left, z up): n_rings elevations from +2 to -24.8
    deg times n_azimuth azimuths, ray-cast against a ground plane z = `ground` and 30 boxes (buildings, cars) 4-40 m
    away; rays that hit nothing return at max_range.  Ranges get N(0, noise) errors (noise = 0: ground points lie
    exactly on the plane).  Returns dict(xyz [3, n_rings * n_azimuth] float32, intensity [n] float32 in [0, 1),
    ground [n] bool)."""
    rng = np.random.default_rng(seed + 0x5CA)
    lo, hi = [], []
    for _ in range(30):
        a, r = rng.uniform(-math.pi, math.pi), rng.uniform(4.0, 40.0)
        half = rng.uniform(0.8, 6.0, 2)
        h = rng.uniform(1.2, 12.0)
        c = np.array([r * math.cos(a), r * math.sin(a)])
        if np.hypot(*c) < 2.0 + float(np.hypot(*half)):
            continue
        lo.append([c[0] - half[0], c[1] - half[1], ground - 1.0])
        hi.append([c[0] + half[0], c[1] + half[1], ground + h])
    lo, hi = np.array(lo), np.array(hi)
    el = np.deg2rad(np.linspace(2.0, -24.8, n_rings))
    az = np.linspace(-math.pi, math.pi, n_azimuth, endpoint=False)
    e, a = np.meshgrid(el, az, indexing="ij")
    d = np.stack([np.cos(e) * np.cos(a), np.cos(e) * np.sin(a), np.sin(e)], -1).reshape(-1, 3)
    tb = _ray_boxes(np.zeros(3), d, lo, hi)
    with np.errstate(divide="ignore", invalid="ignore"):
        tg = np.where(d[:, 2] < -1e-9, ground / d[:, 2], np.inf)
    on_ground = tg < tb
    t = np.minimum(np.minimum(tb, tg), max_range)
    on_ground &= t < max_range
    t = t + (rng.normal(0.0, noise, t.shape) if noise > 0 else 0.0)
    xyz = d * t[:, None]
    if noise == 0:
        xyz[on_ground, 2] = ground
    inten = rng.random(t.shape[0], dtype=np.float32)
    return dict(xyz=xyz.T.astype(np.float32), intensity=inten, ground=on_ground)


def _rigid(rng, rot_amp, t_amp):
    a = rng.uniform(-rot_amp, rot_amp, 3)
    c, s = np.cos(a), np.sin(a)
    Rx = np.array([[1, 0, 0], [0, c[0], -s[0]], [0, s[0], c[0]]])
    Ry = np.array([[c[1], 0, s[1]], [0, 1, 0], [-s[1], 0, c[1]]])
    Rz = np.array([[c[2], -s[2], 0], [s[2], c[2], 0], [0, 0, 1]])
    P = np.eye(4)
    P[:3, :3] = Rz @ Ry @ Rx
    P[:3, 3] = rng.uniform(-t_amp, t_amp, 3)
    return P


def make_loader_sample(seed, shape="kitti", n_rings=64, n_azimuth=512):
    """One seeded loader sample for deepi2p_b200.assemble.  kitti: 7 make_lidar_scan frames (the anchor first, then
    3 before and 3 after it, each moved by a small rigid frame_T as search_for_accumulation composes Pc^-1 P_ij Pc),
    unit normals, Pc (camera <- velodyne) and Pji; oxford: one frame in camera axes (x right, y down, z forward), no
    normals, and P_cam_pc.  Returns dict(frames [(xyz [3,n] f32, intensity [n] f32, sn [3,n] f32 or None)], frame_T
    [T,4,4], K [3,3], and Pc / Pji (kitti) or P_cam_pc (oxford))."""
    rng = np.random.default_rng(seed + 0x10AD)
    K = np.array([[358.0, 0.0, 256.0], [0.0, 358.0, 80.0], [0.0, 0.0, 1.0]])
    if shape == "kitti":
        frames, Ts = [], []
        for t in range(7):
            sc = make_lidar_scan(seed * 16 + t, n_rings=n_rings, n_azimuth=n_azimuth)
            nrm = rng.normal(0.0, 0.2, sc["xyz"].shape) + np.array([[0.0], [0.0], [1.0]])
            nrm = (nrm / np.linalg.norm(nrm, axis=0)).astype(np.float32)
            frames.append((sc["xyz"], sc["intensity"], nrm))
            Ts.append(np.eye(4) if t == 0 else _rigid(rng, 0.02, 6.0))
        Pc = np.eye(4)
        Pc[:3, :3] = np.array([[0.0, -1.0, 0.0], [0.0, 0.0, -1.0], [1.0, 0.0, 0.0]]) @ _rigid(rng, 0.01, 0.0)[:3, :3]
        Pc[:3, 3] = [0.06, -0.08, -0.27]
        return dict(frames=frames, frame_T=np.stack(Ts), K=K, Pc=Pc, Pji=_rigid(rng, 0.05, 3.0))
    if shape == "oxford":
        sc = make_lidar_scan(seed * 16, n_rings=n_rings, n_azimuth=n_azimuth)
        x, y, z = sc["xyz"]
        cam = np.stack([-y, -z, x]).astype(np.float32)
        return dict(frames=[(cam, sc["intensity"], None)], frame_T=np.eye(4)[None], K=K,
                    P_cam_pc=_rigid(rng, 0.1, 5.0))
    raise ValueError(f"shape must be 'kitti' or 'oxford' (got {shape!r})")


def write_icp_handoff(data_dir, monodepth_dir, seeds, shape="oxford"):
    """make_icp_frame frames as a hand-off directory (<id>_pc_label.npy / _K.npy / _P.npy, labels = the GT inside
    mask) plus the <monodepth_dir>/<id>_pc.npy depth clouds registration_icp.py:204 reads.  Returns the frames by id."""
    import os
    from . import handoff
    os.makedirs(monodepth_dir, exist_ok=True)
    frames = {}
    for i, s in enumerate(seeds):
        f = make_icp_frame(s, shape)
        name = "%06d_%02d" % (i, 0)
        lab = inside_mask(f["src"], f["P_gt"], f["K"], f["H"], f["W"]).astype(np.int32)
        handoff.save_record(data_dir, name, f["src"], lab, lab, lab, lab, f["K"], f["P_gt"][:3])
        np.save(os.path.join(monodepth_dir, name + "_pc.npy"), f["tgt"])
        frames[name] = f
    return frames


def make_index_max_inputs(seed, B=64, C=64, N=16384, K=64):
    rng = np.random.default_rng(seed)
    data = rng.standard_normal((B, C, N), dtype=np.float32)
    index = rng.integers(0, K, (B, N), dtype=np.int32)
    return data, index


def make_ball_query_inputs(seed, B=64, M=64, N=16384, K=64, cube=20.0):
    """True node->point Euclidean distances in a cube; radius chosen so the median row has ~K hits."""
    rng = np.random.default_rng(seed)
    pts = rng.uniform(0, cube, (B, N, 3)).astype(np.float32)
    nodes = rng.uniform(0, cube, (B, M, 3)).astype(np.float32)
    dist = np.sqrt(((nodes[:, :, None, :] - pts[:, None, :, :]) ** 2).sum(-1, dtype=np.float32)).astype(np.float32)
    kth = np.partition(dist, K - 1, axis=2)[:, :, K - 1]
    radius = float(np.median(kth))
    return dist, radius
