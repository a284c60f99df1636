"""Seeded synthetic workloads of the shapes BASELINE.json names (SURVEY.md section 8d).

No dataset or checkpoint is reachable offline, so every benchmark / parity input is generated
here; seed = sample id so the CPU oracle and the GPU path consume identical arrays.

KITTI-shaped: N=20480 points, H=160, W=512, intrinsics of KITTI odometry P2 after the
loader's crop/scale (data/kitti_pc_img_pose_loader.py:329-349, kitti/options.py:23-28).
Oxford-shaped: H=384, W=640 (data/oxford_pc_img_pose_loader.py:221-259).
"""
import math
import os
import struct
import zlib

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


NUSCENES_CAMERAS = ("CAM_FRONT", "CAM_FRONT_LEFT", "CAM_FRONT_RIGHT", "CAM_BACK", "CAM_BACK_LEFT", "CAM_BACK_RIGHT")
EGO_POINTS = 512


def make_nuscenes_sweep(seed, n_rings=32, n_azimuth=1085):
    """One seeded LIDAR_TOP-shaped sweep as the .pcd.bin records hold it: [n, 5] float32 (x, y, z, intensity, ring),
    a make_lidar_scan of n_rings x n_azimuth rays (intensity 0-255) followed by EGO_POINTS points drawn in and around
    the ego-vehicle box (-0.8 < x < 0.8, -2.7 < y < 2.7)."""
    sc = make_lidar_scan(seed, n_rings=n_rings, n_azimuth=n_azimuth, ground=-1.84)
    rng = np.random.default_rng(seed + 0xE60)
    ego = rng.uniform([-1.0, -3.0, -1.5], [1.0, 3.0, 0.5], (EGO_POINTS, 3)).T
    xyz = np.concatenate([sc["xyz"], ego.astype(np.float32)], 1)
    inten = np.concatenate([sc["intensity"] * 255.0, rng.uniform(0.0, 255.0, EGO_POINTS)])
    ring = np.concatenate([np.repeat(np.arange(n_rings), n_azimuth), np.zeros(EGO_POINTS)])
    return np.stack([xyz[0], xyz[1], xyz[2], inten, ring], 1).astype(np.float32)


def make_nuscenes_sample(seed, n_sweeps=7, n_rings=32, n_azimuth=1085):
    """One seeded nuScenes sample for assemble_batch(**nuscenes_args): n_sweeps make_nuscenes_sweep frames (the anchor
    first with the identity, the others moved by small rigid frame_T as the sweep chain composes them) and P_cam_pc.
    Returns dict(frames [(xyz [3,n] f32, intensity [n] f32, None)], frame_T [T,4,4], P_cam_pc [4,4])."""
    rng = np.random.default_rng(seed + 0x4E5)
    frames, Ts = [], []
    for t in range(n_sweeps):
        r = make_nuscenes_sweep(seed * 16 + t, n_rings, n_azimuth)
        frames.append((np.ascontiguousarray(r[:, :3].T), np.ascontiguousarray(r[:, 3]), None))
        Ts.append(np.eye(4) if t == 0 else _rigid(rng, 0.02, 4.0))
    P = np.eye(4)
    P[:3, :3] = np.array([[0.0, -1.0, 0.0], [0.0, 0.0, -1.0], [1.0, 0.0, 0.0]]) @ _rigid(rng, 0.05, 0.0)[:3, :3]
    P[:3, 3] = rng.uniform(-1.0, 1.0, 3)
    return dict(frames=frames, frame_T=np.stack(Ts), P_cam_pc=P)


def _quaternion(rng, yaw, tilt=0.01):
    """A near-unit (w, x, y, z) list: yaw about z plus small tilts, not renormalised."""
    return [math.cos(yaw / 2), float(rng.normal(0.0, tilt)), float(rng.normal(0.0, tilt)), math.sin(yaw / 2)]


def write_nuscenes_dataroot(root, chains, seed=0, jpeg=None, version="v1.0-mini", n_rings=8, n_azimuth=128,
                            sweeps=True):
    """A seeded devkit-layout dataroot for deepi2p_b200.nuscenes: <root>/<version>/{sample_data, ego_pose,
    calibrated_sensor}.json, <root>/dataset_info.list and, with `sweeps`, one make_nuscenes_sweep .pcd.bin per
    LIDAR_TOP record.  chains: [(length, anchor)] -- one scene per entry, `length` LIDAR_TOP sweeps linked by next /
    prev, the dataset entry at sweep `anchor`.  Each scene has one record per camera whose file holds `jpeg` (bytes)
    when given.  Returns the dataset_info list."""
    import json
    import pickle
    rng = np.random.default_rng(seed + 0x4E5C)
    sd, ego, cal = [], [], []
    cal.append(dict(token="calib-LIDAR_TOP", sensor_token="LIDAR_TOP", translation=[0.943713, 0.0, 1.84023],
                    rotation=_quaternion(rng, -math.pi / 2), camera_intrinsic=[]))
    for k, name in enumerate(NUSCENES_CAMERAS):
        yaw = [0.0, 0.95, -0.95, math.pi, 1.9, -1.9][k]
        cal.append(dict(token=f"calib-{name}", sensor_token=name, translation=[1.7, 0.0 + 0.1 * k, 1.5],
                        rotation=_quaternion(rng, yaw - math.pi / 2),
                        camera_intrinsic=[[1266.4, 0.0, 816.3 + k], [0.0, 1266.4, 491.5], [0.0, 0.0, 1.0]]))
    items = []
    for c, (length, anchor) in enumerate(chains):
        x0 = rng.uniform(300.0, 900.0, 2)
        heading = rng.uniform(-math.pi, math.pi)
        for i in range(length):
            tok = f"lidar-{c}-{i}"
            fn = f"sweeps/LIDAR_TOP/scene{c}_{i:03d}.pcd.bin"
            sd.append(dict(token=tok, filename=fn, ego_pose_token=f"ego-{c}-{i}",
                           calibrated_sensor_token="calib-LIDAR_TOP",
                           next=f"lidar-{c}-{i + 1}" if i + 1 < length else "",
                           prev=f"lidar-{c}-{i - 1}" if i > 0 else ""))
            yaw = heading + 0.01 * i
            ego.append(dict(token=f"ego-{c}-{i}", rotation=_quaternion(rng, yaw),
                            translation=[x0[0] + 0.45 * i * math.cos(heading), x0[1] + 0.45 * i * math.sin(heading),
                                         float(rng.normal(0.0, 0.02))]))
            if sweeps:
                os.makedirs(os.path.join(root, os.path.dirname(fn)), exist_ok=True)
                make_nuscenes_sweep(seed * 4096 + c * 64 + i, n_rings, n_azimuth).tofile(os.path.join(root, fn))
        cams = {}
        for name in NUSCENES_CAMERAS:
            tok = f"cam-{c}-{name}"
            fn = f"samples/{name}/scene{c}.jpg"
            sd.append(dict(token=tok, filename=fn, ego_pose_token=f"ego-{tok}", calibrated_sensor_token=f"calib-{name}",
                           next="", prev=""))
            ego.append(dict(token=f"ego-{tok}", rotation=_quaternion(rng, heading + 0.01 * anchor),
                            translation=[x0[0] + 0.45 * anchor * math.cos(heading) + float(rng.normal(0.0, 0.1)),
                                         x0[1] + 0.45 * anchor * math.sin(heading), 0.0]))
            if jpeg is not None:
                os.makedirs(os.path.join(root, os.path.dirname(fn)), exist_ok=True)
                with open(os.path.join(root, fn), "wb") as f:
                    f.write(jpeg)
            cams[name] = [tok]
        items.append((f"lidar-{c}-{anchor}", cams))
    os.makedirs(os.path.join(root, version), exist_ok=True)
    for name, recs in (("sample_data", sd), ("ego_pose", ego), ("calibrated_sensor", cal)):
        with open(os.path.join(root, version, name + ".json"), "w") as f:
            json.dump(recs, f)
    with open(os.path.join(root, "dataset_info.list"), "wb") as f:
        pickle.dump(items, f)
    return items


NUSCENES_RAW_RATES = (("LIDAR_TOP", "lidar", 20.0),) + tuple((c, "camera", 12.0) for c in NUSCENES_CAMERAS) + (
    ("RADAR_FRONT", "radar", 13.0),)
NUSCENES_NIGHT_TOKEN = "e59a4d0cc6a84ed59f78fb21a45cdcb4"     # the first of make_datasets.py's test_night_scene_tokens
NUSCENES_TIE_XY = (1000.0, 500.0)          # the tie scene's LIDAR_TOP position; its ties lie 10 m from it


def _track(rng, times):
    """Along-track distance at `times` for piecewise-constant speeds: stops (0 m/s, one segment in five), driving
    (1-12 m/s) and reversing (-3 to -1 m/s), each 0.5-3 s long."""
    edges, speeds = [0.0], []
    while edges[-1] <= times[-1]:
        edges.append(edges[-1] + float(rng.uniform(0.5, 3.0)))
        u = rng.uniform()
        speeds.append(0.0 if u < 0.2 else -float(rng.uniform(1.0, 3.0)) if u < 0.3 else float(rng.uniform(1.0, 12.0)))
    edges, speeds = np.array(edges), np.array(speeds)
    at_edge = np.concatenate([[0.0], np.cumsum(np.diff(edges) * speeds)])
    k = np.searchsorted(edges, times, side="right") - 1
    return at_edge[k] + speeds[k] * (times - edges[k])


def write_nuscenes_raw(root, n_scenes=8, seed=0, version="v1.0-mini", seconds=(3.0, 8.0), special=True,
                       all_night=False, jpeg=None, n_rings=4, n_azimuth=64, max_translation=10.0):
    """A seeded raw devkit-layout root: <root>/<version>/{scene, sample, sample_data, sensor, calibrated_sensor,
    ego_pose}.json.  LIDAR_TOP at 20 Hz, six cameras at 12 Hz and RADAR_FRONT at 13 Hz, each record with its own ego
    pose; key frames at 2 Hz, the record of each channel nearest a sample's time.  Scenes last `seconds` (a range) and
    drive at global positions 300-2000 m from the origin with stops and reversals.  With `special`, the first five
    scenes are instead: a tie scene (identity rotations; camera translations whose t_lc is exactly (max_translation,
    0, 0), (-max_translation, 0, 0) or (0, max_translation, 0), or one float32 ulp either side of it), a one-sweep
    scene, a night scene, a day scene with a hard-coded night token and a scene whose camera chains end at the first
    neighbour.  all_night marks every scene's description as night.  With jpeg (bytes), every LIDAR_TOP record gets a
    make_nuscenes_sweep file and every camera record the JPEG, so the root feeds nuscenes.nuscenes_batch.  Returns
    dict(tie_scene, tie_lanes: the (camera, chain position) of each planted exact tie)."""
    import json
    rng = np.random.default_rng(seed + 0x4E5D)
    tabs = {k: [] for k in ("scene", "sample", "sample_data", "sensor", "calibrated_sensor", "ego_pose")}
    for k, (ch, mod, _) in enumerate(NUSCENES_RAW_RATES):
        tabs["sensor"].append(dict(token=f"sensor-{ch}", channel=ch, modality=mod))
        cam = mod == "camera"
        yaw = [0.0, 0.95, -0.95, math.pi, 1.9, -1.9][k - 1] if cam else 0.0
        tabs["calibrated_sensor"].append(dict(
            token=f"calib-{ch}", sensor_token=f"sensor-{ch}", translation=[1.7 if cam else 0.94, 0.1 * k, 1.5],
            rotation=_quaternion(rng, yaw - math.pi / 2 if cam else -math.pi / 2),
            camera_intrinsic=[[1266.4, 0.0, 816.3 + k], [0.0, 1266.4, 491.5], [0.0, 0.0, 1.0]] if cam else []))
    f32 = lambda v: float(np.float32(v))
    ulp = lambda v, d: float(np.nextafter(np.float32(v), np.float32(d)))
    m = float(max_translation)
    Lx, Ly = NUSCENES_TIE_XY
    # tie scene, camera chain positions 2.. : (camera, position) -> (x, y) relative offsets from the lidar
    ties = {("CAM_FRONT", 2): (Lx + m, Ly), ("CAM_FRONT_RIGHT", 2): (Lx - m, Ly), ("CAM_BACK", 2): (Lx, Ly + m),
            ("CAM_BACK_LEFT", 3): (Lx + m, Ly)}
    near = {("CAM_FRONT_LEFT", 2): (ulp(Lx + m, 0), Ly), ("CAM_FRONT_LEFT", 3): (ulp(Lx + m, 4096), Ly),
            ("CAM_BACK_LEFT", 2): (Lx + m - 1.0, Ly), ("CAM_BACK_RIGHT", 2): (ulp(Lx + m, 4096), Ly)}
    info = dict(tie_scene=None, tie_lanes=sorted(ties))
    for c in range(n_scenes):
        kind = ("tie", "one", "night", "token", "short")[c] if special and c < 5 else "drive"
        T = dict(tie=1.2, one=0.04, short=0.1).get(kind, float(rng.uniform(*seconds)))
        token = NUSCENES_NIGHT_TOKEN if kind == "token" else f"scene-{seed}-{c:04d}"
        night = all_night or kind == "night"
        desc = ["Night, rain, parked cars", "night driving"][c % 2] if night else ["Day, busy street", "Turn left"][c % 2]
        if kind == "tie":
            info["tie_scene"] = token
        ns = max(1, int(math.ceil(T / 0.5 - 1e-9)))
        s_tok = [f"sample-{seed}-{c}-{j}" for j in range(ns)]
        for j in range(ns):
            tabs["sample"].append(dict(token=s_tok[j], timestamp=int(1.5e15 + c * 1e8 + j * 5e5), scene_token=token,
                                       prev=s_tok[j - 1] if j else "", next=s_tok[j + 1] if j + 1 < ns else ""))
        tabs["scene"].append(dict(token=token, log_token=f"log-{c}", nbr_samples=ns, first_sample_token=s_tok[0],
                                  last_sample_token=s_tok[-1], name=f"scene-{c:04d}", description=desc))
        r0 = rng.uniform(300.0, 2000.0)
        phi, heading = rng.uniform(-math.pi, math.pi, 2)
        x0, y0 = r0 * math.cos(phi), r0 * math.sin(phi)
        grid = np.arange(0.0, T + 1.0, 0.01)
        s_grid = _track(rng, grid)
        for k, (ch, mod, hz) in enumerate(NUSCENES_RAW_RATES):
            off = 0.0 if k == 0 else 0.007 * k
            times = off + np.arange(int(math.floor((T - off) * hz)) + 1) / hz if T > off else np.array([off])
            n = len(times)
            s = np.interp(times, grid, s_grid)
            wob = 0.5 * np.sin(0.1 * s)
            xs = x0 + s * math.cos(heading) - wob * math.sin(heading)
            ys = y0 + s * math.sin(heading) + wob * math.cos(heading)
            zs = 0.01 * np.sin(times)
            keys = {int(np.argmin(np.abs(times - 0.5 * j))): j for j in range(ns)}
            near_s = np.minimum(np.rint(times / 0.5).astype(int), ns - 1)
            toks = [f"sd-{seed}-{c}-{ch}-{i}" for i in range(n)]
            for i in range(n):
                key = i in keys
                if ch == "LIDAR_TOP":
                    fn = f"{'samples' if key else 'sweeps'}/{ch}/s{c}_{i:04d}.pcd.bin"
                else:
                    fn = f"{'samples' if key else 'sweeps'}/{ch}/s{c}_{i:04d}.{'jpg' if mod == 'camera' else 'pcd'}"
                if kind == "tie":
                    rot = [1.0, 0.0, 0.0, 0.0]
                    x, y = (Lx, Ly) if ch == "LIDAR_TOP" or mod != "camera" else ties.get(
                        (ch, i), near.get((ch, i), (Lx + 0.25 * i, Ly + 0.5)))
                    t = [f32(x), f32(y), 1.5]
                else:
                    rot = _quaternion(rng, heading + 0.001 * float(s[i]), tilt=0.005)
                    t = [float(xs[i]), float(ys[i]), float(zs[i])]
                ego_tok = f"ego-{seed}-{c}-{ch}-{i}"
                tabs["ego_pose"].append(dict(token=ego_tok, timestamp=int(1.5e15 + c * 1e8 + times[i] * 1e6),
                                             rotation=rot, translation=t))
                tabs["sample_data"].append(dict(
                    token=toks[i], sample_token=s_tok[keys[i]] if key else s_tok[near_s[i]], ego_pose_token=ego_tok,
                    calibrated_sensor_token=f"calib-{ch}", timestamp=int(1.5e15 + c * 1e8 + times[i] * 1e6),
                    fileformat=fn.rsplit(".", 1)[1], is_key_frame=key, height=900 if mod == "camera" else 0,
                    width=1600 if mod == "camera" else 0, filename=fn,
                    prev=toks[i - 1] if i else "", next=toks[i + 1] if i + 1 < n else ""))
                if jpeg is not None and ch == "LIDAR_TOP":
                    os.makedirs(os.path.join(root, os.path.dirname(fn)), exist_ok=True)
                    make_nuscenes_sweep(seed * 65536 + c * 1024 + i, n_rings, n_azimuth).tofile(os.path.join(root, fn))
                elif jpeg is not None and mod == "camera":
                    os.makedirs(os.path.join(root, os.path.dirname(fn)), exist_ok=True)
                    with open(os.path.join(root, fn), "wb") as f:
                        f.write(jpeg)
    os.makedirs(os.path.join(root, version), exist_ok=True)
    for name, recs in tabs.items():
        with open(os.path.join(root, version, name + ".json"), "w") as f:
            json.dump(recs, f)
    return info


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


def seeded_state_dict(model, seed):
    """Seeded weights for a network's state_dict, the same on every machine (numpy draws in sorted key order):
    convolution and linear weights N(0, 1 / fan_in), other weights (the norms') 1 + N(0, 0.1^2), biases and running
    means N(0, 0.1^2), running variances U(0.5, 1.5); num_batches_tracked is kept.  Returns a dict of CPU tensors
    with the dtypes of `model.state_dict()`."""
    import torch
    rng = np.random.default_rng(seed)
    out = {}
    ref = model.state_dict()
    for k in sorted(ref):
        v = ref[k]
        if k.endswith("num_batches_tracked"):
            out[k] = v.detach().cpu().clone()
            continue
        shape = tuple(v.shape)
        if k.endswith("running_var"):
            a = rng.uniform(0.5, 1.5, shape)
        elif k.endswith(".weight") and len(shape) > 1:
            a = rng.standard_normal(shape) / math.sqrt(int(np.prod(shape[1:])))
        elif k.endswith(".weight"):
            a = 1.0 + 0.1 * rng.standard_normal(shape)
        else:
            a = 0.1 * rng.standard_normal(shape)
        out[k] = torch.from_numpy(np.asarray(a, dtype=np.float64)).to(v.dtype)
    return out


def make_network_inputs(seed, B=2, N=2048, Ma=128, Mb=128, H=64, W=128, L=8):
    """Seeded classifier-network inputs (numpy float32): pc, node_a, node_b uniform in a 40 x 6 x 40 m box (drawn
    independently, so no node coincides with a point), intensity U(0, 1), unit normals sn, img U(0, 1) [B,3,H,W], and
    the weights of a linear test loss lw_coarse [B,2,N], lw_fine [B,L,N] ~ N(0, 1)."""
    rng = np.random.default_rng(seed)

    def cloud(n):
        return np.stack([rng.uniform(-20, 20, (B, n)), rng.uniform(-3, 3, (B, n)),
                         rng.uniform(-20, 20, (B, n))], 1).astype(np.float32)
    sn = rng.standard_normal((B, 3, N))
    sn = (sn / np.linalg.norm(sn, axis=1, keepdims=True)).astype(np.float32)
    pc = cloud(N)
    intensity = rng.uniform(0, 1, (B, 1, N)).astype(np.float32)
    node_a, node_b = cloud(Ma), cloud(Mb)
    img = rng.uniform(0, 1, (B, 3, H, W)).astype(np.float32)
    rng = np.random.default_rng(seed + 1)
    lw_coarse = rng.standard_normal((B, 2, N)).astype(np.float32)
    lw_fine = rng.standard_normal((B, L, N)).astype(np.float32)
    return dict(pc=pc, intensity=intensity, sn=sn, node_a=node_a, node_b=node_b, img=img, lw_coarse=lw_coarse,
                lw_fine=lw_fine)


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


def _link_or_copy(src, dst):
    try:
        os.link(src, dst)
    except OSError:
        import shutil
        shutil.copyfile(src, dst)


def _kitti_record(seed, n_rings, n_azimuth):
    """A [7, n] float32 KITTI scan record (xyz, intensity, unit normals) of a make_lidar_scan with a seeded fraction of
    the rays dropped, so record lengths differ."""
    sc = make_lidar_scan(seed, n_rings=n_rings, n_azimuth=n_azimuth)
    rng = np.random.default_rng(seed + 0x7EC)
    keep = rng.random(sc["xyz"].shape[1]) < rng.uniform(0.6, 0.95)
    nrm = rng.normal(0.0, 0.2, sc["xyz"].shape) + np.array([[0.0], [0.0], [1.0]])
    nrm /= np.linalg.norm(nrm, axis=0)
    return np.concatenate([sc["xyz"], sc["intensity"][None], nrm], 0)[:, keep].astype(np.float32)


def write_kitti_root(root, seqs=(0, 9, 10), n_frames=90, seed=0, n_rings=8, n_azimuth=256, image_hw=(376, 1241),
                     n_images=4, images="npy"):
    """A seeded KITTI odometry root in the loader's layout for deepi2p_b200.kitti: calib/<seq>/calib.txt (P0-P3 and
    Tr as KITTI writes them), poses/<seq>/<frame>.npz ['pose'] along a gently turning drive of about 1 m per frame,
    data_odometry_velodyne_NWU/sequences/<seq>/voxel0.1-SNr0.6/<frame>.npy records ([7, n], n differing per frame) and
    data_odometry_color_npy/sequences/<seq>/image_{2,3}/<frame>.npy images (n_images distinct uint8 frames of
    image_hw, linked by frame number).  images="png" writes the same pixels in the official layout instead,
    data_odometry_color/sequences/<seq>/image_{2,3}/<frame>.png (encode_png, the rows cycling through the five
    filters).  Returns {seq: n_frames}."""
    if images not in ("npy", "png"):
        raise ValueError(f"images must be 'npy' or 'png' (got {images!r})")
    rng = np.random.default_rng(seed + 0x4B17)
    os.makedirs(root, exist_ok=True)
    for seq in seqs:
        s = "%02d" % seq
        os.makedirs(os.path.join(root, "calib", s), exist_ok=True)
        fx, cx, cy = 718.856 + seq, 607.1928, 185.2157
        lines = []
        for k, tx in enumerate((0.0, -0.537, 0.06, -0.47)):
            tz = (0.0, 0.0, 2.7e-3, 3.4e-3)[k]
            ty = (0.0, 0.0, -1.2e-5, 2.0e-5)[k]
            m = [fx, 0.0, cx, fx * tx + cx * tz, 0.0, fx, cy, fx * ty + cy * tz, 0.0, 0.0, 1.0, tz]
            lines.append(f"P{k}: " + " ".join("%.12e" % v for v in m))
        R = np.array([[0.0, -1.0, 0.0], [0.0, 0.0, -1.0], [1.0, 0.0, 0.0]]) @ _rigid(rng, 0.01, 0.0)[:3, :3]
        Tr = np.concatenate([R, np.array([[-4.07e-3], [-7.63e-2], [-2.72e-1]])], 1)
        lines.append("Tr: " + " ".join("%.12e" % v for v in Tr.reshape(-1)))
        with open(os.path.join(root, "calib", s, "calib.txt"), "w") as f:
            f.write("\n".join(lines) + "\n")
        pdir = os.path.join(root, "poses", s)
        rdir = os.path.join(root, "data_odometry_velodyne_NWU", "sequences", s, "voxel0.1-SNr0.6")
        for d in (pdir, rdir):
            os.makedirs(d, exist_ok=True)
        yaw, pos = rng.uniform(-math.pi, math.pi), np.zeros(3)
        for i in range(n_frames):
            yaw += rng.normal(0.0, 0.01)
            pos = pos + np.array([math.sin(yaw), 0.0, math.cos(yaw)]) * rng.uniform(0.8, 1.2)
            P = np.eye(4)
            P[:3, :3] = ry_matrix(yaw) @ _rigid(rng, 0.002, 0.0)[:3, :3]
            P[:3, 3] = pos + rng.normal(0.0, 0.01, 3)
            np.savez(os.path.join(pdir, "%06d.npz" % i), pose=P)
            np.save(os.path.join(rdir, "%06d.npy" % i), _kitti_record(seed * 65536 + seq * 1024 + i, n_rings,
                                                                      n_azimuth))
        for cam in ("image_2", "image_3"):
            folder = "data_odometry_color_npy" if images == "npy" else "data_odometry_color"
            idir = os.path.join(root, folder, "sequences", s, cam)
            os.makedirs(idir, exist_ok=True)
            srcs = []
            for k in range(n_images):
                h, w = image_hw
                yy, xx = np.mgrid[0:h, 0:w]
                img = np.stack([(xx * (3 + k) + yy) % 256, (yy * (2 + k)) % 256, (xx + 7 * yy * k) % 256], -1)
                img = (img + rng.integers(0, 24, img.shape)).clip(0, 255).astype(np.uint8)
                srcs.append(os.path.join(idir, "%06d.%s" % (k, images)))
                if images == "npy":
                    np.save(srcs[-1], img)
                else:
                    with open(srcs[-1], "wb") as f:
                        f.write(encode_png(img, filters=np.arange(h) % 5))
            for i in range(n_images, n_frames):
                _link_or_copy(srcs[i % n_images], os.path.join(idir, "%06d.%s" % (i, images)))
    return {seq: n_frames for seq in seqs}


def write_kitti_velodyne_root(root, velodyne_root, seq, scans, sizes, K=(718.856, 718.856, 607.1928, 185.2157),
                              images="npy"):
    """A KITTI root for the camera-frame build (deepi2p_b200.kitti_depth): velodyne_root/sequences/<seq>/velodyne/
    <frame>.bin from `scans` ([4, n] float32 each), root/calib/<seq>/calib.txt and the frames' images.  The calibration
    has the intrinsics K = (fx, fy, cx, cy) for every camera; P0 and P2 have no translation (so P2 = I and
    Pc = Tr exactly), P1 and P3 KITTI's baselines; Tr is the axis permutation x_cam = -y, y_cam = -z, z_cam = x.
    sizes: per frame (H, W), or ((H2, W2), (H3, W3)) per camera.  images "npy" writes zero uint8 [H, W, 3] frames to
    data_odometry_color_npy, "png" grey PNGs to the official data_odometry_color layout."""
    if images not in ("npy", "png"):
        raise ValueError(f"images must be 'npy' or 'png' (got {images!r})")
    s = "%02d" % seq
    fx, fy, cx, cy = K
    lines = []
    for k, tx in enumerate((0.0, -0.537, 0.0, -0.47)):
        tz = (0.0, 0.0, 0.0, 3.4e-3)[k]
        ty = (0.0, 0.0, 0.0, 2.0e-5)[k]
        m = [fx, 0.0, cx, fx * tx + cx * tz, 0.0, fy, cy, fy * ty + cy * tz, 0.0, 0.0, 1.0, tz]
        lines.append(f"P{k}: " + " ".join("%.12e" % v for v in m))
    lines.append("Tr: " + " ".join("%.12e" % v for v in (0, -1, 0, 0, 0, 0, -1, 0, 1, 0, 0, 0)))
    os.makedirs(os.path.join(root, "calib", s), exist_ok=True)
    with open(os.path.join(root, "calib", s, "calib.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")
    vdir = os.path.join(velodyne_root, "sequences", s, "velodyne")
    os.makedirs(vdir, exist_ok=True)
    for i, scan in enumerate(scans):
        np.ascontiguousarray(np.asarray(scan, dtype="<f4").T).tofile(os.path.join(vdir, "%06d.bin" % i))
    folder = "data_odometry_color_npy" if images == "npy" else "data_odometry_color"
    for c, cam in enumerate(("image_2", "image_3")):
        idir = os.path.join(root, folder, "sequences", s, cam)
        os.makedirs(idir, exist_ok=True)
        for i, hw in enumerate(sizes):
            h, w = hw[c] if isinstance(hw[0], (tuple, list)) else hw
            if images == "npy":
                np.save(os.path.join(idir, "%06d.npy" % i), np.zeros((h, w, 3), dtype=np.uint8))
            else:
                with open(os.path.join(idir, "%06d.png" % i), "wb") as f:
                    f.write(encode_png(np.zeros((h, w), dtype=np.uint8)))
    return root


def write_oxford_root(root, train=("2014-05-19-13-20-57", "2014-06-26-08-53-56"), val=("2014-07-14-14-49-50",),
                      n_clouds=24, cams_per_cloud=3, seed=0, n_rings=8, n_azimuth=256, image_hw=(960, 1280),
                      n_images=3, quality=90):
    """A seeded Oxford root in the loader's layout for deepi2p_b200.oxford: train.txt / val.txt, and per traversal
    pc_timestamps.npy / camera_timestamps.npy (int64 microseconds, cams_per_cloud camera frames per cloud),
    pc_poses.npy / camera_poses.npy ([n,4,4] float64 along a drive, 2 m between clouds, in the frame the loader
    conjugates by P_convert), lms_front/<ts>.npy records ([4, n] in camera axes, n differing per cloud) and
    stereo/centre/<ts>.jpg frames (n_images distinct Pillow JPEGs of image_hw, linked by timestamp).  Returns
    {traversal: n_clouds}."""
    from PIL import Image
    rng = np.random.default_rng(seed + 0x0CF)
    os.makedirs(root, exist_ok=True)
    for name, trs in (("train.txt", train), ("val.txt", val)):
        with open(os.path.join(root, name), "w") as f:
            f.write("".join(t + "\n" for t in trs))
    jpegs = []
    for k in range(n_images):
        h, w = image_hw
        yy, xx = np.mgrid[0:h, 0:w]
        img = np.stack([(xx // (2 + k) + yy // 3) % 256, (yy // (1 + k)) % 256, (xx // 5 + 11 * k) % 256], -1)
        img = (img + rng.integers(0, 16, img.shape)).clip(0, 255).astype(np.uint8)
        jpegs.append(img)

    def pose(yaw, p):
        P = np.eye(4)
        c, s = math.cos(yaw), math.sin(yaw)
        P[:3, :3] = np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]]) @ _rigid(rng, 0.003, 0.0)[:3, :3]
        P[:3, 3] = p
        return P

    for t_i, tr in enumerate(tuple(train) + tuple(val)):
        d = os.path.join(root, tr)
        for sub in ("lms_front", os.path.join("stereo", "centre")):
            os.makedirs(os.path.join(d, sub), exist_ok=True)
        t0 = 1400000000000000 + t_i * 10**9
        yaw, pos = rng.uniform(-math.pi, math.pi), np.array([rng.uniform(-500, 500), rng.uniform(-500, 500), 0.0])
        pc_ts, pc_P, cam_ts, cam_P = [], [], [], []
        for i in range(n_clouds):
            ts = t0 + i * 250000 + int(rng.integers(0, 1000))
            for c in range(cams_per_cloud):
                cts = ts - 100000 + c * (250000 // cams_per_cloud) + int(rng.integers(0, 500))
                cyaw = yaw + rng.normal(0.0, 0.01)
                cp = pos + np.array([math.cos(yaw), math.sin(yaw), 0.0]) * (c * 2.0 / cams_per_cloud - 0.8)
                cam_ts.append(cts)
                cam_P.append(pose(cyaw, cp))
            pc_ts.append(ts)
            pc_P.append(pose(yaw, pos))
            sc = make_lidar_scan(seed * 65536 + t_i * 1024 + i, n_rings=n_rings, n_azimuth=n_azimuth)
            keep = rng.random(sc["xyz"].shape[1]) < rng.uniform(0.6, 0.95)
            x, y, z = sc["xyz"]
            rec = np.stack([-y, -z, x, sc["intensity"]])[:, keep].astype(np.float32)
            np.save(os.path.join(d, "lms_front", "%d.npy" % ts), rec)
            yaw += rng.normal(0.0, 0.02)
            pos = pos + np.array([math.cos(yaw), math.sin(yaw), 0.0]) * 2.0
        order = np.argsort(cam_ts, kind="stable")
        cam_ts = [cam_ts[k] for k in order]
        cam_P = [cam_P[k] for k in order]
        np.save(os.path.join(d, "pc_timestamps.npy"), np.array(pc_ts, dtype=np.int64))
        np.save(os.path.join(d, "pc_poses.npy"), np.stack(pc_P))
        np.save(os.path.join(d, "camera_timestamps.npy"), np.array(cam_ts, dtype=np.int64))
        np.save(os.path.join(d, "camera_poses.npy"), np.stack(cam_P))
        srcs = []
        for k, cts in enumerate(cam_ts):
            p = os.path.join(d, "stereo", "centre", "%d.jpg" % cts)
            if k < n_images:
                Image.fromarray(jpegs[k]).save(p, quality=quality)
                srcs.append(p)
            else:
                _link_or_copy(srcs[k % n_images], p)
    return {tr: n_clouds for tr in tuple(train) + tuple(val)}


OXFORD_CAMERA_MODEL = ("964.828979 964.828979 643.788025 484.407990\n"
                       "0 0 1 0\n1 0 0 0\n0 1 0 0\n0 0 0 1\n")
OXFORD_EXTRINSICS = {"lms_front": "1.7042 -0.021 0.1052 -0.0017 0.0152 -0.0001\n",
                     "stereo": "0 0 0 0 0 0\n"}


def write_oxford_sdk(sdk):
    """The SDK text files the Oxford build reads: models/stereo_narrow_left.txt and extrinsics/{lms_front,stereo}.txt
    (the loader's K_CENTRE, a camera-from-image permutation and plausible mounting offsets)."""
    os.makedirs(os.path.join(sdk, "models"), exist_ok=True)
    os.makedirs(os.path.join(sdk, "extrinsics"), exist_ok=True)
    with open(os.path.join(sdk, "models", "stereo_narrow_left.txt"), "w") as f:
        f.write(OXFORD_CAMERA_MODEL)
    for name, line in OXFORD_EXTRINSICS.items():
        with open(os.path.join(sdk, "extrinsics", name + ".txt"), "w") as f:
            f.write(line)


def write_oxford_raw(raw, lms, sdk, traversals=("2014-05-19-13-20-57",), night=("2014-12-10-18-10-50",), seconds=30.0,
                     speed=5.0, stops=((8.0, 9.5), (14.0, 17.0)), curve=(6.0, 11.0), yaw_rate=0.15, zero_reflectance_after=None,
                     n_returns=60, missing_scans=0.03, missing_images=0.05, vo_on_cameras=False, seed=0,
                     image_shape=None):
    """Seeded raw RobotCar traversals in the layout build_dataset.py reads: <raw>/<t>/vo/vo.csv (16 Hz rows whose
    chain abs_k = abs_{k-1} se3(row k) is the drive: `speed` m/s, standing still during each of `stops` (seconds from
    the start), turning at yaw_rate rad/s during `curve`), <raw>/<t>/stereo.timestamps (16 Hz; with vo_on_cameras the
    VO rows are sourced at the camera frames and end on the last one, as in a RobotCar download, otherwise they are
    offset from them and run 120 ms past the last), empty placeholder
    <raw>/<t>/stereo/centre/<ts>.png files (a fraction missing_images absent), <raw>/<t>/tags.csv, and
    <lms>/<t>/lms_front.timestamps with 50 Hz <lms>/<t>/lms_front/<ts>.bin scans of n_returns float64 (x, y,
    reflectance) triples (a fraction missing_scans absent; some x exactly 0.1; reflectance zero from
    zero_reflectance_after seconds on).  night names traversals tagged night.  Also writes the SDK files into sdk.
    With image_shape=(h, w) the PNGs are seeded 8-bit GBRG Bayer mosaics of that size (oxford_mosaic) and the SDK gets
    a seeded radial models/stereo_narrow_left_distortion_lut.bin (oxford_distortion_lut); the other files are the same
    as without.  Returns {traversal: dict(vo=..., lms=..., cameras=...)} of timestamp lists."""
    write_oxford_sdk(sdk)
    if image_shape is not None:
        h, w = (int(v) for v in image_shape)
        lut = oxford_distortion_lut(h, w, seed)
        np.concatenate([lut[:, 0], lut[:, 1]]).tofile(os.path.join(sdk, "models", "stereo_narrow_left_distortion_lut.bin"))
    out = {}
    for t_i, t in enumerate(tuple(traversals) + tuple(night)):
        rng = np.random.default_rng(seed * 1000 + t_i + 0x0B5)
        t0 = 1400000000000000 + t_i * 10**10
        end = t0 + int(seconds * 1e6)
        cams = list(range(t0 + 30002, end, 62500))
        vo_ts = list(cams) if vo_on_cameras else list(range(t0 + 1, end + 120001, 60000))
        rows = [[0.0] * 6]
        for a, b in zip(vo_ts[:-1], vo_ts[1:]):
            tm = (b - t0) / 1e6
            dt = (b - a) / 1e6
            moving = not any(a_ <= tm <= b_ for a_, b_ in stops)
            v = speed * dt if moving else 0.0
            w = yaw_rate * dt if (moving and curve[0] <= tm <= curve[1]) else 0.0
            n = rng.normal(0.0, 1e-4, 4) if moving else np.zeros(4)
            rows.append([v, n[0], n[1], n[2], n[3], w])
        d = os.path.join(raw, t)
        os.makedirs(os.path.join(d, "vo"), exist_ok=True)
        os.makedirs(os.path.join(d, "stereo", "centre"), exist_ok=True)
        with open(os.path.join(d, "vo", "vo.csv"), "w") as f:
            f.write("source_timestamp,destination_timestamp,x,y,z,roll,pitch,yaw\n")
            for k, (ts, r) in enumerate(zip(vo_ts, rows)):
                f.write(",".join([str(ts), str(vo_ts[max(k - 1, 0)])] + [repr(float(x)) for x in r]) + "\n")
        with open(os.path.join(d, "stereo.timestamps"), "w") as f:
            f.write("".join("%d 1\n" % c for c in cams))
        for c in cams:
            if rng.random() >= missing_images:
                path = os.path.join(d, "stereo", "centre", "%d.png" % c)
                if image_shape is None:
                    open(path, "wb").close()
                else:
                    with open(path, "wb") as f:
                        f.write(encode_png(oxford_mosaic(image_shape, c)))
        with open(os.path.join(d, "tags.csv"), "w") as f:
            f.write("night,rain\n" if t in night else "overcast,roadworks\n")
        ld = os.path.join(lms, t, "lms_front")
        os.makedirs(ld, exist_ok=True)
        lts = list(range(t0 + 10004, end, 20000))
        with open(os.path.join(lms, t, "lms_front.timestamps"), "w") as f:
            f.write("".join("%d 1\n" % x for x in lts))
        for x in lts:
            if rng.random() < missing_scans:
                continue
            s = np.empty((n_returns, 3))
            s[:, 0] = rng.uniform(-3.0, 1.0, n_returns)
            s[rng.random(n_returns) < 0.05, 0] = 0.1
            s[:, 1] = rng.uniform(-25.0, 25.0, n_returns)
            s[:, 2] = rng.uniform(0.0, 1500.0, n_returns)
            if zero_reflectance_after is not None and x - t0 >= zero_reflectance_after * 1e6:
                s[:, 2] = 0.0
            s.astype(np.float64).tofile(os.path.join(ld, "%d.bin" % x))
        out[t] = dict(vo=vo_ts, lms=lts, cameras=cams)
    return out


def oxford_mosaic(shape, seed):
    """A seeded 8-bit Bayer mosaic of shape (h, w): smooth gradients and a disc under noise, with saturated and black
    specks, so that demosaicing, the borders and the JPEG encoder's 0xFF bytes all get exercised."""
    h, w = (int(v) for v in shape)
    rng = np.random.default_rng(int(seed) & 0xFFFFFFFF)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    a, b, c = rng.uniform(0.5, 3.0, 3)
    img = 128 + 60 * np.sin(a * xx / w * 6.28 + b) * np.cos(c * yy / h * 6.28)
    cy, cx, r = rng.uniform(0, h), rng.uniform(0, w), rng.uniform(0.1, 0.4) * min(h, w)
    img += np.where((yy - cy) ** 2 + (xx - cx) ** 2 < r * r, 70.0, 0.0)
    img += rng.normal(0.0, 12.0, (h, w))
    img[rng.random((h, w)) < 0.01] = 255
    img[rng.random((h, w)) < 0.01] = 0
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def oxford_distortion_lut(h, w, seed=0):
    """A seeded radial undistortion LUT in the SDK's layout: float64 [h w, 2] of (x, y) source coordinates, (x - cx)
    scaled by 1 + k r^2 about a centre near the middle; the corners map slightly outside the image."""
    rng = np.random.default_rng(int(seed) + 0x1C7)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    cx, cy = (w - 1) / 2 + rng.uniform(-2, 2), (h - 1) / 2 + rng.uniform(-2, 2)
    k = rng.uniform(0.05, 0.15) / ((w / 2) ** 2 + (h / 2) ** 2)
    r2 = (xx - cx) ** 2 + (yy - cy) ** 2
    return np.stack([(cx + (xx - cx) * (1 + k * r2)).ravel(), (cy + (yy - cy) * (1 + k * r2)).ravel()], 1)


def png_chunk(ctype, data, crc=None):
    """One PNG chunk: length, type, data and CRC-32 (the correct one unless `crc` is given)."""
    c = zlib.crc32(ctype + data) if crc is None else crc
    return struct.pack(">I", len(data)) + ctype + data + struct.pack(">I", c & 0xFFFFFFFF)


def png_filter(img, filters):
    """The filtered scanlines of an HWC uint8 RGB image (or an HW grey one): each row prefixed by its filter type
    (filters: one int for every row, or one per row) and filtered with 3 (grey: 1) bytes per pixel, mod 256."""
    h, w = img.shape[:2]
    bpp = 1 if img.ndim == 2 else 3
    x = img.reshape(h, bpp * w).astype(np.int64)
    up = np.vstack([np.zeros((1, bpp * w), np.int64), x[:-1]])
    left = np.hstack([np.zeros((h, bpp), np.int64), x[:, :-bpp]])
    ul = np.hstack([np.zeros((h, bpp), np.int64), up[:, :-bpp]])
    p = left + up - ul
    pa, pb, pc = np.abs(p - left), np.abs(p - up), np.abs(p - ul)
    paeth = np.where((pa <= pb) & (pa <= pc), left, np.where(pb <= pc, up, ul))
    preds = [np.zeros_like(x), left, up, (left + up) >> 1, paeth]
    f = np.broadcast_to(np.asarray(filters, np.int64), (h,))
    out = np.empty((h, bpp * w + 1), np.uint8)
    out[:, 0] = f
    for k in range(5):
        out[f == k, 1:] = (x - preds[k])[f == k] & 255
    return out.tobytes()


def encode_png(img, filters=4, level=6, wbits=15, idat=8192, zdata=None, ancillary=True):
    """A PNG stream of an HWC uint8 RGB image (an HW one: 8-bit grey) from the standard library: png_filter's
    scanlines through zlib at `level` with a 2^wbits window, split into IDAT chunks of `idat` bytes (an int, or a list
    of chunk lengths, the last taking the rest); zdata replaces the zlib stream.  ancillary adds a tEXt chunk before
    the IDATs."""
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape[:2]
    if zdata is None:
        co = zlib.compressobj(level, zlib.DEFLATED, wbits)
        zdata = co.compress(png_filter(img, filters)) + co.flush()
    ctype = 0 if img.ndim == 2 else 2
    parts = [b"\x89PNG\r\n\x1a\n", png_chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, ctype, 0, 0, 0))]
    if ancillary:
        parts.append(png_chunk(b"tEXt", b"Software\0deepi2p_b200"))
    sizes = list(idat) if isinstance(idat, (list, tuple)) else None
    p = 0
    while p < len(zdata) or p == 0:
        n = (sizes.pop(0) if sizes else len(zdata) - p) if sizes is not None else idat
        parts.append(png_chunk(b"IDAT", zdata[p:p + n]))
        p += n
        if sizes is not None and not sizes and p < len(zdata):
            parts.append(png_chunk(b"IDAT", zdata[p:]))
            p = len(zdata)
    parts.append(png_chunk(b"IEND", b""))
    return b"".join(parts)
