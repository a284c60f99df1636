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
