"""numpy oracle of the KITTI camera-frame records and depth maps -- TEST INFRASTRUCTURE ONLY.

Only tests/, tests/golden/ generators, __graft_entry__.smoke() and the benchmark scripts may import this package;
deepi2p_b200 never does.  It restates data/kitti/kitti_pc_bin_to_npy_in_img_frame.py process_kitti one scan and one
camera at a time, in the reference's own structure, with the project's documented contract (DESIGN.md 4.33):

  - the per-point competition is the reference's loop, in file order, with its comparison d < (double) stored;
  - the transform is the fixed fp64 association ((Pc0 x + Pc1 y) + Pc2 z) + Pc3, and the projection
    (K0 X + K1 Y) + K2 Z, in place of np.dot's BLAS order;
  - the distance transform is the exact nearest filled pixel, the smallest column and then the smallest row among
    the nearest (the index scipy.ndimage.distance_transform_edt returns), with scipy's (-1, 0) when nothing is filled;
  - the voxel grid, normals and nearest-point intensity are oracle_prep's (DESIGN.md 4.10).

project_rule is the order-independent form of the competition the kernels compute; the tests hold it against
project_loop.
"""
import math
import os

import numpy as np

import oracle_prep

CAMERAS = ("P2", "P3")


def affine(P, p):
    """Rows ((P0 x + P1 y) + P2 z) + P3 in fp64 of points p [3,n] (any float dtype, widened)."""
    x, y, z = (np.asarray(p[a]).astype(np.float64) for a in range(3))
    return np.stack([((P[r, 0] * x + P[r, 1] * y) + P[r, 2] * z) + P[r, 3] for r in range(3)])


def project(pc_np, Pc, K):
    """(P_pc_homo [3,N] f64, u, v, w [N] f64) of a float32 scan [3,N] under Pc [4,4] and the float32 K [3,3]."""
    X = affine(Pc, pc_np)
    Kd = np.asarray(K, dtype=np.float32).astype(np.float64)
    u, v, w = ((Kd[r, 0] * X[0] + Kd[r, 1] * X[1]) + Kd[r, 2] * X[2] for r in range(3))
    return X, u, v, w


def project_loop(pc_np, Pc, K, H, W):
    """The reference's loop (lines 117-136), point by point in file order.  Returns (img_depth [H,W] f32,
    img_depth_dist_to_nn_pc [H,W] f32, img_depth_mask [H,W] bool).  A point with w = 0 is not projected (the
    reference's round(inf) raises)."""
    img_depth = np.zeros((H, W), dtype=np.float32)
    img_depth_dist_to_nn_pc = np.zeros((H, W), dtype=np.float32) + H * W
    img_depth_mask = np.zeros((H, W), dtype=bool)
    P_pc_homo, u, v, w = project(pc_np, Pc, K)
    with np.errstate(divide="ignore", invalid="ignore"):
        KP_pc_pxpy = np.stack([u / w, v / w])
    for j in range(KP_pc_pxpy.shape[1]):
        if w[j] == 0:
            continue
        px = KP_pc_pxpy[0, j]
        py = KP_pc_pxpy[1, j]
        px_round = int(round(px))
        py_round = int(round(py))
        pz = P_pc_homo[2, j]
        if pz > 0.1 and px_round >= 0 and px_round <= W - 1 and py_round >= 0 and py_round <= H - 1:
            dx = px - float(px_round)
            dy = py - float(py_round)
            dist_to_nn_pc = math.sqrt(dx * dx + dy * dy)
            if dist_to_nn_pc < float(img_depth_dist_to_nn_pc[py_round, px_round]):
                img_depth[py_round, px_round] = pz
                img_depth_dist_to_nn_pc[py_round, px_round] = dist_to_nn_pc
                img_depth_mask[py_round, px_round] = True
    return img_depth, img_depth_dist_to_nn_pc, img_depth_mask


def project_rule(pc_np, Pc, K, H, W):
    """The same three arrays from the order-independent rule: per pixel m = min float32(d); the winner is the largest
    index with d < m if there is one, else the smallest index with float32(d) = m."""
    X, u, v, w = project(pc_np, Pc, K)
    ok = w != 0
    with np.errstate(divide="ignore", invalid="ignore"):
        px, py = np.where(ok, u / w, 0.0), np.where(ok, v / w, 0.0)
    rx, ry = np.rint(px), np.rint(py)
    ok &= (X[2] > 0.1) & (rx >= 0) & (rx <= W - 1) & (ry >= 0) & (ry <= H - 1)
    dx, dy = px - rx, py - ry
    d = np.sqrt(dx * dx + dy * dy)
    f = d.astype(np.float32)
    idx = np.nonzero(ok)[0]
    pix = (ry[idx] * W + rx[idx]).astype(np.int64)
    m = np.full(H * W, np.inf, dtype=np.float32)
    np.minimum.at(m, pix, f[idx])
    hi = np.full(H * W, -1, dtype=np.int64)
    below = d[idx] < m[pix].astype(np.float64)
    np.maximum.at(hi, pix[below], idx[below])
    lo = np.full(H * W, np.iinfo(np.int64).max, dtype=np.int64)
    eq = f[idx] == m[pix]
    np.minimum.at(lo, pix[eq], idx[eq])
    mask = np.isfinite(m)
    win = np.where(hi >= 0, hi, lo)[mask]
    img_depth = np.zeros(H * W, dtype=np.float32)
    img_depth[mask] = X[2][win].astype(np.float32)
    dist = np.full(H * W, np.float32(H * W))
    dist[mask] = m[mask]
    return img_depth.reshape(H, W), dist.reshape(H, W), mask.reshape(H, W)


def edt(mask_inv):
    """distance_transform_edt(mask_inv, return_indices=True) under the rule above: (edt_val [H,W] f64, edt_idx
    [2,H,W] int64).  The feature pixels are those where mask_inv is False."""
    H, W = mask_inv.shape
    filled = ~np.asarray(mask_inv, dtype=bool)
    rows, cols = np.mgrid[0:H, 0:W]
    if not filled.any():
        idx = np.stack([np.full((H, W), -1), np.zeros((H, W), dtype=np.int64)])
        return np.sqrt(((rows + 1) ** 2 + cols ** 2).astype(np.float64)), idx
    # nearest filled row of each pixel within its column, the lower row on ties (-1: the column has none)
    near = np.full((H, W), -1, dtype=np.int64)
    above = np.full(W, -1, dtype=np.int64)
    for r in range(H):
        above = np.where(filled[r], r, above)
        near[r] = above
    below = np.full(W, -1, dtype=np.int64)
    for r in range(H - 1, -1, -1):
        below = np.where(filled[r], r, below)
        up = near[r]
        take = (below >= 0) & ((up < 0) | (below - r < r - up))
        near[r] = np.where(take, below, up)
    idx = np.zeros((2, H, W), dtype=np.int64)
    d2 = np.zeros((H, W), dtype=np.int64)
    c = np.arange(W)
    big = np.iinfo(np.int64).max // 4
    for r in range(H):
        f = np.where(near[r] >= 0, (r - near[r]) ** 2, big)
        D = (c[:, None] - c[None, :]) ** 2 + f[None, :]          # [pixel column, source column]
        q = np.argmin(D, axis=1)                                  # the first minimum: the smallest column
        idx[0, r], idx[1, r] = near[r][q], q
        d2[r] = D[c, q]
    return np.sqrt(d2.astype(np.float64)), idx


def depth_map(pc_np, Pc, K, H, W):
    """One camera's [2, H, W] float32 depth map (lines 117-145 with project_loop and edt)."""
    img_depth, img_depth_dist_to_nn_pc, img_depth_mask = project_loop(pc_np, Pc, K, H, W)
    img_depth_mask_inv = np.logical_not(img_depth_mask)
    edt_val, edt_idx = edt(img_depth_mask_inv)
    img_depth_dist_to_nn_pc = img_depth_mask * img_depth_dist_to_nn_pc + img_depth_mask_inv * edt_val
    img_depth = img_depth[edt_idx[0], edt_idx[1]]
    return np.stack((img_depth, img_depth_dist_to_nn_pc), axis=0).astype(np.float32)


def coordinate_NWU_to_cam(pc_np):
    out = np.copy(pc_np)
    out[0, :] = -pc_np[1, :]
    out[1, :] = -pc_np[2, :]
    out[2, :] = pc_np[0, :]
    return out


def downsample(pc_np, intensity_np, voxel_size=0.1, sn_radius=0.6, sn_max_nn=30):
    """(pc_down_np [3,M] f64, intensity_down_np [1,M] f32, pc_down_sn_np [3,M] f64) of a float32 scan."""
    down, _ = oracle_prep.voxel_downsample(pc_np, voxel_size)
    sn, _ = oracle_prep.estimate_normals(down.astype(np.float32), sn_radius, sn_max_nn)
    I = oracle_prep.nearest(pc_np, down)
    return down, np.asarray(intensity_np, dtype=np.float32).reshape(1, -1)[:, I], sn


def camera_record(down, intensity_down_np, sn, Pc):
    """One camera's [7, M] float32 record from downsample's outputs."""
    pc_down_img_np = affine(Pc, down)
    pc_down_sn_img_np = coordinate_NWU_to_cam(sn)
    return np.concatenate((pc_down_img_np, intensity_down_np, pc_down_sn_img_np), axis=0).astype(np.float32)


def read_velodyne_bin(path):
    return np.fromfile(path, dtype="<f4").reshape(-1, 4).T.astype(np.float32)


def process_sequence(root, velodyne_root, seq, Pc, K, sizes, voxel_size=0.1, sn_radius=0.6, sn_max_nn=30,
                     frames=None):
    """process_kitti for one sequence without writing: Pc {key: [4,4]}, K {key: [3,3] f32}, sizes {key: [(H, W)] per
    frame}.  Returns (records {(i, key): [7, M]}, maps {(i, key): [2, H, W]})."""
    folder = os.path.join(velodyne_root, "sequences", "%02d" % seq, "velodyne")
    sample_num = round(len(os.listdir(folder)))
    records, maps = {}, {}
    for i in range(sample_num) if frames is None else frames:
        data_np = read_velodyne_bin(os.path.join(folder, "%06d.bin" % i))
        pc_np, intensity_np = data_np[0:3, :], data_np[3:, :]
        down, inten, sn = downsample(pc_np, intensity_np, voxel_size, sn_radius, sn_max_nn)
        for key in CAMERAS:
            records[(i, key)] = camera_record(down, inten, sn, Pc[key])
            H, W = sizes[key][i]
            maps[(i, key)] = depth_map(pc_np, Pc[key], K[key], H, W)
    return records, maps
