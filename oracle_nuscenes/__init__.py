"""numpy oracle of the nuScenes point side -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and the benchmark scripts may import this package; deepi2p_b200 never does.  It
restates DESIGN.md 4.20 one sample at a time: the ego-vehicle box tested in float32 on each sweep's own coordinates,
the fixed-association fp64 transform kept in fp64, the voxel grid on the fp64 cloud (the kernels' order: ascending
(ix, iy, iz), sums in ascending point index), and then oracle_assemble's resample, jitter, transform and node sets.
"""
import numpy as np

import oracle_assemble as oa

EGO_BOX = (-0.8, 0.8, -2.7, 2.7)


def ego_mask(xyz, box=EGO_BOX):
    """Keep mask of float32 points xyz [3,n]: not (x_lo < x < x_hi and y_lo < y < y_hi), compared in float32."""
    x, y = np.asarray(xyz[0], dtype=np.float32), np.asarray(xyz[1], dtype=np.float32)
    lo_x, hi_x, lo_y, hi_y = (np.float32(v) for v in box)
    inside = np.logical_and(np.logical_and(x < hi_x, x > lo_x), np.logical_and(y < hi_y, y > lo_y))
    return np.logical_not(inside)


def affine64(M, p):
    """Rows ((M0 x + M1 y) + M2 z) + M3 in fp64 of float32 points p [3,n], kept in fp64."""
    x, y, z = (np.asarray(p[a], dtype=np.float32).astype(np.float64) for a in range(3))
    return np.stack([((M[r, 0] * x + M[r, 1] * y) + M[r, 2] * z) + M[r, 3] for r in range(3)])


def accumulate(frames, frame_T, box=EGO_BOX):
    """One sample's sweeps [(xyz [3,n] f32, intensity [n] f32, None)] masked by the box in their own frame, moved by
    frame_T [T,4,4] and concatenated.  Returns (xyz [3,n] float64, intensity [n] float32)."""
    xs, its = [], []
    for (x, it, _), M in zip(frames, frame_T):
        keep = ego_mask(x, box) if box is not None else np.ones(np.asarray(x).shape[1], dtype=bool)
        xs.append(affine64(np.asarray(M, dtype=np.float64), np.asarray(x)[:, keep]))
        its.append(np.asarray(it, dtype=np.float32).reshape(-1)[keep])
    return np.concatenate(xs, 1), np.concatenate(its)


def voxel_downsample64(xyz, voxel_size, attr):
    """The voxel grid on fp64 points xyz [3,n] with attributes attr [C,n] f64: min_bound = min - 0.5 v, voxel =
    floor((p - min_bound) / v), voxels in ascending (ix, iy, iz), each mean a sequential sum in ascending point index
    divided by the count.  Returns (xyz [3,m] f64, attr [C,m] f64)."""
    p = np.asarray(xyz, dtype=np.float64)
    A = np.asarray(attr, dtype=np.float64)
    mb = p.min(1) - 0.5 * voxel_size
    idx = np.maximum(np.floor((p - mb[:, None]) / voxel_size), 0.0).astype(np.int64)
    order = np.lexsort((idx[2], idx[1], idx[0]))          # stable: ascending point index within a voxel
    k = idx[:, order]
    head = np.ones(order.size, dtype=bool)
    head[1:] = np.any(k[:, 1:] != k[:, :-1], axis=0)
    start = np.nonzero(head)[0]
    count = np.diff(np.append(start, order.size))
    vals = np.concatenate([p, A])[:, order]
    acc = np.zeros((vals.shape[0], start.size))
    for j in range(int(count.max())):
        live = count > j
        acc[:, live] = acc[:, live] + vals[:, start[live] + j]
    mean = acc / count.astype(np.float64)
    return mean[:3], mean[3:]


def voxel_step(xyz, inten, voxel_size=0.2):
    """downsample_with_reflectance on the fp64 cloud (reflectance / max in float32, means in fp64, times max), then
    both rounded to float32."""
    imax = np.max(inten)
    px, A = voxel_downsample64(xyz, voxel_size, (inten / imax).astype(np.float64)[None])
    return px.astype(np.float32), (A[0] * imax).astype(np.float32)


def assemble_sample(frames, frame_T, s, seed, M, N=20480, node_a_num=128, node_b_num=128, voxel_size=0.2,
                    box=EGO_BOX, jitter_channels=(), sigma=0.01, clip=0.05):
    """Sample s of assemble_batch(**nuscenes_args): M = Pr pre [4,4] (fp64).  Returns oracle_assemble.assemble_sample's
    dict (sn zeros)."""
    x64, it = accumulate(frames, frame_T, box)
    if x64.shape[1] > 2 * N:
        x, it = voxel_step(x64, it, voxel_size)
    else:
        x = x64.astype(np.float32)
    n = x.shape[1]
    src = oa.resample_index(n, N, s, seed)
    p = x[:, src]
    i_ = it[src]
    if "pc" in jitter_channels:
        p = p + oa.jitter(oa.normals3(N, s, oa.STREAM_JITTER_PC, seed), sigma, clip)
    if "intensity" in jitter_channels:
        i_ = i_ + oa.jitter(oa.normals3(N, s, oa.STREAM_JITTER_INTENSITY, seed)[0], sigma, clip)
    pc = oa.affine(M, p)
    out = dict(pc=pc, intensity=i_[None], sn=np.zeros((3, N), dtype=np.float32), src=src, n_before_resample=n)
    for name, m, stream in (("node_a", node_a_num, oa.STREAM_NODE_A), ("node_b", node_b_num, oa.STREAM_NODE_B)):
        cand = oa.key_order(N, s, stream, seed)[:8 * m]
        fi, nodes = oa.fps(pc[:, cand], m, 0)
        out[name] = nodes
        out[name + "_idx"] = cand[fi]
    return out
