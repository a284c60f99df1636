"""numpy oracle of the batch-assembly path -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and the benchmark scripts may import this package; deepi2p_b200.assemble never
does.  It restates DESIGN.md "Batch assembly" one sample at a time from the same Philox streams: a vectorised uint32
Philox4x32-10, the key order, the repeat rule of downsample_np, Box-Muller jitter, the fixed-association transforms and
farthest-point sampling written the reference's way.  The voxel step is oracle_prep's (C++) voxel grid.
"""
import numpy as np

import oracle_prep

STREAM_RESAMPLE, STREAM_JITTER_PC, STREAM_JITTER_SN, STREAM_NODE_A, STREAM_NODE_B, STREAM_JITTER_INTENSITY = 1, 2, 3, 4, \
    5, 6
M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
MASK32 = 0xFFFFFFFF


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al., SC'11) on counters ctr [4, n] (uint32-valued) with key (k0, k1).  Returns [4, n]
    uint64 arrays holding uint32 words."""
    c = [np.asarray(x, dtype=np.uint64) & MASK32 for x in ctr]
    n = max(x.size for x in c)
    c = [np.broadcast_to(x, (n,)).copy() for x in c]
    k0, k1 = np.uint64(key[0] & MASK32), np.uint64(key[1] & MASK32)
    for _ in range(10):
        p0 = np.uint64(M0) * c[0]
        p1 = np.uint64(M1) * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & np.uint64(MASK32)
        hi1, lo1 = p1 >> np.uint64(32), p1 & np.uint64(MASK32)
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0 = (k0 + np.uint64(W0)) & np.uint64(MASK32)
        k1 = (k1 + np.uint64(W1)) & np.uint64(MASK32)
    return np.stack(c)


def words(n, s, stream, seed):
    """The four Philox words of positions 0..n-1 of sample s in a stream: counter (pos, s, stream, 0), key = seed."""
    seed = int(seed) & (2**64 - 1)
    return philox4x32_10([np.arange(n), s, stream, 0], (seed & MASK32, seed >> 32))


def key_order(n, s, stream, seed):
    """Positions 0..n-1 sorted by (64-bit key = w0 << 32 | w1, position)."""
    w = words(n, s, stream, seed)
    return np.argsort((w[0] << np.uint64(32)) | w[1], kind="stable")


def resample_index(n, N, s, seed):
    """downsample_np's choice for a cloud of n points: N in key order, or r copies of range(n) then N - r n in key
    order, r >= 1 the smallest with (r + 1) n >= N."""
    order = key_order(n, s, STREAM_RESAMPLE, seed)
    if n >= N:
        return order[:N]
    r = 1
    while n + r * n < N:
        r += 1
    return np.concatenate([np.tile(np.arange(n), r), order[:N - r * n]])


def normals3(n, s, stream, seed):
    """Box-Muller on the words of each position: z0 = r0 cos t0, z1 = r0 sin t0, z2 = r1 cos t1, r_i = sqrt(-2 log
    u(w_2i)), t_i = 2 pi u(w_2i+1), u(w) = (w + 0.5) 2^-32.  Returns [3, n] float64."""
    w = words(n, s, stream, seed).astype(np.float64)
    u = (w + 0.5) * 2.3283064365386963e-10
    r0, t0 = np.sqrt(-2.0 * np.log(u[0])), 6.283185307179586 * u[1]
    r1, t1 = np.sqrt(-2.0 * np.log(u[2])), 6.283185307179586 * u[3]
    return np.stack([r0 * np.cos(t0), r0 * np.sin(t0), r1 * np.cos(t1)])


def jitter(z, sigma=0.01, clip=0.05):
    return np.clip(sigma * z, -clip, clip).astype(np.float32)


def affine(M, p):
    """Rows ((M0 x + M1 y) + M2 z) + M3 in fp64 of float32 points p [3, n], rounded to float32."""
    x, y, z = (p[a].astype(np.float64) for a in range(3))
    return np.stack([((M[r, 0] * x + M[r, 1] * y) + M[r, 2] * z) + M[r, 3] for r in range(3)]).astype(np.float32)


def rotate(M, p):
    x, y, z = (p[a].astype(np.float64) for a in range(3))
    return np.stack([(M[r, 0] * x + M[r, 1] * y) + M[r, 2] * z for r in range(3)]).astype(np.float32)


def compose(A, B):
    """A @ B with the association ((a0 b0 + a1 b1) + a2 b2) + a3 b3."""
    out = np.zeros((4, 4))
    for i in range(4):
        for j in range(4):
            out[i, j] = ((A[i, 0] * B[0, j] + A[i, 1] * B[1, j]) + A[i, 2] * B[2, j]) + A[i, 3] * B[3, j]
    return out


def fps(pts, k, start=0):
    """FarthestSampler.sample with a given start: pts [D, n] (D = 2 or 3), fp64 distances (dx dx + dy dy) + dz dz, the
    running minimum, np.argmax (first maximum).  Returns (idx int64 [k], nodes [D, k] in pts' dtype)."""
    P = np.asarray(pts).astype(np.float64)
    idx = np.zeros(k, dtype=np.int64)
    idx[0] = start
    dmin = np.full(P.shape[1], np.inf)
    for i in range(k):
        w = idx[i]
        d = (P[0] - P[0, w]) * (P[0] - P[0, w]) + (P[1] - P[1, w]) * (P[1] - P[1, w])
        if P.shape[0] == 3:
            d = d + (P[2] - P[2, w]) * (P[2] - P[2, w])
        dmin = np.minimum(dmin, d)
        if i + 1 < k:
            idx[i + 1] = int(np.argmax(dmin))
    return idx, np.asarray(pts)[:, idx]


def accumulate(frames, frame_T, range_max=None):
    """One sample's frames [(xyz [3,n] f32, intensity [n] f32, sn [3,n] f32 or None)] moved by frame_T [T,4,4] and
    concatenated; range_max keeps float32 x^2 + z^2 < range_max^2."""
    xs, its, ns = [], [], []
    for (x, it, sn), M in zip(frames, frame_T):
        p = affine(M, x)
        keep = np.ones(p.shape[1], dtype=bool)
        if range_max is not None:
            keep = p[0] * p[0] + p[2] * p[2] < np.float32(range_max * range_max)
        xs.append(p[:, keep])
        its.append(np.asarray(it, dtype=np.float32)[keep])
        if sn is not None:
            ns.append(rotate(M, sn)[:, keep])
    return np.concatenate(xs, 1), np.concatenate(its), (np.concatenate(ns, 1) if ns else None)


def voxel_step(xyz, inten, sn, voxel_size):
    """downsample_with_intensity_sn / downsample_with_reflectance as the pointprep drop-ins compute them, then float32."""
    imax = np.max(inten)
    rows = [(inten / imax).astype(np.float64)] + ([sn[a].astype(np.float64) for a in range(3)] if sn is not None else [])
    px, A = oracle_prep.voxel_downsample(xyz, voxel_size, np.stack(rows))
    return (px.astype(np.float32), (A[0] * imax).astype(np.float32),
            A[1:4].astype(np.float32) if sn is not None else None)


def assemble_sample(frames, frame_T, s, seed, M, N=20480, node_a_num=128, node_b_num=128, voxel_size=0.3,
                    range_max=None, jitter_channels=(), sigma=0.01, clip=0.05):
    """Sample s of assemble_batch: frames and frame_T as accumulate, M = Pr pre [4,4] (fp64).  Returns dict(pc, intensity
    [1,N], sn, src, n_before_resample, node_a, node_a_idx, node_b, node_b_idx)."""
    x, it, sn = accumulate(frames, frame_T, range_max)
    if x.shape[1] > 2 * N:
        x, it, sn = voxel_step(x, it, sn, voxel_size)
    n = x.shape[1]
    src = resample_index(n, N, s, seed)
    p = x[:, src]
    i_ = it[src]
    q = sn[:, src] if sn is not None else np.zeros((3, N), dtype=np.float32)
    if "pc" in jitter_channels:
        p = p + jitter(normals3(N, s, STREAM_JITTER_PC, seed), sigma, clip)
    if "sn" in jitter_channels and sn is not None:
        q = q + jitter(normals3(N, s, STREAM_JITTER_SN, seed), sigma, clip)
    if "intensity" in jitter_channels:
        i_ = i_ + jitter(normals3(N, s, STREAM_JITTER_INTENSITY, seed)[0], sigma, clip)
    pc = affine(M, p)
    out = dict(pc=pc, intensity=i_[None], sn=rotate(M, q), src=src, n_before_resample=n)
    for name, m, stream in (("node_a", node_a_num, STREAM_NODE_A), ("node_b", node_b_num, STREAM_NODE_B)):
        cand = key_order(N, s, stream, seed)[:8 * m]
        fi, nodes = fps(pc[:, cand], m, 0)
        out[name] = nodes
        out[name + "_idx"] = cand[fi]
    return out
