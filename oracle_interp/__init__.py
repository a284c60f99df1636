"""numpy oracle of the decoder's inverse-distance interpolation -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and the benchmark scripts may import this package; deepi2p_b200.point_ops never
does.  It restates DESIGN.md 4.12 one operation at a time: the forward in float32 (numpy rounds every elementwise
operation once and never contracts a multiply-add), the feature gradient as an fp64 sum of the exact fp32 products.
"""
import numpy as np


def interp_weights(topk_idx, query, node):
    """w [B,Nq,k] f32 and a validity mask [B,Nq] (every index in [0, M)).  Invalid points get NaN weights."""
    idx = np.asarray(topk_idx).astype(np.int64)
    q = np.asarray(query, dtype=np.float32)
    nd = np.asarray(node, dtype=np.float32)
    B, Nq, k = idx.shape
    M = nd.shape[2]
    valid = ((idx >= 0) & (idx < M)).all(axis=2)
    safe = np.where(valid[..., None], idx, 0)
    w = np.empty((B, Nq, k), np.float32)
    with np.errstate(invalid="ignore", divide="ignore"):
        for b in range(B):
            d = []
            for j in range(k):
                nj = nd[b][:, safe[b, :, j]]                                     # [3, Nq]
                dx, dy, dz = q[b, 0] - nj[0], q[b, 1] - nj[1], q[b, 2] - nj[2]
                d.append(np.sqrt((dx * dx + dy * dy) + dz * dz))
            S = d[0]
            for j in range(1, k):
                S = S + d[j]
            for j in range(k):
                w[b, :, j] = np.float32(1) - d[j] / S
    w[~valid] = np.nan
    return w, valid


def interp_forward(topk_idx, query, node, features):
    """out [B,C,Nq] f32 = ((w_0 F[:, i_0] + w_1 F[:, i_1]) + ...), NaN columns for points with a bad index."""
    F = np.asarray(features, dtype=np.float32)
    w, valid = interp_weights(topk_idx, query, node)
    idx = np.where(valid[..., None], np.asarray(topk_idx).astype(np.int64), 0)
    B, Nq, k = idx.shape
    out = np.empty((B, F.shape[1], Nq), np.float32)
    with np.errstate(invalid="ignore"):
        for b in range(B):
            acc = w[b, :, 0][None] * F[b][:, idx[b, :, 0]]
            for j in range(1, k):
                acc = acc + w[b, :, j][None] * F[b][:, idx[b, :, j]]
            out[b] = acc
    out[np.broadcast_to(~valid[:, None, :], out.shape)] = np.nan
    return out


def interp_backward(topk_idx, query, node, grad_out, M, with_abs=False):
    """gF [B,C,M] f32: the fp64 sum over (n, j) with idx[b,n,j] = m of float64(w) * float64(g[b,c,n]) (exact products),
    rounded once.  Points with a bad index contribute nothing.  with_abs also returns sum |w g| in fp64, the scale of
    the contract's absolute term."""
    g = np.asarray(grad_out, dtype=np.float32).astype(np.float64)
    w, valid = interp_weights(topk_idx, query, node)
    idx = np.asarray(topk_idx).astype(np.int64)
    B, Nq, k = idx.shape
    C = g.shape[1]
    gF = np.zeros((B, C, M), np.float64)
    ab = np.zeros((B, C, M), np.float64)
    for b in range(B):
        n_ok = np.nonzero(valid[b])[0]
        for j in range(k):
            p = w[b, n_ok, j].astype(np.float64)[None] * g[b][:, n_ok]          # [C, n_ok]
            m = idx[b, n_ok, j]
            for c in range(C):
                gF[b, c] += np.bincount(m, weights=p[c], minlength=M)
                if with_abs:
                    ab[b, c] += np.bincount(m, weights=np.abs(p[c]), minlength=M)
    out = gF.astype(np.float32)
    return (out, ab) if with_abs else out
