"""numpy oracle of the point encoder's cluster max-pool and node kNN grouping -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and the benchmark scripts may import this package; deepi2p_b200.point_ops never
does.  It restates DESIGN.md 4.16: the forwards in float32 on top of oracle.index_max and oracle.cluster_assign's key
order (numpy rounds every elementwise operation once and never contracts a multiply-add), the feature gradients as
fp64 sums of the incoming float32 terms, rounded once.
"""
import numpy as np

import oracle


def pool_select(features, min_idx, M):
    """sel [B,C,M] int32 (index_max with points outside [0, M) left out) and mask [B,M] float32."""
    F = np.asarray(features, dtype=np.float32)
    idx = np.asarray(min_idx).astype(np.int64)
    valid = (idx >= 0) & (idx < M)
    # a left-out point gets -inf, which never wins a segment (index_max drops values <= -1000), and segment 0
    data = np.where(valid[:, None, :], F, np.float32(-np.inf)).astype(np.float32)
    sel = oracle.index_max(data, np.where(valid, idx, 0).astype(np.int32), M)
    B = idx.shape[0]
    mask = np.zeros((B, M), np.float32)
    for b in range(B):
        mask[b, idx[b][valid[b]]] = 1.0
    return sel, mask


def cluster_max_pool(features, min_idx, M, broadcast=False):
    """pooled [B,C,M] = features[b,c,sel] * mask (one f32 multiply) and, with broadcast, scattered [B,C,N] =
    pooled[b,c,min_idx], NaN for a point outside [0, M).  Returns (pooled, scattered or None, sel, mask)."""
    F = np.asarray(features, dtype=np.float32)
    idx = np.asarray(min_idx).astype(np.int64)
    sel, mask = pool_select(F, idx, M)
    with np.errstate(invalid="ignore"):
        pooled = np.take_along_axis(F, sel.astype(np.int64), axis=2) * mask[:, None, :]
    scattered = None
    if broadcast:
        valid = (idx >= 0) & (idx < M)
        safe = np.where(valid, idx, 0)
        scattered = np.take_along_axis(pooled, np.broadcast_to(safe[:, None, :], F.shape), axis=2).copy()
        scattered[np.broadcast_to(~valid[:, None, :], F.shape)] = np.nan
    return pooled.astype(np.float32), scattered, sel, mask


def cluster_max_pool_backward(features, min_idx, M, grad_pooled=None, grad_scattered=None, with_abs=False):
    """gF [B,C,N] f32 = sum over m with sel = n of mask * (gP + sum over n' with min_idx = m of gS), in fp64, rounded
    once.  Either gradient may be None.  with_abs also returns the fp64 sum of the terms' magnitudes."""
    F = np.asarray(features, dtype=np.float32)
    idx = np.asarray(min_idx).astype(np.int64)
    B, C, N = F.shape
    sel, mask = pool_select(F, idx, M)
    valid = (idx >= 0) & (idx < M)
    t = np.zeros((B, C, M), np.float64)
    ta = np.zeros((B, C, M), np.float64)
    if grad_pooled is not None:
        gp = np.asarray(grad_pooled, dtype=np.float32).astype(np.float64)
        t += gp
        ta += np.abs(gp)
    if grad_scattered is not None:
        gs = np.asarray(grad_scattered, dtype=np.float32).astype(np.float64)
        for b in range(B):
            m = idx[b][valid[b]]
            for c in range(C):
                t[b, c] += np.bincount(m, weights=gs[b, c][valid[b]], minlength=M)
                ta[b, c] += np.bincount(m, weights=np.abs(gs[b, c][valid[b]]), minlength=M)
    with np.errstate(invalid="ignore"):
        t = t * mask[:, None, :].astype(np.float64)
    ta = ta * mask[:, None, :]
    gF = np.zeros((B, C, N), np.float64)
    ab = np.zeros((B, C, N), np.float64)
    for b in range(B):
        for c in range(C):
            gF[b, c] = np.bincount(sel[b, c], weights=t[b, c], minlength=N)
            ab[b, c] = np.bincount(sel[b, c], weights=ta[b, c], minlength=N)
    out = gF.astype(np.float32)
    return (out, ab) if with_abs else out


def knn_indices(query, database, K):
    """knn_idx [B,M,K] int32: stable sort of the f32 key ((dx*dx + dy*dy) + dz*dz), so ties go to the lower index,
    +inf after finite keys and NaN last."""
    q = np.asarray(query, dtype=np.float32)
    db = np.asarray(database, dtype=np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        d = q[:, :, :, None] - db[:, :, None, :]                 # [B,3,M,N], query - database
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
    return np.argsort(d2, axis=2, kind="stable")[:, :, :K].astype(np.int32)


def knn_group(query, database, features, K):
    """(knn_idx [B,M,K] int32, grouped [B,3+C,M,K] f32): rows 0-2 database[idx] - query, rows 3.. features[idx]."""
    q = np.asarray(query, dtype=np.float32)
    db = np.asarray(database, dtype=np.float32)
    F = np.asarray(features, dtype=np.float32)
    idx = knn_indices(q, db, K)
    B, M, _ = idx.shape
    C = F.shape[1]
    grouped = np.empty((B, 3 + C, M, K), np.float32)
    with np.errstate(over="ignore", invalid="ignore"):
        for b in range(B):
            grouped[b, :3] = db[b][:, idx[b]] - q[b][:, :, None]
            grouped[b, 3:] = F[b][:, idx[b]]
    return idx, grouped


def knn_group_backward(knn_idx, grad_grouped, N, with_abs=False):
    """gF [B,C,N] f32 = sum over (m, j) with knn_idx = n of grad_grouped[b, 3 + c, m, j], in fp64, rounded once."""
    idx = np.asarray(knn_idx).astype(np.int64)
    g = np.asarray(grad_grouped, dtype=np.float32).astype(np.float64)
    B = idx.shape[0]
    C = g.shape[1] - 3
    gF = np.zeros((B, C, N), np.float64)
    ab = np.zeros((B, C, N), np.float64)
    for b in range(B):
        flat = idx[b].ravel()
        for c in range(C):
            gF[b, c] = np.bincount(flat, weights=g[b, 3 + c].ravel(), minlength=N)
            ab[b, c] = np.bincount(flat, weights=np.abs(g[b, 3 + c].ravel()), minlength=N)
    out = gF.astype(np.float32)
    return (out, ab) if with_abs else out
