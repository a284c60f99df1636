"""Float64 restatement of point_ops.knn_fusion and point_ops.pointwise_mlp_max (csrc/knn_fusion.cu, DESIGN.md 4.26)
with a running error bound.

It follows the kernel's formulation: the first "after" layer's input [max; x] is split, W [max; x] = W_p max + W_x x,
with the max projected once per node; weights, grouped values and the activations fed to the next layer are rounded
by oracle_pointwise.tf32_round; the per-node max is taken over the rounded activations; the output max is over the
unrounded last layer; a NaN anywhere in a group gives NaN (torch.max(dim)'s rule).

The bound follows oracle_pointwise's rules: an f32 accumulation of K products contributes (K + 8) U32 |W| |x|, an input
error e contributes |W| e, ReLU is 1-Lipschitz, re-rounding an activation that is off by e gives e (1 + U_TF32) +
2 U_TF32 |y|, and a max of values each within its bound is within the largest of those bounds.  Where the oracle's
value is not finite the bound is 0: the device must then hold the same NaN or infinity.  Tests, smoke() and nothing
else use this module.
"""
import numpy as np

from oracle_pointwise import U_32, U_TF32, relu, tf32_round


def group(query, database, features, idx):
    """knn_group's grouped tensor [B,3+C,M,K] float32 for the given indices [B,M,K]: rows 0-2 database[idx] - query
    (one float32 subtraction), rows 3.. features[idx]."""
    query, database, features = (np.asarray(t, dtype=np.float32) for t in (query, database, features))
    idx = np.asarray(idx, dtype=np.int64)
    B, M, K = idx.shape
    take = lambda a: np.take_along_axis(a, idx.reshape(B, 1, M * K), axis=2).reshape(B, a.shape[1], M, K)
    return np.concatenate((take(database) - query[:, :, :, None], take(features)), axis=1)


def knn_indices(query, database, K):
    """The K nearest database nodes of each query by knn_group's key (float32 ((dx*dx + dy*dy) + dz*dz), ties to the
    lower index; no NaN handling): [B,M,K]."""
    q, d = np.asarray(query, dtype=np.float32), np.asarray(database, dtype=np.float32)
    diff = d[:, :, None, :] - q[:, :, :, None]                               # [B,3,M,N] float32
    sq = diff * diff
    key = (sq[:, 0] + sq[:, 1]) + sq[:, 2]
    return np.argsort(key, axis=2, kind="stable")[:, :, :K].astype(np.int32)


def _matmul(W, x):
    """W [O,C] applied to x [B,C,...] -> [B,O,...]."""
    B, C = x.shape[:2]
    return np.matmul(W, x.reshape(B, C, -1)).reshape((B, W.shape[0]) + x.shape[2:])


def _max(y, e, axis):
    """torch.max(dim)'s value (NaN wins) and the largest bound over the finite members."""
    with np.errstate(invalid="ignore"):
        v = np.where(np.isnan(y).any(axis=axis), np.nan, np.max(np.where(np.isnan(y), -np.inf, y), axis=axis))
    return v, np.max(np.where(np.isfinite(y), e, 0.0), axis=axis)


class _Rules:
    def __init__(self, tf32):
        self.rnd = (lambda a: tf32_round(a).astype(np.float64)) if tf32 else (lambda a: np.asarray(a, np.float64))
        self.u32, self.u_tf = (U_32, U_TF32) if tf32 else (0.0, 0.0)

    def store(self, y, err):
        """An activation fed to the next layer: rounded, its bound widened by the re-rounding."""
        x = self.rnd(y)
        return x, np.where(np.isfinite(x), err * (1 + self.u_tf) + 2 * self.u_tf * np.abs(x), 0.0)

    def product(self, W, x, e):
        """(W x, |W| |x|, its error) for rounded weights."""
        Wr = self.rnd(W)
        mag = _matmul(np.abs(Wr), np.abs(x))
        return _matmul(Wr, x), mag, _matmul(np.abs(Wr), e) + (x.shape[1] + 8) * self.u32 * mag

    def finish(self, z, mag, err, b, act, terms):
        if b is not None:
            bb = np.asarray(b, dtype=np.float64).reshape((1, -1) + (1,) * (z.ndim - 2))
            z, mag = z + bb, mag + np.abs(bb)
        err = err + terms * self.u32 * mag
        return (relu(z) if act else z), np.where(np.isfinite(z), err, 0.0)


def _chain(R, x, e, layers, last_rounded):
    y = err = None
    for i, (W, b, act) in enumerate(layers):
        if i > 0:
            x, e = R.store(y, err)
        z, mag, err = R.product(W, x, e)
        y, err = R.finish(z, mag, err, b, act, 2)
    if last_rounded:
        return R.store(y, err)
    return y, err


def knn_fusion(grouped, before, after, tf32=True):
    """grouped [B,3+C,M,K] (group()); before, after: [(W [C_out,C_in], b [C_out] or None, relu)], the first after
    layer's W [C_a, 2 C_b] with the max's columns first.  Returns dict(out [B,C_out,M] float64, bound (same shape)).
    tf32=False drops every rounding and is the exact module (the bound is then all zero)."""
    R = _Rules(tf32)
    with np.errstate(all="ignore"):
        x0 = R.rnd(grouped)
        x, e = _chain(R, x0, np.zeros_like(x0), before, True)                  # rounded, as the kernel stores them
        pooled, ep = _max(x, e, axis=3)                                         # [B,C_b,M]
        W, b, act = after[0]
        Cb = x.shape[1]
        W = np.asarray(W)
        zx, mx, ex = R.product(W[:, Cb:], x, e)
        zp, mp, epp = R.product(W[:, :Cb], pooled, ep)
        y, err = R.finish(zx + zp[..., None], mx + mp[..., None], ex + epp[..., None], b, act, 3)
        for W, b, act in after[1:]:
            x, e = R.store(y, err)
            z, mag, err = R.product(W, x, e)
            y, err = R.finish(z, mag, err, b, act, 2)
        out, bound = _max(y, err, axis=3)
    return dict(out=out, bound=np.where(np.isfinite(out), bound, 0.0))


def pointwise_mlp_max(sources, layers, tf32=True):
    """sources: dense arrays [B,C,N] (concatenated along C); layers as pointwise_mlp's.  Returns dict(out [B,C_out,1]
    float64, bound): the max over the N columns of the chain."""
    R = _Rules(tf32)
    with np.errstate(all="ignore"):
        x0 = R.rnd(np.concatenate([np.asarray(s, dtype=np.float32) for s in sources], axis=1))
        y, err = _chain(R, x0, np.zeros_like(x0), layers, False)
        out, bound = _max(y, err, axis=2)
    return dict(out=out[:, :, None], bound=np.where(np.isfinite(out), bound, 0.0)[:, :, None])
