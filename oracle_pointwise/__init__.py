"""Float64 restatement of point_ops.pointwise_mlp (csrc/pointwise_mlp.cu, DESIGN.md 4.21) with a running error bound.

It follows the kernel's formulation, not the unfused network's: an interpolated source's block of W1 is applied to
the node features first and the projected rows are interpolated per point; weights, source values and the activations
fed to the next layer are rounded to TF32 by tf32_round (nearest, ties away from zero: the kernel's tf32_rna); the
products and sums are float64 here and float32 on the device; bias, ReLU (NaN stays NaN) and the arg-max follow.

Next to the values it returns, per element, a bound on |device - oracle| by forward analysis: operands rounded the
same way on both sides contribute nothing, an f32 accumulation of K products contributes (K + 8) U32 |W| |x| (U32 =
2^-23 covers a truncating accumulator), an input error e contributes |W| e, ReLU is 1-Lipschitz, and re-rounding an
activation that is off by e gives e (1 + U_TF32) + 2 U_TF32 |y|.  Where the oracle's value is not finite the bound is
0: the device must then hold the same NaN or infinity.  Tests, smoke() and nothing else use this module.
"""
import numpy as np

U_TF32 = 2.0 ** -11 * (1 + 2.0 ** -12)      # half a TF32 ulp, plus the float64 -> float32 step before it
U_32 = 2.0 ** -23


def tf32_round(x):
    """float32 -> the nearest value with 10 mantissa bits, ties away from zero; a value that rounds past the largest
    finite float becomes infinity, NaN is returned unchanged."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    nan = (u & np.uint32(0x7fffffff)) > np.uint32(0x7f800000)
    r = (u + np.uint32(0x1000)) & np.uint32(0xffffe000)
    return np.where(nan, u, r).astype(np.uint32).view(np.float32)


def relu(z):
    """torch.relu: NaN stays NaN."""
    return np.where(z < 0, 0.0, z)


def argmax_rule(scores):
    """torch.max's index over axis 1 of [B,C,N]: the first NaN if there is one, else the first maximum."""
    nan = np.isnan(scores)
    first_nan = np.argmax(nan, axis=1)
    with np.errstate(invalid="ignore"):
        best = np.argmax(np.where(nan, -np.inf, scores), axis=1)
    return np.where(nan.any(axis=1), first_nan, best)


def gather(P, w, idx):
    """sum_j w[b,n,j] P[b,:,idx[b,n,j]] -> [B,C,N]; a point with an index outside [0, M) is NaN in every channel.
    Also returns sum_j |w| |P| and the mask of those points."""
    B, C, M = P.shape
    bad = ((idx < 0) | (idx >= M)).any(axis=2)                       # [B,N]
    safe = np.where((idx < 0) | (idx >= M), 0, idx)
    out = np.zeros((B, C, idx.shape[1]))
    mag = np.zeros_like(out)
    for j in range(idx.shape[2]):
        g = np.take_along_axis(P, np.broadcast_to(safe[:, None, :, j], (B, C, idx.shape[1])), axis=2)
        wj = w[:, None, :, j].astype(np.float64)
        out += wj * g
        mag += np.abs(wj) * np.abs(g)
    out[np.broadcast_to(bad[:, None, :], out.shape)] = np.nan
    return out, mag, bad


def pointwise_mlp(sources, layers, c_split=None, tf32=True):
    """sources: arrays [B,C,N] (dense) or tuples (features [B,C,M], w [B,N,k] float32, idx [B,N,k]); layers: [(W
    [C_out,C_in], b [C_out] or None, relu)].  Returns dict(out [B,C_out,N] float64, bound (same shape), and with
    c_split pred_a, pred_b (None when [c_split, C_out) is empty) and margin_a, margin_b: the gap between the best
    and the second-best score of each range (inf for a one-channel range)).  tf32=False drops every rounding and is
    the exact layer chain over the interpolated rows (the bound is then all zero)."""
    rnd = (lambda a: tf32_round(a).astype(np.float64)) if tf32 else (lambda a: np.asarray(a, dtype=np.float64))
    u32 = U_32 if tf32 else 0.0
    u_tf = U_TF32 if tf32 else 0.0
    with np.errstate(all="ignore"):
        W1, b1, relu1 = layers[0]
        W1r = rnd(W1)
        C1 = W1r.shape[0]
        col = 0
        z = mag = err = None
        dense_x, dense_w = [], []
        for s in sources:
            if isinstance(s, (tuple, list)):
                F, w, idx = s
                Ws = W1r[:, col:col + F.shape[1]]
                Fr = rnd(F)
                P = Ws @ Fr                                              # [B,C1,M]
                eP = (F.shape[1] + 8) * u32 * (np.abs(Ws) @ np.abs(Fr)) + u32 * np.abs(P)
                val, m, bad = gather(P, w, np.asarray(idx))
                e, _, _ = gather(eP, np.abs(np.asarray(w, dtype=np.float64)), np.asarray(idx))
                e = np.where(np.isnan(e), 0.0, e) + (np.asarray(idx).shape[2] * len(sources) + 2) * u32 * m
                col += F.shape[1]
            else:
                dense_x.append(rnd(s))
                dense_w.append(W1r[:, col:col + s.shape[1]])
                col += s.shape[1]
                continue
            z = val if z is None else z + val
            mag = np.abs(val) if mag is None else mag + np.abs(val)
            err = e if err is None else err + e
        if dense_x:
            x, Wd = np.concatenate(dense_x, axis=1), np.concatenate(dense_w, axis=1)
            val = Wd @ x
            e = (x.shape[1] + 8) * u32 * (np.abs(Wd) @ np.abs(x))
            z = val if z is None else z + val
            mag = np.abs(val) if mag is None else mag + np.abs(val)
            err = e if err is None else err + e
        assert col == W1r.shape[1], (col, W1r.shape)
        if b1 is not None:
            bb = np.asarray(b1, dtype=np.float64)[None, :, None]
            z = z + bb
            mag = mag + np.abs(bb)
        err = err + 3 * u32 * mag
        y = relu(z) if relu1 else z
        err = np.where(np.isfinite(z), err, 0.0)
        for W, b, act in layers[1:]:
            x = rnd(y)
            e_in = err * (1 + u_tf) + 2 * u_tf * np.abs(x)
            e_in = np.where(np.isfinite(x), e_in, 0.0)
            Wr = rnd(W)
            z = Wr @ x
            mag = np.abs(Wr) @ np.abs(x)
            err = np.abs(Wr) @ e_in + (x.shape[1] + 8) * u32 * mag
            if b is not None:
                bb = np.asarray(b, dtype=np.float64)[None, :, None]
                z = z + bb
                mag = mag + np.abs(bb)
            err = err + 2 * u32 * mag
            y = relu(z) if act else z
            err = np.where(np.isfinite(z), err, 0.0)
        res = dict(out=y, bound=np.where(np.isfinite(y), err, 0.0))
        if c_split is not None:
            for name, lo, hi in (("a", 0, c_split), ("b", c_split, y.shape[1])):
                if lo >= hi:
                    res["pred_" + name], res["margin_" + name] = None, None
                    continue
                part = y[:, lo:hi]
                res["pred_" + name] = argmax_rule(part)
                if hi - lo == 1:
                    res["margin_" + name] = np.full(part[:, 0].shape, np.inf)
                else:
                    top = np.sort(np.where(np.isnan(part), np.inf, part), axis=1)
                    res["margin_" + name] = top[:, -1] - top[:, -2]
        return res
