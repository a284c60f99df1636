"""Float64 restatement of point_ops.node_mlp (csrc/node_mlp.cu, DESIGN.md 4.27) with a running error bound.

It follows the kernel's formulation: layer 1's input rows are split into the dense sources' rows, multiplied per
column, and the per-sample sources' rows, projected once per sample and output row and added like a bias; weights,
source values and the activations fed to the next layer are rounded by oracle_pointwise.tf32_round; the last layer is
not rounded.

The per-sample projection is evaluated as the kernel evaluates it: a float32 fma chain in ascending input row.  A
product of two TF32 values has at most 22 significant bits, so it is exact in float32 whenever it lies in float32's
normal range (or is zero, infinite or NaN); a float32 multiply followed by a float32 add then equals the fma, and the
chain here is the device's bit for bit.  The projection's bound term covers exactly that: it is zero for every
(sample, output row) whose products are all exact, and where one is not (it underflows below 2^-126), it is twice
n (U32 sum |w| |v| + 2^-148), n the chain's length, which covers both chains' distance from the exact sum.

The rest of the bound is oracle_pointwise's: an f32 accumulation of K products contributes (K + 8) U32 |W| |x|, the
two f32 additions of the projection and the bias contribute U32 each of |W| |x| + |W_p| |v| + |b|, ReLU is
1-Lipschitz, and re-rounding an activation that is off by e gives e (1 + U_TF32) + 2 U_TF32 |y|.  Where the oracle's value is not
finite the bound is 0: the device must then hold the same NaN or infinity.  Tests, smoke() and nothing else use this
module.
"""
import numpy as np

from oracle_knn_fusion import _Rules
from oracle_pointwise import U_32


def project(W, v, tf32=True):
    """The per-sample projection: W [C_out, C] applied to v [B, C] as an fp32 fma chain in ascending c (tf32=True, W
    and v rounded to TF32) or exactly in float64 (tf32=False).  Returns (proj [B, C_out] float64, magnitude sum |W|
    |v|, bound on |device - proj|)."""
    R = _Rules(tf32)
    Wr, vr = R.rnd(W), R.rnd(v)
    mag = np.abs(vr) @ np.abs(Wr).T
    if not tf32:
        return vr @ Wr.T, mag, np.zeros_like(mag)
    W32, v32 = Wr.astype(np.float32), vr.astype(np.float32)
    acc = np.zeros((v.shape[0], W.shape[0]), dtype=np.float32)
    inexact = np.zeros(acc.shape, dtype=bool)
    for c in range(W.shape[1]):
        p32 = v32[:, c:c + 1] * W32[None, :, c]
        p64 = vr[:, c:c + 1] * Wr[None, :, c]
        inexact |= np.isfinite(p64) & (p32.astype(np.float64) != p64)
        acc = acc + p32
    n = W.shape[1]
    bound = np.where(inexact, 2 * n * (U_32 * mag + 2.0 ** -148), 0.0)
    return acc.astype(np.float64), mag, bound


def node_mlp(sources, layers, tf32=True, M=None):
    """sources: arrays in input-row order, dense [B,C,M] or per sample [B,C] (M is needed only when every source is
    per sample); layers: [(W [C_out,C_in], b [C_out] or None, relu)].  Returns dict(out [B,C_out,M] float64, bound (same shape)).  tf32=False drops every rounding and is
    the exact layer chain over the concatenated input (the bound is then all zero)."""
    R = _Rules(tf32)
    sources = [np.asarray(s, dtype=np.float32) for s in sources]
    B = sources[0].shape[0]
    M = next((s.shape[2] for s in sources if s.ndim == 3), M)
    W1, b1, act1 = layers[0]
    W1 = np.asarray(W1)
    col, dense_cols, bc_cols, dense, bc = 0, [], [], [], []
    for s in sources:
        cols = list(range(col, col + s.shape[1]))
        col += s.shape[1]
        (dense_cols if s.ndim == 3 else bc_cols).extend(cols)
        (dense if s.ndim == 3 else bc).append(s)
    with np.errstate(all="ignore"):
        C1 = W1.shape[0]
        if dense:
            x = R.rnd(np.concatenate(dense, axis=1))
            z, mag, err = R.product(W1[:, dense_cols], x, np.zeros_like(x))
        else:
            z, mag, err = (np.zeros((B, C1, M)) for _ in range(3))
        terms = 2
        if bc:
            p, pmag, perr = project(W1[:, bc_cols], np.concatenate(bc, axis=1), tf32)
            z, mag, err = z + p[..., None], mag + pmag[..., None], err + perr[..., None]
            terms = 3
        y, err = R.finish(z, mag, err, b1, act1, terms)
        for W, b, act in layers[1:]:
            x, e = R.store(y, err)
            z, mag, err = R.product(W, x, e)
            y, err = R.finish(z, mag, err, b, act, 2)
    return dict(out=y, bound=np.where(np.isfinite(y), err, 0.0))
