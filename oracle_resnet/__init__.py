"""Float64 restatement of resnet.conv2d_fused and the stem (csrc/resnet.cu, DESIGN.md 4.30) with a per-output error
bound, and a float64 chain of the whole folded backbone.

conv() follows the kernel's formulation: an implicit GEMM over the zero-padded input, K = k^2 C_in columns in the
packed [C_out][k][k][C_in] order (then the fused shortcut's C2 columns), weights and input values rounded by
oracle_pointwise.tf32_round, products and sums in float64 here and float32 on the device; then the bias, the residual
and ReLU (NaN stays NaN).

The bound follows oracle_pointwise's rules: an f32 accumulation of K products in any order contributes (K + 8) U32
|W| |x| (U32 = 2^-23 covers a truncating accumulator), the two f32 additions of the bias and the residual contribute
U32 each of |W| |x| + |b| + |residual|, and ReLU is 1-Lipschitz.  The 3x3 stride-2 max-pool of values each within its
bound is within the largest bound of its window.  Where the oracle's value is not finite the bound is 0: the device
must then hold the same NaN or infinity.  Tests, smoke() and nothing else use this module.
"""
import numpy as np

from oracle_pointwise import U_32, relu, tf32_round


def _cols(x, k, stride, pad):
    """im2col of NHWC x [B,H,W,C] float64: [B,Ho,Wo,k*k*C] in (kh, kw, C) order over the zero-padded input."""
    B, H, W, C = x.shape
    xp = np.pad(x, ((0, 0), (pad, pad), (pad, pad), (0, 0)))
    win = np.lib.stride_tricks.sliding_window_view(xp, (k, k), axis=(1, 2))[:, ::stride, ::stride]   # [B,Ho,Wo,C,k,k]
    return np.ascontiguousarray(win.transpose(0, 1, 2, 4, 5, 3)).reshape(win.shape[:3] + (k * k * C,))


def conv(x, W, b, stride, residual=None, relu_=True, shortcut=None, nchw_input=False, tf32=True):
    """x: NHWC [B,H,W,C] (or NCHW [B,C,H,W] with nchw_input) float32; W [C_out,k,k,C] and b [C_out] float32 (the
    packed bias: with a shortcut already b2 + bd); padding k // 2; residual NHWC [B,Ho,Wo,C_out] or None; shortcut =
    (x2 NHWC [B,H2,W2,C2], Wd [C_out,1,1,C2], stride2) or None.  Returns dict(out [B,Ho,Wo,C_out] float64, bound).
    tf32=False drops the rounding (the bound is then all zero)."""
    rnd = (lambda a: tf32_round(a).astype(np.float64)) if tf32 else (lambda a: np.asarray(a, np.float64))
    u32 = U_32 if tf32 else 0.0
    x = np.asarray(x, np.float32)
    if nchw_input:
        x = x.transpose(0, 2, 3, 1)
    k = W.shape[1]
    cols = _cols(rnd(x), k, stride, k // 2)
    Wm = rnd(W).reshape(W.shape[0], -1)
    if shortcut is not None:
        x2, Wd, s2 = shortcut
        cols = np.concatenate((cols, rnd(np.asarray(x2, np.float32))[:, ::s2, ::s2]), axis=3)
        Wm = np.concatenate((Wm, rnd(Wd).reshape(Wd.shape[0], -1)), axis=1)
    K = cols.shape[3]
    with np.errstate(all="ignore"):
        z = cols @ Wm.T
        mag = np.abs(cols) @ np.abs(Wm).T
        bb = np.asarray(b, np.float64)
        z, mag = z + bb, mag + np.abs(bb)
        if residual is not None:
            r = np.asarray(residual, np.float64)
            z, mag = z + r, mag + np.abs(r)
        err = (K + 8) * u32 * mag + 2 * u32 * mag
        y = relu(z) if relu_ else z
    return dict(out=y, bound=np.where(np.isfinite(y), err, 0.0))


def max_pool(y, e):
    """torch.nn.MaxPool2d(3, 2, 1) over NHWC y [B,H,W,C] (NaN wins) and the largest bound of each window's finite
    members."""
    B, H, W, C = y.shape
    yp = np.pad(y, ((0, 0), (1, 1), (1, 1), (0, 0)), constant_values=-np.inf)
    ep = np.pad(e, ((0, 0), (1, 1), (1, 1), (0, 0)))
    wy = np.lib.stride_tricks.sliding_window_view(yp, (3, 3), axis=(1, 2))[:, ::2, ::2].reshape(
        B, (H - 1) // 2 + 1, (W - 1) // 2 + 1, C, 9)
    we = np.lib.stride_tricks.sliding_window_view(ep, (3, 3), axis=(1, 2))[:, ::2, ::2].reshape(wy.shape)
    with np.errstate(invalid="ignore"):
        nan = np.isnan(wy).any(axis=4)
        v = np.where(nan, np.nan, np.max(np.where(np.isnan(wy), -np.inf, wy), axis=4))
    return v, np.where(np.isfinite(v), np.max(np.where(np.isfinite(wy), we, 0.0), axis=4), 0.0)


def stem(img, W, b, tf32=True):
    """conv1 + bn1 + relu (folded) + the max-pool from the [B,3,H,W] image: dict(out NHWC float64, bound)."""
    r = conv(img, W, b, 2, nchw_input=True, tf32=tf32)
    out, bound = max_pool(r["out"], r["bound"])
    return dict(out=out, bound=bound)


def backbone(folded, img):
    """The whole backbone in float64 from network.fold_resnet34's dict (torch tensors, any device; use
    dtype=torch.float64 for a reference) with torch.nn.functional's convolution, bias, residual, ReLU and max-pool:
    img [B,3,H,W] -> (s16 [B,256,P16], s32 [B,512,P32], img_global [B,512]) in the dtype of `folded`."""
    import torch
    import torch.nn.functional as F

    def cv(x, name, stride, pad):
        W, bias = folded[name]
        return F.conv2d(x, W.permute(0, 3, 1, 2), bias, stride=stride, padding=pad)

    x = F.max_pool2d(F.relu(cv(img.to(folded["conv1"][0].dtype), "conv1", 2, 3)), 3, 2, 1)
    s16 = None
    for s in range(1, 5):
        j = 0
        while f"layer{s}.{j}.conv1" in folded:
            stride = 2 if s > 1 and j == 0 else 1
            y = F.relu(cv(x, f"layer{s}.{j}.conv1", stride, 1))
            down = f"layer{s}.{j}.downsample"
            x = F.relu(cv(y, f"layer{s}.{j}.conv2", 1, 1) + (cv(x, down, stride, 0) if down in folded else x))
            j += 1
        if s == 3:
            s16 = x
    B = img.shape[0]
    return s16.reshape(B, 256, -1), x.reshape(B, 512, -1), torch.mean(x.reshape(B, 512, -1), dim=2)
