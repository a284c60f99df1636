"""numpy fp64 oracle of the classifier's training targets and losses -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and the benchmark scripts may import this package; deepi2p_b200.classifier never
does.  It restates DESIGN.md 4.15: the label rule (the projection evaluated in fp64 from the float32 coordinates in
the order of csrc/project.cuh; numpy never contracts a multiply-add, so the labels are the kernel's bit for bit), the
focal loss with both eps terms and the inside-only cross-entropy in fp64, their analytic gradients, torch.max's argmax
rule and the accuracies from integer counts.
"""
import math

import numpy as np


def project(pc, P, K, H, W):
    """u, v [B,N] f64 and the inside mask [B,N] bool.  pc [B,3,N] f32, P [B,3|4,4], K [B,3,3]."""
    x, y, z = (np.asarray(pc, dtype=np.float32).astype(np.float64)[:, i] for i in range(3))
    P = np.asarray(P, dtype=np.float64)
    K = np.asarray(K, dtype=np.float64)
    c = lambda M, i, j: M[:, i, j][:, None]  # noqa: E731
    X = c(P, 0, 0) * x + c(P, 0, 1) * y + c(P, 0, 2) * z + c(P, 0, 3)
    Y = c(P, 1, 0) * x + c(P, 1, 1) * y + c(P, 1, 2) * z + c(P, 1, 3)
    Z = c(P, 2, 0) * x + c(P, 2, 1) * y + c(P, 2, 2) * z + c(P, 2, 3)
    kx = c(K, 0, 0) * X + c(K, 0, 1) * Y + c(K, 0, 2) * Z
    ky = c(K, 1, 0) * X + c(K, 1, 1) * Y + c(K, 1, 2) * Z
    kz = c(K, 2, 0) * X + c(K, 2, 1) * Y + c(K, 2, 2) * Z
    with np.errstate(divide="ignore", invalid="ignore"):
        u, v = kx / kz, ky / kz
        inside = (u >= 0.0) & (u <= W - 1.0) & (v >= 0.0) & (v <= H - 1.0) & (Z > 0.1)
    return u, v, inside


def labels(pc, P, K, H, W, fine_scale=32):
    """coarse int8 [B,N] (1 inside), fine int32 [B,N] (floor(u/s) + floor(v/s) W_f inside, -1 outside)."""
    u, v, inside = project(pc, P, K, H, W)
    W_f = int(round(W / fine_scale))
    with np.errstate(invalid="ignore"):
        fu = np.floor(np.where(inside, u, 0.0) / fine_scale)
        fv = np.floor(np.where(inside, v, 0.0) / fine_scale)
    fine = np.where(inside, fu + fv * W_f, -1).astype(np.int32)
    return inside.astype(np.int8), fine


def argmax(z, axis=1):
    """torch.max's index: the first maximal entry, a NaN counting as maximal (the first NaN wins)."""
    z = np.asarray(z)
    nan = np.isnan(z)
    first_nan = np.argmax(nan, axis=axis)
    best = np.argmax(np.where(nan, -np.inf, z), axis=axis)
    # a row of -inf only: np.argmax of all -inf is 0, as torch's
    return np.where(nan.any(axis=axis), first_nan, best)


def softmax(z, axis=1):
    m = np.max(z, axis=axis, keepdims=True)
    e = np.exp(z - m)
    return e / np.sum(e, axis=axis, keepdims=True)


def focal(z, label, alpha=0.5, gamma=2, eps=1e-6):
    """kornia's focal loss as the reference calls it, per point, and its gradient with respect to the logits.
    z [B,C,N] f64, label [B,N] in [0, C).  p = softmax(z) + eps, f_c = -alpha (1 - p_c)^gamma log p_c,
    loss = sum_c (onehot_c + eps) f_c."""
    z = np.asarray(z, dtype=np.float64)
    s = softmax(z)
    p = s + eps
    q = 1.0 - p
    w = (np.arange(z.shape[1])[None, :, None] == np.asarray(label)[:, None, :]).astype(np.float64) + eps
    lg = np.log(p)
    qg = q ** gamma
    loss = np.sum(w * (-alpha * qg * lg), axis=1)
    dp = alpha * (gamma * q ** (gamma - 1) * lg - qg / p) if gamma > 0 else -alpha / p
    a = w * dp                                                   # d loss / d s_c
    dz = s * (a - np.sum(a * s, axis=1, keepdims=True))
    return loss, dz


def cross_entropy(z, label):
    """-log_softmax(z)[label] per point and its gradient softmax - onehot; label [B,N], -1 = not counted (0, 0)."""
    z = np.asarray(z, dtype=np.float64)
    lab = np.asarray(label)
    m = np.max(z, axis=1, keepdims=True)
    lse = m[:, 0] + np.log(np.sum(np.exp(z - m), axis=1))
    safe = np.where(lab >= 0, lab, 0)
    zl = np.take_along_axis(z, safe[:, None, :], axis=1)[:, 0]
    inside = lab >= 0
    ce = np.where(inside, lse - zl, 0.0)
    g = np.exp(z - lse[:, None]) - (np.arange(z.shape[1])[None, :, None] == safe[:, None, :])
    return ce, np.where(inside[:, None], g, 0.0)


def classifier_loss(coarse, fine, pc, P, K, H, W, fine_scale=32, coarse_loss_alpha=50.0, focal_alpha=0.5,
                    focal_gamma=2, eps=1e-6, grads=(1.0, 0.0, 0.0)):
    """Every output of deepi2p_b200.classifier.classifier_loss in fp64, plus grad_coarse [B,2,N] and grad_fine
    [B,L,N] for the upstream gradients grads = (g_loss, g_coarse, g_fine)."""
    coarse = np.asarray(coarse, dtype=np.float32).astype(np.float64)
    B, _, N = coarse.shape
    c_lab, f_lab = labels(pc, P, K, H, W, fine_scale)
    fl, dz_c = focal(coarse, c_lab.astype(np.int64), focal_alpha, focal_gamma, eps)
    coarse_loss = coarse_loss_alpha * math.fsum(fl.ravel()) / (B * N)
    c_pred = argmax(coarse).astype(np.int8)
    c_ok = (c_pred == c_lab).sum(axis=1)
    g_loss, g_coarse, g_fine = grads
    out = dict(coarse=coarse_loss, coarse_labels=c_lab, coarse_predictions=c_pred, coarse_correct=c_ok.astype(np.int32),
               n_inside=c_lab.astype(np.int64).sum(axis=1).astype(np.int32),
               coarse_accuracy=c_ok.sum() / (B * N),
               grad_coarse=dz_c * ((g_loss + g_coarse) * coarse_loss_alpha / (B * N)))
    if fine is None:
        out.update(loss=coarse_loss, fine=None)
        return out
    fine = np.asarray(fine, dtype=np.float32).astype(np.float64)
    ce, g_ce = cross_entropy(fine, f_lab)
    n_in = int((f_lab >= 0).sum())
    fine_loss = math.fsum(ce.ravel()) / n_in if n_in else 0.0
    f_pred = argmax(fine).astype(np.int32)
    f_ok = ((f_pred == f_lab) & (f_lab >= 0)).sum(axis=1)
    out.update(loss=coarse_loss + fine_loss, fine=fine_loss, fine_labels=f_lab, fine_predictions=f_pred,
               fine_correct=f_ok.astype(np.int32), fine_accuracy=f_ok.sum() / n_in if n_in else float("nan"),
               grad_fine=g_ce * ((g_loss + g_fine) / n_in) if n_in else np.zeros_like(fine))
    return out
