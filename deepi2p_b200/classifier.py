"""The classifier's training targets and losses as one fused, differentiable op (DESIGN.md 4.15).

classifier_loss replaces the tail of MMClassifer.foraward_pass (models/multimodal_classifier.py:135-191, the
coarse-only variant :482-508): the projected coarse and fine labels, kornia's focal loss on the coarse scores, the
cross-entropy of the fine scores over the inside points, the accuracies and the predictions, with no host
synchronisation, so a training step can be captured in a CUDA graph.  The kernels are in csrc/classifier_loss.cu;
there is no CPU fallback.
"""
import math
import numbers

import torch

from . import _native


def fine_grid(H, W, fine_scale):
    """(H_f, W_f) of the fine cell grid as the reference computes them: Python's round of H / s and W / s."""
    return int(round(H / fine_scale)), int(round(W / fine_scale))


def _check_scores(t, name, C=None):
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a torch.Tensor")
    if t.dtype != torch.float32:
        raise RuntimeError(f"{name} must have dtype {torch.float32}")
    if t.dim() != 3 or (C is not None and t.shape[1] != C):
        raise RuntimeError(f"{name} must be [B,{C if C is not None else 'L'},N]")


def _check_args(coarse_scores, fine_scores, pc, P, K, H, W, fine_scale, focal_gamma):
    """Shape, dtype, value and autograd checks first (they need no device), then device placement.
    Returns (B, N, L, H_f, W_f)."""
    _check_scores(coarse_scores, "coarse_scores", 2)
    B, _, N = coarse_scores.shape
    L = H_f = W_f = 0
    if fine_scores is not None:
        _check_scores(fine_scores, "fine_scores")
        L = fine_scores.shape[1]
        if fine_scores.shape[0] != B or fine_scores.shape[2] != N:
            raise RuntimeError("fine_scores must be [B,L,N] with the B and N of coarse_scores")
    for t, name in ((pc, "pc"), (P, "P"), (K, "K")):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{name} must be a torch.Tensor")
    if pc.dtype != torch.float32 or tuple(pc.shape) != (B, 3, N):
        raise RuntimeError("pc must be a float32 [B,3,N] tensor with the B and N of coarse_scores")
    if P.dtype not in (torch.float32, torch.float64) or P.dim() != 3 or P.shape[0] != B or P.shape[2] != 4 \
            or P.shape[1] not in (3, 4):
        raise RuntimeError("P must be a float32 or float64 [B,3,4] or [B,4,4] tensor")
    if K.dtype not in (torch.float32, torch.float64) or tuple(K.shape) != (B, 3, 3):
        raise RuntimeError("K must be a float32 or float64 [B,3,3] tensor")
    if not (1 <= B <= 65535 and N >= 1 and B * N < 2 ** 31):
        raise RuntimeError(f"need 1 <= B <= 65535, N >= 1 and B * N < 2^31, got B = {B}, N = {N}")
    if isinstance(focal_gamma, bool) or not isinstance(focal_gamma, numbers.Real) \
            or float(focal_gamma) != int(focal_gamma) or focal_gamma < 0:
        raise ValueError(f"focal_gamma must be a non-negative integer, got {focal_gamma!r}")
    if not (H >= 1 and W >= 1 and fine_scale > 0):
        raise ValueError(f"need H, W >= 1 and fine_scale > 0, got H = {H}, W = {W}, fine_scale = {fine_scale}")
    if fine_scores is not None:
        H_f, W_f = fine_grid(H, W, fine_scale)
        if L != H_f * W_f:
            raise ValueError(f"fine_scores has L = {L} channels, but the {H} x {W} image in cells of {fine_scale} px "
                             f"has H_f * W_f = {H_f} * {W_f} = {H_f * W_f}")
        if math.floor((W - 1) / fine_scale) >= W_f or math.floor((H - 1) / fine_scale) >= H_f:
            raise ValueError(f"the last pixel row or column of the {H} x {W} image falls outside the {H_f} x {W_f} "
                             f"cell grid of fine_scale {fine_scale}")
    for t, name in ((pc, "pc"), (P, "P"), (K, "K")):
        if t.requires_grad:
            raise RuntimeError(f"classifier_loss has no gradient with respect to {name}: detach it")
    dev = coarse_scores.device
    for t, name in ((coarse_scores, "coarse_scores"), (fine_scores, "fine_scores"), (pc, "pc"), (P, "P"), (K, "K")):
        if t is None:
            continue
        if not t.is_cuda:
            raise RuntimeError(f"{name} must be a CUDA tensor/variable")
        if t.device != dev:
            raise RuntimeError(f"{name} must be on {dev}")
    return B, N, L, H_f, W_f


def _scores_view(t):
    """The kernels take (channel, point) strides (N, 1) with any batch stride: a channel slice of one [B,2+L,N] score
    tensor needs no copy.  Returns (tensor, batch stride)."""
    B, C, N = t.shape
    if (C > 1 and t.stride(1) != N) or (N > 1 and t.stride(2) != 1):
        t = t.contiguous()
    return t, (t.stride(0) if B > 1 else 0)


def _ptr(t):
    return t.data_ptr() if t is not None else None


class _ClassifierLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, coarse_scores, fine_scores, pc, P12, K9, cfg, extras):
        B, N, L, H, W, s, H_f, W_f, coarse_alpha, focal_alpha, gamma, eps = cfg
        lib = _native.load()
        dev = coarse_scores.device
        has_fine = fine_scores is not None
        coarse, cbs = _scores_view(coarse_scores)
        fine, fbs = _scores_view(fine_scores) if has_fine else (None, 0)
        with torch.cuda.device(dev):
            i8, i32, f32 = dict(dtype=torch.int8, device=dev), dict(dtype=torch.int32, device=dev), \
                dict(dtype=torch.float32, device=dev)
            coarse_labels, coarse_pred = torch.empty((B, N), **i8), torch.empty((B, N), **i8)
            fine_labels = torch.empty((B, N), **i32) if has_fine else None
            fine_pred = torch.empty((B, N), **i32) if has_fine else None
            lse = torch.empty((2, B, N), **f32) if has_fine else None     # row max, log of the shifted sum
            loss, coarse_loss, fine_loss = torch.empty((), **f32), torch.empty((), **f32), torch.empty((), **f32)
            accuracy = torch.empty((2,), **f32)
            n_inside, coarse_correct = torch.empty((B,), **i32), torch.empty((B,), **i32)
            fine_correct = torch.empty((B,), **i32) if has_fine else None
            n_inside_total = torch.empty((1,), **i32)
            # per-CTA partials: from torch's allocator on every call, so that a captured graph owns its own
            ws = torch.empty((max(lib.classifier_loss_workspace_bytes(B, N), 8),), dtype=torch.uint8, device=dev)
            rc = lib.classifier_loss_forward_f32(
                coarse.data_ptr(), cbs, _ptr(fine), fbs, L, pc.data_ptr(), P12.data_ptr(), K9.data_ptr(), B, N,
                float(H), float(W), float(s), H_f, W_f, float(coarse_alpha), float(focal_alpha), gamma, float(eps),
                coarse_labels.data_ptr(), _ptr(fine_labels), coarse_pred.data_ptr(), _ptr(fine_pred), _ptr(lse),
                loss.data_ptr(), coarse_loss.data_ptr(), fine_loss.data_ptr(), accuracy.data_ptr(),
                n_inside.data_ptr(), coarse_correct.data_ptr(), _ptr(fine_correct), n_inside_total.data_ptr(),
                ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
        _native.check(rc, "classifier_loss_forward_f32")
        extras.update(coarse_labels=coarse_labels, fine_labels=fine_labels, coarse_predictions=coarse_pred,
                      fine_predictions=fine_pred, n_inside=n_inside, coarse_accuracy=accuracy[0],
                      fine_accuracy=accuracy[1] if has_fine else None, coarse_correct=coarse_correct,
                      fine_correct=fine_correct)
        ctx.save_for_backward(coarse, fine, coarse_labels, fine_labels, lse, n_inside_total)
        ctx.cfg = cfg
        ctx.strides = (cbs, fbs)
        return loss, coarse_loss, fine_loss

    @staticmethod
    def backward(ctx, g_loss, g_coarse, g_fine):
        want_c, want_f = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if not (want_c or want_f):
            return None, None, None, None, None, None, None
        coarse, fine, coarse_labels, fine_labels, lse, n_inside_total = ctx.saved_tensors
        B, N, L, _, _, _, _, _, coarse_alpha, focal_alpha, gamma, eps = ctx.cfg
        cbs, fbs = ctx.strides
        dev = coarse.device
        g_loss, g_coarse, g_fine = (g.float().contiguous() for g in (g_loss, g_coarse, g_fine))
        lib = _native.load()
        with torch.cuda.device(dev):
            gc = torch.empty((B, 2, N), dtype=torch.float32, device=dev) if want_c else None
            gf = torch.empty((B, L, N), dtype=torch.float32, device=dev) if want_f else None
            rc = lib.classifier_loss_backward_f32(
                coarse.data_ptr(), cbs, _ptr(fine), fbs, L, B, N, coarse_labels.data_ptr(), _ptr(fine_labels),
                _ptr(lse), n_inside_total.data_ptr(), g_loss.data_ptr(), g_coarse.data_ptr(), g_fine.data_ptr(),
                float(coarse_alpha), float(focal_alpha), gamma, float(eps), _ptr(gc), _ptr(gf),
                torch.cuda.current_stream().cuda_stream)
        _native.check(rc, "classifier_loss_backward_f32")
        return gc, gf, None, None, None, None, None


def classifier_loss(coarse_scores, fine_scores, pc, P, K, H, W, fine_scale=32, coarse_loss_alpha=50.0,
                    focal_alpha=0.5, focal_gamma=2, eps=1e-6):
    """Labels, losses, accuracies and predictions of one classifier step (models/multimodal_classifier.py:135-191;
    with fine_scores=None the coarse-only classifier, :482-508).

    coarse_scores [B,2,N], fine_scores [B,L,N] or None, pc [B,3,N], all float32; P [B,3,4] or [B,4,4] and K [B,3,3]
    float32 or float64 (read as fp64); all on one CUDA device.  Scores with (channel, point) strides (N, 1), such as
    the channel slices of the network's [B,2+L,N] output, are read without a copy.  L must be H_f * W_f with
    H_f = round(H / fine_scale), W_f = round(W / fine_scale).

    Returns a dict:
      loss, coarse, fine      0-dim float32, differentiable with respect to the scores (loss = coarse + fine).
                              coarse: the mean over all B*N points of kornia's focal loss as the reference calls it
                              (softmax + eps, one-hot + eps), times coarse_loss_alpha; fine: the mean cross-entropy
                              over the inside points, 0 with a zero gradient when there is none.  For coarse-only,
                              fine is None.
      coarse_labels           int8 [B,N]: 1 inside the image (the rule of frustum.inside_mask_batch, bit for bit).
      fine_labels             int32 [B,N]: floor(u/s) + floor(v/s) * W_f inside, -1 outside.
      coarse_predictions      int8 [B,N] and fine_predictions int32 [B,N]: torch.max's argmax over the classes
                              (first maximal index, NaN maximal), for every point; register_batch and pnp_ransac_batch
                              take them as they are.
      n_inside, coarse_correct, fine_correct   int32 [B] per sample (fine_correct counts inside points).
      coarse_accuracy, fine_accuracy           0-dim float32 from the integer counts (fine: NaN with no inside point).
    The fine_* entries are None for coarse-only.  No host synchronisation: the call is capturable in a CUDA graph.
    pc, P and K must not require grad."""
    B, N, L, H_f, W_f = _check_args(coarse_scores, fine_scores, pc, P, K, H, W, fine_scale, focal_gamma)
    P12 = P[:, :3, :].to(torch.float64).reshape(B, 12).contiguous()
    K9 = K.to(torch.float64).reshape(B, 9).contiguous()
    pc = pc.contiguous()
    cfg = (B, N, L, H, W, fine_scale, H_f, W_f, coarse_loss_alpha, focal_alpha, int(focal_gamma), eps)
    extras = {}
    loss, coarse, fine = _ClassifierLoss.apply(coarse_scores, fine_scores, pc, P12, K9, cfg, extras)
    return dict(loss=loss, coarse=coarse, fine=fine if fine_scores is not None else None, **extras)
