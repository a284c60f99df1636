"""Classifier training targets and losses (DESIGN.md 4.15) without a GPU: the fp64 numpy oracle against a torch
restatement of the reference's formulation (models/multimodal_classifier.py:135-191 with kornia's focal loss,
models/focal_loss.py:55-112), its analytic gradients against autograd, and the host-side argument checks of
classifier.classifier_loss and of the C ABI."""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle_cls
from deepi2p_b200 import classifier


def formulation(coarse, fine, pc, P, K, H, W, fine_scale=32, coarse_loss_alpha=50.0, focal_alpha=0.5, focal_gamma=2,
                eps=1e-6, dtype=torch.float64):
    """The reference's arithmetic in torch, in `dtype`: projection by two matmuls, the label rule, kornia's focal loss
    (softmax + eps, one-hot + eps), the cross-entropy of the inside rows, torch.max predictions and the accuracies.
    The inside rows are selected with a boolean mask instead of the reference's sort + gather (the same rows).  With no
    inside point the fine loss is returned as 0 (the reference raises there)."""
    B, _, N = coarse.shape
    dev = coarse.device
    H_f, W_f = classifier.fine_grid(H, W, fine_scale)
    pc_homo = torch.cat((pc.to(dtype), torch.ones((B, 1, N), dtype=dtype, device=dev)), dim=1)
    P_pc = torch.matmul(P[:, :3].to(dtype), pc_homo)
    KP = torch.matmul(K.to(dtype), P_pc)
    pxpy = KP[:, 0:2] / KP[:, 2:3]
    inside = ((pxpy[:, 0] >= 0) & (pxpy[:, 0] <= W - 1) & (pxpy[:, 1] >= 0) & (pxpy[:, 1] <= H - 1)
              & (KP[:, 2] > 0.1))
    cell = torch.floor(pxpy / fine_scale).to(torch.long)
    fine_idx = cell[:, 0] + cell[:, 1] * W_f
    coarse_labels = inside.to(torch.long)
    # kornia focal_loss(reduction='mean') with the FocalLoss module's eps
    soft = F.softmax(coarse.to(dtype), dim=1) + eps
    one_hot = torch.zeros_like(soft).scatter_(1, coarse_labels.unsqueeze(1), 1.0) + eps
    focal = -focal_alpha * torch.pow(-soft + 1.0, focal_gamma) * torch.log(soft)
    coarse_loss = torch.mean(torch.sum(one_hot * focal, dim=1)) * coarse_loss_alpha
    _, coarse_pred = torch.max(coarse, dim=1)
    out = dict(coarse=coarse_loss, loss=coarse_loss, coarse_labels=coarse_labels, coarse_predictions=coarse_pred,
               coarse_accuracy=torch.sum(torch.eq(coarse_labels, coarse_pred).to(dtype)) / (B * N))
    if fine is None:
        return out
    L = fine.shape[1]
    mask = inside.reshape(B * N)
    rows = fine.to(dtype).permute(0, 2, 1).reshape(B * N, L)[mask]
    lab = fine_idx.reshape(B * N)[mask]
    fine_loss = F.cross_entropy(rows, lab) if rows.shape[0] else torch.zeros((), dtype=dtype, device=dev)
    _, fine_pred = torch.max(fine, dim=1)
    out.update(fine=fine_loss, loss=coarse_loss + fine_loss, fine_labels=torch.where(inside, fine_idx, -1),
               fine_predictions=fine_pred,
               fine_accuracy=torch.sum(torch.eq(lab, torch.max(rows, dim=1)[1]).to(dtype)) / rows.shape[0])
    return out


KITTI_K = np.array([[380.0, 0.0, 256.0], [0.0, 380.0, 80.0], [0.0, 0.0, 1.0]])


def make_case(seed, B, N, H=160, W=512, fine_scale=32, with_fine=True, scale=3.0):
    """Points in front of, beside and behind a camera looking down +z; logits ~ N(0, scale)."""
    rng = np.random.default_rng(seed)
    pc = np.stack([rng.uniform(-30, 30, (B, N)), rng.uniform(-6, 6, (B, N)), rng.uniform(-20, 60, (B, N))],
                  axis=1).astype(np.float32)
    P = np.tile(np.eye(4), (B, 1, 1))
    for b in range(B):
        a = rng.uniform(-0.2, 0.2)
        P[b, :3, :3] = [[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]]
        P[b, :3, 3] = rng.uniform(-1, 1, 3)
    K = np.tile(KITTI_K * [[W / 512], [H / 160], [1]], (B, 1, 1))
    L = int(np.prod(classifier.fine_grid(H, W, fine_scale)))
    coarse = (rng.normal(0, scale, (B, 2, N))).astype(np.float32)
    fine = (rng.normal(0, scale, (B, L, N))).astype(np.float32) if with_fine else None
    return coarse, fine, pc, P, K, H, W


def torch_args(case):
    coarse, fine, pc, P, K, H, W = case
    t = lambda a: torch.from_numpy(a) if a is not None else None  # noqa: E731
    return t(coarse), t(fine), t(pc), t(P), t(K), H, W


def assert_matches_formulation(case, **kw):
    ref = formulation(*torch_args(case), **kw)
    got = oracle_cls.classifier_loss(*case, **kw)
    np.testing.assert_array_equal(got["coarse_labels"], ref["coarse_labels"].numpy())
    np.testing.assert_array_equal(got["coarse_predictions"], ref["coarse_predictions"].numpy())
    for k in ("coarse", "loss", "coarse_accuracy") + (("fine", "fine_accuracy") if case[1] is not None else ()):
        want = float(ref[k])
        assert (math.isnan(got[k]) and math.isnan(want)) or abs(got[k] - want) <= 1e-12 * max(abs(want), 1e-300), k
    if case[1] is not None:
        np.testing.assert_array_equal(got["fine_labels"], ref["fine_labels"].numpy())
        np.testing.assert_array_equal(got["fine_predictions"], ref["fine_predictions"].numpy())
    return got


@pytest.mark.parametrize("seed,B,N,H,W", [(0, 2, 3000, 160, 512), (1, 3, 800, 384, 640), (2, 1, 2000, 160, 320)])
def test_oracle_matches_formulation_random(seed, B, N, H, W):
    got = assert_matches_formulation(make_case(seed, B, N, H, W))
    assert 0 < got["n_inside"].sum() < B * N
    assert_matches_formulation(make_case(seed, B, N, H, W, with_fine=False))


def adversarial_case():
    """Ties, +-1e4 logits, an all-outside sample (sample 1 looks away) and an exactly-representable boundary set."""
    coarse, fine, pc, P, K, H, W = make_case(7, 3, 600)
    coarse[:, :, :50] = 0.25                             # coarse ties
    fine[:, :, 50:100] = -1.5                            # whole fine rows tied
    fine[:, 3:7, 100:150] = 2.0                          # a tie at the top
    rng = np.random.default_rng(3)
    coarse[:, :, 150:300] = rng.choice([-1e4, 1e4], (3, 2, 150))
    fine[:, :, 150:300] = rng.choice([-1e4, 0.0, 1e4], (3, fine.shape[1], 150))
    P[1, :3, :3] = np.diag([1.0, 1.0, -1.0]) * [[1], [-1], [1]]     # turned around: every point behind or beside
    P[1, :3, 3] = [0.0, 0.0, -100.0]
    return coarse, fine, pc, P, K, H, W


def test_oracle_matches_formulation_adversarial():
    case = adversarial_case()
    got = assert_matches_formulation(case)
    assert got["n_inside"][1] == 0 and got["n_inside"][0] > 0
    assert got["fine_correct"][1] == 0


def test_all_outside_batch():
    coarse, fine, pc, P, K, H, W = make_case(8, 2, 500)
    P[:, 2, 3] = -1000.0                                 # everything behind the camera
    got = oracle_cls.classifier_loss(coarse, fine, pc, P, K, H, W, grads=(1.0, 0.5, 2.0))
    assert got["n_inside"].sum() == 0 and (got["fine_labels"] == -1).all()
    assert got["fine"] == 0.0 and math.isnan(got["fine_accuracy"]) and not got["grad_fine"].any()
    ref = formulation(*torch_args((coarse, fine, pc, P, K, H, W)))
    assert abs(got["coarse"] - float(ref["coarse"])) <= 1e-12 * float(ref["coarse"])
    assert got["loss"] == got["coarse"]


@pytest.mark.parametrize("gamma", [0, 1, 2, 3])
@pytest.mark.parametrize("case_name", ["random", "adversarial", "coarse_only"])
def test_oracle_gradients_match_autograd(gamma, case_name):
    if case_name == "adversarial":
        case = adversarial_case()
    else:
        case = make_case(11 + gamma, 2, 700, with_fine=case_name == "random")
    coarse, fine, pc, P, K, H, W = torch_args(case)
    grads = (0.7, -0.3, 1.9)
    c = coarse.double().requires_grad_(True)
    f = fine.double().requires_grad_(True) if fine is not None else None
    ref = formulation(c, f, pc, P, K, H, W, focal_gamma=gamma)
    total = ref["loss"] * grads[0] + ref["coarse"] * grads[1] + (ref["fine"] * grads[2] if f is not None else 0)
    total.backward()
    got = oracle_cls.classifier_loss(*case, focal_gamma=gamma, grads=grads)
    pairs = [(got["grad_coarse"], c.grad.numpy())] + ([(got["grad_fine"], f.grad.numpy())] if f is not None else [])
    for g, want in pairs:
        np.testing.assert_allclose(g, want, rtol=1e-12, atol=1e-12 * np.abs(want).max())


def test_argmax_rule_matches_torch():
    z = np.array([[[1.0, np.nan, 2.0, 2.0, -np.inf, np.inf, np.nan, 0.0],
                   [1.0, 5.0, np.nan, 2.0, -np.inf, np.inf, np.nan, -0.0],
                   [0.5, np.nan, np.nan, 1.0, -np.inf, 1.0, 3.0, 0.0]]], dtype=np.float32)
    np.testing.assert_array_equal(oracle_cls.argmax(z), torch.max(torch.from_numpy(z), dim=1)[1].numpy())


def test_labels_at_cell_lines():
    """u on a cell line belongs to the cell on its right; u = W - 1 and v = H - 1 to the last cell."""
    K = np.eye(3)[None]
    H, W = 160, 512
    u = np.array([0.0, 31.0, 32.0, 511.0, 511.0, 100.0])
    v = np.array([0.0, 0.0, 31.5, 159.0, 0.0, 64.0])
    pc = np.stack([u, v, np.ones_like(u)])[None].astype(np.float32)
    c, f = oracle_cls.labels(pc, np.eye(4)[None], K, H, W)
    np.testing.assert_array_equal(c[0], 1)
    np.testing.assert_array_equal(f[0], [0, 0, 1, 15 + 4 * 16, 15, 3 + 2 * 16])


# ---- host-side checks ------------------------------------------------------------------------------------------------

def _args(B=2, N=10, H=160, W=512, s=32, L=None):
    L = L if L is not None else int(np.prod(classifier.fine_grid(H, W, s)))
    return dict(coarse_scores=torch.zeros(B, 2, N), fine_scores=torch.zeros(B, L, N), pc=torch.zeros(B, 3, N),
                P=torch.zeros(B, 4, 4, dtype=torch.float64), K=torch.zeros(B, 3, 3), H=H, W=W, fine_scale=s)


def _with(**kw):
    a = _args()
    a.update(kw)
    return a


@pytest.mark.parametrize("kwargs,exc,match", [
    (_args(L=79), ValueError, r"L = 79 .* 5 \* 16"),
    (dict(_args(H=160, W=80, L=10), ), ValueError, "last pixel row or column"),       # round(2.5) = 2 < 79 // 32 + 1
    (_with(coarse_scores=torch.zeros(2, 2, 10, dtype=torch.float64)), RuntimeError, "coarse_scores must have dtype"),
    (_with(fine_scores=torch.zeros(2, 80, 10, dtype=torch.float16)), RuntimeError, "fine_scores must have dtype"),
    (_with(pc=torch.zeros(2, 3, 10, dtype=torch.float64)), RuntimeError, "pc must be a float32"),
    (_with(P=torch.zeros(2, 4, 4, dtype=torch.int32)), RuntimeError, "P must be"),
    (_with(K=torch.zeros(2, 3, 3, dtype=torch.float16)), RuntimeError, "K must be"),
    (_with(coarse_scores=torch.zeros(2, 3, 10)), RuntimeError, r"coarse_scores must be \[B,2,N\]"),
    (_with(coarse_scores=torch.zeros(2, 10)), RuntimeError, r"coarse_scores must be \[B,2,N\]"),
    (_with(fine_scores=torch.zeros(2, 80, 11)), RuntimeError, "fine_scores must be"),
    (_with(pc=torch.zeros(2, 2, 10)), RuntimeError, "pc must be"),
    (_with(P=torch.zeros(2, 2, 4)), RuntimeError, "P must be"),
    (_with(P=torch.zeros(3, 4, 4)), RuntimeError, "P must be"),
    (_with(K=torch.zeros(2, 4, 4)), RuntimeError, "K must be"),
    (_with(coarse_scores=torch.zeros(2, 2, 0), fine_scores=torch.zeros(2, 80, 0), pc=torch.zeros(2, 3, 0)),
     RuntimeError, "N >= 1"),
    (_with(focal_gamma=1.5), ValueError, "non-negative integer"),
    (_with(focal_gamma=-1), ValueError, "non-negative integer"),
    (_with(focal_gamma="2"), ValueError, "non-negative integer"),
    (_with(fine_scale=0), ValueError, "fine_scale > 0"),
    (_with(pc=torch.zeros(2, 3, 10, requires_grad=True)), RuntimeError, "respect to pc"),
    (_with(P=torch.zeros(2, 3, 4, dtype=torch.float64, requires_grad=True)), RuntimeError, "respect to P"),
    (_with(K=torch.zeros(2, 3, 3, requires_grad=True)), RuntimeError, "respect to K"),
    (_args(), RuntimeError, "CUDA"),
])
def test_host_side_rejection(kwargs, exc, match):
    with pytest.raises(exc, match=match):
        classifier.classifier_loss(**kwargs)


def test_valid_shapes_pass_the_host_checks():
    """Integer-valued float gamma, P [B,3,4], H = W = s (L = 1) and coarse-only reach the device check only."""
    for kw in (_with(focal_gamma=2.0), _with(P=torch.zeros(2, 3, 4)), _args(H=32, W=32, s=32),
               _with(fine_scores=None), _args(H=384, W=640), _args(H=160, W=320)):
        with pytest.raises(RuntimeError, match="CUDA"):
            classifier.classifier_loss(**kw)


def test_c_abi_validates_on_host():
    from deepi2p_b200 import _native
    lib = _native.load()
    buf = ctypes.create_string_buffer(1 << 12)
    a = ctypes.addressof(buf)

    def fwd(L=80, B=2, N=10, H_f=5, W_f=16, W=512.0, gamma=2, ws_bytes=1 << 12):
        return lib.classifier_loss_forward_f32(a, 20, a, 800, L, a, a, a, B, N, 160.0, W, 32.0, H_f, W_f, 50.0, 0.5,
                                               gamma, 1e-6, a, a, a, a, a, a, a, a, a, a, a, a, a, a, ws_bytes, None)
    assert fwd(L=79) == -22 and b"H_f * W_f" in lib.dib_last_error()
    assert fwd(L=32, W_f=2, H_f=16, W=80.0) == -22 and b"cell grid" in lib.dib_last_error()
    assert fwd(gamma=-1) == -22 and b"focal_gamma" in lib.dib_last_error()
    assert fwd(B=0) == -22 and fwd(N=0) == -22 and fwd(B=65536) == -22
    assert fwd(ws_bytes=8) == -22 and b"workspace" in lib.dib_last_error()
    assert lib.classifier_loss_backward_f32(a, -1, None, 0, 0, 1, 4, a, None, None, None, a, a, a, 50.0, 0.5, 2, 1e-6,
                                            a, None, None) == -22
    assert lib.classifier_loss_workspace_bytes(0, 10) == 0
    # per-CTA partials of 256 points: two doubles and three int32 each
    assert lib.classifier_loss_workspace_bytes(8, 20480) == 8 * 80 * 28
