"""Classifier training targets and losses on the H100 (DESIGN.md 4.15): labels against inside_mask_batch, the oracle
and exact rational evaluation; predictions against torch.max; losses and gradients against the fp64 oracle and fp64
autograd of the reference's formulation; determinism, strided score slices, no host synchronisation, CUDA-graph
capture, a conv head trained one step, and the predictions fed to the registration entry points."""
from fractions import Fraction

import numpy as np
import pytest
import torch

import oracle_cls
from deepi2p_b200 import classifier, frustum, pnp, synthetic as syn
from test_classifier_loss_cpu import adversarial_case, formulation, make_case

pytestmark = pytest.mark.gpu

CASES = {  # (B, N, H, W, fine_scale, with_fine)
    "kitti": (8, 20480, 160, 512, 32, True),
    "oxford": (8, 20480, 384, 640, 32, True),
    "nuscenes": (12, 20480, 160, 320, 32, True),
    "B1": (1, 3000, 160, 512, 32, True),
    "N1": (2, 1, 160, 512, 32, True),
    "N20479": (2, 20479, 160, 512, 32, True),
    "L1": (3, 5000, 32, 32, 32, True),
    "coarse_only": (8, 20480, 160, 512, 32, False),
}
GRADS = (0.75, -0.5, 1.5)


def to_dev(case, dev, requires_grad=False):
    coarse, fine, pc, P, K, H, W = case
    t = lambda a: torch.from_numpy(a).to(dev) if a is not None else None  # noqa: E731
    c, f = t(coarse), t(fine)
    if requires_grad:
        c.requires_grad_(True)
        if f is not None:
            f.requires_grad_(True)
    return c, f, t(pc), t(P), t(K), H, W


def run(case, dev, grads=GRADS, **kw):
    c, f, pc, P, K, H, W = to_dev(case, dev, requires_grad=True)
    out = classifier.classifier_loss(c, f, pc, P, K, H, W, **kw)
    outs = [out["loss"], out["coarse"]] + ([out["fine"]] if f is not None else [])
    torch.autograd.backward(outs, [torch.tensor(g, device=dev) for g in grads[:len(outs)]])
    return out, c.grad, (f.grad if f is not None else None)


def grad_ok(got, want):
    got = got.detach().cpu().numpy().astype(np.float64)
    tol = 1e-5 * np.abs(want) + 1e-6 * np.abs(want).max()
    bad = np.abs(got - want) > tol
    assert not bad.any(), (bad.sum(), np.abs(got - want).max())


def rel_ok(got, want, rtol=1e-6):
    assert abs(float(got) - want) <= rtol * abs(want) + 1e-30, (float(got), want)


@pytest.mark.parametrize("name", list(CASES))
def test_against_oracle(cuda, name):
    B, N, H, W, s, with_fine = CASES[name]
    case = make_case(list(CASES).index(name), B, N, H, W, s, with_fine=with_fine)
    out, gc, gf = run(case, cuda, fine_scale=s)
    ref = oracle_cls.classifier_loss(*case, fine_scale=s, grads=GRADS)
    np.testing.assert_array_equal(out["coarse_labels"].cpu().numpy(), ref["coarse_labels"])
    np.testing.assert_array_equal(out["coarse_predictions"].cpu().numpy(), ref["coarse_predictions"])
    np.testing.assert_array_equal(out["n_inside"].cpu().numpy(), ref["n_inside"])
    np.testing.assert_array_equal(out["coarse_correct"].cpu().numpy(), ref["coarse_correct"])
    assert out["coarse_accuracy"].item() == np.float32(ref["coarse_accuracy"])
    rel_ok(out["coarse"], ref["coarse"])
    rel_ok(out["loss"], ref["loss"])
    assert out["loss"].item() == np.float32(out["coarse"].item() + (out["fine"].item() if with_fine else 0.0))
    grad_ok(gc, ref["grad_coarse"])
    assert out["coarse_labels"].dtype == torch.int8 and out["coarse_predictions"].dtype == torch.int8
    if not with_fine:
        assert out["fine"] is None and out["fine_labels"] is None and gf is None
        return
    np.testing.assert_array_equal(out["fine_labels"].cpu().numpy(), ref["fine_labels"])
    np.testing.assert_array_equal(out["fine_predictions"].cpu().numpy(), ref["fine_predictions"])
    np.testing.assert_array_equal(out["fine_correct"].cpu().numpy(), ref["fine_correct"])
    if ref["n_inside"].sum():
        rel_ok(out["fine"], ref["fine"])
        assert out["fine_accuracy"].item() == np.float32(ref["fine_accuracy"])
    assert out["fine_labels"].dtype == torch.int32 and out["fine_predictions"].dtype == torch.int32
    grad_ok(gf, ref["grad_fine"])
    print("%s: %d of %d points inside" % (name, int(ref["n_inside"].sum()), B * N))


def test_adversarial_against_oracle(cuda):
    """Ties, +-1e4 logits and a sample with no inside point."""
    case = adversarial_case()
    out, gc, gf = run(case, cuda)
    ref = oracle_cls.classifier_loss(*case, grads=GRADS)
    for k in ("coarse_labels", "fine_labels", "coarse_predictions", "fine_predictions", "n_inside", "fine_correct"):
        np.testing.assert_array_equal(out[k].cpu().numpy(), ref[k], err_msg=k)
    assert out["n_inside"][1].item() == 0
    for k in ("loss", "coarse", "fine"):
        rel_ok(out[k], ref[k])
    grad_ok(gc, ref["grad_coarse"])
    grad_ok(gf, ref["grad_fine"])


def test_all_outside_batch(cuda):
    case = make_case(8, 2, 500)
    case[3][:, 2, 3] = -1000.0                            # everything behind the camera
    out, gc, gf = run(case, cuda)
    assert out["n_inside"].sum().item() == 0 and (out["fine_labels"] == -1).all()
    assert out["fine"].item() == 0.0 and torch.isnan(out["fine_accuracy"]) and not gf.any()
    ref = oracle_cls.classifier_loss(*case, grads=GRADS)
    rel_ok(out["coarse"], ref["coarse"])
    grad_ok(gc, ref["grad_coarse"])


def test_gradients_match_fp64_autograd(cuda):
    for gamma in (0, 2, 3):
        case = make_case(21 + gamma, 2, 4096)
        out, gc, gf = run(case, cuda, focal_gamma=gamma)
        c, f, pc, P, K, H, W = to_dev(case, cuda)
        c, f = c.double().requires_grad_(True), f.double().requires_grad_(True)
        ref = formulation(c, f, pc, P, K, H, W, focal_gamma=gamma)
        (ref["loss"] * GRADS[0] + ref["coarse"] * GRADS[1] + ref["fine"] * GRADS[2]).backward()
        grad_ok(gc, c.grad.cpu().numpy())
        grad_ok(gf, f.grad.cpu().numpy())


def test_coarse_labels_equal_inside_mask_batch(cuda):
    from test_metrics_gpu import EXACT_H, EXACT_K, EXACT_W, exact_boundary_cases
    xyz, P, want = exact_boundary_cases()                 # u = 0, u = W-1, v = 0, v = H-1, Z = 0.1 and one ulp off
    S = len(want)
    pc = torch.from_numpy(np.ascontiguousarray(xyz)).to(cuda)
    Kb = np.tile(EXACT_K, (S, 1, 1))
    L = int(np.prod(classifier.fine_grid(EXACT_H, EXACT_W, 32)))
    out = classifier.classifier_loss(torch.zeros(S, 2, 1, device=cuda), torch.zeros(S, L, 1, device=cuda), pc,
                                     torch.from_numpy(P).to(cuda), torch.from_numpy(Kb).to(cuda), EXACT_H, EXACT_W)
    np.testing.assert_array_equal(out["coarse_labels"][:, 0].cpu().numpy(), want)
    for seed in (41, 42):
        shape = "kitti" if seed == 41 else "oxford"
        smps = [syn.make_sample(seed + 10 * b, 4096, shape=shape) for b in range(3)]
        pc = torch.from_numpy(np.stack([m["points"] for m in smps])).to(cuda)
        Pb = torch.from_numpy(np.stack([m["P_gt"] for m in smps])).to(cuda)
        K, H, W = smps[0]["K"], smps[0]["H"], smps[0]["W"]
        mask = frustum.inside_mask_batch(pc, None, Pb, K, H, W)
        L = int(np.prod(classifier.fine_grid(H, W, 32)))
        out = classifier.classifier_loss(torch.zeros(3, 2, 4096, device=cuda), torch.zeros(3, L, 4096, device=cuda),
                                         pc, Pb, torch.from_numpy(np.tile(K, (3, 1, 1))).to(cuda), H, W)
        assert torch.equal(out["coarse_labels"], mask)


def exact_fine(x, y, z, P, K, W_f, s=32):
    """Exact label and the distance of (u, v) to the nearest cell line, or None outside."""
    P = [[Fraction(float(v)) for v in row] for row in np.asarray(P, dtype=np.float64)[:3]]
    K = [[Fraction(float(v)) for v in row] for row in np.asarray(K, dtype=np.float64)]
    x, y, z = Fraction(float(x)), Fraction(float(y)), Fraction(float(z))
    c = [P[i][0] * x + P[i][1] * y + P[i][2] * z + P[i][3] for i in range(3)]
    k = [K[i][0] * c[0] + K[i][1] * c[1] + K[i][2] * c[2] for i in range(3)]
    u, v = k[0] / k[2], k[1] / k[2]
    fu, fv = u // s, v // s
    dist = min(u - fu * s, (fu + 1) * s - u, v - fv * s, (fv + 1) * s - v)
    return int(fu + fv * W_f), float(dist)


def test_fine_labels_exact(cuda):
    """Cell lines u = 32k and v = 32j exactly (cameras with K = diag(1, 1, 1)), the last column and row, and random
    points against exact rational evaluation away from the cell lines."""
    H, W = 160, 512
    us = [0.0, 31.0, 32.0, 64.0, 480.0, 511.0, 255.5]
    vs = [0.0, 32.0, 96.0, 128.0, 159.0, 31.75]
    uu, vv = np.meshgrid(us, vs)
    pts = np.stack([uu.ravel(), vv.ravel(), np.ones(uu.size)]).astype(np.float32)[None]
    n = pts.shape[2]
    out = classifier.classifier_loss(torch.zeros(1, 2, n, device=cuda), torch.zeros(1, 80, n, device=cuda),
                                     torch.from_numpy(pts).to(cuda), torch.eye(4, device=cuda)[None],
                                     torch.eye(3, device=cuda)[None], H, W)
    want = [int(u // 32) + int(v // 32) * 16 for u, v in zip(uu.ravel(), vv.ravel())]
    np.testing.assert_array_equal(out["fine_labels"][0].cpu().numpy(), want)
    assert (out["coarse_labels"] == 1).all()
    case = make_case(5, 1, 4096)
    c, f, pc, P, K, H, W = to_dev(case, cuda)
    got = classifier.classifier_loss(c, f, pc, P, K, H, W)["fine_labels"][0].cpu().numpy()
    near = 0
    for i in np.nonzero(got >= 0)[0]:
        lab, dist = exact_fine(*case[2][0, :, i], case[3][0], case[4][0], 16)
        if dist <= 1e-9:
            near += 1
            continue
        assert got[i] == lab, i
    assert near <= 2 and (got >= 0).sum() > 500


def test_fp32_formulation_disagrees_only_at_boundaries(cuda):
    """The reference computes the labels in fp32: a point may switch label only within fp32 rounding of the image
    border, a cell line or Z = 0.1."""
    case = make_case(9, *CASES["kitti"][:4])
    c, f, pc, P, K, H, W = to_dev(case, cuda)
    got = classifier.classifier_loss(c, f, pc, P, K, H, W)
    ref = formulation(c, f, pc, P.float(), K.float(), H, W, dtype=torch.float32)
    cl = got["coarse_labels"].long() != ref["coarse_labels"]
    fl = got["fine_labels"].long() != ref["fine_labels"]
    bad = (cl | fl).cpu().numpy()
    u, v, _ = oracle_cls.project(case[2], case[3], case[4], H, W)
    print("fp32 formulation: %d coarse and %d fine label disagreements of %d points"
          % (int(cl.sum()), int(fl.sum()), bad.size))
    for b, n in zip(*np.nonzero(bad)):
        du = min(abs(u[b, n] - 32 * round(u[b, n] / 32)), abs(u[b, n] - (W - 1)))
        dv = min(abs(v[b, n] - 32 * round(v[b, n] / 32)), abs(v[b, n] - (H - 1)))
        z = case[3][b, 2, :3] @ case[2][b, :, n].astype(np.float64) + case[3][b, 2, 3]
        assert min(du, dv) <= 2e-3 or abs(z - 0.1) <= 1e-5, (b, n, u[b, n], v[b, n], z)
    assert bad.sum() <= 1e-3 * bad.size


def test_predictions_follow_torch_max(cuda):
    B, N, L = 2, 4096, 80
    g = torch.Generator(device=cuda).manual_seed(3)
    c = torch.randint(-2, 3, (B, 2, N), device=cuda, generator=g).float()          # many ties
    f = torch.randint(-2, 3, (B, L, N), device=cuda, generator=g).float()
    special = torch.tensor([float("nan"), float("inf"), -float("inf")], device=cuda)
    pick = torch.rand((B, 2, N), device=cuda, generator=g) < 0.1
    c[pick] = special[torch.randint(0, 3, (int(pick.sum()),), device=cuda, generator=g)]
    pick = torch.rand((B, L, N), device=cuda, generator=g) < 0.01
    f[pick] = special[torch.randint(0, 3, (int(pick.sum()),), device=cuda, generator=g)]
    f[:, :, :16] = float("nan")                                                     # all-NaN rows
    f[:, :, 16:32] = -float("inf")                                                  # all -inf rows
    pc = torch.randn(B, 3, N, device=cuda)
    eye = torch.eye(4, device=cuda).expand(B, 4, 4)
    out = classifier.classifier_loss(c, f, pc, eye, torch.eye(3, device=cuda).expand(B, 3, 3), 160, 512)
    assert torch.equal(out["coarse_predictions"].long(), torch.max(c, dim=1)[1])
    assert torch.equal(out["fine_predictions"].long(), torch.max(f, dim=1)[1])


def _all_outputs(out, gc, gf):
    return [t for t in list(out.values()) + [gc, gf] if isinstance(t, torch.Tensor)]


def _bits_equal(a, b):
    return all(torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x,
                           y.view(torch.int32) if y.dtype == torch.float32 else y) for x, y in zip(a, b))


def test_deterministic_and_side_stream(cuda):
    case = make_case(13, *CASES["oxford"][:4])
    first = _all_outputs(*run(case, cuda))
    assert _bits_equal(first, _all_outputs(*run(case, cuda)))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        side = _all_outputs(*run(case, cuda))
    torch.cuda.current_stream().wait_stream(s)
    assert _bits_equal(first, side)


def test_slices_of_one_score_tensor(cuda):
    """The network returns [B,2+L,N]; its channel slices are read in place and give the contiguous results."""
    case = make_case(17, 4, 5000)
    c, f, pc, P, K, H, W = to_dev(case, cuda)
    whole = torch.cat((c, f), dim=1).requires_grad_(True)
    out = classifier.classifier_loss(whole[:, 0:2], whole[:, 2:], pc, P, K, H, W)
    torch.autograd.backward([out["loss"], out["coarse"], out["fine"]],
                            [torch.tensor(g, device=cuda) for g in GRADS])
    ref, gc, gf = run(case, cuda)
    assert _bits_equal([t for t in out.values() if isinstance(t, torch.Tensor)],
                       [t for t in ref.values() if isinstance(t, torch.Tensor)])
    assert torch.equal(whole.grad, torch.cat((gc, gf), dim=1))


def test_no_host_synchronisation(cuda):
    case = make_case(19, 2, 4096)
    run(case, cuda)                                       # loads the library
    c, f, pc, P, K, H, W = to_dev(case, cuda, requires_grad=True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = classifier.classifier_loss(c, f, pc, P, K, H, W)
        out["loss"].backward()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert c.grad is not None and f.grad is not None


def test_cuda_graph_capture(cuda):
    case = make_case(23, 4, 6000)
    c, f, pc, P, K, H, W = to_dev(case, cuda, requires_grad=True)

    def step():
        out = classifier.classifier_loss(c, f, pc, P, K, H, W)
        gc, gf = torch.autograd.grad(out["loss"], (c, f))
        return out, gc, gf

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    new = make_case(29, 4, 6000)
    with torch.no_grad():
        for t, a in ((c, new[0]), (f, new[1]), (pc, new[2]), (P, new[3]), (K, new[4])):
            t.copy_(torch.from_numpy(a))
    graph.replay()
    torch.cuda.synchronize()
    eager = step()
    assert _bits_equal(_all_outputs(*captured), _all_outputs(*eager))
    assert not torch.equal(eager[0]["coarse_labels"],
                           classifier.classifier_loss(*to_dev(case, cuda))["coarse_labels"])


class Head(torch.nn.Module):
    def __init__(self, L):
        super().__init__()
        self.a = torch.nn.Conv1d(16, 64, 1)
        self.b = torch.nn.Conv1d(64, 2 + L, 1)

    def forward(self, x):
        y = self.b(torch.relu(self.a(x)))
        return y[:, 0:2], y[:, 2:]


def test_conv_head_end_to_end(cuda):
    B, N, H, W = 4, 4096, 160, 512
    case = make_case(31, B, N, H, W)
    _, _, pc, P, K, _, _ = to_dev(case, cuda)
    torch.manual_seed(0)
    feat = torch.randn(B, 16, N, device=cuda)
    heads = [Head(80).to(cuda), Head(80).to(cuda)]
    heads[1].load_state_dict(heads[0].state_dict())
    out = classifier.classifier_loss(*heads[0](feat), pc, P, K, H, W)
    out["loss"].backward()
    ref = formulation(*heads[1](feat), pc, P, K, H, W)
    ref["loss"].backward()
    torch.testing.assert_close(out["loss"].double(), ref["loss"], rtol=1e-5, atol=0)
    for p0, p1 in zip(heads[0].parameters(), heads[1].parameters()):
        torch.testing.assert_close(p0.grad, p1.grad, rtol=1e-4, atol=1e-6)


def test_predictions_feed_registration(cuda):
    """coarse_predictions (int8) and fine_predictions (int32) go to register_batch and pnp_ransac_batch as they are."""
    smps = [syn.make_sample(60 + b, 4096) for b in range(2)]
    pc = torch.from_numpy(np.stack([m["points"] for m in smps])).to(cuda)
    P = torch.from_numpy(np.stack([m["P_gt"] for m in smps])).to(cuda)
    K, H, W = smps[0]["K"], smps[0]["H"], smps[0]["W"]
    Kb = torch.from_numpy(np.tile(K, (2, 1, 1))).to(cuda)
    L = int(np.prod(classifier.fine_grid(H, W, 32)))
    lab = classifier.classifier_loss(torch.zeros(2, 2, 4096, device=cuda), torch.zeros(2, L, 4096, device=cuda), pc, P,
                                     Kb, H, W)
    # scores that predict the ground truth
    coarse = torch.nn.functional.one_hot(lab["coarse_labels"].long(), 2).permute(0, 2, 1).float() * 5
    fine = torch.nn.functional.one_hot(lab["fine_labels"].long().clamp(min=0), L).permute(0, 2, 1).float() * 5
    out = classifier.classifier_loss(coarse, fine, pc, P, Kb, H, W)
    assert torch.equal(out["coarse_predictions"], out["coarse_labels"])
    reg = frustum.register_batch(pc, out["coarse_predictions"], 4096, K, H, W, n_inits=4)
    assert torch.isfinite(reg["P"]).all()
    res = pnp.pnp_ransac_batch(pc, out["coarse_predictions"], out["fine_predictions"], None, K, H, W)
    assert torch.isfinite(res["P"]).all() and (res["inliers"] > 0).all()
