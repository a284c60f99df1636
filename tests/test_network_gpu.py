"""The classifier network on the H100 (DESIGN.md 4.18): eval- and train-mode scores and parameter gradients against the
reference's own network (tests/golden/network_small.npz), a bit-reproducible KITTI training step under
torch.use_deterministic_algorithms, and classify_and_register against its parts."""
import os

import numpy as np
import pytest
import torch

from deepi2p_b200 import classifier, frustum, network, synthetic

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "network_small.npz")
# |gpu - ref64| <= TOL_FACTOR max|ref32 - ref64| + 1e-6 max|ref64| per tensor, ref32 / ref64 the reference network
# in float32 / float64 on the CPU (DESIGN.md 4.18 records the measured ratios)
TOL_FACTOR = 4.0


@pytest.fixture(autouse=True)
def no_tf32():
    flags = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = flags


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def within(name, got, g, key):
    """got: the full GPU tensor; the fixture keeps the float64 reference at a stride (make_network_golden.py)."""
    if key.startswith("grad_"):
        got = got.reshape(-1)[::int(g["grad_stride"][int(key[5:])])]
    else:
        got = got[..., ::int(g["point_stride"])]
    ref64, spread = g[key], float(g["spread_" + key])
    assert got.shape == ref64.shape, (name, got.shape, ref64.shape)
    err = np.abs(got.astype(np.float64) - ref64).max()
    bound = TOL_FACTOR * spread + 1e-6 * np.abs(ref64).max()
    print(f"{name}: max|gpu - ref64| {err:.3e}, max|ref32 - ref64| {spread:.3e}, ratio {err / spread:.3f}")
    assert err <= bound, (name, err, bound)


def small_model(g):
    model = network.KeypointDetector(img_H=64, img_W=128)
    model.load_state_dict(synthetic.seeded_state_dict(model, int(g["weight_seed"])), strict=True)
    return model.cuda()


def small_inputs(g):
    """The fixture's inputs and loss weights, regenerated from its seed (test_network_cpu checks the fingerprint)."""
    x = synthetic.make_network_inputs(int(g["input_seed"]))
    return {k: torch.from_numpy(v).cuda() for k, v in x.items()}


ORDER = ("pc", "intensity", "sn", "node_a", "node_b", "img")


def test_eval_matches_reference(golden):
    model = small_model(golden).eval()
    x = small_inputs(golden)
    with torch.no_grad():
        coarse, fine = model(*(x[k] for k in ORDER))
    within("eval coarse", coarse.cpu().numpy(), golden, "eval_coarse")
    within("eval fine", fine.cpu().numpy(), golden, "eval_fine")


def test_train_and_gradients_match_reference(golden):
    model = small_model(golden).train()
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.eval()
    x = small_inputs(golden)
    coarse, fine = model(*(x[k] for k in ORDER))
    loss = (coarse * x["lw_coarse"]).sum() + (fine * x["lw_fine"]).sum()
    loss.backward()
    within("train coarse", coarse.detach().cpu().numpy(), golden, "train_coarse")
    within("train fine", fine.detach().cpu().numpy(), golden, "train_fine")
    params = dict(model.named_parameters())
    for i, k in enumerate(golden["grad_keys"]):
        within("grad " + str(k), params[str(k)].grad.cpu().numpy(), golden, f"grad_{i}")


def kitti_batch(B, seed, dev):
    """B KITTI-shaped samples: make_sample clouds, seeded intensities, normals, node sets (subsets of the cloud),
    images, P and K."""
    gen = torch.Generator().manual_seed(seed)
    smps = [synthetic.make_sample(seed + s, 20480, "kitti") for s in range(B)]
    pc = torch.from_numpy(np.stack([s["points"] for s in smps]))
    idx = torch.stack([torch.randperm(20480, generator=gen)[:256] for _ in range(B)])
    nodes = torch.gather(pc, 2, idx.unsqueeze(1).expand(B, 3, 256))
    sn = torch.nn.functional.normalize(torch.randn(B, 3, 20480, generator=gen), dim=1)
    P = torch.from_numpy(np.stack([s["P_gt"][:3] for s in smps])).float()
    K = torch.from_numpy(np.stack([s["K"] for s in smps])).float()
    out = dict(pc=pc, intensity=torch.rand(B, 1, 20480, generator=gen), sn=sn, node_a=nodes[:, :, :128].contiguous(),
               node_b=nodes[:, :, 128:].contiguous(), img=torch.rand(B, 3, 160, 512, generator=gen), P=P, K=K)
    return {k: v.to(dev) for k, v in out.items()}


def test_training_step_is_bit_reproducible():
    dev = torch.device("cuda")
    batch = kitti_batch(8, 400, dev)
    base = network.KeypointDetector(**network.SHAPES["kitti"])
    state = synthetic.seeded_state_dict(base, 1)
    flags = (torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark, torch.are_deterministic_algorithms_enabled())
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    torch.use_deterministic_algorithms(True)
    try:
        results = []
        for _ in range(2):
            model = network.KeypointDetector(**network.SHAPES["kitti"])
            model.load_state_dict(state)
            model = model.to(dev).train()
            opt = torch.optim.Adam(model.parameters(), lr=1e-3)
            torch.manual_seed(123)                          # the dropout masks
            coarse, fine = model(*(batch[k] for k in ("pc", "intensity", "sn", "node_a", "node_b", "img")))
            out = classifier.classifier_loss(coarse, fine, batch["pc"], batch["P"], batch["K"], 160, 512)
            opt.zero_grad()
            out["loss"].backward()
            unused = [k for k, p in model.named_parameters() if p.grad is None]
            assert unused == ["img_encoder.backbone.fc.weight", "img_encoder.backbone.fc.bias"]
            grads = [p.grad.clone() for p in model.parameters() if p.grad is not None]
            opt.step()
            results.append((out["loss"].detach().clone(), grads, [p.detach().clone() for p in model.parameters()]))
        (l0, g0, p0), (l1, g1, p1) = results
        assert torch.isfinite(l0) and torch.equal(l0, l1)
        assert all(torch.equal(a, b) for a, b in zip(g0, g1))
        assert all(torch.equal(a, b) for a, b in zip(p0, p1))
        assert all(bool(g.abs().sum() > 0) for g in g0)
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = flags[:2]
        torch.use_deterministic_algorithms(flags[2])


def oxford_batch(S, seed, dev):
    gen = torch.Generator().manual_seed(seed)
    smps = [synthetic.make_sample(seed + s, 20480, "oxford") for s in range(S)]
    pc = torch.from_numpy(np.stack([s["points"] for s in smps]))
    idx = torch.stack([torch.randperm(20480, generator=gen)[:256] for _ in range(S)])
    nodes = torch.gather(pc, 2, idx.unsqueeze(1).expand(S, 3, 256))
    out = dict(pc=pc, intensity=torch.rand(S, 1, 20480, generator=gen),
               sn=torch.nn.functional.normalize(torch.randn(S, 3, 20480, generator=gen), dim=1),
               node_a=nodes[:, :, :128].contiguous(), node_b=nodes[:, :, 128:].contiguous(),
               img=torch.rand(S, 3, 384, 640, generator=gen))
    out = {k: v.to(dev) for k, v in out.items()}
    out["K"] = torch.from_numpy(np.stack([s["K"] for s in smps])).float().to(dev)
    return out


ARGS = ("pc", "intensity", "sn", "node_a", "node_b", "img")


@pytest.fixture(scope="module")
def oxford():
    dev = torch.device("cuda")
    model = network.KeypointDetector(**network.SHAPES["oxford"])
    model.load_state_dict(synthetic.seeded_state_dict(model, 2))
    return model.to(dev), oxford_batch(6, 500, dev)


def chunked_scores(model, b, chunk):
    with torch.no_grad():
        outs = [model(*(b[k][a:a + chunk] for k in ARGS)) for a in range(0, b["pc"].shape[0], chunk)]
    return torch.cat([o[0] for o in outs]), torch.cat([o[1] for o in outs])


def test_classify_and_register_equals_its_parts(oxford):
    model, b = oxford
    model.train()
    out = network.classify_and_register(model, *(b[k] for k in ARGS), b["K"], chunk=4)
    assert model.training                                   # the flag is restored
    model.eval()
    coarse, fine = chunked_scores(model, b, 4)
    c, f = network.predict(coarse, fine)
    assert torch.equal(out["coarse_pred"], c) and torch.equal(out["fine_pred"], f)
    reg = frustum.register_batch(b["pc"], c, 20480, b["K"], 384, 640)
    for k in ("P", "cost", "degenerate"):
        assert torch.equal(out[k], reg[k]), k


def test_classify_and_register_all_outside(oxford):
    model, b = oxford
    with torch.no_grad():
        bias = model.per_point_pn.layers[2].conv.bias
        saved = bias.clone()
        bias[0] = 1e6                                       # class 0 (outside) wins everywhere
        try:
            out = network.classify_and_register(model, *(b[k] for k in ARGS), b["K"], chunk=4)
        finally:
            bias.copy_(saved)
    assert int(out["coarse_pred"].abs().sum()) == 0
    eye = torch.eye(4, dtype=torch.float64, device=b["pc"].device)
    for s in range(6):
        assert torch.equal(out["P"][s], eye) and float(out["cost"][s]) == 1e4 and int(out["degenerate"][s]) == 1


def test_chunk_size_changes_rounding_only(oxford):
    model, b = oxford
    model.eval()
    c2, f2 = chunked_scores(model, b, 2)
    c6, f6 = chunked_scores(model, b, 6)
    for x, y in ((c2, c6), (f2, f6)):
        assert float((x - y).abs().max()) <= 1e-4 * float(y.abs().max())
