"""bfloat16 autocast (DESIGN.md 4.37): the five differentiable ops' bf16 paths against their one contract (the float32
call on the widened inputs, rounded to bf16, bit for bit), the network under autocast, the bf16 trainer, and the
raises."""
import os

import numpy as np
import pytest
import torch

from deepi2p_b200 import classifier, kitti, network, point_ops, synthetic, train

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
ORDER = ("pc", "intensity", "sn", "node_a", "node_b", "img")
# (H, W, B) of the three datasets' image sizes and batch sizes (train.DEFAULTS); the ops are tested at B = 2
SHAPES = {"kitti": (160, 512, 8), "oxford": (384, 640, 8), "nuscenes": (160, 320, 12)}


def _bits(t):
    t = t.detach().contiguous()
    v = t.view(torch.int16 if t.dtype == BF else torch.int32)
    return torch.where(torch.isnan(t), torch.zeros_like(v), v)


def _same(a, b):
    """Bit for bit, any NaN equal to any NaN."""
    assert a.dtype == b.dtype and a.shape == b.shape, (a.dtype, b.dtype, a.shape, b.shape)
    assert torch.equal(torch.isnan(a), torch.isnan(b))
    assert torch.equal(_bits(a), _bits(b))


def _contract(op, feats, seed=0, strided=False):
    """op(*feats) -> tensor or tuple of differentiable tensors.  The bf16 call's outputs and feature gradients must be
    the float32 call's on the widened features (and the widened bf16 output gradient), rounded to bf16.  strided: the
    outputs reach the loss through a torch.cat, so their gradients are channel slices with a batch stride."""
    xb = [f.detach().clone().requires_grad_(True) for f in feats]
    xf = [f.detach().float().requires_grad_(True) for f in feats]
    ob, of = op(*xb), op(*xf)
    ob, of = (ob,) if torch.is_tensor(ob) else tuple(ob), (of,) if torch.is_tensor(of) else tuple(of)
    for a, b in zip(ob, of):
        assert a.dtype == BF
        _same(a, b.to(BF))
    gen = torch.Generator(device="cuda").manual_seed(seed)
    if strided:
        ob = [torch.cat((o, torch.zeros_like(o[:, :3])), 1) for o in ob]
        of = [torch.cat((o, torch.zeros_like(o[:, :3])), 1) for o in of]
    gs = [torch.randn(o.shape, generator=gen, device="cuda").to(BF) for o in ob]
    torch.autograd.backward(ob, gs)
    torch.autograd.backward(of, [g.float() for g in gs])
    for a, b in zip(xb, xf):
        assert a.grad.dtype == BF
        _same(a.grad, b.grad.to(BF))


def _batch(name, B, seed):
    H, W, _ = SHAPES[name]
    gen = torch.Generator().manual_seed(seed)
    smps = [synthetic.make_sample(seed + s, 20480, "oxford" if name == "oxford" else "kitti") for s in range(B)]
    pc = torch.from_numpy(np.stack([s["points"] for s in smps]))
    idx = torch.stack([torch.randperm(20480, generator=gen)[:256] for _ in range(B)])
    nodes = torch.gather(pc, 2, idx.unsqueeze(1).expand(B, 3, 256))
    sn = torch.nn.functional.normalize(torch.randn(B, 3, 20480, generator=gen), dim=1)
    P = torch.from_numpy(np.stack([s["P_gt"][:3] for s in smps])).float()
    K = torch.from_numpy(np.stack([s["K"] for s in smps])).float()
    out = dict(pc=pc, intensity=torch.rand(B, 1, 20480, generator=gen), sn=sn, node_a=nodes[:, :, :128].contiguous(),
               node_b=nodes[:, :, 128:].contiguous(), img=torch.rand(B, 3, H, W, generator=gen), P=P, K=K)
    return {k: v.cuda() for k, v in out.items()}


def _bf(shape, seed, levels=None):
    """Seeded bf16 normals; with levels, rounded to that many values per unit (exact ties)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(shape, generator=g, device="cuda")
    if levels:
        x = torch.round(x * levels) / levels
    return x.to(BF)


# -- the ops at the network's call shapes ------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(SHAPES))
def test_ops_at_network_shapes(name):
    H, W, _ = SHAPES[name]
    b = _batch(name, 2, 10)
    pc, node_a, node_b = b["pc"], b["node_a"], b["node_b"]
    ca = point_ops.cluster_assign_forward(pc, node_a, k=3)
    # the encoder's two max-pools: first_pn_out [B,32,N] with its scatter, second_pn_out [B,64,N]
    _contract(lambda f: point_ops.cluster_max_pool(f, ca["min_idx"], 128, broadcast=True), [_bf((2, 32, 20480), 1)],
              strided=True)
    _contract(lambda f: point_ops.cluster_max_pool(f, ca["min_idx"], 128), [_bf((2, 64, 20480), 2)])
    # the kNN module's grouping: node_b over the cluster means, node_a_features [B,64,128], K = 16
    _contract(lambda f: point_ops.knn_group(node_b, ca["cluster_mean"], f, 16)[1], [_bf((2, 64, 128), 3)],
              strided=True)
    # the decoder's three interpolations
    pb_idx = point_ops.cluster_assign_forward(pc, node_b, k=3, want_centers=False)["min_k_idx"]
    ab_idx = point_ops.cluster_assign_forward(node_a, node_b, k=3, want_centers=False)["min_k_idx"]
    _contract(lambda f: point_ops.upsample_by_interpolation(ca["min_k_idx"], pc, node_a, f), [_bf((2, 128, 128), 4)],
              strided=True)
    _contract(lambda f: point_ops.upsample_by_interpolation(pb_idx, pc, node_b, f), [_bf((2, 512, 128), 5)],
              strided=True)
    _contract(lambda f: point_ops.upsample_by_interpolation(ab_idx, node_a, node_b, f), [_bf((2, 512, 128), 6)],
              strided=True)
    # the two attention fusions: the stride-32 map with node_b's attention, the stride-16 map with node_a's
    L = classifier.fine_grid(H, W, 32)
    L = L[0] * L[1]
    _contract(point_ops.attention_fusion, [_bf((2, 512, L), 7), _bf((2, L, 128), 8)], strided=True)
    _contract(point_ops.attention_fusion, [_bf((2, 256, 4 * L), 9), _bf((2, 4 * L, 128), 10)], strided=True)
    # the loss on the channel slices of one [B,2+L,N] score tensor
    _loss_contract(_bf((2, 2 + L, 20480), 11, levels=4), b, H, W)


def _loss_contract(scores, b, H, W, fine=True):
    """classifier_loss on scores[:, :2] and scores[:, 2:]: every output of the float32 call on scores.float() outright,
    the score gradient rounded to bf16."""
    sb = scores.detach().clone().requires_grad_(True)
    sf = scores.detach().float().requires_grad_(True)
    ob = classifier.classifier_loss(sb[:, :2], sb[:, 2:] if fine else None, b["pc"], b["P"], b["K"], H, W)
    of = classifier.classifier_loss(sf[:, :2], sf[:, 2:] if fine else None, b["pc"], b["P"], b["K"], H, W)
    for k in of:
        if of[k] is None:
            assert ob[k] is None
        else:
            assert ob[k].dtype == of[k].dtype, k
            if of[k].is_floating_point():
                _same(ob[k].detach(), of[k].detach())
            else:
                assert torch.equal(ob[k], of[k]), k
    ob["loss"].backward()
    of["loss"].backward()
    _same(sb.grad, sf.grad.to(BF))
    return ob


def test_loss_predictions_are_torch_argmax_of_tied_bf16_scores():
    b = _batch("kitti", 3, 20)
    scores = _bf((3, 82, 20480), 21, levels=1)            # integers in [-5, 5]: most rows tie at their max
    top = scores[:, 2:].float().max(1, keepdim=True)[0]
    assert float((scores[:, 2:].float() == top).sum(1).float().mean()) > 2
    out = _loss_contract(scores, b, 160, 512)
    assert torch.equal(out["fine_predictions"], torch.argmax(scores[:, 2:], 1).to(torch.int32))
    assert torch.equal(out["coarse_predictions"], torch.argmax(scores[:, :2], 1).to(torch.int8))
    _loss_contract(scores[:, :2], b, 160, 512, fine=False)


# -- edge cases ----------------------------------------------------------------------------------------------------------
def test_cluster_max_pool_ties_all_equal_groups_and_nan():
    g = torch.Generator(device="cuda").manual_seed(30)
    for B, C, N, M in ((1, 5, 300, 7), (2, 33, 1001, 40), (3, 16, 64, 64)):
        min_idx = torch.randint(0, M, (B, N), generator=g, device="cuda", dtype=torch.int32)
        min_idx[:, :3] = -1                                # joins no segment
        f = _bf((B, C, N), 31 + N, levels=1)               # many ties
        f[:, 0][min_idx == 1] = 2.0                        # an all-equal group in channel 0
        f[0, 1, 10] = float("nan")
        f[0, 2, :] = -2000.0                               # nothing above index_max's floor
        _contract(lambda x: point_ops.cluster_max_pool(x, min_idx, M, broadcast=True), [f], seed=N)
        _contract(lambda x: point_ops.cluster_max_pool(x, min_idx, M), [f], seed=N + 1)


@pytest.mark.parametrize("B,M,N,K", [(1, 5, 7, 1), (2, 40, 32, 32), (1, 16, 16, 16), (3, 128, 128, 16)])
def test_knn_group_edges(B, M, N, K):
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + K)
    q = torch.round(torch.randn(B, 3, M, generator=g, device="cuda") * 2) / 2    # tied distances
    d = torch.round(torch.randn(B, 3, N, generator=g, device="cuda") * 2) / 2
    f = _bf((B, 9, N), K, levels=2)
    f[0, 0, 0] = float("nan")
    _contract(lambda x: point_ops.knn_group(q, d, x, K)[1], [f], seed=K, strided=True)
    _contract(lambda x: point_ops.knn_group(q, d, x, K)[1], [f[:, :0]], seed=K)                   # C = 0


@pytest.mark.parametrize("k", [1, 3, 8])
def test_interpolation_edges(k):
    g = torch.Generator(device="cuda").manual_seed(k)
    B, Nq, M = 2, 500, 37
    q, n = torch.randn(B, 3, Nq, generator=g, device="cuda"), torch.randn(B, 3, M, generator=g, device="cuda")
    idx = torch.randint(0, M, (B, Nq, k), generator=g, device="cuda", dtype=torch.int32)
    idx[0, 3, 0] = M                                       # out of range: a NaN column, no gradient
    f = _bf((B, 20, M), 40 + k)
    f[1, 2, 5] = float("nan")
    _contract(lambda x: point_ops.upsample_by_interpolation(idx, q, n, x), [f], seed=k, strided=True)
    _contract(lambda x: point_ops.upsample_by_interpolation(idx[:1], q[:1], n[:1], x), [f[:1]], seed=k + 10)


@pytest.mark.parametrize("B,C,P,M", [(1, 1, 1, 1), (2, 70, 33, 130), (1, 512, 80, 128), (9, 64, 320, 65)])
def test_attention_fusion_edges(B, C, P, M):
    F, A = _bf((B, C, P), C), _bf((B, P, M), M)
    F[0, 0, 0] = float("nan") if C > 1 else F[0, 0, 0]
    _contract(point_ops.attention_fusion, [F, A], seed=P, strided=True)
    # one input without a gradient
    out_b = point_ops.attention_fusion(F, A.detach().requires_grad_(True))
    assert out_b.dtype == BF


# -- the network under autocast --------------------------------------------------------------------------------------
def _model(name, seed=1, point_layers="torch"):
    H, W, _ = SHAPES[name]
    m = network.KeypointDetector(img_H=H, img_W=W, point_layers=point_layers)
    m.load_state_dict(synthetic.seeded_state_dict(m, seed))
    return m.cuda()


def _step(model, b, H, W, bf16):
    torch.manual_seed(123)                                # the dropout masks
    with torch.autocast("cuda", dtype=BF, enabled=bf16, cache_enabled=False):
        coarse, fine = model(*(b[k] for k in ORDER))
        out = classifier.classifier_loss(coarse, fine, b["pc"], b["P"], b["K"], H, W)
    model.zero_grad(set_to_none=True)
    out["loss"].backward()
    grads = [p.grad.clone() for p in model.parameters() if p.grad is not None]
    return coarse.detach(), fine.detach(), {k: out[k].detach() for k in ("loss", "coarse", "fine")}, grads


# The bf16 losses must be within LOSS_RTOL (relative) of the fp32 model's on the same batch, weights and dropout
# masks.  bf16 keeps 8 significant bits (relative rounding 2^-9 = 2.0e-3); the forward rounds at about 20 layers and
# BatchNorm renormalises after each, and the losses are means over 2 x 20480 points.  On an H100 the largest relative
# difference of the three losses over the three shapes was 1.45e-2 (KITTI's coarse loss; 2.6e-3 to 1.45e-2 in all);
# the tolerance is about three times that.
LOSS_RTOL = 0.05


@pytest.mark.parametrize("name", list(SHAPES))
def test_network_under_autocast_is_deterministic_and_near_fp32(name):
    H, W, _ = SHAPES[name]
    b = _batch(name, 2, 50)
    flags = (torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark,
             torch.are_deterministic_algorithms_enabled())
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    torch.use_deterministic_algorithms(True)
    try:
        model = _model(name).train()
        runs = [_step(model, b, H, W, True) for _ in range(2)]
        ref = _step(model, b, H, W, False)
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = flags[:2]
        torch.use_deterministic_algorithms(flags[2])
    (c0, f0, l0, g0), (c1, f1, l1, g1) = runs
    assert c0.dtype == f0.dtype == BF and l0["loss"].dtype == torch.float32
    _same(c0, c1)
    _same(f0, f1)
    for k in l0:
        _same(l0[k], l1[k])
    assert len(g0) == len(g1) == len(ref[3]) and all(g.dtype == torch.float32 for g in g0)
    assert all(torch.equal(a, b_) for a, b_ in zip(g0, g1))
    assert all(bool(torch.isfinite(g).all()) for g in g0)
    for k in ("loss", "coarse", "fine"):
        rel = abs(float(l0[k]) - float(ref[2][k])) / abs(float(ref[2][k]))
        print(f"{name} {k}: bf16 {float(l0[k]):.6f} fp32 {float(ref[2][k]):.6f} relative difference {rel:.3e}")
        assert rel < LOSS_RTOL, (name, k, rel)
    # eval mode under autocast runs too
    model.eval()
    with torch.no_grad(), torch.autocast("cuda", dtype=BF, cache_enabled=False):
        c, f = model(*(b[k] for k in ORDER))
    assert c.dtype == BF and bool(torch.isfinite(c).all())


def test_autocast_raises_for_fused_modes_and_float16():
    b = _batch("kitti", 1, 60)
    for mode in ("fused", "fused_all"):
        for training in (True, False):
            m = _model("kitti", point_layers=mode).train(training)
            with torch.no_grad(), torch.autocast("cuda", dtype=BF):
                with pytest.raises(ValueError, match="point_layers='torch'"):
                    m(*(b[k] for k in ORDER))
    m = _model("kitti")
    with torch.autocast("cuda", dtype=torch.float16):
        with pytest.raises(ValueError, match="bfloat16 only"):
            m(*(b[k] for k in ORDER))
    with pytest.raises(RuntimeError, match="features must have dtype"):
        point_ops.cluster_max_pool(torch.zeros(1, 2, 8, device="cuda", dtype=torch.float16),
                                   torch.zeros(1, 8, device="cuda", dtype=torch.int32), 2)


# -- the trainer in bf16 ---------------------------------------------------------------------------------------------
@pytest.fixture
def deterministic():
    flags = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    yield
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = flags


def _state(model, opt):
    out = {("model", k): v.clone() for k, v in model.state_dict().items()}
    for i, p in enumerate(model.parameters()):
        for k, v in opt.state[p].items():
            out[("adam", i, k)] = v.clone()
    return out


@pytest.mark.parametrize("dropout", [True, False])
def test_bf16_captured_step_is_the_eager_loop_bit_for_bit(deterministic, dropout):
    batches = [_batch("kitti", 2, 100 + k) for k in range(7)]

    def run(capture):
        model = _model("kitti")
        if not dropout:
            model.per_point_pn.layers[0].dropout = model.per_point_pn.layers[1].dropout = None
        opt = train.make_optimizer(model)
        static = {k: torch.empty_like(v) for k, v in batches[0].items()}
        stats, losses = torch.zeros(5, device="cuda"), []
        torch.cuda.manual_seed(7)
        graph = None
        for k, b in enumerate(batches):
            for n, v in b.items():
                static[n].copy_(v)
            if not capture or k < train.WARMUP_STEPS:
                stats.copy_(train._stats(train.train_step(model, opt, static, "bf16")))
            else:
                if graph is None:
                    opt.zero_grad(set_to_none=True)
                    graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graph):
                        stats.copy_(train._stats(train.train_step(model, opt, static, "bf16")))
                graph.replay()
            losses.append(stats.clone())
        torch.cuda.synchronize()
        return _state(model, opt), torch.stack(losses)

    s_eager, l_eager = run(False)
    s_graph, l_graph = run(True)
    assert torch.equal(l_eager, l_graph)
    assert s_eager.keys() == s_graph.keys()
    assert all(v.dtype != BF for v in s_eager.values())      # parameters, buffers and Adam state stay float32
    bad = [k for k in s_eager if not torch.equal(s_eager[k], s_graph[k])]
    assert not bad, f"{len(bad)} tensors differ, first {bad[:3]}"


def test_bf16_run_learns_and_its_checkpoint_evaluates_in_fp32(tmp_path):
    """test_train_gpu.py's learning test with precision="bf16": train on sequence 9, test on 10; held-out coarse
    accuracy clearly above the all-outside baseline.  The float32 checkpoint then loads and evaluates without autocast
    to nearly the same accuracy: 0.8045 against the bf16 test pass's 0.8142 on an H100, where the baseline is 0.767."""
    def source(root, seq):
        ds = kitti.KittiDataset(root, "val", seqs=(seq,))
        return len(ds), lambda items, seed, rng, stream: kitti.kitti_batch(ds, items, "val", seed, rng=rng,
                                                                           stream=stream)
    root = str(tmp_path / "root")
    synthetic.write_kitti_root(root, seqs=(9, 10), n_frames=200, seed=4)
    tr, te = source(root, 9), source(root, 10)
    lines = []
    t = train.Trainer(_model("kitti", 3), tr, te, "kitti", str(tmp_path / "out"), batch_size=4, epochs=6,
                      log=lines.append, precision="bf16")
    last = t.run()
    inside = []
    for items in train.test_batches(te[0], 4):
        vals = te[1](items, 0, 0, None)
        pc, P, K = vals[0], vals[5].cuda(), vals[7].cuda().float()
        z = torch.zeros(pc.shape[0], 2, pc.shape[2], device="cuda")
        inside.append(classifier.classifier_loss(z, None, pc, P, K, 160, 512)["coarse_labels"].float().mean().item())
    baseline = 1.0 - float(np.mean(inside))
    acc = float(os.path.basename(last)[:-4].split("-")[-1])
    print("bf16 held-out coarse accuracy", acc, "all-outside baseline", baseline, lines[-6:])
    assert acc > baseline + 0.04

    sd = torch.load(last, weights_only=True)
    assert all(v.dtype in (torch.float32, torch.int64) for v in sd.values())
    m = network.KeypointDetector(**network.SHAPES["kitti"])
    network.load_checkpoint(m, last)
    t32 = train.Trainer(m.cuda(), tr, te, "kitti", str(tmp_path / "eval"), batch_size=4, log=lambda s: None)
    losses, acc32 = t32.test(0)
    print("fp32 evaluation of the bf16 checkpoint", losses, acc32)
    assert abs(acc32["coarse_accuracy"] - acc) < 0.02
    assert acc32["coarse_accuracy"] > baseline + 0.02
