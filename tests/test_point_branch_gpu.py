"""point_ops.point_branch and KeypointDetector(point_layers="fused_all") (DESIGN.md 4.36) on the device: the kNN
module, final_pointnet + global max and the four node-level PointNets at the KITTI, Oxford and nuScenes widths against
float64 copies of the model's own layers (outputs, running statistics, num_batches_tracked and every gradient), the
group max and group sum against exact restatements, edge shapes, bit-identical reruns, a captured "fused_all" step
against the eager one, the whole model against the torch layers, eval mode against FusedInference, and peak memory."""
import copy

import numpy as np
import pytest
import torch

from deepi2p_b200 import network, point_ops, synthetic, train

pytestmark = pytest.mark.gpu
TOL = 2.0 ** -10
# Outputs and running statistics: |fused - float64| <= C_OUT 2^-10 max|float64| for every element.
C_OUT = 16
# Gradients: |fused - float64| <= C_GRAD 2^-10 sum|terms| per element, sum|terms| being the backward with every term
# replaced by its magnitude (the form of tests/test_point_chain_gpu.py), for all but a share FRAC of the elements.  The
# float64 restatement takes each group max at the index the fused path chose (gathered, not its own arg-max), so what
# remains to flip is a ReLU input within TF32 rounding of zero, which moves that element's gradient completely; with as
# few as 256 columns (K = 1, B = 1) one such flip moves a whole row of a weight gradient.  The largest share measured on
# an H100 was 7.8e-3: 2 of the 256 BatchNorm-bias gradients of the kNN module's last layer at K = 1, whose batch has
# only 256 columns; the shares are printed (pytest -s).
C_GRAD, FRAC = 16, 1e-2


def _check(got, want, what, c=C_OUT):
    want = want.double()
    scale = want.abs().max().item()
    err = (got.double() - want).abs()
    bad = (err > c * TOL * scale).double().mean().item()
    print(f"{what}: max error {err.max().item() / max(scale, 1e-300):.2e} of max|ref|")
    assert bad == 0, f"{what}: {bad:.2e} of the elements exceed {c} 2^-10 max|ref|"


def _check_sum(got, want, scale, what, frac=FRAC, c=C_GRAD):
    bad = ((got.double() - want.double()).abs() > c * TOL * scale.double()).double().mean().item()
    print(f"{what}: share past {c} 2^-10 sum|terms|: {bad:.2e}")
    assert bad <= frac, f"{what}: {bad:.2e} of the elements exceed {c} 2^-10 sum|terms|"


class _BnReluAbs(torch.autograd.Function):
    """The magnitude graph of train-mode BatchNorm + ReLU over [B, C, cols]: forward gives |a|, backward the sum of
    |terms| of the BatchNorm backward (dY = k1 (dZ - mean dZ - x^ mean(dZ x^))) and of dgamma, dbeta."""

    @staticmethod
    def forward(ctx, ya, ga, bea, a_abs, keep, xhat_abs, k1_abs):
        ctx.save_for_backward(keep, xhat_abs, k1_abs)
        return a_abs.clone()

    @staticmethod
    def backward(ctx, g):
        keep, xa, k1 = ctx.saved_tensors
        gz = g * keep
        M = gz.shape[0] * gz.shape[2]
        gy = k1[None, :, None] * (gz + gz.sum(dim=(0, 2), keepdim=True) / M
                                  + xa * (gz * xa).sum(dim=(0, 2), keepdim=True) / M)
        return gy, (gz * xa).sum(dim=(0, 2)), gz.sum(dim=(0, 2)), None, None, None, None


def _ref_layer(layer, x, xa, before):
    """One _PointLayer in float64 over [B, C, cols] (a Conv2d layer's [B, C, M, K] viewed as [B, C, M K]), beside
    its magnitude graph over xa.  before: the layer's (running_mean, running_var) as the fused call found them.
    Returns (a, a_abs, [(fused param, float64 leaf, magnitude leaf)], (running_mean, running_var) or None)."""
    conv, norm = layer.conv, layer.norm
    C = conv.out_channels
    leaf = lambda t, *shape: t.detach().double().reshape(*shape).clone().requires_grad_()
    mag = lambda t: t.detach().abs().requires_grad_()
    W, b = leaf(conv.weight, C, conv.in_channels), leaf(conv.bias, C)
    Wa, ba = mag(W), mag(b)
    y = torch.einsum("ck,bkn->bcn", W, x) + b[None, :, None]
    ya = torch.einsum("ck,bkn->bcn", Wa, xa) + ba[None, :, None]
    params = [(conv.weight, W, Wa)] + ([] if norm is not None else [(conv.bias, b, ba)])
    if norm is None:
        return y, ya, params, None
    g, be = leaf(norm.weight, C), leaf(norm.bias, C)
    mean, var = y.mean(dim=(0, 2)), y.var(dim=(0, 2), unbiased=False)
    M = y.shape[0] * y.shape[2]
    run = ((1 - norm.momentum) * before[0].double() + norm.momentum * mean.detach(),
           (1 - norm.momentum) * before[1].double() + norm.momentum * var.detach() * M / (M - 1))
    invstd = 1 / torch.sqrt(var + norm.eps)
    xhat = (y - mean[None, :, None]) * invstd[None, :, None]
    z = xhat * g[None, :, None] + be[None, :, None]
    a = torch.relu(z)
    ga, bea = mag(g), mag(be)
    aa = _BnReluAbs.apply(ya, ga, bea, a.detach().abs(), (z > 0).double().detach(), xhat.detach().abs(),
                          (g * invstd).detach().abs())
    return a, aa, params + [(norm.weight, g, ga), (norm.bias, be, bea)], run


def _ref_chain(layers, x, xa, before):
    params, runs = [], []
    for layer, bf in zip(layers, before):
        x, xa, p, r = _ref_layer(layer, x, xa, bf)
        params += p
        runs.append((layer, r))
    return x, xa, params, runs


def _gmax(y, idx, G):
    """The max over groups of G columns taken at the fused path's in-group indices idx [B, C, cols / G]."""
    B, C, N = y.shape
    return y.reshape(B, C, N // G, G).gather(3, idx.long().unsqueeze(3)).squeeze(3)


def _group_idx(act, G):
    B, C, N = act.shape
    return torch.max(act.reshape(B, C, N // G, G), dim=3).indices


def _buffers(layers):
    return [(l.norm.running_mean.clone(), l.norm.running_var.clone(), l.norm.num_batches_tracked.clone())
            if l.norm is not None else None for l in layers]


def _compare(params, runs, before, what):
    """Every parameter gradient against the float64 one within C_GRAD 2^-10 sum|terms|, the running statistics within
    C_OUT 2^-10 max|ref| and num_batches_tracked one up."""
    for i, (pf, p64, pa) in enumerate(params):
        got = pf.grad.reshape(p64.shape)
        _check_sum(got, p64.grad, pa.grad, f"{what} param {i} {tuple(p64.shape)} grad")
    for (layer, r), bf in zip(runs, before):
        if r is not None:
            _check(layer.norm.running_mean, r[0], f"{what} running_mean")
            _check(layer.norm.running_var, r[1], f"{what} running_var")
            assert layer.norm.num_batches_tracked.item() == bf[2].item() + 1


def _model(shape="kitti", seed=0, fine=True, point_layers="fused_all"):
    m = network.KeypointDetector(**network.SHAPES[shape], fine=fine, point_layers=point_layers)
    m.load_state_dict(synthetic.seeded_state_dict(m, 1 + seed))
    m = m.cuda().train()
    torch.manual_seed(seed)
    with torch.no_grad():                    # non-trivial BN parameters and running statistics
        for mod in m.modules():
            if isinstance(mod, (torch.nn.BatchNorm1d, torch.nn.BatchNorm2d)):
                C = mod.num_features
                mod.weight.copy_(torch.rand(C) + 0.5)
                mod.bias.copy_(torch.randn(C) * 0.1)
                mod.running_mean.copy_(torch.randn(C) * 0.1)
                mod.running_var.copy_(torch.rand(C) + 0.5)
    return m


def _randn(shape, g, scale=1.0):
    return (torch.randn(shape, device="cuda", generator=g) * scale).requires_grad_()


def _leaf64(t):
    x = t.detach().double().requires_grad_()
    return x, x.detach().abs().requires_grad_()


def _run_knn(m, B, Ma, Mb, K, seed):
    """The kNN module through KeypointDetector._fused_knn and its float64 restatement (module order: before-chain,
    max over K expanded and concatenated in front, after-chain, max over K), the maxes at the fused indices."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    m.k_ab = K
    knn = m.pc_encoder.knnlayer
    twin = copy.deepcopy(knn)                   # the same call again, with outputs="both", for the fused indices
    lb, la = list(knn.layers_before), list(knn.layers_after)
    before_b, before_a = _buffers(lb), _buffers(la)
    naf = _randn((B, 64, Ma), g)
    cm = torch.randn((B, 3, Ma), device="cuda", generator=g)
    nb = torch.randn((B, 3, Mb), device="cuda", generator=g)
    out = m._fused_knn(nb, cm, naf)
    gout = torch.randn(out.shape, device="cuda", generator=g)
    out.backward(gout)
    naf2 = naf.detach().clone().requires_grad_()
    _, x = point_ops.knn_group(nb, cm, naf2, K)
    xf = x.reshape(B, x.shape[1], Mb * K)
    with torch.no_grad():
        act_b, mx_b = point_ops.point_branch([xf.detach()], list(twin.layers_before), None, max_group=K,
                                             output="both")
        proj = point_ops.channel_product(twin.layers_after[0].conv.weight[:, :mx_b.shape[1], 0, 0], mx_b)
        act_a, _ = point_ops.point_branch([act_b], list(twin.layers_after), None, cols=[mx_b.shape[1]], add=proj,
                                          add_group=K, max_group=K, output="both")
    idx_b, idx_a = _group_idx(act_b, K), _group_idx(act_a, K)
    x64, xa = _leaf64(xf)
    a, aa, p1, r1 = _ref_chain(lb, x64, xa, before_b)
    pooled = lambda t: _gmax(t, idx_b, K).unsqueeze(3).expand(-1, -1, -1, K).reshape(t.shape)
    y, ya = torch.cat((pooled(a), a), dim=1), torch.cat((pooled(aa), aa), dim=1)
    y, ya, p2, r2 = _ref_chain(la, y, ya, before_a)
    ref, ref_a = _gmax(y, idx_a, K), _gmax(ya, idx_a, K)
    ref.backward(gout.double())
    ref_a.backward(gout.double().abs())
    naf_ref = torch.autograd.grad(xf, naf2, x64.grad.float(), retain_graph=True)[0]
    naf_abs = torch.autograd.grad(xf, naf2, xa.grad.float())[0]
    return dict(out=out, ref=ref, naf=(naf.grad, naf_ref, naf_abs), params=p1 + p2, runs=r1 + r2,
                before=before_b + before_a, knn=knn)


KNN_CASES = [("kitti", 2, 128, 128, 16), ("oxford", 2, 128, 128, 16), ("nuscenes", 3, 128, 128, 16),
             ("K1", 2, 128, 128, 1), ("K_is_M", 2, 16, 16, 16), ("M77", 2, 77, 77, 8), ("B1", 1, 128, 128, 16)]


@pytest.mark.parametrize("case", KNN_CASES, ids=[c[0] for c in KNN_CASES])
def test_knn_module_matches_float64(case):
    name, B, Ma, Mb, K = case
    m = _model(name if name in network.SHAPES else "kitti")
    r = _run_knn(m, B, Ma, Mb, K, 3)
    _check(r["out"], r["ref"], f"knn {name} out")
    _compare(r["params"], r["runs"], r["before"], f"knn {name}")
    got, want, scale = r["naf"]
    _check_sum(got, want, scale, f"knn {name} node_a_features grad")


def _node_inputs(B, M, g):
    return dict(nbf=_randn((B, 256, M), g), naf=_randn((B, 64, M), g), ws32=_randn((B, 512, M), g),
                ws16=_randn((B, 256, M), g), ab=_randn((B, 512, M), g), ig=_randn((B, 512), g),
                gf=_randn((B, 512), g), nb=_randn((B, 3, M), g))


# name -> (module getter, fused call, the torch.cat rows of the float64 reference)
NODE = {
    "att_b": (lambda m: m.node_b_attention_pn,
              lambda m, i, M: m._fused_node(m.node_b_attention_pn, [i["nbf"]], [0], [(256, i["ig"])], M),
              lambda i, M: [i["nbf"], i["ig"][:, :, None].expand(-1, -1, M)]),
    "node_b": (lambda m: m.node_b_pn,
               lambda m, i, M: m._fused_node(m.node_b_pn, [i["nbf"], i["ws32"]], [0, 768],
                                             [(256, i["gf"]), (1280, i["ig"])], M),
               lambda i, M: [i["nbf"], i["gf"][:, :, None].expand(-1, -1, M), i["ws32"],
                             i["ig"][:, :, None].expand(-1, -1, M)]),
    "att_a": (lambda m: m.node_a_attention_pn,
              lambda m, i, M: m._fused_node(m.node_a_attention_pn, [i["naf"]], [0], [(64, i["ig"])], M),
              lambda i, M: [i["naf"], i["ig"][:, :, None].expand(-1, -1, M)]),
    "node_a": (lambda m: m.node_a_pn,
               lambda m, i, M: m._fused_node(m.node_a_pn, [i["naf"], i["ab"], i["ws16"]], None, [], M),
               lambda i, M: [i["naf"], i["ab"], i["ws16"]]),
    "final": (lambda m: m.pc_encoder.final_pointnet,
              lambda m, i, M: point_ops.point_branch([i["nb"], i["nbf"]], list(m.pc_encoder.final_pointnet.layers),
                                                     None, max_group=M, output="max"),
              lambda i, M: [i["nb"], i["nbf"]]),
}


def _run_node(name, shape, B, M, seed):
    m = _model(shape)
    get, fused, rows = NODE[name]
    pn = get(m)
    layers = list(pn.layers)
    twin, before = copy.deepcopy(pn), _buffers(layers)
    g = torch.Generator(device="cuda").manual_seed(seed)
    inp = _node_inputs(B, M, g)
    out = fused(m, inp, M)
    gout = torch.randn(out.shape, device="cuda", generator=g)
    out.backward(gout)
    pairs = {k: _leaf64(v) for k, v in inp.items()}
    rows64 = rows({k: v[0] for k, v in pairs.items()}, M)
    rows_a = rows({k: v[1] for k, v in pairs.items()}, M)
    ref, ref_a, params, runs = _ref_chain(layers, torch.cat(rows64, 1), torch.cat(rows_a, 1), before)
    if name == "final":
        with torch.no_grad():
            act, _ = point_ops.point_branch([inp["nb"].detach(), inp["nbf"].detach()], list(twin.layers), None,
                                            max_group=M, output="both")
        idx = _group_idx(act, M)
        ref, ref_a = _gmax(ref, idx, M), _gmax(ref_a, idx, M)
    ref.backward(gout.double())
    ref_a.backward(gout.double().abs())
    return dict(out=out, ref=ref, params=params, runs=runs, before=before, pn=pn,
                inputs={k: (v.grad, pairs[k][0].grad, pairs[k][1].grad) for k, v in inp.items() if v.grad is not None})


@pytest.mark.parametrize("shape", ["kitti", "oxford", "nuscenes"])
@pytest.mark.parametrize("name", list(NODE))
def test_node_pointnets_and_final_match_float64(name, shape):
    r = _run_node(name, shape, 3 if shape == "nuscenes" else 2, 128, 5)
    _check(r["out"], r["ref"], f"{name} {shape} out")
    _compare(r["params"], r["runs"], r["before"], f"{name} {shape}")
    for k, (got, want, scale) in r["inputs"].items():
        _check_sum(got, want, scale, f"{name} {shape} {k} grad")


@pytest.mark.parametrize("width", [1, 300, 512, 1024])
def test_widths_with_a_group_max(width):
    torch.manual_seed(width)
    pn = network._PointNet(40, [width], True).cuda()
    layers, before = list(pn.layers), _buffers(list(pn.layers))
    g = torch.Generator(device="cuda").manual_seed(1)
    x = _randn((2, 40, 77 * 4), g)
    act, mx = point_ops.point_branch([x], layers, None, max_group=4, output="both")
    ga, gm = torch.randn(act.shape, device="cuda", generator=g), torch.randn(mx.shape, device="cuda", generator=g)
    torch.autograd.backward([act, mx], [ga, gm])
    x64, xa = _leaf64(x)
    a64, aa, params, runs = _ref_chain(layers, x64, xa, before)
    idx = _group_idx(act, 4)
    m64 = _gmax(a64, idx, 4)
    torch.autograd.backward([a64, m64], [ga.double(), gm.double()])
    torch.autograd.backward([aa, _gmax(aa, idx, 4)], [ga.double().abs(), gm.double().abs()])
    _check(act, a64, f"width {width} act")
    _check(mx, m64, f"width {width} max")
    _check_sum(x.grad, x64.grad, xa.grad, f"width {width} x grad")
    _compare(params, runs, before, f"width {width}")


def test_sources_out_of_column_order():
    """Sources that feed layer 1's columns in another order than theirs: the weight gradient lands on each source's
    own columns, as the float64 restatement over the columns in layer order has it."""
    torch.manual_seed(3)
    pn = network._PointNet(7, [32, 16], True).cuda()
    layers, before = list(pn.layers), _buffers(list(pn.layers))
    g = torch.Generator(device="cuda").manual_seed(2)
    a, b = _randn((2, 3, 500), g), _randn((2, 4, 500), g)          # b feeds columns 0-3, a columns 4-6
    out = point_ops.point_branch([a, b], layers, None, cols=[4, 0])
    gout = torch.randn(out.shape, device="cuda", generator=g)
    out.backward(gout)
    (b64, ba), (a64, aa) = _leaf64(b), _leaf64(a)
    ref, ref_a, params, runs = _ref_chain(layers, torch.cat((b64, a64), 1), torch.cat((ba, aa), 1), before)
    ref.backward(gout.double())
    ref_a.backward(gout.double().abs())
    _check(out, ref, "out of order out")
    _compare(params, runs, before, "out of order")
    _check_sum(a.grad, a64.grad, aa.grad, "out of order source a grad")
    _check_sum(b.grad, b64.grad, ba.grad, "out of order source b grad")


def _group_max_rule(x, G):
    """torch.max(dim)'s rule restated: the first maximal value of each group, a NaN (the first) over any number."""
    B, C, N = x.shape
    v = x.reshape(B, C, N // G, G)
    best, idx = v[..., 0].copy(), np.zeros(v.shape[:3], dtype=np.int32)
    for k in range(1, G):
        take = (v[..., k] > best) | (np.isnan(v[..., k]) & ~np.isnan(best))
        best = np.where(take, v[..., k], best)
        idx = np.where(take, k, idx)
    return best, idx


@pytest.mark.parametrize("G", [1, 4, 16, 77])
def test_group_max_and_sum_against_exact_restatements(G):
    rng = np.random.default_rng(G)
    x = rng.integers(-3, 4, size=(2, 5, 77 * 16)).astype(np.float32)        # many ties
    x[0, 0, :G] = 2.0                                                        # a group of all-equal values
    x[1, 2, 3] = np.nan                                                      # a NaN in a group
    x[1, 3, 1], x[1, 3, 2] = np.nan, np.nan
    xt = torch.from_numpy(x).cuda()
    with torch.cuda.device(0):
        _, mx, idx = point_ops._chain_group_max(point_ops._chain_operand([xt]), 2, 77 * 16, 5, G, False)
        s = point_ops._chain_group_sum(point_ops._chain_operand([xt]), 2, 77 * 16, 5, G)
    best, bi = _group_max_rule(x, G)
    assert np.array_equal(mx.cpu().numpy(), best, equal_nan=True)
    assert np.array_equal(idx.cpu().numpy(), bi)
    tv, ti = torch.max(xt.view(2, 5, -1, G), dim=3)
    assert torch.equal(tv.isnan(), mx.isnan()) and torch.equal(tv[~tv.isnan()], mx[~mx.isnan()])
    assert torch.equal(ti.int()[~tv.isnan()], idx[~tv.isnan()])
    want = np.cumsum(x.astype(np.float64).reshape(2, 5, -1, G), axis=3)[..., -1].astype(np.float32)
    assert np.array_equal(s.cpu().numpy(), want, equal_nan=True)


def _run_once():
    m = _model("kitti")
    a = _run_knn(m, 2, 128, 128, 16, 7)
    res = [a["out"].detach(), a["naf"][0]] + [p.grad for p in a["knn"].parameters()] + \
        [b.clone() for b in a["knn"].buffers()]
    b = _run_node("node_b", "kitti", 2, 128, 8)
    res += [b["out"].detach()] + [p.grad for p in b["pn"].parameters()] + [v[0] for v in b["inputs"].values()]
    return res


def test_two_runs_are_bit_identical():
    a, b = _run_once(), _run_once()
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def _inputs(S, seed):
    rng = np.random.default_rng(seed)
    smps = [synthetic.make_sample(seed + s, 20480, "kitti") for s in range(S)]
    pc = torch.from_numpy(np.stack([s["points"] for s in smps])).cuda()
    idx = torch.from_numpy(np.stack([rng.permutation(20480)[:256] for _ in range(S)])).cuda()
    nodes = torch.gather(pc, 2, idx.unsqueeze(1).expand(S, 3, 256))
    return dict(pc=pc, intensity=torch.from_numpy(rng.random((S, 1, 20480), dtype=np.float32)).cuda(),
                sn=torch.from_numpy(rng.standard_normal((S, 3, 20480), dtype=np.float32)).cuda(),
                node_a=nodes[:, :, :128].contiguous(), node_b=nodes[:, :, 128:].contiguous(),
                img=torch.from_numpy(rng.random((S, 3, 160, 512), dtype=np.float32)).cuda(),
                K=torch.from_numpy(np.stack([s["K"] for s in smps])).float().cuda(),
                P=torch.from_numpy(np.stack([s["P_gt"][:3] for s in smps])).float().cuda())


ARGS = ("pc", "intensity", "sn", "node_a", "node_b", "img")


def _seeded(point_layers, fine=True):
    m = network.KeypointDetector(**network.SHAPES["kitti"], fine=fine, point_layers=point_layers)
    m.load_state_dict(synthetic.seeded_state_dict(m, 1))
    return m.cuda()


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm()).item()


# The whole model's scores in train mode, "fused_all" against the torch layers with dropout off, as a relative 2-norm:
# measured 7.9e-3 on an H100 (TF32 products in every point layer against cuDNN's, and max-pool arg-maxes that move
# where rounding reorders near-equal features), so 2^-6 leaves a margin while a wiring error would be of order one.
MODEL_SCORE_REL = 2 ** -6
# Its parameter gradients, the same way.  Unlike the module tests, the two models' max-pools (cluster_max_pool, the kNN
# module's two maxes, the global max) each pick their own arg-max, so a near-tie that rounds the other way sends a
# group's whole gradient to another column, and that reaches every layer below it.  The largest difference measured on
# an H100 was 2.4e-1, first_pointnet's first weight, below cluster_max_pool (the bound of test_point_chain_gpu.py's
# whole-model test for the same reason); a wiring error would be of order one.
MODEL_GRAD_REL = 2 ** -1


def _normed_bias(mod, k):
    """A conv bias followed by BatchNorm: its gradient is 0 plus rounding on both sides, so it is not compared."""
    return k.endswith("conv.bias") and mod.get_submodule(k[:-len(".conv.bias")]).norm is not None


# Gradients that are zero plus rounding: each is a sum over the whole batch of a gradient that reaches the loss only
# through batch-statistics BatchNorm layers (via weights that sum to one: a broadcast over the nodes, the
# interpolations), and BatchNorm's input gradient sums to zero over the batch.  What is left is rounding on both sides
# (cuDNN's TF32 products against the fused path's), so they are not compared.
BATCH_CANCELLING = {"pc_encoder.final_pointnet.layers.1.norm.bias", "node_b_pn.layers.2.conv.bias",
                    "node_a_pn.layers.2.conv.bias"}


def test_train_mode_model_matches_the_torch_layers_without_dropout():
    inp = _inputs(2, 60)
    args = [inp[k] for k in ARGS]
    models, outs = {}, {}
    for mode in ("torch", "fused_all"):
        m = _seeded(mode).train()
        for layer in m.per_point_pn.layers:
            layer.dropout = None
        scores = torch.cat(m(*args), dim=1)
        g = torch.Generator(device="cuda").manual_seed(4)
        (scores * torch.randn(scores.shape, device="cuda", generator=g)).sum().backward()
        models[mode], outs[mode] = m, scores.detach()
    rel = _rel(outs["fused_all"], outs["torch"])
    print(f"whole model scores: relative 2-norm difference {rel:.2e}")
    assert rel < MODEL_SCORE_REL
    t, f = models["torch"], models["fused_all"]
    rels = {k: _rel(pf.grad, pt.grad) for (k, pt), pf in zip(t.named_parameters(), f.parameters())
            if pt.grad is not None and "img_encoder" not in k and not _normed_bias(t, k) and k not in BATCH_CANCELLING}
    worst = max(rels, key=rels.get)
    print(f"whole model parameter gradients: largest relative 2-norm difference {rels[worst]:.2e} ({worst})")
    bad = [(k, v) for k, v in rels.items() if v >= MODEL_GRAD_REL]
    assert not bad, bad
    for (k, bt), bf in zip(t.named_buffers(), f.buffers()):
        if bt.dtype == torch.int64:
            assert torch.equal(bt, bf), k
        elif "running" in k:
            assert _rel(bf, bt) < 2 ** -6, k


@pytest.mark.parametrize("fine", [True, False])
def test_eval_mode_is_fused_inference_bit_for_bit(fine):
    inp = _inputs(2, 40)
    args = [inp[k] for k in ARGS]
    m = _seeded("fused_all", fine).eval()
    with torch.no_grad():
        got = m(*args)
        want = network.FusedInference(m, encoder="fused", decoder="fused").classify(*args, return_scores=True)[-1]
    got = torch.cat(got, dim=1) if fine else got
    assert torch.equal(got, want)
    with pytest.raises(RuntimeError, match="no backward"):
        m(*args)


def _state(model, opt):
    out = {("model", k): v.clone() for k, v in model.state_dict().items()}
    for i, p in enumerate(model.parameters()):
        for k, v in opt.state[p].items():
            out[("adam", i, k)] = v.clone()
    return out


def test_captured_fused_all_step_is_the_eager_step_bit_for_bit():
    flags = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark, \
        torch.are_deterministic_algorithms_enabled()
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    torch.use_deterministic_algorithms(True)
    try:
        batches = [_inputs(2, 100 + k) for k in range(6)]

        def run(capture):
            model = _seeded("fused_all")
            model.point_chain_state.copy_(point_ops.new_dropout_state(11, "cuda"))
            opt = train.make_optimizer(model)
            static = {k: torch.empty_like(v) for k, v in batches[0].items()}
            stats, losses = torch.zeros(5, device="cuda"), []
            torch.cuda.manual_seed(7)
            graph = None
            for k, b in enumerate(batches):
                for n, v in b.items():
                    static[n].copy_(v)
                if not capture or k < train.WARMUP_STEPS:
                    stats.copy_(train._stats(train.train_step(model, opt, static)))
                else:
                    if graph is None:
                        opt.zero_grad(set_to_none=True)
                        graph = torch.cuda.CUDAGraph()
                        with torch.cuda.graph(graph):
                            stats.copy_(train._stats(train.train_step(model, opt, static)))
                    graph.replay()
                losses.append(stats.clone())
            torch.cuda.synchronize()
            return _state(model, opt), torch.stack(losses), model.point_chain_state.clone()

        s_eager, l_eager, d_eager = run(False)
        s_graph, l_graph, d_graph = run(True)
        assert torch.equal(l_eager, l_graph)
        assert torch.equal(d_eager, d_graph)
        bad = [k for k in s_eager if not torch.equal(s_eager[k], s_graph[k])]
        assert not bad, f"{len(bad)} tensors differ, first {bad[:3]}"
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = flags[:2]
        torch.use_deterministic_algorithms(flags[2])


def _step_peak(mode, B=8):
    inp = _inputs(B, 200)
    m = _seeded(mode).train()
    opt = train.make_optimizer(m)
    train.train_step(m, opt, inp)                 # allocator and workspaces warm
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    train.train_step(m, opt, inp)
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def test_eager_step_peak_memory_in_each_mode():
    peaks = {mode: _step_peak(mode) for mode in network.POINT_LAYERS}
    print("eager KITTI step peak above the resident state, B = 8 (MiB):",
          {k: round(v / 2 ** 20) for k, v in peaks.items()})
    assert peaks["fused_all"] < peaks["fused"]
