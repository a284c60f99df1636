"""The fused kNN module and global feature on the H100 (DESIGN.md 4.26): point_ops.knn_fusion and pointwise_mlp_max
against oracle_knn_fusion within the oracle's own error bound at the shipped shape and at the edges,
network.FusedInference(encoder="fused") against the reference network's float64 scores
(tests/golden/network_small.npz) and against the float32 path, and classify_and_register(head="fused_encoder")
against its parts."""
import os

import numpy as np
import pytest
import torch

import oracle_knn_fusion
from deepi2p_b200 import frustum, network, point_ops, synthetic

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "network_small.npz")
# |fused encoder - ref64| <= ENCODER_TOL_FACTOR * 2^-10 * max|ref64| per score tensor (DESIGN.md 4.26 records the
# measured ratio)
ENCODER_TOL_FACTOR = 8.0
ORDER = ("pc", "intensity", "sn", "node_a", "node_b", "img")


def make_layers(rng, c_in, widths, bias_scale=0.1, relu=True):
    layers = []
    for c in widths:
        layers.append((rng.normal(0, np.sqrt(2.0 / c_in), (c, c_in)).astype(np.float32),
                       rng.normal(0, bias_scale, c).astype(np.float32), relu))
        c_in = c
    return layers


def knn_layers(rng, C, before, after):
    b = make_layers(rng, 3 + C, before)
    return b, make_layers(rng, 2 * before[-1], after)


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def gpu_layers(layers):
    return [(cu(W), cu(b), r) for W, b, r in layers]


def check(name, got, ref):
    """|gpu - oracle| <= the oracle's bound where the oracle is finite; the same NaN / infinity elsewhere."""
    got = got.astype(np.float64)
    fin = np.isfinite(ref["out"])
    assert got.shape == ref["out"].shape, name
    assert np.array_equal(got[~fin], ref["out"][~fin], equal_nan=True), name
    err, bound = np.abs(got - ref["out"])[fin], ref["bound"][fin]
    if err.size:
        print(f"{name}: max err {err.max():.3e}, max err / bound {np.max(err / np.maximum(bound, 1e-300)):.3f}")
    assert (err <= bound).all(), (name, float(err.max()))


def knn_inputs(rng, B, M, N, C):
    return (rng.uniform(-5, 5, (B, 3, M)).astype(np.float32), rng.uniform(-5, 5, (B, 3, N)).astype(np.float32),
            rng.normal(0, 1, (B, C, N)).astype(np.float32))


def run_knn(q, d, f, K, before, after):
    """(device out, device idx, oracle) for numpy inputs; the oracle groups by knn_group's own output."""
    qg, dg, fg = cu(q), cu(d), cu(f)
    with torch.no_grad():
        out, idx = point_ops.knn_fusion(qg, dg, fg, K, (gpu_layers(before), gpu_layers(after)), return_idx=True)
        gidx, grouped = point_ops.knn_group(qg, dg, fg, K)
    assert torch.equal(idx, gidx)
    ref = oracle_knn_fusion.knn_fusion(grouped.cpu().numpy(), before, after)
    return out.cpu().numpy(), idx.cpu().numpy(), ref


KNN_CASES = {
    # name: (B, M, N, C, K, before, after)
    "shipped": (2, 128, 128, 64, 16, (256, 256), (512, 256)),
    "shipped_ragged_M": (2, 13, 128, 64, 16, (256, 256), (512, 256)),
    "K1": (2, 37, 50, 9, 1, (24, 40), (48, 20)),
    "K32": (2, 20, 40, 9, 32, (24, 40), (48, 20)),
    "K_equals_N": (3, 11, 7, 5, 7, (16, 16), (32, 16)),
    "K3_M1": (1, 1, 9, 5, 3, (16,), (8,)),
    "odd_widths": (2, 21, 30, 13, 5, (13, 21), (37, 5)),
    "one_layer_each": (2, 17, 25, 6, 4, (40,), (9,)),
    "three_layers_each": (2, 19, 33, 7, 6, (24, 40, 17), (33, 19, 11)),
    "widest": (1, 6, 24, 509, 8, (512, 512, 512), (512, 512, 512)),
}


@pytest.mark.parametrize("name", list(KNN_CASES))
def test_knn_fusion_within_the_oracle_bound(name):
    B, M, N, C, K, before, after = KNN_CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    q, d, f = knn_inputs(rng, B, M, N, C)
    out, idx, ref = run_knn(q, d, f, K, *knn_layers(rng, C, before, after))
    assert out.shape == (B, after[-1], M) and idx.shape == (B, M, K)
    assert np.isfinite(out).all()
    check(name, out, ref)


def test_nan_and_infinities_in_the_features():
    rng = np.random.default_rng(3)
    q, d, f = knn_inputs(rng, 2, 40, 64, 16)
    f[0, 3, 5] = np.nan
    f[1, 7, 9] = np.inf
    f[1, 2, 30] = -np.inf
    out, idx, ref = run_knn(q, d, f, 8, *knn_layers(rng, 16, (32, 32), (48, 24)))
    assert (~np.isfinite(ref["out"])).any()
    nan_nodes = (idx[0] == 5).any(axis=1)
    assert nan_nodes.any() and np.isnan(out[0][:, nan_nodes]).all() and not np.isnan(out[0][:, ~nan_nodes]).any()
    check("nan_inf", out, ref)


def test_all_negative_preactivations_zero_a_layer():
    rng = np.random.default_rng(4)
    q, d, f = knn_inputs(rng, 2, 30, 40, 8)
    before, after = knn_layers(rng, 8, (24, 16), (32, 12))
    W, b, r = after[-1]
    after[-1] = (W, np.full_like(b, -1e6), r)
    out, _, ref = run_knn(q, d, f, 6, before, after)
    assert (out == 0).all() and not np.signbit(out).any()
    check("zeroed", out, ref)


def test_stream_and_repeatability():
    rng = np.random.default_rng(5)
    B, M, N, C, K, before, after = KNN_CASES["shipped"]
    q, d, f = (cu(a) for a in knn_inputs(rng, B, M, N, C))
    packed = point_ops.pack_knn_fusion(C, *(gpu_layers(x) for x in knn_layers(rng, C, before, after)))
    with torch.no_grad():
        want = point_ops.knn_fusion(q, d, f, K, packed)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            runs = [point_ops.knn_fusion(q, d, f, K, packed) for _ in range(3)]
        torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    for r in runs:
        assert torch.equal(r.view(torch.int32), want.view(torch.int32))


def test_requires_grad_raises():
    rng = np.random.default_rng(6)
    q, d, f = (cu(a) for a in knn_inputs(rng, 1, 8, 16, 4))
    layers = tuple(gpu_layers(x) for x in knn_layers(rng, 4, (8,), (8,)))
    fg = f.clone().requires_grad_(True)
    with pytest.raises(RuntimeError):
        point_ops.knn_fusion(q, d, fg, 4, layers)
    W = layers[0][0][0].clone().requires_grad_(True)
    with pytest.raises(RuntimeError):
        point_ops.knn_fusion(q, d, f, 4, ([(W, layers[0][0][1], True)], layers[1]))
    with pytest.raises(RuntimeError):
        point_ops.pointwise_mlp_max([fg], gpu_layers(make_layers(rng, 4, [8])))
    with torch.no_grad():
        point_ops.knn_fusion(q, d, fg, 4, layers)


MAX_CASES = {
    # name: (B, N, source widths, layer widths)
    "final_pointnet": (3, 128, (3, 256), (256, 512)),
    "one_column": (2, 1, (3, 5), (7,)),
    "ragged_tile": (2, 33, (4,), (17, 9, 3)),
    "widest": (1, 70, (500, 12), (512, 512, 512)),
}


@pytest.mark.parametrize("name", list(MAX_CASES))
def test_pointwise_mlp_max_within_the_oracle_bound(name):
    B, N, widths, layers = MAX_CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    src = [rng.normal(0, 1, (B, c, N)).astype(np.float32) for c in widths]
    lay = make_layers(rng, sum(widths), layers)
    with torch.no_grad():
        out = point_ops.pointwise_mlp_max([cu(s) for s in src], gpu_layers(lay)).cpu().numpy()
    assert out.shape == (B, layers[-1], 1)
    check(name, out, oracle_knn_fusion.pointwise_mlp_max(src, lay))


def test_pointwise_mlp_max_channel_slice_nan_and_inf():
    rng = np.random.default_rng(8)
    wide = rng.normal(0, 1, (2, 40, 50)).astype(np.float32)
    wide[0, 12, 7] = np.nan
    wide[1, 20, 3] = np.inf
    lay = make_layers(rng, 3 + 20, (16, 24))
    xyz = rng.normal(0, 1, (2, 3, 50)).astype(np.float32)
    with torch.no_grad():
        out = point_ops.pointwise_mlp_max([cu(xyz), cu(wide)[:, 10:30]], gpu_layers(lay)).cpu().numpy()
    ref = oracle_knn_fusion.pointwise_mlp_max([xyz, wide[:, 10:30]], lay)
    assert np.isnan(out[0]).all()
    check("slice_nan_inf", out, ref)


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


@pytest.fixture()
def no_tf32():
    flags = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = flags


def small_model(g, seed=None):
    model = network.KeypointDetector(img_H=64, img_W=128)
    model.load_state_dict(synthetic.seeded_state_dict(model, int(g["weight_seed"]) if seed is None else seed))
    return model.cuda()


def small_inputs(g):
    x = synthetic.make_network_inputs(int(g["input_seed"]))
    return [torch.from_numpy(x[k]).cuda() for k in ORDER]


def test_fused_encoder_matches_the_reference_network(golden, no_tf32):
    model = small_model(golden).eval()
    x = small_inputs(golden)
    fused = network.FusedInference(model, encoder="fused")
    with torch.no_grad():
        c, f, scores = fused.classify(*x, return_scores=True)
        c2, f2, scores2 = fused.classify(*x, return_scores=True)
        tc, tf = model(*x)
        pc, pf = network.predict(tc, tf)
    assert torch.equal(scores.view(torch.int32), scores2.view(torch.int32))
    assert torch.equal(c, c2) and torch.equal(f, f2)
    stride = int(golden["point_stride"])
    for name, got, key, torch_scores, pred, tpred in (("coarse", scores[:, :2], "eval_coarse", tc, c, pc),
                                                      ("fine", scores[:, 2:], "eval_fine", tf, f, pf)):
        ref64 = golden[key]
        unit = 2.0 ** -10 * np.abs(ref64).max()
        err = np.abs(got[..., ::stride].cpu().numpy().astype(np.float64) - ref64).max()
        print(f"fused encoder {name}: max|fused - ref64| {err:.3e} = {err / unit:.3f} x 2^-10 max|ref64|")
        assert err <= ENCODER_TOL_FACTOR * unit, (name, err / unit)
        top = torch.topk(torch_scores, 2, dim=1)[0]
        sure = (top[:, 0] - top[:, 1]) > 2 * ENCODER_TOL_FACTOR * unit
        print(f"fused encoder {name}: predictions agree with the float32 path at "
              f"{(pred == tpred).float().mean():.4f} of the points; {sure.float().mean():.4f} are decided beyond "
              f"the tolerance")
        assert torch.equal(pred[sure], tpred[sure]), name


def test_torch_encoder_is_the_default(golden):
    model = small_model(golden).eval()
    x = small_inputs(golden)
    with torch.no_grad():
        a = network.FusedInference(model).classify(*x, return_scores=True)
        b = network.FusedInference(model, encoder="torch").classify(*x, return_scores=True)
    for u, v in zip(a, b):
        assert torch.equal(u.view(torch.int32) if u.dtype == torch.float32 else u,
                           v.view(torch.int32) if v.dtype == torch.float32 else v)


def test_new_encoder_weights_are_picked_up(golden):
    model = small_model(golden).eval()
    x = small_inputs(golden)
    fused = network.FusedInference(model, encoder="fused")
    with torch.no_grad():
        _, _, s0 = fused.classify(*x, return_scores=True)
        model.pc_encoder.knnlayer.layers_after[0].norm.running_mean.add_(0.5)
        _, _, s1 = fused.classify(*x, return_scores=True)
        _, _, want = network.FusedInference(model, encoder="fused").classify(*x, return_scores=True)
    assert not torch.equal(s0, s1) and torch.equal(s1, want)


def test_classify_and_register_fused_encoder_equals_its_parts():
    dev = torch.device("cuda")
    gen = torch.Generator().manual_seed(601)
    S = 3
    smps = [synthetic.make_sample(610 + s, 20480, "kitti") for s in range(S)]
    pc = torch.from_numpy(np.stack([s["points"] for s in smps]))
    idx = torch.stack([torch.randperm(20480, generator=gen)[:256] for _ in range(S)])
    nodes = torch.gather(pc, 2, idx.unsqueeze(1).expand(S, 3, 256))
    b = [pc, torch.rand(S, 1, 20480, generator=gen),
         torch.nn.functional.normalize(torch.randn(S, 3, 20480, generator=gen), dim=1),
         nodes[:, :, :128].contiguous(), nodes[:, :, 128:].contiguous(), torch.rand(S, 3, 160, 512, generator=gen)]
    b = [t.to(dev) for t in b]
    K = torch.from_numpy(np.stack([s["K"] for s in smps])).float().to(dev)
    model = network.KeypointDetector(**network.SHAPES["kitti"])
    model.load_state_dict(synthetic.seeded_state_dict(model, 3))
    model = model.to(dev).train()
    out = network.classify_and_register(model, *b, K, chunk=2, head="fused_encoder")
    assert model.training
    fused = network.FusedInference(model, encoder="fused")
    with torch.no_grad():
        parts = [fused.classify(*(t[a:a + 2] for t in b)) for a in (0, 2)]
    c, f = torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts])
    assert torch.equal(out["coarse_pred"], c) and torch.equal(out["fine_pred"], f)
    reg = frustum.register_batch(b[0], c, 20480, K, 160, 512)
    for k in ("P", "cost", "degenerate"):
        assert torch.equal(out[k], reg[k]), k
