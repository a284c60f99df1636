"""The fused per-point layers on the H100 (DESIGN.md 4.21): point_ops.pointwise_mlp against oracle_pointwise within the
oracle's own error bound at every shipped chain and at the edges, network.FusedInference against the reference
network's float64 scores (tests/golden/network_small.npz) and against the unfused float32 path, and
classify_and_register(head="fused") against its parts."""
import os

import numpy as np
import pytest
import torch

import oracle_pointwise
from deepi2p_b200 import frustum, network, point_ops, synthetic

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "network_small.npz")
# |fused - ref64| <= FUSED_TOL_FACTOR * 2^-10 * max|ref64| per score tensor (DESIGN.md 4.21 records the measured ratio)
FUSED_TOL_FACTOR = 8.0
ORDER = ("pc", "intensity", "sn", "node_a", "node_b", "img")


def make_layers(rng, c_in, widths, relus, bias_scale=0.1):
    layers = []
    for c, r in zip(widths, relus):
        layers.append((rng.normal(0, np.sqrt(2.0 / c_in), (c, c_in)).astype(np.float32),
                       rng.normal(0, bias_scale, c).astype(np.float32), r))
        c_in = c
    return layers


def dense_sources(rng, B, N, widths):
    return [rng.normal(0, 1, (B, c, N)).astype(np.float32) for c in widths]


def interp_source(rng, B, N, C, M, k=3, bad=()):
    """Node features and the weights / indices interp_weights_f32 writes for random points and nodes; the points in
    `bad` get an out-of-range neighbour."""
    pc = torch.from_numpy(rng.uniform(-10, 10, (B, 3, N)).astype(np.float32)).cuda()
    nd = torch.from_numpy(rng.uniform(-10, 10, (B, 3, M)).astype(np.float32)).cuda()
    topk = point_ops.cluster_assign_forward(pc, nd, k=k, want_centers=False)["min_k_idx"]
    for b, n in bad:
        topk[b, n, k - 1] = M + 7
    w, idx = point_ops.interpolation_weights(topk, pc, nd)
    return rng.normal(0, 1, (B, C, M)).astype(np.float32), w.cpu().numpy(), idx.cpu().numpy()


def to_gpu(sources, layers):
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    src = [tuple(cu(t) for t in s) if isinstance(s, tuple) else cu(s) for s in sources]
    lay = [(cu(W), None if b is None else cu(b), r) for W, b, r in layers]
    return src, lay


def check_scores(name, got, ref):
    """|gpu - oracle| <= the oracle's bound where the oracle is finite; the same NaN / infinity elsewhere."""
    got = got.astype(np.float64)
    fin = np.isfinite(ref["out"])
    assert np.array_equal(got[~fin], ref["out"][~fin], equal_nan=True), name
    err, bound = np.abs(got - ref["out"])[fin], ref["bound"][fin]
    if err.size:
        print(f"{name}: max err {err.max():.3e}, max err / bound {np.max(err / np.maximum(bound, 1e-300)):.3f}")
    assert (err <= bound).all(), (name, float(err.max()))


def check_argmax(name, pred_a, pred_b, scores, ref, c_split):
    """The predictions are torch.max's rule on the kernel's own scores exactly, and the oracle's wherever the
    oracle's top-two margin exceeds twice the bound."""
    pairs = ((pred_a, 0, c_split, "a"), (pred_b, c_split, scores.shape[1], "b"))
    for pred, lo, hi, r in pairs:
        if lo >= hi:
            assert pred is None and ref["pred_" + r] is None
            continue
        assert np.array_equal(pred.astype(np.int64), oracle_pointwise.argmax_rule(scores[:, lo:hi].astype(np.float64)))
        bound = ref["bound"][:, lo:hi].max(axis=1)
        with np.errstate(invalid="ignore"):
            sure = (ref["margin_" + r] > 2 * bound) | np.isnan(ref["out"][:, lo:hi]).any(axis=1)
        print(f"{name} range {r}: {sure.mean():.4f} of the points are decided beyond the bound")
        assert np.array_equal(pred[sure], ref["pred_" + r][sure]), (name, r)


def run(sources, layers, c_split=None):
    src, lay = to_gpu(sources, layers)
    with torch.no_grad():
        if c_split is None:
            return point_ops.pointwise_mlp(src, lay).cpu().numpy()
        a, b, s = point_ops.pointwise_mlp(src, lay, output="argmax", c_split=c_split, return_scores=True)
    return a.cpu().numpy(), None if b is None else b.cpu().numpy(), s.cpu().numpy()


CHAINS = {
    "first_pointnet": dict(dense=[3, 1, 3], widths=[32, 32, 32], relus=[True, True, True]),
    "second_pointnet": dict(dense=[32, 32], widths=[64, 64], relus=[True, True]),
    "head_L50": dict(interp=True, dense=[32, 64], widths=[256, 256, 52], relus=[True, True, False]),
    "head_L80": dict(interp=True, dense=[32, 64], widths=[256, 256, 82], relus=[True, True, False]),
    "head_L240": dict(interp=True, dense=[32, 64], widths=[256, 256, 242], relus=[True, True, False]),
    "head_coarse_only": dict(interp=True, dense=[32, 64], widths=[128, 128, 2], relus=[True, True, False]),
    "golden_small_head": dict(interp=True, dense=[32, 64], widths=[256, 256, 10], relus=[True, True, False]),
}


def chain_case(name, B=2, N=333, seed=0, bad=()):
    c = CHAINS[name]
    rng = np.random.default_rng(seed)
    sources = []
    if c.get("interp"):
        sources += [interp_source(rng, B, N, 128, 128, bad=bad), interp_source(rng, B, N, 512, 128)]
    sources += dense_sources(rng, B, N, c["dense"])
    c_in = sum(s[0].shape[1] if isinstance(s, tuple) else s.shape[1] for s in sources)
    return sources, make_layers(rng, c_in, c["widths"], c["relus"])


@pytest.mark.parametrize("name", list(CHAINS))
def test_every_output_mode_within_the_oracle_bound(name):
    sources, layers = chain_case(name)
    C = layers[-1][0].shape[0]
    ref = oracle_pointwise.pointwise_mlp(sources, layers, c_split=min(2, C))
    act = run(sources, layers)
    check_scores(name + " activations", act, ref)
    a, b, s = run(sources, layers, c_split=min(2, C))
    assert np.array_equal(s, act)                          # the scores of the arg-max mode are the activations
    check_argmax(name, a, b, s, ref, min(2, C))
    src, lay = to_gpu(sources, layers)
    with torch.no_grad():
        a2, b2 = point_ops.pointwise_mlp(src, lay, output="argmax", c_split=min(2, C))
    assert np.array_equal(a2.cpu().numpy(), a) and (b is None or np.array_equal(b2.cpu().numpy(), b))
    assert a2.dtype == torch.int8 and (b2 is None or b2.dtype == torch.int32)


def test_single_point_and_odd_widths():
    rng = np.random.default_rng(1)
    for N, dense, widths in ((1, [5], [1]), (1, [7, 2], [17, 3]), (65, [9], [250, 33, 7]), (130, [1000, 24], [40])):
        sources = dense_sources(rng, 3, N, dense)
        layers = make_layers(rng, sum(dense), widths, [True] * (len(widths) - 1) + [False])
        ref = oracle_pointwise.pointwise_mlp(sources, layers)
        check_scores(f"N={N} {dense}->{widths}", run(sources, layers), ref)


def test_narrow_layers_after_interpolated_sources():
    """First layers narrower than one 128-channel gather step, and one that ends inside a step."""
    rng = np.random.default_rng(7)
    for widths in ([40, 24, 8], [200], [5, 3]):
        sources = [interp_source(rng, 2, 150, 24, 16), interp_source(rng, 2, 150, 9, 40, k=2)]
        sources += dense_sources(rng, 2, 150, [8])
        layers = make_layers(rng, 24 + 9 + 8, widths, [True] * (len(widths) - 1) + [False])
        check_scores(f"interpolated -> {widths}", run(sources, layers), oracle_pointwise.pointwise_mlp(sources, layers))
    sources = [interp_source(rng, 2, 150, 24, 16)]                       # no dense source at all
    layers = make_layers(rng, 24, [48, 6], [True, False])
    check_scores("interpolated only", run(sources, layers), oracle_pointwise.pointwise_mlp(sources, layers))


def test_bad_interpolation_index_gives_nan_scores_and_index_zero():
    sources, layers = chain_case("head_L50", bad=((0, 5), (1, 332)))
    assert (sources[0][2][0, 5] == -1).all() and np.isnan(sources[0][1][1, 332]).all()
    ref = oracle_pointwise.pointwise_mlp(sources, layers, c_split=2)
    a, b, s = run(sources, layers, c_split=2)
    check_scores("bad index", s, ref)
    assert np.isnan(s[0, :, 5]).all() and np.isnan(s[1, :, 332]).all() and np.isnan(s).sum() == 2 * s.shape[1]
    assert a[0, 5] == 0 and b[0, 5] == 0 and a[1, 332] == 0 and b[1, 332] == 0
    check_argmax("bad index", a, b, s, ref, 2)


def test_nan_and_infinities_in_a_dense_source():
    sources, layers = chain_case("head_L50", seed=2)
    sources[2][0, 3, 10] = np.nan
    sources[3][1, 0, 20] = np.inf
    sources[3][1, 1, 21] = -np.inf
    ref = oracle_pointwise.pointwise_mlp(sources, layers, c_split=2)
    a, b, s = run(sources, layers, c_split=2)
    check_scores("non-finite", s, ref)
    assert np.isnan(s[0, :, 10]).all() and a[0, 10] == 0 and b[0, 10] == 0
    assert not np.isfinite(s[1, :, 20]).any() and not np.isfinite(s[1, :, 21]).any()
    check_argmax("non-finite", a, b, s, ref, 2)
    other = np.ones(s.shape, dtype=bool)
    other[0, :, 10] = other[1, :, 20] = other[1, :, 21] = False
    assert np.isfinite(s[other]).all()                      # the other points of the tile are untouched


def test_exact_ties_take_the_lowest_index():
    sources, layers = chain_case("head_L80", seed=3)
    W, b, r = layers[2]
    W[:] = W[0]
    b[:] = b[0]
    a, f, s = run(sources, layers, c_split=2)
    assert (s == s[:, :1]).all()                            # equal rows give bit-equal scores
    assert not a.any() and not f.any()
    W[40], b[40] = 2 * W[0], 2 * b[0]                       # channel 40 wins where the score is positive
    a, f, s = run(sources, layers, c_split=2)
    assert np.array_equal(f, np.where(s[:, 0] > 0, 38, 0)) and (s[:, 0] > 0).any() and (s[:, 0] < 0).any()


def test_all_negative_preactivations_zero_a_layer():
    sources, layers = chain_case("head_L50", seed=4)
    layers[0][1][:] = -1e6
    ref = oracle_pointwise.pointwise_mlp(sources, layers)
    got = run(sources, layers)
    check_scores("relu zeros layer 1", got, ref)
    assert (got == got[:1, :, :1]).all()                    # a constant: the later layers see zeros only


def test_channel_slice_stream_and_repeatability():
    sources, layers = chain_case("second_pointnet", N=1000, seed=5)
    src, lay = to_gpu(sources, layers)
    wide = torch.randn(2, 80, 1000, device="cuda")
    wide[:, 7:39] = src[0]
    with torch.no_grad():
        want = point_ops.pointwise_mlp(src, lay)
        again = point_ops.pointwise_mlp(src, lay)
        sliced = point_ops.pointwise_mlp([wide[:, 7:39], src[1]], lay)
        stream = torch.cuda.Stream()
        stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(stream):
            other = point_ops.pointwise_mlp(src, lay)
        stream.synchronize()
        packed = point_ops.pack_pointwise_mlp([(32, 0, 0), (32, 0, 0)], lay)
        pre = point_ops.pointwise_mlp(src, packed)
    for t in (again, sliced, other, pre):
        assert torch.equal(t, want)
    sources, layers = chain_case("head_L240", seed=6)
    assert all(np.array_equal(x, y) for x, y in zip(run(sources, layers, c_split=2), run(sources, layers, c_split=2)))


def test_requires_grad_raises():
    src, lay = to_gpu(*chain_case("first_pointnet"))
    src[0].requires_grad_(True)
    with pytest.raises(RuntimeError):
        point_ops.pointwise_mlp(src, lay)
    with torch.no_grad():
        point_ops.pointwise_mlp(src, lay)


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


def test_fused_inference_matches_the_reference_network(golden, no_tf32):
    model = small_model(golden).train()
    x = small_inputs(golden)
    fused = network.FusedInference(model)
    with pytest.raises(RuntimeError):
        fused.classify(*x)                                   # inference only
    with torch.no_grad():
        c, f, scores = fused.classify(*x, return_scores=True)
        assert model.training                                # the flag is restored
        c2, f2 = fused.classify(*x)
        model.eval()
        tc, tf = model(*x)
        pc, pf = network.predict(tc, tf)
    assert torch.equal(c, c2) and torch.equal(f, f2)
    assert c.dtype == torch.int8 and f.dtype == torch.int32
    stride = int(golden["point_stride"])
    for name, got, key, torch_scores, pred, tpred in (("coarse", scores[:, :2], "eval_coarse", tc, c, pc),
                                                      ("fine", scores[:, 2:], "eval_fine", tf, f, pf)):
        ref64 = golden[key]
        tol = FUSED_TOL_FACTOR * 2.0 ** -10 * np.abs(ref64).max()
        err = np.abs(got[..., ::stride].cpu().numpy().astype(np.float64) - ref64).max()
        print(f"fused {name}: max|fused - ref64| {err:.3e} = {err / (2.0 ** -10 * np.abs(ref64).max()):.3f} "
              f"x 2^-10 max|ref64|")
        assert err <= tol, (name, err, tol)
        top = torch.topk(torch_scores, 2, dim=1)[0]
        sure = (top[:, 0] - top[:, 1]) > 2 * tol
        print(f"fused {name}: predictions agree with the float32 path at {(pred == tpred).float().mean():.4f} of the "
              f"points; {sure.float().mean():.4f} are decided beyond the tolerance")
        assert torch.equal(pred[sure], tpred[sure]), name


def test_new_weights_are_picked_up(golden):
    model = small_model(golden).eval()
    x = small_inputs(golden)
    fused = network.FusedInference(model)
    with torch.no_grad():
        _, _, s0 = fused.classify(*x, return_scores=True)
        model.load_state_dict(synthetic.seeded_state_dict(model, 77))
        _, _, s1 = fused.classify(*x, return_scores=True)
        _, _, want = network.FusedInference(model).classify(*x, return_scores=True)
    assert not torch.equal(s0, s1) and torch.equal(s1, want)


def test_classify_and_register_fused_equals_its_parts():
    dev = torch.device("cuda")
    gen = torch.Generator().manual_seed(600)
    S = 3
    smps = [synthetic.make_sample(600 + s, 20480, "oxford") for s in range(S)]
    pc = torch.from_numpy(np.stack([s["points"] for s in smps]))
    idx = torch.stack([torch.randperm(20480, generator=gen)[:256] for _ in range(S)])
    nodes = torch.gather(pc, 2, idx.unsqueeze(1).expand(S, 3, 256))
    b = [pc, torch.rand(S, 1, 20480, generator=gen),
         torch.nn.functional.normalize(torch.randn(S, 3, 20480, generator=gen), dim=1),
         nodes[:, :, :128].contiguous(), nodes[:, :, 128:].contiguous(), torch.rand(S, 3, 384, 640, generator=gen)]
    b = [t.to(dev) for t in b]
    K = torch.from_numpy(np.stack([s["K"] for s in smps])).float().to(dev)
    model = network.KeypointDetector(**network.SHAPES["oxford"])
    model.load_state_dict(synthetic.seeded_state_dict(model, 2))
    model = model.to(dev).train()
    out = network.classify_and_register(model, *b, K, chunk=2, head="fused")
    assert model.training
    fused = network.FusedInference(model)
    with torch.no_grad():
        parts = [fused.classify(*(t[a:a + 2] for t in b)) for a in (0, 2)]
    c, f = torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts])
    assert torch.equal(out["coarse_pred"], c) and torch.equal(out["fine_pred"], f)
    reg = frustum.register_batch(b[0], c, 20480, K, 384, 640)
    for k in ("P", "cost", "degenerate"):
        assert torch.equal(out[k], reg[k]), k
    with pytest.raises(ValueError):
        network.classify_and_register(model, *b, K, chunk=2, head="cudnn")
