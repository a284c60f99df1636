"""The fused ResNet-34 image encoder on the H100 (DESIGN.md 4.30): every layer kind of resnet.conv2d_fused and the stem
against oracle_resnet within the oracle's own error bound at the layer shapes of the KITTI, Oxford and nuScenes images
and at the edges, NaN and infinity agreement with torch's rules, repeatability on any stream, the whole backbone
against the float64 module, network.FusedInference(image="fused") against the reference network's float64 scores
(tests/golden/network_small.npz), and classify_and_register(head="fused_image")."""
import os

import numpy as np
import pytest
import torch

import oracle_resnet
from deepi2p_b200 import frustum, network, resnet, synthetic

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "network_small.npz")
# |fused - ref64| <= TOL_FACTOR * 2^-10 * max|ref64| per output tensor (DESIGN.md 4.30 records the measured ratios)
TOL_FACTOR = 8.0
ORDER = ("pc", "intensity", "sn", "node_a", "node_b", "img")


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def check(name, got, ref):
    """got (torch) against the oracle: the same NaN and infinities, every finite value within its bound."""
    got = got.double().cpu().numpy()
    out, bound = ref["out"], ref["bound"]
    assert got.shape == out.shape, (name, got.shape, out.shape)
    assert np.array_equal(np.isnan(got), np.isnan(out)), name
    inf = np.isinf(out)
    assert np.array_equal(got[inf], out[inf]) and not np.isinf(got[~inf]).any(), name
    fin = np.isfinite(out)
    excess = np.abs(got[fin] - out[fin]) - bound[fin]
    assert excess.max(initial=-1.0) <= 0, (name, excess.max())


def make_conv(rng, C_in, C_out, k, shortcut_c=0):
    W = rng.normal(0, np.sqrt(2.0 / (k * k * C_in)), (C_out, k, k, C_in)).astype(np.float32)
    b = rng.normal(0, 0.1, C_out).astype(np.float32)
    if not shortcut_c:
        return W, b, None, resnet.pack_conv(cu(W), cu(b))
    Wd = rng.normal(0, np.sqrt(1.0 / shortcut_c), (C_out, 1, 1, shortcut_c)).astype(np.float32)
    bd = rng.normal(0, 0.1, C_out).astype(np.float32)
    return W, b + bd, Wd, resnet.pack_conv(cu(W), cu(b), shortcut=(cu(Wd), cu(bd)))


def act(rng, *shape):
    return np.maximum(rng.normal(0, 1, shape), 0).astype(np.float32)


def run_conv(rng, B, H, W_, C_in, C_out, k, stride, kind):
    """One layer of `kind` ("plain", "residual", "shortcut", "stage_end", "last") on the device and in the oracle."""
    x = act(rng, B, H, W_, C_in)
    Ho, Wo = (H + 2 * (k // 2) - k) // stride + 1, (W_ + 2 * (k // 2) - k) // stride + 1
    if kind == "shortcut":                      # the block's second conv: its input is y, its shortcut the block input
        W, b, Wd, layer = make_conv(rng, C_out, C_out, 3, shortcut_c=C_in)
        y = act(rng, B, Ho, Wo, C_out)
        got = resnet.conv2d_fused(cu(y), layer, 1, shortcut=cu(x), shortcut_stride=stride)
        return got, oracle_resnet.conv(y, W, b, 1, shortcut=(x, Wd, stride))
    W, b, _, layer = make_conv(rng, C_in, C_out, k)
    res = rng.normal(0, 1, (B, Ho, Wo, C_out)).astype(np.float32) if kind in ("residual", "stage_end", "last") else None
    ref = oracle_resnet.conv(x, W, b, stride, residual=res)
    r = None if res is None else cu(res)
    if kind == "stage_end":
        nhwc, cm = resnet.conv2d_fused(cu(x), layer, stride, residual=r, channel_major=True)
        assert torch.equal(cm, nhwc.reshape(B, Ho * Wo, C_out).transpose(1, 2))
        return cm, dict(out=ref["out"].reshape(B, Ho * Wo, C_out).transpose(0, 2, 1),
                        bound=ref["bound"].reshape(B, Ho * Wo, C_out).transpose(0, 2, 1))
    if kind == "last":
        nhwc, cm = resnet.conv2d_fused(cu(x), layer, stride, residual=r, channel_major=True, nhwc=False)
        assert nhwc is None
        return cm, dict(out=ref["out"].reshape(B, Ho * Wo, C_out).transpose(0, 2, 1),
                        bound=ref["bound"].reshape(B, Ho * Wo, C_out).transpose(0, 2, 1))
    return resnet.conv2d_fused(cu(x), layer, stride, residual=r), ref


def map_sizes(H, W):
    """(h, w) after the stem + max-pool and after each stage (strides 4, 4, 8, 16, 32)."""
    down = lambda n, k, p: (n + 2 * p - k) // 2 + 1
    h, w = down(down(H, 7, 3), 3, 1), down(down(W, 7, 3), 3, 1)
    out = [(h, w)]
    for _ in range(3):
        h, w = down(h, 3, 1), down(w, 3, 1)
        out.append((h, w))
    return out


@pytest.mark.parametrize("shape", ["kitti", "oxford", "nuscenes"])
def test_layer_kinds_within_the_oracle_bound(shape):
    H, W = network.SHAPES[shape]["img_H"], network.SHAPES[shape]["img_W"]
    rng = np.random.default_rng(sum(map(ord, shape)))
    B = 1 if shape == "oxford" else 2
    img = rng.normal(0, 1, (B, 3, H, W)).astype(np.float32)
    Ws, bs, _, stem = make_conv(rng, 3, 64, 7)
    got = resnet.stem(cu(img), resnet.PackedResNet34(stem, []))
    check(f"{shape} stem", got, oracle_resnet.stem(img, Ws, bs))
    sizes = map_sizes(H, W)
    (h4, w4), (h8, w8), (h16, w16), (h32, w32) = sizes
    check(f"{shape} layer1 3x3 s1 + residual", *run_conv(rng, B, h4, w4, 64, 64, 3, 1, "residual"))
    check(f"{shape} layer2 3x3 s2", *run_conv(rng, B, h4, w4, 64, 128, 3, 2, "plain"))
    check(f"{shape} layer2 downsample", *run_conv(rng, B, h4, w4, 64, 128, 3, 2, "shortcut"))
    check(f"{shape} layer3 3x3 s2", *run_conv(rng, B, h8, w8, 128, 256, 3, 2, "plain"))
    check(f"{shape} layer4 downsample", *run_conv(rng, B, h16, w16, 256, 512, 3, 2, "shortcut"))
    check(f"{shape} layer3 end", *run_conv(rng, B, h16, w16, 256, 256, 3, 1, "stage_end"))
    check(f"{shape} layer4 end", *run_conv(rng, B, h32, w32, 512, 512, 3, 1, "last"))


@pytest.mark.parametrize("case", [
    (1, 5, 7, 64, 64, 3, 1, "residual"),        # B = 1, odd H and W
    (2, 1, 1, 64, 64, 3, 1, "residual"),        # a 1 x 1 output
    (1, 2, 2, 128, 256, 3, 2, "plain"),         # 1 x 1 from stride 2
    (1, 1, 129, 32, 72, 3, 1, "plain"),         # M one more than a tile, C_out not a multiple of 64
    (3, 1, 43, 64, 64, 3, 1, "stage_end"),      # M = 129 over three samples
    (1, 3, 5, 64, 128, 3, 2, "shortcut"),       # odd sizes through the fused downsample
    (2, 2, 4, 512, 512, 3, 1, "last"),          # the golden shape's stride-32 map
])
def test_edges_within_the_oracle_bound(case):
    B, H, W, C_in, C_out, k, stride, kind = case
    check(str(case), *run_conv(np.random.default_rng(H * 1000 + W), B, H, W, C_in, C_out, k, stride, kind))


def test_stem_edges():
    rng = np.random.default_rng(11)
    Ws, bs, _, stem = make_conv(rng, 3, 64, 7)
    for B, H, W in ((1, 1, 1), (2, 5, 9), (1, 33, 65)):
        img = rng.normal(0, 1, (B, 3, H, W)).astype(np.float32)
        check(f"stem {B}x{H}x{W}", resnet.stem(cu(img), resnet.PackedResNet34(stem, [])),
              oracle_resnet.stem(img, Ws, bs))


def seeded_backbone(seed):
    torch.manual_seed(seed)
    bb = network._ResNet34()
    with torch.no_grad():
        for m in bb.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.running_mean.normal_(0, 0.3)
                m.running_var.uniform_(0.5, 2.0)
                m.weight.uniform_(0.5, 1.5)
                m.bias.normal_(0, 0.2)
    return bb.cuda().eval()


def test_nan_and_infinities_follow_torch():
    bb = seeded_backbone(21)
    folded = network.fold_resnet34(bb)
    packed = resnet.pack_resnet34(folded)
    # the float64 reference runs on the CPU, whose direct convolution propagates NaN and infinity element by element
    folded64 = {k: (W.cpu(), b.cpu()) for k, (W, b) in network.fold_resnet34(bb, dtype=torch.float64).items()}
    gen = torch.Generator().manual_seed(21)
    img = torch.randn(3, 3, 64, 128, generator=gen).cuda()
    with torch.no_grad():
        clean = resnet.resnet34_features(img, packed)
        bad = img.clone()
        bad[1, 0, 10, 20] = float("nan")
        bad[1, 2, 40, 100] = float("inf")
        got = resnet.resnet34_features(bad, packed)
        want = [t.cuda() for t in oracle_resnet.backbone(folded64, bad.double().cpu())]
    for name, c, g, w in zip(("s16", "s32", "img_global"), clean, got, want):
        for s in (0, 2):                               # the other samples are untouched, bit for bit
            assert torch.equal(c[s].view(torch.int32), g[s].view(torch.int32)), (name, s)
        assert torch.isnan(g[1]).any(), name
        assert torch.equal(torch.isnan(g), torch.isnan(w)), name
        assert torch.equal(torch.isinf(g), torch.isinf(w)), name
    # a NaN weight: every sample's output channel 5 of layer3.1.conv1 is NaN, and whatever torch spreads it to
    folded["layer3.1.conv1"][0][5, 1, 1, 7] = float("nan")
    folded64["layer3.1.conv1"][0][5, 1, 1, 7] = float("nan")
    with torch.no_grad():
        got = resnet.resnet34_features(img, resnet.pack_resnet34(folded))
        want = [t.cuda() for t in oracle_resnet.backbone(folded64, img.double().cpu())]
    for name, g, w in zip(("s16", "s32", "img_global"), got, want):
        assert torch.isnan(g).any(), name
        assert torch.equal(torch.isnan(g), torch.isnan(w)), name


def test_repeatable_on_any_stream():
    bb = seeded_backbone(22)
    packed = resnet.pack_resnet34(network.fold_resnet34(bb))
    img = torch.rand(3, 3, 160, 320, generator=torch.Generator().manual_seed(22)).cuda()
    with torch.no_grad():
        a = resnet.resnet34_features(img, packed)
        b = resnet.resnet34_features(img, packed)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            c = resnet.resnet34_features(img, packed)
        torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for x, y, z in zip(a, b, c):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))
        assert torch.equal(x.view(torch.int32), z.view(torch.int32))
    assert [tuple(t.shape) for t in a] == [(3, 256, 10 * 20), (3, 512, 5 * 10), (3, 512)]


@pytest.mark.parametrize("shape", ["kitti", "oxford"])
def test_backbone_against_the_float64_module(shape):
    bb = seeded_backbone(23)
    H, W = network.SHAPES[shape]["img_H"], network.SHAPES[shape]["img_W"]
    img = torch.rand(2, 3, H, W, generator=torch.Generator().manual_seed(23)).cuda()
    with torch.no_grad():
        got = resnet.resnet34_features(img, resnet.pack_resnet34(network.fold_resnet34(bb)))
        bb64 = bb.double()
        s16, s32 = bb64(img.double())
        want = (s16.reshape(2, 256, -1), s32.reshape(2, 512, -1), s32.mean(dim=(2, 3)))
    ratios = []
    for name, g, w in zip(("s16", "s32", "img_global"), got, want):
        unit = 2.0 ** -10 * float(w.abs().max())
        ratios.append(float((g.double() - w).abs().max()) / unit)
        print(f"{shape} {name}: max|fused - ref64| = {ratios[-1]:.3f} x 2^-10 max|ref64|")
    assert max(ratios) <= TOL_FACTOR, ratios


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def small_model(g):
    model = network.KeypointDetector(img_H=64, img_W=128)
    model.load_state_dict(synthetic.seeded_state_dict(model, int(g["weight_seed"])))
    return model.cuda()


def small_inputs(g):
    x = synthetic.make_network_inputs(int(g["input_seed"]))
    return [torch.from_numpy(x[k]).cuda() for k in ORDER]


def test_fused_image_matches_the_reference_network(golden):
    model = small_model(golden).eval()
    x = small_inputs(golden)
    fused = network.FusedInference(model, encoder="fused", decoder="fused", image="fused")
    with torch.no_grad():
        c, f, scores = fused.classify(*x, return_scores=True)
        c2, f2, scores2 = fused.classify(*x, return_scores=True)
    assert torch.equal(scores.view(torch.int32), scores2.view(torch.int32))
    assert torch.equal(c, c2) and torch.equal(f, f2)
    stride = int(golden["point_stride"])
    for name, got, key in (("coarse", scores[:, :2], "eval_coarse"), ("fine", scores[:, 2:], "eval_fine")):
        ref64 = golden[key]
        unit = 2.0 ** -10 * np.abs(ref64).max()
        err = np.abs(got[..., ::stride].cpu().numpy().astype(np.float64) - ref64).max()
        print(f"fused encoder + decoder + image {name}: max|fused - ref64| {err:.3e} = {err / unit:.3f} x 2^-10 "
              f"max|ref64|")
        assert err <= TOL_FACTOR * unit, (name, err / unit)


def test_classify_and_register_fused_image():
    dev = torch.device("cuda")
    gen = torch.Generator().manual_seed(801)
    S = 3
    smps = [synthetic.make_sample(810 + s, 20480, "kitti") for s in range(S)]
    pc = torch.from_numpy(np.stack([s["points"] for s in smps]))
    idx = torch.stack([torch.randperm(20480, generator=gen)[:256] for _ in range(S)])
    nodes = torch.gather(pc, 2, idx.unsqueeze(1).expand(S, 3, 256))
    b = [pc, torch.rand(S, 1, 20480, generator=gen),
         torch.nn.functional.normalize(torch.randn(S, 3, 20480, generator=gen), dim=1),
         nodes[:, :, :128].contiguous(), nodes[:, :, 128:].contiguous(), torch.rand(S, 3, 160, 512, generator=gen)]
    b = [t.to(dev) for t in b]
    K = torch.from_numpy(np.stack([s["K"] for s in smps])).float().to(dev)
    model = network.KeypointDetector(**network.SHAPES["kitti"])
    model.load_state_dict(synthetic.seeded_state_dict(model, 4))
    model = model.to(dev).train()
    out = network.classify_and_register(model, *b, K, chunk=2, head="fused_image")
    assert model.training
    assert out["coarse_pred"].dtype == torch.int8 and out["fine_pred"].dtype == torch.int32
    assert out["P"].dtype == torch.float64 and tuple(out["P"].shape) == (S, 4, 4)
    assert out["cost"].dtype == torch.float64 and out["degenerate"].dtype == torch.int32
    fused = network.FusedInference(model, encoder="fused", decoder="fused", image="fused")
    ref_head = network.FusedInference(model, encoder="fused", decoder="fused")
    with torch.no_grad():
        parts = [fused.classify(*(t[a:a + 2] for t in b)) for a in (0, 2)]
        ref = [ref_head.classify(*(t[a:a + 2] for t in b), return_scores=True) for a in (0, 2)]
    c, f = torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts])
    assert torch.equal(out["coarse_pred"], c) and torch.equal(out["fine_pred"], f)
    reg = frustum.register_batch(b[0], c, 20480, K, 160, 512)
    for k in ("P", "cost", "degenerate"):
        assert torch.equal(out[k], reg[k]), k
    # against head="fused_all": the same predictions wherever the top two scores do not nearly tie
    scores = torch.cat([r[2] for r in ref])
    for name, pred, sc, want in (("coarse", c, scores[:, :2], torch.cat([r[0] for r in ref])),
                                 ("fine", f, scores[:, 2:], torch.cat([r[1] for r in ref]))):
        top = torch.topk(sc, 2, dim=1)[0]
        unit = 2.0 ** -10 * float(sc.abs().max())
        sure = (top[:, 0] - top[:, 1]) > 2 * TOL_FACTOR * unit
        print(f"fused_image {name}: {(pred == want).float().mean():.4f} of the predictions equal fused_all's; "
              f"{sure.float().mean():.4f} are decided beyond the tolerance")
        assert torch.equal(pred[sure], want[sure]), name
