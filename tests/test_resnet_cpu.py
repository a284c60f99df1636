"""The host side of the fused ResNet-34 image encoder (DESIGN.md 4.30): BatchNorm folding of every convolution
(downsample branches included) against the module in float64, the oracle without rounding against the module and its
bound against a float32 evaluation in another summation order, the argument checks of resnet.py and of the C ABI, and
FusedInference's re-fold after a weight change, none of which needs a GPU."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle_resnet
from oracle_pointwise import tf32_round
from deepi2p_b200 import network, resnet


def seeded_backbone(seed):
    """A float64 _ResNet34 in eval mode whose BatchNorm layers have non-trivial statistics and affine parameters."""
    torch.manual_seed(seed)
    bb = network._ResNet34().double()
    with torch.no_grad():
        for m in bb.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.running_mean.normal_(0, 0.3)
                m.running_var.uniform_(0.5, 2.0)
                m.weight.uniform_(0.5, 1.5)
                m.bias.normal_(0, 0.2)
    return bb.eval()


def test_fold_equals_the_module_in_float64():
    bb = seeded_backbone(1)
    img = torch.randn(2, 3, 64, 96, dtype=torch.float64, generator=torch.Generator().manual_seed(2))
    folded = network.fold_resnet34(bb, dtype=torch.float64)
    assert len(folded) == 1 + 2 * 16 + 3 and "fc" not in " ".join(folded)
    assert [k for k in folded if k.endswith("downsample")] == ["layer2.0.downsample", "layer3.0.downsample",
                                                               "layer4.0.downsample"]
    assert folded["conv1"][0].shape == (64, 7, 7, 3) and folded["layer3.0.downsample"][0].shape == (256, 1, 1, 128)
    with torch.no_grad():
        s16, s32 = bb(img)
        f16, f32, g = oracle_resnet.backbone(folded, img)
    for want, got in ((s16, f16), (s32, f32)):
        want = want.reshape(got.shape)
        assert torch.allclose(got, want, rtol=1e-10, atol=1e-10 * want.abs().max().item())
    assert torch.allclose(g, s32.mean(dim=(2, 3)), rtol=1e-10, atol=1e-12)
    f32_ = network.fold_resnet34(bb)
    assert all(W.dtype == torch.float32 and b.dtype == torch.float32 for W, b in f32_.values())
    assert torch.equal(f32_["layer2.0.conv2"][0], folded["layer2.0.conv2"][0].float())


def np_layer(folded, name):
    W, b = folded[name]
    return W.float().numpy(), b.float().numpy()


def test_oracle_without_rounding_equals_the_module():
    bb = seeded_backbone(3)
    folded = network.fold_resnet34(bb, dtype=torch.float64)
    rng = np.random.default_rng(3)
    img = rng.normal(0, 1, (2, 3, 37, 50)).astype(np.float32)
    W, b = np_layer(folded, "conv1")
    got = oracle_resnet.stem(img, W, b, tf32=False)
    with torch.no_grad():
        t = torch.from_numpy(img).double()
        want = F.max_pool2d(F.relu(F.conv2d(t, torch.from_numpy(W).double().permute(0, 3, 1, 2),
                                            torch.from_numpy(b).double(), stride=2, padding=3)), 3, 2, 1)
    np.testing.assert_allclose(got["out"], want.permute(0, 2, 3, 1).numpy(), rtol=1e-12, atol=1e-12)
    assert not got["bound"].any()
    # layer2's first block: 3x3 stride 2, then 3x3 with the downsample as the shortcut
    x = np.maximum(rng.normal(0, 1, (2, 9, 13, 64)), 0).astype(np.float32)
    W1, b1 = np_layer(folded, "layer2.0.conv1")
    W2, b2 = np_layer(folded, "layer2.0.conv2")
    Wd, bd = np_layer(folded, "layer2.0.downsample")
    y = oracle_resnet.conv(x, W1, b1, 2, tf32=False)["out"].astype(np.float32)
    out = oracle_resnet.conv(y, W2, (b2.astype(np.float64) + bd).astype(np.float32), 1, shortcut=(x, Wd, 2),
                             tf32=False)["out"]
    with torch.no_grad():
        xt = torch.from_numpy(x).permute(0, 3, 1, 2).double()
        yt = torch.from_numpy(y).permute(0, 3, 1, 2).double()
        c2 = F.conv2d(yt, torch.from_numpy(W2).double().permute(0, 3, 1, 2), torch.from_numpy(b2).double(), padding=1)
        sc = F.conv2d(xt, torch.from_numpy(Wd).double().permute(0, 3, 1, 2), torch.from_numpy(bd).double(), stride=2)
        want = F.relu(c2 + sc).permute(0, 2, 3, 1).numpy()
    np.testing.assert_allclose(out, want, rtol=1e-6, atol=1e-6 * np.abs(want).max())


def test_oracle_bound_covers_float32_evaluation():
    """torch's float32 convolution of the TF32-rounded operands sums in its own order; the oracle's bound covers it,
    including the residual, the fused shortcut and the stem's max-pool."""
    rng = np.random.default_rng(5)
    x = np.maximum(rng.normal(0, 1, (2, 7, 11, 64)), 0).astype(np.float32)
    W = rng.normal(0, 0.05, (64, 3, 3, 64)).astype(np.float32)
    b = rng.normal(0, 0.3, 64).astype(np.float32)
    res = rng.normal(0, 1, (2, 7, 11, 64)).astype(np.float32)
    ref = oracle_resnet.conv(x, W, b, 1, residual=res)
    t = lambda a: torch.from_numpy(tf32_round(a))
    with torch.no_grad():
        z = F.conv2d(t(x).permute(0, 3, 1, 2), t(W).permute(0, 3, 1, 2), torch.from_numpy(b), padding=1)
        got = F.relu(z.permute(0, 2, 3, 1) + torch.from_numpy(res)).double().numpy()
    assert np.all(np.abs(got - ref["out"]) <= ref["bound"]) and ref["bound"].max() > 0
    # with a fused shortcut: the two products are two float32 sums added once
    x2 = np.maximum(rng.normal(0, 1, (2, 13, 21, 32)), 0).astype(np.float32)
    Wd = rng.normal(0, 0.1, (64, 1, 1, 32)).astype(np.float32)
    ref = oracle_resnet.conv(x, W, b, 1, shortcut=(x2, Wd, 2))
    with torch.no_grad():
        z = F.conv2d(t(x).permute(0, 3, 1, 2), t(W).permute(0, 3, 1, 2), torch.from_numpy(b), padding=1)
        z = z + F.conv2d(t(x2).permute(0, 3, 1, 2), t(Wd).permute(0, 3, 1, 2), stride=2)
        got = F.relu(z).permute(0, 2, 3, 1).double().numpy()
    assert np.all(np.abs(got - ref["out"]) <= ref["bound"])
    img = rng.normal(0, 1, (2, 3, 33, 41)).astype(np.float32)
    Ws = rng.normal(0, 0.1, (64, 7, 7, 3)).astype(np.float32)
    ref = oracle_resnet.stem(img, Ws, b)
    with torch.no_grad():
        z = F.conv2d(t(img), t(Ws).permute(0, 3, 1, 2), torch.from_numpy(b), stride=2, padding=3)
        got = F.max_pool2d(F.relu(z), 3, 2, 1).permute(0, 2, 3, 1).double().numpy()
    assert got.shape == ref["out"].shape == (2, 9, 11, 64)
    assert np.all(np.abs(got - ref["out"]) <= ref["bound"])


def test_oracle_max_pool_propagates_nan():
    y = np.zeros((1, 4, 4, 1))
    y[0, 0, 0, 0] = np.nan
    y[0, 3, 3, 0] = np.inf
    v, e = oracle_resnet.max_pool(y, np.ones_like(y))
    # output (i, j) covers input rows and columns 2i-1 .. 2i+1: only (0, 0) sees the NaN, only (1, 1) the infinity
    assert np.isnan(v[0, 0, 0, 0]) and v[0, 0, 1, 0] == 0 and v[0, 1, 0, 0] == 0 and v[0, 1, 1, 0] == np.inf
    assert e[0, 0, 0, 0] == 0 and e[0, 1, 1, 0] == 0 and v.shape == (1, 2, 2, 1)


def test_argument_validation_without_gpu():
    layer = resnet.PackedConv(torch.zeros(64 * 576), torch.zeros(64), 3, 64, 64)
    with pytest.raises(TypeError):
        resnet.conv2d_fused(torch.zeros(1, 4, 4, 64), "not a layer", 1)
    with pytest.raises(ValueError, match="stride"):
        resnet.conv2d_fused(torch.zeros(1, 4, 4, 64), layer, 3)
    with pytest.raises(ValueError, match="channels"):
        resnet.conv2d_fused(torch.zeros(1, 4, 4, 32), layer, 1)
    with pytest.raises(TypeError, match="float32"):
        resnet.conv2d_fused(torch.zeros(1, 4, 4, 64, dtype=torch.float64), layer, 1)
    with pytest.raises(RuntimeError, match="CUDA"):
        resnet.conv2d_fused(torch.zeros(1, 4, 4, 64), layer, 1)
    with pytest.raises(TypeError):
        resnet.resnet34_features(torch.zeros(1, 3, 64, 64), "not packed")
    packed = resnet.PackedResNet34(layer, [])
    with pytest.raises(ValueError, match="too small"):
        resnet.resnet34_features(torch.zeros(1, 3, 31, 64), packed)
    with pytest.raises(ValueError, match=r"\[B,3,H,W\]"):
        resnet.resnet34_features(torch.zeros(1, 4, 64, 64), packed)
    with pytest.raises(RuntimeError, match="CUDA"):
        resnet.resnet34_features(torch.zeros(1, 3, 64, 64), packed)
    with pytest.raises(ValueError, match="C_out"):
        resnet.pack_conv(torch.zeros(12, 3, 3, 64), torch.zeros(12))
    with pytest.raises(ValueError, match="fold_resnet34"):
        resnet.pack_resnet34({})


def test_native_validation_without_gpu():
    from deepi2p_b200 import _native
    lib = _native.load()
    assert lib.resnet_conv_packed_bytes(64, 147) == 64 * 160 * 4
    assert lib.resnet_conv_packed_bytes(128, 9 * 64 + 64) == 128 * 640 * 4
    assert lib.resnet_conv_packed_bytes(0, 147) == 0
    buf = (ctypes.c_float * 1024)()
    a = ctypes.addressof(buf)
    aligned = a + (-a) % 16
    assert lib.resnet_conv_pack_f32(None, 64, 147, aligned, 1 << 20, None) == -22
    assert lib.resnet_conv_pack_f32(aligned, 64, 147, aligned, 16, None) == -12
    args = lambda **kw: [kw.get(k, v) for k, v in (
        ("x", aligned), ("nchw", 0), ("B", 2), ("H", 8), ("W", 8), ("C_in", 64), ("kernel", 3), ("stride", 1),
        ("pad", 1), ("shortcut", None), ("H2", 0), ("W2", 0), ("C2", 0), ("stride2", 2), ("packed", aligned),
        ("packed_bytes", 1 << 30), ("bias", aligned), ("residual", None), ("relu", 1), ("C_out", 64),
        ("out_nhwc", aligned), ("out_cm", None), ("stream", None))]
    for kw, text in ((dict(C_out=12), b"multiple of 8"), (dict(C_in=48), b"C_in % 32"), (dict(x=None), b"NULL"),
                     (dict(out_nhwc=None), b"both outputs"), (dict(stride=3), b"stride"),
                     (dict(kernel=3, pad=3), b"pad"), (dict(B=0), b"B"), (dict(x=aligned + 4), b"16-byte"),
                     (dict(packed_bytes=64), b"packed"), (dict(H=1, W=1, pad=0), b"smaller than the kernel"),
                     (dict(shortcut=aligned, H2=18, W2=16, C2=64), b"strided size"),
                     (dict(shortcut=aligned, H2=16, W2=16, C2=48), b"shortcut"),
                     (dict(nchw=1, C_in=3, kernel=7, stride=2, pad=3, shortcut=aligned, H2=4, W2=4, C2=64),
                      b"shortcut")):
        assert lib.resnet_conv_f32(*args(**kw)) == -22, kw
        assert text in lib.dib_last_error(), (kw, lib.dib_last_error())
    assert lib.resnet_maxpool_f32(None, 1, 4, 4, 64, aligned, None) == -22
    assert lib.resnet_maxpool_f32(aligned, 1, 0, 4, 64, aligned, None) == -22
    assert lib.resnet_mean_f32(aligned, 4, 0, aligned, None) == -22
    assert b"P >= 1" in lib.dib_last_error()


def test_fused_inference_refolds_after_a_weight_change(monkeypatch):
    """The backbone is folded once and folded again when a parameter or buffer it reads has changed."""
    model = network.KeypointDetector(img_H=64, img_W=128).eval()
    calls = []

    def fake_pack(folded):
        calls.append(folded)
        return len(calls)
    monkeypatch.setattr(resnet, "pack_resnet34", fake_pack)
    with pytest.raises(ValueError, match="image"):
        network.FusedInference(model, image="cudnn")
    fused = network.FusedInference(model, encoder="fused", decoder="fused", image="fused")
    assert fused._chain("resnet") == 1 and fused._chain("resnet") == 1
    assert calls[0]["layer4.0.downsample"][0].shape == (512, 1, 1, 256)
    with torch.no_grad():
        model.img_encoder.backbone.layer3[2].bn2.running_var.mul_(2.0)
    assert fused._chain("resnet") == 2
    assert not torch.equal(calls[0]["layer3.2.conv2"][0], calls[1]["layer3.2.conv2"][0])
    assert torch.equal(calls[0]["layer3.1.conv2"][0], calls[1]["layer3.1.conv2"][0])
    assert "fused_image" in network.HEADS and network.HEADS[0] == "torch"
