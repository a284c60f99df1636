"""The host side of the fused node-level PointNets (DESIGN.md 4.27): BatchNorm folding with the per-sample columns split
off against the modules in float64, the oracle's once-per-sample projection against a float64 evaluation of the
modules and against a float32 evaluation, the argument and limit checks of point_ops.node_mlp and of the C ABI, and
FusedInference's re-fold after a weight change, none of which needs a GPU."""
import numpy as np
import pytest
import torch

import oracle_node_mlp
from oracle_pointwise import tf32_round
from deepi2p_b200 import network, point_ops


def seeded_pointnet(c_in, widths, seed, norm_act_at_last=False):
    """A float64 _PointNet in eval mode whose BatchNorm layers have non-trivial statistics and affine parameters."""
    torch.manual_seed(seed)
    pn = network._PointNet(c_in, widths, norm_act_at_last).double()
    with torch.no_grad():
        for layer in pn.layers:
            layer.conv.bias.normal_(0, 0.3)
            if layer.norm is not None:
                layer.norm.running_mean.normal_(0, 0.5)
                layer.norm.running_var.uniform_(0.3, 2.0)
                layer.norm.weight.uniform_(0.5, 1.5)
                layer.norm.bias.normal_(0, 0.2)
    return pn.eval()


def module_input(sources, M):
    """torch.cat of the sources with each per-sample [B,C] source expanded over the M columns, as network.py does."""
    return torch.cat([torch.from_numpy(np.asarray(s, np.float64)) if s.ndim == 3 else
                      torch.from_numpy(np.asarray(s, np.float64))[:, :, None].expand(-1, -1, M) for s in sources], dim=1)


def layers_np(folded):
    return [(W.numpy(), b.numpy(), act) for W, b, act in folded]


def make_sources(rng, B, M, spec):
    return [rng.normal(0, 1, (B, c) if bc else (B, c, M)).astype(np.float32) for c, bc in spec]


# node_b_pn's layout at small widths: dense, per sample, dense, per sample
SPEC = ((6, False), (5, True), (7, False), (4, True))


def test_fold_with_per_sample_columns_equals_the_module():
    pn = seeded_pointnet(22, [16, 12, 9], 1)
    rng = np.random.default_rng(1)
    src = make_sources(rng, 3, 11, SPEC)
    with torch.no_grad():
        want = pn(module_input(src, 11))
    folded = network.fold_pointnet(pn, dtype=torch.float64)
    assert [act for _, _, act in folded] == [True, True, False]
    W1 = folded[0][0]
    dense = torch.cat([torch.from_numpy(s).double() for s in src if s.ndim == 3], dim=1)
    bc = torch.cat([torch.from_numpy(s).double() for s in src if s.ndim == 2], dim=1)
    dcols = list(range(0, 6)) + list(range(11, 18))
    bcols = list(range(6, 11)) + list(range(18, 22))
    x = torch.einsum("oc,bcm->bom", W1[:, dcols], dense) + (bc @ W1[:, bcols].T)[:, :, None] \
        + folded[0][1][None, :, None]
    x = torch.relu(x)
    for W, b, act in folded[1:]:
        x = torch.einsum("oc,bcm->bom", W, x) + b[None, :, None]
        x = torch.relu(x) if act else x
    assert float((x - want).abs().max()) <= 1e-12 * float(want.abs().max())


@pytest.mark.parametrize("spec", [SPEC, ((9, False),), ((5, True), (4, True)), ((3, True), (8, False), (2, False))])
def test_oracle_without_rounding_equals_the_module(spec):
    c_in = sum(c for c, _ in spec)
    pn = seeded_pointnet(c_in, [14, 10], 2)
    rng = np.random.default_rng(2)
    M = 9
    src = make_sources(rng, 3, M, spec)
    bc = [i for i, (_, b) in enumerate(spec) if b]
    if bc:
        src[bc[0]][1, 2] = np.nan                             # a NaN per-sample value: every column of sample 1
    with torch.no_grad():
        want = pn(module_input(src, M)).numpy()
    got = oracle_node_mlp.node_mlp(src, layers_np(network.fold_pointnet(pn, dtype=torch.float64)), tf32=False, M=M)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got["out"]), nan)
    if bc:
        assert nan[1].all() and not nan[[0, 2]].any()
    assert np.nanmax(np.abs(got["out"] - want)) <= 1e-12 * np.nanmax(np.abs(want))
    assert not got["bound"].any()


def test_oracle_bound_covers_float32_evaluation():
    """The bound covers a float32 evaluation of the concatenated formulation on the same rounded operands, the
    projection is the kernel's float32 fma chain, and TF32 rounding moves the output by more than float32 could."""
    pn = seeded_pointnet(22, [40, 24, 17], 3)
    rng = np.random.default_rng(3)
    M = 13
    src = make_sources(rng, 2, M, SPEC)
    layers = layers_np(network.fold_pointnet(pn))
    ref = oracle_node_mlp.node_mlp(src, layers)
    exact = oracle_node_mlp.node_mlp(src, layers, tf32=False)
    assert np.isfinite(ref["out"]).all() and (ref["bound"] > 0).all()
    assert np.abs(ref["out"] - exact["out"]).max() > 10 * np.finfo(np.float32).eps
    r = tf32_round
    x = r(module_input(src, M).numpy().astype(np.float32))
    for i, (W, b, act) in enumerate(layers):
        x = np.einsum("oc,bcm->bom", r(W), x, dtype=np.float32) + b[None, :, None]
        x = np.maximum(x, 0) if act else x
        if i < len(layers) - 1:
            x = r(x)
    assert (np.abs(x.astype(np.float64) - ref["out"]) <= ref["bound"]).all()
    # the projection equals a float32 fma chain (float64 product, one rounding per step) in ascending row
    W1 = r(layers[0][0])
    v = r(np.concatenate([s for s in src if s.ndim == 2], axis=1))
    Wb = W1[:, [6, 7, 8, 9, 10, 18, 19, 20, 21]]
    p, _, bound = oracle_node_mlp.project(layers[0][0][:, [6, 7, 8, 9, 10, 18, 19, 20, 21]], v)
    acc = np.zeros(p.shape, dtype=np.float32)
    for c in range(Wb.shape[1]):
        acc = (v[:, c:c + 1].astype(np.float64) * Wb[None, :, c] + acc).astype(np.float32)
    assert np.array_equal(acc.astype(np.float64), p) and not bound.any()


def test_projection_bound_where_a_product_underflows():
    """A product of two TF32 values below float32's normal range can be inexact: only there is the term non-zero."""
    t = 2.0 ** -70 * (1 + 2.0 ** -10)                         # t * t needs a bit at 2^-160, below float32's 2^-149
    W = np.array([[t, 1.0]], dtype=np.float32)
    v = np.array([[t, 3.0]], dtype=np.float32)
    p, mag, bound = oracle_node_mlp.project(W, v)
    assert p[0, 0] == 3.0 and bound[0, 0] >= 2 * 2 * 2.0 ** -148
    p, _, bound = oracle_node_mlp.project(np.array([[1.0, 2.0]], np.float32), np.array([[3.0, 4.0]], np.float32))
    assert p[0, 0] == 11.0 and bound[0, 0] == 0


def gpu_free_layers(c_in, widths):
    return [(torch.zeros(c, ci), torch.zeros(c), True) for ci, c in zip([c_in] + list(widths), widths)]


def test_argument_validation_without_gpu():
    d, g = torch.zeros(2, 6, 9), torch.zeros(2, 5)
    ok = gpu_free_layers(11, [8])
    bad = [
        ([], ok), ([d, g], gpu_free_layers(10, [8])),                        # no source; W does not match the rows
        ([d, g], gpu_free_layers(11, [8] * 4)), ([d, g], []),                # four layers; none
        ([d, g], gpu_free_layers(11, [1025])),                               # a layer wider than 1024
        ([d, torch.zeros(3, 5)], ok),                                        # sample counts differ
        ([d, torch.zeros(2, 6, 8)], gpu_free_layers(12, [8])),               # column counts differ
        ([torch.zeros(2, 6, 9, 1)], gpu_free_layers(6, [8])),                # a 4-D source
        ([torch.zeros(2, 1025, 3)], gpu_free_layers(1025, [8])),             # more than 1024 dense rows
        ([torch.zeros(2, 600, 3), torch.zeros(2, 500, 3)], gpu_free_layers(1100, [8])),
        ([d, torch.zeros(2, 65537)], gpu_free_layers(65543, [8])),          # more than 65536 per-sample rows
        ([d] * 5, gpu_free_layers(30, [8])),                                 # five dense sources
        ([torch.zeros(2, 6, 0)], gpu_free_layers(6, [8])),                   # no columns
        ([g], gpu_free_layers(5, [8])),                                      # per sample only, M not given
        ([torch.zeros(2, 0, 9)], gpu_free_layers(0, [8])),                   # a source without channels
    ]
    for sources, layers in bad:
        with pytest.raises(ValueError):
            point_ops.node_mlp(sources, layers)
    with pytest.raises(RuntimeError):                         # well-formed but not on a GPU: no CPU fallback
        point_ops.node_mlp([d, g], ok)
    with pytest.raises(RuntimeError):
        point_ops.node_mlp([g], gpu_free_layers(5, [8]), M=4)
    with pytest.raises(RuntimeError):                         # no backward
        point_ops.node_mlp([d, g.clone().requires_grad_(True)], ok)
    for spec in ([], [(0, False)], [(3, False)] * 5, [(600, False), (500, False)], [(70000, True)]):
        with pytest.raises(ValueError):
            point_ops.pack_node_mlp(spec, gpu_free_layers(sum(c for c, _ in spec), [4]))
    with pytest.raises(ValueError):
        network.FusedInference(network.KeypointDetector(img_H=64, img_W=128), decoder="cudnn")
    assert "fused_all" in network.HEADS


def test_native_validation_without_gpu():
    from deepi2p_b200 import _native
    lib = _native.load()
    src = np.zeros((4, 8), dtype=np.int64)
    src[:, 2], src[:, 7] = (6, 5, 7, 4), (0, 1, 0, 1)
    lay = np.zeros((3, 4), dtype=np.int64)
    lay[:, 2], lay[:, 3] = (20, 12, 9), (1, 1, 0)
    # 13 dense rows (padded to 16) -> 20 (padded to 32) -> 12 -> 9: the fragments of 32 x 16, 16 x 32 and 16 x 16
    # weights, the biases 32 + 16 + 16 and the per-sample columns transposed, 9 x 32
    want = (32 * 16 + 16 * 32 + 16 * 16 + 32 + 16 + 16 + 9 * 32) * 4
    assert lib.node_mlp_packed_bytes(src.ctypes.data, 4, lay.ctypes.data, 3) == want
    assert lib.node_mlp_workspace_bytes(src.ctypes.data, 4, lay.ctypes.data, 3, 64) == 64 * 32 * 4
    dense = src[[0, 2]].copy()
    assert lib.node_mlp_workspace_bytes(dense.ctypes.data, 2, lay.ctypes.data, 3, 64) == 0
    lay[0, 2] = 1025
    assert lib.node_mlp_packed_bytes(src.ctypes.data, 4, lay.ctypes.data, 3) == 0
    assert b"C_out <= 1024" in lib.dib_last_error()
    lay[0, 2] = 1024
    assert lib.node_mlp_packed_bytes(src.ctypes.data, 4, lay.ctypes.data, 3) > 0
    assert lib.node_mlp_packed_bytes(src.ctypes.data, 4, lay.ctypes.data, 4) == 0
    assert b"1 to 3 layers" in lib.dib_last_error()
    src[1, 7] = 2
    assert lib.node_mlp_packed_bytes(src.ctypes.data, 4, lay.ctypes.data, 3) == 0
    assert b"BCAST" in lib.dib_last_error()
    src[1, 7], src[1, 3] = 1, 16                               # an interpolated source is not supported
    assert lib.node_mlp_packed_bytes(src.ctypes.data, 4, lay.ctypes.data, 3) == 0
    assert b"NODES" in lib.dib_last_error()
    src[1, 3], src[0, 2] = 0, 1018                             # 1018 + 7 dense rows
    assert lib.node_mlp_packed_bytes(src.ctypes.data, 4, lay.ctypes.data, 3) == 0
    assert b"1024 rows" in lib.dib_last_error()
    src[0, 2], src[1, 2] = 1017, 65533                          # 1024 dense and 65537 per-sample rows
    assert lib.node_mlp_packed_bytes(src.ctypes.data, 4, lay.ctypes.data, 3) == 0
    assert b"65536 per-sample" in lib.dib_last_error()
    src[1, 2] = 65532
    assert lib.node_mlp_packed_bytes(src.ctypes.data, 4, lay.ctypes.data, 3) > 0
    src[1, 2] = 5
    five = np.zeros((5, 8), dtype=np.int64)
    five[:, 2] = 3
    assert lib.node_mlp_packed_bytes(five.ctypes.data, 5, lay.ctypes.data, 3) == 0
    assert b"4 dense" in lib.dib_last_error()
    five[:, 7] = 1                                             # any number of per-sample sources
    assert lib.node_mlp_packed_bytes(five.ctypes.data, 5, lay.ctypes.data, 3) > 0
    src[0, 2] = 6
    # a NULL source, a short batch stride and a NULL packed buffer are rejected before anything is launched
    assert lib.node_mlp_f32(src.ctypes.data, 4, lay.ctypes.data, 3, None, 0, 2, 9, None, None, 0, None) == -22
    assert b"NULL" in lib.dib_last_error()
    src[:, 0] = 256
    src[:, 1] = (6 * 9, 5, 7 * 9 - 1, 4)
    assert lib.node_mlp_f32(src.ctypes.data, 4, lay.ctypes.data, 3, None, 0, 2, 9, None, None, 0, None) == -22
    assert b"batch stride" in lib.dib_last_error()
    assert lib.node_mlp_f32(src.ctypes.data, 4, lay.ctypes.data, 3, None, 0, 0, 9, None, None, 0, None) == 0


def test_fused_inference_refolds_after_a_weight_change(monkeypatch):
    """The node chains are folded once and folded again when a parameter or buffer they read has changed."""
    model = network.KeypointDetector(img_H=64, img_W=128).eval()
    calls = []

    def fake_pack(spec, layers):
        calls.append((list(spec), [W.clone() for W, _, _ in layers]))
        return len(calls)
    monkeypatch.setattr(point_ops, "pack_node_mlp", fake_pack)
    fused = network.FusedInference(model, encoder="fused", decoder="fused")
    assert fused._chain("node_b") == 1 and fused._chain("node_b") == 1
    assert calls[0][0] == [(256, False), (512, True), (512, False), (512, True)]
    assert [W.shape for W in calls[0][1]] == [(1024, 1792), (512, 1024), (512, 512)]
    with torch.no_grad():
        model.node_b_pn.layers[0].norm.running_var.mul_(2.0)
    assert fused._chain("node_b") == 2
    assert not torch.equal(calls[0][1][0], calls[1][1][0])
    assert fused._chain("att_b") == 3 and fused._chain("att_b") == 3
    assert calls[2][0] == [(256, False), (512, True)] and calls[2][1][-1].shape == (model.node_b_attention_pn.layers[
        -1].conv.out_channels, 256)
    assert fused._chain("att_a") == 4 and calls[3][0] == [(64, False), (512, True)]
    assert fused._chain("node_a") == 5 and calls[4][0] == [(64, False), (512, False), (256, False)]
