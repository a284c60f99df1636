"""The host side of the fused kNN module and global feature (DESIGN.md 4.26): BatchNorm folding against _KnnFusion,
the oracle's [max; x] split against the module's own forward and against final_pointnet + max in float64, the bound
against a float32 evaluation, and the argument checks of point_ops.knn_fusion / pointwise_mlp_max and of the C ABI,
none of which needs a GPU."""
import numpy as np
import pytest
import torch

import oracle_knn_fusion
from deepi2p_b200 import network, point_ops


def seeded_knn_fusion(c_in, before, after, seed):
    """A float64 _KnnFusion in eval mode whose BatchNorm layers have non-trivial statistics and affine parameters."""
    torch.manual_seed(seed)
    mod = network._KnnFusion(c_in, before, after).double()
    with torch.no_grad():
        for layer in list(mod.layers_before) + list(mod.layers_after):
            layer.conv.bias.normal_(0, 0.3)
            layer.norm.running_mean.normal_(0, 0.5)
            layer.norm.running_var.uniform_(0.3, 2.0)
            layer.norm.weight.uniform_(0.5, 1.5)
            layer.norm.bias.normal_(0, 0.2)
    return mod.eval()


def seeded_pointnet(c_in, widths, seed):
    torch.manual_seed(seed)
    pn = network._PointNet(c_in, widths, True).double()
    with torch.no_grad():
        for layer in pn.layers:
            layer.conv.bias.normal_(0, 0.3)
            layer.norm.running_mean.normal_(0, 0.5)
            layer.norm.running_var.uniform_(0.3, 2.0)
            layer.norm.weight.uniform_(0.5, 1.5)
            layer.norm.bias.normal_(0, 0.2)
    return pn.eval()


def knn_case(seed, B=2, M=7, N=11, C=5, K=4):
    rng = np.random.default_rng(seed)
    q = rng.uniform(-3, 3, (B, 3, M)).astype(np.float32)
    d = rng.uniform(-3, 3, (B, 3, N)).astype(np.float32)
    f = rng.normal(0, 1, (B, C, N)).astype(np.float32)
    return q, d, f, oracle_knn_fusion.knn_indices(q, d, K)


def numpy_knn_group(idx):
    """A stand-in for point_ops.knn_group (CUDA only) that groups by the given indices."""
    def knn_group(query, database, features, K):
        g = oracle_knn_fusion.group(query.float().numpy(), database.float().numpy(), features.float().numpy(), idx)
        return torch.from_numpy(idx), torch.from_numpy(g.astype(np.float64))
    return knn_group


def layers_np(folded):
    return [(W.numpy(), b.numpy(), act) for W, b, act in folded]


def test_fold_knn_fusion_equals_the_module(monkeypatch):
    mod = seeded_knn_fusion(3 + 5, (12, 9), (14, 6), 3)
    q, d, f, idx = knn_case(1)
    monkeypatch.setattr(point_ops, "knn_group", numpy_knn_group(idx))
    with torch.no_grad():
        want = mod(torch.from_numpy(q).double(), torch.from_numpy(d).double(), torch.from_numpy(f).double(), 4)
    before, after = network.fold_knn_fusion(mod, dtype=torch.float64)
    assert [W.shape for W, _, _ in before] == [(12, 8), (9, 12)]
    assert [W.shape for W, _, _ in after] == [(14, 18), (6, 14)]
    assert all(act for _, _, act in before + after)
    x = torch.from_numpy(oracle_knn_fusion.group(q, d, f, idx)).double()
    for W, b, _ in before:
        x = torch.relu(torch.einsum("oc,bcmk->bomk", W, x) + b[None, :, None, None])
    x = torch.cat((x.max(dim=3, keepdim=True)[0].expand_as(x), x), dim=1)
    for W, b, _ in after:
        x = torch.relu(torch.einsum("oc,bcmk->bomk", W, x) + b[None, :, None, None])
    got = x.max(dim=3)[0]
    assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max())
    b32, a32 = network.fold_knn_fusion(mod)
    assert all(W.dtype == torch.float32 and torch.equal(W, W64.float()) for (W, _, _), (W64, _, _) in
               zip(b32 + a32, before + after))


@pytest.mark.parametrize("K", [1, 4, 11])
def test_oracle_without_rounding_equals_the_module(monkeypatch, K):
    """The [max; x] split with the max projected once per node is the module's torch.cat formulation."""
    mod = seeded_knn_fusion(3 + 5, (12, 9), (14, 6), 4)
    q, d, f, idx = knn_case(2, K=K)
    f[1, 2, 3] = np.nan                                       # a NaN feature: every query that groups node 3 is NaN
    monkeypatch.setattr(point_ops, "knn_group", numpy_knn_group(idx))
    with torch.no_grad():
        want = mod(torch.from_numpy(q).double(), torch.from_numpy(d).double(), torch.from_numpy(f).double(), K)
    before, after = network.fold_knn_fusion(mod, dtype=torch.float64)
    got = oracle_knn_fusion.knn_fusion(oracle_knn_fusion.group(q, d, f, idx), layers_np(before), layers_np(after),
                                       tf32=False)
    nan = torch.isnan(want).numpy()
    assert np.array_equal(np.isnan(got["out"]), nan)
    assert nan[1].any() == (idx[1] == 3).any() and not nan[0].any()
    assert np.nanmax(np.abs(got["out"] - want.numpy())) <= 1e-12 * float(np.nanmax(np.abs(want.numpy())))
    assert not got["bound"].any()


def test_oracle_bound_covers_float32_evaluation(monkeypatch):
    """The bound covers a float32 evaluation of the torch formulation on the same rounded operands, and TF32 rounding
    moves the output by more than float32 accumulation could."""
    mod = seeded_knn_fusion(3 + 6, (24, 20), (32, 16), 5)
    q, d, f, idx = knn_case(3, B=2, M=9, N=13, C=6, K=5)
    grouped = oracle_knn_fusion.group(q, d, f, idx)
    before, after = (layers_np(t) for t in network.fold_knn_fusion(mod))
    ref = oracle_knn_fusion.knn_fusion(grouped, before, after)
    exact = oracle_knn_fusion.knn_fusion(grouped, before, after, tf32=False)
    fin = np.isfinite(ref["out"])
    assert fin.all() and (ref["bound"] > 0).all()
    assert np.abs(ref["out"] - exact["out"]).max() > 10 * np.finfo(np.float32).eps
    assert (ref["bound"] < 0.1 * np.abs(exact["out"]).max()).all()           # four layers of |W| e growth
    # float32 evaluation of the concatenated formulation with the kernel's rounded operands
    r = oracle_knn_fusion.tf32_round
    x = r(grouped)
    for i, (W, b, _) in enumerate(before):
        x = r(np.maximum(np.einsum("oc,bcmk->bomk", r(W), x, dtype=np.float32) + b[None, :, None, None], 0))
    x = np.concatenate((np.broadcast_to(x.max(axis=3, keepdims=True), x.shape), x), axis=1)
    for i, (W, b, _) in enumerate(after):
        x = np.maximum(np.einsum("oc,bcmk->bomk", r(W), x, dtype=np.float32) + b[None, :, None, None], 0)
        if i < len(after) - 1:
            x = r(x)
    f32 = x.max(axis=3).astype(np.float64)
    assert (np.abs(f32 - ref["out"]) <= ref["bound"]).all()


def test_pointwise_mlp_max_oracle_equals_the_module_and_bounds_float32():
    pn = seeded_pointnet(3 + 10, [24, 40], 6)
    rng = np.random.default_rng(7)
    s1, s2 = (rng.normal(0, 1, (3, c, 29)).astype(np.float32).astype(np.float64) for c in (3, 10))
    s2[2, 4, 17] = np.nan
    with torch.no_grad():
        want = torch.max(pn(torch.from_numpy(np.concatenate((s1, s2), axis=1))), dim=2, keepdim=True)[0].numpy()
    folded64 = layers_np(network.fold_pointnet(pn, dtype=torch.float64))
    got = oracle_knn_fusion.pointwise_mlp_max([s1, s2], folded64, tf32=False)
    assert got["out"].shape == (3, 40, 1)
    assert np.array_equal(np.isnan(got["out"]), np.isnan(want))
    assert np.isnan(want[2]).all() and not np.isnan(want[:2]).any()
    assert np.nanmax(np.abs(got["out"] - want)) <= 1e-12 * np.nanmax(np.abs(want))
    layers = layers_np(network.fold_pointnet(pn))
    s1, s2 = s1.astype(np.float32), s2.astype(np.float32)
    ref = oracle_knn_fusion.pointwise_mlp_max([s1, s2], layers)
    r = oracle_knn_fusion.tf32_round
    x = r(np.concatenate((s1, s2), axis=1))
    (W1, b1, _), (W2, b2, _) = layers
    x = r(np.maximum(np.einsum("oc,bcn->bon", r(W1), x, dtype=np.float32) + b1[None, :, None], 0))
    x = np.maximum(np.einsum("oc,bcn->bon", r(W2), x, dtype=np.float32) + b2[None, :, None], 0)
    f32 = x.max(axis=2, keepdims=True).astype(np.float64)
    fin = np.isfinite(ref["out"])
    assert np.array_equal(fin, ~np.isnan(want))
    assert (np.abs(f32 - ref["out"])[fin] <= ref["bound"][fin]).all()


def test_argument_validation_without_gpu():
    q, d, f = torch.zeros(2, 3, 7), torch.zeros(2, 3, 11), torch.zeros(2, 5, 11)
    lay = lambda c_in, widths: [(torch.zeros(c, ci), torch.zeros(c), True) for ci, c in zip([c_in] + widths, widths)]
    ok = (lay(8, [12]), lay(24, [6]))
    bad = [
        ((q, d, f, 4, (lay(8, [12]), lay(20, [6]))), {}),         # the first after layer must take 2 C_b rows
        ((q, d, f, 4, (lay(8, [12] * 4), lay(24, [6]))), {}),     # more than three before layers
        ((q, d, f, 4, ([], lay(24, [6]))), {}),                   # no before layer
        ((q, d, f, 4, (lay(8, [513]), lay(1026, [6]))), {}),      # a layer wider than 512
        ((q, d, f, 0, ok), {}), ((q, d, f, 33, ok), {}), ((q, d, f, 12, ok), {}),   # K outside [1, min(32, N)]
        ((q, torch.zeros(2, 3, 2049), torch.zeros(2, 5, 2049), 4, ok), {}),        # N > 2048
        ((q, d, torch.zeros(2, 5, 10), 4, ok), {}),               # features do not match the database
        ((torch.zeros(2, 3, 0), d, f, 4, ok), {}),                # no queries
        ((q, d, torch.zeros(2, 510, 11), 4, (lay(513, [12]), lay(24, [6]))), {}),   # 3 + C > 512
        ((q, d, f, 4, ok[0]), {}),
    ]
    for args, kw in bad:
        with pytest.raises(ValueError):
            point_ops.knn_fusion(*args, **kw)
    with pytest.raises(RuntimeError):                         # well-formed but not on a GPU: no CPU fallback
        point_ops.knn_fusion(q, d, f, 4, ok)
    with pytest.raises(RuntimeError):                         # no backward
        point_ops.knn_fusion(q, d, f.clone().requires_grad_(True), 4, ok)
    s = [torch.zeros(2, 3, 9), torch.zeros(2, 5, 9)]
    for sources, layers in (([], lay(8, [4])), (s, lay(7, [4])), (s, lay(8, [4] * 4)), (s, lay(8, [513])),
                            ([torch.zeros(2, 513, 9)], lay(513, [4])), ([torch.zeros(2, 3, 0)], lay(3, [4])),
                            ([(s[0], s[0], s[0])], lay(3, [4]))):
        with pytest.raises(ValueError):
            point_ops.pointwise_mlp_max(sources, layers)
    with pytest.raises(RuntimeError):
        point_ops.pointwise_mlp_max(s, lay(8, [4]))
    with pytest.raises(RuntimeError):
        point_ops.pointwise_mlp_max([s[0], s[1].clone().requires_grad_(True)], lay(8, [4]))
    with pytest.raises(ValueError):
        network.FusedInference(network.KeypointDetector(img_H=64, img_W=128), encoder="cudnn")


def test_native_validation_without_gpu():
    from deepi2p_b200 import _native
    lib = _native.load()
    lay = np.zeros((4, 4), dtype=np.int64)
    lay[:, 2], lay[:, 3] = (12, 9, 14, 6), 1
    # before 8 -> 12 -> 9, after 18 -> 14 -> 6: the fragments of 16 x 8, 16 x 16, 16 x 16 (the x half), 16 x 16 weights,
    # four 16-float biases and the transposed max half 9 x 16
    want = (16 * 8 + 16 * 16 + 16 * 16 + 16 * 16 + 4 * 16 + 9 * 16) * 4
    assert lib.knn_fusion_packed_bytes(8, lay.ctypes.data, 2, 2) == want
    assert lib.knn_fusion_packed_bytes(8, lay.ctypes.data, 2, 0) == 0
    assert b"each side" in lib.dib_last_error()
    assert lib.knn_fusion_packed_bytes(513, lay.ctypes.data, 2, 2) == 0
    lay[1, 2] = 513
    assert lib.knn_fusion_packed_bytes(8, lay.ctypes.data, 2, 2) == 0
    assert b"C_out <= 512" in lib.dib_last_error()
    lay[1, 2] = 9
    # K > N and N > 2048 are rejected before any pointer is read
    assert lib.knn_fusion_f32(None, None, None, 1, 5, 4, 3, 4, lay.ctypes.data, 2, 2, None, 0, None, None, None) == -22
    assert b"K <= min(32, N)" in lib.dib_last_error()
    assert lib.knn_fusion_f32(None, None, None, 1, 5, 4, 2049, 4, lay.ctypes.data, 2, 2, None, 0, None, None,
                              None) == -22
    assert lib.knn_fusion_f32(None, None, None, 1, 5, 4, 16, 4, lay.ctypes.data, 2, 2, None, 0, None, None,
                              None) == -22                    # NULL pointers
    assert b"NULL" in lib.dib_last_error()
    assert lib.pointwise_mlp_max_packed_bytes(8, lay.ctypes.data, 2) == (16 * 8 + 16 * 16 + 2 * 16) * 4
    assert lib.pointwise_mlp_max_workspace_bytes(512, 64, 128) == 64 * 512 * 4 * 4
    src = np.zeros((1, 8), dtype=np.int64)
    src[0, 2], src[0, 3] = 8, 16                              # an interpolated source is not supported
    assert lib.pointwise_mlp_max_f32(src.ctypes.data, 1, lay.ctypes.data, 2, None, 0, 1, 5, None, None, 0, None) == -22
    assert b"dense" in lib.dib_last_error()
