"""The host side of the fused per-point layers (DESIGN.md 4.21): BatchNorm folding against the module itself, the
oracle's formulation against the unfused layers in float64, the TF32 rounding rule at its edges, and the argument
checks of point_ops.pointwise_mlp, none of which needs a GPU."""
import numpy as np
import pytest
import torch

import oracle_pointwise
from deepi2p_b200 import network, point_ops


def seeded_pointnet(c_in, widths, norm_act_at_last, seed):
    """A float64 _PointNet in eval mode whose BatchNorm layers have non-trivial statistics and affine parameters."""
    torch.manual_seed(seed)
    pn = network._PointNet(c_in, widths, norm_act_at_last, dropouts=[0.5] * len(widths)).double()
    with torch.no_grad():
        for layer in pn.layers:
            layer.conv.bias.normal_(0, 0.3)
            if layer.norm is not None:
                layer.norm.running_mean.normal_(0, 0.5)
                layer.norm.running_var.uniform_(0.3, 2.0)
                layer.norm.weight.uniform_(0.5, 1.5)
                layer.norm.bias.normal_(0, 0.2)
    return pn.eval()


def chain(folded, x):
    for W, b, act in folded:
        x = torch.einsum("oc,bcn->bon", W, x) + b[None, :, None]
        if act:
            x = torch.relu(x)
    return x


@pytest.mark.parametrize("norm_act_at_last", [True, False])
def test_fold_pointnet_equals_the_module(norm_act_at_last):
    pn = seeded_pointnet(11, [24, 17, 9], norm_act_at_last, 3)
    x = torch.randn(2, 11, 50, dtype=torch.float64)
    with torch.no_grad():
        want = pn(x)
    folded = network.fold_pointnet(pn, dtype=torch.float64)
    assert [a for _, _, a in folded] == [True, True, norm_act_at_last]
    got = chain(folded, x)
    assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max())
    f32 = network.fold_pointnet(pn)
    assert all(W.dtype == torch.float32 and b.dtype == torch.float32 for W, b, _ in f32)
    assert all(torch.equal(W32, W.float()) for (W32, _, _), (W, _, _) in zip(f32, folded))


def small_head_case(seed=5):
    rng = np.random.default_rng(seed)
    B, N, Ma, Mb, k = 2, 37, 6, 5, 3
    Fa, Fb = rng.normal(0, 1, (B, 4, Ma)), rng.normal(0, 1, (B, 7, Mb))
    d1, d2 = rng.normal(0, 1, (B, 3, N)), rng.normal(0, 1, (B, 2, N))
    wa, wb = rng.uniform(0, 1, (B, N, k)).astype(np.float32), rng.uniform(0, 1, (B, N, k)).astype(np.float32)
    ia, ib = rng.integers(0, Ma, (B, N, k)).astype(np.int32), rng.integers(0, Mb, (B, N, k)).astype(np.int32)
    ia[0, 4], wa[0, 4] = -1, np.nan                          # what interp_weights writes for a bad point
    ib[1, 9], wb[1, 9] = -1, np.nan
    return (Fa, wa, ia), (Fb, wb, ib), d1, d2


def torch_interp(F, w, idx):
    F, w, idx = torch.from_numpy(F), torch.from_numpy(w).double(), torch.from_numpy(idx).long()
    B, C, _ = F.shape
    out = torch.zeros(B, C, idx.shape[1], dtype=torch.float64)
    for j in range(idx.shape[2]):
        out += w[:, None, :, j] * torch.gather(F, 2, idx[:, None, :, j].clamp(min=0).expand(B, C, -1))
    out[(idx < 0).any(dim=2)[:, None, :].expand_as(out)] = float("nan")
    return out


def test_oracle_without_rounding_equals_the_unfused_layers():
    a, b, d1, d2 = small_head_case()
    pn = seeded_pointnet(4 + 7 + 3 + 2, [12, 10, 2 + 6], False, 8)
    x = torch.cat((torch_interp(*a), torch_interp(*b), torch.from_numpy(d1), torch.from_numpy(d2)), dim=1)
    with torch.no_grad():
        want = pn(x)
    layers = [(W.numpy(), bb.numpy(), act) for W, bb, act in network.fold_pointnet(pn, dtype=torch.float64)]
    got = oracle_pointwise.pointwise_mlp([a, b, d1, d2], layers, c_split=2, tf32=False)
    nan = torch.isnan(want).numpy()
    assert nan[0, :, 4].all() and nan[1, :, 9].all() and nan.sum() == 2 * want.shape[1]
    assert np.array_equal(np.isnan(got["out"]), nan)
    assert np.nanmax(np.abs(got["out"] - want.numpy())) <= 1e-12 * float(want[~torch.isnan(want)].abs().max())
    assert not got["bound"].any()
    c, f = network.predict(want[:, :2], want[:, 2:])
    assert np.array_equal(got["pred_a"], c.numpy()) and np.array_equal(got["pred_b"], f.numpy())
    assert got["pred_a"][0, 4] == 0 and got["pred_b"][1, 9] == 0          # NaN is maximal: the first index


def test_oracle_bound_covers_float32_evaluation():
    """The bound is an upper bound on what any float32 evaluation of the same rounded operands can be off by."""
    a, b, d1, d2 = small_head_case(6)
    f32 = [np.float32(t) for t in (d1, d2)]
    a, b = (np.float32(a[0]), a[1], a[2]), (np.float32(b[0]), b[1], b[2])
    pn = seeded_pointnet(16, [12, 10, 8], False, 9)
    layers = [(W.numpy(), bb.numpy(), act) for W, bb, act in network.fold_pointnet(pn)]
    ref = oracle_pointwise.pointwise_mlp([a, b, *f32], layers, c_split=2)
    exact = oracle_pointwise.pointwise_mlp([a, b, *f32], layers, tf32=False)
    fin = np.isfinite(ref["out"])
    assert fin.sum() > 0 and (ref["bound"][fin] > 0).all()
    # TF32 rounding moves the scores by far more than float32 accumulation could: the bound must not hide that
    assert np.abs(ref["out"] - exact["out"])[fin].max() > 10 * np.finfo(np.float32).eps
    assert (ref["bound"][fin] < 0.05 * np.abs(exact["out"][fin]).max()).all()


def test_tf32_rounding_rule():
    r = oracle_pointwise.tf32_round
    one = np.float32(1.0)
    ulp = np.float32(2.0 ** -10)                             # a TF32 ulp at 1.0
    assert r(one + ulp / 2) == one + ulp                     # a tie goes away from zero
    assert r(-(one + ulp / 2)) == -(one + ulp)
    assert r(one + ulp * np.float32(1.5)) == one + 2 * ulp   # ... also when the kept mantissa is odd
    assert r(np.float32(1.0 + 2.0 ** -11 - 2.0 ** -23)) == one   # just below a tie goes down
    assert r(np.float32(2.0 - 2.0 ** -12)) == np.float32(2.0)    # rounds up into the next binade
    sub = np.float32(2.0 ** -136)                            # subnormals keep multiples of 2^-136
    assert r(sub) == sub and r(np.float32(2.0 ** -137)) == sub and r(np.float32(2.0 ** -149)) == 0.0
    assert r(np.float32(2.0 ** -149 * 0x0fff)) == 0.0
    assert np.isposinf(r(np.float32(np.inf))) and np.isneginf(r(np.float32(-np.inf)))
    assert np.isposinf(r(np.finfo(np.float32).max))              # overflow is defined: infinity
    nan = np.array([np.nan, -np.nan], dtype=np.float32)
    assert np.array_equal(r(nan).view(np.uint32), nan.view(np.uint32))
    x = np.random.default_rng(0).normal(0, 100, 10000).astype(np.float32)
    assert (r(x).view(np.uint32) & 0x1fff == 0).all() and np.abs(r(x) - x).max() <= np.abs(x).max() * 2.0 ** -11
    assert np.array_equal(r(r(x)), r(x))


def test_argmax_rule_is_torch_max():
    s = np.array([[[1.0, 3.0, np.nan, 2.0], [3.0, 3.0, 0.0, np.nan], [2.0, 5.0, np.nan, np.nan]]]).transpose(0, 1, 2)
    want = torch.max(torch.from_numpy(s), dim=1)[1].numpy()
    assert np.array_equal(oracle_pointwise.argmax_rule(s), want)


def test_argument_validation_without_gpu():
    x = torch.zeros(2, 3, 10)
    W = torch.zeros(4, 3)
    ok = [(W, None, True)]
    bad = [
        (([x] * 5, [(torch.zeros(4, 15), None, True)]), {}),                       # more than four sources
        (([x, torch.zeros(2, 3, 11)], [(torch.zeros(4, 6), None, True)]), {}),     # mismatched N
        (([x], [(torch.zeros(257, 3), None, True)]), {}),                          # a layer wider than 256
        (([x], [(torch.zeros(4, 5), None, True)]), {}),                            # W does not match the input rows
        (([x], ok * 4), {}),                                                       # more than three layers
        (([torch.zeros(2, 1025, 10)], [(torch.zeros(4, 1025), None, True)]), {}),  # more than 1024 input rows
        (([(torch.zeros(2, 3, 6), torch.zeros(2, 10, 9), torch.zeros(2, 10, 9, dtype=torch.int32))], ok), {}),  # k > 8
        (([(torch.zeros(2, 3, 2049), torch.zeros(2, 10, 3), torch.zeros(2, 10, 3, dtype=torch.int32))], ok), {}),
        (([x], [(W, torch.zeros(5), True)]), {}),                                  # bias of the wrong length
        (([x], ok), dict(output="argmax")),                                        # c_split missing
        (([x], ok), dict(output="argmax", c_split=5)),                             # c_split > C_out
        (([x], ok), dict(output="scores")),
        (([x], ok), dict(return_scores=True)),
        (([torch.zeros(2, 3, 0)], ok), {}),                                        # no points
    ]
    for (sources, layers), kw in bad:
        with pytest.raises(ValueError):
            point_ops.pointwise_mlp(sources, layers, **kw)
    with pytest.raises(RuntimeError):                         # well-formed but not on a GPU: no CPU fallback
        point_ops.pointwise_mlp([x], ok)
    with pytest.raises(RuntimeError):                         # no backward
        point_ops.pointwise_mlp([x.clone().requires_grad_(True)], ok)


def test_native_validation_without_gpu():
    from deepi2p_b200 import _native
    lib = _native.load()
    src = np.zeros((1, 8), dtype=np.int64)
    lay = np.zeros((1, 4), dtype=np.int64)
    src[0, 2], lay[0, 2] = 3, 300
    assert lib.pointwise_mlp_packed_bytes(src.ctypes.data, 1, lay.ctypes.data, 1) == 0
    assert b"C_out" in lib.dib_last_error()
    lay[0, 2] = 10
    # one layer 3 -> 10: 16 padded rows x 8 padded columns of weights and 16 biases
    assert lib.pointwise_mlp_packed_bytes(src.ctypes.data, 1, lay.ctypes.data, 1) == (16 * 8 + 16) * 4
    assert lib.pointwise_mlp_workspace_bytes(src.ctypes.data, 1, lay.ctypes.data, 1, 4) == 0
    src[0, 3], src[0, 6] = 128, 3
    assert lib.pointwise_mlp_workspace_bytes(src.ctypes.data, 1, lay.ctypes.data, 1, 4) == 4 * 128 * 16 * 4
    assert lib.pointwise_mlp_f32(src.ctypes.data, 5, lay.ctypes.data, 1, None, 0, 1, 1, 0, None, None, None, None, 0,
                                 None) == -22
    src[0, 6] = 9
    assert lib.pointwise_mlp_f32(src.ctypes.data, 1, lay.ctypes.data, 1, None, 0, 1, 1, 0, None, None, None, None, 0,
                                 None) == -22
    assert b"k <= 8" in lib.dib_last_error()
