"""point_ops.point_branch's host side and KeypointDetector(point_layers="fused_all") (DESIGN.md 4.36): argument errors
and their messages, the new header constants against the host tables, the state_dict across the three modes, the
script option, and numpy restatements of the group max's index rule and the group sum's order."""
import re

import numpy as np
import pytest
import torch

from deepi2p_b200 import _native, network, point_ops


def _layers(c_in, widths, last=True):
    return list(network._PointNet(c_in, widths, last, 0.1).layers)


def test_header_constants_match_the_host_tables():
    with open(_native._build.HEADER) as f:
        text = f.read()
    const = dict((m.group(1), int(m.group(2))) for m in re.finditer(r"#define (DIB_PC_\w+) (\d+)", text))
    assert const["DIB_PC_MODE_MAX_GRAD"] == point_ops._OP_MAX_GRAD
    assert const["DIB_PC_MAX_WIDTH"] == point_ops.BRANCH_MAX_WIDTH == point_ops.CHAIN_MAX_IN
    sigs = _native.parse_header(text)
    for name in ("point_chain_gemm_group_f32", "point_chain_group_max_f32", "point_chain_group_sum_f32"):
        assert name in sigs
    # the max-gradient operand: one source row (compact gradient), then the transform row with the indices in Y and
    # the group in LAYER
    g, idx = torch.zeros((2, 5, 3)), torch.zeros((2, 5, 3), dtype=torch.int32)
    t = point_ops._chain_max_grad_operand(g, idx, 4)
    assert t.shape == (point_ops._PC_SRC + point_ops._PC_OP,)
    assert list(t[:3]) == [g.data_ptr(), 15, 5]
    op = t[3:]
    assert op[const["DIB_PC_OP_MODE"]] == 3 and op[const["DIB_PC_OP_Y"]] == idx.data_ptr()
    assert op[const["DIB_PC_OP_LAYER"]] == 4


def _args(**kw):
    a = dict(sources=[torch.zeros((2, 7, 16))], layers=_layers(7, [32, 32]), drop_state=None, cols=[0], add=None,
             add_group=1, max_group=None, output="activations")
    a.update(kw)
    return a


@pytest.mark.parametrize("bad, exc, msg", [
    (dict(layers=[]), ValueError, "layers"),
    (dict(layers=_layers(7, [1025])), ValueError, r"layers\[0\]: need 1 <= C_out <= 1024"),
    (dict(sources=[]), ValueError, "sources"),
    (dict(sources=[torch.zeros((2, 7, 16), dtype=torch.float64)]), TypeError, r"sources\[0\]"),
    (dict(sources=[torch.zeros((2, 3, 16)), torch.zeros((3, 4, 16))], cols=[0, 3]), ValueError, r"sources\[1\]"),
    (dict(cols=[-1]), ValueError, "cols"),
    (dict(cols=[0, 1]), ValueError, "cols"),
    (dict(cols=[1]), ValueError, "cols"),
    (dict(sources=[torch.zeros((2, 3, 16)), torch.zeros((2, 4, 16))], cols=[0, 2]), ValueError, "overlap"),
    (dict(sources=[torch.zeros((2, 3, 16))], cols=[0]), ValueError, "sources"),
    (dict(max_group=5, output="max"), ValueError, "max_group"),
    (dict(max_group=4), ValueError, "max_group"),
    (dict(output="max"), ValueError, "max_group"),
    (dict(output="min"), ValueError, "output"),
    (dict(sources=[torch.zeros((2, 3, 16))], add=torch.zeros((2, 32, 16)), add_group=4), ValueError, "add must be"),
    (dict(sources=[torch.zeros((2, 3, 16))], add=torch.zeros((2, 32, 4)), add_group=3), ValueError, "add_group"),
    (dict(sources=[torch.zeros((2, 3, 16))], add=[0.0], add_group=1), TypeError, "add"),
    (dict(layers=_layers(7, [32], last=False), max_group=4, output="max"), ValueError, "max_group"),
])
def test_argument_errors_name_the_argument(bad, exc, msg):
    a = _args(**bad)
    with pytest.raises(exc, match=msg):
        point_ops._check_branch_args(a["sources"], a["layers"], a["drop_state"], a["cols"], a["add"], a["add_group"],
                                     a["max_group"], a["output"])


def test_conv2d_layers_are_taken_and_checked_last_for_device():
    knn = network._KnnFusion(7, (8,), (8,))
    a = _args(sources=[torch.zeros((2, 7, 64))], layers=list(knn.layers_before), max_group=16, output="both")
    # the layers' own tensors are checked last for device and dtype (CPU tensors here): the shapes passed
    with pytest.raises(TypeError, match="float32 CUDA"):
        point_ops._check_branch_args(a["sources"], a["layers"], None, a["cols"], None, 1, 16, "both")
    k3 = torch.nn.Conv2d(7, 8, 3)
    bad = network._PointLayer(7, 8, True, dims=2)
    bad.conv = k3
    with pytest.raises(TypeError, match="1x1 Conv1d or Conv2d"):
        point_ops._check_branch_args(a["sources"], [bad], None, a["cols"], None, 1, None, "activations")


def test_state_dict_is_the_same_in_every_mode():
    sds = [network.KeypointDetector(**network.SHAPES["kitti"], point_layers=m).state_dict()
           for m in network.POINT_LAYERS]
    assert network.POINT_LAYERS == ("torch", "fused", "fused_all")
    for sd in sds[1:]:
        assert list(sd) == list(sds[0])
        assert all(sd[k].shape == sds[0][k].shape and sd[k].dtype == sds[0][k].dtype for k in sd)


def test_script_takes_fused_all():
    import importlib.util
    import os
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts", "train_classifier.py")
    spec = importlib.util.spec_from_file_location("train_classifier_script_fa", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    base = ["--dataset", "kitti", "--root", "r", "--out", "o"]
    assert mod.parse_args(base + ["--point-layers", "fused_all"]).point_layers == "fused_all"


def test_eval_mode_under_grad_raises():
    m = network.KeypointDetector(**network.SHAPES["kitti"], point_layers="fused_all").eval()
    with pytest.raises(RuntimeError, match="no backward"):
        m(*[None] * 6)


def _group_max_rule(v):
    """torch.max(dim=-1)'s rule over the last axis, sequentially: the first maximal value; a NaN, the first one, over
    any number.  What chain_group_max_kernel does per group."""
    best, idx = v[..., 0].copy(), np.zeros(v.shape[:-1], dtype=np.int64)
    for k in range(1, v.shape[-1]):
        take = (v[..., k] > best) | (np.isnan(v[..., k]) & ~np.isnan(best))
        best, idx = np.where(take, v[..., k], best), np.where(take, k, idx)
    return best, idx


def test_group_max_rule_matches_torch_max_on_the_cpu():
    rng = np.random.default_rng(0)
    v = rng.integers(-2, 3, size=(4, 6, 16)).astype(np.float32)              # many ties
    v[0, 0] = 1.0                                                              # all equal
    v[1, 1, 5] = np.nan
    v[2, 2, [3, 9]] = np.nan
    best, idx = _group_max_rule(v)
    tv, ti = torch.max(torch.from_numpy(v), dim=-1)
    assert np.array_equal(best, tv.numpy(), equal_nan=True)
    ok = ~np.isnan(best)
    assert np.array_equal(idx[ok], ti.numpy()[ok])
    assert idx[0, 0] == 0 and idx[1, 1] == 5 and idx[2, 2] == 3


def test_group_sum_order_is_sequential_fp64():
    # the add gradient sums each group's G columns in column order in fp64, rounded once: for these values a pairwise
    # or float32 order gives other bits, so the restatement pins the order
    x = np.array([1.0, 2.0 ** -30, -1.0, 2.0 ** -30] * 4, dtype=np.float32).reshape(1, 1, 16)
    seq = np.cumsum(x.astype(np.float64), axis=-1)[..., -1].astype(np.float32)
    f32 = np.float32(0)
    for t in x.ravel():
        f32 = np.float32(f32 + t)
    assert seq[0, 0] == np.float32(8 * 2.0 ** -30) and f32 != seq[0, 0]
