"""point_ops.point_chain's host side (DESIGN.md 4.34): argument checks and their messages, the operand tables against
pointwise_mlp's source layout and the header, the running-statistics rule restated in numpy against nn.BatchNorm1d,
and the fused model's state_dict against the default one."""
import numpy as np
import pytest
import torch

from deepi2p_b200 import _native, network, point_ops, train


def _layers(c_in, widths, last, dropouts=None):
    return list(network._PointNet(c_in, widths, last, 0.1, dropouts).layers)


def test_header_constants_match_the_host_tables():
    with open(_native._build.HEADER) as f:
        text = f.read()
    const = dict((m.group(1), int(m.group(2))) for m in
                 __import__("re").finditer(r"#define (DIB_PC_\w+) (\d+)", text))
    assert const["DIB_PC_SRC"] == point_ops._PC_SRC and const["DIB_PC_OP"] == point_ops._PC_OP
    assert (const["DIB_PC_SRC_DATA"], const["DIB_PC_SRC_BSTRIDE"], const["DIB_PC_SRC_CHANNELS"]) == (0, 1, 2)
    assert [const[f"DIB_PC_OP_{k}"] for k in ("MODE", "STATS", "Y", "DROP_STATE", "DROP_PPM", "LAYER")] == \
        list(range(6))
    assert const["DIB_PC_ACT"] == 5
    sigs = _native.parse_header(text)
    for name in ("point_chain_gemm_f32", "point_chain_bn_f32", "point_chain_dw_f32", "point_chain_dropout_mask",
                 "point_chain_partial_bytes", "point_chain_dw_workspace_bytes"):
        assert name in sigs


def test_operand_table_layout():
    a = torch.zeros((2, 3, 10))
    b = torch.zeros((2, 5, 10))
    t = point_ops._chain_operand([a, b])
    assert t.dtype == np.int64 and t.shape == (2 * 3 + 6,)
    assert list(t[:3]) == [a.data_ptr(), 30, 3] and list(t[3:6]) == [b.data_ptr(), 50, 5]
    assert list(t[6:]) == [0, 0, 0, 0, 0, 0]
    st, state = torch.zeros((4, 5)), torch.zeros(2, dtype=torch.int64)
    t = point_ops._chain_operand([b], point_ops._OP_ACT, st, drop=(state, 0.5), layer=1)
    assert list(t[3:]) == [1, st.data_ptr(), 0, state.data_ptr(), 500000, 1]
    # a single sample passes channels x N as its batch stride, as pointwise_mlp does
    one = torch.zeros((1, 4, 7))
    assert point_ops._chain_operand([one])[1] == 28
    row = point_ops._chain_act_row(st, None, 2)
    assert list(row) == [st.data_ptr(), 0, 0, 0, 2]


def test_dense_pack_spec_is_pointwise_mlps():
    # point_chain packs layer 1 as pointwise_mlp packs a chain of dense sources: same source and layer tables
    src, lay = point_ops._mlp_tables([(32, 0, 0), (64, 0, 0)], [(256, False)])
    assert src[:, 2].tolist() == [32, 64] and src[:, 3].tolist() == [0, 0] and lay[0, 2] == 256


@pytest.mark.parametrize("bad, exc, msg", [
    (dict(layers=[]), ValueError, "layers"),
    (dict(sources=[]), ValueError, "sources"),
    (dict(sources="x"), ValueError, "sources"),
    (dict(sources=[torch.zeros((2, 7, 16), dtype=torch.float64)]), TypeError, r"sources\[0\]"),
    (dict(sources=[torch.zeros((2, 7))]), ValueError, r"sources\[0\]"),
    (dict(sources=[torch.zeros((2, 3, 16)), torch.zeros((3, 4, 16))]), ValueError, r"sources\[1\]"),
    (dict(sources=[torch.zeros((2, 6, 16))]), ValueError, "sources"),
    (dict(in_col=-1), TypeError, "in_col"),
    (dict(in_col=1), ValueError, "sources"),
])
def test_argument_errors_name_the_argument(bad, exc, msg):
    args = dict(sources=[torch.zeros((2, 7, 16))], layers=_layers(7, [32, 32], True), in_col=0, add=None)
    args.update(bad)
    with pytest.raises(exc, match=msg):
        point_ops._check_chain_args(args["sources"], args["layers"], None, args["add"], args["in_col"], True)


def test_layer_errors():
    layers = _layers(7, [32, 16], True)
    with pytest.raises(ValueError, match=r"layers\[1\]"):
        point_ops._check_chain_args([torch.zeros((2, 7, 16))], [layers[1], layers[0]], None, None, 0, True)
    nolast = _layers(7, [32, 16], False)
    with pytest.raises(ValueError, match=r"layers\[0\]: only the last"):
        point_ops._check_chain_args([torch.zeros((2, 7, 16))], [nolast[1].__class__(7, 16, False), nolast[1]],
                                    None, None, 0, True)
    wide = _layers(7, [300], True)
    with pytest.raises(ValueError, match="C_out"):
        point_ops._check_chain_args([torch.zeros((2, 7, 16))], wide, None, None, 0, True)
    conv2 = list(network._KnnFusion(7, (8,), (8,)).layers_before)
    with pytest.raises(TypeError, match="Conv1d"):
        point_ops._check_chain_args([torch.zeros((2, 7, 16))], conv2, None, None, 0, True)
    drop = _layers(736, [256, 256, 82], False, [0.5, 0.5, 0])
    srcs = [torch.zeros((2, 32, 16)), torch.zeros((2, 64, 16))]
    add = torch.zeros((2, 256, 16))
    with pytest.raises(TypeError, match="drop_state"):
        point_ops._check_chain_args(srcs, drop, None, add, 640, True)
    with pytest.raises(ValueError, match="drop_state"):
        point_ops._check_chain_args(srcs, drop, torch.zeros(3, dtype=torch.int64), add, 640, True)
    with pytest.raises(ValueError, match="exceed"):
        point_ops._check_chain_args(srcs, drop, torch.zeros(2, dtype=torch.int64), add, 700, True)
    with pytest.raises(ValueError, match="add must be"):
        point_ops._check_chain_args(srcs, drop, torch.zeros(2, dtype=torch.int64), add[:, :128], 640, True)
    # the layers' own tensors are checked for device and dtype last (CPU tensors here)
    with pytest.raises(TypeError, match="float32 CUDA"):
        point_ops._check_chain_args(srcs, drop, torch.zeros(2, dtype=torch.int64), add, 640, True)


def test_eval_mode_refuses_add():
    with pytest.raises(ValueError, match="add"):
        point_ops.point_chain([torch.zeros((2, 7, 16))], _layers(7, [32], True), False, add=torch.zeros((2, 32, 16)))


def _running_update(rm, rv, y, momentum):
    """The running statistics of nn.BatchNorm1d in train mode, restated: mean and unbiased variance over (B, N)."""
    y = y.astype(np.float64)
    M = y.shape[0] * y.shape[2]
    mean = y.mean(axis=(0, 2))
    var = ((y - mean[None, :, None]) ** 2).sum(axis=(0, 2)) / (M - 1)
    return (1 - momentum) * rm + momentum * mean, (1 - momentum) * rv + momentum * var


@pytest.mark.parametrize("momentum", [0.1, 0.5])
def test_running_statistics_rule_matches_batchnorm1d(momentum):
    rng = np.random.default_rng(0)
    bn = torch.nn.BatchNorm1d(6, momentum=momentum).train()
    rm, rv = np.zeros(6), np.ones(6)
    for k in range(3):
        y = (rng.standard_normal((4, 6, 50)) * (k + 1) + k).astype(np.float32)
        bn(torch.from_numpy(y))
        rm, rv = _running_update(rm, rv, y, momentum)
        assert np.allclose(bn.running_mean.numpy(), rm, rtol=1e-5, atol=1e-6)
        assert np.allclose(bn.running_var.numpy(), rv, rtol=1e-5, atol=1e-6)
    assert bn.num_batches_tracked.item() == 3


def test_fused_model_has_the_same_state_dict():
    a = network.KeypointDetector(**network.SHAPES["kitti"]).state_dict()
    b = network.KeypointDetector(**network.SHAPES["kitti"], point_layers="fused").state_dict()
    assert list(a) == list(b)
    assert all(a[k].shape == b[k].shape and a[k].dtype == b[k].dtype for k in a)
    with pytest.raises(ValueError, match="point_layers"):
        network.KeypointDetector(point_layers="triton")


def test_script_takes_point_layers():
    import importlib.util
    import os
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts", "train_classifier.py")
    spec = importlib.util.spec_from_file_location("train_classifier_script", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    base = ["--dataset", "kitti", "--root", "r", "--out", "o"]
    assert mod.parse_args(base).point_layers == "torch"
    assert mod.parse_args(base + ["--point-layers", "fused"]).point_layers == "fused"
    with pytest.raises(SystemExit):
        mod.parse_args(base + ["--point-layers", "x"])
    assert train.Trainer  # the trainer takes the model as built, so the option travels with it


def test_eval_mode_under_grad_raises_instead_of_cutting_the_graph():
    layers = _layers(7, [32], True)
    with pytest.raises(RuntimeError, match="no backward"):
        point_ops.point_chain([torch.zeros((2, 7, 16))], layers, False)
    for p in (q for layer in layers for q in layer.parameters()):
        p.requires_grad_(False)
    with pytest.raises(RuntimeError, match="no backward"):
        point_ops.point_chain([torch.zeros((2, 7, 16), requires_grad=True)], layers, False)


@pytest.mark.parametrize("W, x, exc, msg", [
    ([[1.0]], torch.zeros((1, 1, 4)), TypeError, "W must be a torch.Tensor"),
    (torch.zeros((2, 3)), torch.zeros((1, 3, 4), dtype=torch.float64), TypeError, "x must have dtype"),
    (torch.zeros((2, 3)), torch.zeros((1, 3, 4)), ValueError, "CUDA"),
])
def test_channel_product_argument_errors(W, x, exc, msg):
    with pytest.raises(exc, match=msg):
        point_ops.channel_product(W, x)
