"""Decoder interpolation (DESIGN.md 4.12) without a GPU: the numpy oracle against a torch restatement of the
reference's formulation (models/networks_united.py:76-103), the reference's quirks, and the host-side argument checks
of point_ops.upsample_by_interpolation and of the C ABI."""
import ctypes

import numpy as np
import pytest
import torch

import oracle_interp
from deepi2p_b200 import point_ops


def formulation(idx, query, node, features):
    """The reference's arithmetic in torch: gather the k nodes, their norm, 1 - d / sum d, gather the k feature
    columns, weight and sum over k.  Works in the dtype of its inputs."""
    B, Nq, k = idx.shape
    C, M = features.shape[1], features.shape[2]
    idx = idx.long()
    nk = torch.gather(node.unsqueeze(3).expand(B, 3, M, k), 2, idx.unsqueeze(1).expand(B, 3, Nq, k))
    d = torch.norm(query.unsqueeze(3) - nk, p=2, dim=1)                                   # [B, Nq, k]
    w = 1 - d / torch.sum(d, dim=2, keepdim=True)
    fk = torch.gather(features.unsqueeze(3).expand(B, C, M, k), 2, idx.unsqueeze(1).expand(B, C, Nq, k))
    return torch.sum(w.unsqueeze(1) * fk, dim=3)


def make_case(seed, B, Nq, M, C, k):
    rng = np.random.default_rng(seed)
    query = rng.uniform(-10, 10, (B, 3, Nq)).astype(np.float32)
    node = rng.uniform(-10, 10, (B, 3, M)).astype(np.float32)
    d = np.linalg.norm(query[:, :, :, None] - node[:, :, None, :], axis=1)                  # [B, Nq, M]
    idx = np.argsort(d, axis=2, kind="stable")[:, :, :k].astype(np.int64)
    F = rng.normal(0, 1, (B, C, M)).astype(np.float32)
    return idx, query, node, F


@pytest.mark.parametrize("B,Nq,M,C,k", [(2, 50, 16, 5, 3), (1, 33, 7, 1, 1), (3, 17, 40, 9, 8)])
def test_oracle_forward_matches_formulation(B, Nq, M, C, k):
    idx, q, nd, F = make_case(B * 100 + k, B, Nq, M, C, k)
    got = oracle_interp.interp_forward(idx, q, nd, F)
    ref = formulation(*[torch.from_numpy(a) for a in (idx, q, nd, F)]).numpy()
    # the formulations differ in the norm's rounding (torch's reduction order) and nothing else: a few float32 ulps
    # of the weights, times |F|
    np.testing.assert_allclose(got, ref, rtol=1e-5, atol=1e-5 * k)


@pytest.mark.parametrize("B,Nq,M,C,k", [(2, 50, 16, 5, 3), (1, 64, 8, 3, 8)])
def test_oracle_backward_matches_fp64_autograd(B, Nq, M, C, k):
    idx, q, nd, F = make_case(7 + k, B, Nq, M, C, k)
    g = np.random.default_rng(1).normal(0, 1, (B, C, Nq)).astype(np.float32)
    Ft = torch.from_numpy(F).double().requires_grad_(True)
    out = formulation(torch.from_numpy(idx), torch.from_numpy(q).double(), torch.from_numpy(nd).double(), Ft)
    out.backward(torch.from_numpy(g).double())
    got = oracle_interp.interp_backward(idx, q, nd, g, M)
    # the oracle weights are float32 (rel. error ~1e-7 each), the autograd restatement's are float64
    np.testing.assert_allclose(got, Ft.grad.numpy(), rtol=1e-5, atol=1e-5)


def test_adjoint_identity():
    idx, q, nd, F = make_case(3, 2, 80, 12, 6, 3)
    g = np.random.default_rng(2).normal(0, 1, (2, 6, 80)).astype(np.float32)
    lhs = np.sum(oracle_interp.interp_forward(idx, q, nd, F).astype(np.float64) * g)
    rhs = np.sum(F.astype(np.float64) * oracle_interp.interp_backward(idx, q, nd, g, 12).astype(np.float64))
    assert abs(lhs - rhs) <= 1e-5 * np.sum(np.abs(F)) * 3


def test_weights_sum_to_k_minus_1():
    for k in (2, 3, 8):
        idx, q, nd, _ = make_case(k, 1, 40, 10, 1, k)
        w, valid = oracle_interp.interp_weights(idx, q, nd)
        assert valid.all()
        np.testing.assert_allclose(w.astype(np.float64).sum(axis=2), k - 1, atol=4 * k * 2.0 ** -23)


def test_quirks_zero_sum_single_neighbour_and_point_on_node():
    nd = np.array([[[0, 1, 2, 3], [0, 0, 0, 0], [0, 0, 0, 0]]], np.float32)                 # 4 nodes on the x axis
    F = np.arange(2 * 4, dtype=np.float32).reshape(1, 2, 4) + 1
    # query 0 sits on node 0 and all its indices are 0: S = 0 -> NaN
    # query 1 sits on node 1 with neighbours (1, 0, 2): w = (1, 1 - 1/2, 1 - 1/2)
    q = np.array([[[0, 1], [0, 0], [0, 0]]], np.float32)
    idx = np.array([[[0, 0, 0], [1, 0, 2]]])
    out = oracle_interp.interp_forward(idx, q, nd, F)
    assert np.isnan(out[0, :, 0]).all()
    np.testing.assert_array_equal(out[0, :, 1], F[0, :, 1] + 0.5 * F[0, :, 0] + 0.5 * F[0, :, 2])
    ref = formulation(*[torch.from_numpy(a) for a in (idx, q, nd, F)]).numpy()
    assert np.isnan(ref[0, :, 0]).all() and np.array_equal(ref[0, :, 1], out[0, :, 1])
    # k = 1: the weight is 1 - d / d = 0 (NaN on a node, where d = 0)
    q1 = np.array([[[0.5, 3.0], [0, 0], [0, 0]]], np.float32)
    out1 = oracle_interp.interp_forward(np.array([[[0], [3]]]), q1, nd, F)
    np.testing.assert_array_equal(out1[0, :, 0], 0)
    assert np.isnan(out1[0, :, 1]).all()


def test_out_of_range_index_gives_nan_column_and_no_gradient():
    idx, q, nd, F = make_case(5, 1, 20, 6, 3, 3)
    bad = idx.copy()
    bad[0, 4, 1] = 6
    bad[0, 9, 2] = -1
    out = oracle_interp.interp_forward(bad, q, nd, F)
    assert np.isnan(out[0, :, [4, 9]]).all() and np.isfinite(np.delete(out, [4, 9], axis=2)).all()
    g = np.random.default_rng(0).normal(0, 1, (1, 3, 20)).astype(np.float32)
    keep = [n for n in range(20) if n not in (4, 9)]
    np.testing.assert_array_equal(oracle_interp.interp_backward(bad, q, nd, g, 6),
                                  oracle_interp.interp_backward(idx[:, keep], q[:, :, keep], nd, g[:, :, keep], 6))


def _args(B=2, Nq=10, M=6, C=4, k=3, idx_dtype=torch.int64):
    return (torch.zeros(B, Nq, k, dtype=idx_dtype), torch.zeros(B, 3, Nq), torch.zeros(B, 3, M), torch.zeros(B, C, M))


@pytest.mark.parametrize("change,match", [
    (lambda a: (a[0].float(), *a[1:]), "topk_idx must have dtype"),
    (lambda a: (a[0].short(), *a[1:]), "topk_idx must have dtype"),
    (lambda a: (*a[:3], a[3].double()), "features must have dtype"),
    (lambda a: (a[0], a[1].half(), *a[2:]), "query must have dtype"),
    (lambda a: (a[0][0], *a[1:]), "topk_idx must have 3 dimensions"),
    (lambda a: (*a[:3], a[3][0]), "features must have 3 dimensions"),
    (lambda a: (a[0], a[1][:, :2], *a[2:]), r"query \[B,3,Nq\]"),
    (lambda a: (*a[:3], a[3][:, :, :5]), r"features \[B,C,M\]"),
    (lambda a: _args(k=9), "k <= 8"),
    (lambda a: _args(k=0), "1 <= k"),
    (lambda a: _args(M=2049), "M <= 2048"),
    (lambda a: (a[0], a[1].requires_grad_(True), *a[2:]), "detach"),
    (lambda a: (*a[:2], a[2].requires_grad_(True), a[3]), "detach"),
    (lambda a: a, "CUDA"),
])
def test_host_side_rejection(change, match):
    with pytest.raises(RuntimeError, match=match):
        point_ops.upsample_by_interpolation(*change(_args()))


def test_m_at_the_bound_passes_the_host_checks():
    with pytest.raises(RuntimeError, match="CUDA"):          # only the device check is left
        point_ops.upsample_by_interpolation(*_args(M=2048, k=8, idx_dtype=torch.int32))


def test_c_abi_validates_on_host():
    from deepi2p_b200 import _native
    lib = _native.load()
    buf = ctypes.create_string_buffer(256)
    a = ctypes.addressof(buf)
    assert lib.interp_weights_f32(a, 8, a, a, 1, 4, 6, 9, a, a, None) == -22                   # k > 8
    assert b"k" in lib.dib_last_error()
    assert lib.interp_weights_f32(a, 2, a, a, 1, 4, 6, 3, a, a, None) == -22                   # idx_bytes
    assert lib.interp_forward_f32(a, a, a, 1, 4, 4, 4096, 3, a, None) == -22                   # M > 2048
    assert lib.interp_backward_f32(a, 16, a, a, 1, 4, 4, 6, 3, a, a, 0, None) == -22           # no workspace
    assert b"workspace" in lib.dib_last_error()
    assert lib.interp_backward_f32(a, -1, a, a, 1, 4, 4, 6, 3, a, a, 256, None) == -22         # negative stride
    assert lib.interp_backward_workspace_bytes(0, 4, 4, 6) == 0
    # the fp64 slice partials: B x slices x C x M doubles, with at least one slice
    assert lib.interp_backward_workspace_bytes(8, 512, 20480, 128) % (8 * 512 * 128 * 8) == 0
    assert lib.interp_backward_workspace_bytes(1, 1, 1, 1) == 8
