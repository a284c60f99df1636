"""The attention-weighted image-feature fusion's oracle and host checks without a GPU (DESIGN.md 4.17): oracle_fusion
against fp64 torch restatements of models/networks_united.py:149-150 / 172-174 (forward and autograd backward), the
adjoint identity, the non-finite and signed-zero rules, and every argument check of point_ops.attention_fusion and of
the C entry points."""
import ctypes

import numpy as np
import pytest
import torch

import oracle_fusion
from deepi2p_b200 import point_ops

SHAPES = [(1, 1, 1, 1), (2, 33, 50, 129), (3, 7, 1, 5), (1, 1, 960, 1), (2, 64, 80, 32)]
U64 = 2.0 ** -53


def reference_lines(F, A):
    """The reference's two lines, any dtype: [B,C,P] x [B,P,M] -> [B,C,M]."""
    return torch.mean(F.unsqueeze(3) * A.unsqueeze(1), dim=2)


def case(seed, B, C, P, M):
    rng = np.random.default_rng(seed)
    F = rng.normal(0, 1, (B, C, P)).astype(np.float32)
    A = (rng.normal(0, 3, (B, P, M))).astype(np.float32)
    g = rng.normal(0, 1, (B, C, M)).astype(np.float32)
    return F, A, g


def close64(got, ref, scale, n):
    """Two fp64 sums of the same n terms in different orders: |got - ref| <= 2 (n + 1) 2^-53 sum |terms|."""
    return bool(np.all(np.abs(got - ref) <= 2 * (n + 1) * U64 * scale + 1e-300))


@pytest.mark.parametrize("shape", SHAPES)
def test_oracle_forward_matches_reference_lines_in_fp64(shape):
    B, C, P, M = shape
    F, A, _ = case(sum(shape), *shape)
    ref = reference_lines(torch.from_numpy(F).double(), torch.from_numpy(A).double()).numpy()
    got, scale = oracle_fusion.forward(F, A, f64=True, with_abs=True)
    assert got.shape == (B, C, M) and close64(got, ref, scale, P)
    out = oracle_fusion.forward(F, A)
    assert out.dtype == np.float32 and np.array_equal(out, got.astype(np.float32))


@pytest.mark.parametrize("shape", SHAPES)
def test_oracle_backward_matches_fp64_autograd(shape):
    B, C, P, M = shape
    F, A, g = case(1 + sum(shape), *shape)
    F64 = torch.from_numpy(F).double().requires_grad_(True)
    A64 = torch.from_numpy(A).double().requires_grad_(True)
    reference_lines(F64, A64).backward(torch.from_numpy(g).double())
    gF, sF = oracle_fusion.backward_features(A, g, f64=True, with_abs=True)
    gA, sA = oracle_fusion.backward_attention(F, g, f64=True, with_abs=True)
    assert gF.shape == (B, C, P) and gA.shape == (B, P, M)
    # autograd divides g by P before the products: one more rounding per term
    assert close64(gF, F64.grad.numpy(), sF, M + 1) and close64(gA, A64.grad.numpy(), sA, C + 1)
    assert np.array_equal(oracle_fusion.backward_features(A, g), gF.astype(np.float32))
    assert np.array_equal(oracle_fusion.backward_attention(F, g), gA.astype(np.float32))


@pytest.mark.parametrize("shape", SHAPES)
def test_oracle_adjoint_identity(shape):
    """<gO, op(F, A)> = <gF, F> = <gA, A>: all three are (1 / P) sum over (b, c, p, m) of gO F A."""
    F, A, g = case(2 + sum(shape), *shape)
    out = oracle_fusion.forward(F, A, f64=True)
    gF = oracle_fusion.backward_features(A, g, f64=True)
    gA = oracle_fusion.backward_attention(F, g, f64=True)
    lhs = (g.astype(np.float64) * out).sum()
    P = shape[2]
    scale = np.abs(F.astype(np.float64))[:, :, :, None] * np.abs(A.astype(np.float64))[:, None, :, :]
    scale = (scale * np.abs(g.astype(np.float64))[:, :, None, :]).sum() / P
    tol = 1e-12 * scale + 1e-300
    assert abs(lhs - (gF * F).sum()) <= tol and abs(lhs - (gA * A).sum()) <= tol


def test_oracle_nonfinite_and_signed_zero_rules():
    """The sum starts at +0.0, so all-(-0) products give +0; inf meets 0 as NaN; products that overflow float32 but
    cancel in fp64 give a finite result where the reference's float32 products give NaN."""
    F = np.zeros((1, 4, 4), np.float32)
    A = np.zeros((1, 4, 2), np.float32)
    F[0, 0] = -0.0                                     # at m = 1 every term is (-0) * (+1 or +0) = -0
    F[0, 1, 0], A[0, 0, 1] = np.inf, 1.0               # inf * 0 at m = 0, inf * 1 at m = 1
    F[0, 2, 1] = np.nan
    F[0, 3, 2], F[0, 3, 3] = 3e38, 3e38                # 3e38 * +-3e38 overflows float32, not fp64
    A[0, 2, 0], A[0, 3, 0] = 3e38, -3e38
    out = oracle_fusion.forward(F, A)
    assert out[0, 0, 1] == 0 and not np.signbit(out[0, 0, 1])
    assert np.isnan(out[0, 1, 0]) and out[0, 1, 1] == np.inf
    assert np.isnan(out[0, 2]).all()
    assert out[0, 3, 0] == 0 and not np.signbit(out[0, 3, 0])
    with np.errstate(over="ignore", invalid="ignore"):
        ref = reference_lines(torch.from_numpy(F), torch.from_numpy(A)).numpy()
    assert np.isnan(ref[0, 3, 0])


def _cpu_args():
    return torch.zeros(2, 5, 7), torch.zeros(2, 7, 3)


def _meta(*shape):
    return torch.empty(*shape, device="meta")


@pytest.mark.parametrize("bad, msg", [
    (lambda F, A: (F.numpy(), A), "img_features must be a torch.Tensor"),
    (lambda F, A: (F, A.numpy()), "attention must be a torch.Tensor"),
    (lambda F, A: (F[0], A), "img_features must have 3 dimensions"),
    (lambda F, A: (F, A.unsqueeze(0)), "attention must have 3 dimensions"),
    (lambda F, A: (F.double(), A), "img_features must have dtype"),
    (lambda F, A: (F, A.half()), "attention must have dtype"),
    (lambda F, A: (F, A[:1]), r"img_features must be \[B,C,P\] and attention \[B,P,M\]"),
    (lambda F, A: (F, A[:, :6]), r"img_features must be \[B,C,P\] and attention \[B,P,M\]"),
    (lambda F, A: (F[:0], A[:0]), "need 1 <= B <= 65535"),
    (lambda F, A: (_meta(65536, 1, 1), _meta(65536, 1, 1)), "need 1 <= B <= 65535"),
    (lambda F, A: (F[:, :0], A), "need C, P, M >= 1"),
    (lambda F, A: (F[:, :, :0], A[:, :0]), "need C, P, M >= 1"),
    (lambda F, A: (F, A[:, :, :0]), "need C, P, M >= 1"),
    (lambda F, A: (_meta(1, 2097121, 1), _meta(1, 1, 1)), "need C, P <= 2097120"),
    (lambda F, A: (_meta(1, 1, 2097121), _meta(1, 2097121, 1)), "need C, P <= 2097120"),
    (lambda F, A: (_meta(1, 1, 1), _meta(1, 1, 2 ** 31)), "M < 2"),
    (lambda F, A: (F, A), "img_features must be a CUDA tensor"),
    (lambda F, A: (_meta(2, 5, 7), A), "img_features must be a CUDA tensor"),
])
def test_host_checks_raise_before_any_device_work(bad, msg):
    F, A = _cpu_args()
    with pytest.raises((RuntimeError, TypeError), match=msg):
        point_ops.attention_fusion(*bad(F, A))


def test_c_entry_points_validate_on_host():
    from deepi2p_b200 import _native
    lib = _native.load()
    buf = ctypes.create_string_buffer(64)
    a = ctypes.addressof(buf)
    assert lib.attn_fusion_forward_f32(a, a, 0, 1, 1, 1, a, None) == -22
    assert b"1 <= B <= 65535" in lib.dib_last_error()
    assert lib.attn_fusion_forward_f32(a, a, 65536, 1, 1, 1, a, None) == -22
    assert lib.attn_fusion_forward_f32(a, a, 1, 0, 1, 1, a, None) == -22
    assert lib.attn_fusion_forward_f32(a, a, 1, 1, 2097121, 1, a, None) == -22
    assert b"C, P <= 2097120" in lib.dib_last_error()
    assert lib.attn_fusion_forward_f32(None, a, 1, 1, 1, 1, a, None) == -22
    assert b"NULL" in lib.dib_last_error()
    assert lib.attn_fusion_backward_f32(a, -1, a, a, 1, 1, 1, 1, a, a, None) == -22
    assert lib.attn_fusion_backward_f32(None, 0, a, a, 1, 1, 1, 1, a, None, None) == -22
    assert lib.attn_fusion_backward_f32(a, 0, a, None, 1, 1, 1, 1, a, None, None) == -22     # gF reads attention
    assert lib.attn_fusion_backward_f32(a, 0, None, a, 1, 1, 1, 1, None, a, None) == -22     # gA reads features
    assert lib.attn_fusion_backward_f32(None, 0, None, None, 1, 1, 1, 1, None, None, None) == 0   # nothing asked
