"""The attention-weighted image-feature fusion on the H100 (DESIGN.md 4.17): forward and both gradients bit-exact against
oracle_fusion at the shipped and ragged shapes and with non-finite and signed-zero inputs, agreement with the
reference's float32 mul + mean within the stated bound, determinism (repeat, second stream, batch split, TF32 flags),
gradient plumbing (torch.cat slices, every needs_input_grad combination) and a mini fusion block against the torch
formulation."""
import numpy as np
import pytest
import torch

import oracle_fusion
from deepi2p_b200 import point_ops
from test_fusion_cpu import reference_lines

pytestmark = pytest.mark.gpu

# (B, C, P, M): the s32 call (C = 512, node_b) and the s16 call (C = 256, node_a) at KITTI 160 x 512 (B = 8), Oxford
# 384 x 640 (B = 8) and nuScenes 160 x 320 (B = 12)
SHIPPED = [(8, 512, 80, 128), (8, 256, 320, 128), (8, 512, 240, 128), (8, 256, 960, 128), (12, 512, 50, 128),
           (12, 256, 200, 128)]
RAGGED = [(1, 1, 1, 1), (2, 33, 50, 129), (3, 7, 1, 5), (1, 1, 960, 1), (2, 513, 81, 127),
          (6, 700, 333, 450)]      # all three products on the 64 x 64 tiles, every dimension ragged


def case(seed, B, C, P, M, dev):
    g = torch.Generator().manual_seed(seed)
    F = torch.randn(B, C, P, generator=g)
    A = torch.randn(B, P, M, generator=g) * 3
    gO = torch.randn(B, C, M, generator=g)
    return F.to(dev), A.to(dev), gO.to(dev)


def run(F, A, gO, need_F=True, need_A=True):
    """(out, gF, gA) of the op, gradients None where not asked."""
    Fr = F.clone().requires_grad_(need_F)
    Ar = A.clone().requires_grad_(need_A)
    out = point_ops.attention_fusion(Fr, Ar)
    if need_F or need_A:
        out.backward(gO)
    return out.detach(), Fr.grad, Ar.grad


def assert_bits(got, ref):
    """Equal values, NaN at the same positions, and the same sign on every zero."""
    got = got.cpu().numpy()
    np.testing.assert_array_equal(got, ref)
    nz = ~np.isnan(ref)
    assert np.array_equal(np.signbit(got[nz]), np.signbit(ref[nz]))


def check_against_oracle(F, A, gO):
    out, gF, gA = run(F, A, gO)
    Fn, An, gn = F.cpu().numpy(), A.cpu().numpy(), gO.cpu().numpy()
    assert_bits(out, oracle_fusion.forward(Fn, An))
    assert_bits(gF, oracle_fusion.backward_features(An, gn))
    assert_bits(gA, oracle_fusion.backward_attention(Fn, gn))


@pytest.mark.parametrize("shape", SHIPPED + RAGGED)
def test_forward_and_gradients_bit_exact(cuda, shape):
    check_against_oracle(*case(sum(shape), *shape, cuda))


def test_nonfinite_and_signed_zero_inputs(cuda):
    """inf, NaN, all-(-0) products (+0 out), inf - inf, and float32-overflowing products that cancel in fp64, at a
    shape on 32 x 32 tiles and one whose forward runs on 64 x 64 tiles."""
    for B, C, P, M in ((2, 96, 70, 130), (6, 700, 40, 450)):
        F, A, gO = case(40 + B, B, C, P, M, cuda)
        F[:, 0] = -0.0                                  # row 0 at m = 1: (-0) * (+|a|) in every term
        A[:, :, 1] = A[:, :, 1].abs()
        F[:, 1, 3] = float("inf")                       # inf * finite, inf * 0 -> NaN
        A[:, 3, 5] = 0.0
        F[:, 2, 4], F[:, 2, 9] = float("inf"), float("-inf")      # inf - inf -> NaN wherever both A > 0
        F[:, 3, 7] = float("nan")
        A[:, 11, 17] = float("nan")                     # column 17 NaN for every c
        F[:, 4, 20], F[:, 4, 21] = 3e38, 3e38            # 3e38 * +-3e38: inf - inf in float32, 0 in fp64
        A[:, 20, 6], A[:, 21, 6] = 3e38, -3e38
        gO[:, 5, 8] = -0.0
        gO[:, 6, 9] = float("inf")
        check_against_oracle(F, A, gO)
        out = point_ops.attention_fusion(F, A).cpu()
        assert (out[:, 0, 1] == 0).all() and not torch.signbit(out[:, 0, 1]).any()
        assert torch.isnan(out[:, :, 17]).all() and torch.isfinite(out[:, 4, 6]).all()
        assert torch.isnan(reference_lines(F, A)[:, 4, 6]).all()


def bound_ok(got, ref, scale, n):
    """|got - ref| <= (n + 1) 2^-24 scale + 1 ulp_f32, scale = sum |terms| / P from the oracle."""
    got, ref = got.detach().cpu().numpy().astype(np.float64), ref.detach().cpu().numpy().astype(np.float64)
    ulp = np.spacing(np.abs(got).astype(np.float32)).astype(np.float64)
    return bool(np.all(np.abs(got - ref) <= (n + 1) * 2.0 ** -24 * scale + ulp))


@pytest.mark.parametrize("shape", SHIPPED)
def test_agrees_with_reference_formulation_within_bound(cuda, shape):
    B, C, P, M = shape
    F, A, gO = case(7 + sum(shape), *shape, cuda)
    out, gF, gA = run(F, A, gO)
    Fr, Ar = F.clone().requires_grad_(True), A.clone().requires_grad_(True)
    ref = reference_lines(Fr, Ar)
    ref.backward(gO)
    Fn, An, gn = F.cpu().numpy(), A.cpu().numpy(), gO.cpu().numpy()
    _, s = oracle_fusion.forward(Fn, An, with_abs=True)
    assert bound_ok(out, ref, s, P)
    # the reference's backward divides gO by P before its products: one more rounding per term
    _, s = oracle_fusion.backward_features(An, gn, with_abs=True)
    assert bound_ok(gF, Fr.grad, s, M + 1)
    _, s = oracle_fusion.backward_attention(Fn, gn, with_abs=True)
    assert bound_ok(gA, Ar.grad, s, C + 1)


@pytest.mark.parametrize("shape", [(8, 256, 960, 128), (8, 512, 80, 128), (2, 513, 81, 127)])
def test_deterministic_repeat_stream_batch_split_and_tf32(cuda, shape):
    F, A, gO = case(3 + sum(shape), *shape, cuda)
    first = run(F, A, gO)
    again = run(F, A, gO)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        other = run(F, A, gO)
    torch.cuda.current_stream().wait_stream(s)
    flags = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    try:
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = True
        tf32 = run(F, A, gO)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = flags
    for r in (again, other, tf32):
        for x, y in zip(first, r):
            assert torch.equal(x, y)
    for b in {0, shape[0] - 1}:          # one sample alone: other tile sizes, the same bits
        alone = run(F[b:b + 1].contiguous(), A[b:b + 1].contiguous(), gO[b:b + 1].contiguous())
        for x, y in zip(first, alone):
            assert torch.equal(x[b:b + 1], y)


@pytest.mark.parametrize("shape", [(4, 512, 80, 128), (3, 1, 50, 128), (3, 64, 50, 1), (2, 1, 7, 1)])
def test_cat_slice_gradient_equals_contiguous(cuda, shape):
    """out joins a torch.cat along channels, as node_b_pn's input does (networks_united.py:152-156): its gradient is a
    strided channel slice, read in place.  A cat along the node dimension gives a slice the op copies."""
    B, C, P, M = shape
    F, A, _ = case(5 + sum(shape), *shape, cuda)
    g = torch.Generator().manual_seed(9)
    node = torch.randn(B, 64, M, generator=g).to(cuda)
    glob = torch.randn(B, 32, 1, generator=g).to(cuda)
    G = torch.randn(B, 64 + 32 + C + 32, M, generator=g).to(cuda)
    Fr, Ar = F.clone().requires_grad_(True), A.clone().requires_grad_(True)
    out = point_ops.attention_fusion(Fr, Ar)
    torch.cat((node, glob.expand(B, 32, M), out, glob.expand(B, 32, M)), dim=1).backward(G)
    _, gF, gA = run(F, A, G[:, 96:96 + C].contiguous())
    assert torch.equal(Fr.grad, gF) and torch.equal(Ar.grad, gA)
    G2 = torch.randn(B, C, 3 * M, generator=g).to(cuda)
    Fr, Ar = F.clone().requires_grad_(True), A.clone().requires_grad_(True)
    out = point_ops.attention_fusion(Fr, Ar)
    torch.cat((out.new_zeros(B, C, M), out, out.new_zeros(B, C, M)), dim=2).backward(G2)
    _, gF, gA = run(F, A, G2[:, :, M:2 * M].contiguous())
    assert torch.equal(Fr.grad, gF) and torch.equal(Ar.grad, gA)


def test_every_needs_input_grad_combination(cuda):
    F, A, gO = case(21, 2, 40, 90, 33, cuda)
    full = run(F, A, gO)
    for need_F, need_A in ((True, False), (False, True)):
        out, gF, gA = run(F, A, gO, need_F, need_A)
        assert torch.equal(out, full[0])
        assert (gF is None) == (not need_F) and (gA is None) == (not need_A)
        if need_F:
            assert torch.equal(gF, full[1])
        if need_A:
            assert torch.equal(gA, full[2])
    out, gF, gA = run(F, A, gO, False, False)
    assert not out.requires_grad and gF is None and gA is None and torch.equal(out, full[0])


def test_layout_and_device_checks(cuda):
    F, A, _ = case(22, 2, 5, 7, 3, cuda)
    with pytest.raises(RuntimeError, match="img_features must be contiguous"):
        point_ops.attention_fusion(F.transpose(1, 2).contiguous().transpose(1, 2), A)
    with pytest.raises(RuntimeError, match="attention must be a CUDA tensor"):
        point_ops.attention_fusion(F, A.cpu())


def test_mini_fusion_block(cuda):
    """A conv1d attention head produces A from node features, the op fuses an image feature map, a conv1d and a loss
    follow.  Loss and weight gradients match the torch formulation within float32 tolerance and are bit-identical
    across two runs."""
    B, Cn, C, P, M = 4, 64, 256, 320, 128
    flags = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32
    # float32 convolutions: both paths then differ only by the fusion's rounding
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32 = True, False, False
    try:
        g = torch.Generator().manual_seed(31)
        node = torch.randn(B, Cn, M, generator=g).to(cuda)
        img = torch.randn(B, C, 16, 20, generator=g).to(cuda)
        torch.manual_seed(0)
        head = torch.nn.Conv1d(Cn, P, 1).to(cuda)
        tail = torch.nn.Conv1d(C, 32, 1).to(cuda)

        def step(fuse):
            for p in list(head.parameters()) + list(tail.parameters()):
                p.grad = None
            Fi = img.clone().requires_grad_(True)
            A = head(node)
            y = tail(fuse(Fi.view(B, C, -1), A))
            loss = (y * y).mean()
            loss.backward()
            return [loss.detach(), head.weight.grad.clone(), head.bias.grad.clone(), tail.weight.grad.clone(),
                    Fi.grad.clone()]

        got = step(point_ops.attention_fusion)
        again = step(point_ops.attention_fusion)
        ref = step(reference_lines)
        for x, y, r in zip(got, again, ref):
            assert torch.equal(x, y)
            torch.testing.assert_close(x, r, rtol=1e-4, atol=1e-5 * float(r.abs().max()))
    finally:
        torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark, torch.backends.cudnn.allow_tf32 = flags
