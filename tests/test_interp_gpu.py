"""Decoder interpolation on the H100 (DESIGN.md 4.12): bit-exact forward against the numpy oracle, a deterministic
feature gradient within the contract bound of the fp64 oracle, strided gradients, bad indices, memory, and a tiny
decoder trained one step against the reference's formulation."""
import numpy as np
import pytest
import torch

import oracle_interp
from deepi2p_b200 import point_ops
from test_interp_cpu import formulation

pytestmark = pytest.mark.gpu

SHIPPED = [  # (B, Nq, M, C, k): points <- node_b, node_a <- node_b, points <- node_a (KITTI / Oxford options)
    (8, 20480, 128, 512, 3),
    (8, 128, 128, 512, 3),
    (8, 20480, 128, 128, 3),
]
RAGGED = [
    (1, 1, 5, 7, 3),
    (2, 300, 100, 70, 3),          # M below the backward's node range, C not a multiple of any chunk
    (2, 257, 129, 33, 8),          # two node ranges in the backward, one point past a forward tile
    (3, 1000, 37, 1, 1),
    (2, 700, 2048, 20, 8),         # M at the bound: forward chunks of 8 channels, 16 node ranges in the backward
    (1, 4096, 300, 96, 4),
]


def cloud_case(seed, B, Nq, M, C, k, dev):
    """Query points, nodes and features with indices from cluster_assign_forward (nearest first)."""
    g = torch.Generator().manual_seed(seed)
    q = (torch.rand(B, 3, Nq, generator=g) * 40 - 20).to(dev)
    nd = (torch.rand(B, 3, M, generator=g) * 40 - 20).to(dev)
    F = torch.randn(B, C, M, generator=g).to(dev)
    idx = point_ops.cluster_assign_forward(q, nd, k=k, want_centers=False)["min_k_idx"]
    return idx, q, nd, F


def contract_ok(got, ref, ab):
    """|gpu - oracle| <= 1 ulp_f32(oracle) + 1e-10 * sum |w g|, NaN where the oracle is NaN."""
    got = got.astype(np.float64)
    ulp = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
    ok = np.abs(got - ref) <= ulp + 1e-10 * ab
    return bool(np.all(ok | (np.isnan(got) & np.isnan(ref))))


@pytest.mark.parametrize("shape", SHIPPED + RAGGED)
@pytest.mark.parametrize("idx_dtype", [torch.int32, torch.int64])
def test_forward_bit_exact(cuda, shape, idx_dtype):
    idx, q, nd, F = cloud_case(sum(shape), *shape, cuda)
    idx = idx.to(idx_dtype)
    out = point_ops.upsample_by_interpolation(idx, q, nd, F)
    ref = oracle_interp.interp_forward(idx.cpu().numpy(), q.cpu().numpy(), nd.cpu().numpy(), F.cpu().numpy())
    assert out.shape == ref.shape and out.dtype == torch.float32
    np.testing.assert_array_equal(out.cpu().numpy(), ref)


@pytest.mark.parametrize("shape", SHIPPED)
def test_forward_close_to_formulation(cuda, shape):
    idx, q, nd, F = cloud_case(5, *shape, cuda)
    out = point_ops.upsample_by_interpolation(idx, q, nd, F)
    ref = formulation(idx, q, nd, F)
    # the weights differ by the norm's rounding only (a few ulps): tolerance scaled by |F| and k
    torch.testing.assert_close(out, ref, rtol=1e-5, atol=1e-5 * shape[4], equal_nan=False)


@pytest.mark.parametrize("shape", SHIPPED + RAGGED)
def test_backward_contract_and_determinism(cuda, shape):
    B, Nq, M, C, k = shape
    idx, q, nd, F = cloud_case(11 + sum(shape), *shape, cuda)
    g = torch.randn(B, C, Nq, device=cuda)

    def grad():
        Fr = F.clone().requires_grad_(True)
        point_ops.upsample_by_interpolation(idx, q, nd, Fr).backward(g)
        return Fr.grad

    g1 = grad()
    ref, ab = oracle_interp.interp_backward(idx.cpu().numpy(), q.cpu().numpy(), nd.cpu().numpy(), g.cpu().numpy(), M,
                                            with_abs=True)
    assert contract_ok(g1.cpu().numpy(), ref, ab)
    assert torch.equal(grad(), g1)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        g2 = grad()
    torch.cuda.current_stream().wait_stream(s)
    assert torch.equal(g2, g1)


def test_grad_from_torch_cat_slice(cuda):
    """In the network the output feeds torch.cat: its gradient arrives as a batch-strided slice."""
    B, Nq, M, C, k = 4, 3000, 128, 96, 3
    idx, q, nd, F = cloud_case(21, B, Nq, M, C, k, cuda)
    other = torch.randn(B, 40, Nq, device=cuda)
    G = torch.randn(B, C + 40, Nq, device=cuda)
    seen = []
    Fa = F.clone().requires_grad_(True)
    out = point_ops.upsample_by_interpolation(idx, q, nd, Fa)
    out.register_hook(lambda t: seen.append((t.is_contiguous(), t.stride())))
    (torch.cat((other, out), dim=1) * G).sum().backward()
    assert seen and not seen[0][0], seen                 # the slice really was strided
    Fb = F.clone().requires_grad_(True)
    point_ops.upsample_by_interpolation(idx, q, nd, Fb).backward(G[:, 40:].contiguous())
    assert torch.equal(Fa.grad, Fb.grad)


def test_out_of_range_index(cuda):
    B, Nq, M, C, k = 2, 500, 64, 48, 3
    idx, q, nd, F = cloud_case(31, B, Nq, M, C, k, cuda)
    bad = idx.clone().long()
    bad[0, 7, 1] = M
    bad[1, 100, 0] = -3
    bad[1, 101, 2] = 1 << 40                             # wraps to a valid int32 if narrowed: must still be caught
    Fr = F.clone().requires_grad_(True)
    out = point_ops.upsample_by_interpolation(bad, q, nd, Fr)
    o = out.detach().cpu()
    assert torch.isnan(o[0, :, 7]).all() and torch.isnan(o[1, :, 100]).all() and torch.isnan(o[1, :, 101]).all()
    o[0, :, 7] = 0
    o[1, :, 100:102] = 0
    assert torch.isfinite(o).all()
    g = torch.randn(B, C, Nq, device=cuda)
    out.backward(g)
    assert torch.isfinite(Fr.grad).all()
    # the oracle with those points removed (batch by batch: the removed sets differ)
    for b, drop in ((0, [7]), (1, [100, 101])):
        keep = [n for n in range(Nq) if n not in drop]
        sl = lambda t: t[b:b + 1].cpu().numpy()  # noqa: E731
        ref, ab = oracle_interp.interp_backward(sl(idx)[:, keep], sl(q)[:, :, keep], sl(nd), sl(g)[:, :, keep], M,
                                                with_abs=True)
        assert contract_ok(Fr.grad[b:b + 1].cpu().numpy(), ref, ab), b


def test_peak_memory(cuda):
    """Beyond its output the op allocates O(B Nq k): the weights and int32 indices it keeps for the backward."""
    B, Nq, M, C, k = SHIPPED[0]
    idx, q, nd, F = cloud_case(41, B, Nq, M, C, k, cuda)
    Fr = F.clone().requires_grad_(True)
    g = torch.randn(B, C, Nq, device=cuda)
    point_ops.upsample_by_interpolation(idx, q, nd, Fr).backward(g)      # warm: the per-stream workspace exists
    Fr.grad = None
    torch.cuda.synchronize()
    small = 2 * B * Nq * k * 4 + (1 << 20)
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = point_ops.upsample_by_interpolation(idx, q, nd, Fr)
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - base <= out.numel() * 4 + small
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out.backward(g)
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - base <= Fr.numel() * 4 + small


class Decoder(torch.nn.Module):
    """conv on node features -> interpolation to the points -> cat with per-point features -> conv."""

    def __init__(self, interp):
        super().__init__()
        self.interp = interp
        self.node_pn = torch.nn.Conv1d(16, 64, 1)
        self.point_pn = torch.nn.Conv1d(64 + 8, 4, 1)

    def forward(self, idx, pc, node, node_feat, point_feat):
        up = self.interp(idx, pc, node, torch.relu(self.node_pn(node_feat)))
        return self.point_pn(torch.cat((up, point_feat), dim=1))


def test_decoder_end_to_end(cuda):
    B, N, M, k = 4, 4096, 128, 3
    torch.manual_seed(0)
    pc = torch.randn(B, 3, N, device=cuda) * 10
    node = torch.randn(B, 3, M, device=cuda) * 10
    idx = point_ops.cluster_assign_forward(pc, node, k=k, want_centers=False)["min_k_idx"]
    node_feat = torch.randn(B, 16, M, device=cuda)
    point_feat = torch.randn(B, 8, N, device=cuda)
    target = torch.randn(B, 4, N, device=cuda)
    nets = [Decoder(point_ops.upsample_by_interpolation).to(cuda), Decoder(formulation).to(cuda)]
    nets[1].load_state_dict(nets[0].state_dict())
    losses = []
    for net in nets:
        loss = torch.nn.functional.mse_loss(net(idx, pc, node, node_feat, point_feat), target)
        loss.backward()
        losses.append(loss.detach())
    # fp32 on both sides; they differ by the norm's rounding and the gradient's summation order
    torch.testing.assert_close(losses[0], losses[1], rtol=1e-5, atol=0)
    for p0, p1 in zip(nets[0].parameters(), nets[1].parameters()):
        torch.testing.assert_close(p0.grad, p1.grad, rtol=1e-4, atol=1e-6)
