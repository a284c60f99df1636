"""The encoder's cluster max-pool and node kNN grouping on the H100 (DESIGN.md 4.16): bit-exact forwards against the
numpy oracle and the reference's torch composition, deterministic feature gradients within the contract bound of the
fp64 oracle, strided and missing gradients, and a mini encoder against the torch formulation."""
import numpy as np
import pytest
import torch

import oracle_encoder
from deepi2p_b200 import point_ops
from test_encoder_ops_cpu import reference_knn, reference_pool

pytestmark = pytest.mark.gpu

POOL_SHIPPED = [(8, 32, 20480, 128), (8, 64, 20480, 128)]      # (B, C, N, M): the two pools of PCEncoder.forward
POOL_RAGGED = [(1, 1, 1, 1), (2, 33, 1000, 37), (1, 7, 3000, 129), (1, 33, 5000, 2048), (3, 1, 257, 5)]
KNN_SHIPPED = [(8, 64, 128, 128, 16)]                           # (B, C, M, N, K): node_b <- node_a, k_ab = 16
KNN_RAGGED = [(1, 1, 1, 1, 1), (2, 33, 37, 40, 16), (1, 5, 129, 32, 32), (2, 3, 2048, 200, 1), (1, 33, 50, 2048, 32),
              (2, 1, 300, 16, 16),
              (2, 4, 50, 3, 3),        # K between instantiated widths and the width above N: the all-keys pass fills it
              (1, 6, 70, 40, 5)]       # K between instantiated widths: only the first K of 8 sorted slots are written


def pool_case(seed, B, C, N, M, dev):
    """Features and the cluster assignment of a random cloud to M random nodes (cluster_assign_forward)."""
    g = torch.Generator().manual_seed(seed)
    pc = (torch.rand(B, 3, N, generator=g) * 40 - 20).to(dev)
    nodes = (torch.rand(B, 3, M, generator=g) * 40 - 20).to(dev)
    F = torch.randn(B, C, N, generator=g).to(dev)
    min_idx = point_ops.cluster_assign_forward(pc, nodes, k=1, want_centers=False)["min_idx"]
    return F, min_idx


def knn_case(seed, B, C, M, N, dev):
    g = torch.Generator().manual_seed(seed)
    q = (torch.rand(B, 3, M, generator=g) * 40 - 20).to(dev)
    db = (torch.rand(B, 3, N, generator=g) * 40 - 20).to(dev)
    F = torch.randn(B, C, N, generator=g).to(dev)
    return q, db, F


def contract_ok(got, ref, ab):
    """|gpu - oracle| <= 1 ulp_f32(oracle) + 1e-10 * sum |terms|, NaN where the oracle is NaN."""
    got = got.astype(np.float64)
    ulp = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
    ok = np.abs(got - ref) <= ulp + 1e-10 * ab
    return bool(np.all(ok | (np.isnan(got) & np.isnan(ref))))


def deterministic(grad_fn):
    """grad_fn() twice on the current stream and once on a second stream: all bit-identical."""
    g1 = grad_fn()
    assert torch.equal(grad_fn(), g1)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        g2 = grad_fn()
    torch.cuda.current_stream().wait_stream(s)
    assert torch.equal(g2, g1)
    return g1


@pytest.mark.parametrize("shape", POOL_SHIPPED + POOL_RAGGED)
def test_pool_forward_bit_exact(cuda, shape):
    B, C, N, M = shape
    F, idx = pool_case(sum(shape), *shape, cuda)
    pooled, scattered = point_ops.cluster_max_pool(F, idx, M, broadcast=True)
    rp, rs, _, _ = oracle_encoder.cluster_max_pool(F.cpu().numpy(), idx.cpu().numpy(), M, broadcast=True)
    assert pooled.shape == (B, C, M) and scattered.shape == (B, C, N)
    np.testing.assert_array_equal(pooled.cpu().numpy(), rp)
    np.testing.assert_array_equal(scattered.cpu().numpy(), rs)
    only = point_ops.cluster_max_pool(F, idx, M)
    assert isinstance(only, torch.Tensor) and torch.equal(only, pooled)


@pytest.mark.parametrize("shape", POOL_SHIPPED + [(2, 33, 1000, 37)])
def test_pool_forward_equals_reference_composition(cuda, shape):
    B, C, N, M = shape
    F, idx = pool_case(3 + sum(shape), *shape, cuda)
    # the reference lines on the device: index_max_forward, .long(), gather, times mask_row_max, gather
    rp, rs = reference_pool(F, idx, point_ops.index_max_forward(F, idx, M), M)
    pooled, scattered = point_ops.cluster_max_pool(F, idx, M, broadcast=True)
    assert torch.equal(pooled, rp) and torch.equal(scattered, rs)


def test_pool_forward_quirks(cuda):
    """Empty segments (features[b, c, 0] * 0.0f: -0.0 and NaN), segments at or below -1000, all-NaN segments and
    points outside [0, M)."""
    B, C, N, M = 2, 6, 700, 40
    F, idx = pool_case(5, B, C, N, M, cuda)
    idx = idx.clone()
    idx[idx == 7] = 8                                    # segment 7 is empty
    F = F.clone()
    F[:, 0, 0], F[:, 1, 0], F[:, 2, 0] = -2.5, float("nan"), float("inf")
    F[0, 3][idx[0] == 11] = -1000.0                       # at the floor: no winner
    F[1, 4][idx[1] == 12] = float("nan")                  # all NaN: no winner
    idx[0, 5], idx[1, 6], idx[1, 9] = M, -1, 1 << 30
    pooled, scattered = point_ops.cluster_max_pool(F, idx, M, broadcast=True)
    rp, rs, sel, mask = oracle_encoder.cluster_max_pool(F.cpu().numpy(), idx.cpu().numpy(), M, broadcast=True)
    np.testing.assert_array_equal(pooled.cpu().numpy(), rp)
    np.testing.assert_array_equal(scattered.cpu().numpy(), rs)
    p = pooled.cpu()
    assert p[0, 0, 7] == 0 and torch.signbit(p[0, 0, 7]) and torch.isnan(p[:, 1:3, 7]).all()
    assert torch.isnan(scattered[0, :, 5]).all() and torch.isnan(scattered[1, :, 6]).all()
    assert sel[0, 3, 11] == 0 and sel[1, 4, 12] == 0

    def grad():
        Fr = F.clone().requires_grad_(True)
        a, b = point_ops.cluster_max_pool(Fr, idx, M, broadcast=True)
        torch.autograd.backward((a, b), (torch.ones_like(a), torch.ones_like(b)))
        return Fr.grad

    g = deterministic(grad)
    ref, ab = oracle_encoder.cluster_max_pool_backward(F.cpu().numpy(), idx.cpu().numpy(), M,
                                                       np.ones((B, C, M), np.float32), np.ones((B, C, N), np.float32),
                                                       with_abs=True)
    assert contract_ok(g.cpu().numpy(), ref, ab)
    assert (g[0, :, 5] == 0).all() and (g[1, :, 6] == 0).all() and (g[1, :, 9] == 0).all()


@pytest.mark.parametrize("shape", POOL_SHIPPED + POOL_RAGGED)
def test_pool_backward_contract_and_determinism(cuda, shape):
    B, C, N, M = shape
    F, idx = pool_case(11 + sum(shape), *shape, cuda)
    gP = torch.randn(B, C, M, device=cuda)
    gS = torch.randn(B, C, N, device=cuda)

    def grad():
        Fr = F.clone().requires_grad_(True)
        a, b = point_ops.cluster_max_pool(Fr, idx, M, broadcast=True)
        torch.autograd.backward((a, b), (gP, gS))
        return Fr.grad

    g = deterministic(grad)
    ref, ab = oracle_encoder.cluster_max_pool_backward(F.cpu().numpy(), idx.cpu().numpy(), M, gP.cpu().numpy(),
                                                       gS.cpu().numpy(), with_abs=True)
    assert contract_ok(g.cpu().numpy(), ref, ab)


def test_pool_missing_gradients(cuda):
    """broadcast=False, and a pooled or scattered output that takes no part in the loss: the missing gradient is
    treated as zero without being materialised."""
    B, C, N, M = 2, 40, 3000, 64
    F, idx = pool_case(17, B, C, N, M, cuda)
    gP = torch.randn(B, C, M, device=cuda)
    gS = torch.randn(B, C, N, device=cuda)
    Fn, ix = F.cpu().numpy(), idx.cpu().numpy()
    cases = [(False, True, False), (True, True, False), (True, False, True)]   # (broadcast, use pooled, use scattered)
    for broadcast, use_p, use_s in cases:
        Fr = F.clone().requires_grad_(True)
        out = point_ops.cluster_max_pool(Fr, idx, M, broadcast=broadcast)
        pooled, scattered = out if broadcast else (out, None)
        loss = (pooled * gP).sum() if use_p else 0
        if use_s:
            loss = loss + (scattered * gS).sum()
        loss.backward()
        ref, ab = oracle_encoder.cluster_max_pool_backward(Fn, ix, M, gP.cpu().numpy() if use_p else None,
                                                           gS.cpu().numpy() if use_s else None, with_abs=True)
        assert contract_ok(Fr.grad.cpu().numpy(), ref, ab), (broadcast, use_p, use_s)


def test_pool_grad_from_torch_cat_slice(cuda):
    """In the encoder the scattered output feeds torch.cat (networks_pc.py:98): its gradient arrives as a slice."""
    B, C, N, M = 4, 32, 4000, 64
    F, idx = pool_case(21, B, C, N, M, cuda)
    G = torch.randn(B, 2 * C, N, device=cuda)
    seen = []
    Fa = F.clone().requires_grad_(True)
    _, s = point_ops.cluster_max_pool(Fa, idx, M, broadcast=True)
    s.register_hook(lambda t: seen.append(t.is_contiguous()))
    (torch.cat((F, s), dim=1) * G).sum().backward()
    assert seen == [False]
    Fb = F.clone().requires_grad_(True)
    _, s = point_ops.cluster_max_pool(Fb, idx, M, broadcast=True)
    s.backward(G[:, C:].contiguous())
    assert torch.equal(Fa.grad, Fb.grad)


@pytest.mark.parametrize("shape", KNN_SHIPPED + KNN_RAGGED)
def test_knn_forward_bit_exact(cuda, shape):
    B, C, M, N, K = shape
    q, db, F = knn_case(sum(shape), B, C, M, N, cuda)
    idx, grouped = point_ops.knn_group(q, db, F, K)
    ri, rg = oracle_encoder.knn_group(q.cpu().numpy(), db.cpu().numpy(), F.cpu().numpy(), K)
    assert idx.dtype == torch.int32 and idx.shape == (B, M, K) and grouped.shape == (B, 3 + C, M, K)
    np.testing.assert_array_equal(idx.cpu().numpy(), ri)
    np.testing.assert_array_equal(grouped.cpu().numpy(), rg)


def test_knn_forward_ties_and_non_finite(cuda):
    """Exact ties (duplicated database nodes) go to the lower index; +inf and NaN keys come last, in that order."""
    B, C, M, N, K = 2, 4, 100, 64, 32
    q, db, F = knn_case(41, B, C, M, N, cuda)
    db = db.clone()
    db[:, :, 32:48] = db[:, :, 0:16]                       # duplicates: equal keys
    q = torch.round(q)
    db[:, :, 48:56] = torch.round(db[:, :, 48:56])         # integer grids: many equal keys
    db[0, 0, 60] = float("inf")
    db[1, 1, 61] = float("nan")
    db[0, 2, 62] = 3e38                                    # the key overflows to +inf
    idx, grouped = point_ops.knn_group(q, db, F, K)
    ri, rg = oracle_encoder.knn_group(q.cpu().numpy(), db.cpu().numpy(), F.cpu().numpy(), K)
    np.testing.assert_array_equal(idx.cpu().numpy(), ri)
    np.testing.assert_array_equal(grouped.cpu().numpy(), rg)
    # K = N over the last 32 nodes (duplicates, integer grid, non-finite): every node appears, the non-finite keys last
    qs, dbs, Fs = q[:, :, :5].contiguous(), db[:, :, 32:].contiguous(), F[:, :, 32:].contiguous()
    idx, _ = point_ops.knn_group(qs, dbs, Fs, 32)
    ri, _ = oracle_encoder.knn_group(qs.cpu().numpy(), dbs.cpu().numpy(), Fs.cpu().numpy(), 32)
    np.testing.assert_array_equal(idx.cpu().numpy(), ri)
    assert sorted(idx[0, 0].tolist()) == list(range(32)) and set(idx[0, :, -2:].flatten().tolist()) <= {28, 30}
    assert (idx[1, :, -1] == 29).all()


@pytest.mark.parametrize("shape", KNN_SHIPPED + [(2, 33, 37, 40, 16)])
def test_knn_forward_equals_torch_formulation(cuda, shape):
    B, C, M, N, K = shape
    q, db, F = knn_case(7 + sum(shape), B, C, M, N, cuda)
    idx, grouped = point_ops.knn_group(q, db, F, K)
    ri, norm, rg = reference_knn(q, db, F, K)
    srt = torch.sort(norm, dim=2)[0][:, :, :K + 1]
    clean = (torch.diff(srt, dim=2) > 0).all(dim=2)        # no two keys tie or round to the same norm
    assert clean.float().mean() > 0.9
    assert torch.equal(idx[clean], ri.int()[clean])
    assert torch.equal(grouped.permute(0, 2, 1, 3)[clean], rg.permute(0, 2, 1, 3)[clean])


@pytest.mark.parametrize("shape", KNN_SHIPPED + KNN_RAGGED)
def test_knn_backward_contract_and_determinism(cuda, shape):
    B, C, M, N, K = shape
    q, db, F = knn_case(13 + sum(shape), B, C, M, N, cuda)
    g = torch.randn(B, 3 + C, M, K, device=cuda)

    def grad():
        Fr = F.clone().requires_grad_(True)
        _, grouped = point_ops.knn_group(q, db, Fr, K)
        grouped.backward(g)
        return Fr.grad

    gF = deterministic(grad)
    idx, _ = point_ops.knn_group(q, db, F, K)
    ref, ab = oracle_encoder.knn_group_backward(idx.cpu().numpy(), g.cpu().numpy(), N, with_abs=True)
    assert contract_ok(gF.cpu().numpy(), ref, ab)


def test_knn_grad_from_torch_cat_slice(cuda):
    B, C, M, N, K = 3, 20, 64, 100, 16
    q, db, F = knn_case(23, B, C, M, N, cuda)
    G = torch.randn(B, 3 + C + 5, M, K, device=cuda)
    other = torch.randn(B, 5, M, K, device=cuda)
    Fa = F.clone().requires_grad_(True)
    _, grouped = point_ops.knn_group(q, db, Fa, K)
    (torch.cat((other, grouped), dim=1) * G).sum().backward()
    Fb = F.clone().requires_grad_(True)
    _, grouped = point_ops.knn_group(q, db, Fb, K)
    grouped.backward(G[:, 5:].contiguous())
    assert torch.equal(Fa.grad, Fb.grad)


def test_knn_grad_strided_rows_at_one_query_one_neighbour(cuda):
    """At M = K = 1 a slice of a torch.cat along dim 3 has row stride 2, not M * K = 1: it must not be read as if
    its rows were packed."""
    B, C, M, N, K = 2, 4, 1, 10, 1
    q, db, F = knn_case(29, B, C, M, N, cuda)
    other = torch.randn(B, 3 + C, M, 1, device=cuda)
    G = torch.randn(B, 3 + C, M, 2, device=cuda)
    seen = []
    Fa = F.clone().requires_grad_(True)
    _, grouped = point_ops.knn_group(q, db, Fa, K)
    grouped.register_hook(lambda t: seen.append(t.stride()))
    (torch.cat((grouped, other), dim=3) * G).sum().backward()
    assert seen and seen[0][1] != M * K, seen                 # the slice really was strided along the rows
    Fb = F.clone().requires_grad_(True)
    _, grouped = point_ops.knn_group(q, db, Fb, K)
    grouped.backward(G[:, :, :, :1].contiguous())
    assert torch.equal(Fa.grad, Fb.grad)
    idx, _ = point_ops.knn_group(q, db, F, K)
    ref = oracle_encoder.knn_group_backward(idx.cpu().numpy(), G[:, :, :, :1].cpu().numpy(), N)
    np.testing.assert_array_equal(Fa.grad.cpu().numpy(), ref)      # one term per (b, c, n): exact


class MiniEncoder(torch.nn.Module):
    """PCEncoder's point branch at the shipped layer widths, shortened: conv -> pool with broadcast -> cat -> conv ->
    pool -> kNN grouping -> conv2d -> max over the neighbours."""

    def __init__(self):
        super().__init__()
        g = torch.Generator().manual_seed(0)
        self.first = torch.nn.Conv1d(7, 32, 1)
        self.second = torch.nn.Conv1d(64, 64, 1)
        self.knn = torch.nn.Conv2d(3 + 64, 128, 1)
        for p in self.parameters():
            p.data = torch.randn(p.shape, generator=g) * 0.2

    def forward(self, pc_aug, pc, node_a, node_b, k_ab, project_ops):
        B, _, N = pc.shape
        Ma = node_a.shape[2]
        ca = point_ops.cluster_assign_forward(pc, node_a, k=1, want_centers=False)
        min_idx, cluster_mean = ca["min_idx"], ca["cluster_mean"]
        first = torch.relu(self.first(pc_aug))
        if project_ops:
            _, scattered = point_ops.cluster_max_pool(first, min_idx, Ma, broadcast=True)
        else:
            _, scattered = reference_pool(first, min_idx, point_ops.index_max_forward(first.detach(), min_idx, Ma), Ma)
        second = torch.relu(self.second(torch.cat((first, scattered), dim=1)))
        if project_ops:
            node_a_features = point_ops.cluster_max_pool(second, min_idx, Ma)
            _, grouped = point_ops.knn_group(node_b, cluster_mean, node_a_features, k_ab)
        else:
            node_a_features, _ = reference_pool(second, min_idx,
                                                point_ops.index_max_forward(second.detach(), min_idx, Ma), Ma)
            _, _, grouped = reference_knn(node_b, cluster_mean, node_a_features, k_ab)
        feature, _ = torch.max(torch.relu(self.knn(grouped)), dim=3)
        return (feature ** 2).mean()


def test_mini_encoder_matches_torch_and_is_deterministic(cuda):
    torch.backends.cudnn.deterministic = True
    try:
        g = torch.Generator().manual_seed(3)
        B, N, Ma, Mb, k_ab = 2, 4096, 128, 128, 16
        pc = (torch.rand(B, 3, N, generator=g) * 40 - 20).to(cuda)
        pc_aug = torch.cat((pc / 20, torch.rand(B, 4, N, generator=g).to(cuda)), dim=1)
        node_a = pc[:, :, torch.randperm(N, generator=g)[:Ma].to(cuda)].contiguous()
        node_b = pc[:, :, torch.randperm(N, generator=g)[:Mb].to(cuda)].contiguous()
        net = MiniEncoder().to(cuda)

        def run(project_ops):
            net.zero_grad()
            loss = net(pc_aug, pc, node_a, node_b, k_ab, project_ops)
            loss.backward()
            return loss.detach().clone(), [p.grad.clone() for p in net.parameters()]

        loss_op, grads_op = run(True)
        loss_ref, grads_ref = run(False)
        torch.testing.assert_close(loss_op, loss_ref, rtol=1e-5, atol=0)
        for a, b in zip(grads_op, grads_ref):
            torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5 * float(b.abs().max()))
        loss_again, grads_again = run(True)
        assert torch.equal(loss_again, loss_op)
        assert all(torch.equal(a, b) for a, b in zip(grads_again, grads_op))
    finally:
        torch.backends.cudnn.deterministic = False
