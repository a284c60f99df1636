"""The encoder ops' oracle (DESIGN.md 4.16) against torch restatements of the reference lines, their quirks, and the
host argument checks of point_ops.cluster_max_pool / point_ops.knn_group (no device needed)."""
import numpy as np
import pytest
import torch

import oracle_encoder
from deepi2p_b200 import point_ops


def reference_pool(F, min_idx, sel, M):
    """models/networks_pc.py:66-69 and :88-97 in torch, at F's dtype: gather by sel, times mask_row_max, gather by
    min_idx.  Every index must be in [0, M)."""
    B, C, N = F.shape
    idx = min_idx.long()
    mask = torch.eq(idx.unsqueeze(2).expand(B, N, M), torch.arange(M, device=F.device).view(1, 1, M).expand(B, N, M))
    mask_row_max, _ = torch.max(mask, dim=1, keepdim=False)
    pooled = F.gather(dim=2, index=sel.long()) * mask_row_max.unsqueeze(1).to(dtype=F.dtype)
    scattered = torch.gather(pooled, dim=2, index=idx.unsqueeze(1).expand(B, C, N))
    return pooled, scattered


def reference_knn(query, database, features, K):
    """models/layers_pc.py:795-807 in torch at the inputs' dtype."""
    B, M, N, C = query.size(0), query.size(2), database.size(2), features.size(1)
    q = query.detach().unsqueeze(3)
    d = database.detach().unsqueeze(2)
    norm = torch.norm(q - d, dim=1, keepdim=False)
    knn_D, knn_I = torch.topk(norm, k=K, dim=2, largest=False, sorted=True)
    I3 = knn_I.unsqueeze(1).expand(B, 3, M, K).contiguous().view(B, 3, M * K)
    IC = knn_I.unsqueeze(1).expand(B, C, M, K).contiguous().view(B, C, M * K)
    coord = torch.gather(database, dim=2, index=I3).view(B, 3, M, K)
    feat = torch.gather(features, dim=2, index=IC).view(B, C, M, K)
    return knn_I, norm, torch.cat(((coord - q).detach(), feat), dim=1)


def pool_case(seed, B, C, N, M, empty=()):
    rng = np.random.default_rng(seed)
    F = rng.normal(0, 1, (B, C, N)).astype(np.float32)
    idx = rng.integers(0, M, (B, N)).astype(np.int32)
    for m in empty:
        idx[idx == m] = (m + 1) % M
    return F, idx


def within_contract(got, ref64, ab):
    ulp = np.spacing(np.abs(ref64).astype(np.float32)).astype(np.float64)
    return bool(np.all(np.abs(got.astype(np.float64) - ref64) <= ulp + 1e-10 * ab))


@pytest.mark.parametrize("shape", [(2, 5, 300, 16), (1, 3, 64, 1), (3, 1, 1000, 37)])
def test_pool_oracle_against_reference_lines(shape):
    B, C, N, M = shape
    F, idx = pool_case(1, *shape)
    pooled, scattered, sel, mask = oracle_encoder.cluster_max_pool(F, idx, M, broadcast=True)
    rp, rs = reference_pool(torch.from_numpy(F), torch.from_numpy(idx), torch.from_numpy(sel), M)
    np.testing.assert_array_equal(pooled, rp.numpy())
    np.testing.assert_array_equal(scattered, rs.numpy())
    # fp64 autograd through the same lines against the oracle's gradient
    rng = np.random.default_rng(2)
    gP = rng.normal(0, 1, (B, C, M)).astype(np.float32)
    gS = rng.normal(0, 1, (B, C, N)).astype(np.float32)
    F64 = torch.from_numpy(F).double().requires_grad_(True)
    p64, s64 = reference_pool(F64, torch.from_numpy(idx), torch.from_numpy(sel), M)
    ((p64 * torch.from_numpy(gP).double()).sum() + (s64 * torch.from_numpy(gS).double()).sum()).backward()
    got, ab = oracle_encoder.cluster_max_pool_backward(F, idx, M, gP, gS, with_abs=True)
    assert within_contract(got, F64.grad.numpy(), ab)


def test_pool_adjoint_identity():
    B, C, N, M = 2, 4, 500, 24
    F, idx = pool_case(3, B, C, N, M, empty=(5,))
    rng = np.random.default_rng(4)
    gP = rng.normal(0, 1, (B, C, M)).astype(np.float32)
    gS = rng.normal(0, 1, (B, C, N)).astype(np.float32)
    pooled, scattered, _, _ = oracle_encoder.cluster_max_pool(F, idx, M, broadcast=True)
    gF = oracle_encoder.cluster_max_pool_backward(F, idx, M, gP, gS)
    lhs = (pooled.astype(np.float64) * gP).sum() + (scattered.astype(np.float64) * gS).sum()
    rhs = (F.astype(np.float64) * gF).sum()
    assert abs(lhs - rhs) <= 1e-5 * (np.abs(pooled * gP).sum() + np.abs(scattered * gS).sum())


def test_pool_missing_gradients_are_zero():
    F, idx = pool_case(5, 2, 3, 200, 8)
    rng = np.random.default_rng(6)
    gP = rng.normal(0, 1, (2, 3, 8)).astype(np.float32)
    gS = rng.normal(0, 1, (2, 3, 200)).astype(np.float32)
    both = oracle_encoder.cluster_max_pool_backward(F, idx, 8, gP, gS).astype(np.float64)
    only_p = oracle_encoder.cluster_max_pool_backward(F, idx, 8, gP, None).astype(np.float64)
    only_s = oracle_encoder.cluster_max_pool_backward(F, idx, 8, None, gS).astype(np.float64)
    np.testing.assert_allclose(both, only_p + only_s, rtol=1e-6, atol=1e-6)
    assert np.array_equal(oracle_encoder.cluster_max_pool_backward(F, idx, 8, np.zeros_like(gP), None),
                          np.zeros_like(F))


def test_pool_empty_segments_follow_the_float_multiply():
    """An empty segment keeps index_max's default 0: pooled = features[b, c, 0] * 0.0f, so -0.0 for a negative value
    and NaN for a non-finite one.  All the empty segments' gradients land on point 0, in ascending m."""
    B, C, N, M = 1, 4, 50, 6
    F, idx = pool_case(7, B, C, N, M, empty=(2, 4))
    F[0, 0, 0], F[0, 1, 0], F[0, 2, 0], F[0, 3, 0] = -3.0, np.inf, np.nan, 2.0
    pooled, scattered, sel, mask = oracle_encoder.cluster_max_pool(F, idx, M, broadcast=True)
    assert mask[0, 2] == 0 and mask[0, 4] == 0 and mask[0, [0, 1, 3, 5]].all()
    assert (sel[0, :, 2] == 0).all() and (sel[0, :, 4] == 0).all()
    assert pooled[0, 0, 2] == 0 and np.signbit(pooled[0, 0, 2])
    assert np.isnan(pooled[0, 1, 2]) and np.isnan(pooled[0, 2, 4])
    assert pooled[0, 3, 2] == 0 and not np.signbit(pooled[0, 3, 2])
    gP = np.ones((B, C, M), np.float32)
    gF = oracle_encoder.cluster_max_pool_backward(F, idx, M, gP, None)
    # point 0 collects its own segment's term (if it wins there) plus two zero-masked terms
    own = (sel[0, :, idx[0, 0]] == 0).astype(np.float32)
    np.testing.assert_array_equal(gF[0, :, 0], own)


def test_pool_floor_and_nan_segments():
    """Segments whose values are all <= -1000 or all NaN never get a winner: sel = 0 and their term goes to point 0."""
    B, C, N, M = 1, 2, 40, 4
    F, idx = pool_case(8, B, C, N, M)
    idx[0, 0] = 3
    F[0, 0, idx[0] == 1] = -1000.0
    F[0, 1, idx[0] == 2] = np.nan
    pooled, _, sel, mask = oracle_encoder.cluster_max_pool(F, idx, M)
    assert mask[0].all()
    assert sel[0, 0, 1] == 0 and sel[0, 1, 2] == 0
    assert pooled[0, 0, 1] == F[0, 0, 0] and pooled[0, 1, 2] == F[0, 1, 0]
    gP = np.arange(1, C * M + 1, dtype=np.float32).reshape(B, C, M)
    gF = oracle_encoder.cluster_max_pool_backward(F, idx, M, gP, None)
    assert gF[0, 0, 0] == gP[0, 0, 1] + (gP[0, 0, 3] if sel[0, 0, 3] == 0 else 0)
    assert gF[0, 1, 0] == gP[0, 1, 2] + (gP[0, 1, 3] if sel[0, 1, 3] == 0 else 0)


def test_pool_out_of_range_points():
    B, C, N, M = 2, 3, 100, 5
    F, idx = pool_case(9, B, C, N, M)
    idx[0, 10], idx[1, 20], idx[1, 21] = M, -1, 1 << 30
    F[0, :, 10] = 1e6                                  # would win its segment if it joined one
    pooled, scattered, sel, mask = oracle_encoder.cluster_max_pool(F, idx, M, broadcast=True)
    assert np.isnan(scattered[0, :, 10]).all() and np.isnan(scattered[1, :, 20:22]).all()
    assert not (sel[0] == 10).any()
    gS = np.ones((B, C, N), np.float32)
    gF = oracle_encoder.cluster_max_pool_backward(F, idx, M, None, gS)
    assert (gF[0, :, 10] == 0).all() and (gF[1, :, 20:22] == 0).all()
    # the segments' winners collect one unit per valid member: every channel's total is the valid point count
    n_valid = ((idx >= 0) & (idx < M)).sum(axis=1)
    np.testing.assert_array_equal(gF.sum(axis=2), np.broadcast_to(n_valid[:, None], (B, C)).astype(np.float32))


@pytest.mark.parametrize("shape", [(2, 16, 64, 7, 5), (1, 1, 1, 3, 1), (1, 40, 32, 2, 32)])
def test_knn_oracle_against_reference_lines(shape):
    B, M, N, C, K = shape
    rng = np.random.default_rng(11)
    q = rng.uniform(-20, 20, (B, 3, M)).astype(np.float32)
    db = rng.uniform(-20, 20, (B, 3, N)).astype(np.float32)
    F = rng.normal(0, 1, (B, C, N)).astype(np.float32)
    idx, grouped = oracle_encoder.knn_group(q, db, F, K)
    ri, norm, rg = reference_knn(*(torch.from_numpy(a) for a in (q, db, F)), K)
    # compare rows whose K + 1 smallest norms are distinct (no tie and no two keys rounding to one norm)
    srt = np.sort(norm.numpy(), axis=2)[:, :, :K + 1]
    clean = (np.diff(srt, axis=2) > 0).all(axis=2)
    assert clean.mean() > 0.9
    np.testing.assert_array_equal(idx[clean], ri.numpy()[clean])
    np.testing.assert_array_equal(grouped.transpose(0, 2, 1, 3)[clean], rg.numpy().transpose(0, 2, 1, 3)[clean])
    # fp64 autograd through the reference lines with the oracle's indices
    g = rng.normal(0, 1, (B, 3 + C, M, K)).astype(np.float32)
    F64 = torch.from_numpy(F).double().requires_grad_(True)
    IC = torch.from_numpy(idx).long().unsqueeze(1).expand(B, C, M, K).reshape(B, C, M * K)
    feat = torch.gather(F64, dim=2, index=IC).view(B, C, M, K)
    (feat * torch.from_numpy(g[:, 3:]).double()).sum().backward()
    got, ab = oracle_encoder.knn_group_backward(idx, g, N, with_abs=True)
    assert within_contract(got, F64.grad.numpy(), ab)
    # adjoint identity of the feature rows
    lhs = (grouped[:, 3:].astype(np.float64) * g[:, 3:]).sum()
    assert abs(lhs - (F.astype(np.float64) * got).sum()) <= 1e-5 * np.abs(grouped[:, 3:] * g[:, 3:]).sum()


def test_knn_key_ties_inf_and_nan():
    """Exact ties go to the lower index; +inf keys come after every finite one and NaN keys after +inf."""
    q = np.zeros((1, 3, 1), np.float32)
    db = np.array([[[np.nan, 1.0, -1.0, 3e38, 0.5, 1.0, 2.0, 0.0]], [[0] * 8], [[0] * 8]], np.float32).reshape(1, 3, 8)
    F = np.arange(8, dtype=np.float32).reshape(1, 1, 8)
    idx, grouped = oracle_encoder.knn_group(q, db, F, 8)
    # keys: nan, 1, 1, inf (3e38^2 overflows), 0.25, 1, 4, 0
    assert idx[0, 0].tolist() == [7, 4, 1, 2, 5, 6, 3, 0]
    np.testing.assert_array_equal(grouped[0, 3, 0], F[0, 0, idx[0, 0]])


def _cpu_pool_args():
    return torch.zeros(2, 3, 10), torch.zeros(2, 10, dtype=torch.int32)


@pytest.mark.parametrize("bad, msg", [
    (lambda F, i: (F.double(), i, 4), "features must have dtype"),
    (lambda F, i: (F, i.long(), 4), "min_idx must have dtype"),
    (lambda F, i: (F[0], i, 4), r"features must be \[B,C,N\]"),
    (lambda F, i: (F, i[:, :5], 4), r"features must be \[B,C,N\]"),
    (lambda F, i: (F, i[:1], 4), r"features must be \[B,C,N\]"),
    (lambda F, i: (F[:, :, :0], i[:, :0], 4), "need N >= 1"),
    (lambda F, i: (F, i, 0), "M must be an integer >= 1"),
    (lambda F, i: (F, i, 2.5), "M must be an integer >= 1"),
    (lambda F, i: (F, i, 4), "must be a CUDA tensor"),
    (lambda F, i: (F.numpy(), i, 4), "must be a torch.Tensor"),
])
def test_pool_host_checks(bad, msg):
    F, i = _cpu_pool_args()
    with pytest.raises((RuntimeError, TypeError), match=msg):
        point_ops.cluster_max_pool(*bad(F, i))


def _cpu_knn_args():
    return torch.zeros(2, 3, 6), torch.zeros(2, 3, 40), torch.zeros(2, 5, 40)


@pytest.mark.parametrize("bad, msg", [
    (lambda q, d, f: (q.double(), d, f, 4), "query must have dtype"),
    (lambda q, d, f: (q, d, f.half(), 4), "features must have dtype"),
    (lambda q, d, f: (q[0], d, f, 4), "query must have 3 dimensions"),
    (lambda q, d, f: (q[:, :2], d, f, 4), r"query must be \[B,3,M\]"),
    (lambda q, d, f: (q, d[:1], f, 4), r"query must be \[B,3,M\]"),
    (lambda q, d, f: (q, d, f[:, :, :39], 4), r"query must be \[B,3,M\]"),
    (lambda q, d, f: (q, d, f, 0), "need 1 <= K <= 32"),
    (lambda q, d, f: (q, d, f, 33), "need 1 <= K <= 32"),
    (lambda q, d, f: (q, d[:, :, :3], f[:, :, :3], 4), "need K <= N"),
    (lambda q, d, f: (q, torch.zeros(2, 3, 2049), torch.zeros(2, 5, 2049), 4), "need 1 <= N <= 2048"),
    (lambda q, d, f: (q.requires_grad_(True), d, f, 4), "detach them"),
    (lambda q, d, f: (q, d.requires_grad_(True), f, 4), "detach them"),
    (lambda q, d, f: (q, d, f, 4), "must be a CUDA tensor"),
    (lambda q, d, f: (q, d.numpy(), f, 4), "must be a torch.Tensor"),
])
def test_knn_host_checks(bad, msg):
    q, d, f = _cpu_knn_args()
    with pytest.raises((RuntimeError, TypeError), match=msg):
        point_ops.knn_group(*bad(q, d, f))
