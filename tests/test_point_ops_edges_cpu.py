"""Edge cases of the classifier's point ops without a GPU: cluster_assign (DESIGN.md 4.6), ball_query_xyz (4.5), the
batched farthest-point sampler (4.11) and the decoder interpolation (4.12).

The builders below make adversarial inputs; the references are written from the contracts, not from the oracles:
top-k as a lexicographic sort on (fp32 key, node index), cluster sums as exact rationals, radius hits as an fp32 brute
force with the padding done in Python, farthest points by the line-by-line FarthestSampler, feature gradients by fp64
autograd.  Each test here checks that its cases really land on their edge and that the oracle agrees with the exact
reference; tests/test_point_ops_edges_gpu.py runs the same cases through the kernels."""
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

import oracle
import oracle_assemble as oa
import oracle_interp
from test_assemble_cpu import _RefFarthestSampler
from test_interp_cpu import formulation

F32 = np.float32
NAN_KEY = 0x7f800001                     # every NaN d2 sorts here: after +inf
FIXED_LIMIT = 2.0 ** 39                  # |x| * 2^24 < 2^63


def f32_round(fr):
    """The rational fr rounded once to float32 (nearest, ties to even)."""
    fr = Fraction(fr)
    if fr == 0:
        return F32(0)
    a = abs(fr)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if a < Fraction(2) ** e:
        e -= 1                                                  # now 2^e <= a < 2^(e + 1)
    s = max(e - 23, -149)
    with np.errstate(over="ignore"):
        return F32(math.copysign(math.ldexp(round(a / Fraction(2) ** s), s), fr))


def d2_f32(p, q):
    """fp32 ((dx*dx + dy*dy) + dz*dz) with d = p - q, one rounding per operation; p [3,N,1] / q [3,1,M] broadcast."""
    with np.errstate(over="ignore", invalid="ignore"):
        d = p.astype(F32) - q.astype(F32)
        return (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]


# ---- cluster_assign -------------------------------------------------------------------------------------------------

def exact_topk(pts, nodes, k):
    """[B,N,k]: the k smallest (key, node index) pairs in lexicographic order, key = the bits of the fp32 d2 (>= +0,
    so the bit order is the value order) with every NaN placed after +inf."""
    B, _, N = pts.shape
    M = nodes.shape[2]
    out = np.empty((B, N, k), np.int64)
    for b in range(B):
        d2 = d2_f32(pts[b][:, :, None], nodes[b][:, None, :])
        key = np.where(np.isnan(d2), np.uint32(NAN_KEY), d2.view(np.uint32)).astype(np.uint64)
        out[b] = (np.sort((key << np.uint64(32)) | np.arange(M, dtype=np.uint64), axis=1)[:, :k]
                  & np.uint64(0xffffffff)).astype(np.int64)
    return out


def _ulp_steps():
    """Nodes on the x axis at 32 consecutive floats from 1.5 and their mirror images (shuffled): fl(x * x) moves by
    one or two ulps between neighbours, and +x / -x tie exactly."""
    rng = np.random.default_rng(1)
    xs = [F32(1.5)]
    for _ in range(31):
        xs.append(np.nextafter(xs[-1], F32(2)))
    xs = np.array(xs, F32)
    nodes = np.zeros((1, 3, 64), F32)
    nodes[0, 0] = np.concatenate([xs, -xs])[rng.permutation(64)]
    pts = np.zeros((1, 3, 4), F32)
    pts[0, 1, 1] = 2.0 ** -12
    pts[0, 2, 2] = 1e-3
    pts[0, 0, 3] = 2.0 ** -30
    return pts, nodes


def _half_lattice(seed, k):
    """Integer points and half-integer nodes: every point has its 8 cube corners at d2 = 0.75 exactly."""
    rng = np.random.default_rng(seed)
    g = np.arange(-2, 3, dtype=F32)
    pts = np.stack(np.meshgrid(g, g, g, indexing="ij")).reshape(1, 3, -1)
    h = np.arange(-2.5, 3.0, dtype=F32)
    nodes = np.stack(np.meshgrid(h, h, h, indexing="ij")).reshape(3, -1)
    return pts, nodes[:, rng.permutation(nodes.shape[1])][None], k


def topk_cases():
    """(name, pts [B,3,N], nodes [B,3,M], k)."""
    rng = np.random.default_rng(2)
    cases = [("ulp_steps", *_ulp_steps(), 8)]
    cases += [(f"ties_k{k}", *_half_lattice(k, k)) for k in range(1, 9)]
    nodes = rng.integers(-6, 7, (1, 3, 2048)).astype(F32)
    pts = (rng.integers(-14, 15, (1, 3, 4096)) * 0.5).astype(F32)
    cases.append(("M2048", pts, nodes, 8))
    for M in (1, 3, 8):
        cases.append((f"k_eq_M{M}", rng.integers(-2, 3, (2, 3, 600)).astype(F32),
                      rng.integers(-1, 2, (2, 3, M)).astype(F32), M))
    base = rng.integers(-3, 4, (3, 40)).astype(F32)
    nodes = np.repeat(base, 3, axis=1)[:, rng.permutation(120)][None]
    cases.append(("duplicate_nodes", rng.integers(-4, 5, (1, 3, 700)).astype(F32), nodes, 8))
    # fewer than k ordered keys: two finite nodes, five whose d2 overflows to +inf, five with a NaN coordinate
    nodes = np.zeros((1, 3, 12), F32)
    nodes[0, :, [0, 3, 4, 7, 10]] = F32(4e19)
    nodes[0, 1, [1, 2, 6, 8, 11]] = np.nan
    nodes[0, :, 5] = [1, 0, 0]
    nodes[0, :, 9] = [-1, 0, 0]
    pts = np.array([[[0.25, -0.5, 0.0, np.nan, 1e30, 4e19]], [[0, 0, 0, 0, 0, 4e19]], [[0, 0, 0, 0, 0, 4e19]]],
                   F32).reshape(1, 3, 6)
    cases.append(("inf_and_nan_keys", pts, nodes, 8))
    return cases


SUM_MAGNITUDES = [1e-6, 0.3, 0.5, 40.0, 1e4, 2.0 ** 38, 2.0 ** 39 - 2.0 ** 15, 2.0 ** 39, 1e12, 1e20, 1e30, 3.4e38]


def sum_case():
    """One batch item per magnitude v: nodes at the origin and +-(v, v, v); 32 points around each, near +-v at a few
    ulps from v (both signs), near the origin at +-v / 1000."""
    rng = np.random.default_rng(3)
    B, N = len(SUM_MAGNITUDES), 96
    pts = np.zeros((B, 3, N), F32)
    nodes = np.zeros((B, 3, 3), F32)
    for b, v in enumerate(SUM_MAGNITUDES):
        v = F32(v)
        nodes[b, :, 1], nodes[b, :, 2] = v, -v
        bits = rng.integers(-40, 41, (3, 32)) + v.view(np.int32)
        near = bits.astype(np.int32).view(F32)
        pts[b, :, :32] = near
        pts[b, :, 32:64] = -near
        pts[b, :, 64:] = (rng.choice([-1, 1], (3, 32)) * rng.uniform(0.5, 1.5, (3, 32)) * (v / F32(1000))).astype(F32)
    return pts, nodes


def exact_sums(pts, min_idx, M):
    """Per (b, axis, node): count of summed points, the exact sum and the sum of the 2^-24-grid images (Fractions).
    A point is summed when every coordinate has magnitude < 2^39 (which also leaves out inf and NaN)."""
    B, _, N = pts.shape
    cnt = np.zeros((B, M), np.int64)
    exact = [[[Fraction(0)] * M for _ in range(3)] for _ in range(B)]
    grid = [[[Fraction(0)] * M for _ in range(3)] for _ in range(B)]
    for b in range(B):
        for n in range(N):
            p = pts[b, :, n]
            if not all(abs(float(x)) < FIXED_LIMIT for x in p):
                continue
            m = int(min_idx[b, n])
            cnt[b, m] += 1
            for a in range(3):
                x = Fraction(float(p[a]))
                exact[b][a][m] += x
                grid[b][a][m] += Fraction(round(x * 2 ** 24), 2 ** 24)   # Fraction rounds half to even
    return cnt, exact, grid


def mean_from_grid(cnt, grid):
    B, M = cnt.shape
    out = np.zeros((B, 3, M), F32)
    for b in range(B):
        for a in range(3):
            for m in range(M):
                out[b, a, m] = f32_round(grid[b][a][m]) / (F32(cnt[b, m]) + F32(1e-5))
    return out


# ---- ball_query_xyz -------------------------------------------------------------------------------------------------

def exact_ball(points, nodes, radius, K):
    """fp32 brute force: hit <=> d2 <= fl(r * r) (NaN never hits); the first K hits in ascending n, padded in Python
    by repeating them cyclically; no hit -> zeros."""
    B, _, N = points.shape
    M = nodes.shape[2]
    r2 = F32(radius) * F32(radius)
    out = np.zeros((B, M, K), np.int32)
    for b in range(B):
        d2 = d2_f32(points[b][:, None, :], nodes[b][:, :, None])          # [M, N]
        for m in range(M):
            hits = [int(n) for n in np.flatnonzero(d2[m] <= r2)][:K]
            if hits:
                out[b, m] = [hits[i % len(hits)] for i in range(K)]
    return out


def grid_cells(points, radius):
    """The cell of every point in the search grid (DESIGN.md 4.5: cell = (extent / dim) * 1.0001, dim = floor(extent /
    radius) clamped to [1, 16]); used only to show that a case straddles cell boundaries."""
    r = F32(radius)
    cells = []
    for c in range(3):
        v = points[c][np.isfinite(points[c])]
        lo, hi = v.min(), v.max()
        ext = F32(max(hi - lo, F32(0)))
        dim = int(np.floor(ext / r)) if r > 0 and ext > 0 else 1
        dim = min(max(dim, 1), 16)
        cell = (ext / F32(dim)) * F32(1.0001) if ext > 0 else F32(1)
        inv = F32(1) / cell
        cells.append(np.clip(np.floor((points[c] - lo) * inv), 0, dim - 1))
    return np.stack(cells)


def sphere_points(nodes, radius, rng):
    """For each node (positive coordinates), points at fp32 d2 = r2 - 1 ulp, r2 and r2 + 1 ulp: start on the sphere
    in a direction with a small x component and step x one ulp at a time (each step moves d2 by under one ulp)."""
    r2 = F32(radius) * F32(radius)
    targets = [np.nextafter(r2, F32(0)), r2, np.nextafter(r2, F32(np.inf))]
    out = []
    for n in nodes.T:
        u = rng.normal(size=3)
        u[0] = 0.05 * math.copysign(1.0, u[0])
        u[1:] *= math.sqrt(1 - u[0] ** 2) / np.linalg.norm(u[1:])
        p0 = (n.astype(np.float64) + radius * u).astype(F32)
        xs = (p0[0].view(np.int32) + np.arange(-600, 601)).astype(np.int32).view(F32)
        d2 = d2_f32(np.stack([xs, np.full_like(xs, p0[1]), np.full_like(xs, p0[2])])[:, :, None], n[:, None, None])[:, 0]
        for t in targets:
            j = np.flatnonzero(d2 == t)
            if len(j):
                out.append([xs[j[0]], p0[1], p0[2]])
    return np.array(out, F32).T


def ball_cases():
    """(name, points [B,3,N], nodes [B,3,M], radius, K)."""
    rng = np.random.default_rng(4)
    cases = []

    def cloud(ext, n, m, r, B=1):
        """n points in all: the sphere points of m nodes, the rest uniform in the cube [0, ext]^3."""
        pts, nds = [], []
        for _ in range(B):
            nd = rng.uniform(0.1 * ext, 0.9 * ext, (3, m)).astype(F32)
            sp = sphere_points(nd, r, rng)
            p = np.concatenate([rng.uniform(0, ext, (3, n - sp.shape[1])).astype(F32), sp], axis=1)
            pts.append(p[:, rng.permutation(p.shape[1])])
            nds.append(nd)
        return np.stack(pts), np.stack(nds)

    cases.append(("sphere_ties_across_cells", *cloud(8.0, 3000, 48, 1.0), 1.0, 16))
    # extent / radius one ulp below, at and one ulp above an integer, one batch item each
    r = F32(0.55)                   # fl(e / r) moves by under one ulp of 7 per ulp of e: every quotient is reachable
    items_p, items_n = [], []
    for q, step in ((7, -1), (7, 0), (7, 1)):
        want = np.nextafter(F32(q), F32(q + step)) if step else F32(q)
        e = F32(q) * r
        for _ in range(64):
            if e / r == want:
                break
            e = np.nextafter(e, F32(np.inf) if e / r < want else F32(0))
        p, nd = cloud(float(e), 1500, 24, float(r))
        p[0, :, :2] = np.array([[0, 0, 0], [e, e, e]], F32).T
        p = np.clip(p, 0, e)
        items_p.append(p[0])
        items_n.append(nd[0])
    cases.append(("extent_over_radius_at_integer", np.stack(items_p), np.stack(items_n), float(r), 32))
    cases.append(("cell_cap_16", *cloud(100.0, 20000, 64, 0.5), 0.5, 8))
    dup = np.repeat(rng.integers(0, 6, (3, 300)).astype(F32), 3, axis=1)[:, rng.permutation(900)]
    nd = np.concatenate([dup[:, :20], np.nextafter(dup[:, 20:21], F32(10))], axis=1)
    cases.append(("radius_zero_duplicates", dup[None], nd[None], 0.0, 4))
    p = rng.uniform(0, 10, (3, 2000)).astype(F32)
    p[:, :6] = [[0, 10, 3, 3, 0, 10], [5, 5, 0, 10, 0, 10], [5, 5, 5, 5, 0, 10]]
    nd = p[:, :6].copy()
    nd[0, 0] -= 0.5; nd[0, 1] += 0.5; nd[1, 2] -= 0.9; nd[1, 3] += 0.9; nd[:, 4] -= 0.3; nd[:, 5] += 0.3
    cases.append(("nodes_outside_box", p[None], nd[None], 1.0, 8))
    p = rng.uniform(0, 5, (3, 1000)).astype(F32)
    p[0, 10], p[1, 11], p[2, 12], p[0, 13], p[1, 14] = np.nan, np.inf, -np.inf, np.inf, np.nan
    nd = p[:, 8:20].copy()
    nd[0, 2:6] = p[0, 8:12] + F32(0.1)
    nd = np.nan_to_num(nd, nan=2.5, posinf=2.5, neginf=2.5)
    cases.append(("non_finite_points", p[None], nd[None], 1.0, 8))
    p = np.full((3, 4096), 50.0, F32) + rng.uniform(0, 5, (3, 4096)).astype(F32)
    runs = np.r_[28:41, 1016:1041, 2040:2101, 4090:4096]
    p[:, runs] = rng.uniform(-0.5, 0.5, (3, len(runs))).astype(F32)
    nd = np.zeros((3, 3), F32)
    nd[:, 1] = [0.4, 0.4, 0.4]                                    # hits only a few of the run points
    nd[:, 2] = [52, 52, 52]
    cases.append(("hits_across_bitmap_words", p[None], nd[None], 1.0, 50))
    cases.append(("N65536", *cloud(20.0, 65536, 64, 1.5), 1.5, 32))
    return cases


# ---- farthest-point sampling ----------------------------------------------------------------------------------------

def fps_cloud(kind, n, seed):
    """[3, n] float64 (exact in float32): duplicated points (each 4 times) or a shuffled integer lattice."""
    rng = np.random.default_rng(seed)
    if kind == "dup":
        base = rng.normal(0, 10, (3, (n + 3) // 4)).astype(F32).astype(np.float64)
        pts = np.repeat(base, 4, axis=1)[:, :n]
    else:
        g = int(math.ceil(n ** (1 / 3)))
        a = np.arange(g, dtype=np.float64)
        pts = np.stack(np.meshgrid(a, a, a, indexing="ij")).reshape(3, -1)[:, :n]
    return pts[:, rng.permutation(n)]


def ref_sampler(pts, k, start):
    """The line-by-line FarthestSampler started at `start` (its own start is np.random.randint(3))."""
    seed = next(s for s in range(100) if (np.random.seed(s), np.random.randint(3))[1] == start)
    np.random.seed(seed)
    return _RefFarthestSampler(3).sample(pts, k)[1]


FPS_SIZES = [8192, 8193, 16385, 65536]


# ---- interpolation --------------------------------------------------------------------------------------------------

def interp_case(seed, B, Nq, M, C, k, lo, hi):
    """Indices drawn from nodes [lo, hi): distinct per row where hi - lo >= k; rows 3 (all k equal), 5 (one pair
    equal) and 9 (all equal and the query on that node: S = 0) in the first 32-point tile among distinct rows."""
    rng = np.random.default_rng(seed)
    q = rng.uniform(-10, 10, (B, 3, Nq)).astype(F32)
    nd = rng.uniform(-10, 10, (B, 3, M)).astype(F32)
    F = rng.normal(0, 1, (B, C, M)).astype(F32)
    if hi - lo >= k:
        idx = np.stack([np.stack([rng.choice(np.arange(lo, hi), k, replace=False) for _ in range(Nq)])
                        for _ in range(B)])
    else:
        idx = rng.integers(lo, hi, (B, Nq, k))
    idx[:, 3, :] = idx[:, 3, :1]
    if k > 1:
        idx[:, 5, 1] = idx[:, 5, 0]
    idx[:, 9, :] = idx[:, 9, :1]
    for b in range(B):
        q[b, :, 9] = nd[b, :, idx[b, 9, 0]]
    return idx.astype(np.int64), q, nd, F


INTERP_CASES = [  # (B, Nq, M, C, k, lo, hi)
    (2, 200, 10, 40, 3, 0, 10),
    (1, 100, 20, 33, 8, 0, 20),
    (2, 64, 10, 5, 1, 0, 10),
    (1, 300, 129, 48, 3, 0, 128),           # every index in the first node range of the backward
    (1, 300, 129, 48, 3, 128, 129),         # ... in the last one, which holds one node
    (1, 500, 2048, 40, 4, 0, 128),
    (1, 500, 2048, 40, 4, 1920, 2048),
]


def autograd_fp64(idx, q, nd, F, g):
    Ft = torch.from_numpy(F).double().requires_grad_(True)
    formulation(torch.from_numpy(idx), torch.from_numpy(q).double(), torch.from_numpy(nd).double(), Ft).backward(
        torch.from_numpy(g).double())
    return Ft.grad.numpy()


# ---- tests ----------------------------------------------------------------------------------------------------------

def test_topk_cases_land_on_their_edges():
    cases = {c[0]: c[1:] for c in topk_cases()}
    pts, nodes, _ = cases["ulp_steps"]
    d2 = np.sort(d2_f32(pts[0][:, :1, None], nodes[0][:, None, :])[0])
    steps = (d2[1:].view(np.int32) - d2[:-1].view(np.int32))
    assert (steps == 0).sum() >= 31 and (steps == 1).any() and (steps == 2).any()
    for k in range(1, 9):
        pts, nodes, _ = cases[f"ties_k{k}"]
        d2 = np.sort(d2_f32(pts[0][:, :, None], nodes[0][:, None, :]), axis=1)
        assert (d2[:, :8] == F32(0.75)).all() and (d2[:, 8] > F32(0.75)).all()
    assert cases["M2048"][1].shape[2] == 2048
    pts, nodes, _ = cases["inf_and_nan_keys"]
    d2 = d2_f32(pts[0][:, :, None], nodes[0][:, None, :])
    assert np.isfinite(d2[0]).sum() == 2 and np.isinf(d2[0]).sum() == 5 and np.isnan(d2[0]).sum() == 5
    assert np.isnan(d2[3]).all() and not np.isfinite(d2[4]).any()


@pytest.mark.parametrize("case", topk_cases(), ids=lambda c: c[0])
def test_cluster_topk_oracle_matches_lexsort(case):
    _, pts, nodes, k = case
    got = oracle.cluster_assign(pts, nodes, k)
    want = exact_topk(pts, nodes, k)
    np.testing.assert_array_equal(got["min_k_idx"], want)
    assert all(len(set(row)) == k for row in want.reshape(-1, k))           # k distinct nodes, whatever the keys


def test_sum_case_lands_on_its_edges():
    pts, nodes = sum_case()
    min_idx = exact_topk(pts, nodes, 1)[:, :, 0]
    cnt, exact, grid = exact_sums(pts, min_idx, 3)
    for b, v in enumerate(SUM_MAGNITUDES):
        summed = (np.abs(pts[b]) < FIXED_LIMIT).all(axis=0)
        assert cnt[b].sum() == summed.sum()
        if v <= 2.0 ** 38:
            assert cnt[b, 1] == 32 and cnt[b, 2] == 32, v               # +-v points reach their own node
        elif v > FIXED_LIMIT:
            assert cnt[b, 1] == 0 and cnt[b, 2] == 0, v
        on_grid = all(Fraction(float(x)) * 2 ** 24 == round(Fraction(float(x)) * 2 ** 24) for x in pts[b].ravel()
                      if abs(float(x)) < FIXED_LIMIT)
        assert on_grid == (v >= 0.5 * 1000), v                          # the origin's points are v / 1000
    b38 = SUM_MAGNITUDES.index(2.0 ** 38)
    assert abs(grid[b38][0][1]) * 2 ** 24 >= 2 ** 63                    # an int64 sum would wrap
    bmax = SUM_MAGNITUDES.index(2.0 ** 39 - 2.0 ** 15)
    assert 0 < cnt[bmax, 1] < 32                                        # the limit splits this node's points


def test_cluster_sums_oracle_matches_exact_rationals():
    pts, nodes = sum_case()
    got = oracle.cluster_assign(pts, nodes, 1)
    min_idx = exact_topk(pts, nodes, 1)[:, :, 0]
    np.testing.assert_array_equal(got["min_idx"], min_idx)
    cnt, exact, grid = exact_sums(pts, min_idx, 3)
    np.testing.assert_array_equal(got["count"], cnt)
    np.testing.assert_array_equal(got["cluster_mean"], mean_from_grid(cnt, grid))
    for b in range(len(SUM_MAGNITUDES)):
        for a in range(3):
            for m in range(3):
                assert abs(grid[b][a][m] - exact[b][a][m]) <= Fraction(int(cnt[b, m]), 2 ** 25)
                if SUM_MAGNITUDES[b] >= 500 and m:
                    assert grid[b][a][m] == exact[b][a][m]              # multiples of 2^-24: exact


def test_old_fixed_point_cast_got_the_sign_wrong_at_1e12():
    """The earlier oracle cast rint(x * 2^24) to int64 without a range check: at x = 1e12 numpy's x86-64 cast gives
    INT64_MIN, a mean of -5.5e11 for a point at +1e12.  Such a point now joins no count or sum."""
    x = np.float64(F32(1e12))
    with np.errstate(invalid="ignore"):
        old_fixed = np.rint(np.array([x]) * 16777216.0).astype(np.int64)[0]
    assert old_fixed != round(Fraction(x) * 2 ** 24)
    old_mean = F32(old_fixed * (1.0 / 16777216.0)) / (F32(1) + F32(1e-5))
    assert old_mean < 0 or old_fixed == np.iinfo(np.int64).max           # wrapped (x86-64) or saturated
    pts = np.array([[[1e12], [0.0], [0.0]]], F32)
    nodes = np.array([[[1e12, 0.0], [0.0, 0.0], [0.0, 0.0]]], F32)
    out = oracle.cluster_assign(pts, nodes, 1)
    assert out["min_idx"][0, 0] == 0 and out["count"][0, 0] == 0 and (out["cluster_mean"] == 0).all()


def test_int_to_f32_rounds_once():
    for v in (0, 1, -1, 2 ** 53 + 1, 2 ** 60 + 2 ** 36, 2 ** 60 + 2 ** 36 + 1, -(2 ** 94) - 3, 2 ** 77 - 1):
        assert oracle.int_to_f32(v) == f32_round(v), v


@pytest.mark.parametrize("case", ball_cases(), ids=lambda c: c[0])
def test_ball_oracle_matches_brute_force(case):
    _, pts, nodes, radius, K = case
    np.testing.assert_array_equal(oracle.ball_query_xyz(pts, nodes, radius, K), exact_ball(pts, nodes, radius, K))


def test_ball_cases_land_on_their_edges():
    cases = {c[0]: c[1:] for c in ball_cases()}
    pts, nodes, r, _ = cases["sphere_ties_across_cells"]
    r2 = F32(r) * F32(r)
    d2 = d2_f32(pts[0][:, None, :], nodes[0][:, :, None])
    cp, cn = grid_cells(pts[0], r), grid_cells(nodes[0], r)    # nodes inside the box: the same cells as points
    cross = (cp[:, None, :] != cn[:, :, None]).any(axis=0)
    for t in (np.nextafter(r2, F32(0)), r2, np.nextafter(r2, F32(np.inf))):
        assert ((d2 == t) & cross).sum() >= 20, t
    pts, nodes, r, _ = cases["extent_over_radius_at_integer"]
    quot = [F32(pts[b, 0].max() - pts[b, 0].min()) / F32(r) for b in range(3)]
    assert quot == [np.nextafter(F32(7), F32(0)), F32(7), np.nextafter(F32(7), F32(8))]
    pts, _, r, _ = cases["cell_cap_16"]
    assert np.floor(F32(np.ptp(pts[0, 0])) / F32(r)) > 16
    pts, nodes, r, _ = cases["radius_zero_duplicates"]
    assert r == 0 and (exact_ball(pts, nodes, r, 4)[0, :20] != exact_ball(pts, nodes, r, 1)[0, :20, :1]).any()
    pts, nodes, r, K = cases["nodes_outside_box"]
    outside = ((nodes[0] < pts[0].min(axis=1, keepdims=True)) | (nodes[0] > pts[0].max(axis=1, keepdims=True))).any(0)
    assert outside.all() and (d2_f32(pts[0][:, None, :], nodes[0][:, :, None]).min(axis=1) <= 1).all()
    pts, _, _, _ = cases["non_finite_points"]
    assert np.isnan(pts).any() and np.isposinf(pts).any() and np.isneginf(pts).any()
    pts, nodes, r, K = cases["hits_across_bitmap_words"]
    hits = np.flatnonzero(d2_f32(pts[0][:, None, :], nodes[0][:, :1, None])[0] <= F32(r) * F32(r))
    assert len(hits) > K and len(set(hits[:K] // 32)) > 2 and hits[K - 1] // 32 == hits[K] // 32
    assert cases["N65536"][0].shape[2] == 65536


@pytest.mark.parametrize("n", FPS_SIZES)
@pytest.mark.parametrize("kind", ["dup", "lattice"])
def test_fps_oracle_matches_reference_sampler(kind, n):
    pts = fps_cloud(kind, n, n)
    for start in (0, 2):
        np.testing.assert_array_equal(oa.fps(pts, 48, start)[0], ref_sampler(pts, 48, start))
    # ties really are settled: some step has several points at the winning distance
    P, idx = pts, oa.fps(pts, 48, 0)[0]
    dmin = np.full(n, np.inf)
    tied = 0
    for i in idx[:-1]:
        dmin = np.minimum(dmin, ((P - P[:, i:i + 1]) ** 2).sum(axis=0))
        tied += (dmin == dmin.max()).sum() > 1
    assert tied >= 5


def test_fps_oracle_takes_more_nodes_than_points():
    pts = fps_cloud("lattice", 100, 1)
    idx, _ = oa.fps(pts, 130, 7)
    assert sorted(set(idx[:100].tolist())) == list(range(100)) and (idx[100:] == 0).all()
    np.testing.assert_array_equal(oa.fps(pts, 130, 2)[0], ref_sampler(pts, 130, 2))


@pytest.mark.parametrize("case", INTERP_CASES)
def test_interp_cases_and_oracle_against_fp64_autograd(case):
    B, Nq, M, C, k, lo, hi = case
    idx, q, nd, F = interp_case(sum(case), B, Nq, M, C, k, lo, hi)
    assert ((idx >= lo) & (idx < hi)).all()
    rows = [len(set(r)) for r in idx[0, :32]]
    if k > 1:
        assert rows[3] == 1 and rows[5] < k and rows.count(k) >= 20 or hi - lo < k
    w, valid = oracle_interp.interp_weights(idx, q, nd)
    assert valid.all() and np.isnan(w[:, 9]).all()                                   # S = 0
    if k == 1:
        assert (w[:, [i for i in range(Nq) if i != 9]] == 0).all()
    g = np.random.default_rng(1).normal(0, 1, (B, C, Nq)).astype(F32)
    got = oracle_interp.interp_backward(idx, q, nd, g, M)
    ref = autograd_fp64(idx, q, nd, F, g)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    fin = np.isfinite(ref)
    assert fin.any()
    np.testing.assert_allclose(got[fin], ref[fin], rtol=1e-5, atol=1e-5 * k)
