"""The point ops' kernels on the edge cases of tests/test_point_ops_edges_cpu.py: bit-exact against their oracles and
against the exact references built from the contracts (DESIGN.md 4.5, 4.6, 4.11, 4.12)."""
from fractions import Fraction

import numpy as np
import pytest
import torch

import oracle
import oracle_assemble as oa
import oracle_interp
from deepi2p_b200 import _native, assemble, point_ops
from test_interp_gpu import contract_ok
from test_point_ops_edges_cpu import (FPS_SIZES, INTERP_CASES, SUM_MAGNITUDES, autograd_fp64, ball_cases, exact_ball,
                                      exact_sums, exact_topk, fps_cloud, interp_case, mean_from_grid, ref_sampler,
                                      sum_case, topk_cases)

pytestmark = pytest.mark.gpu


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _cluster(pts, nodes, k):
    got = point_ops.cluster_assign_forward(_dev(pts), _dev(nodes), k)
    got = {name: t.cpu().numpy() for name, t in got.items()}
    want = oracle.cluster_assign(pts, nodes, k)
    for name in want:
        np.testing.assert_array_equal(got[name], want[name], err_msg=name)
    return got


@pytest.mark.parametrize("case", topk_cases(), ids=lambda c: c[0])
def test_cluster_topk_against_lexsort(cuda, case):
    _, pts, nodes, k = case
    got = _cluster(pts, nodes, k)
    np.testing.assert_array_equal(got["min_k_idx"], exact_topk(pts, nodes, k))


def test_cluster_sums_against_exact_rationals(cuda):
    """Every magnitude from 1e-6 to 3.4e38 at both signs: count and mean follow the exact sums of the points below
    2^39 rounded to the 2^-24 grid (no error at all for multiples of 2^-24), within 2^-25 per point of the exact sum;
    an int64 sum of the 2^38 points would wrap, the two-word one does not.  Bit-identical on a repeat."""
    pts, nodes = sum_case()
    got = _cluster(pts, nodes, 1)
    min_idx = exact_topk(pts, nodes, 1)[:, :, 0]
    np.testing.assert_array_equal(got["min_idx"], min_idx)
    cnt, exact, grid = exact_sums(pts, min_idx, 3)
    np.testing.assert_array_equal(got["count"], cnt)
    np.testing.assert_array_equal(got["cluster_mean"], mean_from_grid(cnt, grid))
    for b in range(len(SUM_MAGNITUDES)):
        for a in range(3):
            for m in range(3):
                assert abs(grid[b][a][m] - exact[b][a][m]) <= Fraction(int(cnt[b, m]), 2 ** 25)
    again = point_ops.cluster_assign_forward(_dev(pts), _dev(nodes), 1)
    np.testing.assert_array_equal(again["cluster_mean"].cpu().numpy(), got["cluster_mean"])


def test_cluster_sums_many_points_per_ctas(cuda):
    """20,000 points of magnitude ~2^38.9 in one node spread over 79 CTAs: the CTA partials and their global sum both
    carry into the high word."""
    rng = np.random.default_rng(8)
    v = np.float32(2.0 ** 38.9)
    pts = (v * rng.uniform(0.99, 1.0, (1, 3, 20000))).astype(np.float32)
    pts[0, :, ::7] *= -1
    nodes = np.array([[[0.0, 1.0]] * 3], np.float32).reshape(1, 3, 2) * v
    got = _cluster(pts, nodes, 1)
    cnt, exact, grid = exact_sums(pts, got["min_idx"], 2)
    np.testing.assert_array_equal(got["count"], cnt)
    np.testing.assert_array_equal(got["cluster_mean"], mean_from_grid(cnt, grid))


@pytest.mark.parametrize("case", ball_cases(), ids=lambda c: c[0])
def test_ball_query_xyz_against_brute_force(cuda, case):
    _, pts, nodes, radius, K = case
    got = point_ops.ball_query_xyz_forward(_dev(pts), _dev(nodes), radius, K).cpu().numpy()
    np.testing.assert_array_equal(got, exact_ball(pts, nodes, radius, K))
    np.testing.assert_array_equal(got, oracle.ball_query_xyz(pts, nodes, radius, K))


def _fps_abi(x, n_pts, k, start):
    """fps_batch through the C ABI (the Python wrapper rejects k > n_pts)."""
    x = x.contiguous()
    S, _, n = x.shape
    idx = torch.empty((S, k), dtype=torch.int32, device="cuda")
    nodes = torch.empty((S, 3, k), dtype=x.dtype, device="cuda")
    lib = _native.load()
    fn = lib.fps_batch_f32 if x.dtype == torch.float32 else lib.fps_batch_f64
    rc = fn(x.data_ptr(), n_pts.data_ptr(), n, S, k, start.data_ptr(), idx.data_ptr(), nodes.data_ptr(),
            torch.cuda.current_stream().cuda_stream)
    _native.check(rc, "fps_batch")
    return idx.cpu().numpy(), nodes.cpu().numpy()


@pytest.mark.parametrize("n", FPS_SIZES)
@pytest.mark.parametrize("kind", ["dup", "lattice"])
def test_fps_cluster_ties(cuda, kind, n):
    """Ties settled across the CTAs of a cluster (and on one CTA at 8192), from set 0's start 0 and set 1's start in a
    later slice."""
    pts = np.stack([fps_cloud(kind, n, n), fps_cloud(kind, n, n + 1)])
    start = [0, min(n - 1, 8192 + 77)]
    for dt in (np.float32, np.float64):
        x = _dev(pts.astype(dt))
        idx, nodes = assemble.farthest_point_sample(x, None, 64, start=torch.tensor(start, dtype=torch.int32,
                                                                                    device="cuda"))
        for s in range(2):
            ri, rn = oa.fps(pts[s].astype(dt), 64, start[s])
            np.testing.assert_array_equal(idx[s].cpu().numpy(), ri, err_msg=f"{dt} {s}")
            np.testing.assert_array_equal(nodes[s].cpu().numpy(), rn, err_msg=f"{dt} {s}")
        np.testing.assert_array_equal(idx[0].cpu().numpy(), ref_sampler(pts[0], 64, 0))


def test_fps_empty_slices_and_more_nodes_than_points(cuda):
    """n_stride 65,536 (8 CTAs) with 1, 100 and 8193 points: whole slices are empty; k = 150 exceeds two of the
    counts, so the sampler must keep returning index 0 once every point is taken."""
    pts = np.stack([fps_cloud("lattice", 65536, 5 + s) for s in range(3)])
    counts = [1, 100, 8193]
    start = [0, 99, 8192]
    for dt in (np.float32, np.float64):
        x = _dev(pts.astype(dt))
        n_pts = torch.tensor(counts, dtype=torch.int32, device="cuda")
        st = torch.tensor(start, dtype=torch.int32, device="cuda")
        idx, nodes = _fps_abi(x, n_pts, 150, st)
        for s, m in enumerate(counts):
            ri, rn = oa.fps(pts[s, :, :m].astype(dt), 150, start[s])
            np.testing.assert_array_equal(idx[s], ri, err_msg=f"{dt} {s}")
            np.testing.assert_array_equal(nodes[s], rn, err_msg=f"{dt} {s}")
        assert (idx[0] == 0).all() and (idx[1, 100:] == 0).all()
        got, _ = assemble.farthest_point_sample(x, n_pts, 1, start=st)
        np.testing.assert_array_equal(got.cpu().numpy()[:, 0], start)


@pytest.mark.parametrize("case", INTERP_CASES)
def test_interp_repeated_indices_and_quirks(cuda, case):
    B, Nq, M, C, k, lo, hi = case
    idx, q, nd, F = interp_case(sum(case), B, Nq, M, C, k, lo, hi)
    g = np.random.default_rng(1).normal(0, 1, (B, C, Nq)).astype(np.float32)
    for dt in (torch.int32, torch.int64):
        Fr = _dev(F).requires_grad_(True)
        out = point_ops.upsample_by_interpolation(_dev(idx).to(dt), _dev(q), _dev(nd), Fr)
        np.testing.assert_array_equal(out.detach().cpu().numpy(), oracle_interp.interp_forward(idx, q, nd, F))
        out.backward(_dev(g))
        got = Fr.grad.cpu().numpy()
        ref, ab = oracle_interp.interp_backward(idx, q, nd, g, M, with_abs=True)
        assert contract_ok(got, ref, ab)
        np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
        auto = autograd_fp64(idx, q, nd, F, g)
        np.testing.assert_array_equal(np.isnan(got), np.isnan(auto))
        fin = np.isfinite(auto)
        np.testing.assert_allclose(got[fin], auto[fin], rtol=1e-5, atol=1e-5 * k)
