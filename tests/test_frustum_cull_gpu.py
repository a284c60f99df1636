"""The solver's fp32 frustum cull at rounding-level distances from the image and depth boundaries (GPU half).

The adversarial clouds of test_frustum_cull_cpu.py (points 1e-9 .. 1e-1 px / m from the five planes the cull tests,
ulp-neighbour groups, straddling and mixed-label groups) go through every pass that culls -- frustum_evaluate, the
solver's first traced pass, the cost-only pass of an infeasible start (lm_begin -> phase 3 -> one eval_slice pass,
the same culled code path as every other pass), a (label, Morton)-sorted copy, and the disabled-cull fallback -- and
must give the sums of oracle.evaluate at the same x to the tolerances of test_evaluate_matches_oracle.  The CPU half
shows that each active point moves a sum by >= 100x those tolerances, so a point the cull drops by mistake fails
here.
"""
import numpy as np
import pytest
import torch

import oracle
from deepi2p_b200 import frustum
from test_frustum_cull_cpu import CONFIGS, OVERFLOW_CONFIGS, POSES, boundary_cloud, config_id, oracle_noise

pytestmark = pytest.mark.gpu

WIDE = ((-1e3,) * 3, (1e3,) * 3)          # translation bounds that hold every boundary pose


def _groups(configs):
    """Configurations grouped by image size (evaluate_batch / solve_batch take one H, W per call)."""
    out = {}
    for cfg in configs:
        cl = boundary_cloud(*cfg)
        out.setdefault((cl["H"], cl["W"]), []).append(cfg)
    return out


def _pack(cfgs, dtype, sort=False):
    """One device batch of clouds, each padded to the longest with ignored points (label -1)."""
    clouds = [boundary_cloud(*c) for c in cfgs]
    n = max(len(c["labels"]) for c in clouds)
    pts = np.zeros((len(clouds), 3, n), dtype=dtype)
    labs = np.full((len(clouds), n), -1, dtype=np.int64)
    for s, c in enumerate(clouds):
        pts[s, :, :len(c["labels"])] = c["points"]
        labs[s, :len(c["labels"])] = c["labels"]
    xyz, lab, n_pts = frustum.pack_clouds(pts, labs, n_pts=np.full(len(clouds), n, dtype=np.int32), dtype=dtype)
    if sort:
        xyz, lab, n_pts = frustum.sort_clouds(xyz, lab, n)
    K = np.stack([c["K"].reshape(9) for c in clouds])
    return clouds, xyz, lab, n_pts, K


def _x(cl, is_2d):
    """The cloud's pose in the layout of is_2d (a 4-DoF pose as 6-DoF: rotation (0, ry, 0))."""
    if cl["is_2d"] == is_2d:
        return cl["x"].copy()
    assert cl["is_2d"] and not is_2d
    x = np.zeros(6)
    x[1], x[3:6] = cl["x"][0], cl["x"][1:4]
    return x


def _init(cl):
    """A solve's init (ry, tx, ty, tz) at the cloud's pose (rotation about y only)."""
    x = cl["x"]
    if cl["is_2d"]:
        return x[:4].copy()
    assert x[0] == 0 and x[2] == 0
    return np.array([x[1], x[3], x[4], x[5]])


def _oracle(cl, x, is_2d):
    P = 4 if is_2d else 6
    return oracle.evaluate(cl["points"].astype(np.float64), cl["labels"], cl["K"], x[:P], cl["H"], cl["W"], is_2d)


def _compare(cfg, c, g, A, ref, x=None, is_2d=None):
    """None if (c, g, A) match the oracle's (co, go, Ao) to test_evaluate_matches_oracle's tolerances, else why not.
    g and A additionally get the oracle's own rounding bound (test_frustum_cull_cpu.oracle_noise)."""
    co, go, Ao = ref
    why = []
    if not abs(c - co) <= 1e-10 * max(1.0, abs(co)):
        why.append("cost %.17g vs %.17g" % (c, co))
    if g is not None or A is not None:
        ng, nA = oracle_noise(cfg, x, is_2d)
    if g is not None and not np.all(np.abs(g - go) <= 1e-9 * np.abs(go) + 1e-9 * np.abs(go).max() + ng):
        why.append("gradient max rel %.3g" % (np.abs(g - go).max() / np.abs(go).max()))
    if A is not None and not np.all(np.abs(A - Ao) <= 1e-9 * np.abs(Ao) + 1e-9 * np.abs(Ao).max() + nA):
        why.append("J^T J max rel %.3g" % (np.abs(A - Ao).max() / np.abs(Ao).max()))
    return None if not why else "%s: %s" % (config_id(cfg), "; ".join(why))


def _configs(dt, is_2d, overflow=False):
    pool = OVERFLOW_CONFIGS if overflow else CONFIGS
    return [c for c in pool if c[2] == dt and boundary_cloud(*c)["is_2d"] == is_2d]


def _solve_configs(dt, is_2d):
    """Clouds a solve can start at: its init is (ry, tx, ty, tz), so a 6-DoF solve starts at rotation (0, ry, 0) --
    the 4-DoF clouds (rotation about y) and 6dof_y."""
    return [c for c in CONFIGS if c[2] == dt and (POSES[c[0]][0] or (not is_2d and c[0] == "6dof_y"))]


@pytest.mark.parametrize("slice_rounds", [0, 4], ids=["one_piece", "sliced"])
@pytest.mark.parametrize("is_2d", [True, False], ids=["4dof", "6dof"])
@pytest.mark.parametrize("dt", ["f32", "f64"])
def test_evaluate_boundary_clouds(cuda, dt, is_2d, slice_rounds):
    """frustum.evaluate_batch on every adversarial cloud of this record / DoF vs oracle.evaluate; a second call
    returns the same bits."""
    bad = []
    for (H, W), cfgs in _groups(_configs(dt, is_2d)).items():
        clouds, xyz, lab, n_pts, K = _pack(cfgs, np.float32 if dt == "f32" else np.float64)
        x = np.stack([_x(c, is_2d) for c in clouds])
        c, g, A = frustum.evaluate_batch(xyz, lab, n_pts, K, x, H, W, is_2d, slice_rounds=slice_rounds)
        c2, g2, A2 = frustum.evaluate_batch(xyz, lab, n_pts, K, x, H, W, is_2d, slice_rounds=slice_rounds)
        assert torch.equal(c, c2) and torch.equal(g, g2) and torch.equal(A, A2)
        c, g, A = c.cpu().numpy(), g.cpu().numpy(), A.cpu().numpy()
        for s, (cfg, cl) in enumerate(zip(cfgs, clouds)):
            why = _compare(cfg, c[s], g[s], A[s], _oracle(cl, x[s], is_2d), x[s], is_2d)
            if why:
                bad.append(why)
    assert not bad, bad


@pytest.mark.parametrize("is_2d", [True, False], ids=["4dof", "6dof"])
def test_traced_solve_first_pass(cuda, is_2d):
    """The solver's own first pass: field [6] (the pass's cost) of trace record 0 of a solve started at the boundary
    pose (float32 record; the traced entry takes float32 only)."""
    bad = []
    for (H, W), cfgs in _groups(_solve_configs("f32", is_2d)).items():
        clouds, xyz, lab, n_pts, K = _pack(cfgs, np.float32)
        x = np.stack([_x(c, is_2d) for c in clouds])
        init = np.stack([[_init(c)] for c in clouds])
        out = frustum.solve_batch(xyz, lab, n_pts, K, init, H, W, WIDE[0], WIDE[1], 2, is_2d, return_all=True,
                                  trace_cap=4)
        tr = out["trace"].cpu().numpy()
        for s, (cfg, cl) in enumerate(zip(cfgs, clouds)):
            assert tr[s, 0, 0, 15] == 1.0 and tr[s, 0, 0, 10] == 0          # a valid record of the initial pass
            why = _compare(cfg, tr[s, 0, 0, 6], None, None, _oracle(cl, x[s], is_2d))
            if why:
                bad.append(why)
    assert not bad, bad


def _infeasible(cfgs, dtype, is_2d, sort=False):
    """Cost of a solve started at the boundary pose with ty bounds that exclude it (termination 6): lm_begin asks for
    one cost-only pass at the init (phase 3), run by the same culled eval_slice as every other pass."""
    bad = []
    for (H, W), group in _groups(cfgs).items():
        clouds, xyz, lab, n_pts, K = _pack(group, dtype, sort=sort)
        x = np.stack([_x(c, is_2d) for c in clouds])
        init = np.stack([[_init(c)] for c in clouds])
        ty = float(init[:, 0, 2].max())
        out = frustum.solve_batch(xyz, lab, n_pts, K, init, H, W, (-1e3, ty + 1.0, -1e3), (1e3, ty + 2.0, 1e3), 500,
                                  is_2d, return_all=True)
        assert (out["stats"][:, 0, 3] == 6).all()
        costs = out["costs"].cpu().numpy()
        for s, (cfg, cl) in enumerate(zip(group, clouds)):
            why = _compare(cfg, costs[s, 0], None, None, _oracle(cl, x[s], is_2d))
            if why:
                bad.append(why)
    return bad


@pytest.mark.parametrize("is_2d", [True, False], ids=["4dof", "6dof"])
@pytest.mark.parametrize("dt", ["f32", "f64"])
def test_infeasible_start_cost(cuda, dt, is_2d):
    bad = _infeasible(_solve_configs(dt, is_2d), np.float32 if dt == "f32" else np.float64, is_2d)
    assert not bad, bad


@pytest.mark.parametrize("is_2d", [True, False], ids=["4dof", "6dof"])
def test_sorted_clouds_infeasible_start_cost(cuda, is_2d):
    """The same clouds after frustum.sort_clouds, which gathers the boundary points into spatially compact,
    label-pure groups (the box level then sees groups made only of near-boundary points)."""
    bad = _infeasible(_solve_configs("f32", is_2d), np.float32, is_2d, sort=True)
    assert not bad, bad


@pytest.mark.parametrize("is_2d", [True, False], ids=["4dof", "6dof"])
@pytest.mark.parametrize("dt", ["f32", "f64"])
def test_disabled_cull_fallback(cuda, dt, is_2d):
    """fx, fy > FLT_MAX: make_class's fp32 coefficients overflow, the cull is disabled (cc.enabled == 0, see the CPU
    model) and every labelled point takes the exact path -- in frustum_evaluate and in an infeasible start's pass."""
    cfgs = _configs(dt, is_2d, overflow=True)
    assert cfgs
    bad = []
    for (H, W), group in _groups(cfgs).items():
        clouds, xyz, lab, n_pts, K = _pack(group, np.float32 if dt == "f32" else np.float64)
        x = np.stack([_x(c, is_2d) for c in clouds])
        for slice_rounds in (0, 4):
            c, g, A = frustum.evaluate_batch(xyz, lab, n_pts, K, x, H, W, is_2d, slice_rounds=slice_rounds)
            c, g, A = c.cpu().numpy(), g.cpu().numpy(), A.cpu().numpy()
            for s, (cfg, cl) in enumerate(zip(group, clouds)):
                why = _compare(cfg, c[s], g[s], A[s], _oracle(cl, x[s], is_2d), x[s], is_2d)
                if why:
                    bad.append(why)
    bad += _infeasible(cfgs, np.float32 if dt == "f32" else np.float64, is_2d)
    assert not bad, bad
