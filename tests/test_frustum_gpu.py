"""GPU parity tests of the registration solver: CUDA path (through the C ABI) vs the CPU oracle.

Tolerances (BASELINE.json north_star): pose within 1e-4 rad / 1e-3 m of the oracle; single
evaluations (cost / gradient / J^T J) agree to 1e-9 relative (fp64 both sides, different
summation order and analytic-vs-dual-number derivatives).
"""
import math

import numpy as np
import pytest
import torch

import oracle
from deepi2p_b200 import frustum, synthetic as syn

pytestmark = pytest.mark.gpu

ROT_TOL = 1e-4
TRANS_TOL = 1e-3


def rot_angle(Ra, Rb):
    c = (np.trace(Ra.T @ Rb) - 1.0) / 2.0
    return math.acos(max(-1.0, min(1.0, c)))


def pose_err(Pa, Pb):
    return rot_angle(Pa[:3, :3], Pb[:3, :3]), float(np.linalg.norm(Pa[:3, 3] - Pb[:3, 3]))


def small_sample(seed, n=2048):
    return syn.make_sample(seed, n_points=n)


@pytest.mark.parametrize("is_2d", [True, False])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_evaluate_matches_oracle(cuda, is_2d, dtype):
    rng = np.random.default_rng(7)
    S = 4
    samples = [small_sample(100 + s, 3000 + 17 * s) for s in range(S)]
    P = 4 if is_2d else 6
    for s, smp in enumerate(samples):
        pts = smp["points"].astype(np.float64)
        if dtype == np.float64:
            pts = pts + rng.normal(0, 1e-9, pts.shape)      # not float32-representable
        xyz, lab, n_pts = frustum.pack_clouds(pts, smp["pred"], dtype=dtype)
        assert xyz.dtype == (torch.float32 if dtype == np.float32 else torch.float64)
        x = np.zeros(6)
        if is_2d:
            x[:4] = [smp["ry_gt"] + 0.05, smp["t_gt"][0] + 0.3, 0.02, smp["t_gt"][2] - 0.5]
        else:
            x[:6] = [0.02, smp["ry_gt"] + 0.05, -0.03, smp["t_gt"][0] + 0.3, 0.02, smp["t_gt"][2] - 0.5]
        c, g, A = frustum.evaluate_batch(xyz, lab, n_pts, smp["K"], x[None], smp["H"], smp["W"], is_2d)
        co, go, Ao = oracle.evaluate(pts, smp["pred"], smp["K"], x[:P], smp["H"], smp["W"], is_2d)
        assert abs(c.item() - co) <= 1e-10 * max(1.0, abs(co))
        np.testing.assert_allclose(g[0].cpu().numpy(), go, rtol=1e-9, atol=1e-9 * np.abs(go).max())
        np.testing.assert_allclose(A[0].cpu().numpy(), Ao, rtol=1e-9, atol=1e-9 * np.abs(Ao).max())


def test_evaluate_small_angle_branch(cuda):
    smp = small_sample(3)
    pts = smp["points"].astype(np.float64)
    xyz, lab, n_pts = frustum.pack_clouds(pts, smp["pred"])
    for is_2d, x in ((True, [1e-9, 0.1, 0.0, 0.2, 0, 0]), (False, [1e-9, -2e-9, 3e-9, 0.1, 0.0, 0.2]),
                     (False, [1e-5, 2e-5, -1e-5, 0.1, 0.0, 0.2])):
        P = 4 if is_2d else 6
        x = np.asarray(x, dtype=np.float64)
        c, g, A = frustum.evaluate_batch(xyz, lab, n_pts, smp["K"], x[None], smp["H"], smp["W"], is_2d)
        co, go, Ao = oracle.evaluate(pts, smp["pred"], smp["K"], x[:P], smp["H"], smp["W"], is_2d)
        assert abs(c.item() - co) <= 1e-10 * max(1.0, abs(co))
        np.testing.assert_allclose(g[0].cpu().numpy(), go, rtol=1e-8, atol=1e-8 * np.abs(go).max())
        np.testing.assert_allclose(A[0].cpu().numpy(), Ao, rtol=1e-8, atol=1e-8 * np.abs(Ao).max())


@pytest.mark.parametrize("is_2d", [True, False])
def test_solve_matches_oracle(cuda, is_2d):
    """Trajectory-level parity.  The objective is piecewise smooth with thousands of kinks and the
    solver stops on a 1e-6 relative function tolerance, so trajectories are chaotic at the rounding
    level: even the CPU oracle against itself with an algebraically equivalent linear solver moves
    ~3-4 % of full-size solves by > 1e-7 (tests/tools/parity_sensitivity_cpu.py).  The gate is therefore
    statistical: at least 97 % of the (sample, init) solves within 1e-4 rad / 1e-3 m of the oracle, 93 % with
    identical iteration / evaluation / termination records, a tiny median difference, and per registration either the
    same best-of-I pose or a GPU best cost that is not worse than the oracle's.  (tests/tools/trace_divergence.py
    traces an out-of-gate solve to its first divergent evaluation; DESIGN.md 3.1 explains why such solves leave the
    gate when either implementation's own input is moved by one ulp.)"""
    S, I, n = 10, 12, 4096
    xs, ls, inits, Ks = [], [], [], []
    smps = []
    for s in range(S):
        smp = small_sample(200 + s, n)
        iy, _, _, _ = oracle.initial_guess(smp["points"], smp["pred"])
        ry, t = syn.make_inits(200 + s, iy, I)
        smps.append((smp, ry, t))
        xs.append(smp["points"]); ls.append(smp["pred"]); Ks.append(smp["K"].reshape(9))
        inits.append(np.concatenate([ry[:, None], t], axis=1))
    xyz, lab, n_pts = frustum.pack_clouds(np.stack(xs), np.stack(ls))
    out = frustum.solve_batch(xyz, lab, n_pts, np.stack(Ks), np.stack(inits), smps[0][0]["H"], smps[0][0]["W"],
                              syn.T_LB, syn.T_UB, 500, is_2d, return_all=True)
    params = out["params"].cpu().numpy()
    costs = out["costs"].cpu().numpy()
    stats = out["stats"].cpu().numpy()
    drs, dts, same_counts, best_ok = [], [], 0, 0
    for s, (smp, ry, t) in enumerate(smps):
        ms = oracle.solve_multistart(smp["points"], smp["pred"], smp["K"], ry, t, smp["H"], smp["W"], syn.T_LB,
                                     syn.T_UB, 500, is_2d)
        for i in range(I):
            if is_2d:
                dr = abs(params[s, i, 0] - ms["params"][i, 0])
                dt = np.linalg.norm(params[s, i, 1:4] - ms["params"][i, 1:4])
            else:
                dr = np.linalg.norm(params[s, i, 0:3] - ms["params"][i, 0:3])
                dt = np.linalg.norm(params[s, i, 3:6] - ms["params"][i, 3:6])
            drs.append(dr); dts.append(dt)
            if dr < ROT_TOL and dt < TRANS_TOL:
                assert abs(costs[s, i] - ms["costs"][i]) <= 1e-5 * max(1.0, ms["costs"][i])
            same_counts += int(stats[s, i, 0] == ms["stats"][i]["iterations"]
                               and stats[s, i, 1] == ms["stats"][i]["unique_evals"]
                               and stats[s, i, 3] == ms["stats"][i]["termination"])
        # arg-min over inits and the 4x4 (only meaningful where the winning solve agreed)
        er, et = pose_err(out["P"][s].cpu().numpy(), ms["P"])
        best_ok += int((er < ROT_TOL and et < TRANS_TOL and int(out["best"][s]) == ms["best"])
                       or out["cost"][s].item() <= ms["cost"] * (1 + 1e-9))
        # the reported pose/cost are those of the reported best init
        b = int(out["best"][s])
        assert out["cost"][s].item() == costs[s, b] and b == int(np.argmin(costs[s]))
    drs, dts = np.array(drs), np.array(dts)
    within = (drs < ROT_TOL) & (dts < TRANS_TOL)
    print("solves within gate %d/%d, identical counters %d/%d, best-of-I agree %d/%d, median rot %.2e trans %.2e, "
          "max rot %.2e trans %.2e" % (within.sum(), within.size, same_counts, within.size, best_ok, S,
                                       np.median(drs), np.median(dts), drs.max(), dts.max()))
    assert within.mean() >= 0.97
    assert same_counts >= 0.93 * within.size
    assert np.median(drs) < 1e-8 and np.median(dts) < 1e-7
    assert best_ok == S


def test_known_answer_zero_cost_start(cuda):
    """Exact GT labels + start at the GT pose => cost 0 => the init pose comes back bit for bit."""
    smp = small_sample(5)
    xyz, lab, n_pts = frustum.pack_clouds(smp["points"], smp["gt"])
    init = np.array([[[smp["ry_gt"], *smp["t_gt"]]]])
    for is_2d in (True, False):
        out = frustum.solve_batch(xyz, lab, n_pts, smp["K"], init, smp["H"], smp["W"], [-100] * 3, [100] * 3, 500,
                                  is_2d, return_all=True)
        assert out["cost"].item() == 0.0
        st = out["stats"][0, 0].tolist()
        assert st[0] == 0 and st[1] == 1 and st[3] == 0
        p = out["params"][0, 0].cpu().numpy()
        if is_2d:
            assert p[0] == smp["ry_gt"] and np.array_equal(p[1:4], smp["t_gt"])
        else:
            assert p[1] == smp["ry_gt"] and p[0] == 0 and p[2] == 0 and np.array_equal(p[3:6], smp["t_gt"])
        er, et = pose_err(out["P"][0].cpu().numpy(), smp["P_gt"])
        assert er < 1e-12 and et < 1e-12


def test_infeasible_start_returns_init(cuda):
    smp = small_sample(6)
    xyz, lab, n_pts = frustum.pack_clouds(smp["points"], smp["pred"])
    init = np.array([[[0.3, 0.0, 0.5, 1.0]]])       # ty = 0.5 outside [-0.1, 0.1]
    out = frustum.solve_batch(xyz, lab, n_pts, smp["K"], init, smp["H"], smp["W"], syn.T_LB, syn.T_UB, 500, True,
                              return_all=True)
    assert out["stats"][0, 0, 3].item() == 6
    np.testing.assert_array_equal(out["params"][0, 0, :4].cpu().numpy(), [0.3, 0.0, 0.5, 1.0])
    Po, co, _, st, _ = oracle.solve(smp["points"], smp["pred"], smp["K"], 0.3, [0.0, 0.5, 1.0], smp["H"], smp["W"],
                                    syn.T_LB, syn.T_UB)
    assert st["termination"] == 6
    er, et = pose_err(out["P"][0].cpu().numpy(), Po)
    assert er < 1e-12 and et < 1e-12
    # the cost of an infeasible start is the cost AT the untouched init (registration.cpp:150-155 evaluates after the
    # failed solve), not 0 -- a zero would win every arg-min over inits
    assert co > 0 and abs(out["cost"][0].item() - co) <= 1e-10 * co
    assert out["stats"][0, 0, 0].item() == 0 and out["stats"][0, 0, 1].item() == 0


def test_mixed_feasible_and_infeasible_inits(cuda):
    """One infeasible init among feasible ones must not win the arg-min with a fake zero cost."""
    smp = small_sample(6)
    xyz, lab, n_pts = frustum.pack_clouds(smp["points"], smp["pred"])
    iy, _, _, _ = oracle.initial_guess(smp["points"], smp["pred"])
    ry, t = syn.make_inits(6, iy, 3)
    init = np.concatenate([ry[:, None], t], axis=1)
    init = np.concatenate([np.array([[0.3, 0.0, 0.5, 1.0]]), init], axis=0)[None]      # init 0 infeasible (ty = 0.5)
    out = frustum.solve_batch(xyz, lab, n_pts, smp["K"], init, smp["H"], smp["W"], syn.T_LB, syn.T_UB, 500, True,
                              return_all=True)
    costs = out["costs"][0].cpu().numpy()
    assert out["stats"][0, 0, 3].item() == 6 and costs[0] > 0
    assert int(out["best"][0]) == int(np.argmin(costs))
    ms = oracle.solve_multistart(smp["points"], smp["pred"], smp["K"], init[0, :, 0], init[0, :, 1:4], smp["H"],
                                 smp["W"], syn.T_LB, syn.T_UB, 500, True)
    assert abs(costs[0] - ms["costs"][0]) <= 1e-10 * ms["costs"][0]


def test_ragged_empty_and_ignored_labels(cuda):
    """n_pts shorter than the stride, an empty cloud, labels outside {0,1} ignored, n not a
    multiple of the tile or of 16."""
    n = 3001
    smp = small_sample(9, n)
    pred = smp["pred"].copy()
    pred[::7] = 5                     # ignored (registration.cpp:89,106)
    pts = np.stack([smp["points"], smp["points"], smp["points"]])
    labs = np.stack([pred, pred, pred])
    n_pts = np.array([n, 1777, 0], dtype=np.int32)
    xyz, lab, npd = frustum.pack_clouds(pts, labs, n_pts=n_pts)
    iy, _, _, _ = oracle.initial_guess(smp["points"], smp["pred"])
    ry, t = syn.make_inits(9, iy, 3)
    init = np.concatenate([ry[:, None], t], axis=1)[None].repeat(3, axis=0)
    out = frustum.solve_batch(xyz, lab, npd, smp["K"], init, smp["H"], smp["W"], syn.T_LB, syn.T_UB, 500, True,
                              return_all=True)
    ok = total = 0
    for s, m in enumerate(n_pts):
        for i in range(3):
            Po, co, _, st, xo = oracle.solve(smp["points"][:, :m], pred[:m], smp["K"], ry[i], t[i], smp["H"],
                                             smp["W"], syn.T_LB, syn.T_UB)
            p = out["params"][s, i].cpu().numpy()
            total += 1
            ok += int(abs(p[0] - xo[0]) < ROT_TOL and np.linalg.norm(p[1:4] - xo[1:4]) < TRANS_TOL
                      and out["stats"][s, i, 3].item() == st["termination"])
            # whatever the trajectory, the reported cost is the cost AT the reported pose for THIS cloud
            # (checks n_pts / ignored labels / the tail of the last group exactly)
            co_at, _, _ = oracle.evaluate(smp["points"][:, :m], pred[:m], smp["K"], p[:4], smp["H"], smp["W"], True) \
                if m > 0 else (0.0, None, None)
            assert abs(out["costs"][s, i].item() - co_at) <= 1e-9 * max(1.0, co_at)
    assert ok >= total - 1      # trajectory-level agreement is statistical, see test_solve_matches_oracle
    # empty cloud: zero cost, init returned
    assert out["costs"][2, 0].item() == 0.0


def test_sort_clouds_is_a_permutation(cuda):
    """frustum_sort_batch_f32 (the drop-in's pre-sort): every point kept, labels other than 0 / 1 become -1 and sort
    last, label 0 before label 1, and the cost at a pose is the unsorted cloud's up to summation order."""
    S, n = 3, 3001
    smps = [small_sample(30 + s, n) for s in range(S)]
    pts = np.stack([s["points"] for s in smps]); prd = np.stack([s["pred"] for s in smps]).astype(np.int64)
    prd[:, ::97] = 7                                           # some ignored labels
    xyz, l8, n_pts = frustum.pack_clouds(pts, prd)
    sx, sl, sn = frustum.sort_clouds(xyz, l8, n)
    assert sn.tolist() == [n] * S and sx.shape[-1] == (n + 15) // 16 * 16
    for s in range(S):
        a = np.concatenate([xyz[s, :, :n].cpu().numpy().T, l8[s, :n].cpu().numpy()[:, None].astype(np.float32)], 1)
        b = np.concatenate([sx[s, :, :n].cpu().numpy().T, sl[s, :n].cpu().numpy()[:, None].astype(np.float32)], 1)
        assert np.array_equal(a[np.lexsort(a.T[::-1])], b[np.lexsort(b.T[::-1])])      # same multiset of (x, y, z, label)
        lab = sl[s, :n].cpu().numpy()
        cls = np.where(lab == 0, 0, np.where(lab == 1, 1, 2))
        assert (np.diff(cls) >= 0).all()                                              # 0s, then 1s, then ignored
        assert (sl[s, n:].cpu().numpy() == -1).all()
    K, H, W = smps[0]["K"], smps[0]["H"], smps[0]["W"]
    x = torch.zeros(S, 6, dtype=torch.float64, device="cuda"); x[:, 0] = 0.3; x[:, 3] = 1.0
    c0, g0, _ = frustum.evaluate_batch(xyz, l8, n_pts, K, x, H, W, True)
    c1, g1, _ = frustum.evaluate_batch(sx, sl, sn, K, x, H, W, True)
    assert torch.allclose(c0, c1, rtol=1e-12, atol=0) and torch.allclose(g0, g1, rtol=1e-9, atol=1e-9)


def test_residual_vector_and_dropin(cuda):
    import deepi2p_b200
    deepi2p_b200.install_dropins()
    import FrustumRegistration
    smp = small_sample(11, 2500)
    iy, pf, lf, _ = oracle.initial_guess(smp["points"], smp["pred"])
    for is_2d in (True, False):
        P, cost, res = FrustumRegistration.solvePGivenK(pf.astype(np.float64), lf.astype(np.int64), smp["K"], iy,
                                                        np.array([0.0, 0.0, 1.5]), smp["H"], smp["W"],
                                                        [-5, -0.1, -10], [5, 0.1, 10], 500, False, is_2d)
        Po, co, ro, st, xo = oracle.solve(pf, lf, smp["K"], iy, [0.0, 0.0, 1.5], smp["H"], smp["W"], syn.T_LB,
                                          syn.T_UB, 500, is_2d)
        assert isinstance(P, np.ndarray) and P.shape == (4, 4) and isinstance(cost, float)
        assert res.shape == ro.shape and res.dtype == np.float64
        # residual vector and cost at the RETURNED pose (independent of the trajectory)
        if is_2d:
            x_ret = np.array([math.atan2(P[0, 2], P[0, 0]), P[0, 3], P[1, 3], P[2, 3]])
        else:
            from scipy.spatial.transform import Rotation
            x_ret = np.concatenate([Rotation.from_matrix(P[:3, :3]).as_rotvec(), P[:3, 3]])
        r_at, c_at = oracle.residuals(pf, lf, smp["K"], x_ret, smp["H"], smp["W"], is_2d)
        np.testing.assert_allclose(res, r_at, rtol=0, atol=1e-6)
        assert abs(cost - c_at) <= 1e-8 * max(1.0, c_at)
        er, et = pose_err(P, Po)
        print("drop-in pose vs oracle: rot %.2e rad, trans %.2e m (is_2d=%s)" % (er, et, is_2d))
        assert cost <= co * (1 + 1e-3) or (er < ROT_TOL and et < TRANS_TOL)
    assert FrustumRegistration.solve is FrustumRegistration.solvePGivenK


def philox4x32_10(c, k0, k1):
    c = [np.asarray(v, dtype=np.uint64) for v in c]
    k0 = np.uint64(k0); k1 = np.uint64(k1)
    M0, M1, MASK = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0 = M0 * c[0]; p1 = M1 * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & MASK
        hi1, lo1 = p1 >> np.uint64(32), p1 & MASK
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0 = (k0 + np.uint64(0x9E3779B9)) & MASK
        k1 = (k1 + np.uint64(0xBB67AE85)) & MASK
    return c


def test_prepare_matches_initial_guess(cuda):
    """On-device get_initial_guess / front filter / inits vs the CPU restatement."""
    S, n, I, seed = 5, 3333, 60, 1234
    smps = [small_sample(300 + s, n) for s in range(S)]
    # make the front filter bite: clean predictions for sample 0, no inside prediction for sample 4
    smps[0]["pred"] = smps[0]["gt"].copy()
    smps[4]["pred"] = np.zeros(n, dtype=np.int32)
    xyz_in, pred_in, _ = frustum.pack_clouds(np.stack([s["points"] for s in smps]),
                                             np.stack([s["pred"] for s in smps]))
    prep = frustum.prepare_batch(xyz_in, pred_in, n, I, seed=seed, sort=False)
    prep_sorted = frustum.prepare_batch(xyz_in, pred_in, n, I, seed=seed, sort=True)
    npts = prep["n_pts"].cpu().numpy()
    for s, smp in enumerate(smps):
        if s == 4:
            assert prep["degenerate"][s].item() == 1 and npts[s] == n
            continue
        iy, pf, lf, mask = oracle.initial_guess(smp["points"], smp["pred"])
        assert prep["degenerate"][s].item() == 0
        assert abs(prep["init_y_angle"][s].item() - iy) < 1e-12
        assert npts[s] == mask.sum()
        np.testing.assert_array_equal(prep["xyz"][s, :, :npts[s]].cpu().numpy(), pf.astype(np.float32))
        np.testing.assert_array_equal(prep["label"][s, :npts[s]].cpu().numpy(), lf.astype(np.int8))
        assert (prep["label"][s, npts[s]:] == -1).all()
        # sorted variant: same multiset of points, label-0 block then label-1 block, same inits
        assert prep_sorted["n_pts"][s].item() == npts[s]
        xs = prep_sorted["xyz"][s, :, :npts[s]].cpu().numpy()
        ls_ = prep_sorted["label"][s, :npts[s]].cpu().numpy()
        assert (np.diff(ls_.astype(np.int32)) >= 0).all()
        a = np.concatenate([xs, ls_[None].astype(np.float32)], axis=0)
        b = np.concatenate([pf.astype(np.float32), lf[None].astype(np.float32)], axis=0)
        np.testing.assert_array_equal(a[:, np.lexsort(a)], b[:, np.lexsort(b)])
        assert (prep_sorted["label"][s, npts[s]:] == -1).all()
        np.testing.assert_array_equal(prep_sorted["init"][s].cpu().numpy(), prep["init"][s].cpu().numpy())
        c = philox4x32_10([np.arange(I), np.full(I, s), np.zeros(I), np.zeros(I)], seed & 0xFFFFFFFF, seed >> 32)
        u1 = 1.0 - ((c[0] >> np.uint64(5)).astype(np.float64) * 67108864.0
                    + (c[1] >> np.uint64(6)).astype(np.float64)) / 9007199254740992.0
        u2 = (c[2].astype(np.float64) + 0.5) / 4294967296.0
        u3 = (c[3].astype(np.float64) + 0.5) / 4294967296.0
        ry = iy + frustum.RY_SIGMA * np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)
        tz = (2.0 * u3 - 1.0) * frustum.T_AMPLITUDE
        got = prep["init"][s].cpu().numpy()
        np.testing.assert_allclose(got[:, 0], ry, rtol=0, atol=1e-12)
        np.testing.assert_allclose(got[:, 3], tz, rtol=0, atol=1e-12)
        assert (got[:, 1:3] == 0).all()
    assert npts[0] < n      # the filter removed something
    # distribution sanity of the inits
    allr = (prep["init"][:4, :, 0] - prep["init_y_angle"][:4, None]).cpu().numpy().ravel()
    assert abs(allr.std() - frustum.RY_SIGMA) < 0.25 * frustum.RY_SIGMA
    # full batched registration == oracle multistart on the prepared inputs
    out = frustum.register_batch(xyz_in, pred_in, n, smps[0]["K"], smps[0]["H"], smps[0]["W"], n_inits=4, seed=seed)
    prep4 = frustum.prepare_batch(xyz_in, pred_in, n, 4, seed=seed)
    for s in (0, 1):
        smp = smps[s]
        _, pf, lf, _ = oracle.initial_guess(smp["points"], smp["pred"])
        ini = prep4["init"][s].cpu().numpy()
        ms = oracle.solve_multistart(pf, lf, smp["K"], ini[:, 0], ini[:, 1:4], smp["H"], smp["W"], syn.T_LB, syn.T_UB)
        er, et = pose_err(out["P"][s].cpu().numpy(), ms["P"])
        assert er < ROT_TOL and et < TRANS_TOL
    assert out["cost"][4].item() == 1e4
    np.testing.assert_array_equal(out["P"][4].cpu().numpy(), np.eye(4))


def test_one_call_path_and_traces(cuda):
    """(a) the ONE-call C entry (frustum_register_batch_f32) gives the bits of prepare + solve; (b) the traced solve
    gives the bits of the plain solve, writes one record per cloud pass, and its records agree with the oracle's trace
    (same evaluated points and decisions) on solves that end within the gate; (c) a second run reproduces the first
    bit for bit (fixed-order sums, slice sums independent of which warp computed them)."""
    S, I, n = 3, 5, 6000
    smps = [small_sample(700 + s, n) for s in range(S)]
    xyz_in, pred_in, _ = frustum.pack_clouds(np.stack([s["points"] for s in smps]), np.stack([s["pred"] for s in smps]))
    K, H, W = smps[0]["K"], smps[0]["H"], smps[0]["W"]
    reg = frustum.register_batch(xyz_in, pred_in, n, K, H, W, n_inits=I, seed=11, return_all=True)
    prep = frustum.prepare_batch(xyz_in, pred_in, n, I, seed=11)
    assert torch.equal(prep["init"], reg["init"]) and torch.equal(prep["n_pts"], reg["n_pts"])
    plain = frustum.solve_batch(prep["xyz"], prep["label"], prep["n_pts"], K, prep["init"], H, W, return_all=True)
    traced = frustum.solve_batch(prep["xyz"], prep["label"], prep["n_pts"], K, prep["init"], H, W, return_all=True,
                                 trace_cap=256)
    again = frustum.register_batch(xyz_in, pred_in, n, K, H, W, n_inits=I, seed=11, return_all=True)
    for key in ("P", "cost", "best", "params", "costs", "stats"):
        assert torch.equal(reg[key], plain[key]), key
        assert torch.equal(traced[key], plain[key]), key
        assert torch.equal(again[key], reg[key]), key
    tr = traced["trace"].cpu().numpy()
    stats = plain["stats"].cpu().numpy()
    params = plain["params"].cpu().numpy()
    inits = prep["init"].cpu().numpy()
    agree = total = 0
    for s, smp in enumerate(smps):
        _, pf, lf, _ = oracle.initial_guess(smp["points"], smp["pred"])
        for i in range(I):
            rec = tr[s, i][tr[s, i][:, 15] > 0]
            assert len(rec) == stats[s, i, 1]                       # one record per cloud pass
            assert rec[-1, 12] == stats[s, i, 3]                     # the last record carries the termination code
            assert rec[0, 10] == 0 and np.array_equal(rec[0, :4], inits[s, i])
            o = oracle.solve(pf, lf, K, inits[s, i, 0], inits[s, i, 1:4], H, W, syn.T_LB, syn.T_UB, 500, True,
                             want_residuals=False, trace_cap=256)
            if abs(params[s, i, 0] - o[4][0]) < ROT_TOL and np.linalg.norm(params[s, i, 1:4] - o[4][1:4]) < TRANS_TOL:
                total += 1
                to = o[5]
                same = (len(to) == len(rec) and np.allclose(to[:, :4], rec[:, :4], rtol=0, atol=1e-6)
                        and np.array_equal(to[:, 10:13], rec[:, 10:13]))
                agree += int(same)
    assert total >= S * I - 2 and agree >= total - 1


def test_helped_passes_are_reproducible(cuda):
    """Six full-size problems on six CTAs: every pass is cut into 10 slices and the 19 idle warps of each CTA race for
    them.  Which warp computes which slice changes from run to run; the results must not (a slice's sum depends only
    on the cloud, the pose and the slice, and the slice sums are added in slice order)."""
    S, I = 2, 3
    smps = [syn.make_sample(820 + s) for s in range(S)]
    xyz_in, pred_in, _ = frustum.pack_clouds(np.stack([s["points"] for s in smps]), np.stack([s["pred"] for s in smps]))
    K, H, W = smps[0]["K"], smps[0]["H"], smps[0]["W"]
    ref = frustum.register_batch(xyz_in, pred_in, 20480, K, H, W, n_inits=I, seed=5, return_all=True)
    ref = {k: v.clone() for k, v in ref.items()}
    for _ in range(12):
        out = frustum.register_batch(xyz_in, pred_in, 20480, K, H, W, n_inits=I, seed=5, return_all=True)
        for key in ("P", "cost", "params", "costs", "stats"):
            assert torch.equal(out[key], ref[key]), key
    # and the sums of such a helped pass are the ones frustum_evaluate forms with the same slicing
    from deepi2p_b200 import _native
    lib = _native.load()
    assert lib.frustum_solve_slice_after(S, I, 1, 0) == 0
    rounds = lib.frustum_solve_slice_rounds(S, I, 1, 0)
    prep = frustum.prepare_batch(xyz_in, pred_in, 20480, I, seed=5)
    x = ref["params"][:, int(ref["best"][0])].contiguous()
    c, _, _ = frustum.evaluate_batch(prep["xyz"], prep["label"], prep["n_pts"], K, x, H, W, True, slice_rounds=rounds)
    for s in range(S):
        if int(ref["best"][s]) == int(ref["best"][0]):
            assert c[s].item() == ref["costs"][s, int(ref["best"][0])].item()      # bit for bit


def test_large_batch_late_problems(cuda, monkeypatch):
    """A batch of more than four waves of problems: passes are sliced only from a problem's 48th pass on, except for the
    LAST resident-grid's worth of queue positions, which are sliced from their first pass (they run while the batch
    drains).  Which problems are late is a function of the batch alone: two runs give the same bits.  Against the same
    batch with the rule switched off the sums differ at rounding level only: the usual statistical gate applies."""
    from deepi2p_b200 import _native
    lib = _native.load()
    S, I = 200, 60
    if lib.frustum_solve_slice_after(S, I, 1, 0) == 0:
        pytest.skip("this GPU holds the whole batch in fewer than four waves")
    base = [syn.make_sample(950 + s) for s in range(8)]
    pts = np.stack([base[s % 8]["points"] for s in range(S)])
    prd = np.stack([base[s % 8]["pred"] for s in range(S)])
    xyz_in, pred_in, _ = frustum.pack_clouds(pts, prd)
    K, H, W = base[0]["K"], base[0]["H"], base[0]["W"]
    a = frustum.register_batch(xyz_in, pred_in, 20480, K, H, W, n_inits=I, seed=21, return_all=True)
    a = {k: v.clone() for k, v in a.items()}
    b = frustum.register_batch(xyz_in, pred_in, 20480, K, H, W, n_inits=I, seed=21, return_all=True)
    for key in ("P", "cost", "params", "costs", "stats"):
        assert torch.equal(a[key], b[key]), key
    monkeypatch.setenv("DIB_LATE_PROBLEMS", "0")
    c = frustum.register_batch(xyz_in, pred_in, 20480, K, H, W, n_inits=I, seed=21, return_all=True)
    pa, pc = a["params"].cpu().numpy(), c["params"].cpu().numpy()
    rot = np.abs(pa[..., 0] - pc[..., 0]); tr = np.linalg.norm(pa[..., 1:4] - pc[..., 1:4], axis=-1)
    within = (rot < 1e-4) & (tr < 1e-3)
    assert within.mean() >= 0.97, within.mean()
    rel = (a["cost"] - c["cost"]).abs() / c["cost"].abs().clamp_min(1e-30)
    assert (rel < 1e-6).float().mean().item() >= 0.95    # best-of-I cost of nearly every registration unchanged


def test_full_size_properties(cuda):
    """BASELINE-size cloud (20480 points): size-independent properties instead of the oracle --
    the returned cost equals a fresh evaluation at the returned pose, the cost never exceeds the
    start cost, translations respect the box, and a solve restarted from its own solution stops
    immediately at the same pose (idempotence)."""
    S, I = 4, 6
    smps = [syn.make_sample(400 + s) for s in range(S)]
    xyz, lab, n_pts = frustum.pack_clouds(np.stack([s["points"] for s in smps]), np.stack([s["pred"] for s in smps]))
    inits = []
    for s, smp in enumerate(smps):
        iy, _, _, _ = oracle.initial_guess(smp["points"], smp["pred"])
        ry, t = syn.make_inits(400 + s, iy, I)
        inits.append(np.concatenate([ry[:, None], t], axis=1))
    inits = np.stack(inits)
    K = smps[0]["K"]; H = smps[0]["H"]; W = smps[0]["W"]
    out = frustum.solve_batch(xyz, lab, n_pts, K, inits, H, W, syn.T_LB, syn.T_UB, 500, True, return_all=True)
    params = out["params"].cpu().numpy()
    for i in range(I):
        x = np.zeros((S, 6)); x[:, :4] = params[:, i, :4]
        c, _, _ = frustum.evaluate_batch(xyz, lab, n_pts, K, x, H, W, True)
        np.testing.assert_allclose(c.cpu().numpy(), out["costs"][:, i].cpu().numpy(), rtol=1e-12)
        x0 = np.zeros((S, 6)); x0[:, :4] = inits[:, i]
        c0, _, _ = frustum.evaluate_batch(xyz, lab, n_pts, K, x0, H, W, True)
        assert (out["costs"][:, i] <= c0 * (1 + 1e-12)).all()
    assert (params[:, :, 1:4] >= np.array(syn.T_LB) - 1e-15).all() and (params[:, :, 1:4] <= np.array(syn.T_UB) + 1e-15).all()
    # best-of-I equals the min of the per-init costs, lowest index on ties
    costs = out["costs"].cpu().numpy()
    np.testing.assert_array_equal(out["best"].cpu().numpy(), np.argmin(costs, axis=1))
    # restart from the solution: the cost can only go down, and only marginally (the first solve
    # stopped on the 1e-6 relative function tolerance, not at a stationary point)
    re_init = params[:, :, :4].copy()
    out2 = frustum.solve_batch(xyz, lab, n_pts, K, re_init, H, W, syn.T_LB, syn.T_UB, 500, True, return_all=True)
    c2 = out2["costs"].cpu().numpy()
    assert (c2 <= costs * (1 + 1e-12)).all()
    assert ((costs - c2) <= 1e-3 * costs).all()
    # one oracle cross-check at full size
    ms = oracle.solve(smps[0]["points"], smps[0]["pred"], K, inits[0, 0, 0], inits[0, 0, 1:4], H, W, syn.T_LB, syn.T_UB)
    assert abs(params[0, 0, 0] - ms[4][0]) < ROT_TOL and np.linalg.norm(params[0, 0, 1:4] - ms[4][1:4]) < TRANS_TOL


def test_f64_coordinates_solve(cuda):
    """Coordinates that are not float32-representable take the f64 device record end to end."""
    smp = small_sample(21, 3000)
    rng = np.random.default_rng(3)
    pts = smp["points"].astype(np.float64) + rng.normal(0, 1e-7, smp["points"].shape)
    xyz, lab, n_pts = frustum.pack_clouds(pts, smp["pred"])
    assert xyz.dtype == torch.float64
    iy, _, _, _ = oracle.initial_guess(pts, smp["pred"])
    ry, t = syn.make_inits(21, iy, 4)
    init = np.concatenate([ry[:, None], t], axis=1)[None]
    out = frustum.solve_batch(xyz, lab, n_pts, smp["K"], init, smp["H"], smp["W"], syn.T_LB, syn.T_UB, 500, True,
                              return_all=True)
    ok = 0
    for i in range(4):
        _, co, _, st, xo = oracle.solve(pts, smp["pred"], smp["K"], ry[i], t[i], smp["H"], smp["W"], syn.T_LB, syn.T_UB)
        p = out["params"][0, i].cpu().numpy()
        ok += int(abs(p[0] - xo[0]) < ROT_TOL and np.linalg.norm(p[1:4] - xo[1:4]) < TRANS_TOL)
        c_at = oracle.evaluate(pts, smp["pred"], smp["K"], p[:4], smp["H"], smp["W"], True)[0]
        assert abs(out["costs"][0, i].item() - c_at) <= 1e-9 * max(1.0, c_at)
    assert ok >= 3


def test_large_cloud_unsorted_fallback_and_oxford_6dof(cuda):
    """(a) a cloud larger than the in-shared-memory sort window (32768 points) goes through prepare
    unsorted and through the solver's multi-chunk box table; (b) Oxford-shaped intrinsics, 6-DoF."""
    n = 40000
    smp = syn.make_sample(31, n_points=n, shape="oxford")
    xyz_in, pred_in, _ = frustum.pack_clouds(smp["points"], smp["pred"])
    prep = frustum.prepare_batch(xyz_in, pred_in, n, 3, seed=5)
    iy, pf, lf, mask = oracle.initial_guess(smp["points"], smp["pred"])
    m = int(prep["n_pts"][0])
    assert m == mask.sum()
    np.testing.assert_array_equal(prep["xyz"][0, :, :m].cpu().numpy(), pf.astype(np.float32))   # original order kept
    for is_2d in (True, False):
        out = frustum.solve_batch(prep["xyz"], prep["label"], prep["n_pts"], smp["K"], prep["init"], smp["H"],
                                  smp["W"], syn.T_LB, syn.T_UB, 500, is_2d, return_all=True)
        ini = prep["init"][0].cpu().numpy()
        ok = 0
        for i in range(3):
            _, co, _, st, xo = oracle.solve(pf, lf, smp["K"], ini[i, 0], ini[i, 1:4], smp["H"], smp["W"], syn.T_LB,
                                            syn.T_UB, 500, is_2d)
            P = 4 if is_2d else 6
            p = out["params"][0, i].cpu().numpy()
            nr = P - 3
            ok += int(np.linalg.norm(p[:nr] - xo[:nr]) < ROT_TOL and np.linalg.norm(p[nr:P] - xo[nr:P]) < TRANS_TOL)
            c_at = oracle.evaluate(pf, lf, smp["K"], p[:P], smp["H"], smp["W"], is_2d)[0]
            assert abs(out["costs"][0, i].item() - c_at) <= 1e-9 * max(1.0, c_at)
        assert ok >= 2


def test_inside_mask_and_pose_error_ops(cuda):
    """N3 ops: label projection rule and the RTE/RRE metric, vs line-by-line restatements of the reference's
    numpy/scipy code (oracle.inside_img_mask / oracle.pose_diff)."""
    from scipy.spatial.transform import Rotation
    S, n = 5, 3000
    smps = [small_sample(500 + s, n) for s in range(S)]
    xyz, _, n_pts = frustum.pack_clouds(np.stack([s["points"] for s in smps]), np.stack([s["pred"] for s in smps]),
                                        n_pts=np.array([n, n, 2000, 17, 0], dtype=np.int32))
    P = np.stack([s["P_gt"] for s in smps])
    mask = frustum.inside_mask_batch(xyz, n_pts, P, smps[0]["K"], smps[0]["H"], smps[0]["W"]).cpu().numpy()
    for s, m in enumerate([n, n, 2000, 17, 0]):
        want = oracle.inside_img_mask(smps[s]["points"][:, :m], P[s], smps[s]["K"], smps[s]["H"], smps[s]["W"])
        np.testing.assert_array_equal(mask[s, :m], want.astype(np.int8))
        assert (mask[s, m:] == -1).all()
        if m == n:
            np.testing.assert_array_equal(mask[s, :n], smps[s]["gt"].astype(np.int8))   # the generator's own labels
    # pose errors
    rng = np.random.default_rng(0)
    Pp, Pg = [], []
    for i in range(64):
        A = np.eye(4); B = np.eye(4)
        A[:3, :3] = Rotation.from_euler("yxz", rng.uniform(-3, 3, 3)).as_matrix(); A[:3, 3] = rng.uniform(-10, 10, 3)
        d = Rotation.from_euler("xzy", rng.normal(0, 0.05 if i % 2 else 0.5, 3)).as_matrix()
        B[:3, :3] = A[:3, :3] @ d; B[:3, 3] = A[:3, 3] + rng.normal(0, 1.0 if i % 2 else 3.0, 3)
        Pp.append(A); Pg.append(B)
    out = frustum.pose_error_batch(np.stack(Pp), np.stack(Pg))
    te, re, ok = out["t_err"].cpu().numpy(), out["r_err"].cpu().numpy(), out["success"].cpu().numpy()
    for i in range(64):
        t_want, r_want = oracle.pose_diff(Pp[i], Pg[i])
        assert abs(te[i] - t_want) < 1e-9 and abs(re[i] - r_want) < 1e-7, (i, te[i], t_want, re[i], r_want)
        assert ok[i] == int(t_want < 2 and r_want < 5)
    assert abs(out["success_rate"].item() - ok.mean()) < 1e-12
    assert 0 < ok.sum() < 64


def test_register_directory_legacy_handoff(cuda, tmp_path):
    """8(f) N2: a directory in the reference's file-triple layout gives the same poses as the in-memory
    contract, plus the result files and summary of registration_lsq.py:396-398 / registration_result_analysis.py."""
    from deepi2p_b200 import handoff

    S, n = 5, 2048
    samples = [small_sample(700 + s, n) for s in range(S)]
    for s, smp in enumerate(samples):
        handoff.save_record(str(tmp_path / "data"), "%06d_%02d" % (s * 30, 0), smp["points"], smp["pred"], smp["gt"],
                            smp["pred"], smp["gt"], smp["K"], smp["P_gt"][:3])
    res = handoff.register_directory(str(tmp_path / "data"), syn.KITTI["H"], syn.KITTI["W"], n_inits=12, seed=3,
                                     out_dir=str(tmp_path / "out"))
    xyz = torch.from_numpy(np.stack([smp["points"].astype(np.float32) for smp in samples])).cuda()
    pred = torch.from_numpy(np.stack([smp["pred"].astype(np.int8) for smp in samples])).cuda()
    K = np.stack([smp["K"].reshape(9) for smp in samples])
    ref = frustum.register_batch(xyz, pred, n, K, syn.KITTI["H"], syn.KITTI["W"], n_inits=12, seed=3)
    np.testing.assert_array_equal(res["P_pred"], ref["P"].cpu().numpy())
    np.testing.assert_array_equal(res["cost"], ref["cost"].cpu().numpy())
    np.testing.assert_array_equal(np.load(tmp_path / "out" / "P_pred_all_np.npy"), res["P_pred"])
    np.testing.assert_array_equal(np.load(tmp_path / "out" / "P_gt_all_np.npy"),
                                  np.stack([smp["P_gt"] for smp in samples]))
    for s, smp in enumerate(samples):
        t, r = oracle.pose_diff(res["P_pred"][s], smp["P_gt"])
        assert abs(t - res["t_err"][s]) < 1e-9 and abs(r - res["r_err"][s]) < 1e-7
    sm = res["summary"]
    assert sm["n"] == S and 0.0 <= sm["success_rate"] <= 1.0 and np.isfinite(sm["rte_mean"])


@pytest.mark.parametrize("is_2d", [True, False])
def test_committed_golden_vectors(cuda, is_2d):
    """CUDA path against tests/golden/frustum_small.npz (oracle outputs committed with their generating script):
    evaluations to the same tolerance as test_evaluate_matches_oracle, solves statistically (see
    test_solve_matches_oracle for why)."""
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "frustum_small.npz"))
    S, I, H, W = int(g["S"]), int(g["I"]), float(g["H"]), float(g["W"])
    P = 4 if is_2d else 6
    xyz, lab, n_pts = frustum.pack_clouds(g["points"], g["pred"])
    K = g["K"].reshape(S, 9)
    x = np.zeros((S, 6))
    x[:, :P] = g["x4"] if is_2d else g["x6"]
    c, gr, A = frustum.evaluate_batch(xyz, lab, n_pts, K, x, H, W, is_2d)
    ev = g["eval4"] if is_2d else g["eval6"]
    for s in range(S):
        co, go, Ao = ev[s, 0], ev[s, 1:1 + P], ev[s, 1 + P:].reshape(P, P)
        assert abs(c[s].item() - co) <= 1e-10 * max(1.0, abs(co))
        np.testing.assert_allclose(gr[s].cpu().numpy(), go, rtol=1e-9, atol=1e-9 * np.abs(go).max())
        np.testing.assert_allclose(A[s].cpu().numpy(), Ao, rtol=1e-9, atol=1e-9 * np.abs(Ao).max())
    out = frustum.solve_batch(xyz, lab, n_pts, K, g["inits"], H, W, syn.T_LB, syn.T_UB, 500, is_2d, return_all=True)
    params = out["params"].cpu().numpy()
    sol = g["solve4"] if is_2d else g["solve6"]
    nr = P - 3
    d_rot = np.linalg.norm(params[:, :, :nr] - sol[:, :, :nr], axis=2)
    d_tr = np.linalg.norm(params[:, :, nr:P] - sol[:, :, nr:P], axis=2)
    within = (d_rot < ROT_TOL) & (d_tr < TRANS_TOL)
    print("golden solves within gate %d/%d" % (within.sum(), within.size))
    assert within.sum() >= within.size - 1        # the fixture's solves were picked stable under a 1e-13 input change
    costs = out["costs"].cpu().numpy()
    assert np.all(np.abs(costs[within] - sol[:, :, 6][within]) <= 1e-5 * np.maximum(1.0, sol[:, :, 6][within]))
