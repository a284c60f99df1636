"""PnP-RANSAC contract on the CPU: the oracle (oracle_pnp) against cv2.solvePnP(SOLVEPNP_EPNP) where OpenCV is
installed, the stopping rule, the reference's edge rules, and the host-side argument checks of the C ABI."""
import ctypes

import numpy as np
import pytest

import oracle_pnp
from deepi2p_b200 import _native, pnp, synthetic

KF = np.array([[353.5 / 32, 0.0, 250.5 / 32], [0.0, 353.5 / 32, 66.5 / 32], [0.0, 0.0, 1.0]])


def _rot(rng, amp=0.3):
    a = rng.normal(size=3) * amp
    th = np.linalg.norm(a)
    k = a / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def _problem(rng, n, noise, planar=False):
    R = _rot(rng)
    t = np.array([rng.uniform(-2, 2), rng.uniform(-1, 1), rng.uniform(5, 10)])
    Xc = np.stack([rng.uniform(-4, 4, n), rng.uniform(-2, 2, n), rng.uniform(4, 20, n)], 1)
    if planar:
        Xc[:, 1] = 0.5 * Xc[:, 0] + 0.01 * rng.normal(size=n)       # near-planar: thin slab
    Xw = (Xc - t) @ R
    uv = Xc[:, :2] / Xc[:, 2:3] * np.array([KF[0, 0], KF[1, 1]]) + np.array([KF[0, 2], KF[1, 2]])
    return Xw, uv + rng.normal(size=uv.shape) * noise, R, t


def test_epnp_noise_free_recovers_pose():
    rng = np.random.default_rng(1)
    for n in (6, 50, 5000):
        for _ in range(20):
            Xw, uv, R, t = _problem(rng, n, 0.0)
            ok, Ro, to = oracle_pnp.epnp(Xw, uv, KF)
            assert ok
            assert np.abs(Ro - R).max() < 1e-9 and np.abs(to - t).max() < 1e-9 * max(1.0, np.linalg.norm(t))


def test_epnp_against_opencv():
    """Noise-free sets of 6 or more points (general and near-planar) agree with cv2 to 1e-9 (5 points leave EPnP a
    two-dimensional null space, where the two implementations may settle on different solutions).  With 0.05 px pixel noise the two EPnP
    implementations differ at the 1e-3 level (neither is closer to the truth); that distribution is printed and
    only bounded loosely."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(2)
    exact, noisy = [], []
    for n in (5, 6, 50, 5000):
        for trial in range(400 if n < 5000 else 40):
            for noise, bucket in ((0.0, exact), (0.05, noisy)):
                Xw, uv, R, t = _problem(rng, n, noise, planar=(trial % 4 == 3))
                ok, Ro, to = oracle_pnp.epnp(Xw, uv, KF)
                ok2, rv, tv = cv2.solvePnP(Xw, uv, KF, None, flags=cv2.SOLVEPNP_EPNP)
                if not (ok and ok2):
                    continue
                Rc = cv2.Rodrigues(rv)[0]
                bucket.append((n, max(np.abs(Ro - Rc).max(), np.abs(to - tv[:, 0]).max() / np.linalg.norm(tv))))
    e = np.array([d for n, d in exact if n >= 6])
    e5 = np.array([d for n, d in exact if n == 5])
    z = np.array([d for _, d in noisy])
    print("noise-free (n>=6): median %.1e p99 %.1e max %.1e (%d sets); n=5: median %.1e; "
          "0.05 px noise: median %.1e p99 %.1e (%d sets)" % (np.median(e), np.quantile(e, 0.99), e.max(), e.size,
                                                            np.median(e5), np.median(z), np.quantile(z, 0.99), z.size))
    assert e.size >= 800 and np.mean(e < 1e-9) >= 0.99
    assert np.median(z) < 1e-2


def test_stopping_rule_formula():
    n = 1000
    for cnt in (5, 50, 200, 500, 900, 1000):
        w = cnt / n
        den = np.log(1.0 - w ** 5)
        expect = 500 if not den < 0 else min(500, int(np.ceil(np.log(1 - 0.99) / den)))
        assert oracle_pnp.update_niters(500, cnt, n, 0.99) == expect
    assert oracle_pnp.update_niters(500, 5, 20480, 0.99) == 500       # 1 - w^5 rounds to 1: no bound
    assert oracle_pnp.update_niters(500, n, n, 0.99) == 0              # every point an inlier: stop at once
    assert oracle_pnp.update_niters(40, 300, n, 0.99) == 40            # never raises niters


def test_samples_are_distinct_and_deterministic():
    for h in range(200):
        a = oracle_pnp.sample(h, 3, 7, 42)
        assert len(set(a.tolist())) == 5 and a.min() >= 0 and a.max() < 7
        assert np.array_equal(a, oracle_pnp.sample(h, 3, 7, 42))
    assert not np.array_equal(oracle_pnp.sample(0, 0, 10 ** 6, 1), oracle_pnp.sample(0, 1, 10 ** 6, 1))


def _frame(n_sel, n=50, seed=0):
    rng = np.random.default_rng(seed)
    pts = np.stack([rng.uniform(-4, 4, n), rng.uniform(-2, 1, n), rng.uniform(5, 30, n)]).astype(np.float32)
    coarse = np.zeros(n, np.int32)
    coarse[:n_sel] = 1
    return pts, coarse, rng.integers(0, 80, n).astype(np.int32)


def test_edge_rules():
    K, H, W = synthetic.KITTI["K"], 160, 512
    for n_sel in (0, 1, 3):
        r = oracle_pnp.ransac_frame(*_frame(n_sel), K, H, W)
        assert r["n_sel"] == n_sel and np.array_equal(r["P"], np.eye(4)) and r["outlier_ratio"] == 1.0
        assert r["hyp_used"] == 0 and r["winner"] == -1
    for n_sel in (4, 5):                 # EPnP on all points, no sampling
        r = oracle_pnp.ransac_frame(*_frame(n_sel), K, H, W)
        assert r["hyp_used"] == 0 and r["winner"] == -1 and r["n_sel"] == n_sel
        if not np.array_equal(r["P"], np.eye(4)):
            assert r["outlier_ratio"] == 1.0 - r["inliers"] / n_sel
    # all hypotheses invalid: every selected point is the same point -> degenerate control points
    pts = np.ones((3, 30), np.float32)
    r = oracle_pnp.ransac_frame(pts, np.ones(30, np.int32), np.zeros(30, np.int32), K, H, W, iterations=20)
    assert r["winner"] == -1 and r["hyp_used"] == 20 and (r["hyp_inliers"] == 0).all()
    assert np.array_equal(r["P"], np.eye(4)) and r["outlier_ratio"] == 1.0


def test_far_solution_is_rejected():
    """|t| >= 14.14 -> P = I, outlier_ratio = 1 (registration_pnp.py:134)."""
    rng = np.random.default_rng(4)
    K, W, H = synthetic.KITTI["K"], 512, 160
    Xc = np.stack([rng.uniform(-10, 10, 400), rng.uniform(-3, 3, 400), rng.uniform(30, 60, 400)])
    t = np.array([0.0, 0.0, 40.0])
    Xw = (Xc - t[:, None]).astype(np.float32)          # identity rotation, |t| = 40
    q = Xw.astype(np.float64) + t[:, None]
    u, v = K[0, 0] * q[0] / q[2] + K[0, 2], K[1, 1] * q[1] / q[2] + K[1, 2]
    fine = (np.floor(u) + np.floor(v) * W).astype(np.int32)          # scale 1: one cell per pixel
    r = oracle_pnp.ransac_frame(Xw, np.ones(400, np.int32), fine, K, H, W, scale=1.0)
    assert r["winner"] >= 0 and r["inliers"] > 100
    assert np.array_equal(r["P"], np.eye(4)) and r["outlier_ratio"] == 1.0


def test_ransac_recovers_synthetic_poses():
    """Oracle RANSAC on simulated grid classifications: success (2 m / 5 deg) on a fair share of frames, and the
    decoded pixels follow the corner convention."""
    ok = 0
    for seed in range(12):
        s = synthetic.make_sample(seed, 8192)
        fine = synthetic.make_fine_labels(s, noise=0.3, seed=seed)
        r = oracle_pnp.ransac_frame(s["points"], s["pred"], fine, s["K"], s["H"], s["W"], s=seed)
        D = np.linalg.inv(r["P"]) @ s["P_gt"]
        c = np.clip((np.trace(D[:3, :3]) - 1) / 2, -1, 1)
        ok += int(np.linalg.norm(D[:3, 3]) < 2.0 and np.degrees(np.arccos(c)) < 5.0)
        assert r["n_sel"] == int((s["pred"] == 1).sum())
    assert ok >= 3, ok


def test_fine_labels_rule():
    s = synthetic.make_sample(5, 4096)
    f0 = synthetic.make_fine_labels(s, noise=0.0)
    m = s["gt"] == 1
    q = s["P_gt"][:3, :3] @ s["points"].astype(np.float64) + s["P_gt"][:3, 3:4]
    u = s["K"][0, 0] * q[0] / q[2] + s["K"][0, 2]
    v = s["K"][1, 1] * q[1] / q[2] + s["K"][1, 2]
    assert np.array_equal(f0[m], (np.floor(u[m] / 32) + np.floor(v[m] / 32) * 16).astype(np.int32))
    f1 = synthetic.make_fine_labels(s, noise=0.3, seed=1)
    assert 0.2 < np.mean(f1 != f0) < 0.35 and np.array_equal(f1, synthetic.make_fine_labels(s, noise=0.3, seed=1))


def test_solve_pnp_rejects_other_methods():
    with pytest.raises(ValueError):
        pnp.solve_pnp(np.zeros((3, 4)), np.ones(4), np.zeros(4), np.eye(3), 160, 512, 1 / 32, 500, 0)


def test_host_argument_checks():
    lib = _native.load()
    assert lib.dib_abi_version() == 4
    buf = (ctypes.c_char * 1024)()
    d = ctypes.cast(buf, ctypes.c_void_p).value
    good = dict(xyz=d, coarse=d, fine=d, n_pts=None, n_stride=16, S=1, K9=d, H=160.0, W=512.0, scale=1 / 32,
                iterations=500, thr=0.6, conf=0.99, seed=0, P=d, ratio=d, inl=d)

    def call(**kw):
        a = dict(good, **kw)
        return lib.pnp_ransac_batch_f32(a["xyz"], a["coarse"], a["fine"], a["n_pts"], a["n_stride"], a["S"], a["K9"],
                                        a["H"], a["W"], a["scale"], a["iterations"], a["thr"], a["conf"], a["seed"],
                                        a["P"], a["ratio"], a["inl"], None, None, None, None, None, d, 0, None)
    for bad in (dict(xyz=None), dict(P=None), dict(S=-1), dict(n_stride=0), dict(iterations=0), dict(W=0.0),
                dict(scale=-1.0), dict(thr=0.0), dict(conf=1.0), dict(conf=0.0), dict(S=65536)):
        assert call(**bad) == -22, bad
    assert call() == -22                  # workspace of 0 bytes is too small
    assert lib.pnp_ransac_workspace_bytes(4, 1024, 500) > lib.pnp_ransac_workspace_bytes(2, 1024, 500) > 0
    assert lib.epnp_batch_f64(None, d, d, 1, d, d, d, None) == -22
    assert lib.epnp_batch_f64(d, d, d, -1, d, d, d, None) == -22


# ---- tests/golden/pnp_small.npz (tests/golden/make_pnp_golden.py) ----
import os  # noqa: E402
import sys  # noqa: E402

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pnp_small.npz")


def test_oracle_reproduces_golden():
    import make_pnp_golden as mk
    g = np.load(GOLDEN)
    smps, fines = mk.oracle_frames()
    assert np.array_equal(np.stack(fines), g["oracle_fine"])
    assert np.array_equal(np.stack([s["points"] for s in smps]), g["oracle_xyz"])
    for s in range(mk.ORACLE_FRAMES):
        r = oracle_pnp.ransac_frame(g["oracle_xyz"][s], g["oracle_coarse"][s], g["oracle_fine"][s], g["oracle_K"],
                                    160, 512, s=s, iterations=mk.ORACLE_ITERS, seed=mk.ORACLE_SEED)
        n_sel, used, win, inl = g["oracle_ints"][s]
        assert (r["n_sel"], r["hyp_used"], r["winner"], r["inliers"]) == (n_sel, used, win, inl)
        assert np.array_equal(r["hyp_inliers"], g["oracle_hyp_inliers"][s, :used])
        assert np.array_equal(r["hyp_pose"], g["oracle_hyp_pose"][s, :used])
        assert np.array_equal(r["P"], g["oracle_P"][s]) and r["outlier_ratio"] == g["oracle_ratio"][s]


def test_oracle_epnp_against_stored_opencv_poses():
    """Noise-free sets: the oracle's EPnP equals the stored cv2.solvePnP(SOLVEPNP_EPNP) poses to 1e-9."""
    g = np.load(GOLDEN)
    offs = g["epnp_offsets"]
    for b in range(len(offs) - 1):
        ok, R, t = oracle_pnp.epnp(g["epnp_xyz"][offs[b]:offs[b + 1]], g["epnp_uv"][offs[b]:offs[b + 1]], g["epnp_K"])
        ref = g["epnp_cv2_pose"][b]
        assert ok and np.abs(np.concatenate([R.reshape(9), t]) - ref).max() <= 1e-9 * max(1.0, np.abs(ref).max()), b


def test_oracle_success_rate_matches_stored_opencv_ransac():
    """Success (2 m / 5 deg) of the oracle's RANSAC on the 64 frames the golden file holds cv2.solvePnPRansac results
    for: within 5 percentage points of cv2's (the random samples differ, so only the rate can be compared)."""
    import make_pnp_golden as mk
    g = np.load(GOLDEN)
    smps, fines = mk.cv2_frames()
    ok = np.zeros(mk.CV2_FRAMES, np.int32)
    ratio = np.zeros(mk.CV2_FRAMES)
    for i, (u, f) in enumerate(zip(smps, fines)):
        r = oracle_pnp.ransac_frame(u["points"], u["pred"], f, u["K"], u["H"], u["W"], s=i)
        ok[i] = mk.success(r["P"], u["P_gt"])
        ratio[i] = r["outlier_ratio"]
    print("success: oracle %d/64, cv2 %d/64; mean outlier ratio oracle %.3f, cv2 %.3f"
          % (ok.sum(), g["cv2r_success"].sum(), ratio.mean(), g["cv2r_ratio"].mean()))
    assert abs(ok.mean() - g["cv2r_success"].mean()) <= 0.05
    assert abs(ratio.mean() - g["cv2r_ratio"].mean()) <= 0.05
