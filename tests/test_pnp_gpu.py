"""PnP-RANSAC path on the GPU (deepi2p_b200.pnp) against the CPU oracle (oracle_pnp).

The oracle restates the kernels' arithmetic order (warp-order sums, the parallel Jacobi ordering, no FMA), so the
comparison is exact: selection / decoding, the sampled indices and every hypothesis pose, per-hypothesis inlier
counts, the stopping replay, the winner, the refit pose, the inlier mask, plus run-to-run and cross-stream bit
identity.  (The one place the two sides could part is the stopping rule's log, should it land within an ulp of an
integer; no such frame occurs in these inputs.)"""
import numpy as np
import pytest
import torch

import oracle_pnp
from deepi2p_b200 import pnp, synthetic

pytestmark = pytest.mark.gpu

SCALE = 1 / 32.0


def _frames(seeds, n_points=4096, noise=0.3):
    smps = [synthetic.make_sample(s, n_points) for s in seeds]
    fines = [synthetic.make_fine_labels(s, SCALE, noise, seed=i) for i, s in zip(seeds, smps)]
    return smps, fines


def _run(smps, fines, **kw):
    xyz, c8, f32, n_pts = pnp.pack_frames([s["points"] for s in smps], [s["pred"] for s in smps], fines)
    K = np.stack([s["K"] for s in smps])
    out = pnp.pnp_ransac_batch(xyz, c8, f32, n_pts, K, smps[0]["H"], smps[0]["W"], return_all=True, **kw)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}, (xyz, c8, f32, n_pts, K)


def _oracle(smps, fines, **kw):
    return [oracle_pnp.ransac_frame(s["points"], s["pred"], f, s["K"], s["H"], s["W"], s=i, **kw)
            for i, (s, f) in enumerate(zip(smps, fines))]


@pytest.fixture(scope="module")
def batch():
    smps, fines = _frames(range(500, 524))
    g, _ = _run(smps, fines, seed=11)
    o = _oracle(smps, fines, seed=11)
    return smps, fines, g, o


def test_selection_and_stopping_match_oracle(batch):
    smps, fines, g, o = batch
    same_winner = 0
    hyp_total = hyp_same = 0
    for s, r in enumerate(o):
        assert g["n_sel"][s] == r["n_sel"]
        used = r["hyp_used"]
        gi = g["hyp_inliers"][s, :used]
        hyp_same += int((gi == r["hyp_inliers"]).sum())
        hyp_total += used
        if np.array_equal(gi, r["hyp_inliers"]):
            # equal counts -> the sequential replay must give the same number of hypotheses and the same winner
            assert g["hyp_used"][s] == used
            assert g["inliers"][s] == r["inliers"]
        same_winner += int(g["hyp_used"][s] == used and g["inliers"][s] == r["inliers"])
    print("hypotheses with identical counts %d/%d, frames with the same winner %d/%d"
          % (hyp_same, hyp_total, same_winner, len(o)))
    assert hyp_same == hyp_total
    assert same_winner == len(o)


def test_hypothesis_poses_match_oracle(batch):
    """Same Philox samples -> the same minimal problems -> bit-identical hypothesis poses."""
    smps, fines, g, o = batch
    diffs = []
    for s, r in enumerate(o):
        used = r["hyp_used"]
        a, b = g["hyp_pose"][s, :used], r["hyp_pose"]
        valid = (r["hyp_inliers"] > 0) & (g["hyp_inliers"][s, :used] > 0)
        d = np.abs(a - b).max(axis=1) / np.maximum(1.0, np.abs(b).max(axis=1))
        diffs.append(d[valid])
    d = np.concatenate(diffs)
    print("hypothesis pose rel diff: median %.2e p99 %.2e max %.2e (n=%d)" % (np.median(d), np.quantile(d, 0.99),
                                                                            d.max(), d.size))
    assert d.max() == 0.0


def test_final_pose_and_ratio_match_oracle(batch):
    smps, fines, g, o = batch
    for s, r in enumerate(o):
        assert np.array_equal(g["P"][s], r["P"]), s
        assert g["outlier_ratio"][s] == r["outlier_ratio"]
        assert np.array_equal(g["inlier_mask"][s, :len(r["mask"])], r["mask"])
        assert not g["inlier_mask"][s, len(r["mask"]):].any()


def test_run_to_run_and_streams_bit_identical(batch):
    smps, fines, g, _ = batch
    g2, args = _run(smps, fines, seed=11)
    for k in g:
        assert np.array_equal(g[k], g2[k]), k
    xyz, c8, f32, n_pts, K = args
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        out = pnp.pnp_ransac_batch(xyz, c8, f32, n_pts, K, smps[0]["H"], smps[0]["W"], seed=11, return_all=True,
                                   stream=side)
    side.synchronize()
    out2 = pnp.pnp_ransac_batch(xyz, c8, f32, n_pts, K, smps[0]["H"], smps[0]["W"], seed=11, return_all=True, out=out)
    assert out2 is out
    torch.cuda.synchronize()
    for k in ("P", "outlier_ratio", "inliers", "hyp_used", "inlier_mask"):
        assert np.array_equal(out[k].cpu().numpy(), g[k]), k


def test_edge_rules():
    """n < 4 -> identity; 4 <= n <= 5 -> EPnP on all points; far-away solutions -> identity; ragged n_pts."""
    rng = np.random.default_rng(3)
    K = synthetic.KITTI["K"]
    H, W = 160, 512
    frames = []
    for n_in in (0, 3, 4, 5, 6, 40):
        pts = np.stack([rng.uniform(-4, 4, 50), rng.uniform(-2, 1, 50), rng.uniform(5, 30, 50)]).astype(np.float32)
        coarse = np.zeros(50, np.int32)
        coarse[:n_in] = 1
        fine = rng.integers(0, 16 * 5, 50).astype(np.int32)
        frames.append((pts, coarse, fine))
    smps = [dict(points=p, pred=c, K=K, H=H, W=W) for p, c, _ in frames]
    fines = [f for _, _, f in frames]
    g, _ = _run(smps, fines, seed=5)
    o = _oracle(smps, fines, seed=5)
    for s, r in enumerate(o):
        assert g["n_sel"][s] == r["n_sel"] == min(frames[s][1].sum(), 50)
        if r["n_sel"] < 4:
            assert np.array_equal(g["P"][s], np.eye(4)) and g["outlier_ratio"][s] == 1.0 and g["inliers"][s] == 0
        if r["n_sel"] <= 5:
            assert g["hyp_used"][s] == 0
        assert g["hyp_used"][s] == r["hyp_used"] and g["inliers"][s] == r["inliers"]
        assert np.array_equal(g["P"][s], r["P"]) and g["outlier_ratio"][s] == r["outlier_ratio"]


def test_far_solution_is_rejected():
    """|t| >= 14.14 -> P = I and outlier_ratio = 1, as in the oracle (scale 1: one cell per pixel)."""
    rng = np.random.default_rng(4)
    K, W, H = synthetic.KITTI["K"], 512, 160
    Xc = np.stack([rng.uniform(-10, 10, 400), rng.uniform(-3, 3, 400), rng.uniform(30, 60, 400)])
    Xw = (Xc - np.array([[0.0], [0.0], [40.0]])).astype(np.float32)
    u, v = K[0, 0] * Xc[0] / Xc[2] + K[0, 2], K[1, 1] * Xc[1] / Xc[2] + K[1, 2]
    fine = (np.floor(u) + np.floor(v) * W).astype(np.int32)
    smps = [dict(points=Xw, pred=np.ones(400, np.int32), K=K, H=H, W=W)]
    g, _ = _run(smps, [fine], scale=1.0)
    r = _oracle(smps, [fine], scale=1.0)[0]
    assert r["inliers"] > 100 and g["inliers"][0] == r["inliers"]
    assert np.array_equal(g["P"][0], np.eye(4)) and g["outlier_ratio"][0] == 1.0


def test_single_frame_and_solve_pnp_signature():
    smps, fines = _frames([77], n_points=20480)
    s = smps[0]
    P, ratio = pnp.solve_pnp(s["points"], s["pred"], fines[0], s["K"], s["H"], s["W"], SCALE, 500, 1)
    r = oracle_pnp.ransac_frame(s["points"], s["pred"], fines[0], s["K"], s["H"], s["W"])
    assert np.array_equal(P, r["P"]) and ratio == r["outlier_ratio"]
    with pytest.raises(ValueError):
        pnp.solve_pnp(s["points"], s["pred"], fines[0], s["K"], s["H"], s["W"], SCALE, 500, 0)


def test_epnp_hook_matches_oracle():
    rng = np.random.default_rng(9)
    K = np.array([[11.0, 0, 7.8], [0, 11.0, 2.1], [0, 0, 1]])
    sets = []
    for n in (5, 6, 50, 2000):
        for _ in range(20):
            Xc = np.stack([rng.uniform(-4, 4, n), rng.uniform(-2, 2, n), rng.uniform(4, 20, n)], 1)
            uv = Xc[:, :2] / Xc[:, 2:3] * 11.0 + np.array([7.8, 2.1]) + rng.normal(size=(n, 2)) * 0.05
            sets.append((Xc + rng.normal(size=3), uv))
    pose, ok = pnp.epnp_batch(sets, K)
    for b, (x, u) in enumerate(sets):
        ok_o, R, t = oracle_pnp.epnp(x, u, K)
        assert ok[b] == ok_o
        if ok_o:
            ref = np.concatenate([R.reshape(9), t])
            assert np.array_equal(pose[b], ref), b


def test_large_batch_runs():
    """S = 4096 frames (64 distinct ones tiled, ~450 selected points each): every frame is selected and solved, and
    the first 64 frames equal the oracle exactly."""
    n = 2048
    S = 4096
    smps = [synthetic.make_sample(1000 + (s % 64), n) for s in range(64)]
    fines = [synthetic.make_fine_labels(smps[s], SCALE, 0.3, seed=s) for s in range(64)]
    xyz, c8, f32, n_pts = pnp.pack_frames([smps[s % 64]["points"] for s in range(S)],
                                          [smps[s % 64]["pred"] for s in range(S)], [fines[s % 64] for s in range(S)])
    out = pnp.pnp_ransac_batch(xyz, c8, f32, n_pts, smps[0]["K"], smps[0]["H"], smps[0]["W"], seed=1)
    torch.cuda.synchronize()
    res = {k: v.cpu().numpy() for k, v in out.items()}
    assert (res["n_sel"] == np.array([int((smps[s % 64]["pred"] == 1).sum()) for s in range(S)])).all()
    assert np.isfinite(res["P"]).all()
    for s, r in enumerate(_oracle(smps, fines, seed=1)):
        assert res["hyp_used"][s] == r["hyp_used"] and res["inliers"][s] == r["inliers"], s
        assert np.array_equal(res["P"][s], r["P"]) and res["outlier_ratio"][s] == r["outlier_ratio"], s


def test_ragged_batch_matches_oracle():
    """Frames of different sizes in one batch (n_pts < stride), including frames with fewer than 4 points next to
    full ones, each equal to the oracle on its own points."""
    sizes = [20480, 3, 0, 4096, 5, 777, 2, 12000]
    smps = [synthetic.make_sample(300 + i, max(n, 1)) for i, n in enumerate(sizes)]
    pts, pred, fines = [], [], []
    for s, n in zip(smps, sizes):
        p, c = s["points"][:, :n], s["pred"][:n].copy()
        if n < 6:
            c[:] = 1
        pts.append(p)
        pred.append(c)
        fines.append(synthetic.make_fine_labels(s, SCALE, 0.3, seed=n)[:n])
    xyz, c8, f32, n_pts = pnp.pack_frames(pts, pred, fines)
    assert n_pts.cpu().tolist() == sizes
    K = smps[0]["K"]
    out = pnp.pnp_ransac_batch(xyz, c8, f32, n_pts, K, 160, 512, seed=2, return_all=True)
    torch.cuda.synchronize()
    g = {k: v.cpu().numpy() for k, v in out.items()}
    for s in range(len(sizes)):
        r = oracle_pnp.ransac_frame(pts[s], pred[s], fines[s], K, 160, 512, s=s, seed=2)
        assert g["n_sel"][s] == r["n_sel"] == int((pred[s] == 1).sum()), s
        assert g["hyp_used"][s] == r["hyp_used"] and g["inliers"][s] == r["inliers"], s
        assert np.array_equal(g["P"][s], r["P"]) and g["outlier_ratio"][s] == r["outlier_ratio"], s
        assert np.array_equal(g["inlier_mask"][s, :sizes[s]], r["mask"]) and not g["inlier_mask"][s, sizes[s]:].any()
        if sizes[s] < 4:
            assert np.array_equal(g["P"][s], np.eye(4)) and g["outlier_ratio"][s] == 1.0


# ---- tests/golden/pnp_small.npz: anchors that need neither OpenCV nor the oracle on this machine ----
import os  # noqa: E402
import sys  # noqa: E402

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pnp_small.npz")


def test_stored_oracle_frames_exact():
    import make_pnp_golden as mk
    g = np.load(GOLDEN)
    F, Nn = mk.ORACLE_FRAMES, mk.ORACLE_N
    xyz = torch.from_numpy(np.ascontiguousarray(g["oracle_xyz"])).cuda()
    c8 = torch.from_numpy(np.ascontiguousarray(g["oracle_coarse"])).cuda()
    f32 = torch.from_numpy(np.ascontiguousarray(g["oracle_fine"])).cuda()
    out = pnp.pnp_ransac_batch(xyz, c8, f32, None, g["oracle_K"], 160, 512, iterations=mk.ORACLE_ITERS,
                               seed=mk.ORACLE_SEED, return_all=True)
    torch.cuda.synchronize()
    r = {k: v.cpu().numpy() for k, v in out.items()}
    for s in range(F):
        n_sel, used, win, inl = g["oracle_ints"][s]
        assert (r["n_sel"][s], r["hyp_used"][s], r["inliers"][s]) == (n_sel, used, inl), s
        assert np.array_equal(r["hyp_inliers"][s, :used], g["oracle_hyp_inliers"][s, :used])
        assert np.array_equal(r["hyp_pose"][s, :used], g["oracle_hyp_pose"][s, :used])
        assert np.array_equal(r["P"][s], g["oracle_P"][s]) and r["outlier_ratio"][s] == g["oracle_ratio"][s]


def test_epnp_hook_against_stored_opencv_poses():
    """epnp_batch_f64 on noise-free sets equals the stored cv2.solvePnP(SOLVEPNP_EPNP) poses to 1e-9."""
    g = np.load(GOLDEN)
    offs = g["epnp_offsets"]
    sets = [(g["epnp_xyz"][offs[b]:offs[b + 1]], g["epnp_uv"][offs[b]:offs[b + 1]]) for b in range(len(offs) - 1)]
    pose, ok = pnp.epnp_batch(sets, g["epnp_K"])
    assert ok.all()
    ref = g["epnp_cv2_pose"]
    err = np.abs(pose - ref).max(axis=1) / np.maximum(1.0, np.abs(ref).max(axis=1))
    print("epnp_batch_f64 vs stored cv2: max rel diff %.1e over %d sets" % (err.max(), len(sets)))
    assert err.max() <= 1e-9


def test_success_rate_matches_stored_opencv_ransac():
    """GPU success (2 m / 5 deg rotation angle) on the 64 frames of the stored cv2.solvePnPRansac run: within 5
    percentage points of cv2's, and the mean outlier ratio within 0.05."""
    import make_pnp_golden as mk
    g = np.load(GOLDEN)
    smps, fines = mk.cv2_frames()
    out, _ = _run(smps, fines)
    ok = np.array([mk.success(out["P"][i], smps[i]["P_gt"]) for i in range(mk.CV2_FRAMES)])
    print("success: GPU %d/64, cv2 %d/64; mean outlier ratio GPU %.3f, cv2 %.3f"
          % (ok.sum(), g["cv2r_success"].sum(), out["outlier_ratio"].mean(), g["cv2r_ratio"].mean()))
    assert abs(ok.mean() - g["cv2r_success"].mean()) <= 0.05
    assert abs(out["outlier_ratio"].mean() - g["cv2r_ratio"].mean()) <= 0.05


def test_register_directory_pnp_matches_oracle(tmp_path):
    """register_dir.py --method pnp on a save_record directory: per-frame poses / costs and the summary equal the
    oracle's on the same frames (the batch seed of frame i is seed + batch start, its frame index within the batch)."""
    import json
    import subprocess
    from test_handoff_pnp_cpu import write_pnp_dir
    from deepi2p_b200 import frustum, handoff
    recs = write_pnp_dir(tmp_path / "data")
    res = handoff.register_directory_pnp(str(tmp_path / "data"), 160, 512, seed=4, batch=3,
                                         out_dir=str(tmp_path / "out"))
    P_o, cost_o = [], []
    for i, (name, smp, fine) in enumerate(recs):
        a = i // 3 * 3
        r = oracle_pnp.ransac_frame(smp["points"], smp["pred"], fine, smp["K"], 160, 512, s=i - a, seed=4 + a)
        P_o.append(r["P"])
        cost_o.append(r["outlier_ratio"])
    assert np.array_equal(res["P_pred"], np.stack(P_o)) and np.array_equal(res["cost"], np.array(cost_o))
    assert np.array_equal(np.load(tmp_path / "out" / "cost_all_np.npy"), np.array(cost_o))
    err = frustum.pose_error_batch(np.stack(P_o), np.stack([s["P_gt"] for _, s, _ in recs]))
    expect = handoff.summarize(err["t_err"].cpu().numpy(), err["r_err"].cpu().numpy(), np.array(cost_o),
                               err["success"].cpu().numpy())
    assert res["summary"] == expect
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cli = subprocess.run([sys.executable, os.path.join(root, "scripts", "register_dir.py"), str(tmp_path / "data"),
                          "--H", "160", "--W", "512", "--method", "pnp", "--seed", "4", "--batch", "3"],
                         capture_output=True, text=True, check=True)
    assert json.loads(cli.stdout.strip().splitlines()[-1]) == json.loads(json.dumps(expect))
