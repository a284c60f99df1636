"""Write tests/golden/pnp_small.npz: fixtures of the PnP-RANSAC path that do not need OpenCV or the oracle at test time.

    python tests/golden/make_pnp_golden.py        # needs cv2 (OpenCV) and the built oracle_pnp

The tests import this module only for the frame definitions below; OpenCV is imported when writing the file.

Contents:
  oracle_*   8 small frames (make_sample(700+i, 1024) + make_fine_labels, 200 iterations, seed 5): inputs and the
             oracle's n_sel, hyp_used, winner, per-hypothesis poses / counts, final P and outlier ratio
  epnp_*     noise-free point sets (6, 50 and 1000 points, general and near-planar) packed with offsets, and
             cv2.solvePnP(SOLVEPNP_EPNP) on each (R row-major | t)
  cv2r_*     cv2.solvePnPRansac (EPNP, 500 iterations, 0.6 px, registration_pnp.py:125-132) on 64 frames
             make_sample(800+i, 8192) + make_fine_labels(seed=i): P, outlier ratio, success (2 m / 5 deg)
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import oracle_pnp  # noqa: E402
from deepi2p_b200 import synthetic  # noqa: E402

ORACLE_FRAMES, ORACLE_N, ORACLE_ITERS, ORACLE_SEED = 8, 1024, 200, 5
CV2_FRAMES, CV2_N = 64, 8192
KF = np.array([[353.5 / 32, 0.0, 250.5 / 32], [0.0, 353.5 / 32, 66.5 / 32], [0.0, 0.0, 1.0]])


def oracle_frames():
    smps = [synthetic.make_sample(700 + i, ORACLE_N) for i in range(ORACLE_FRAMES)]
    return smps, [synthetic.make_fine_labels(s, seed=i) for i, s in enumerate(smps)]


def cv2_frames():
    smps = [synthetic.make_sample(800 + i, CV2_N) for i in range(CV2_FRAMES)]
    return smps, [synthetic.make_fine_labels(s, seed=i) for i, s in enumerate(smps)]


def success(P, P_gt):
    D = np.linalg.inv(P) @ P_gt
    c = np.clip((np.trace(D[:3, :3]) - 1) / 2, -1, 1)
    return bool(np.linalg.norm(D[:3, 3]) < 2.0 and np.degrees(np.arccos(c)) < 5.0)


def epnp_sets():
    import cv2
    rng = np.random.default_rng(12)
    sets = []
    for n in (6, 50, 1000):
        for trial in range(8):
            a = rng.normal(size=3) * 0.3
            R = cv2.Rodrigues(a)[0]
            t = np.array([rng.uniform(-2, 2), rng.uniform(-1, 1), rng.uniform(5, 10)])
            Xc = np.stack([rng.uniform(-4, 4, n), rng.uniform(-2, 2, n), rng.uniform(4, 20, n)], 1)
            if trial % 4 == 3:
                Xc[:, 1] = 0.5 * Xc[:, 0] + 0.01 * rng.normal(size=n)
            uv = Xc[:, :2] / Xc[:, 2:3] * np.array([KF[0, 0], KF[1, 1]]) + np.array([KF[0, 2], KF[1, 2]])
            sets.append(((Xc - t) @ R, uv))
    return sets


def main():
    import cv2
    out = {}
    smps, fines = oracle_frames()
    out["oracle_xyz"] = np.stack([s["points"] for s in smps])
    out["oracle_coarse"] = np.stack([s["pred"] for s in smps]).astype(np.int8)
    out["oracle_fine"] = np.stack(fines)
    out["oracle_K"] = smps[0]["K"]
    hp = np.zeros((ORACLE_FRAMES, ORACLE_ITERS, 12))
    hi = np.zeros((ORACLE_FRAMES, ORACLE_ITERS), np.int32)
    ints = np.zeros((ORACLE_FRAMES, 4), np.int32)
    P = np.zeros((ORACLE_FRAMES, 4, 4))
    ratio = np.zeros(ORACLE_FRAMES)
    for s, (smp, f) in enumerate(zip(smps, fines)):
        r = oracle_pnp.ransac_frame(smp["points"], smp["pred"], f, smp["K"], smp["H"], smp["W"], s=s,
                                    iterations=ORACLE_ITERS, seed=ORACLE_SEED)
        u = r["hyp_used"]
        hp[s, :u], hi[s, :u] = r["hyp_pose"], r["hyp_inliers"]
        ints[s] = (r["n_sel"], u, r["winner"], r["inliers"])
        P[s], ratio[s] = r["P"], r["outlier_ratio"]
    out.update(oracle_hyp_pose=hp, oracle_hyp_inliers=hi, oracle_ints=ints, oracle_P=P, oracle_ratio=ratio)

    sets = epnp_sets()
    offs = np.zeros(len(sets) + 1, np.int32)
    for b, (x, _) in enumerate(sets):
        offs[b + 1] = offs[b] + len(x)
    pose = np.zeros((len(sets), 12))
    for b, (x, u) in enumerate(sets):
        ok, rv, tv = cv2.solvePnP(x, u, KF, None, flags=cv2.SOLVEPNP_EPNP)
        assert ok
        pose[b, :9], pose[b, 9:] = cv2.Rodrigues(rv)[0].reshape(9), tv[:, 0]
    out.update(epnp_xyz=np.concatenate([x for x, _ in sets]), epnp_uv=np.concatenate([u for _, u in sets]),
               epnp_offsets=offs, epnp_K=KF, epnp_cv2_pose=pose)

    smps, fines = cv2_frames()
    Pc = np.zeros((CV2_FRAMES, 4, 4))
    rc = np.ones(CV2_FRAMES)
    okc = np.zeros(CV2_FRAMES, np.int32)
    for i, (u, f) in enumerate(zip(smps, fines)):        # registration_pnp.py:95-148 with the reference's call
        m = u["pred"] == 1
        W = u["W"] / 32.0
        py = np.floor(f[m] / W)
        pix = np.stack((f[m] - py * W, py)).astype(np.float64)
        Ks = u["K"] / 32.0
        Ks[2, 2] = 1
        Pc[i] = np.eye(4)
        if m.sum() >= 4:
            good, rv, tv, inl = cv2.solvePnPRansac(u["points"][:, m].T.astype(np.float64), pix.T, Ks, None,
                                                   useExtrinsicGuess=False, iterationsCount=500,
                                                   reprojectionError=0.6, flags=cv2.SOLVEPNP_EPNP)
            if good and np.linalg.norm(tv) < 14.14:
                Pc[i, :3, :3], Pc[i, :3, 3] = cv2.Rodrigues(rv)[0], tv[:, 0]
                rc[i] = 1 - len(inl) / m.sum()
        okc[i] = success(Pc[i], u["P_gt"])
    out.update(cv2r_P=Pc, cv2r_ratio=rc, cv2r_success=okc)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pnp_small.npz")
    np.savez_compressed(path, **out)
    print(path, "cv2 RANSAC success %d/%d" % (okc.sum(), CV2_FRAMES))


if __name__ == "__main__":
    main()
