"""Throughput of the PnP-RANSAC path (deepi2p_b200.pnp.pnp_ransac_batch) on KITTI-shaped synthetic frames.

    python scripts/bench_pnp.py [--frames 4096] [--reps 3] [--out FILE.json]

Frames: synthetic.make_sample (20480 points, about 4700 predicted inside) with make_fine_labels (30 % random cells);
64 distinct frames are tiled to the batch size.  Prints one JSON line: frames/s at S = --frames, latency at S = 1,
success rate (2 m / 5 deg) against GT, and a cv2.solvePnPRansac CPU baseline on the same frames when OpenCV imports.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepi2p_b200 import frustum, pnp, synthetic  # noqa: E402


def _time(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) / 1e3)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    uniq = [synthetic.make_sample(s) for s in range(64)]
    ufine = [synthetic.make_fine_labels(s, seed=i) for i, s in enumerate(uniq)]
    S = a.frames
    xyz, c8, f32, n_pts = pnp.pack_frames([uniq[s % 64]["points"] for s in range(S)],
                                          [uniq[s % 64]["pred"] for s in range(S)], [ufine[s % 64] for s in range(S)])
    K, H, W = uniq[0]["K"], uniq[0]["H"], uniq[0]["W"]
    res = {}
    out = pnp.pnp_ransac_batch(xyz, c8, f32, n_pts, K, H, W)
    t_big = _time(lambda: pnp.pnp_ransac_batch(xyz, c8, f32, n_pts, K, H, W, out=out), a.reps)
    x1, c1, f1, n1 = xyz[:1].contiguous(), c8[:1].contiguous(), f32[:1].contiguous(), n_pts[:1].contiguous()
    o1 = pnp.pnp_ransac_batch(x1, c1, f1, n1, K, H, W)
    t_one = _time(lambda: pnp.pnp_ransac_batch(x1, c1, f1, n1, K, H, W, out=o1), max(a.reps, 5))
    P = out["P"][:64].cpu().numpy()
    err = frustum.pose_error_batch(P, np.stack([u["P_gt"] for u in uniq]))
    res.update(frames=S, mean_selected=float(out["n_sel"].float().mean()),
               mean_hypotheses=float(out["hyp_used"].float().mean()), seconds=t_big, frames_per_s=S / t_big,
               latency_s1_ms=t_one * 1e3, success_rate=float(err["success"].float().mean()),
               gpu=torch.cuda.get_device_name(0))
    try:
        import cv2
        n_cv, t_cv, ok_cv = 64, 0.0, 0
        for i in range(n_cv):
            u, f = uniq[i], ufine[i]
            m = u["pred"] == 1
            Ks = K / 32.0
            Ks[2, 2] = 1
            py = np.floor(f[m] / (W / 32.0))
            pix = np.stack((f[m] - py * (W / 32.0), py)).astype(np.float64)
            t0 = time.perf_counter()
            good, rv, tv, inl = cv2.solvePnPRansac(u["points"][:, m].T.astype(np.float64), pix.T, Ks, None,
                                                   iterationsCount=500, reprojectionError=0.6, flags=cv2.SOLVEPNP_EPNP)
            t_cv += time.perf_counter() - t0
            Pc = np.eye(4)
            if good and np.linalg.norm(tv) < 14.14:
                Pc[:3, :3] = cv2.Rodrigues(rv)[0]
                Pc[:3, 3] = tv[:, 0]
            ok_cv += int(frustum.pose_error_batch(Pc[None], u["P_gt"][None])["success"][0])
        res["cv2_cpu"] = dict(frames=n_cv, ms_per_frame=1e3 * t_cv / n_cv, success_rate=ok_cv / n_cv)
    except ImportError:
        res["cv2_cpu"] = "not available"
    line = json.dumps(dict(pnp=res))
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
