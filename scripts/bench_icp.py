"""Throughput of the ICP path (deepi2p_b200.icp.icp_register_batch) on Oxford-shaped synthetic frames.

    python scripts/bench_icp.py [--frames 64] [--inits 60] [--reps 3] [--cpu-frames 1] [--out FILE.json]

Frames: synthetic.make_icp_frame (20480 LiDAR points, a 640 x 384 depth cloud = 245,760 points), scale-calibrated as
registration_icp.py:215-218 does; 8 distinct frames are tiled to the batch size.  max_iteration 30, 60 inits.  Prints
one JSON line: frames/s at S = --frames, latency at S = 1, the index build alone at S = --frames and S = 1 (CUDA
events around icp_build_index_f32, which runs exactly the build launches of a call), mean update steps per problem,
nearest-neighbour queries/s and mean point distance evaluations per query (device counters of a counted call),
success rate (2 m / 5 deg) against GT, the GPU and its power limit, and a CPU baseline: the oracle on all host cores
over --cpu-frames frames (and Open3D's registration_icp when it imports).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepi2p_b200 import handoff, icp, synthetic  # noqa: E402


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


def _power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--inits", type=int, default=60)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--cpu-frames", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    uniq = [synthetic.make_icp_frame(s, "oxford") for s in range(8)]
    srcs = [u["src"] for u in uniq]
    tgts = [(u["tgt"] * icp.calibrate_scale(u["src"], u["P_gt"], u["K"], u["H"], u["W"], u["tgt"])).astype(np.float32)
            for u in uniq]
    S, I = a.frames, a.inits
    src, n = icp.pack_clouds([srcs[s % 8] for s in range(S)])
    tgt, m = icp.pack_clouds([tgts[s % 8] for s in range(S)])
    init = torch.from_numpy(icp.random_inits(S, I, seed=0)).cuda()
    out = icp.icp_register_batch(src, n, tgt, m, init, return_all=True)
    counters = torch.zeros(2, dtype=torch.int64, device=src.device)
    icp.icp_register_batch(src, n, tgt, m, init, return_all=True, out=out, counters=counters)
    queries, evals = (int(v) for v in counters.cpu().tolist())
    t_big = _time(lambda: icp.icp_register_batch(src, n, tgt, m, init, return_all=True, out=out), a.reps)
    s1, n1, t1, m1, i1 = (x[:1].contiguous() for x in (src, n, tgt, m, init))
    o1 = icp.icp_register_batch(s1, n1, t1, m1, i1)
    t_one = _time(lambda: icp.icp_register_batch(s1, n1, t1, m1, i1, out=o1), max(a.reps, 5))
    t_build = _time(lambda: icp.build_index(tgt, m), max(a.reps, 5))
    t_build1 = _time(lambda: icp.build_index(t1, m1), max(a.reps, 5))
    steps = out["stats"][..., 0].double()
    P = out["P"][:8].cpu().numpy()
    t_err, r_err = handoff.get_p_diff(P, np.stack([u["P_gt"] for u in uniq]))
    res = dict(frames=S, inits=I, target_points=int(m[0]), source_points=int(n[0]), seconds=t_big,
               frames_per_s=S / t_big, latency_s1_ms=t_one * 1e3,
               index_build_ms=t_build * 1e3, index_build_s1_ms=t_build1 * 1e3,
               mean_update_steps=float(steps.mean()), nn_queries_per_s=queries / t_big,
               evals_per_query=evals / max(queries, 1),
               success_rate=float(((t_err < 2.0) & (r_err < 5.0)).mean()), gpu=torch.cuda.get_device_name(0),
               power_limit=_power_limit())
    import oracle_icp
    t0 = time.perf_counter()
    for f in range(a.cpu_frames):
        oracle_icp.register_frame(srcs[f], tgts[f], icp.random_inits(1, I, seed=f)[0])
    res["oracle_cpu"] = dict(frames=a.cpu_frames, cores=os.cpu_count(),
                             s_per_frame=(time.perf_counter() - t0) / max(a.cpu_frames, 1))
    try:
        import open3d as o3d
        reg = o3d.pipelines.registration
        t0 = time.perf_counter()
        sp, tp = o3d.geometry.PointCloud(), o3d.geometry.PointCloud()
        sp.points = o3d.utility.Vector3dVector(srcs[0].T.astype(np.float64))
        tp.points = o3d.utility.Vector3dVector(tgts[0].T.astype(np.float64))
        for T0 in icp.random_inits(1, I, seed=0)[0]:
            reg.registration_icp(sp, tp, 1.0, T0, reg.TransformationEstimationPointToPoint())
        res["open3d_cpu"] = dict(frames=1, s_per_frame=time.perf_counter() - t0)
    except ImportError:
        res["open3d_cpu"] = "not available"
    line = json.dumps(dict(icp=res))
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
