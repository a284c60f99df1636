"""Benchmark of the Oxford RobotCar cloud build (deepi2p_b200.oxford_build) on a full-size synthetic segment: 541
returns per LMS scan at 50 Hz, 100 m windows, a cloud every 2 m, batches of S clouds.  Writes BENCH_OXFORD_BUILD.json
(or --out):

  - store load time (reading the window's .bin files into the device store) and the host plan time;
  - per-stage device times from CUDA events (plan, gather = count + scatter, voxel grid, pack), median of --reps;
  - clouds/s and input points/s with and without file I/O (with: store load + build + writing the .npy records);
  - the oracle's time per cloud on the host (single-threaded numpy / Python);
  - the card name and power limit, read in the same run.

The reference's own build cannot be timed here: it needs Open3D and the RobotCar SDK's Python code.

    python scripts/bench_oxford_build.py [--batch 64] [--reps 5] [--seconds 90] [--out PATH]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (x.strip() for x in q.split(","))
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # noqa: BLE001 - the card is still named by torch
        return dict(name=torch.cuda.get_device_name(0), power_limit=f"unknown ({e})")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seconds", type=float, default=90.0)
    ap.add_argument("--oracle-clouds", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "BENCH_OXFORD_BUILD.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_oxford_build needs a CUDA device")
    import oracle_oxford_build as oo
    from deepi2p_b200 import oxford_build as ob, pointprep, synthetic as syn
    dev = torch.device("cuda:0")
    res = dict(card=card(), batch=a.batch, reps=a.reps)
    with tempfile.TemporaryDirectory() as tmp:
        raw, lms, sdk, out = (os.path.join(tmp, d) for d in ("raw", "lms", "sdk", "out"))
        syn.write_oxford_raw(raw, lms, sdk, seconds=a.seconds, speed=10.0, stops=((40.0, 41.0),), curve=(45.0, 60.0),
                             n_returns=541, seed=7)
        t = sorted(os.listdir(raw))[0]
        t0 = time.perf_counter()
        plan = ob.plan_traversal(raw, lms, out, t, sdk)
        res["plan_s"] = time.perf_counter() - t0
        n = len(plan["centres"])
        S = min(a.batch, n)
        ids = list(range(S))
        win = [hi - lo for _, lo, hi, _ in plan["centres"][:S]]
        t0 = time.perf_counter()
        store = ob.RawScanStore(plan, dev)
        res["store_load_s"] = time.perf_counter() - t0
        res["store"] = dict(scans=int(store.present_host.sum()), points=store.n_points, bytes=store.nbytes)
        in_pts = int(sum(store.counts_host[lo - store.lo:hi - store.lo].sum() for _, lo, hi, _ in plan["centres"][:S]))
        res["segment"] = dict(clouds=n, clouds_timed=S, mean_window_scans=float(np.mean(win)),
                              input_points_per_batch=in_pts)
        ob.build_clouds(store, plan, ids)                       # warm-up of every shape
        torch.cuda.synchronize()
        stages = {k: [] for k in ("plan", "gather", "voxel", "pack", "total")}
        for _ in range(a.reps):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
            ev[0].record()
            planned = ob.plan_clouds(store, plan, ids)
            ev[1].record()
            g = ob.gather_clouds(store, plan, ids, planned)
            ev[2].record()
            down = pointprep.voxel_downsample(g["xyz"], g["n_pts"], 0.1, attr=g["attr"])
            ev[3].record()
            rec, m = ob.pack_clouds(plan, g, down)
            ev[4].record()
            torch.cuda.synchronize()
            for k, (i, j) in zip(("plan", "gather", "voxel", "pack", "total"),
                                 ((0, 1), (1, 2), (2, 3), (3, 4), (0, 4))):
                stages[k].append(ev[i].elapsed_time(ev[j]))
        res["stage_ms_median"] = {k: float(np.median(v)) for k, v in stages.items()}
        wall = []
        for _ in range(a.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = ob.build_clouds(store, plan, ids)
            r["records"].cpu()
            wall.append(time.perf_counter() - t0)
        w = float(np.median(wall))
        res["without_io"] = dict(batch_s=w, clouds_per_s=S / w, input_points_per_s=in_pts / w)
        t0 = time.perf_counter()
        summary = ob.build_traversal(raw, lms, out, t, sdk, batch=a.batch, device=dev)
        w = time.perf_counter() - t0
        all_pts = int(sum(store.counts_host[lo - store.lo:hi - store.lo].sum() for _, lo, hi, _ in plan["centres"]))
        res["with_io"] = dict(traversal_s=w, clouds=summary["clouds_built"], clouds_per_s=summary["clouds_built"] / w,
                              input_points_per_s=all_pts / w,
                              note="plan, store load, all batches and the .npy / table writes of the whole segment")
        t0 = time.perf_counter()
        scans = oo.read_scans(plan, range(plan["centres"][0][1], plan["centres"][a.oracle_clouds - 1][2]))
        for c in range(a.oracle_clouds):
            oo.build_cloud(plan, c, scans)
        res["oracle_s_per_cloud"] = (time.perf_counter() - t0) / a.oracle_clouds
        res["oracle_note"] = "one host core, numpy / Python; the reference needs Open3D and the SDK and is not timed"
    with open(a.out, "w") as f:
        json.dump(res, f)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
