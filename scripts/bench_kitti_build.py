"""Benchmark of the KITTI accumulated-frame build (deepi2p_b200.kitti_build) on a synthetic sequence of HDL-64-shaped
prepared scans (64 rings x 1024 azimuths, about 50k points per record after the seeded ray drop), at the published
parameters (stride 4 m, radius 50 m, voxel 0.4 m).  Writes BENCH_KITTI_BUILD.json (or --out):

  - outputs/s from a device store at batch 1 and at --batch, with CUDA-synchronised host clocks around whole
    build_frames calls (the count read-back and allocations included), median of --reps;
  - the whole sequence from files to files (build_sequence: plan, store load, every batch, the .npy writes);
  - the numpy oracle's time per output frame on one host core;
  - the card name and power limit, read in the same run.

The reference itself cannot be timed here: it needs Open3D.

    python scripts/bench_kitti_build.py [--frames 160] [--batch 64] [--reps 5] [--out PATH]
"""
import os

os.environ.setdefault("OMP_NUM_THREADS", "1")          # the oracle runs on one host core
os.environ.setdefault("OPENBLAS_NUM_THREADS", "1")
os.environ.setdefault("MKL_NUM_THREADS", "1")

import argparse  # noqa: E402
import json  # noqa: E402
import subprocess  # noqa: E402
import sys  # noqa: E402
import tempfile  # noqa: E402
import time  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402

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


def timed(fn, reps):
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t0)
    return float(np.median(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=160)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--single", type=int, default=16, help="outputs timed one per call")
    ap.add_argument("--oracle-frames", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "BENCH_KITTI_BUILD.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_kitti_build needs a CUDA device")
    import oracle_kitti_build as okb
    from deepi2p_b200 import kitti, kitti_build as kb, synthetic as syn
    res = dict(card=card(), batch=a.batch, reps=a.reps, params=dict(stride=4, radius=50, voxel=0.4))
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, "kitti")
        t0 = time.perf_counter()
        syn.write_kitti_root(root, seqs=(0,), n_frames=a.frames, seed=1, n_rings=64, n_azimuth=1024, image_hw=(8, 8),
                             n_images=1)
        res["write_root_s"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        plan = kb.plan_sequence(root, 0)
        res["plan_s"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        store = kb.stride_store(plan)
        torch.cuda.synchronize()
        res["store_load_s"] = time.perf_counter() - t0
        n = plan["n"]
        win = plan["windows"][:, 1] - plan["windows"][:, 0] + 1
        res["sequence"] = dict(frames=n, stride_frames=len(plan["strides"]), mean_window=float(win.mean()),
                               record_points=float(store.counts.mean()), store_bytes=store.nbytes)
        mid = max(0, n // 2 - a.batch // 2)
        frames = list(range(mid, min(n, mid + a.batch)))
        B = len(frames)
        strides, first, P = kb.frame_pairs(plan, frames)
        ids = [store.index(j) for j in strides]
        out = kb.build_frames(store, ids, first, P)               # warm-up
        res["batch_points_in"] = int(out["n_pts"].sum())
        res["batch_points_out"] = int(out["m_host"].sum())
        t = timed(lambda: kb.build_frames(store, ids, first, P), a.reps)
        res["device_store_batch"] = dict(frames=B, seconds=t, outputs_per_s=B / t,
                                         input_points_per_s=res["batch_points_in"] / t)
        singles = [kb.frame_pairs(plan, [i]) for i in frames[:a.single]]
        sargs = [([store.index(j) for j in s], f, p) for s, f, p in singles]
        kb.build_frames(store, *sargs[0])

        def one_by_one():
            for x in sargs:
                kb.build_frames(store, *x)
        t1 = timed(one_by_one, a.reps)
        res["device_store_batch1"] = dict(frames=len(sargs), seconds=t1, outputs_per_s=len(sargs) / t1)
        out_dir = kb.output_dir(root, 0)
        t0 = time.perf_counter()
        kb.build_sequence(root, 0, batch=a.batch, log=lambda s: None)
        res["files_to_files"] = dict(seconds=time.perf_counter() - t0, frames=n)
        res["files_to_files"]["outputs_per_s"] = n / res["files_to_files"]["seconds"]
        chk = np.load(os.path.join(out_dir, "%06d.npy" % frames[0]))
        o_frames = frames[:a.oracle_frames]
        Tr = kitti.read_calib(root, 0)["Tr"]
        t0 = time.perf_counter()
        o = okb.accumulate_sequence(root, 0, Tr, 4, 50, 0.4, frames=o_frames)
        res["oracle_s_per_frame"] = (time.perf_counter() - t0) / len(o_frames)
        res["oracle_equal"] = bool(np.array_equal(o["records"][frames[0]], chk))
    print(json.dumps(res))
    with open(a.out, "w") as f:
        f.write(json.dumps(res) + "\n")


if __name__ == "__main__":
    main()
