"""Throughput of the scan-preparation path (deepi2p_b200.pointprep) on HDL-64-shaped synthetic scans.

    python scripts/bench_prep.py [--scans 64] [--reps 5] [--cpu-scans 4] [--out FILE.json]

Scans: synthetic.make_lidar_scan (64 rings x 2048 azimuths = 131,072 points); 8 distinct scans are tiled to the batch
size.  KITTI parameters: voxel 0.1 m, normals with radius 0.6 m and max_nn 30, orientation (0, 0, 1).  Prints one JSON
line: prepare_scans scans/s at S = --scans and latency at S = 1; per-stage times at S = --scans (CUDA events around
the three C-ABI calls: voxel_downsample_batch_f32, estimate_normals_batch_f32, nearest_batch_f32); the mean number of
neighbours per normal; the loader workload (8 clouds, each 7 scans downsampled at 0.1 m and moved by a random pose,
through downsample_with_intensity_sn(..., 0.3) with numpy in and out); the GPU and its power limit; and the CPU
baseline, the oracle (oracle_prep) on all host cores.  Open3D's time is not measured (it is not installed).
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
from deepi2p_b200 import pointprep, synthetic  # noqa: E402
from deepi2p_b200.icp import pack_clouds  # noqa: E402


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
    except Exception:  # noqa: BLE001
        return "unknown"


def _stages(xyz, inten, n, reps):
    """Median ms of each C-ABI call of prepare_scans, each timed on its own with CUDA events."""
    down = pointprep.voxel_downsample(xyz, n, 0.1)
    d32 = down["xyz"].to(torch.float32)
    m = down["m_pts"]
    nrm, cnt = pointprep.estimate_normals(d32, m, 0.6, 30, counts=True)
    t_vox = _time(lambda: pointprep.voxel_downsample(xyz, n, 0.1), reps)
    t_nrm = _time(lambda: pointprep.estimate_normals(d32, m, 0.6, 30), reps)
    t_nn = _time(lambda: pointprep.nearest(down["xyz"], m, xyz, n), reps)
    nbr = float(cnt.sum()) / float(m.sum())
    return dict(voxel_downsample_ms=t_vox * 1e3, estimate_normals_ms=t_nrm * 1e3, nearest_ms=t_nn * 1e3,
                mean_points_per_scan=float(m.double().mean()), mean_neighbours=nbr)


def _loader_clouds(rng, n_clouds=8, frames=7):
    """Loader-shaped inputs: per cloud, 7 scans downsampled at 0.1 m (as the stored records are), each moved by a
    random planar pose, concatenated; intensity [1, N] and surface normals [3, N] alongside."""
    clouds = []
    for c in range(n_clouds):
        pcs, its, sns = [], [], []
        for f in range(frames):
            sc = synthetic.make_lidar_scan(100 + 7 * c + f)
            xyz, n = pack_clouds([sc["xyz"]])
            down = pointprep.voxel_downsample(xyz, n, 0.1)
            m = int(down["m_pts"][0])
            p = down["xyz"][0, :, :m].cpu().numpy()
            a = rng.uniform(-0.2, 0.2)
            R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
            pcs.append((R @ p + np.array([[rng.uniform(-3, 3)], [rng.uniform(-1, 1)], [0.0]])).astype(np.float32))
            its.append(rng.random((1, m)).astype(np.float32))
            sn = rng.standard_normal((3, m))
            sns.append((sn / np.linalg.norm(sn, axis=0)).astype(np.float32))
        clouds.append((np.concatenate(pcs, 1), np.concatenate(its, 1), np.concatenate(sns, 1)))
    return clouds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-scans", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_prep.py needs a CUDA device")
    base = [synthetic.make_lidar_scan(s) for s in range(8)]
    scans = [base[s % 8] for s in range(a.scans)]
    xyz, n = pack_clouds([s["xyz"] for s in scans])
    inten = torch.from_numpy(np.stack([s["intensity"] for s in scans])).cuda()
    t_big = _time(lambda: pointprep.prepare_scans(xyz, inten, n), a.reps)
    t_one = _time(lambda: pointprep.prepare_scans(xyz[:1], inten[:1], n[:1]), max(a.reps, 10))
    stages = _stages(xyz, inten, n, a.reps)

    rng = np.random.default_rng(0)
    clouds = _loader_clouds(rng)
    for c in clouds[:1]:
        pointprep.downsample_with_intensity_sn(c[0], c[1], c[2], 0.3)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(a.reps):
        for c in clouds:
            pointprep.downsample_with_intensity_sn(c[0], c[1], c[2], 0.3)
    t_loader = (time.perf_counter() - t0) / (a.reps * len(clouds))

    import oracle_prep
    t0 = time.perf_counter()
    for s in range(a.cpu_scans):
        oracle_prep.prepare_scan(base[s]["xyz"], base[s]["intensity"])
    t_cpu = (time.perf_counter() - t0) / max(a.cpu_scans, 1)

    res = {"prep": {
        "scans": a.scans, "points_per_scan": int(xyz.shape[2]), "voxel": 0.1, "sn_radius": 0.6, "sn_max_nn": 30,
        "seconds": t_big, "scans_per_s": a.scans / t_big, "latency_s1_ms": t_one * 1e3,
        "stages_ms": {k: v for k, v in stages.items() if k.endswith("_ms")},
        "mean_points_after_downsample": stages["mean_points_per_scan"],
        "mean_neighbours_per_query": stages["mean_neighbours"],
        "loader": {"clouds": len(clouds), "mean_points_in": float(np.mean([c[0].shape[1] for c in clouds])),
                   "voxel": 0.3, "ms_per_cloud": t_loader * 1e3},
        "gpu": torch.cuda.get_device_name(0), "power_limit": _power_limit(),
        "oracle_cpu": {"scans": a.cpu_scans, "cores": os.cpu_count(), "s_per_scan": t_cpu},
        "open3d_cpu": "not measured"}}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
