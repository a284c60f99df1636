"""Throughput of the nuScenes classifier batch (deepi2p_b200.assemble with nuscenes_args, deepi2p_b200.nuscenes) on
seeded nuScenes-shaped synthetic samples.

    python scripts/bench_nuscenes.py [--samples 12,64] [--reps 5] [--cpu-samples 2] [--out FILE.json]

Samples: synthetic.make_nuscenes_sample (7 LIDAR_TOP-shaped sweeps of 32 rings x 1085 azimuths plus 512 points in and
around the ego-vehicle box, 246,624 points per sample, so every sample takes the voxel-0.2 step on the fp64 cloud); 8
distinct samples are tiled to the batch size.  train mode with nuscenes_args (rotation about z, jitter on pc and
intensity), N = 20480, Ma = Mb = 128.  Prints one JSON line with, per batch size S: samples/s of the point side from
host sweep arrays (pack_frames + assemble_batch) and from device buffers (assemble_batch); per-stage times (CUDA
events around each call: accumulate with its count read-back, the voxel step, resample, and the two candidate +
farthest-point calls); and nuscenes_batch end to end on a dataroot written to a temporary directory (sweep files read
on the host, the JSON tables, 1600 x 900 JPEG frames decoded on the device).  Beside them: the GPU and its power
limit, and oracle_nuscenes per sample on one host core.  The reference loader itself is not timed: it needs
nuscenes-devkit and Open3D.
"""
import os

os.environ.setdefault("OMP_NUM_THREADS", "1")      # the CPU baseline is one host core

import argparse  # noqa: E402
import json  # noqa: E402
import sys  # noqa: E402
import tempfile  # noqa: E402
import time  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from deepi2p_b200 import assemble, nuscenes, synthetic  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_prep import _power_limit, _time  # noqa: E402


def _jpeg_1600x900():
    g = np.load(os.path.join(ROOT, "tests", "golden", "jpeg_small.npz"))
    so = np.concatenate([[0], np.cumsum(g["stream_lens"])])
    i = int(np.nonzero((g["shapes"][:, 0] == 900) & (g["shapes"][:, 1] == 1600))[0][0])
    return g["streams"][so[i]:so[i + 1]].tobytes()


def _stages(frames, args, N, M, reps):
    acc = lambda: assemble.accumulate(frames["xyz"], frames["intensity"], None, frames["n_pts"],  # noqa: E731
                                      frames["frame_sample"], frames["frame_T"], None, None, args["exclude_box"], True)
    x, i, _, cnt, cnt_h = acc()
    S = cnt_h.shape[0]
    t_acc = _time(acc, reps)
    t_clone = _time(lambda: (x.clone(), i.clone()), reps)
    t_vox = _time(lambda: assemble._voxel_step(x.clone(), i.clone(), None, cnt, cnt_h, N, 0.2, None), reps) - t_clone
    i2 = i.clone()
    x2, c2, _ = assemble._voxel_step(x, i2, None, cnt, cnt_h, N, 0.2, None)
    Pr, _ = assemble.random_transforms(S, "train", args["amplitudes"], 0, False)
    res = lambda: assemble.resample(x2, i2, None, c2, N, 7, M=Pr, jitter=("pc", "intensity"))  # noqa: E731
    out = res()
    t_res = _time(res, reps)

    def nodes():
        for ns in (0, 1):
            cidx, cxyz = assemble.candidates(out["pc"], 8 * M, 7, ns)
            assemble.farthest_point_sample(cxyz, None, M)

    t_nodes = _time(nodes, reps)
    return dict(accumulate_with_readback=t_acc * 1e3, voxel_step=t_vox * 1e3, resample=t_res * 1e3,
                candidates_and_fps_a_b=t_nodes * 1e3), float(c2.double().mean())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", default="12,64")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-samples", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_nuscenes.py needs a CUDA device")
    N, M = 20480, 128
    base = [synthetic.make_nuscenes_sample(s) for s in range(8)]
    args = assemble.nuscenes_args(base[0]["P_cam_pc"])
    blob = _jpeg_1600x900()
    result = {"gpu": torch.cuda.get_device_name(0), "power_limit": _power_limit(), "input_pt_num": N,
              "node_a_num": M, "node_b_num": M, "mode": "train", "sweeps_per_sample": 7,
              "points_per_sample_in": int(sum(f[0].shape[1] for f in base[0]["frames"])), "batches": {}}
    with tempfile.TemporaryDirectory() as root:
        items = synthetic.write_nuscenes_dataroot(root, [(25, 12)] * 4, seed=1, jpeg=blob, n_rings=32, n_azimuth=1085)
        tables = nuscenes.Tables(root, "v1.0-mini")
        for S in (int(v) for v in a.samples.split(",")):
            smps = [base[s % 8] for s in range(S)]
            host = [(m["frames"], m["frame_T"]) for m in smps]
            frames = assemble.pack_frames(host)

            def run(fr):
                return assemble.assemble_batch(fr, "train", 7, input_pt_num=N, node_a_num=M, node_b_num=M, rng=0,
                                               **args)

            t_dev = _time(lambda: run(frames), a.reps)
            t_host = _time(lambda: run(assemble.pack_frames(host)), a.reps)
            stages, mean_n = _stages(frames, args, N, M, a.reps)
            its = [items[s % len(items)] for s in range(S)]
            t_batch = _time(lambda: nuscenes.nuscenes_batch(tables, its, "train", 7, rng=0), a.reps)
            result["batches"][str(S)] = {
                "samples": S, "point_side_from_host_sweeps": {"seconds": t_host, "samples_per_s": S / t_host},
                "point_side_from_device_buffers": {"seconds": t_dev, "samples_per_s": S / t_dev},
                "stages_ms": stages, "mean_points_before_resample": mean_n,
                "nuscenes_batch_with_jpeg_decode": {"seconds": t_batch, "samples_per_s": S / t_batch}}
    import oracle_nuscenes
    Pr, _ = assemble.random_transforms(a.cpu_samples, "train", args["amplitudes"], 0, False)
    t0 = time.perf_counter()
    for s in range(a.cpu_samples):
        oracle_nuscenes.assemble_sample(base[s]["frames"], base[s]["frame_T"], s, 7, Pr[s], N, M, M,
                                        jitter_channels=("pc", "intensity"))
    t_cpu = (time.perf_counter() - t0) / max(a.cpu_samples, 1)
    result["numpy_oracle_cpu"] = {"samples": a.cpu_samples, "cores": 1, "s_per_sample": t_cpu}
    result["reference_loader"] = "not timed: it needs nuscenes-devkit and Open3D"
    line = json.dumps({"nuscenes": result})
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
