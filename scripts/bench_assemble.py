"""Throughput of classifier-batch assembly (deepi2p_b200.assemble) on KITTI-shaped synthetic samples.

    python scripts/bench_assemble.py [--samples 64] [--reps 5] [--cpu-samples 2] [--out FILE.json]

Samples: synthetic.make_loader_sample (7 frames of 64 rings x 512 azimuths, 229,376 points per sample, so every
sample takes the voxel-0.3 step); 8 distinct samples are tiled to the batch size.  train mode with the KITTI
arguments (Ry augmentation, flip, jitter on pc and sn), N = 20480, Ma = Mb = 128.  Prints one JSON line: samples/s of
assemble_batch at S = --samples from device frames and the latency of one sample; per-stage times at S = --samples
(CUDA events around each call: accumulate with its count read-back, the voxel step, resample, and the two candidate +
farthest-point calls); farthest-point sampling alone for 128 sets of 1024 -> 128 (one CTA per set) and 64 full clouds
of 20480 -> 128 and -> 512 (the cluster path); the GPU and its power limit; and the numpy restatement of the point
side (oracle_assemble, its voxel grid on one thread) per sample on one host core.
"""
import os

os.environ.setdefault("OMP_NUM_THREADS", "1")      # the CPU baseline is one host core

import argparse  # noqa: E402
import json  # noqa: E402
import sys  # noqa: E402
import time  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepi2p_b200 import assemble, synthetic  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_prep import _power_limit, _time  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-samples", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_assemble.py needs a CUDA device")
    N, M = 20480, 128
    base = [synthetic.make_loader_sample(s, "kitti") for s in range(8)]
    smps = [base[s % 8] for s in range(a.samples)]
    frames = assemble.pack_frames([(m["frames"], m["frame_T"]) for m in smps])
    one = assemble.pack_frames([(base[0]["frames"], base[0]["frame_T"])])
    args = assemble.kitti_args(base[0]["Pc"], base[0]["Pji"])

    def run(fr):
        return assemble.assemble_batch(fr, "train", 7, input_pt_num=N, node_a_num=M, node_b_num=M, rng=0, **args)

    t_big = _time(lambda: run(frames), a.reps)
    t_one = _time(lambda: run(one), max(a.reps, 10))

    # stages at S = --samples, each timed on its own
    acc = lambda: assemble.accumulate(frames["xyz"], frames["intensity"], frames["sn"], frames["n_pts"],  # noqa: E731
                                      frames["frame_sample"], frames["frame_T"])
    x, i, sn, cnt, cnt_h = acc()
    S = cnt_h.shape[0]
    t_acc = _time(acc, a.reps)

    def vox():
        x2, i2, s2 = x.clone(), i.clone(), sn.clone()
        return assemble._voxel_step(x2, i2, s2, cnt, cnt_h, N, 0.3, None)

    t_clone = _time(lambda: (x.clone(), i.clone(), sn.clone()), a.reps)
    t_vox = _time(vox, a.reps) - t_clone
    x2, i2, s2 = x.clone(), i.clone(), sn.clone()
    c2, _ = assemble._voxel_step(x2, i2, s2, cnt, cnt_h, N, 0.3, None)
    Pr, _ = assemble.random_transforms(S, "train", args["amplitudes"], 0)
    Mx = assemble.compose(Pr, np.broadcast_to(args["pre"], (S, 4, 4)))
    res = lambda: assemble.resample(x2, i2, s2, c2, N, 7, M=Mx, jitter=("pc", "sn"))  # noqa: E731
    out = res()
    t_res = _time(res, a.reps)

    def nodes():
        for ns in (0, 1):
            cidx, cxyz = assemble.candidates(out["pc"], 8 * M, 7, ns)
            assemble.farthest_point_sample(cxyz, None, M)

    t_nodes = _time(nodes, a.reps)

    rng = np.random.default_rng(1)
    sets = torch.from_numpy(rng.normal(0, 20, (128, 3, 1024)).astype(np.float32)).cuda()
    t_fps_small = _time(lambda: assemble.farthest_point_sample(sets, None, 128), a.reps)
    t_fps_128 = _time(lambda: assemble.farthest_point_sample(out["pc"], None, 128), a.reps)
    t_fps_512 = _time(lambda: assemble.farthest_point_sample(out["pc"], None, 512), a.reps)

    import oracle_assemble
    t0 = time.perf_counter()
    for s in range(a.cpu_samples):
        oracle_assemble.assemble_sample(base[s]["frames"], base[s]["frame_T"], s, 7, Mx[s], N, M, M, 0.3, None,
                                        ("pc", "sn"))
    t_cpu = (time.perf_counter() - t0) / max(a.cpu_samples, 1)

    result = {"assemble": {
        "samples": a.samples, "frames_per_sample": 7, "points_per_sample_in": int(frames["n_pts"][:7].sum()),
        "input_pt_num": N, "node_a_num": M, "node_b_num": M, "mode": "train",
        "seconds": t_big, "samples_per_s": a.samples / t_big, "latency_s1_ms": t_one * 1e3,
        "stages_ms": {"accumulate_with_readback": t_acc * 1e3, "voxel_step": t_vox * 1e3, "resample": t_res * 1e3,
                      "candidates_and_fps_a_b": t_nodes * 1e3},
        "mean_points_before_resample": float(c2.double().mean()),
        "fps_ms": {"sets128_1024_to_128": t_fps_small * 1e3, "clouds64_20480_to_128": t_fps_128 * 1e3,
                   "clouds64_20480_to_512": t_fps_512 * 1e3},
        "gpu": torch.cuda.get_device_name(0), "power_limit": _power_limit(),
        "numpy_cpu": {"samples": a.cpu_samples, "cores": 1, "s_per_sample": t_cpu}}}
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
