"""Training benchmark of the classifier (DESIGN.md 4.32): writes BENCH_TRAIN.json.

- step: one training step (forward in train mode, classifier_loss, backward, Adam) at the shipped KITTI shape (B = 8,
  20480 points, 160 x 512), eager (train.train_step) and replayed from a CUDA graph, timed in alternating blocks on
  two models of the same seeded state; Oxford (B = 8, 384 x 640) and nuScenes (B = 12, 160 x 320): the step alone.
- profile: torch.profiler over eager KITTI steps: the share of the step's wall time in which some kernel runs, and
  the idle gaps between consecutive kernels.
- trainer: train.Trainer epochs on a synthetic KITTI root (one train and one val sequence of 64 x 1024-ray scans)
  from a device scan store, overlapped (batch k + 1 assembled on a side stream while step k runs) and serial (the
  device synchronised after every step, so assembly and step never overlap), in samples/s.
- the GPU name and power limit, read in this run, and the peak memory of each part.

    python scripts/bench_train.py [--reps 20] [--out BENCH_TRAIN.json]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from deepi2p_b200 import network, synthetic, train  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_prep import _power_limit  # noqa: E402

SHAPES = {"kitti": (8, (160, 512)), "oxford": (8, (384, 640)), "nuscenes": (12, (160, 320))}


def inputs(shape, dev, seed=2000):
    """Seeded inputs of the shape's batch: synthetic.make_sample clouds, nodes drawn from them, a random image."""
    S, (H, W) = SHAPES[shape]
    smps = [synthetic.make_sample(seed + s, 20480, "oxford" if shape == "oxford" else "kitti") for s in range(S)]
    pc = torch.from_numpy(np.stack([s["points"] for s in smps])).to(dev)
    gen = torch.Generator(device=dev).manual_seed(seed)
    idx = torch.argsort(torch.rand(S, 20480, device=dev, generator=gen), dim=1)[:, :256]
    nodes = torch.gather(pc, 2, idx.unsqueeze(1).expand(S, 3, 256))
    return dict(pc=pc, intensity=torch.rand(S, 1, 20480, device=dev, generator=gen),
                sn=torch.nn.functional.normalize(torch.randn(S, 3, 20480, device=dev, generator=gen), dim=1),
                node_a=nodes[:, :, :128].contiguous(), node_b=nodes[:, :, 128:].contiguous(),
                img=torch.rand(S, 3, H, W, device=dev, generator=gen),
                K=torch.from_numpy(np.stack([s["K"] for s in smps])).float().to(dev),
                P=torch.from_numpy(np.stack([s["P_gt"][:3] for s in smps])).float().to(dev))


def model_for(shape, dev):
    model = network.KeypointDetector(**network.SHAPES[shape])
    model.load_state_dict(synthetic.seeded_state_dict(model, 1))
    return model.to(dev)


def _block_ms(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def step_times(shape, dev, reps):
    """Eager and captured step of two models of the same seeded state, timed in alternating blocks of `reps` steps;
    medians over the blocks.  Also the peak memory of each."""
    x = inputs(shape, dev)
    me, mg = model_for(shape, dev), model_for(shape, dev)
    oe, og = train.make_optimizer(me), train.make_optimizer(mg)
    eager = lambda: train.train_step(me, oe, x)
    for _ in range(train.WARMUP_STEPS):
        eager()
        train.train_step(mg, og, x)
    og.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        train.train_step(mg, og, x)
    graph_bytes = torch.cuda.memory_allocated() - before
    replay = g.replay
    replay()
    eager()
    torch.cuda.synchronize()
    e_ms, g_ms = [], []
    for _ in range(5):
        e_ms.append(_block_ms(eager, reps))
        g_ms.append(_block_ms(replay, reps))
    torch.cuda.reset_peak_memory_stats()
    eager()
    torch.cuda.synchronize()
    e_peak = torch.cuda.max_memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    replay()
    torch.cuda.synchronize()
    g_peak = torch.cuda.max_memory_allocated()
    S, (H, W) = SHAPES[shape]
    res = {"B": S, "points": 20480, "image": [H, W], "eager_step_ms": float(np.median(e_ms)),
           "captured_step_ms": float(np.median(g_ms)), "eager_blocks_ms": e_ms, "captured_blocks_ms": g_ms,
           "steps_per_block": reps, "graph_private_pool_bytes": graph_bytes,
           "peak_bytes_two_models_eager_step": e_peak, "peak_bytes_two_models_replay": g_peak}
    del g
    return res


def profile_eager(dev, steps=5):
    """Kernel intervals of `steps` eager KITTI steps: busy share = union of kernel time / span from the first kernel
    start to the last kernel end; gaps = idle time between consecutive (merged) kernel intervals."""
    from torch.profiler import ProfilerActivity, profile
    x = inputs("kitti", dev)
    m = model_for("kitti", dev)
    o = train.make_optimizer(m)
    for _ in range(train.WARMUP_STEPS):
        train.train_step(m, o, x)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            train.train_step(m, o, x)
        torch.cuda.synchronize()
    iv = sorted((e.time_range.start, e.time_range.end) for e in prof.events()
                if e.device_type == torch.autograd.DeviceType.CUDA and e.time_range.end > e.time_range.start)
    merged = []
    for s, t in iv:
        if merged and s <= merged[-1][1]:
            merged[-1][1] = max(merged[-1][1], t)
        else:
            merged.append([s, t])
    busy = sum(t - s for s, t in merged)
    span = merged[-1][1] - merged[0][0]
    gaps = np.array([merged[i + 1][0] - merged[i][1] for i in range(len(merged) - 1)], dtype=np.float64)
    return {"steps": steps, "kernels_per_step": len(iv) / steps, "device_busy_share": busy / span,
            "span_ms_per_step": span / steps / 1e3, "busy_ms_per_step": busy / steps / 1e3,
            "gap_ms_per_step": float(gaps.sum()) / steps / 1e3, "gap_us_median": float(np.median(gaps)),
            "gap_us_p90": float(np.percentile(gaps, 90)), "gap_us_max": float(gaps.max()),
            "gaps_over_50us_per_step": float((gaps > 50).sum()) / steps}


def trainer_rates(dev, epochs=3):
    """Samples/s of Trainer.train_epoch, overlapped and serial, alternating epochs after one warm-up epoch each."""
    with tempfile.TemporaryDirectory() as d:
        root = os.path.join(d, "kitti")
        synthetic.write_kitti_root(root, seqs=(0, 9), n_frames=120, n_rings=64, n_azimuth=1024, n_images=1)
        tr = train.batch_source("kitti", root, "train", store="cuda", seqs=(0,))
        te = train.batch_source("kitti", root, "val", store="cuda", seqs=(9,))
        out = {"root": "synthetic.write_kitti_root(seqs=(0, 9), n_frames=120, n_rings=64, n_azimuth=1024)",
               "train_entries": tr[0], "batch": 8, "store": "cuda"}
        trainers = {}
        for kind in ("overlapped", "serial"):
            m = model_for("kitti", dev)
            t = train.Trainer(m, tr, te, "kitti", os.path.join(d, kind), log=lambda s: None)
            if kind == "serial":
                step = t._step

                def serial_step(step=step):
                    step()
                    torch.cuda.synchronize()
                t._step = serial_step
            t.train_epoch(0)                  # warm-up and capture
            trainers[kind] = t
        torch.cuda.synchronize()
        times = {"overlapped": [], "serial": []}
        torch.cuda.reset_peak_memory_stats()
        for e in range(1, epochs + 1):
            for kind, t in trainers.items():
                t0 = time.perf_counter()
                t.train_epoch(e)
                torch.cuda.synchronize()
                times[kind].append(time.perf_counter() - t0)
        n = (tr[0] // 8) * 8
        for kind in times:
            out[kind] = {"epoch_seconds": times[kind], "samples_per_s": n / float(np.median(times[kind]))}
        out["peak_bytes_two_trainers"] = torch.cuda.max_memory_allocated()
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="BENCH_TRAIN.json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train.py needs a CUDA device")
    dev = torch.device("cuda")
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit": _power_limit(),
           "torch": torch.__version__, "cudnn_benchmark": torch.backends.cudnn.benchmark}
    res["step"] = {"kitti": step_times("kitti", dev, a.reps)}
    print(json.dumps(res["step"]["kitti"]), flush=True)
    res["profile_eager_kitti"] = profile_eager(dev)
    print(json.dumps(res["profile_eager_kitti"]), flush=True)
    res["trainer_kitti"] = trainer_rates(dev)
    print(json.dumps(res["trainer_kitti"]), flush=True)
    for shape in ("oxford", "nuscenes"):
        res["step"][shape] = step_times(shape, dev, a.reps)
        print(json.dumps(res["step"][shape]), flush=True)
    with open(a.out, "w") as f:
        json.dump({"train": res}, f)
    print(json.dumps({"train": res}))


if __name__ == "__main__":
    main()
