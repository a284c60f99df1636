"""bfloat16 autocast benchmark of the classifier's training step (DESIGN.md 4.37): writes BENCH_AMP.json.

- step: the captured training step (train.train_step replayed from a CUDA graph) in fp32 and bf16 at KITTI (B = 8,
  160 x 512), Oxford (B = 8, 384 x 640) and nuScenes (B = 12, 160 x 320), timed in alternating blocks of the two
  precisions on two models of the same seeded state (medians over the blocks), and the peak allocation of one eager
  step of each precision on its own.
- ops: forward + backward of the five differentiable ops at the network's own call shapes (KITTI, B = 8), float32
  against bfloat16 operands, alternating blocks, medians.
- profile: torch.profiler over eager bf16 KITTI steps, profiled apart from the timed runs: kernel time split between
  cuDNN convolutions and BatchNorm, the project's ops and the rest.
- the GPU name and power limit, read in this run.

    python scripts/bench_amp.py [--reps 20] [--out BENCH_AMP.json]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from deepi2p_b200 import classifier, point_ops, train  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_prep import _power_limit  # noqa: E402
from bench_train import SHAPES, _block_ms, inputs, model_for  # noqa: E402

PRECISIONS = ("fp32", "bf16")


def step_times(shape, dev, reps, blocks=5):
    x = inputs(shape, dev)
    out = {"B": SHAPES[shape][0], "points": 20480, "image": list(SHAPES[shape][1])}
    replays = {}
    for p in PRECISIONS:                                  # the eager step's peak, each precision on its own
        m = model_for(shape, dev)
        o = train.make_optimizer(m)
        for _ in range(train.WARMUP_STEPS):
            train.train_step(m, o, x, p)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        train.train_step(m, o, x, p)
        torch.cuda.synchronize()
        out[f"{p}_eager_step_peak_bytes"] = torch.cuda.max_memory_allocated() - base
        o.zero_grad(set_to_none=True)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            train.train_step(m, o, x, p)
        g.replay()
        replays[p] = (g, m, o)
    torch.cuda.synchronize()
    ms = {p: [] for p in PRECISIONS}
    for _ in range(blocks):
        for p in PRECISIONS:
            ms[p].append(_block_ms(replays[p][0].replay, reps))
    for p in PRECISIONS:
        out[f"{p}_captured_step_ms"] = float(np.median(ms[p]))
        out[f"{p}_captured_blocks_ms"] = ms[p]
    out["steps_per_block"] = reps
    out["bf16_speedup"] = out["fp32_captured_step_ms"] / out["bf16_captured_step_ms"]
    del replays
    torch.cuda.empty_cache()
    return out


def op_cases(dev):
    """(name, inputs -> differentiable output, feature inputs) of the five ops at the KITTI network's shapes, B = 8."""
    x = inputs("kitti", dev)
    B = x["pc"].shape[0]
    g = torch.Generator(device=dev).manual_seed(5)
    r = lambda *s: torch.randn(*s, device=dev, generator=g)
    ca = point_ops.cluster_assign_forward(x["pc"], x["node_a"], k=3)
    pb_idx = point_ops.cluster_assign_forward(x["pc"], x["node_b"], k=3, want_centers=False)["min_k_idx"]
    cases = [
        ("cluster_max_pool [B,32,N] broadcast", lambda f: point_ops.cluster_max_pool(f, ca["min_idx"], 128, True)[1],
         [r(B, 32, 20480)]),
        ("cluster_max_pool [B,64,N]", lambda f: point_ops.cluster_max_pool(f, ca["min_idx"], 128), [r(B, 64, 20480)]),
        ("knn_group [B,64,128] K=16", lambda f: point_ops.knn_group(x["node_b"], ca["cluster_mean"], f, 16)[1],
         [r(B, 64, 128)]),
        ("upsample_by_interpolation pb [B,512,128] -> N",
         lambda f: point_ops.upsample_by_interpolation(pb_idx, x["pc"], x["node_b"], f), [r(B, 512, 128)]),
        ("upsample_by_interpolation pa [B,128,128] -> N",
         lambda f: point_ops.upsample_by_interpolation(ca["min_k_idx"], x["pc"], x["node_a"], f), [r(B, 128, 128)]),
        ("attention_fusion s16 [B,256,320] x [B,320,128]", point_ops.attention_fusion,
         [r(B, 256, 320), r(B, 320, 128)]),
        ("attention_fusion s32 [B,512,80] x [B,80,128]", point_ops.attention_fusion, [r(B, 512, 80), r(B, 80, 128)]),
        ("classifier_loss [B,82,N]", lambda s: classifier.classifier_loss(s[:, :2], s[:, 2:], x["pc"], x["P"], x["K"],
                                                                            160, 512)["loss"], [r(B, 82, 20480)]),
    ]
    return cases


def op_times(dev, reps, blocks=5):
    out = []
    for name, fn, feats in op_cases(dev):
        runs = {}
        for p, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
            xs = [f.to(dt).requires_grad_(True) for f in feats]
            y = fn(*xs)
            gy = torch.randn_like(y) if y.dim() else None

            def run(xs=xs, gy=gy):
                y = fn(*xs)
                y.backward(gy)
            runs[p] = run
            run()
        torch.cuda.synchronize()
        ms = {p: [] for p in PRECISIONS}
        for _ in range(blocks):
            for p in PRECISIONS:
                ms[p].append(_block_ms(runs[p], reps))
        row = {"op": name, "fp32_fwd_bwd_ms": float(np.median(ms["fp32"])),
               "bf16_fwd_bwd_ms": float(np.median(ms["bf16"]))}
        row["bf16_speedup"] = row["fp32_fwd_bwd_ms"] / row["bf16_fwd_bwd_ms"]
        out.append(row)
    return out


CONV_BN = ("conv", "cudnn", "xmma", "gemm", "implicit", "wgrad", "dgrad", "bn_", "batch_norm", "batchnorm",
           "BatchNorm", "nhwc", "nchw", "cutlass", "sm90_")


def kernel_split(dev, steps=5):
    """Kernel time of `steps` eager bf16 KITTI steps (profiled in a run of their own), by kernel name: the project's
    kernels (namespace dib::), cuDNN convolutions and BatchNorm, and the rest (elementwise, casts, reductions, Adam)."""
    from torch.profiler import ProfilerActivity, profile
    x = inputs("kitti", dev)
    m = model_for("kitti", dev)
    o = train.make_optimizer(m)
    for _ in range(train.WARMUP_STEPS):
        train.train_step(m, o, x, "bf16")
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            train.train_step(m, o, x, "bf16")
        torch.cuda.synchronize()
    split = {"project_ops": 0.0, "conv_and_batchnorm": 0.0, "other": 0.0}
    top = {}
    for e in prof.key_averages():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        t = e.self_device_time_total
        key = "project_ops" if "dib::" in e.key else \
            "conv_and_batchnorm" if any(s in e.key.lower() for s in (c.lower() for c in CONV_BN)) else "other"
        split[key] += t
        top[e.key[:120]] = (key, t)
    total = sum(split.values())
    return {"steps": steps, "kernel_ms_per_step": total / steps / 1e3,
            **{f"{k}_ms_per_step": v / steps / 1e3 for k, v in split.items()},
            **{f"{k}_share": v / total for k, v in split.items()},
            "top_kernels": [{"kernel": k, "class": c, "ms_per_step": t / steps / 1e3}
                            for k, (c, t) in sorted(top.items(), key=lambda kv: -kv[1][1])[:15]]}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(ROOT, "BENCH_AMP.json"))
    ap.add_argument("--parts", default="step,ops,profile")
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_amp.py needs a CUDA device")
    dev = torch.device("cuda")
    torch.backends.cudnn.benchmark = True
    parts = a.parts.split(",")
    res = {"gpu": torch.cuda.get_device_name(dev), "power_limit": _power_limit(), "torch": torch.__version__,
           "cudnn_benchmark": True, "tf32_flags": [torch.backends.cuda.matmul.allow_tf32,
                                                   torch.backends.cudnn.allow_tf32]}
    if "step" in parts:
        res["step"] = {s: step_times(s, dev, a.reps) for s in SHAPES}
    if "ops" in parts:
        res["ops_kitti_B8"] = op_times(dev, a.reps)
    if "profile" in parts:
        res["bf16_kernel_split_kitti"] = kernel_split(dev)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))
    return res


if __name__ == "__main__":
    main()
