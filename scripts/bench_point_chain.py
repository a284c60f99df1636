"""Benchmark of the classifier's per-point chains in training (point_ops.point_chain, DESIGN.md 4.34): writes
BENCH_POINT_CHAIN.json.

- chains: forward + backward of first_pointnet, second_pointnet and per_point_pn (KITTI, Oxford and nuScenes head
  widths, plus the coarse-only head) at the trainer's batch (B = 8, 12 for nuScenes; 20480 points), the model's torch
  layers (torch.cat of the inputs, Conv1d / BatchNorm1d / ReLU / Dropout; for the head the pa and pb interpolations
  and the 736-row cat) against point_chain (for the head: W_a, W_b applied at the nodes, the projected rows
  interpolated, the sum as the additive term), timed in alternating blocks, medians over blocks; peak memory of each
  above the inputs; the fused op's TF32 GEMM work (forward, dX and dW products, from shapes) over its time, against
  the 495 TFLOP/s dense TF32 data-sheet figure of the H100 SXM.  That is a whole-op rate, not a kernel's share.
- step: the captured training step (train.train_step in one CUDA graph) of KeypointDetector(point_layers="torch")
  and "fused" for KITTI, Oxford and nuScenes, alternating blocks, medians.
- step_peak: the peak allocation of one eager step per mode, each measured with the other mode's model freed.
- attribution: torch.profiler over eager steps of the torch-mode model, the kernel time of each chain's forward and
  backward (tied to its forward through the autograd sequence numbers) over the step's kernel time.
- the GPU name and power limit, read in this run.

    python scripts/bench_point_chain.py [--reps 20] [--out BENCH_POINT_CHAIN.json]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from deepi2p_b200 import network, point_ops, synthetic, train  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_prep import _power_limit  # noqa: E402
from bench_train import SHAPES, _block_ms, inputs  # noqa: E402

TF32_PEAK = 495e12
N = 20480
# (name, B, c_in, widths, norm_act_at_last, dropouts, dense source widths)
CHAINS = [("first", 8, 7, [32, 32, 32], True, None, (3, 1, 3)),
          ("second", 8, 64, [64, 64], True, None, (32, 32)),
          ("head_kitti", 8, 736, [256, 256, 82], False, [0.5, 0.5, 0], (32, 64)),
          ("head_oxford", 8, 736, [256, 256, 242], False, [0.5, 0.5, 0], (32, 64)),
          ("head_nuscenes", 12, 736, [256, 256, 52], False, [0.5, 0.5, 0], (32, 64)),
          ("head_coarse", 8, 736, [128, 128, 2], False, [0.5, 0.5, 0], (32, 64))]


def chain_case(spec, dev):
    name, B, c_in, widths, last, drops, src_w = spec
    torch.manual_seed(0)
    pn = network._PointNet(c_in, widths, last, 0.1, drops).to(dev)
    g = torch.Generator(device=dev).manual_seed(1)
    srcs = [torch.randn((B, c, N), device=dev, generator=g).requires_grad_() for c in src_w]
    state = point_ops.new_dropout_state(0, dev)
    if sum(src_w) == c_in:
        torch_fn = lambda: pn(torch.cat(srcs, dim=1))
        fused_fn = lambda: point_ops.point_chain(srcs, list(pn.layers), True, state)
        return torch_fn, fused_fn, pn, srcs, B
    pc = torch.randn((B, 3, N), device=dev, generator=g)
    na, nb = pc[:, :, :128].contiguous(), pc[:, :, 128:256].contiguous()
    ia = point_ops.cluster_assign_forward(pc, na, k=3, want_centers=False)["min_k_idx"]
    ib = point_ops.cluster_assign_forward(pc, nb, k=3, want_centers=False)["min_k_idx"]
    upa = torch.randn((B, 128, 128), device=dev, generator=g).requires_grad_()
    upb = torch.randn((B, 512, 128), device=dev, generator=g).requires_grad_()

    def torch_fn():
        pa = point_ops.upsample_by_interpolation(ia, pc, na, upa)
        pb = point_ops.upsample_by_interpolation(ib, pc, nb, upb)
        return pn(torch.cat((pa, pb, *srcs), dim=1))

    def fused_fn():
        W1 = pn.layers[0].conv.weight[:, :, 0]
        add = point_ops.upsample_by_interpolation(ia, pc, na, point_ops.channel_product(W1[:, :128], upa)) + \
            point_ops.upsample_by_interpolation(ib, pc, nb, point_ops.channel_product(W1[:, 128:640], upb))
        return point_ops.point_chain(srcs, list(pn.layers), True, state, add=add, in_col=640)
    return torch_fn, fused_fn, pn, srcs, B


def gemm_flops(spec, B):
    """TF32 products of the fused op per call, from shapes: forward W x, backward dX = W^T dY and dW = dY x^T for every
    layer (the sources require grad here); layer 1 counts its dense rows only."""
    _, _, c_in, widths, _, _, src_w = spec
    k_in, f = sum(src_w), 0
    for c in widths:
        f += 3 * 2 * B * N * c * k_in
        k_in = c
    return f


def bench_chain(spec, dev, reps):
    torch_fn, fused_fn, pn, srcs, B = chain_case(spec, dev)
    params = list(pn.parameters()) + srcs

    def step(fn):
        for p in params:
            p.grad = None
        fn().sum().backward()

    for _ in range(3):
        step(torch_fn)
        step(fused_fn)
    torch.cuda.synchronize()
    t_ms, f_ms = [], []
    for _ in range(5):
        t_ms.append(_block_ms(lambda: step(torch_fn), reps))
        f_ms.append(_block_ms(lambda: step(fused_fn), reps))
    peaks = {}
    for kind, fn in (("torch", torch_fn), ("fused", fused_fn)):
        for p in params:
            p.grad = None
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        step(fn)
        torch.cuda.synchronize()
        peaks[kind] = torch.cuda.max_memory_allocated() - base
    fused = float(np.median(f_ms))
    flops = gemm_flops(spec, B)
    return {"B": B, "points": N, "widths": spec[3], "torch_fwd_bwd_ms": float(np.median(t_ms)),
            "fused_fwd_bwd_ms": fused, "torch_blocks_ms": t_ms, "fused_blocks_ms": f_ms, "calls_per_block": reps,
            "torch_peak_bytes": peaks["torch"], "fused_peak_bytes": peaks["fused"],
            "fused_gemm_tflop": flops / 1e12, "fused_tf32_tflops_per_s": flops / (fused * 1e-3) / 1e12,
            "fused_share_of_tf32_datasheet": flops / (fused * 1e-3) / TF32_PEAK}


def model_for(shape, dev, point_layers):
    m = network.KeypointDetector(**network.SHAPES[shape], point_layers=point_layers)
    m.load_state_dict(synthetic.seeded_state_dict(m, 1))
    return m.to(dev)


def step_times(shape, dev, reps):
    """The captured step of both modes, replays timed in alternating blocks; medians over the blocks."""
    x = inputs(shape, dev)
    graphs = {}
    for mode in ("torch", "fused"):
        m = model_for(shape, dev, mode)
        o = train.make_optimizer(m)
        for _ in range(train.WARMUP_STEPS):
            train.train_step(m, o, x)
        o.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            train.train_step(m, o, x)
        g.replay()
        torch.cuda.synchronize()
        graphs[mode] = (g, m, o)
    ms = {"torch": [], "fused": []}
    for _ in range(5):
        for mode in ("torch", "fused"):
            ms[mode].append(_block_ms(graphs[mode][0].replay, reps))
    del graphs
    S, (H, W) = SHAPES[shape]
    return {"B": S, "points": N, "image": [H, W], "torch_captured_step_ms": float(np.median(ms["torch"])),
            "fused_captured_step_ms": float(np.median(ms["fused"])), "torch_blocks_ms": ms["torch"],
            "fused_blocks_ms": ms["fused"], "steps_per_block": reps}


def step_peaks(shape, dev):
    """Peak allocation of one eager training step per mode, with only that mode's model, its Adam state and the
    inputs alive (the other mode's model is freed first)."""
    x = inputs(shape, dev)
    out = {}
    for mode in ("torch", "fused"):
        m = model_for(shape, dev, mode)
        o = train.make_optimizer(m)
        for _ in range(train.WARMUP_STEPS):
            train.train_step(m, o, x)
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        train.train_step(m, o, x)
        torch.cuda.synchronize()
        out[mode] = {"peak_bytes": torch.cuda.max_memory_allocated(), "allocated_before_step_bytes": before,
                     "step_peak_above_resident_bytes": torch.cuda.max_memory_allocated() - before}
        del m, o
        torch.cuda.empty_cache()
    return out


def _subtree(e):
    out, stack = [], [e]
    while stack:
        v = stack.pop()
        out.append(v)
        stack.extend(v.cpu_children)
    return out


def _kernel_us(events):
    return sum(k.duration for e in events for k in e.kernels)


def attribution(shape, dev, steps=3):
    """torch.profiler over eager steps of the torch-mode model: the kernel time of each chain's forward (the kernels
    launched inside its module) and backward (the kernels of the autograd nodes whose sequence numbers its forward
    ops recorded), against the step's kernel time.  Eager steps, because graph replays carry no CPU op to tie a kernel
    to; the kernels are the ones the captured step replays."""
    from torch.profiler import ProfilerActivity, profile, record_function
    x = inputs(shape, dev)
    m = model_for(shape, dev, "torch")
    o = train.make_optimizer(m)
    chains = {"first_pointnet": m.pc_encoder.first_pointnet, "second_pointnet": m.pc_encoder.second_pointnet,
              "per_point_pn": m.per_point_pn}
    open_ranges, handles = [], []
    for name, mod in chains.items():
        def pre(_m, _a, name=name):
            r = record_function("chain::" + name)
            r.__enter__()
            open_ranges.append(r)

        def post(_m, _a, _o):
            open_ranges.pop().__exit__(None, None, None)
        handles += [mod.register_forward_pre_hook(pre), mod.register_forward_hook(post)]
    for _ in range(train.WARMUP_STEPS):
        train.train_step(m, o, x)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            train.train_step(m, o, x)
        torch.cuda.synchronize()
    for h in handles:
        h.remove()
    events = list(prof.events())
    total = _kernel_us(events)
    bwd = [e for e in events if e.name.startswith("autograd::engine::evaluate_function")]
    res = {"steps": steps, "step_kernel_ms": total / steps / 1e3, "chains": {}}
    for name in chains:
        ranges = [e for e in events if e.name == "chain::" + name]
        fwd_ev = [v for r in ranges for v in _subtree(r)]
        seq = {v.sequence_nr for v in fwd_ev if v.sequence_nr is not None and v.sequence_nr >= 0}
        bwd_ev = [v for e in bwd if e.sequence_nr in seq for v in _subtree(e)]
        f_us, b_us = _kernel_us(fwd_ev), _kernel_us(bwd_ev)
        res["chains"][name] = {"forward_kernel_ms": f_us / steps / 1e3, "backward_kernel_ms": b_us / steps / 1e3,
                               "backward_nodes": len([e for e in bwd if e.sequence_nr in seq]) // steps,
                               "share_of_step_kernel_time": (f_us + b_us) / total if total else None}
    res["three_chains_share_of_step_kernel_time"] = \
        sum((v["forward_kernel_ms"] + v["backward_kernel_ms"]) for v in res["chains"].values()) / \
        res["step_kernel_ms"] if total else None
    del m, o
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="BENCH_POINT_CHAIN.json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_point_chain.py needs a CUDA device")
    dev = torch.device("cuda")
    torch.backends.cudnn.benchmark = False
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit": _power_limit(), "torch": torch.__version__,
           "tf32_datasheet_flops": TF32_PEAK, "chains": {}, "step": {}}
    for spec in CHAINS:
        res["chains"][spec[0]] = bench_chain(spec, dev, a.reps)
        print(json.dumps({spec[0]: res["chains"][spec[0]]}), flush=True)
    for shape in ("kitti", "oxford", "nuscenes"):
        res["step"][shape] = step_times(shape, dev, a.reps)
        print(json.dumps({shape: res["step"][shape]}), flush=True)
    res["step_peak"], res["attribution"] = {}, {}
    for shape in ("kitti", "oxford", "nuscenes"):
        res["step_peak"][shape] = step_peaks(shape, dev)
        res["attribution"][shape] = attribution(shape, dev)
        print(json.dumps({shape: {"peak": res["step_peak"][shape], "attribution": res["attribution"][shape]}}),
              flush=True)
    with open(a.out, "w") as f:
        json.dump({"point_chain": res}, f)
    print(json.dumps({"point_chain": res}))


if __name__ == "__main__":
    main()
