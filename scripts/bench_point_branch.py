"""Benchmark of the classifier's kNN module, final_pointnet + global max and node-level PointNets in training
(point_ops.point_branch, KeypointDetector(point_layers="fused_all"), DESIGN.md 4.36): writes BENCH_POINT_BRANCH.json.

- modules: forward + backward of each module, the model's torch layers (cuDNN, torch.cat, torch.max) against
  point_branch, at KITTI / Oxford (B = 8) and nuScenes (B = 12) shapes with 128 nodes and K = 16; the two alternate
  run by run, and the median and range of the per-run times and each side's peak allocation are reported;
- fused rate: the fused module's products (2 B N C_in C_out per layer forward, twice that backward) over its time;
- step: the captured KITTI training step (B = 8) of each point_layers mode, and one eager step's peak allocation;
- attribution: torch.profiler over eager steps of the torch-mode KITTI model (B = 8), the kernel time of each
  module's forward (the kernels launched inside it) and backward (the kernels of the autograd nodes its forward ops
  recorded), against the step's kernel time, as bench_point_chain.py does for the per-point chains; final_pointnet's
  global max is a torch.max outside the module and is not in its share;
- the GPU's name and power limit, read in the same run.

    python scripts/bench_point_branch.py [--reps 20] [--out BENCH_POINT_BRANCH.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepi2p_b200 import network, point_ops, synthetic, train  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_point_chain import _kernel_us, _subtree  # noqa: E402


def _time(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return ts


def _peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def _model(shape, mode="fused_all"):
    m = network.KeypointDetector(**network.SHAPES[shape], point_layers=mode)
    m.load_state_dict(synthetic.seeded_state_dict(m, 1))
    return m.cuda().train()


def _modules(shape, B, M=128, K=16):
    """{name: (torch fn, fused fn, fused forward flops)} with fresh leaf inputs per call."""
    m = _model(shape)
    g = torch.Generator(device="cuda").manual_seed(0)
    r = lambda *s: torch.randn(s, device="cuda", generator=g).requires_grad_()
    naf, nbf, nb, cm = r(B, 64, M), r(B, 256, M), torch.randn((B, 3, M), device="cuda"), torch.randn((B, 3, M),
                                                                                                     device="cuda")
    ig, gf, ws32, ws16, ab = r(B, 512), r(B, 512), r(B, 512, M), r(B, 256, M), r(B, 512, M)
    e = lambda v: v[:, :, None].expand(-1, -1, M)
    enc = m.pc_encoder
    L4 = m.node_a_attention_pn.layers[-1].conv.out_channels

    def bwd(out):
        out.sum().backward()

    def flops(cols, layers):
        return sum(2 * B * cols * c_in * c_out for c_in, c_out in layers)

    mods = {
        "knn": (lambda: bwd(enc.knnlayer(nb, cm, naf, K)), lambda: bwd(m._fused_knn(nb, cm, naf)),
                flops(M * K, [(67, 256), (256, 256), (256, 512), (512, 256)]) + flops(M, [(256, 512)])),
        "final_max": (lambda: bwd(torch.max(enc.final_pointnet(torch.cat((nb, nbf), 1)), dim=2)[0]),
                      lambda: bwd(point_ops.point_branch([nb, nbf], list(enc.final_pointnet.layers), None,
                                                         max_group=M, output="max")),
                      flops(M, [(259, 256), (256, 512)])),
        "node_b_attention_pn": (
            lambda: bwd(m.node_b_attention_pn(torch.cat((nbf, e(ig)), 1))),
            lambda: bwd(m._fused_node(m.node_b_attention_pn, [nbf], [0], [(256, ig)], M)),
            flops(M, [(256, 256), (256, L4 // 4)])),
        "node_b_pn": (
            lambda: bwd(m.node_b_pn(torch.cat((nbf, e(gf), ws32, e(ig)), 1))),
            lambda: bwd(m._fused_node(m.node_b_pn, [nbf, ws32], [0, 768], [(256, gf), (1280, ig)], M)),
            flops(M, [(768, 1024), (1024, 512), (512, 512)])),
        "node_a_attention_pn": (
            lambda: bwd(m.node_a_attention_pn(torch.cat((naf, e(ig)), 1))),
            lambda: bwd(m._fused_node(m.node_a_attention_pn, [naf], [0], [(64, ig)], M)),
            flops(M, [(64, 256), (256, L4)])),
        "node_a_pn": (
            lambda: bwd(m.node_a_pn(torch.cat((naf, ab, ws16), 1))),
            lambda: bwd(m._fused_node(m.node_a_pn, [naf, ab, ws16], None, [], M)),
            flops(M, [(832, 512), (512, 128), (128, 128)])),
    }
    return mods


def _inputs(S, seed):
    import numpy as np
    rng = np.random.default_rng(seed)
    smps = [synthetic.make_sample(seed + s, 20480, "kitti") for s in range(S)]
    pc = torch.from_numpy(np.stack([s["points"] for s in smps])).cuda()
    idx = torch.from_numpy(np.stack([rng.permutation(20480)[:256] for _ in range(S)])).cuda()
    nodes = torch.gather(pc, 2, idx.unsqueeze(1).expand(S, 3, 256))
    return dict(pc=pc, intensity=torch.from_numpy(rng.random((S, 1, 20480), dtype=np.float32)).cuda(),
                sn=torch.from_numpy(rng.standard_normal((S, 3, 20480), dtype=np.float32)).cuda(),
                node_a=nodes[:, :, :128].contiguous(), node_b=nodes[:, :, 128:].contiguous(),
                img=torch.from_numpy(rng.random((S, 3, 160, 512), dtype=np.float32)).cuda(),
                K=torch.from_numpy(np.stack([s["K"] for s in smps])).float().cuda(),
                P=torch.from_numpy(np.stack([s["P_gt"][:3] for s in smps])).float().cuda())


def _step(mode, reps, B=8):
    m = _model("kitti", mode)
    opt = train.make_optimizer(m)
    static = _inputs(B, 300)
    stats = torch.zeros(5, device="cuda")
    for _ in range(train.WARMUP_STEPS):
        stats.copy_(train._stats(train.train_step(m, opt, static)))
    eager = statistics.median(_time(lambda: train.train_step(m, opt, static), max(3, reps // 4)))
    peak = _peak(lambda: train.train_step(m, opt, static))
    opt.zero_grad(set_to_none=True)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        stats.copy_(train._stats(train.train_step(m, opt, static)))
    ts = _time(graph.replay, reps)
    return dict(captured_ms=statistics.median(ts), captured_range_ms=[min(ts), max(ts)], eager_ms=eager,
                eager_peak_mib=peak)


def _attribution(B=8, steps=3):
    from torch.profiler import ProfilerActivity, profile, record_function
    m = _model("kitti", "torch")
    opt = train.make_optimizer(m)
    x = _inputs(B, 301)
    mods = {"knn": m.pc_encoder.knnlayer, "final_pointnet": m.pc_encoder.final_pointnet,
            "node_b_attention_pn": m.node_b_attention_pn, "node_b_pn": m.node_b_pn,
            "node_a_attention_pn": m.node_a_attention_pn, "node_a_pn": m.node_a_pn}
    open_ranges, handles = [], []
    for name, mod in mods.items():
        def pre(_m, _a, name=name):
            r = record_function("branch::" + name)
            r.__enter__()
            open_ranges.append(r)

        def post(_m, _a, _o):
            open_ranges.pop().__exit__(None, None, None)
        handles += [mod.register_forward_pre_hook(pre), mod.register_forward_hook(post)]
    for _ in range(train.WARMUP_STEPS):
        train.train_step(m, opt, x)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            train.train_step(m, opt, x)
        torch.cuda.synchronize()
    for h in handles:
        h.remove()
    events = list(prof.events())
    total = _kernel_us(events)
    bwd = [e for e in events if e.name.startswith("autograd::engine::evaluate_function")]
    res = {"steps": steps, "step_kernel_ms": total / steps / 1e3, "modules": {}}
    for name in mods:
        fwd_ev = [v for r in events if r.name == "branch::" + name for v in _subtree(r)]
        seq = {v.sequence_nr for v in fwd_ev if v.sequence_nr is not None and v.sequence_nr >= 0}
        bwd_ev = [v for e in bwd if e.sequence_nr in seq for v in _subtree(e)]
        f_us, b_us = _kernel_us(fwd_ev), _kernel_us(bwd_ev)
        res["modules"][name] = {"forward_kernel_ms": f_us / steps / 1e3, "backward_kernel_ms": b_us / steps / 1e3,
                                "share_of_step_kernel_time": (f_us + b_us) / total if total else None}
    res["six_modules_share_of_step_kernel_time"] = sum(v["share_of_step_kernel_time"] or 0
                                                       for v in res["modules"].values())
    del m, opt
    torch.cuda.empty_cache()
    return res


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="BENCH_POINT_BRANCH.json")
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_point_branch.py needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    res = {"gpu": q[0] if q else torch.cuda.get_device_name(), "modules": {}, "step": {}}
    for shape, B in (("kitti", 8), ("oxford", 8), ("nuscenes", 12)):
        for name, (tf, ff, fl) in _modules(shape, B).items():
            for fn in (tf, ff, tf, ff):          # warm both sides (algorithm choice, workspaces)
                fn()
            tt, tfu = [], []
            for _ in range(a.reps):
                tt += _time(tf, 1)
                tfu += _time(ff, 1)
            res["modules"][f"{shape}/{name}"] = dict(
                B=B, torch_ms=statistics.median(tt), torch_range_ms=[min(tt), max(tt)],
                fused_ms=statistics.median(tfu), fused_range_ms=[min(tfu), max(tfu)],
                torch_peak_mib=_peak(tf), fused_peak_mib=_peak(ff),
                fused_tf32_tflops=3 * fl / (statistics.median(tfu) * 1e-3) / 1e12)
    for mode in network.POINT_LAYERS:
        res["step"][mode] = _step(mode, a.reps)
    res["attribution"] = _attribution()
    with open(a.out, "w") as f:
        json.dump({"point_branch": res}, f)
    print(json.dumps({"point_branch": res}))


if __name__ == "__main__":
    main()
