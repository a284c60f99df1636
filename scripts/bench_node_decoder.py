"""The decoder's four node-level PointNets, torch layers against the fused node_mlp op (DESIGN.md 4.27).

    python scripts/bench_node_decoder.py [--chunk 64] [--reps 7] [--samples 1024] [--out BENCH_NODE_DECODER.json]
    python scripts/bench_node_decoder.py --accounting     # operations from the shapes; needs no GPU

At the Oxford and KITTI shapes (20480 points, 128 + 128 nodes, seeded untrained weights from bench_e2e's builders),
one chunk of `--chunk` samples:
- modules: node_b_attention_pn, node_b_pn, node_a_attention_pn and node_a_pn, each as network.py runs it (torch.cat
  of the expanded per-sample inputs, cuDNN convolutions, BatchNorm, ReLU) against one point_ops.node_mlp call, on the
  same captured inputs;
- forward: FusedInference.classify with encoder="fused" (head "fused_encoder") against encoder="fused",
  decoder="fused" (head "fused_all");
- profile: in a torch.profiler run of its own, one forward of each head, and the share of the device time spent in
  the node-level PointNets (the modules' kernels and their torch.cat copies, or the node_mlp kernels);
and config 5 (network.classify_and_register over `--samples` Oxford samples, 60 inits) with both heads.
The candidates alternate within one run (bench_head.alternate): CUDA events after a warm-up, the median of --reps with
the minimum and maximum; peak is max_memory_allocated above what was resident before the call.  The fused kernels'
share of the TF32 bound is the time their operations (computed here from the shapes) take at the H100 SXM
data-sheet rate, 495 TFLOP/s dense TF32, over the measured time.  Prints one JSON line with the GPU name and power
limit read in the same run; --out writes it to a file.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from deepi2p_b200 import classifier, network, point_ops  # noqa: E402
from bench_head import ARGS, PEAK_TF32, alternate  # noqa: E402

MODULES = ("att_b", "node_b", "att_a", "node_a")
ATTR = {"att_b": "node_b_attention_pn", "node_b": "node_b_pn", "att_a": "node_a_attention_pn", "node_a": "node_a_pn"}


def accounting(shape, chunk, M=128):
    """FLOP of each node-level PointNet for one chunk from the shapes: the torch formulation (every input row per
    column) and the fused one (the per-sample rows once per sample)."""
    H_f, W_f = classifier.fine_grid(network.SHAPES[shape]["img_H"], network.SHAPES[shape]["img_W"], 32)
    L = H_f * W_f
    out = {}
    for name, (get, spec) in network.FusedInference._NODE_CHAINS.items():
        widths = {"att_b": (256, L), "node_b": (1024, 512, 512), "att_a": (256, 4 * L), "node_a": (512, 128, 128)}[name]
        c_in = sum(c for c, _ in spec)
        per_sample = sum(c for c, bc in spec if bc)
        later = sum(a * b for a, b in zip(widths, widths[1:]))
        torch_flop = 2 * chunk * M * (c_in * widths[0] + later)
        fused_flop = 2 * chunk * M * ((c_in - per_sample) * widths[0] + later) + 2 * chunk * per_sample * widths[0]
        out[name] = {"input_rows": c_in, "per_sample_rows": per_sample, "widths": list(widths),
                     "flop_torch_formulation": torch_flop, "flop_fused_formulation": fused_flop,
                     "least_ms_at_tf32_data_sheet_rate": fused_flop / PEAK_TF32 * 1e3}
    return out


def capture(model, b):
    """One forward with hooks: each node-level PointNet's concatenated input."""
    got = {}
    hooks = [getattr(model, ATTR[n]).register_forward_pre_hook(lambda m, x, n=n: got.__setitem__(n, x[0]))
             for n in MODULES]
    with torch.no_grad():
        model(*(b[k] for k in ARGS))
    for h in hooks:
        h.remove()
    return got


def split(name, x):
    """The sources node_mlp takes, from a captured concatenated input: dense slices and per-sample [B, C] columns."""
    _, spec = network.FusedInference._NODE_CHAINS[name]
    out, r = [], 0
    for c, bc in spec:
        out.append(x[:, r:r + c, 0].contiguous() if bc else x[:, r:r + c].contiguous())
        r += c
    return out


def node_level_share(model, b):
    """Device time of one forward per head under torch.profiler, and the part spent in the node-level PointNets: the
    kernels launched inside the four modules (a record_function range around each) and the torch.cat copies for the
    torch layers, the node_mlp kernels for the fused ones."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile, record_function
    heads = {"fused_encoder": network.FusedInference(model, encoder="fused"),
             "fused_all": network.FusedInference(model, encoder="fused", decoder="fused")}

    def enter(m, x):
        m._node_range = record_function("node_level")
        m._node_range.__enter__()

    def leave(m, x, y):
        m._node_range.__exit__(None, None, None)
        del m._node_range

    def kernel_us(e):
        return sum(k.duration for k in e.kernels) + sum(kernel_us(c) for c in e.cpu_children)

    res = {}
    for head, f in heads.items():
        with torch.no_grad():
            f.classify(*(b[k] for k in ARGS))
            torch.cuda.synchronize()
            hooks = [h for n in MODULES for h in (getattr(model, ATTR[n]).register_forward_pre_hook(enter),
                                                   getattr(model, ATTR[n]).register_forward_hook(leave))]
            try:
                with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                    f.classify(*(b[k] for k in ARGS))
                    torch.cuda.synchronize()
            finally:
                for h in hooks:
                    h.remove()
        total = fused = modules = cat = 0.0
        for e in prof.events():
            if e.device_type == DeviceType.CUDA and e.name != "node_level":
                t = e.time_range.elapsed_us()
                total += t
                if "nm_kernel" in e.name or "nm_proj_kernel" in e.name:
                    fused += t
                elif "CatArrayBatchedCopy" in e.name:
                    cat += t
            elif e.device_type == DeviceType.CPU and e.name == "node_level":
                modules += kernel_us(e)
        node = fused + modules + cat
        res[head] = {"device_us": total, "node_level_us": node, "of_which_node_mlp_kernels_us": fused,
                     "of_which_torch_module_kernels_us": modules, "of_which_torch_cat_us": cat,
                     "node_level_share": node / total if total else None}
    return res


def one_shape(shape, a, dev):
    from bench_e2e import batch, model_for
    b = batch(a.chunk, shape, 1000, dev)
    model = model_for(shape, dev).eval()
    enc, full = network.FusedInference(model, encoder="fused"), network.FusedInference(model, encoder="fused",
                                                                                        decoder="fused")
    g = capture(model, b)
    acc = accounting(shape, a.chunk)
    keep = {}
    res = {"modules": {}}
    for n in MODULES:
        x = g[n]
        src = split(n, x)
        _, spec = network.FusedInference._NODE_CHAINS[n]
        parts = [s if not bc else s.unsqueeze(2).expand(-1, -1, x.shape[2]) for s, (_, bc) in zip(src, spec)]
        mod = getattr(model, ATTR[n])

        def run_torch(mod=mod, parts=parts):
            with torch.no_grad():
                keep["y"] = mod(torch.cat(parts, dim=1))

        def run_fused(n=n, src=src):
            with torch.no_grad():
                keep["y"] = point_ops.node_mlp(src, full._chain(n))

        r = alternate({"torch": run_torch, "fused": run_fused}, a.reps)
        with torch.no_grad():
            t, f = mod(x), point_ops.node_mlp(src, full._chain(n))
        r["max_abs_difference_over_max_abs"] = float((t - f).abs().max() / t.abs().max())
        r["fused_faster"] = r["fused"]["ms"] < r["torch"]["ms"]
        r["fused_share_of_tf32_bound"] = acc[n]["least_ms_at_tf32_data_sheet_rate"] / r["fused"]["ms"]
        r["accounting"] = acc[n]
        res["modules"][n] = r
        keep.clear()
    del g

    def fwd(f):
        def run():
            with torch.no_grad():
                keep["fwd"] = f.classify(*(b[k] for k in ARGS))
        return run

    res["forward"] = alternate({"fused_encoder": fwd(enc), "fused_all": fwd(full)}, a.reps)
    res["forward"]["fused_all_faster"] = res["forward"]["fused_all"]["ms"] < res["forward"]["fused_encoder"]["ms"]
    for side, head in (("torch", "fused_encoder"), ("fused", "fused_all")):
        # a cross-check of the profiler's share: the four modules' separately timed medians over the forward's
        res["forward"][head]["node_level_share_from_module_timings"] = \
            sum(res["modules"][n][side]["ms"] for n in MODULES) / res["forward"][head]["ms"]
    with torch.no_grad():
        p0, p1 = enc.classify(*(b[k] for k in ARGS)), full.classify(*(b[k] for k in ARGS))
    res["forward"]["fraction_of_points_predicted_differently"] = {
        "coarse": float((p0[0] != p1[0]).float().mean()), "fine": float((p0[1] != p1[1]).float().mean())}
    keep.clear()
    try:
        res["profile"] = node_level_share(model, b)
    except Exception as e:  # noqa: BLE001 - the timings above stand on their own
        res["profile"] = {"error": repr(e)}
    return res


def config5(a, dev):
    from bench_e2e import batch, model_for
    b = batch(a.samples, "oxford", 1000, dev)
    model = model_for("oxford", dev).eval()
    fns = {h: (lambda h=h: network.classify_and_register(model, *(b[k] for k in ARGS), b["K"], chunk=a.chunk, head=h))
           for h in ("fused_encoder", "fused_all")}
    res = alternate(fns, max(3, a.reps // 2))
    res.update(samples=a.samples, chunk=a.chunk, n_inits=60,
               note="seeded untrained weights: the registration solves meaningless predictions, which can differ "
                    "between the heads, so its time can differ too")
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunk", type=int, default=network.DEFAULT_CHUNK)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--samples", type=int, default=1024)
    ap.add_argument("--accounting", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.accounting:
        print(json.dumps({s: accounting(s, a.chunk) for s in ("oxford", "kitti")}))
        return
    if not torch.cuda.is_available():
        raise SystemExit("bench_node_decoder.py needs a CUDA device (--accounting runs without one)")
    from bench_prep import _power_limit
    dev = torch.device("cuda:0")
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit": _power_limit(),
           "tf32_flags_of_the_torch_path": [torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32],
           "chunk": a.chunk, "reps": a.reps}
    for shape in ("oxford", "kitti"):
        print(f"bench_node_decoder: {shape}", file=sys.stderr, flush=True)
        res[shape] = one_shape(shape, a, dev)
        torch.cuda.empty_cache()
    if a.samples > 0:
        print("bench_node_decoder: config 5", file=sys.stderr, flush=True)
        res["config5_oxford"] = config5(a, dev)
    print(json.dumps({"node_decoder": res}))
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps({"node_decoder": res}) + "\n")


if __name__ == "__main__":
    main()
