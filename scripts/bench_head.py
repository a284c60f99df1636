"""The classifier's per-point layers, unfused (torch) against fused (point_ops.pointwise_mlp, DESIGN.md 4.21).

    python scripts/bench_head.py [--chunk 64] [--reps 7] [--samples 1024] [--out BENCH_HEAD.json]
    python scripts/bench_head.py --accounting          # operations and bytes from the shapes; needs no GPU

At the Oxford and KITTI shapes (20480 points, 128 + 128 nodes, seeded untrained weights from bench_e2e's builders),
one chunk of `--chunk` samples:
- head: the two per-point interpolations, the 736-row torch.cat, per_point_pn and network.predict, against
  interpolation_weights x 2 + one pointwise_mlp call with the arg-max output, on the same captured inputs;
- encoder: first_pointnet and second_pointnet with their torch.cat, against the two pointwise_mlp calls;
- forward: model.forward + predict against FusedInference.classify; and config 5 (network.classify_and_register over
  `--samples` Oxford samples, 60 inits) with head="torch" and head="fused".
Torch and fused alternate within one run; times are CUDA events after a warm-up, reported as the median with the
minimum and maximum; peak is max_memory_allocated above what was resident before the call.  The fraction of points
whose prediction differs between the two heads is measured at the timed size.  The kernel's share of its bounding
peak uses the operations and bytes this script computes from the shapes (the fused formulation; compulsory traffic
only) and the data-sheet rates of the H100 SXM (495 TFLOP/s dense TF32, 3.35 TB/s); the bound that is larger is
named.  A run without a CUDA device fails unless --accounting is given.  Prints one JSON line with the GPU name and
power limit read in the same run; --out writes it to a file.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from deepi2p_b200 import network, point_ops  # noqa: E402

ARGS = ("pc", "intensity", "sn", "node_a", "node_b", "img")
PEAK_TF32, PEAK_BW = 495e12, 3.35e12          # H100 SXM data sheet, dense TF32 FLOP/s and HBM3 bytes/s at 700 W


def accounting(shape, chunk, N=20480, M=128, k=3):
    """Operations and compulsory bytes of the three fused calls for one chunk, from the shapes."""
    H, W = network.SHAPES[shape]["img_H"], network.SHAPES[shape]["img_W"]
    L = round(H / 32) * round(W / 32)
    pts = chunk * N

    def chain(dense_rows, widths, interp_rows=()):
        flop, c_in = 0, dense_rows
        for c in widths:
            flop += 2 * c_in * c * pts
            c_in = c
        flop += sum(2 * r * widths[0] * M * chunk for r in interp_rows)            # node projections
        flop += 2 * len(interp_rows) * k * widths[0] * pts                          # per-point interpolation
        unfused = 2 * pts * sum(a * b for a, b in zip([dense_rows + sum(interp_rows)] + widths[:-1], widths))
        read = 4 * dense_rows * pts + sum(4 * r * M * chunk + 8 * k * pts for r in interp_rows)
        return flop, unfused, read

    head = chain(96, [256, 256, 2 + L], (128, 512))
    first, second = chain(7, [32, 32, 32]), chain(64, [64, 64])
    out = {"L": L, "points": pts,
           "head": {"flop_fused_formulation": head[0], "flop_unfused_formulation": head[1],
                    "bytes_compulsory": head[2] + 5 * pts},
           "encoder": {"flop_fused_formulation": first[0] + second[0], "flop_unfused_formulation": first[1] + second[1],
                       "bytes_compulsory": first[2] + second[2] + 4 * (32 + 64) * pts}}
    for v in (out["head"], out["encoder"]):
        t_flop, t_bw = v["flop_fused_formulation"] / PEAK_TF32, v["bytes_compulsory"] / PEAK_BW
        v["bound"] = "tensor-core TF32 rate" if t_flop >= t_bw else "HBM bandwidth"
        v["least_ms_at_data_sheet_rates"] = max(t_flop, t_bw) * 1e3
    return out


def _timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def alternate(fns, reps):
    """{name: dict(ms median, min, max, peak bytes above the resident set)} with the candidates interleaved."""
    res = {}
    for name, fn in fns.items():
        fn()                                                 # warm-up: module load, algorithm choice, allocator
        fn()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        fn()
        torch.cuda.synchronize()
        res[name] = {"peak_bytes_above_resident": torch.cuda.max_memory_allocated() - base, "ms_all": []}
    for _ in range(reps):
        for name, fn in fns.items():
            res[name]["ms_all"].append(_timed(fn))
    for v in res.values():
        v["ms"], v["ms_min"], v["ms_max"] = float(np.median(v["ms_all"])), min(v["ms_all"]), max(v["ms_all"])
    return res


def capture(model, b):
    """One unfused forward with hooks: the inputs of the per-point layers and the decoder's node features."""
    got = {}
    hooks = [model.pc_encoder.first_pointnet.register_forward_pre_hook(lambda m, x: got.__setitem__("first_in", x[0])),
             model.pc_encoder.second_pointnet.register_forward_pre_hook(lambda m, x: got.__setitem__("second_in", x[0])),
             model.per_point_pn.register_forward_pre_hook(lambda m, x: got.__setitem__("head_in", x[0])),
             model.node_a_pn.register_forward_hook(lambda m, x, y: got.__setitem__("up_a", y)),
             model.node_b_pn.register_forward_hook(lambda m, x, y: got.__setitem__("up_b", y))]
    with torch.no_grad():
        model(*(b[k] for k in ARGS))
    for h in hooks:
        h.remove()
    return got


def one_shape(shape, a, dev):
    from bench_e2e import batch, model_for
    b = batch(a.chunk, shape, 1000, dev)
    model = model_for(shape, dev).eval()
    fused = network.FusedInference(model)
    g = capture(model, b)
    pc, node_a, node_b = b["pc"], b["node_a"], b["node_b"]
    idx_a = point_ops.cluster_assign_forward(pc, node_a, k=3, want_centers=False)["min_k_idx"]
    idx_b = point_ops.cluster_assign_forward(pc, node_b, k=3, want_centers=False)["min_k_idx"]
    first_out, second_out = g["head_in"][:, 640:672].contiguous(), g["head_in"][:, 672:].contiguous()
    first_srcs = [g["first_in"][:, 0:3].contiguous(), g["first_in"][:, 3:4].contiguous(),
                  g["first_in"][:, 4:7].contiguous()]
    scattered = g["second_in"][:, 32:].contiguous()
    up_a, up_b = g["up_a"], g["up_b"]
    del g
    enc = model.pc_encoder
    keep = {}

    def head_torch():
        with torch.no_grad():
            pa = point_ops.upsample_by_interpolation(idx_a, pc, node_a, up_a)
            pb = point_ops.upsample_by_interpolation(idx_b, pc, node_b, up_b)
            s = model.per_point_pn(torch.cat((pa, pb, first_out, second_out), dim=1))
            keep["torch"] = network.predict(s[:, :2], s[:, 2:])

    def head_fused():
        with torch.no_grad():
            wa, ia = point_ops.interpolation_weights(idx_a, pc, node_a)
            wb, ib = point_ops.interpolation_weights(idx_b, pc, node_b)
            keep["fused"] = point_ops.pointwise_mlp([(up_a, wa, ia), (up_b, wb, ib), first_out, second_out],
                                                    fused._chain("head"), output="argmax", c_split=2)

    def enc_torch():
        with torch.no_grad():
            f = enc.first_pointnet(torch.cat(first_srcs, dim=1))
            keep["enc"] = enc.second_pointnet(torch.cat((f, scattered), dim=1))

    def enc_fused():
        with torch.no_grad():
            f = point_ops.pointwise_mlp(first_srcs, fused._chain("first"))
            keep["enc"] = point_ops.pointwise_mlp([f, scattered], fused._chain("second"))

    def fwd_torch():
        with torch.no_grad():
            keep["fwd"] = network.predict(*model(*(b[k] for k in ARGS)))

    def fwd_fused():
        with torch.no_grad():
            keep["fwd"] = fused.classify(*(b[k] for k in ARGS))

    res = {"head": alternate({"torch": head_torch, "fused": head_fused}, a.reps)}
    differ = [float((x != y).float().mean()) for x, y in zip(keep["torch"], keep["fused"])]
    res["head"]["fraction_of_points_predicted_differently"] = {"coarse": differ[0], "fine": differ[1]}
    keep.clear()
    res["encoder"] = alternate({"torch": enc_torch, "fused": enc_fused}, a.reps)
    keep.clear()
    res["forward"] = alternate({"torch": fwd_torch, "fused": fwd_fused}, a.reps)
    keep.clear()
    acc = accounting(shape, a.chunk)
    for part in ("head", "encoder"):
        least = acc[part]["least_ms_at_data_sheet_rates"]
        res[part]["fused_share_of_bounding_peak"] = least / res[part]["fused"]["ms"]
        res[part]["bound"] = acc[part]["bound"]
    res["accounting"] = acc
    return res


def config5(a, dev):
    from bench_e2e import batch, model_for
    b = batch(a.samples, "oxford", 1000, dev)
    model = model_for("oxford", dev).eval()
    fns = {h: (lambda h=h: network.classify_and_register(model, *(b[k] for k in ARGS), b["K"], chunk=a.chunk, head=h))
           for h in ("torch", "fused")}
    res = alternate(fns, max(3, a.reps // 2))
    res.update(samples=a.samples, chunk=a.chunk, n_inits=60,
               note="seeded untrained weights: the registration solves meaningless predictions, which differ "
                    "between the heads, so its time differs too")
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
        raise SystemExit("bench_head.py needs a CUDA device (--accounting runs without one)")
    from bench_prep import _power_limit
    dev = torch.device("cuda:0")
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit": _power_limit(),
           "tf32_flags_of_the_torch_path": [torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32],
           "chunk": a.chunk, "reps": a.reps}
    for shape in ("oxford", "kitti"):
        print(f"bench_head: {shape}", file=sys.stderr, flush=True)
        res[shape] = one_shape(shape, a, dev)
        torch.cuda.empty_cache()
    if a.samples > 0:
        print("bench_head: config 5", file=sys.stderr, flush=True)
        res["config5_oxford"] = config5(a, dev)
    print(json.dumps({"head": res}))
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps({"head": res}) + "\n")


if __name__ == "__main__":
    main()
