"""The point encoder's kNN module and global feature, unfused (torch) against fused (point_ops.knn_fusion and
point_ops.pointwise_mlp_max, DESIGN.md 4.26).

    python scripts/bench_knn_fusion.py [--chunk 64] [--reps 7] [--samples 1024] [--out BENCH_KNN_FUSION.json]
    python scripts/bench_knn_fusion.py --accounting     # operations and bytes from the shapes; needs no GPU

At the Oxford and KITTI shapes (20480 points, 128 + 128 nodes, K = 16, seeded untrained weights from bench_e2e's
builders), one chunk of `--chunk` samples:
- knnlayer: _KnnFusion.forward (knn_group, cuDNN convolutions, BatchNorm, ReLU, torch.cat, two max) against one
  knn_fusion call, on the same captured inputs;
- final: final_pointnet over torch.cat((node_b, node_b_features)) + torch.max over the nodes against one
  pointwise_mlp_max call;
- forward: FusedInference.classify with encoder="torch" against encoder="fused"; and config 5
  (network.classify_and_register over `--samples` Oxford samples, 60 inits) with head="fused" and "fused_encoder".
The candidates alternate within one run (bench_head.alternate): CUDA events after a warm-up, the median of --reps
with the minimum and maximum; peak is max_memory_allocated above what was resident before the call.  The fused
kernels' share of their bounding peak uses the operations and compulsory bytes computed here from the shapes and the
H100 SXM data-sheet rates (495 TFLOP/s dense TF32, 3.35 TB/s); the larger bound is named.  Prints one JSON line with
the GPU name and power limit read in the same run; --out writes it to a file.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from deepi2p_b200 import network, point_ops  # noqa: E402
from bench_head import ARGS, PEAK_BW, PEAK_TF32, alternate  # noqa: E402


def accounting(chunk, M=128, K=16, C=64, before=(256, 256), after=(512, 256), final=(256, 512)):
    """Operations and bytes of the kNN module and of final_pointnet + max for one chunk, from the shapes: the torch
    formulation's products (the [max; x] concatenation fed whole to the first after layer), the fused formulation's
    (its max half once per node), the float32 activations torch writes, and the fused kernels' compulsory traffic."""
    cols = chunk * M * K
    widths = [3 + C, *before]
    macs_before = sum(a * b for a, b in zip(widths, widths[1:]))
    aw = [2 * before[-1], *after]
    macs_after_torch = sum(a * b for a, b in zip(aw, aw[1:]))
    macs_after_fused = macs_after_torch - before[-1] * after[0]
    knn = {
        "columns": cols,
        "flop_torch_formulation": 2 * cols * (macs_before + macs_after_torch),
        "flop_fused_formulation": 2 * cols * (macs_before + macs_after_fused) + 2 * chunk * M * before[-1] * after[0],
        # grouped input, each layer's output, the cat, the max of the last before layer: float32, written once each
        "bytes_torch_activations_written": 4 * cols * (3 + C + sum(before) + 2 * before[-1] + sum(after))
        + 4 * chunk * M * (before[-1] + after[-1]),
        # the fused kernel reads the coordinates, the features and the indices and writes [B, C_out, M]
        "bytes_compulsory": 4 * chunk * (3 * M + 3 * M + C * M + K * M + after[-1] * M),
    }
    fw = [3 + before[-1], *final]
    fin = {
        "columns": chunk * M,
        "flop": 2 * chunk * M * sum(a * b for a, b in zip(fw, fw[1:])),
        "bytes_torch_activations_written": 4 * chunk * M * (fw[0] + sum(final)),
        "bytes_compulsory": 4 * chunk * (fw[0] * M + final[-1]),
    }
    for v, flop in ((knn, knn["flop_fused_formulation"]), (fin, fin["flop"])):
        t_flop, t_bw = flop / PEAK_TF32, v["bytes_compulsory"] / PEAK_BW
        v["bound"] = "tensor-core TF32 rate" if t_flop >= t_bw else "HBM bandwidth"
        v["least_ms_at_data_sheet_rates"] = max(t_flop, t_bw) * 1e3
    return {"knnlayer": knn, "final": fin}


def capture(model, b):
    """One forward with hooks: the kNN module's and final_pointnet's inputs."""
    got = {}
    enc = model.pc_encoder
    hooks = [enc.knnlayer.register_forward_pre_hook(lambda m, x: got.__setitem__("knn_in", x)),
             enc.final_pointnet.register_forward_pre_hook(lambda m, x: got.__setitem__("final_in", x[0]))]
    with torch.no_grad():
        model(*(b[k] for k in ARGS))
    for h in hooks:
        h.remove()
    return got


def one_shape(shape, a, dev):
    from bench_e2e import batch, model_for
    b = batch(a.chunk, shape, 1000, dev)
    model = model_for(shape, dev).eval()
    enc = model.pc_encoder
    fused_torch, fused_enc = network.FusedInference(model), network.FusedInference(model, encoder="fused")
    g = capture(model, b)
    query, database, feats, K = g["knn_in"]
    final_in = g["final_in"]
    node_b, node_b_features = final_in[:, :3].contiguous(), final_in[:, 3:].contiguous()
    del g
    keep = {}

    def knn_torch():
        with torch.no_grad():
            keep["knn"] = enc.knnlayer(query, database, feats, K)

    def knn_fused():
        with torch.no_grad():
            keep["knn"] = point_ops.knn_fusion(query, database, feats, K, fused_enc._chain("knn"))

    def final_torch():
        with torch.no_grad():
            keep["final"] = torch.max(enc.final_pointnet(torch.cat((node_b, node_b_features), dim=1)), dim=2,
                                      keepdim=True)[0]

    def final_fused():
        with torch.no_grad():
            keep["final"] = point_ops.pointwise_mlp_max([node_b, node_b_features], fused_enc._chain("final"))

    def fwd(f):
        def run():
            with torch.no_grad():
                keep["fwd"] = f.classify(*(b[k] for k in ARGS))
        return run

    res = {"knnlayer": alternate({"torch": knn_torch, "fused": knn_fused}, a.reps)}
    with torch.no_grad():
        t = enc.knnlayer(query, database, feats, K)
        f = point_ops.knn_fusion(query, database, feats, K, fused_enc._chain("knn"))
    res["knnlayer"]["max_abs_difference_over_max_abs"] = float((t - f).abs().max() / t.abs().max())
    keep.clear()
    res["final"] = alternate({"torch": final_torch, "fused": final_fused}, a.reps)
    keep.clear()
    res["forward"] = alternate({"encoder_torch": fwd(fused_torch), "encoder_fused": fwd(fused_enc)}, a.reps)
    with torch.no_grad():
        p0, p1 = fused_torch.classify(*(b[k] for k in ARGS)), fused_enc.classify(*(b[k] for k in ARGS))
    res["forward"]["fraction_of_points_predicted_differently"] = {
        "coarse": float((p0[0] != p1[0]).float().mean()), "fine": float((p0[1] != p1[1]).float().mean())}
    keep.clear()
    acc = accounting(a.chunk)
    for part in ("knnlayer", "final"):
        res[part]["fused_share_of_bounding_peak"] = acc[part]["least_ms_at_data_sheet_rates"] / res[part]["fused"]["ms"]
        res[part]["bound"] = acc[part]["bound"]
        res[part]["fused_faster"] = res[part]["fused"]["ms"] < res[part]["torch"]["ms"]
    res["accounting"] = acc
    return res


def config5(a, dev):
    from bench_e2e import batch, model_for
    b = batch(a.samples, "oxford", 1000, dev)
    model = model_for("oxford", dev).eval()
    fns = {h: (lambda h=h: network.classify_and_register(model, *(b[k] for k in ARGS), b["K"], chunk=a.chunk, head=h))
           for h in ("fused", "fused_encoder")}
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
        print(json.dumps(accounting(a.chunk)))
        return
    if not torch.cuda.is_available():
        raise SystemExit("bench_knn_fusion.py needs a CUDA device (--accounting runs without one)")
    from bench_prep import _power_limit
    dev = torch.device("cuda:0")
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit": _power_limit(),
           "tf32_flags_of_the_torch_path": [torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32],
           "chunk": a.chunk, "reps": a.reps}
    for shape in ("oxford", "kitti"):
        print(f"bench_knn_fusion: {shape}", file=sys.stderr, flush=True)
        res[shape] = one_shape(shape, a, dev)
        torch.cuda.empty_cache()
    if a.samples > 0:
        print("bench_knn_fusion: config 5", file=sys.stderr, flush=True)
        res["config5_oxford"] = config5(a, dev)
    print(json.dumps({"knn_fusion": res}))
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps({"knn_fusion": res}) + "\n")


if __name__ == "__main__":
    main()
