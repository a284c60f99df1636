"""The classifier's ResNet-34 image encoder, torch backbone against the fused resnet34_features (DESIGN.md 4.30).

    python scripts/bench_image_encoder.py [--chunk 64] [--reps 7] [--samples 1024] [--out BENCH_IMAGE_ENCODER.json]
    python scripts/bench_image_encoder.py --profile [--out ...]   # device-time split of one forward per head
    python scripts/bench_image_encoder.py --accounting            # operations and bytes from the shapes; no GPU

At the KITTI, Oxford and nuScenes image shapes (seeded untrained weights from bench_e2e's builders), one chunk of
`--chunk` assembled images:
- backbone: model.img_encoder.backbone(img), the mean over H and W and the two reshape/contiguous copies, as
  FusedInference's torch path runs them (cuDNN, with torch's TF32 flags as they are, recorded below), against one
  resnet.resnet34_features call;
- forward (Oxford): FusedInference.classify with head "fused_all" against "fused_image";
and config 5 (network.classify_and_register over `--samples` Oxford samples, 60 inits) with both heads.
The candidates alternate within one run (bench_head.alternate): CUDA events after a warm-up, the median of --reps with
the minimum and maximum; peak is max_memory_allocated above what was resident before the call.  The least time is the
larger of the backbone's operations at the H100 SXM data-sheet rate (495 TFLOP/s dense TF32) and one float32 write
plus one read of every convolution and pool output and one read of the image at 3.35 TB/s; the share of that bound is
the least time over the measured one.  Prints one JSON line with the GPU name and power limit read in the same run;
--out writes it to a file.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from deepi2p_b200 import network, resnet  # noqa: E402
from bench_head import ARGS, PEAK_BW, PEAK_TF32, alternate  # noqa: E402

SHAPES = ("oxford", "kitti", "nuscenes")


def accounting(shape, chunk):
    """FLOP of every convolution and the bytes of one write and one read of every convolution / pool output (plus
    the image read once) for one chunk, from the shapes."""
    H, W = network.SHAPES[shape]["img_H"], network.SHAPES[shape]["img_W"]
    down = lambda n, k, p, s: (n + 2 * p - k) // s + 1
    flop = 0
    out_floats = 0
    h, w = down(H, 7, 3, 2), down(W, 7, 3, 2)
    flop += 2 * chunk * h * w * 64 * 147
    out_floats += chunk * h * w * 64
    h, w = down(h, 3, 1, 2), down(w, 3, 1, 2)
    out_floats += chunk * h * w * 64
    c_in = 64
    for C, n, first in resnet.STAGES:
        for j in range(n):
            s = first if j == 0 else 1
            h, w = down(h, 3, 1, s), down(w, 3, 1, s)
            flop += 2 * chunk * h * w * C * 9 * (c_in + C)
            if s != 1:
                flop += 2 * chunk * h * w * C * c_in
            out_floats += 2 * chunk * h * w * C
            c_in = C
    nbytes = 4 * (2 * out_floats + chunk * 3 * H * W)
    t_flop, t_bytes = flop / PEAK_TF32, nbytes / PEAK_BW
    return {"image": [H, W], "flop": flop, "bytes_one_write_and_read_of_every_output": nbytes,
            "least_ms": max(t_flop, t_bytes) * 1e3, "bound": "tf32_compute" if t_flop >= t_bytes else "hbm_bytes",
            "ms_at_tf32_data_sheet_rate": t_flop * 1e3, "ms_at_hbm_data_sheet_rate": t_bytes * 1e3}


def torch_backbone(model, img):
    s16, s32 = model.img_encoder.backbone(img)
    B = img.shape[0]
    g = s32.mean(dim=(2, 3))
    return s16.reshape(B, s16.shape[1], -1).contiguous(), s32.reshape(B, g.shape[1], -1).contiguous(), g


def one_shape(shape, a, dev):
    from bench_e2e import model_for
    H, W = network.SHAPES[shape]["img_H"], network.SHAPES[shape]["img_W"]
    model = model_for(shape, dev).eval()
    img = torch.rand(a.chunk, 3, H, W, device=dev, generator=torch.Generator(device=dev).manual_seed(1000))
    fused = network.FusedInference(model, encoder="fused", decoder="fused", image="fused")
    packed = fused._chain("resnet")
    keep = {}

    def run_torch():
        with torch.no_grad():
            keep["y"] = torch_backbone(model, img)

    def run_fused():
        with torch.no_grad():
            keep["y"] = resnet.resnet34_features(img, packed)

    res = alternate({"torch": run_torch, "fused": run_fused}, a.reps)
    keep.clear()
    with torch.no_grad():
        t, f = torch_backbone(model, img), resnet.resnet34_features(img, packed)
    res["max_abs_difference_over_max_abs"] = {
        n: float((x - y).abs().max() / x.abs().max()) for n, x, y in zip(("s16", "s32", "img_global"), t, f)}
    del t, f
    acc = accounting(shape, a.chunk)
    res["accounting"] = acc
    res["fused_faster"] = res["fused"]["ms"] < res["torch"]["ms"]
    for side in ("torch", "fused"):
        res[side]["share_of_bound"] = acc["least_ms"] / res[side]["ms"]
    return res


def forward(a, dev):
    from bench_e2e import batch, model_for
    b = batch(a.chunk, "oxford", 1000, dev)
    model = model_for("oxford", dev).eval()
    heads = {"fused_all": network.FusedInference(model, encoder="fused", decoder="fused"),
             "fused_image": network.FusedInference(model, encoder="fused", decoder="fused", image="fused")}
    keep = {}

    def fwd(f):
        def run():
            with torch.no_grad():
                keep["fwd"] = f.classify(*(b[k] for k in ARGS))
        return run

    res = alternate({h: fwd(f) for h, f in heads.items()}, a.reps)
    keep.clear()
    res["fused_image_faster"] = res["fused_image"]["ms"] < res["fused_all"]["ms"]
    with torch.no_grad():
        p0, p1 = (f.classify(*(b[k] for k in ARGS)) for f in heads.values())
    res["fraction_of_points_predicted_differently"] = {
        "coarse": float((p0[0] != p1[0]).float().mean()), "fine": float((p0[1] != p1[1]).float().mean())}
    return res


def config5(a, dev):
    from bench_e2e import batch, model_for
    b = batch(a.samples, "oxford", 1000, dev)
    model = model_for("oxford", dev).eval()
    out = {}
    fns = {}
    for h in ("fused_all", "fused_image"):
        def run(h=h):
            out[h] = network.classify_and_register(model, *(b[k] for k in ARGS), b["K"], chunk=a.chunk, head=h)
        fns[h] = run
    res = alternate(fns, max(3, a.reps // 2))
    res["fraction_of_points_predicted_differently"] = {
        k: float((out["fused_all"][k] != out["fused_image"][k]).float().mean()) for k in ("coarse_pred", "fine_pred")}
    res.update(samples=a.samples, chunk=a.chunk, n_inits=60,
               note="seeded untrained weights: the registration solves meaningless predictions, which can differ "
                    "between the heads, so its time can differ too")
    return res


def profile(a, dev):
    """Device time of one Oxford forward per head under torch.profiler, split into the image encoder (the kernels
    launched inside the torch backbone's forward, or the resnet kernels) and the rest."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile as tprofile, record_function
    from bench_e2e import batch, model_for
    b = batch(a.chunk, "oxford", 1000, dev)
    model = model_for("oxford", dev).eval()
    bb = model.img_encoder.backbone
    heads = {"fused_all": network.FusedInference(model, encoder="fused", decoder="fused"),
             "fused_image": network.FusedInference(model, encoder="fused", decoder="fused", image="fused")}

    def enter(m, x):
        m._range = record_function("image_backbone")
        m._range.__enter__()

    def leave(m, x, y):
        m._range.__exit__(None, None, None)
        del m._range

    def kernel_us(e):
        return sum(k.duration for k in e.kernels) + sum(kernel_us(c) for c in e.cpu_children)

    res = {}
    for head, f in heads.items():
        with torch.no_grad():
            for _ in range(2):
                f.classify(*(b[k] for k in ARGS))
            torch.cuda.synchronize()
            hooks = [bb.register_forward_pre_hook(enter), bb.register_forward_hook(leave)]
            try:
                with tprofile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                    f.classify(*(b[k] for k in ARGS))
                    torch.cuda.synchronize()
            finally:
                for h in hooks:
                    h.remove()
        total = fused = backbone = 0.0
        top = {}
        for e in prof.events():
            if e.device_type == DeviceType.CUDA and e.name != "image_backbone":
                t = e.time_range.elapsed_us()
                total += t
                top[e.name[:100]] = top.get(e.name[:100], 0.0) + t
                if "rn_conv_kernel" in e.name or "rn_maxpool_kernel" in e.name or "rn_mean_kernel" in e.name:
                    fused += t
            elif e.device_type == DeviceType.CPU and e.name == "image_backbone":
                backbone += kernel_us(e)
        image = fused + backbone
        res[head] = {"device_us": total, "image_encoder_us": image, "of_which_resnet_kernels_us": fused,
                     "of_which_torch_backbone_kernels_us": backbone,
                     "image_encoder_share": image / total if total else None,
                     "top_kernels": [{"us": t, "name": n} for n, t in sorted(top.items(), key=lambda kv: -kv[1])[:15]]}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunk", type=int, default=network.DEFAULT_CHUNK)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--samples", type=int, default=1024)
    ap.add_argument("--accounting", action="store_true")
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if a.accounting:
        print(json.dumps({s: accounting(s, a.chunk) for s in SHAPES}))
        return
    if not torch.cuda.is_available():
        raise SystemExit("bench_image_encoder.py needs a CUDA device (--accounting runs without one)")
    from bench_prep import _power_limit
    dev = torch.device("cuda:0")
    res = {"gpu": torch.cuda.get_device_name(0), "power_limit": _power_limit(),
           "tf32_flags_of_the_torch_path": [torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32],
           "chunk": a.chunk, "reps": a.reps}
    if a.profile:
        res["profile_oxford"] = profile(a, dev)
        key = "image_encoder_profile"
    else:
        key = "image_encoder"
        for shape in SHAPES:
            print(f"bench_image_encoder: {shape}", file=sys.stderr, flush=True)
            res[shape] = one_shape(shape, a, dev)
            torch.cuda.empty_cache()
        print("bench_image_encoder: forward", file=sys.stderr, flush=True)
        res["forward_oxford"] = forward(a, dev)
        torch.cuda.empty_cache()
        if a.samples > 0:
            print("bench_image_encoder: config 5", file=sys.stderr, flush=True)
            res["config5_oxford"] = config5(a, dev)
    print(json.dumps({key: res}))
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps({key: res}) + "\n")


if __name__ == "__main__":
    main()
