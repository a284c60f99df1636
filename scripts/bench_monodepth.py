"""Benchmark of the monodepth depth clouds (deepi2p_b200.monodepth) at the Oxford shape: S frames of 384 x 640 to the
mono+stereo_640x192 feed (640 x 192, only the vertical pass of the resize), seeded weights of the shipped shape.
Writes BENCH_MONODEPTH.json (or --out):

  - the resize kernel, the network's forward, the cloud kernel (unscaled fp64 cloud; and scale + float32 target) and
    the whole depth_clouds call, each with CUDA events over --reps calls after --warmup, as ms per call and frames/s;
  - achieved bytes/s of the two kernels (bytes the algorithm must move, computed from the shapes) against 3.35 TB/s;
  - ICP from images (icp.register_images, 60 inits per frame) in frames/s;
  - the reference-shaped loop on the same machine: Pillow's Lanczos on one host core, a batch-1 forward,
    F.interpolate + reciprocal and the numpy back-projection, per frame;
  - a torch.profiler split of the forward into convolutions and the rest, taken after the timed runs;
  - the card name and power limit, read in the same run.

    python scripts/bench_monodepth.py [--frames 64] [--reps 20] [--warmup 3] [--out PATH]
"""
import os

os.environ.setdefault("OMP_NUM_THREADS", "1")          # the host loop runs on one core
os.environ.setdefault("OPENBLAS_NUM_THREADS", "1")

import argparse  # noqa: E402
import json  # noqa: E402
import subprocess  # noqa: E402
import sys  # noqa: E402
import time  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_BYTES = 3.35e12                     # H100 SXM HBM3, NVIDIA data sheet


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (x.strip() for x in q.split(","))
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # noqa: BLE001 - the card is still named by torch
        return dict(name=torch.cuda.get_device_name(0), power_limit=f"unknown ({e})")


def events(fn, reps, warmup):
    """Median ms per call of fn over reps calls, each between two CUDA events, after warmup calls."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return float(np.median(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-frames", type=int, default=4, help="frames of the reference-shaped loop")
    ap.add_argument("--out", default=os.path.join(ROOT, "BENCH_MONODEPTH.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_monodepth.py needs a CUDA device")
    import oracle_monodepth as om
    from PIL import Image
    from deepi2p_b200 import icp, imageprep, monodepth, synthetic

    S, H, W, fh, fw = a.frames, 384, 640, 192, 640
    res = dict(card=card(), frames=S, image=[H, W], feed=[fh, fw], tf32=bool(torch.backends.cudnn.allow_tf32))
    enc, dec = om.seeded_checkpoint(0, fh, fw)
    model = monodepth.DepthNet(fh, fw)
    model.load_state_dict({k: v for k, v in {**enc, **dec}.items() if torch.is_tensor(v)})
    model = model.cuda().eval()
    frames = [synthetic.make_icp_frame(s, "oxford") for s in range(S)]
    rng = np.random.default_rng(0)
    host_imgs = [rng.integers(0, 256, (H, W, 3), dtype=np.uint8) for _ in range(S)]
    images = imageprep.pack_images(host_imgs)
    K = np.stack([f["K"] for f in frames]).astype(np.float32)
    K_inv = monodepth.k_inverse(K)
    K64 = K.astype(np.float64).reshape(S, 9)
    P = np.stack([f["P_gt"] for f in frames])
    src, n = icp.pack_clouds([f["src"] for f in frames])

    x = monodepth.resize_normalise(images, fh, fw)
    with torch.no_grad():
        disp = model(x).contiguous()

    class Fixed(torch.nn.Module):
        feed_height, feed_width = fh, fw

        def forward(self, _):
            return disp
    fixed = Fixed().eval()
    # the cloud kernel alone: depth_clouds with the network's output given (its resize is subtracted below)
    t_resize = events(lambda: monodepth.resize_normalise(images, fh, fw), a.reps, a.warmup)
    with torch.no_grad():
        t_forward = events(lambda: model(x), a.reps, a.warmup)
    t_cloud64 = events(lambda: monodepth.depth_clouds(fixed, images, K_inv), a.reps, a.warmup) - t_resize
    t_scaled = events(lambda: monodepth.depth_clouds(fixed, images, K_inv, src=src, n_pts=n, P_gt=P, K=K64,
                                                     cloud64=False), a.reps, a.warmup) - t_resize
    t_all = events(lambda: monodepth.depth_clouds(model, images, K_inv), a.reps, a.warmup)
    t_all_scaled = events(lambda: monodepth.depth_clouds(model, images, K_inv, src=src, n_pts=n, P_gt=P, K=K64,
                                                         cloud64=False), a.reps, a.warmup)
    P_px, p_px = H * W, fh * fw
    b_resize = S * (H * W * 3 + 3 * p_px * 4)                      # uint8 in, float32 NCHW out (one pass)
    b_cloud64 = S * (fh * fw * 4 + 3 * P_px * 8)                   # disparity in, fp64 cloud out
    b_scaled = S * (2 * fh * fw * 4 + 3 * P_px * 4 + 3 * src.shape[2] * 4)   # two disparity reads, f32 out, LiDAR
    res["ms"] = dict(resize=t_resize, forward=t_forward, cloud_f64=t_cloud64, cloud_scale_f32=t_scaled,
                     depth_clouds_f64=t_all, depth_clouds_scaled_f32=t_all_scaled)
    res["frames_per_s"] = {k: S / (v / 1e3) for k, v in res["ms"].items()}
    res["bytes_per_s"] = dict(resize=b_resize / (t_resize / 1e3), cloud_f64=b_cloud64 / (t_cloud64 / 1e3),
                              cloud_scale_f32=b_scaled / (t_scaled / 1e3))
    res["share_of_3_35_TBps"] = {k: v / PEAK_BYTES for k, v in res["bytes_per_s"].items()}
    res["cloud_times_note"] = "cloud_* = depth_clouds with a fixed disparity minus the resize time (host glue included)"

    init = torch.from_numpy(icp.random_inits(S, 60, 0)).cuda()
    t_icp = events(lambda: icp.register_images(src, n, images, K, P, init, model), 2, 1)
    res["icp_from_images"] = dict(ms=t_icp, frames_per_s=S / (t_icp / 1e3), inits=60)

    # the reference-shaped loop: one frame at a time, PIL on the host, batch-1 forward, numpy back-projection
    def host_frame(s):
        img = Image.fromarray(host_imgs[s]).convert("RGB").resize((fw, fh), Image.LANCZOS)
        t = torch.from_numpy(np.asarray(img)).permute(2, 0, 1)[None].float().div(255).cuda()
        with torch.no_grad():
            dsp = model((t - 0.45) / 0.225)
            dep = torch.reciprocal(F.interpolate(dsp, (H, W), mode="bilinear", align_corners=False))
        return om.convert_depth_to_pointcloud(dep[0, 0].unsqueeze(2).cpu().numpy(), K[s])
    host_frame(0)
    t0 = time.perf_counter()
    for s in range(a.host_frames):
        host_frame(s)
    t_host = (time.perf_counter() - t0) / a.host_frames
    res["reference_loop"] = dict(ms_per_frame=t_host * 1e3, frames_per_s=1.0 / t_host, frames=a.host_frames)

    # the forward's split, in a profiled pass of its own after the timed runs
    from torch.profiler import ProfilerActivity, profile
    with torch.no_grad(), profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            model(x)
        torch.cuda.synchronize()
    split = dict(convolution=0.0, cudnn_layout_and_batchnorm=0.0, torch_glue=0.0)
    kernels = []
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if e.key.startswith("aten::") or e.key.startswith("cuda") or t <= 0:
            continue
        name = e.key.lower()
        kernels.append((t / 3e3, e.key[:90]))
        if any(w in name for w in ("fprop", "conv", "gemm", "xmma", "cutlass", "implicit")):
            split["convolution"] += t / 3e3
        elif "cudnn" in name:
            split["cudnn_layout_and_batchnorm"] += t / 3e3
        else:                            # reflection pad, ELU, ReLU, add, max-pool, nearest upsample, cat, sigmoid
            split["torch_glue"] += t / 3e3
    top = [[k, round(v, 4)] for v, k in sorted(kernels, reverse=True)[:12]]
    res["forward_profile_ms"] = dict(split, top_kernels=top)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
