"""Throughput of the image side of classifier batches (deepi2p_b200.imageprep, DESIGN.md 4.13).

    python scripts/bench_images.py [--samples 64] [--reps 20] [--cpu-samples 8] [--out FILE.json]

Frames: synthetic KITTI-shaped uint8 images (370 x 1226, 375 x 1242, 376 x 1241 in turn), packed once and resident
on the device, as a loader that keeps decoded frames on the GPU would hold them.  KITTI train arguments (50-row cut,
scale 0.5, random 160 x 512 crop, every sample jittered, half flipped).  Prints one JSON line with:
- samples/s of assemble_images at S = --samples (host draws, parameter upload and both kernels; CUDA events around
  each call, median over --reps) and the latency of one sample;
- per-kernel device times from a separate torch.profiler run, and the algorithmic bytes (the source window the
  crop needs, read once, plus the output written) over the assemble kernel's time against the H100 SXM data-sheet
  3.35 TB/s;
- assemble_batch (the point side, bench_assemble.py's KITTI batch) and assemble_images together at S = --samples;
- the host path the loaders run (cv2.resize, crop, torchvision ColorJitter on PIL, flip, float32 CHW) per sample on
  one host core, or a stated skip when cv2 / Pillow / torchvision are missing;
- the GPU and its power limit, read in the same run.
"""
import os

os.environ.setdefault("OMP_NUM_THREADS", "1")      # the host baseline is one core

import argparse  # noqa: E402
import json  # noqa: E402
import sys  # noqa: E402
import time  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import oracle_image  # noqa: E402
from deepi2p_b200 import assemble, imageprep, synthetic  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_prep import _power_limit, _time  # noqa: E402

HBM_BPS = 3.35e12
SHAPES = [(370, 1226), (375, 1242), (376, 1241)]
K = np.array([[718.856, 0.0, 607.1928], [0.0, 718.856, 185.2157], [0.0, 0.0, 1.0]])


def frames_of(S, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    for s in range(S):
        h, w = SHAPES[s % 3]
        y, x = np.mgrid[0:h, 0:w]
        base = np.stack([255 * x / w, 255 * y / h, 127 + 120 * np.sin(x / 17.0 + y / 11.0)], -1)
        out.append(np.clip(base + rng.normal(0, 30, (h, w, 3)), 0, 255).astype(np.uint8))
    return out


def window_bytes(p, w):
    """Source bytes the crop window needs: the span of source rows and columns its resize taps touch."""
    total = 0
    for s in range(len(p["dh"])):
        sx, _, _ = oracle_image.axis_coeffs(int(w[s]), int(p["dw"][s]))
        sy, _, _ = oracle_image.axis_coeffs(int(p["rows"][s]), int(p["dh"][s]))
        x0, y0 = int(p["dx"][s]), int(p["dy"][s])
        cols = min(int(sx[x0 + p["img_W"] - 1]) + 1, int(w[s]) - 1) - int(sx[x0]) + 1
        rows = min(int(sy[y0 + p["img_H"] - 1]) + 1, int(p["rows"][s]) - 1) - int(sy[y0]) + 1
        total += 3 * cols * rows
    return total


def kernel_ms(fn, reps):
    """Mean device time per call of each kernel, from torch.profiler over `reps` calls."""
    fn()
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if "image_" in e.key:
            name = "image_luma_partials_kernel" if "partials" in e.key else "image_assemble_kernel"
            t = getattr(e, "device_time_total", None)
            if t is None:
                t = e.cuda_time_total
            out[name] = out.get(name, 0.0) + t / 1e3 / reps
    return out


def host_path(frames, p, flip, n):
    """The loaders' per-sample host steps, timed on one core."""
    import cv2
    from deepi2p_b200.imageprep import augment_img
    t0 = time.perf_counter()
    for s in range(n):
        img = frames[s][int(p["row0"][s]):]
        img = cv2.resize(img, (int(p["dw"][s]), int(p["dh"][s])), interpolation=cv2.INTER_LINEAR)
        y, x = int(p["dy"][s]), int(p["dx"][s])
        img = img[y:y + p["img_H"], x:x + p["img_W"]]
        img = augment_img(img, s)
        if flip[s]:
            img = np.flip(img, 1)
        torch.from_numpy(img.astype(np.float32)).permute(2, 0, 1).contiguous()
    return (time.perf_counter() - t0) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=64)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--cpu-samples", type=int, default=8)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_images.py needs a CUDA device")
    S = a.samples
    frames = frames_of(S)
    packed = imageprep.pack_images(frames)
    one = imageprep.pack_images(frames[:1])
    args = imageprep.kitti_image_args()
    flip = np.arange(S) % 2 == 1

    def run(pk, fl):
        return imageprep.assemble_images(pk, K, "train", rng=0, flip=fl, **args)

    t_big = _time(lambda: run(packed, flip), a.reps)
    t_one = _time(lambda: run(one, flip[:1]), a.reps)
    params = run(packed, flip)["params"]
    kern = kernel_ms(lambda: imageprep.assemble_images(packed, K, params=params, flip=flip), a.reps)
    H, W = params["img_H"], params["img_W"]
    read_b = window_bytes(params, packed["shapes"][:, 1])
    write_b = S * 3 * H * W * 4
    t_k = kern.get("image_assemble_kernel", float("nan")) * 1e-3
    res = {"samples": S, "img_H": H, "img_W": W, "frame_shapes": SHAPES, "mode": "train",
           "samples_per_s": S / t_big, "batch_ms": t_big * 1e3, "latency_s1_ms": t_one * 1e3,
           "kernel_ms": kern, "algorithmic_bytes": {"window_read": read_b, "output_written": write_b},
           "assemble_kernel_share_of_3_35_TBps": (read_b + write_b) / HBM_BPS / t_k}

    base = [synthetic.make_loader_sample(s, "kitti") for s in range(8)]
    fr = assemble.pack_frames([(base[s % 8]["frames"], base[s % 8]["frame_T"]) for s in range(S)])
    pargs = assemble.kitti_args(base[0]["Pc"], base[0]["Pji"])

    def both():
        pts = assemble.assemble_batch(fr, "train", 7, rng=0, **pargs)
        return imageprep.assemble_images(packed, K, "train", rng=0, flip=pts["flip"], **args)

    t_pts = _time(lambda: assemble.assemble_batch(fr, "train", 7, rng=0, **pargs), max(3, a.reps // 4))
    t_both = _time(both, max(3, a.reps // 4))
    res["with_assemble_batch"] = {"assemble_batch_ms": t_pts * 1e3, "both_ms": t_both * 1e3,
                                  "samples_per_s": S / t_both}
    try:
        import cv2  # noqa: F401
        import torchvision  # noqa: F401
        from PIL import Image  # noqa: F401
        n = min(a.cpu_samples, S)
        res["host_path"] = {"samples": n, "cores": 1, "s_per_sample": host_path(frames, params, flip, n)}
    except ImportError as e:
        res["host_path"] = {"skipped": f"cv2 / Pillow / torchvision not importable here ({e})"}
    res["gpu"] = torch.cuda.get_device_name(0)
    res["power_limit"] = _power_limit()
    line = json.dumps({"images": res})
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
