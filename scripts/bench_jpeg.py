"""Throughput of the batched JPEG decoder (imageprep.decode_jpeg_batch, csrc/jpeg.cu, DESIGN.md 4.19).

    python scripts/bench_jpeg.py [--samples 64] [--reps 10] [--out BENCH_JPEG.json]

Inputs, generated here with a fixed seed: --samples Oxford-shaped frames (1280 x 960) and as many nuScenes-shaped
ones (1600 x 900), each a different synthetic textured image (gradients, edges, Gaussian noise) encoded as the
Oxford build script writes them: cv2.imencode at its defaults (quality 95, 4:2:0, no restart markers).  Prints one
JSON line with, per shape:
- images/s and compressed MB/s of decode_jpeg_batch at S = 1 and S = --samples, from host bytes: header parsing,
  the H2D copy, the kernels and the status read-back are all inside the timed call (wall clock, median of --reps);
- device time per kernel (unstuff, Huffman, IDCT, upsample + colour) from a torch.profiler run at S = --samples,
  and the synchronisation rounds the no-restart Huffman path needed (max and mean over the images);
- for Oxford, decode_jpeg_batch + assemble_images(oxford_image_args(), "val") to [S, 3, 384, 640];
- Pillow's decode (np.asarray(Image.open(...).convert("RGB"))) on one host core and on all host cores with a process
  pool, and torchvision.io.decode_jpeg(device="cuda") (nvJPEG) with the number of pixels where it differs from
  Pillow, for information only;
- the GPU and its power limit, read in the same run.
"""
import argparse
import io
import json
import os
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepi2p_b200 import imageprep  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_prep import _power_limit  # noqa: E402

SHAPES = {"oxford": (960, 1280), "nuscenes": (900, 1600)}
KERNELS = ("jpeg_unstuff_kernel", "jpeg_huffman_kernel", "jpeg_idct_kernel", "jpeg_color_kernel")
K_OXFORD = np.array([[983.044, 0.0, 643.647], [0.0, 983.044, 493.379], [0.0, 0.0, 1.0]])


def frames(shape, S, seed):
    import cv2
    rng = np.random.default_rng(seed)
    h, w = shape
    y, x = np.mgrid[0:h, 0:w]
    out = []
    for s in range(S):
        ph = rng.uniform(0, 6.3)
        base = np.stack([255 * x / w, 255 * y / h, 127 + 120 * np.sin(x / (9.0 + s % 7) + y / 13.0 + ph)], -1)
        base[(x // 97 + y // 61 + s) % 5 == 0] = 250
        img = np.clip(base + rng.normal(0, 12, (h, w, 3)), 0, 255).astype(np.uint8)
        ok, enc = cv2.imencode(".jpg", img)
        assert ok
        out.append(enc.tobytes())
    return out


def wall(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def kernel_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for k in KERNELS:
            if k in e.key:
                t = getattr(e, "device_time_total", None)
                t = e.cuda_time_total if t is None else t
                out[k] = out.get(k, 0.0) + t / 1e3 / reps
    return out


def pillow_one(b):
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(b)).convert("RGB"))


def pillow_shape(b):
    return pillow_one(b).shape


def host_pillow(blobs, reps):
    t0 = time.perf_counter()
    for _ in range(reps):
        for b in blobs:
            pillow_one(b)
    one = (time.perf_counter() - t0) / (reps * len(blobs))
    cores = os.cpu_count() or 1
    with ProcessPoolExecutor(cores) as ex:
        list(ex.map(pillow_shape, blobs))                    # start the workers
        t0 = time.perf_counter()
        for _ in range(reps):
            list(ex.map(pillow_shape, blobs, chunksize=max(1, len(blobs) // cores)))
        pool = (time.perf_counter() - t0) / reps
    return {"one_core_ms_per_image": one * 1e3, "one_core_images_per_s": 1.0 / one, "pool_cores": cores,
            "pool_images_per_s": len(blobs) / pool}


def nvjpeg(blobs, reps):
    try:
        import torchvision
        from torchvision.io import decode_jpeg
    except ImportError as e:
        return {"skipped": f"torchvision not importable ({e})"}
    data = [torch.frombuffer(bytearray(b), dtype=torch.uint8) for b in blobs]
    try:
        t = wall(lambda: decode_jpeg(data, device="cuda"), reps)
        out = decode_jpeg(data, device="cuda")
    except Exception as e:  # noqa: BLE001 - informational only
        return {"skipped": f"torchvision.io.decode_jpeg(device='cuda') failed: {e}"}
    diff = 0
    for img, b in zip(out, blobs):
        diff += int((img.permute(1, 2, 0).cpu().numpy() != pillow_one(b)).any(-1).sum())
    return {"torchvision": torchvision.__version__, "images_per_s": len(blobs) / t, "batch_ms": t * 1e3,
            "pixels_differing_from_pillow": diff, "pixels": int(sum(pillow_one(b).shape[0] * pillow_one(b).shape[1]
                                                                    for b in blobs))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=64)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_jpeg.py needs a CUDA device")
    S = a.samples
    res = {"samples": S, "encoding": "cv2.imencode defaults: quality 95, 4:2:0, no restart markers"}
    for i, (name, shape) in enumerate(SHAPES.items()):
        blobs = frames(shape, S, 100 + i)
        mb = sum(len(b) for b in blobs) / 1e6
        for b in blobs[:2]:
            assert np.array_equal(imageprep.decode_jpeg_batch([b])["data"].cpu().numpy().reshape(shape + (3,)),
                                  pillow_one(b))
        t1 = wall(lambda: imageprep.decode_jpeg_batch(blobs[:1]), a.reps)
        tS = wall(lambda: imageprep.decode_jpeg_batch(blobs), a.reps)
        imageprep.decode_jpeg_batch(blobs)
        rounds = imageprep.decode_jpeg_batch.last_rounds
        r = {"frame_hw": list(shape), "compressed_MB": mb, "mean_KB_per_frame": mb * 1e3 / S,
             "s1": {"ms": t1 * 1e3, "images_per_s": 1.0 / t1, "MB_per_s": len(blobs[0]) / 1e6 / t1},
             f"s{S}": {"ms": tS * 1e3, "images_per_s": S / tS, "MB_per_s": mb / tS},
             "kernel_ms": kernel_ms(lambda: imageprep.decode_jpeg_batch(blobs), a.reps),
             "sync_rounds": {"max": int(rounds.max()), "mean": float(rounds.mean())},
             "pillow": host_pillow(blobs[:16], max(1, a.reps // 5)),
             "nvjpeg": nvjpeg(blobs, a.reps)}
        if name == "oxford":
            def both():
                dec = imageprep.decode_jpeg_batch(blobs)
                return imageprep.assemble_images(dec, K_OXFORD, "val", **imageprep.oxford_image_args())
            t = wall(both, a.reps)
            assert tuple(both()["img"].shape) == (S, 3, 384, 640)
            r["with_assemble_images"] = {"out": [S, 3, 384, 640], "ms": t * 1e3, "samples_per_s": S / t}
        res[name] = r
    res["gpu"] = torch.cuda.get_device_name(0)
    res["power_limit"] = _power_limit()
    line = json.dumps({"jpeg": res})
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
