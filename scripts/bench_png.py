"""Throughput of the batched PNG decoder (imageprep.decode_png_batch, csrc/png.cu, DESIGN.md 4.23).

    python scripts/bench_png.py [--samples 1,8,64] [--reps 5] [--out BENCH_PNG.json]

Inputs, generated here with a fixed seed by the stdlib writer (synthetic.encode_png, zlib level 6, rows cycling
through the five filters): KITTI-shaped frames (1241 x 376), each a different gradient image with +-12 noise.  PNG is
lossless, so the check is equality with the writer's input.  Prints one JSON line with:
- frames/s and compressed MB/s of decode_png_batch at each S, from host bytes: the chunk walk, the H2D copy, the
  kernels and the status read-back are all inside the timed call (wall clock, median of --reps);
- device time per kernel from a torch.profiler run at the largest S;
- cv2.imdecode on the same frames on one host core and on all host cores with a process pool (when cv2 imports);
- decode_png_batch + assemble_images(kitti_image_args(), "val") at the largest S;
- kitti.kitti_batch whole (train, 64 samples) on a synthetic root with PNG frames and on the same root with .npy
  frames, page-cache warm;
- the GPU and its power limit, read in the same run.
"""
import argparse
import json
import os
import sys
import tempfile
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepi2p_b200 import imageprep, kitti, synthetic  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_prep import _power_limit  # noqa: E402

HW = (376, 1241)
KERNELS = ("png_crc_kernel", "png_chunk_kernel", "png_inflate_kernel", "png_unfilter_kernel")
K_KITTI = np.array([[718.856, 0.0, 607.1928], [0.0, 718.856, 185.2157], [0.0, 0.0, 1.0]])


def frames(S, seed):
    rng = np.random.default_rng(seed)
    h, w = HW
    yy, xx = np.mgrid[0:h, 0:w]
    imgs, blobs = [], []
    for k in range(S):
        img = np.stack([(xx * (3 + k % 5) + yy) % 256, (yy * (2 + k % 3)) % 256, (xx + 7 * yy * k) % 256], -1)
        img = (img + rng.integers(-12, 13, img.shape)).clip(0, 255).astype(np.uint8)
        imgs.append(img)
        blobs.append(synthetic.encode_png(img, filters=np.arange(h) % 5))
    return imgs, blobs


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


def cv2_shape(b):
    import cv2
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR).shape


def host_cv2(blobs, reps):
    try:
        import cv2
    except ImportError as e:
        return {"not measured": f"cv2 is not importable ({e})"}
    cv2.setNumThreads(1)
    t0 = time.perf_counter()
    for _ in range(reps):
        for b in blobs:
            cv2_shape(b)
    one = (time.perf_counter() - t0) / (reps * len(blobs))
    cores = os.cpu_count() or 1
    with ProcessPoolExecutor(cores) as ex:
        list(ex.map(cv2_shape, blobs))
        t0 = time.perf_counter()
        for _ in range(reps):
            list(ex.map(cv2_shape, blobs, chunksize=max(1, len(blobs) // cores)))
        pool = (time.perf_counter() - t0) / reps
    return {"opencv": cv2.__version__, "one_core_ms_per_frame": one * 1e3, "one_core_frames_per_s": 1.0 / one,
            "pool_cores": cores, "pool_frames_per_s": len(blobs) / pool}


def kitti_roots(S, reps):
    out = {}
    with tempfile.TemporaryDirectory() as root:
        for fmt in ("npy", "png"):
            r = os.path.join(root, fmt)
            synthetic.write_kitti_root(r, seqs=(0,), n_frames=120, n_rings=64, n_azimuth=1024, n_images=8, images=fmt)
            ds = kitti.KittiDataset(r, "train", seqs=(0,))
            items = list(range(S))
            t = wall(lambda: kitti.kitti_batch(ds, items, "train", 3, rng=5), reps)
            out[fmt] = {"ms": t * 1e3, "samples_per_s": S / t}
            out[fmt + "_img"] = kitti.kitti_batch(ds, items, "train", 3, rng=5)[6]
    assert torch.equal(out.pop("npy_img"), out.pop("png_img")), "the PNG and npy roots differ"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", default="1,8,64")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_png.py needs a CUDA device")
    Ss = [int(v) for v in a.samples.split(",") if v]
    imgs, blobs = frames(max(Ss), 11)
    dec = imageprep.decode_png_batch(blobs)
    data = dec["data"].cpu().numpy()
    for img, o in zip(imgs, dec["offsets"]):
        assert np.array_equal(data[o:o + img.size].reshape(img.shape), img)
    res = {"frame_hw": list(HW), "encoding": "synthetic.encode_png: zlib level 6, 8 KB IDATs, filters 0-4 by row",
           "mean_KB_per_frame": sum(len(b) for b in blobs) / 1e3 / len(blobs)}
    for S in Ss:
        mb = sum(len(b) for b in blobs[:S]) / 1e6
        t = wall(lambda: imageprep.decode_png_batch(blobs[:S]), a.reps)
        res[f"s{S}"] = {"ms": t * 1e3, "frames_per_s": S / t, "MB_per_s": mb / t}
    S = max(Ss)
    res["kernel_ms"] = kernel_ms(lambda: imageprep.decode_png_batch(blobs[:S]), a.reps)
    res["cv2"] = host_cv2(blobs[:16], max(1, a.reps // 2))

    def both():
        d = imageprep.decode_png_batch(blobs[:S])
        return imageprep.assemble_images(d, np.tile(K_KITTI, (S, 1, 1)), "val", **imageprep.kitti_image_args())
    t = wall(both, a.reps)
    res["with_assemble_images"] = {"S": S, "ms": t * 1e3, "samples_per_s": S / t}
    res["kitti_batch_64"] = kitti_roots(64, a.reps)
    res["gpu"] = torch.cuda.get_device_name(0)
    res["power_limit"] = _power_limit()
    line = json.dumps({"png": res})
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
