"""Throughput of the Oxford stereo-centre conversion (grey PNG decode, demosaic + undistort, JPEG encode; DESIGN.md
4.25) on 1280 x 960 RobotCar-shaped frames.

    python scripts/bench_oxford_images.py [--samples 1,64] [--reps 5] [--host-frames 4] [--out BENCH_OXFORD_IMAGES.json]

Inputs, generated here with fixed seeds: synthetic.oxford_mosaic frames written as grey PNGs by the stdlib writer
(zlib level 6) and one synthetic.oxford_distortion_lut.  Prints one JSON line with:
- per S, frames/s from device buffers: decode_grey_png_batch (from host bytes, with its status read-back),
  debayer_undistort_batch and encode_jpeg_batch (to host bytes, with its size read-back), each stage timed with CUDA
  events (median of --reps), and their sum;
- per S, frames/s from files: oxford_images.convert_frames over PNG files to JPEG files in a temporary directory
  (wall clock, page-cache warm);
- the host pipeline build_dataset.py runs (PIL open, the SDK's demosaic and undistort over scipy, cv2.imwrite at
  quality 95) on one host core and on all cores with a process pool, on --host-frames frames (when cv2 imports);
- device time per kernel of the demosaic and the encoder at the largest S (torch.profiler, a run of its own);
- the GPU and its power limit, read in the same run.
The first frame's JPEG is checked against the CPU restatement (oracle_oxford_images) before anything is timed.
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import oracle_oxford_images as oo  # noqa: E402
from deepi2p_b200 import imageprep, oxford_images, synthetic  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_prep import _power_limit  # noqa: E402

HW = (960, 1280)


def events(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def kernel_ms(fn, reps, names):
    """Device time per kernel (torch.profiler, its own run), ms per call."""
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for k in names:
            if k in e.key:
                t = getattr(e, "device_time_total", None)
                t = e.cuda_time_total if t is None else t
                out[k] = out.get(k, 0.0) + t / 1e3 / reps
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


_LUT = None


def _set_lut(lut):
    global _LUT
    _LUT = lut


def host_frame(args):
    """build_dataset.py's conversion of one frame on the host: PIL open, demosaic + undistort, cv2.imwrite."""
    png_path, jpg_path = args
    lut = _LUT
    import cv2
    from PIL import Image
    cfa = np.asarray(Image.open(png_path))
    img = oo.sdk_load_image(cfa, lut)
    cv2.imwrite(jpg_path, cv2.cvtColor(img, cv2.COLOR_BGR2RGB))


def host_pipeline(pngs, tmp, lut, n):
    try:
        import cv2
    except ImportError as e:
        return {"not measured": f"cv2 is not importable ({e})"}
    cv2.setNumThreads(1)
    jobs = [(p, os.path.join(tmp, "host_%d.jpg" % k)) for k, p in enumerate(pngs[:n])]
    _set_lut(lut)
    t0 = time.perf_counter()
    for j in jobs:
        host_frame(j)
    one = (time.perf_counter() - t0) / len(jobs)
    cores = os.cpu_count() or 1
    many = [jobs[k % len(jobs)] for k in range(2 * cores)]
    with ProcessPoolExecutor(cores, initializer=_set_lut, initargs=(lut,)) as ex:
        t0 = time.perf_counter()
        list(ex.map(host_frame, many))
        pool = time.perf_counter() - t0
    return {"opencv": cv2.__version__, "one_core_s_per_frame": one, "one_core_frames_per_s": 1.0 / one,
            "pool_cores": cores, "pool_frames": len(many), "pool_frames_per_s": len(many) / pool}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", default="1,64")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-frames", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_oxford_images.py needs a CUDA device")
    Ss = [int(v) for v in a.samples.split(",") if v]
    S_max = max(Ss)
    lut = synthetic.oxford_distortion_lut(*HW, 7)
    mosaics = [synthetic.oxford_mosaic(HW, 100 + k) for k in range(S_max)]
    blobs = [synthetic.encode_png(m) for m in mosaics]
    table = torch.from_numpy(lut).cuda()
    first = imageprep.encode_jpeg_batch(oxford_images.debayer_undistort_batch(
        imageprep.decode_grey_png_batch(blobs[:1]), table))[0]
    assert first == oo.encode_jpeg(oo.sdk_load_image(mosaics[0], lut)), "the device pipeline differs from the oracle"
    res = {"frame_hw": list(HW), "png": "synthetic.encode_png: grey, zlib level 6, filter 4",
           "mean_png_KB": sum(len(b) for b in blobs) / 1e3 / len(blobs), "mean_jpg_KB": len(first) / 1e3}
    with tempfile.TemporaryDirectory() as tmp:
        pngs = []
        for k, b in enumerate(blobs):
            pngs.append(os.path.join(tmp, "%d.png" % k))
            with open(pngs[-1], "wb") as f:
                f.write(b)
        for S in Ss:
            grey = imageprep.decode_grey_png_batch(blobs[:S])
            rgb = oxford_images.debayer_undistort_batch(grey, table)
            st = {"decode_ms": events(lambda: imageprep.decode_grey_png_batch(blobs[:S]), a.reps),
                  "debayer_undistort_ms": events(lambda: oxford_images.debayer_undistort_batch(grey, table), a.reps),
                  "encode_ms": events(lambda: imageprep.encode_jpeg_batch(rgb), a.reps)}
            st["total_ms"] = sum(st.values())
            st["frames_per_s"] = S / st["total_ms"] * 1e3
            jpgs = [os.path.join(tmp, "out_%d.jpg" % k) for k in range(S)]
            t = wall(lambda: oxford_images.convert_frames(pngs[:S], jpgs, table, batch=S), a.reps)
            st["files"] = {"ms": t * 1e3, "frames_per_s": S / t}
            res[f"s{S}"] = st
        S = S_max
        grey = imageprep.decode_grey_png_batch(blobs[:S])
        rgb = oxford_images.debayer_undistort_batch(grey, table)
        res["kernel_ms"] = {"S": S, **kernel_ms(lambda: oxford_images.debayer_undistort_batch(grey, table), a.reps,
                                                 ("oxford_debayer_kernel",)),
                            **kernel_ms(lambda: imageprep.encode_jpeg_batch(rgb), a.reps,
                                        ("jpege_block", "jpege_dummy", "jpege_length", "DeviceScan", "jpege_emit",
                                         "jpege_count", "jpege_stuff", "Memcpy DtoH", "Memset"))}
        res["host_pipeline"] = host_pipeline(pngs, tmp, lut, a.host_frames)
    res["gpu"] = torch.cuda.get_device_name(0)
    res["power_limit"] = _power_limit()
    line = json.dumps({"oxford_images": res})
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
