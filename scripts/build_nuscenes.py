"""Build a nuScenes dataroot's dataset_info.list from the raw tables (data/nuscenes/make_datasets.py, one GPU):

    python scripts/build_nuscenes.py --dataroot R --version v1.0-trainval [--frame-skip 2] [--max-translation 10]

R holds <version>/{scene, sample, sample_data, sensor, calibrated_sensor, ego_pose}.json; R/dataset_info.list is
(over)written.  Prints the entry, scene and deferral counts and the time of each stage.
"""
import argparse
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def positive(v):
    n = int(v)
    if n < 1:
        raise argparse.ArgumentTypeError(f"must be a positive integer (got {v})")
    return n


def radius(v):
    x = float(v)
    if not math.isfinite(x) or x < 0:
        raise argparse.ArgumentTypeError(f"must be a finite number >= 0 (got {v})")
    return x


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--dataroot", required=True)
    ap.add_argument("--version", required=True, help="the table directory, e.g. v1.0-trainval")
    ap.add_argument("--frame-skip", type=positive, default=2, help="keep every n-th LIDAR_TOP sweep (the script's 2)")
    ap.add_argument("--max-translation", type=radius, default=10.0, help="camera radius in metres (the script's 10)")
    a = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        sys.exit("build_nuscenes.py needs a CUDA device (sm_90a); there is no CPU path")
    from deepi2p_b200 import nuscenes_build
    st = {}
    nuscenes_build.make_dataset_info(a.dataroot, a.version, a.frame_skip, a.max_translation, stats=st)
    print(f"{st['entries']} entries from {st['scenes']} of {st['scenes_total']} scenes "
          f"({st['sample_data']} sample_data records); {st['walks']} camera walks, {st['tokens']} tokens from the "
          f"device, {st['deferred']} walks deferred to the host")
    for k in ("json", "index", "plan", "walk", "assemble", "total"):
        print(f"  {k + ':':<10}{st[k + '_seconds']:9.3f} s")
    print(f"  (device kernels {st['device_seconds'] * 1e3:.3f} ms)")
    print("wrote", os.path.join(a.dataroot, "dataset_info.list"))


if __name__ == "__main__":
    main()
