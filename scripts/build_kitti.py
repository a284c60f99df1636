"""Build a KITTI root's accumulated-frame records from its prepared scans (data/kitti/frame_accumulation.py, one GPU):

    python scripts/build_kitti.py ROOT [--seqs 0-10] [--stride 4] [--radius 50] [--voxel 0.4] [--batch 64]

ROOT holds calib/<seq>/calib.txt, poses/<seq>/<frame>.npz and data_odometry_velodyne_NWU/sequences/<seq>/
voxel0.1-SNr0.6/<frame>.npy (scripts/prepare_scans.py writes them).  Each sequence's records go to
data_odometry_velodyne_NWU/sequences/<seq>/stride<S>-acc<R>-voxel<V>/<frame>.npy; a sequence whose folder exists is
skipped.  Prints one line per batch of frames.
"""
import argparse
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def seq_list(v):
    out = []
    for part in v.split(","):
        lo, _, hi = part.partition("-")
        try:
            out += list(range(int(lo), int(hi or lo) + 1))
        except ValueError:
            raise argparse.ArgumentTypeError(f"sequences are a list of numbers and ranges, e.g. 0-10 or 0,2,5-7 "
                                             f"(got {v!r})") from None
    if not out or min(out) < 0:
        raise argparse.ArgumentTypeError(f"no valid sequence in {v!r}")
    return out


def positive_int(v):
    n = int(v)
    if n < 1:
        raise argparse.ArgumentTypeError(f"must be a positive integer (got {v})")
    return n


def positive(v):
    x = float(v)
    if not (math.isfinite(x) and x > 0):
        raise argparse.ArgumentTypeError(f"must be a positive number (got {v})")
    return x


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("root")
    ap.add_argument("--seqs", type=seq_list, default=list(range(11)), help="sequences, e.g. 0-10 (the script's)")
    ap.add_argument("--stride", type=positive, default=4, help="frame_stride_dist in metres (4)")
    ap.add_argument("--radius", type=positive, default=50, help="accumulate_radius in metres (50)")
    ap.add_argument("--voxel", type=positive, default=0.4, help="voxel size in metres (0.4)")
    ap.add_argument("--batch", type=positive_int, default=64, help="output frames per device call (64)")
    a = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        sys.exit("build_kitti.py needs a CUDA device (sm_90a); there is no CPU path")
    from deepi2p_b200 import kitti_build
    for seq in a.seqs:
        kitti_build.build_sequence(a.root, seq, a.stride, a.radius, a.voxel, a.batch, log=lambda s: print(s, flush=True))


if __name__ == "__main__":
    main()
