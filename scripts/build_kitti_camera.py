"""Build a KITTI root's camera-frame scan records and LiDAR depth maps from the raw velodyne scans
(data/kitti/kitti_pc_bin_to_npy_in_img_frame.py, one GPU):

    python scripts/build_kitti_camera.py ROOT VELODYNE_ROOT [--seqs 0-21] [--batch 32] [--voxel 0.1]
                                         [--sn-radius 0.6] [--sn-max-nn 30]

VELODYNE_ROOT holds sequences/<seq>/velodyne/<frame>.bin; ROOT holds calib/<seq>/calib.txt and the frames' images
(data_odometry_color_npy/, or the official data_odometry_color/ PNGs), whose sizes the depth maps take.  Each
sequence writes data_odometry_velodyne_{P2,P3}_npy/sequences/<seq>/voxel<V>-SNr<R>/<frame>.npy and
data_odometry_color_depth_npy/sequences/<seq>/image_{2,3}/<frame>.npy; a sequence whose folders exist is skipped.
Prints one line per batch of scans.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from build_kitti import positive, positive_int, seq_list  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("root")
    ap.add_argument("velodyne_root")
    ap.add_argument("--seqs", type=seq_list, default=list(range(22)), help="sequences, e.g. 0-21 (the script's)")
    ap.add_argument("--batch", type=positive_int, default=32, help="scans per device call (32)")
    ap.add_argument("--voxel", type=positive, default=0.1, help="voxel size in metres (0.1)")
    ap.add_argument("--sn-radius", type=positive, default=0.6, help="normal search radius in metres (0.6)")
    ap.add_argument("--sn-max-nn", type=positive_int, default=30, help="normal neighbours at most (30)")
    a = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        sys.exit("build_kitti_camera.py needs a CUDA device (sm_90a); there is no CPU path")
    from deepi2p_b200 import kitti_depth
    kitti_depth.build_root(a.root, a.velodyne_root, a.seqs, a.voxel, a.sn_radius, a.sn_max_nn, a.batch,
                           log=lambda s: print(s, flush=True))


if __name__ == "__main__":
    main()
