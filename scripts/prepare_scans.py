"""KITTI scan preparation on the GPU (data/kitti/kitti_pc_bin_to_npy_with_downsample_sn.py without Open3D):

    python scripts/prepare_scans.py VELODYNE_DIR OUT_DIR [--voxel 0.1 --sn-radius 0.6 --sn-max-nn 30 --batch 64]

reads every %06d.bin of VELODYNE_DIR (N x 4 little-endian float32: x, y, z, reflectance) and writes OUT_DIR/%06d.npy,
a [7, M] float32 record (downsampled xyz, intensity of the nearest original point, surface normal) in the reference's
layout.  Scans go through deepi2p_b200.pointprep.prepare_scans --batch at a time.
"""
import argparse
import os
import re
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("velodyne_dir")
    ap.add_argument("out_dir")
    ap.add_argument("--voxel", type=float, default=0.1)
    ap.add_argument("--sn-radius", type=float, default=0.6)
    ap.add_argument("--sn-max-nn", type=int, default=30)
    ap.add_argument("--batch", type=int, default=64)
    a = ap.parse_args(argv)
    import torch
    from deepi2p_b200 import pointprep
    from deepi2p_b200.icp import pack_clouds
    names = sorted(f for f in os.listdir(a.velodyne_dir) if re.fullmatch(r"\d{6}\.bin", f))
    os.makedirs(a.out_dir, exist_ok=True)
    for b in range(0, len(names), a.batch):
        chunk = names[b:b + a.batch]
        scans = [pointprep.read_velodyne_bin(os.path.join(a.velodyne_dir, f)) for f in chunk]
        xyz, n = pack_clouds([s[:3] for s in scans])
        inten = torch.zeros((len(scans), xyz.shape[2]), dtype=torch.float32)
        for s, scan in enumerate(scans):
            inten[s, :scan.shape[1]] = torch.from_numpy(scan[3])
        rec, m = pointprep.prepare_scans(xyz, inten.to(xyz.device), n, a.voxel, a.sn_radius, a.sn_max_nn)
        rec, m = rec.cpu().numpy(), m.cpu().numpy()
        for s, f in enumerate(chunk):
            np.save(os.path.join(a.out_dir, f[:-4] + ".npy"), rec[s, :, :m[s]])
        print(f"{b + len(chunk)}/{len(names)} scans", flush=True)


if __name__ == "__main__":
    main()
