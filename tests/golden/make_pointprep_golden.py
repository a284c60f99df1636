"""Write tests/golden/pointprep_small.npz: oracle_prep results on two small synthetic scans.

    python tests/golden/make_pointprep_golden.py

Scans: make_lidar_scan(40 + s, n_rings=16, n_azimuth=512) (8192 points each), voxel 0.25 m, normals with radius 0.8
and max_nn 30 on the float32-rounded centres, nearest original point of every centre.  tests/test_pointprep_cpu.py
checks that the oracle still reproduces them and tests/test_pointprep_gpu.py that the GPU does."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import oracle_prep  # noqa: E402
from deepi2p_b200 import synthetic  # noqa: E402

VOXEL, RADIUS, MAX_NN = 0.25, 0.8, 30


def scans():
    return [synthetic.make_lidar_scan(40 + s, n_rings=16, n_azimuth=512) for s in range(2)]


def compute():
    out = {}
    for s, sc in enumerate(scans()):
        down, _ = oracle_prep.voxel_downsample(sc["xyz"], VOXEL)
        nrm, cnt = oracle_prep.estimate_normals(down.astype(np.float32), RADIUS, MAX_NN)
        out[f"down{s}"] = down
        out[f"normals{s}"] = nrm
        out[f"count{s}"] = cnt
        out[f"nearest{s}"] = oracle_prep.nearest(sc["xyz"], down)
    return out


if __name__ == "__main__":
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pointprep_small.npz")
    np.savez_compressed(path, **compute())
    print(path, os.path.getsize(path), "bytes")
