#!/usr/bin/env python
"""Write the monodepth depth clouds of a hand-off root on the GPU (evaluation/icp/save_depth_map.py):

    python scripts/save_depth_map.py ROOT --depth-model models/mono+stereo_640x192 [--out DIR] [--batch 64]

For every frame id of ROOT/data (the first 9 characters of the file names), ROOT/visualization/<id>_img.png and
ROOT/data/<id>_K.npy give <out>/<id>_pc.npy (default out: ROOT/monodepth), the float64 [3, H*W] cloud the script
writes: Pillow's Lanczos resize to the checkpoint's feed size, monodepth2's ResNet-18 depth network, the bilinear
upsample of ("disp", 0) to the image size, its reciprocal, and np.linalg.inv(K) (in K's stored dtype) times
(d x, d y, d).  register_dir.py --method icp --monodepth reads the files.  Frames of one size go through the network
together, --batch at a time.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def positive_int(v):
    n = int(v)
    if n < 1:
        raise argparse.ArgumentTypeError(f"must be a positive integer (got {v})")
    return n


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("root", help="hand-off root holding data/ and visualization/")
    ap.add_argument("--depth-model", required=True, help="monodepth2 checkpoint directory (encoder.pth, depth.pth)")
    ap.add_argument("--out", default=None, help="output directory (default ROOT/monodepth)")
    ap.add_argument("--batch", type=positive_int, default=64, help="frames per network call (64)")
    a = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        sys.exit("save_depth_map.py needs a CUDA device (sm_90a); there is no CPU path")
    import numpy as np
    from deepi2p_b200 import imageprep, monodepth

    data_dir = os.path.join(a.root, "data")
    names = sorted({f[0:9] for f in os.listdir(data_dir) if os.path.isfile(os.path.join(data_dir, f))})
    out_dir = a.out if a.out is not None else os.path.join(a.root, "monodepth")
    os.makedirs(out_dir, exist_ok=True)
    model = monodepth.load_monodepth(a.depth_model)
    for i in range(0, len(names), a.batch):
        part = names[i:i + a.batch]
        images = imageprep.read_png_batch([os.path.join(a.root, "visualization", n + "_img.png") for n in part])
        K_inv = monodepth.k_inverse([np.load(os.path.join(data_dir, n + "_K.npy")) for n in part])
        groups = {}
        for s, hw in enumerate(map(tuple, images["shapes"])):
            groups.setdefault(hw, []).append(s)
        for idx in groups.values():
            sub = dict(data=images["data"], offsets=images["offsets"][idx], shapes=images["shapes"][idx])
            pc = monodepth.depth_clouds(model, sub, K_inv[idx])["pc"].cpu().numpy()
            for j, s in enumerate(idx):
                np.save(os.path.join(out_dir, part[s] + "_pc.npy"), pc[j])
                print(part[s], pc[j].shape, flush=True)


if __name__ == "__main__":
    main()
