"""kitti_batch on a KITTI root in the official PNG layout (data_odometry_color/.../<frame>.png, decoded on the GPU)
against the same root with the frames converted to .npy: every output equal, in train, val and val_random_Ry."""
import os

import numpy as np
import pytest
import torch

from deepi2p_b200 import kitti, synthetic

pytestmark = pytest.mark.gpu
KN, KM = 2048, 64


@pytest.fixture(scope="module")
def roots(tmp_path_factory):
    out = {}
    for fmt in ("npy", "png"):
        out[fmt] = str(tmp_path_factory.mktemp("kitti_" + fmt))
        synthetic.write_kitti_root(out[fmt], seqs=(0, 9, 10), n_frames=90, seed=5, images=fmt)
    return out


def test_roots_differ_only_in_the_image_format(roots):
    assert kitti.image_dir(roots["png"], 9, "P2").endswith(os.path.join("data_odometry_color", "sequences", "09",
                                                                        "image_2"))
    assert kitti.image_path(roots["png"], 9, "P3", 5).endswith(os.path.join("image_3", "000005.png"))
    assert kitti.image_path(roots["npy"], 9, "P3", 5).endswith(os.path.join("image_3", "000005.npy"))
    assert kitti.sequence_length(roots["png"], 9) == kitti.sequence_length(roots["npy"], 9) == 90


@pytest.mark.parametrize("mode", ["train", "val", "val_random_Ry"])
def test_png_root_equals_npy_root(cuda, roots, mode):
    seqs = (0,) if mode == "train" else (9, 10)
    got = []
    for fmt in ("npy", "png"):
        ds = kitti.KittiDataset(roots[fmt], mode, seqs=seqs)
        items = [0, 1, 3, 7, len(ds) - 1, 2]
        got.append(kitti.kitti_batch(ds, items, mode, 11, rng=21, input_pt_num=KN, node_a_num=KM, node_b_num=KM))
    torch.cuda.synchronize()
    for a, b in zip(*got):
        assert a.shape == b.shape and torch.equal(a.cpu(), b.cpu())
    assert got[1][6].shape == (6, 3, 160, 512) and got[1][6].abs().sum() > 0
