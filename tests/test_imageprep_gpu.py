"""The image side on the H100 (deepi2p_b200.imageprep): bit-exact against the numpy oracle and the cv2 / Pillow
fixture for ragged KITTI batches, Oxford and nuScenes shapes, every jitter order, the range ends, flip, val mode,
S = 1 and a second stream; deterministic across runs; fed by assemble_batch's flip."""
import itertools

import numpy as np
import pytest
import torch

import oracle_image as oi
from deepi2p_b200 import assemble, imageprep, synthetic
from test_imageprep_cpu import golden, oracle_sample

pytestmark = pytest.mark.gpu

K_KITTI = np.array([[718.856, 0.0, 607.1928], [0.0, 718.856, 185.2157], [0.0, 0.0, 1.0]])


def frames_of(shapes, seed):
    """Smooth gradients plus noise, so resizing and the colour steps see both flat and busy regions."""
    rng = np.random.default_rng(seed)
    out = []
    for h, w in shapes:
        y, x = np.mgrid[0:h, 0:w]
        base = np.stack([255 * x / w, 255 * y / h, 127 + 120 * np.sin(x / 17.0 + y / 11.0)], -1)
        out.append(np.clip(base + rng.normal(0, 30, (h, w, 3)), 0, 255).astype(np.uint8))
    return out


def check(frames, K, out, flip):
    p = out["params"]
    img = out["img"].cpu().numpy()
    for s, fr in enumerate(frames):
        assert np.array_equal(img[s], oracle_sample(fr, p, s, flip[s])), s
    Ks = np.broadcast_to(np.asarray(K, np.float64), (len(frames), 3, 3))
    for s in range(len(frames)):
        ref = oi.camera_K(Ks[s], int(p["row0"][s]), p["scale"], int(p["dx"][s]), int(p["dy"][s]))
        assert np.array_equal(out["K64"][s], ref) and np.array_equal(out["K"][s].numpy(), ref.astype(np.float32)), s


def test_golden_fixture(cuda):
    g = golden()
    packed = imageprep.pack_images(g["frames"])
    out = imageprep.assemble_images(packed, g["K"], params=g["params"], flip=g["flip"])
    assert out["img"].dtype == torch.float32 and out["img"].shape == g["img"].shape
    assert np.array_equal(out["img"].cpu().numpy(), g["img"].astype(np.float32))
    assert np.array_equal(out["K64"], g["K_out"]) and np.array_equal(out["K"].numpy(), g["K_out"].astype(np.float32))
    u8 = imageprep.assemble_images(packed, g["K"], params=g["params"], flip=g["flip"], out_dtype=torch.uint8)
    assert np.array_equal(u8["img"].cpu().numpy(), g["img"])


def test_ragged_kitti_train_batch(cuda):
    shapes = [(370, 1226), (375, 1242), (376, 1241), (376, 1241)]
    frames = frames_of(shapes, 1)
    flip = np.array([False, True, True, False])
    out = imageprep.assemble_images(imageprep.pack_images(frames), K_KITTI, "train", rng=3, flip=flip,
                                    **imageprep.kitti_image_args())
    assert out["params"]["jitter"].all() and list(out["params"]["dw"]) == [613, 621, 620, 620]
    check(frames, K_KITTI, out, flip)
    again = imageprep.assemble_images(imageprep.pack_images(frames), K_KITTI, params=out["params"], flip=flip)
    assert torch.equal(again["img"], out["img"])                       # a repeat is bit-identical


@pytest.mark.parametrize("mode", ["train", "val"])
def test_oxford_and_nuscenes_shapes(cuda, mode):
    frames = frames_of([(960, 1280)] * 3, 2)
    K = np.array([[983.0, 0.0, 643.6], [0.0, 983.0, 484.4], [0.0, 0.0, 1.0]])
    out = imageprep.assemble_images(imageprep.pack_images(frames), K, mode, rng=np.random.default_rng(4),
                                    **imageprep.oxford_image_args())
    assert out["img"].shape == (3, 3, 384, 640)
    check(frames, K, out, np.zeros(3, bool))
    nus = frames_of([(900, 1600)] * 2, 3)
    args = dict(img_H=160, img_W=320, img_scale=0.2, crop_top_rows=100, jitter_prob=1.0)
    out = imageprep.assemble_images(imageprep.pack_images(nus), K, mode, rng=5, **args)
    assert list(out["params"]["dh"]) == [160, 160] and list(out["params"]["dw"]) == [320, 320]
    check(nus, K, out, np.zeros(2, bool))


def test_all_orders_range_ends_and_flip(cuda):
    orders = np.array(list(itertools.permutations(range(4))), np.int32)
    S = len(orders)
    shapes = [(120 + s % 3, 300 + 7 * s) for s in range(S)]
    frames = frames_of(shapes, 6)
    p = imageprep.image_params(shapes, "train", 7, img_H=48, img_W=128, img_scale=0.5, crop_top_rows=5)
    ends = np.array([[0.8, 1.2, 0.8, -0.1], [1.2, 0.8, 1.2, 0.1], [1.2, 1.2, 0.8, -0.1], [0.8, 0.8, 1.2, 0.1]],
                    np.float32)
    p = dict(p, order=orders, factors=ends[np.arange(S) % 4], jitter=np.ones(S, bool))
    for flip in (np.arange(S) % 2 == 1, np.arange(S) % 2 == 0):
        out = imageprep.assemble_images(imageprep.pack_images(frames), K_KITTI, params=p, flip=flip)
        check(frames, K_KITTI, out, flip)


def test_val_mode_single_sample_and_second_stream(cuda):
    frames = frames_of([(376, 1241)], 8)
    packed = imageprep.pack_images(frames)
    out = imageprep.assemble_images(packed, K_KITTI, "val", **imageprep.kitti_image_args())
    p = out["params"]
    assert not p["jitter"].any() and (int(p["dx"][0]), int(p["dy"][0])) == (54, 1)
    check(frames, K_KITTI, out, [False])
    shapes = [(370, 1226), (376, 1241), (375, 1242)]
    frames = frames_of(shapes, 9)
    packed = imageprep.pack_images(frames)
    ref = imageprep.assemble_images(packed, K_KITTI, "train", rng=10, **imageprep.kitti_image_args())
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        other = imageprep.assemble_images(packed, K_KITTI, params=ref["params"], stream=st)
    st.synchronize()
    assert torch.equal(other["img"], ref["img"])
    check(frames, K_KITTI, ref, np.zeros(3, bool))


def test_assemble_batch_flip_feeds_the_images(cuda):
    smps = [synthetic.make_loader_sample(40 + s, "kitti", n_rings=8, n_azimuth=128) for s in range(6)]
    fr = assemble.pack_frames([(m["frames"], m["frame_T"]) for m in smps])
    pts = assemble.assemble_batch(fr, "train", 3, input_pt_num=2048, node_a_num=32, node_b_num=32, rng=2,
                                  **dict(assemble.kitti_args(smps[0]["Pc"]), jitter=()))
    assert pts["flip"].any() and not pts["flip"].all()
    frames = frames_of([(376, 1241)] * 6, 11)
    K = np.stack([m["K"] for m in smps])
    out = imageprep.assemble_images(imageprep.pack_images(frames), K, "train", rng=12, flip=pts["flip"],
                                    **imageprep.kitti_image_args())
    check(frames, K, out, pts["flip"])
    plain = imageprep.assemble_images(imageprep.pack_images(frames), K, params=out["params"])
    f = pts["flip"]
    assert torch.equal(plain["img"][f].flip(-1), out["img"][f]) and torch.equal(plain["img"][~f], out["img"][~f])


def test_rejects_before_launch(cuda):
    frames = frames_of([(376, 1241)], 1)
    packed = imageprep.pack_images(frames)
    with pytest.raises(ValueError, match="smaller than"):
        imageprep.assemble_images(packed, K_KITTI, "train", rng=1, **dict(imageprep.kitti_image_args(), img_W=640))
    with pytest.raises(ValueError, match="flip"):
        imageprep.assemble_images(packed, K_KITTI, "train", rng=1, flip=[True, False], **imageprep.kitti_image_args())
    with pytest.raises(ValueError, match="K must"):
        imageprep.assemble_images(packed, np.eye(4), "train", rng=1, **imageprep.kitti_image_args())
