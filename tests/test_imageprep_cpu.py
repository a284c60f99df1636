"""The image side's numpy oracle (oracle_image) against cv2, Pillow and torchvision where they are importable, and
against tests/golden/image_small.npz always; resize dimensions, K, the host draws and the host argument checks."""
import ctypes
import itertools
import os

import numpy as np
import pytest

import oracle_image as oi
from deepi2p_b200 import imageprep

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "image_small.npz")
ORDERS = list(itertools.permutations(range(4)))


def golden():
    """The fixture as frames, image_params-style params, K and the expected outputs."""
    z = np.load(GOLDEN)
    shapes = z["shapes"]
    sizes = 3 * shapes[:, 0] * shapes[:, 1]
    offsets = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    frames = [z["frames"][o:o + n].reshape(h, w, 3) for o, n, (h, w) in zip(offsets, sizes, shapes)]
    p = z["params"]
    H, W = (int(v) for v in z["img_HW"])
    params = dict(row0=p[:, 0], rows=p[:, 1], dh=p[:, 2], dw=p[:, 3], dy=p[:, 4], dx=p[:, 5], jitter=p[:, 7] == 1,
                  order=p[:, 8:12].astype(np.int32), factors=z["factors"], scale=z["scale"], img_H=H, img_W=W)
    return dict(frames=frames, params=params, flip=p[:, 6] == 1, scale=z["scale"], K=z["K"], K_out=z["K_out"],
                img=z["img"])


def oracle_sample(frame, p, s, flip):
    """oracle_image.assemble_image for sample s of an image_params-style dict."""
    img, _ = oi.assemble_image(frame, None, int(p["row0"][s]), int(p["rows"][s]), int(p["dh"][s]), int(p["dw"][s]),
                               int(p["dy"][s]), int(p["dx"][s]), p["img_H"], p["img_W"], flip=bool(flip),
                               jitter=bool(p["jitter"][s]), order=p["order"][s], factors=p["factors"][s])
    return img


def adversarial_image():
    """Grey pixels, ties of the maximum channel, primaries and secondaries, every level in every channel."""
    rng = np.random.default_rng(11)
    lv = np.arange(256, dtype=np.uint8)
    a = rng.integers(0, 256, (24, 256, 3), dtype=np.uint8)
    a[0] = lv[:, None]                                        # greys, all 256 levels
    for c in range(3):
        a[1 + c, :, :] = 0
        a[1 + c, :, c] = lv                                   # each channel alone, all levels
        a[4 + c] = lv[:, None]
        a[4 + c, :, c] = 255 - lv                             # one channel against two equal ones
    prim = np.array([[255, 0, 0], [0, 255, 0], [0, 0, 255], [255, 255, 0], [0, 255, 255], [255, 0, 255],
                     [0, 0, 0], [255, 255, 255], [7, 7, 3], [3, 7, 7], [7, 3, 7], [1, 1, 0]], np.uint8)
    a[7] = prim[np.arange(256) % len(prim)]
    a[8, :, 0] = lv                                            # r == g ties at every level, b below
    a[8, :, 1] = lv
    a[8, :, 2] = lv // 2
    a[9, :, 1] = lv                                            # g == b ties, r below
    a[9, :, 2] = lv
    a[9, :, 0] = lv // 3
    return a


def test_golden_fixture_matches_oracle():
    g = golden()
    p = g["params"]
    for s, fr in enumerate(g["frames"]):
        assert np.array_equal(oracle_sample(fr, p, s, g["flip"][s]), g["img"][s].astype(np.float32)), s
        K = oi.camera_K(g["K"][s], int(p["row0"][s]), float(g["scale"][s]), int(p["dx"][s]), int(p["dy"][s]))
        assert np.array_equal(K, g["K_out"][s]), s
        assert (int(p["dh"][s]), int(p["dw"][s])) == oi.resize_dims(int(p["rows"][s]), fr.shape[1], g["scale"][s])
    assert np.array_equal(imageprep.camera_K(g["K"], p["row0"], p["scale"], p["dx"], p["dy"]), g["K_out"])


@pytest.mark.parametrize("h,w,s", [(326, 1241, 0.5), (320, 1226, 0.5), (325, 1242, 0.5), (800, 1600, 0.2),
                                   (960, 1280, 0.5), (101, 77, 0.37), (33, 47, 0.9), (50, 60, 1.0)])
def test_resize_matches_cv2(h, w, s):
    cv2 = pytest.importorskip("cv2")
    img = np.random.default_rng(h * w).integers(0, 256, (h, w, 3), dtype=np.uint8)
    dh, dw = oi.resize_dims(h, w, s)
    ref = cv2.resize(img, (dw, dh), interpolation=cv2.INTER_LINEAR)
    assert np.array_equal(oi.resize_window(img, dh, dw), ref)
    assert np.array_equal(oi.resize_window(img, dh, dw, 3, 5, dh - 7, dw - 9), ref[3:dh - 4, 5:dw - 4])


def test_resize_dims_of_kitti_frames():
    """KITTI frames are 370 x 1226, 375 x 1242 or 376 x 1241; after the 50-row cut cv2 gets round(h/2) x round(w/2)
    with ties to even, so 1241 -> 620 and 325 -> 162: not an exact 2x."""
    top = imageprep.kitti_image_args()["crop_top_rows"]
    got = {(h, w): imageprep.resize_dims(h - top, w, 0.5) for h, w in ((370, 1226), (375, 1242), (376, 1241))}
    assert got == {(370, 1226): (160, 613), (375, 1242): (162, 621), (376, 1241): (163, 620)}
    for (h, w), d in got.items():
        assert oi.resize_dims(h - top, w, 0.5) == d
    assert imageprep.resize_dims(800, 1600, 0.2) == (160, 320)
    assert imageprep.resize_dims(960, 1280, 0.5) == (480, 640)


def test_exact_half_is_the_area_average():
    img = np.random.default_rng(3).integers(0, 256, (40, 60, 3), dtype=np.uint8)
    q = img.astype(np.int64)
    avg = (q[0::2, 0::2] + q[0::2, 1::2] + q[1::2, 0::2] + q[1::2, 1::2] + 2) >> 2
    assert np.array_equal(oi.resize_window(img, 20, 30), avg)


FACTORS = (0.0, 0.8, 0.9, 1.0, 1.13, 1.2, 1.7)
HUES = (-0.5, -0.1, -0.05, -0.001, 0.0, 0.013, 0.1, 0.37, 0.5)


@pytest.mark.parametrize("which", ["random", "adversarial"])
def test_each_colour_step_matches_pil(which):
    pytest.importorskip("PIL")
    F = pytest.importorskip("torchvision.transforms.functional")
    from PIL import Image
    img = adversarial_image() if which == "adversarial" else \
        np.random.default_rng(7).integers(0, 256, (48, 160, 3), dtype=np.uint8)
    P = Image.fromarray(img)
    for f in FACTORS:
        assert np.array_equal(np.array(F.adjust_brightness(P, f)), oi.adjust_brightness(img, f)), f
        assert np.array_equal(np.array(F.adjust_contrast(P, f)), oi.adjust_contrast(img, f)), f
        assert np.array_equal(np.array(F.adjust_saturation(P, f)), oi.adjust_saturation(img, f)), f
    for hf in HUES:
        assert np.array_equal(np.array(F.adjust_hue(P, hf)), oi.adjust_hue(img, oi.hue_shift(hf))), hf


def test_all_orders_match_torchvision():
    pytest.importorskip("PIL")
    F = pytest.importorskip("torchvision.transforms.functional")
    from PIL import Image
    img = np.concatenate([adversarial_image()[:, :128],
                          np.random.default_rng(8).integers(0, 256, (24, 128, 3), dtype=np.uint8)])
    steps = (F.adjust_brightness, F.adjust_contrast, F.adjust_saturation, F.adjust_hue)
    for i, order in enumerate(ORDERS):
        fac = np.float32([(0.8, 1.2)[i % 2], (1.2, 0.8)[(i // 2) % 2], (0.8, 1.2)[(i // 4) % 2], (-0.1, 0.1)[i % 3 == 0]])
        P = Image.fromarray(img)
        for op in order:
            P = steps[op](P, float(fac[op]))
        assert np.array_equal(np.array(P), oi.color_jitter(img, order, fac)), order


def test_hue_round_trip_loses_information_at_zero_shift():
    img = adversarial_image()
    out = oi.adjust_hue(img, 0)
    assert not np.array_equal(out, img)                     # the HSV round trip is kept even at hue 0
    grey = img[0]
    assert np.array_equal(out[0], grey)                     # s == 0 gives v exactly


def test_negative_hue_wraps():
    assert [oi.hue_shift(h) for h in (-0.1, 0.1, 0.0, -0.5, 0.5, -0.001)] == [231, 25, 0, 129, 127, 0]
    assert [imageprep.hue_shift(h) for h in (-0.1, 0.1, 0.0, -0.5, 0.5, -0.001)] == [231, 25, 0, 129, 127, 0]
    img = adversarial_image()
    h, s, v = oi.rgb2hsv(img)
    assert np.array_equal(oi.adjust_hue(img, 231), oi.hsv2rgb((h + 231) % 256, s, v))
    assert np.array_equal(oi.adjust_hue(img, 231), oi.hsv2rgb((h - 25) % 256, s, v))


def test_contrast_grey_level_rounds_half_up():
    assert oi.contrast_degenerate(5, 2) == 3 and oi.contrast_degenerate(3, 2) == 2 and oi.contrast_degenerate(0, 7) == 0


def camera_matrix_cropping(K, dx, dy):        # data/kitti_helper.py, restated
    K_crop = np.copy(K)
    K_crop[0, 2] -= dx
    K_crop[1, 2] -= dy
    return K_crop


def camera_matrix_scaling(K, s):
    K_scale = s * K
    K_scale[2, 2] = 1
    return K_scale


def test_K_matches_the_loader_updates():
    rng = np.random.default_rng(4)
    K = np.array([[718.856, 0.0, 607.1928], [0.0, 718.856, 185.2157], [0.0, 0.0, 1.0]])
    for args, shapes in ((imageprep.kitti_image_args(), [(376, 1241), (370, 1226)]),
                         (imageprep.oxford_image_args(), [(960, 1280), (960, 1280)])):
        p = imageprep.image_params(shapes, "train", rng, **args)
        got = imageprep.camera_K(np.stack([K, K]), p["row0"], p["scale"], p["dx"], p["dy"])
        for s in range(2):
            ref = camera_matrix_cropping(K, 0, args["crop_top_rows"])
            ref = camera_matrix_scaling(ref, args["img_scale"])
            ref = camera_matrix_cropping(ref, int(p["dx"][s]), int(p["dy"][s]))
            assert np.array_equal(got[s], ref)
            assert np.array_equal(oi.camera_K(K, int(p["row0"][s]), p["scale"], int(p["dx"][s]), int(p["dy"][s])),
                                  ref)


def test_image_params_draws():
    shapes = [(376, 1241)] * 400
    a = imageprep.image_params(shapes, "train", 3, **imageprep.kitti_image_args())
    b = imageprep.image_params(shapes, "train", 3, **imageprep.kitti_image_args())
    for k in ("dx", "dy", "order", "factors", "jitter"):
        assert np.array_equal(a[k], b[k]), k                 # a seed reproduces the draws
    assert a["jitter"].all()                                  # KITTI jitters every train sample
    assert (a["dh"] == 163).all() and (a["dw"] == 620).all()
    assert a["dx"].min() == 0 and a["dx"].max() == 620 - 512 and a["dy"].max() <= 3
    assert (np.sort(a["order"], 1) == np.arange(4)).all() and len({tuple(o) for o in a["order"]}) == 24
    f = a["factors"]
    assert f.dtype == np.float32 and (f[:, :3] >= 0.8).all() and (f[:, :3] <= 1.2).all()
    assert (np.abs(f[:, 3]) <= np.float32(0.1)).all() and f[:, 3].min() < -0.05 and f[:, 3].max() > 0.05
    o = imageprep.image_params([(960, 1280)] * 400, "train", 5, **imageprep.oxford_image_args())
    assert 150 < o["jitter"].sum() < 250                      # Oxford jitters with probability 1/2
    assert (o["dh"] == 480).all() and o["dy"].max() <= 96
    v = imageprep.image_params([(376, 1241), (370, 1226)], "val", None, **imageprep.kitti_image_args())
    assert list(v["dx"]) == [(620 - 512) // 2, (613 - 512) // 2] and list(v["dy"]) == [1, 0]
    assert not v["jitter"].any()
    n = imageprep.image_params([(900, 1600)], "test", None, img_H=160, img_W=320, img_scale=0.2, crop_top_rows=100)
    assert (int(n["dh"][0]), int(n["dw"][0]), int(n["dx"][0]), int(n["dy"][0])) == (160, 320, 0, 0)


def test_host_argument_rejection():
    args = imageprep.kitti_image_args()
    with pytest.raises(ValueError, match="mode"):
        imageprep.image_params([(376, 1241)], "fit", 0, **args)
    with pytest.raises(ValueError, match="img_scale"):
        imageprep.image_params([(376, 1241)], "train", 0, **dict(args, img_scale=1.5))
    with pytest.raises(ValueError, match="img_scale"):
        imageprep.image_params([(376, 1241)], "train", 0, **dict(args, img_scale=0.0))
    with pytest.raises(ValueError, match="smaller than"):
        imageprep.image_params([(300, 1241)], "train", 0, **args)
    with pytest.raises(ValueError, match="no row"):
        imageprep.image_params([(40, 1241)], "train", 0, **args)
    with pytest.raises(TypeError):
        imageprep.image_params([(376, 1241)], "train", 0, gamma=(0, 1), **args)
    with pytest.raises(ValueError, match="uint8"):
        imageprep.pack_images([np.zeros((4, 4, 3), np.float32)], device="cpu")
    with pytest.raises(ValueError, match="uint8"):
        imageprep.pack_images([np.zeros((4, 4), np.uint8)], device="cpu")
    shapes = np.array([[376, 1241]])
    good = imageprep.image_params(shapes, "train", 0, **args)
    imageprep._pack_params(shapes, good, np.zeros(1, bool))
    for key, val, msg in (("order", [[0, 1, 1, 3]], "permutation"), ("dx", [109], "crop offset"),
                          ("dy", [-1], "crop offset"), ("dw", [1242], "downscale"), ("dh", [150], "smaller"),
                          ("row0", [330], "row cut"), ("factors", [[1, np.nan, 1, 0]], "finite"),
                          ("dx", [0, 0], "one entry")):
        with pytest.raises(ValueError, match=msg):
            imageprep._pack_params(shapes, dict(good, **{key: np.array(val)}), np.zeros(1, bool))


def test_c_abi_rejects_bad_parameters_before_device_work():
    from deepi2p_b200 import _native
    lib = _native.load()
    S, H, W = 1, 16, 32
    ws_bytes = lib.image_assemble_workspace_bytes(S, H, W)
    assert ws_bytes > 0 and lib.image_assemble_workspace_bytes(S, 0, W) == 0
    buf = ctypes.create_string_buffer(64)
    fake = ctypes.addressof(buf)

    def call(params, factors=(1.0, 1.0, 1.0), offsets=(0,), src_bytes=60 * 100 * 3, ws=ws_bytes):
        P = np.zeros((S, imageprep.IMAGE_PARAMS), np.int32)
        P[0, :len(params)] = params
        off = np.asarray(offsets, np.int64)
        fac = np.asarray(factors, np.float32)
        rc = lib.image_assemble_f32(fake, src_bytes, off.ctypes.data, P.ctypes.data, fac.ctypes.data, S, H, W, fake,
                                    fake, ws, None)
        return rc, lib.dib_last_error()

    ok = [60, 100, 4, 50, 25, 50, 3, 10, 0, 1, 0, 1, 2, 3, 231]    # h w row0 rows dh dw dy dx flip jitter order shift
    cases = [
        (dict(params=ok[:4] + [51] + ok[5:]), b"downscale"),
        (dict(params=ok[:4] + [15] + ok[5:]), b"smaller than"),
        (dict(params=ok[:6] + [10] + ok[7:]), b"crop offset"),
        (dict(params=ok[:2] + [20, 41] + ok[4:]), b"rows"),
        (dict(params=ok[:10] + [0, 1, 1, 3, 231]), b"permutation"),
        (dict(params=ok[:14] + [256]), b"hue shift"),
        (dict(params=ok[:8] + [2] + ok[9:]), b"flip and jitter"),
        (dict(params=ok, factors=(1.0, np.inf, 1.0)), b"finite"),
        (dict(params=ok, offsets=(8,)), b"outside"),
        (dict(params=ok, src_bytes=100), b"outside"),
    ]
    for kw, msg in cases:
        rc, err = call(**kw)
        assert rc == -22 and msg in err, (kw, err)
    rc, err = call(ok, ws=ws_bytes - 1)
    assert rc == -12 and b"workspace" in err


def test_augment_img_dropin_matches_oracle():
    pytest.importorskip("torchvision")
    img = np.random.default_rng(9).integers(0, 256, (40, 96, 3), dtype=np.uint8)
    for seed in range(6):
        out = imageprep.augment_img(img, np.random.default_rng(seed))
        order, fac = imageprep._draw_jitter(np.random.default_rng(seed), 1, *imageprep.JITTER_RANGES.values())
        assert out.dtype == np.uint8 and out.shape == img.shape
        assert np.array_equal(out, oi.color_jitter(img, order[0], fac[0])), seed
