"""The Oxford stereo-centre conversion on the device (DESIGN.md 4.25): decode_grey_png_batch, debayer_undistort_batch
and encode_jpeg_batch against tests/golden/oxford_images_small.npz (Pillow's pixels, the SDK pipeline's RGB and
cv2.imencode's bytes) bit for bit, and build_traversal(images=True) end to end."""
import hashlib
import io
import os

import numpy as np
import pytest
import torch

import oracle_oxford_images as o
from deepi2p_b200 import imageprep, oxford, oxford_build as ob, oxford_images as oi, synthetic as syn

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, "tests", "golden", "oxford_images_small.npz"))
T = "2014-05-19-13-20-57"


def _sha(b):
    return hashlib.sha256(b).hexdigest()


def _full(k):
    seed = int(G["full_seeds"][k])
    return syn.oxford_mosaic((960, 1280), seed), syn.oxford_distortion_lut(960, 1280, seed)


def _grey(mosaics):
    return imageprep.decode_grey_png_batch([syn.encode_png(m) for m in mosaics])


def test_decode_grey_png_batch_equals_pillow(cuda):
    n = int(G["png_n"])
    blobs = [G[f"png_blob_{i}"].tobytes() for i in range(n)]
    out = imageprep.decode_grey_png_batch(blobs)
    data = out["data"].cpu().numpy()
    for i in range(n):
        pix = G[f"png_pix_{i}"]
        assert tuple(out["shapes"][i]) == pix.shape
        assert np.array_equal(data[out["offsets"][i]:out["offsets"][i] + pix.size].reshape(pix.shape), pix), i
    one = imageprep.decode_grey_png_batch(blobs[-1:])
    assert np.array_equal(one["data"].cpu().numpy().reshape(G[f"png_pix_{n - 1}"].shape), G[f"png_pix_{n - 1}"])
    with pytest.raises(ValueError, match="image 1: unsupported colour type 0"):
        imageprep.decode_png_batch([syn.encode_png(np.zeros((4, 4, 3), np.uint8)), blobs[0]])
    with pytest.raises(ValueError, match="image 2: unsupported colour type 2"):
        imageprep.decode_grey_png_batch(blobs[:2] + [syn.encode_png(np.zeros((4, 4, 3), np.uint8))])
    bad = bytearray(blobs[3])
    bad[-20] ^= 0x55                                                    # inside the last IDAT: a CRC or inflate error
    with pytest.raises(ValueError, match="image 1: "):
        imageprep.decode_grey_png_batch([blobs[0], bytes(bad)])


def test_debayer_undistort_equals_sdk_pipeline(cuda):
    n = int(G["dm_n"])
    mos = [G[f"dm_mosaic_{i}"] for i in range(n)]
    luts = [G[f"dm_lut_{i}"] for i in range(n)]
    grey = _grey(mos)
    rgb = oi.debayer_undistort_batch(grey, luts)
    data = rgb["data"].cpu().numpy()
    for i in range(n):
        ref = G[f"dm_rgb_{i}"]
        assert np.array_equal(data[rgb["offsets"][i]:rgb["offsets"][i] + ref.size].reshape(ref.shape), ref), i
        alone = oi.debayer_undistort_batch(_grey([mos[i]]), torch.from_numpy(luts[i]).cuda())
        assert np.array_equal(alone["data"].cpu().numpy().reshape(ref.shape), ref), i
    # two full-size frames sharing one LUT upload, and each frame with its own LUT
    frames = [_full(k) for k in range(2)]
    both = oi.debayer_undistort_batch(_grey([m for m, _ in frames]), [lut for _, lut in frames])
    d = both["data"].cpu().numpy()
    for k in range(2):
        assert _sha(d[k * 3 * 960 * 1280:(k + 1) * 3 * 960 * 1280].tobytes()) == str(G[f"full_rgb_sha_{k}"]), k
    shared = oi.debayer_undistort_batch(_grey([frames[0][0]] * 3), frames[0][1])
    assert all(_sha(x.tobytes()) == str(G["full_rgb_sha_0"]) for x in np.split(shared["data"].cpu().numpy(), 3))


def _case_image(i):
    spec = str(G[f"enc_spec_{i}"])
    h, w = (int(v) for v in G[f"enc_shape_{i}"])
    if spec.startswith("dm:"):
        return G[f"dm_rgb_{int(spec[3:])}"]
    if spec.startswith("full:"):
        return None
    return o.fixture_image(spec, h, w)


def test_encode_jpeg_batch_equals_cv2_bytes(cuda):
    n = int(G["enc_n"])
    full = oi.debayer_undistort_batch(_grey([_full(k)[0] for k in range(2)]), [_full(k)[1] for k in range(2)])
    full_imgs = [x.reshape(960, 1280, 3) for x in np.split(full["data"].cpu().numpy(), 2)]
    cases = {}
    for i in range(n):
        img = _case_image(i)
        if img is None:
            img = full_imgs[int(str(G[f"enc_spec_{i}"])[5:])]
        cases.setdefault(int(G[f"enc_q_{i}"]), []).append((i, img))
    streams = {}
    for q, items in cases.items():
        got = imageprep.encode_jpeg_batch(imageprep.pack_images([img for _, img in items]), quality=q)
        again = imageprep.encode_jpeg_batch(imageprep.pack_images([img for _, img in items]), quality=q)
        assert got == again, q                                          # two runs are identical
        for (i, _), b in zip(items, got):
            streams[i] = b
            if f"enc_jpg_{i}" in G:
                assert b == G[f"enc_jpg_{i}"].tobytes(), (i, str(G[f"enc_spec_{i}"]), q)
            else:
                assert _sha(b) == str(G[f"enc_sha_{i}"]), (i, str(G[f"enc_spec_{i}"]), q)
    # each stream alone, and the produced streams through the project's own decoder against Pillow's decode
    for i in (0, 5, n - 1):
        img = _case_image(i) if _case_image(i) is not None else full_imgs[1]
        assert imageprep.encode_jpeg_batch(imageprep.pack_images([img]), quality=int(G[f"enc_q_{i}"]))[0] == streams[i]
    order = sorted(streams)
    dec = imageprep.decode_jpeg_batch([streams[i] for i in order])
    data = dec["data"].cpu().numpy()
    for k, i in enumerate(order):
        h, w = (int(v) for v in G[f"enc_shape_{i}"])
        px = data[dec["offsets"][k]:dec["offsets"][k] + 3 * h * w]
        if f"enc_pil_{i}" in G:
            assert np.array_equal(px.reshape(h, w, 3), G[f"enc_pil_{i}"]), i
        else:
            assert _sha(px.tobytes()) == str(G[f"enc_pilsha_{i}"]), i


def test_bad_inputs_raise(cuda):
    ok = _grey([G["dm_mosaic_0"], G["dm_mosaic_1"]])
    with pytest.raises(ValueError, match="image 1: Incorrect image size"):
        oi.debayer_undistort_batch(ok, [G["dm_lut_0"], G["dm_lut_0"]])
    with pytest.raises(ValueError, match="Incorrect image size"):
        oi.debayer_undistort_batch(ok, G["dm_lut_0"])
    with pytest.raises(ValueError, match="image 1: a 1 x 6 mosaic"):
        oi.debayer_undistort_batch(_grey([G["dm_mosaic_0"], np.zeros((1, 6), np.uint8)]),
                                   [G["dm_lut_0"], np.zeros((6, 2))])
    with pytest.raises(ValueError, match="non-finite"):
        oi.debayer_undistort_batch(ok, [G["dm_lut_0"], np.full_like(G["dm_lut_1"], np.inf)])
    with pytest.raises(ValueError, match="pattern"):
        oi.debayer_undistort_batch(ok, [G["dm_lut_0"], G["dm_lut_1"]], pattern="rggb")
    imgs = imageprep.pack_images([np.zeros((4, 4, 3), np.uint8)])
    with pytest.raises(ValueError, match="quality"):
        imageprep.encode_jpeg_batch(imgs, quality=0)
    bad = dict(imgs, shapes=np.array([[4, 70000]]))
    with pytest.raises(ValueError, match="image 0"):
        imageprep.encode_jpeg_batch(bad)
    assert imageprep.encode_jpeg_batch(imageprep.pack_images([])) == []


def _files(root):
    out = {}
    for d, _, files in os.walk(root):
        for f in files:
            p = os.path.join(d, f)
            with open(p, "rb") as fh:
                out[os.path.relpath(p, root)] = fh.read()
    return out


def test_build_traversal_images(tmp_path_factory, cuda):
    d = tmp_path_factory.mktemp("oximg")
    raw, lms, sdk = (str(d / x) for x in ("raw", "lms", "sdk"))
    syn.write_oxford_raw(raw, lms, sdk, seconds=12.0, stops=((6.0, 7.0),), curve=(3.0, 8.0), n_returns=8, seed=4,
                         image_shape=(96, 128))
    args = dict(accumulation_distance=6.0, ignore_first_n_second=1)
    plain, conv = str(d / "plain"), str(d / "conv")
    s0 = ob.build_traversal(raw, lms, plain, T, sdk, batch=5, **args)
    s1 = ob.build_traversal(raw, lms, conv, T, sdk, batch=5, images=True, **args)
    assert "images_converted" not in s0
    cams = [int(c) for c in np.load(os.path.join(conv, T, "camera_timestamps.npy"))]
    assert s1.pop("images_converted") == len(cams) == s1["camera_frames"] and s1.pop("images_skipped") == 0
    for k in s0:
        assert np.array_equal(s0[k], s1[k]), k
    a, b = _files(plain), _files(conv)
    jpgs = {k for k in b if k.endswith(".jpg")}
    assert {k for k in a if not k.endswith(".jpg")} == set(a) and set(b) - jpgs == set(a)
    assert all(a[k] == b[k] for k in a)
    lut = oi.read_distortion_lut(os.path.join(sdk, "models", oi.LUT_FILE), 96, 128)
    assert len(jpgs) == len(cams)
    for c in cams:
        m = syn.oxford_mosaic((96, 128), int(c))
        assert b[os.path.join(T, "stereo", "centre", "%d.jpg" % c)] == o.encode_jpeg(o.sdk_load_image(m, lut)), c
    # a second run converts nothing and reports every frame as skipped
    again = ob.build_traversal(raw, lms, conv, T, sdk, batch=5, images=True, **args)
    assert again["images_converted"] == 0 and again["images_skipped"] == len(cams)


def test_build_root_full_size_then_oxford_batch(tmp_path_factory, cuda):
    from PIL import Image
    d = tmp_path_factory.mktemp("oxfull")
    raw, lms, sdk, out = (str(d / x) for x in ("raw", "lms", "sdk", "out"))
    syn.write_oxford_raw(raw, lms, sdk, seconds=7.0, stops=(), curve=(2.0, 5.0), n_returns=8, seed=5, night=(),
                         image_shape=(960, 1280))
    os.makedirs(out)
    with open(os.path.join(out, "val.txt"), "w") as f:
        f.write(T + "\n")
    logs = []
    (s,) = ob.build_root(raw, lms, out, sdk, batch=16, log=logs.append, images=True, accumulation_distance=6.0,
                         ignore_first_n_second=1)
    assert s["images_converted"] == s["camera_frames"] > 0 and "images converted" in logs[-1]
    cams = np.load(os.path.join(out, T, "camera_timestamps.npy"))
    c = int(cams[len(cams) // 2])
    lut = oi.read_distortion_lut(os.path.join(sdk, "models", oi.LUT_FILE), 960, 1280)
    with open(os.path.join(out, T, "stereo", "centre", "%d.jpg" % c), "rb") as f:
        jpg = f.read()
    assert jpg == o.encode_jpeg(o.sdk_load_image(syn.oxford_mosaic((960, 1280), c), lut))
    assert np.asarray(Image.open(io.BytesIO(jpg))).shape == (960, 1280, 3)
    res = oxford.oxford_batch(out, [0, 1], "val", seed=5, rng=9, input_pt_num=256, node_a_num=8, node_b_num=8,
                              remove_ground=True)
    img = res[6]
    assert tuple(img.shape) == (2, 3, 384, 640) and float(img.float().std()) > 1.0
