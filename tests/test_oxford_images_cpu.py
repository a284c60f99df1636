"""The Oxford stereo-centre conversion's rules on the CPU (DESIGN.md 4.25): oracle_oxford_images against scipy's own
map_coordinates and the SDK pipeline fixture, the encoder restatement plus deepi2p_b200.jpeg_encode's markers against
cv2.imencode's bytes (tests/golden/oxford_images_small.npz), the host checks and the synthetic raw writer."""
import hashlib
import os

import numpy as np
import pytest

import oracle_oxford_images as o
from deepi2p_b200 import jpeg_encode as je, oxford_images, png, synthetic as syn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, "tests", "golden", "oxford_images_small.npz"))
# write_oxford_raw() with its defaults: the digest of every file it writes, as before image_shape existed.
RAW_DEFAULT_DIGEST = "1308b606afbf1c95b6775fe779cb82d0c7fbbe2383917979d6819000c75a50d7"


def _sha(b):
    return hashlib.sha256(b).hexdigest()


def _enc_image(i):
    spec = str(G[f"enc_spec_{i}"])
    h, w = (int(v) for v in G[f"enc_shape_{i}"])
    if spec.startswith("dm:"):
        return G[f"dm_rgb_{int(spec[3:])}"]
    if spec.startswith("full:"):
        seed = int(G["full_seeds"][int(spec[5:])])
        return o.sdk_load_image(syn.oxford_mosaic((h, w), seed), syn.oxford_distortion_lut(h, w, seed))
    return o.fixture_image(spec, h, w)


def test_map_coordinates_restatement_equals_scipy():
    from scipy.ndimage import map_coordinates
    rng = np.random.default_rng(7)
    for H, W in ((37, 53), (2, 2), (960, 1280)):
        ch = rng.integers(0, 2296, (H, W)).astype(np.float64) * 0.25       # multiples of 0.25 up to 573.75
        n = 1_000_000 if H == 37 else 100_000
        y = rng.uniform(-1.5, H + 0.5, n)
        x = rng.uniform(-1.5, W + 0.5, n)
        sp = np.array([0.0, -0.0, 1.0, H - 1.0, W - 1.0, np.nextafter(H - 1.0, 0), np.nextafter(W - 1.0, 0), -1e-9,
                       H - 1 + 1e-9, W - 1 + 1e-9, 1e-300, -1e-300, np.nextafter(1.0, 0), 0.5, -7.0, H + 9.0])
        sy, sx = np.meshgrid(sp, sp)
        c = np.stack([np.concatenate([y, sy.ravel()]), np.concatenate([x, sx.ravel()])])
        ref = map_coordinates(ch, c, order=1)
        got = o.map_coordinates_order1(ch, c)
        assert np.array_equal(ref.view(np.int64), got.view(np.int64)), (H, W)


def test_demosaic_sums_equal_colour_demosaicing_rules():
    rng = np.random.default_rng(3)
    for shape in ((2, 2), (7, 5), (16, 24)):
        cfa = rng.integers(0, 256, shape, dtype=np.uint8)
        assert np.array_equal(o.demosaic_sums(cfa) * 0.25, o.sdk_demosaic(cfa))


def test_oracle_pipeline_equals_fixture():
    for i in range(int(G["dm_n"])):
        mosaic, lut, rgb = G[f"dm_mosaic_{i}"], G[f"dm_lut_{i}"], G[f"dm_rgb_{i}"]
        assert np.array_equal(o.sdk_load_image(mosaic, lut), rgb), i
        assert np.array_equal(o.debayer_undistort(mosaic, lut), rgb), i


def test_oracle_pipeline_full_frames():
    for k, seed in enumerate(G["full_seeds"]):
        m, lut = syn.oxford_mosaic((960, 1280), int(seed)), syn.oxford_distortion_lut(960, 1280, int(seed))
        got = o.debayer_undistort(m, lut)
        assert _sha(got.tobytes()) == str(G[f"full_rgb_sha_{k}"]), k
        # the reflected borders push demosaiced values past 255; numpy's cast wraps them, and so does the fixture
        assert (o.demosaic_sums(m) > 4 * 255).any()


def test_encoder_restatement_equals_cv2_bytes():
    for i in range(int(G["enc_n"])):
        got = o.encode_jpeg(_enc_image(i), int(G[f"enc_q_{i}"]))
        if f"enc_jpg_{i}" in G:
            assert got == G[f"enc_jpg_{i}"].tobytes(), (i, str(G[f"enc_spec_{i}"]))
        else:
            assert _sha(got) == str(G[f"enc_sha_{i}"]), (i, str(G[f"enc_spec_{i}"]))


def test_header_and_tables():
    # force_baseline clamps to 1..255; quality 100 gives all ones, quality 1 the scaled tables clamped at 255
    assert (je.quant_tables(100) == 1).all()
    assert je.quant_tables(1).max() == 255 and je.quant_tables(50)[0, 0] == 16
    assert je.quality_scaling(0) == 5000 and je.quality_scaling(101) == 0
    assert je.max_block_bits() == 1660 and -(-je.max_block_bits() // 8) == je.MAX_BLOCK_BYTES
    h = je.header(961, 1281, 95)
    assert h[:2] == b"\xFF\xD8" and h[-14:-12] == b"\xFF\xDA"
    assert [h[i + 1] for i in range(len(h) - 1) if h[i] == 0xFF and h[i + 1] in (0xDB, 0xC0, 0xC4)] == \
        [0xDB, 0xDB, 0xC0, 0xC4, 0xC4, 0xC4, 0xC4]
    t = je.device_tables()
    assert t[0, 0] == (2 << 16) | 0 and t[1, 0] == (4 << 16) | 0b1010     # DC luma category 0, AC luma EOB
    g = je.geometry(961, 1281)
    assert (g["mcux"], g["mcuy"], g["ybx"], g["yby"], g["blocks"]) == (81, 61, 161, 121, 6 * 81 * 61)
    for hw in ((0, 5), (5, 0), (65501, 1)):
        with pytest.raises(ValueError, match="image 3"):
            je.check_shape(*hw, "image 3")


def test_lut_errors(tmp_path):
    lut = syn.oxford_distortion_lut(6, 8, 1)
    p = str(tmp_path / "lut.bin")
    np.concatenate([lut[:, 0], lut[:, 1]]).tofile(p)
    assert np.array_equal(oxford_images.read_distortion_lut(p, 6, 8), lut)
    with pytest.raises(ValueError, match="Incorrect image size"):
        oxford_images.read_distortion_lut(p, 8, 8)
    np.concatenate([lut[:, 0], lut[:, 1], [1.0]]).tofile(p)
    with pytest.raises(ValueError, match="Incorrect image size"):
        oxford_images.read_distortion_lut(p, 6, 8)
    bad = lut.copy()
    bad[5, 1] = np.nan
    np.concatenate([bad[:, 0], bad[:, 1]]).tofile(p)
    with pytest.raises(ValueError, match="non-finite"):
        oxford_images.read_distortion_lut(p, 6, 8)
    with pytest.raises(ValueError, match="Incorrect image size"):
        o.lut_coords(lut, 8, 6 + 1)


def test_grey_png_header_rules():
    g = syn.oxford_mosaic((5, 7), 1)
    grey, rgb = syn.encode_png(g), syn.encode_png(np.stack([g] * 3, -1))
    hd = png.parse_png(grey, grey=True)
    assert (hd.H, hd.W) == (5, 7)
    with pytest.raises(ValueError, match="unsupported colour type 0"):
        png.parse_png(grey)                       # the RGB path keeps rejecting grey
    with pytest.raises(ValueError, match="unsupported colour type 2"):
        png.parse_png(rgb, grey=True)
    pk = png.pack_batch([grey, rgb], grey=True)
    assert pk["out_bytes"] == 35 and list(pk["errors"]) == [1] and pk["desc"][0, png.BPP_SLOT] == 1
    assert (png.pack_batch([rgb])["desc"][:, png.BPP_SLOT] == 0).all()


def test_png_writer_grey_streams_match_pillow():
    import io
    from PIL import Image
    for i in range(int(G["png_n"])):
        assert np.array_equal(np.asarray(Image.open(io.BytesIO(G[f"png_blob_{i}"].tobytes()))), G[f"png_pix_{i}"])


def _tree_digest(*roots):
    h = hashlib.sha256()
    for k, root in enumerate(roots):
        for d, dirs, files in sorted(os.walk(root)):
            dirs.sort()
            for f in sorted(files):
                p = os.path.join(d, f)
                h.update(f"{k}/{os.path.relpath(p, root)}\n".encode())
                with open(p, "rb") as fh:
                    h.update(fh.read())
    return h.hexdigest()


def test_write_oxford_raw_default_unchanged(tmp_path):
    r, l, s = (str(tmp_path / x) for x in ("raw", "lms", "sdk"))
    syn.write_oxford_raw(r, l, s)
    assert _tree_digest(r, l, s) == RAW_DEFAULT_DIGEST


def test_write_oxford_raw_images(tmp_path):
    from PIL import Image
    r, l, s = (str(tmp_path / x) for x in ("raw", "lms", "sdk"))
    syn.write_oxford_raw(r, l, s, seconds=3.0, image_shape=(12, 20))
    q, m, t = (str(tmp_path / x) for x in ("raw0", "lms0", "sdk0"))
    syn.write_oxford_raw(q, m, t, seconds=3.0)
    lut = oxford_images.read_distortion_lut(os.path.join(s, "models", oxford_images.LUT_FILE), 12, 20)
    assert np.array_equal(lut, syn.oxford_distortion_lut(12, 20, 0))
    n = 0
    for tr in os.listdir(q):
        cen = os.path.join(q, tr, "stereo", "centre")
        assert sorted(os.listdir(cen)) == sorted(os.listdir(os.path.join(r, tr, "stereo", "centre")))
        for f in os.listdir(cen):
            img = np.asarray(Image.open(os.path.join(r, tr, "stereo", "centre", f)))
            assert img.shape == (12, 20) and np.array_equal(img, syn.oxford_mosaic((12, 20), int(f[:-4])))
            n += 1
    assert n > 40
