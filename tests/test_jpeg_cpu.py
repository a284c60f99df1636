"""The JPEG decoder's CPU side: oracle_jpeg against Pillow's decode stored in tests/golden/jpeg_small.npz (and against
Pillow itself where it is importable), the fixture against its maker, the host parser's rejections with their
reasons, and the batch packing.  No GPU."""
import hashlib
import io
import os
import struct
import sys

import numpy as np
import pytest

import oracle_jpeg
from deepi2p_b200 import jpeg

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "jpeg_small.npz")


def golden():
    g = np.load(GOLDEN)
    so = np.concatenate([[0], np.cumsum(g["stream_lens"])])
    po = np.concatenate([[0], np.cumsum(g["pixel_lens"])])
    out = []
    for i, name in enumerate(g["names"]):
        px = g["pixels"][po[i]:po[i + 1]]
        h, w = g["shapes"][i]
        out.append(dict(name=str(name), blob=g["streams"][so[i]:so[i + 1]].tobytes(), shape=(int(h), int(w)),
                        digest=str(g["digests"][i]), pixels=px.reshape(h, w, 3) if px.size else None))
    return out


CASES = golden()
SMALL = [c for c in CASES if c["pixels"] is not None]
LARGE = [c for c in CASES if c["pixels"] is None]


def maker():
    pytest.importorskip("cv2")
    pytest.importorskip("PIL")
    sys.path.insert(0, os.path.join(HERE, "golden"))
    try:
        import make_jpeg_golden
    finally:
        sys.path.pop(0)
    return make_jpeg_golden


def test_fixture_covers_the_matrix():
    names = {c["name"] for c in CASES}
    for h, w in [(1, 1), (7, 9), (8, 8), (15, 17), (16, 16), (17, 33)]:
        for q in (1, 50, 75, 95, 100):
            for sf in ("444", "422", "420", "440"):
                assert f"cv2_{h}x{w}_q{q}_{sf}" in names
            assert f"pil_{h}x{w}_q{q}_gray" in names
        for kind in ("rst1", "rst4", "rst2", "optimize", "dqt16", "extras", "exif"):
            assert any(n.endswith(f"{h}x{w}_{kind}") for n in names), (h, w, kind)
    assert {"oxford_960x1280_q95_420", "nuscenes_900x1600_q95_420", "cv2_376x1241_q95_420"} <= names
    assert os.path.getsize(GOLDEN) < 512 << 10


@pytest.mark.parametrize("case", SMALL, ids=[c["name"] for c in SMALL])
def test_oracle_matches_pillow_small(case):
    assert np.array_equal(oracle_jpeg.decode(case["blob"]), case["pixels"])


@pytest.mark.parametrize("case", LARGE, ids=[c["name"] for c in LARGE])
def test_oracle_matches_pillow_large(case):
    img = oracle_jpeg.decode(case["blob"])
    assert img.shape == case["shape"] + (3,)
    assert hashlib.sha256(img.tobytes()).hexdigest() == case["digest"]


def test_fixture_matches_its_maker():
    """The maker regenerates the committed streams and Pillow's pixels and digests."""
    ref = maker().build()
    g = np.load(GOLDEN)
    for k in ref:
        assert np.array_equal(ref[k], g[k]), k


def test_oracle_matches_installed_pillow():
    pil = pytest.importorskip("PIL.Image")
    for c in CASES[::7]:
        assert np.array_equal(oracle_jpeg.decode(c["blob"]), np.asarray(pil.open(io.BytesIO(c["blob"])).convert("RGB")))


def test_oracle_stages():
    c = next(c for c in CASES if c["name"] == "cv2_17x33_q75_420")
    st = oracle_jpeg.decode(c["blob"], stages=True)
    assert [a.shape for a in st["coef"]] == [(4, 6, 64), (2, 3, 64), (2, 3, 64)]
    assert [p.shape for p in st["planes"]] == [(32, 48), (16, 24), (16, 24)]
    assert np.array_equal(st["rgb"], c["pixels"])


# --- rejections -------------------------------------------------------------------------------------------------


def _pil(arr, **kw):
    Image = pytest.importorskip("PIL.Image")
    bio = io.BytesIO()
    Image.fromarray(arr).save(bio, "JPEG", **kw)
    return bio.getvalue()


def _rgb(h=24, w=40):
    rng = np.random.default_rng(3)
    return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)


def _set_sof(blob, code):
    b = bytearray(blob)
    i = b.index(b"\xff\xc0")
    b[i + 1] = code
    return bytes(b)


def _adobe(blob, transform):
    """Replace the JFIF APP0 with an Adobe APP14 segment of the given transform."""
    assert blob[2:4] == b"\xff\xe0"
    L = struct.unpack(">H", blob[4:6])[0]
    app14 = b"\xff\xee" + struct.pack(">H", 14) + b"Adobe" + b"\x00\x64\x00\x00\x00\x00" + bytes([transform])
    return blob[:2] + app14 + blob[4 + L:]


def test_rejects_progressive():
    with pytest.raises(ValueError, match="progressive"):
        jpeg.parse_jpeg(_pil(_rgb(), progressive=True))


def test_rejects_arithmetic_sof9():
    with pytest.raises(ValueError, match="arithmetic-coded sequential"):
        jpeg.parse_jpeg(_set_sof(_pil(_rgb()), 0xC9))


def test_rejects_lossless_and_12_bit():
    with pytest.raises(ValueError, match="lossless"):
        jpeg.parse_jpeg(_set_sof(_pil(_rgb()), 0xC3))
    b = bytearray(_pil(_rgb()))
    b[b.index(b"\xff\xc0") + 4] = 12
    with pytest.raises(ValueError, match="12-bit"):
        jpeg.parse_jpeg(bytes(b))


def test_rejects_cmyk():
    Image = pytest.importorskip("PIL.Image")
    bio = io.BytesIO()
    Image.fromarray(_rgb()).convert("CMYK").save(bio, "JPEG")
    with pytest.raises(ValueError, match="CMYK"):
        jpeg.parse_jpeg(bio.getvalue())


def test_rejects_411():
    cv2 = pytest.importorskip("cv2")
    ok, enc = cv2.imencode(".jpg", _rgb(), [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411])
    with pytest.raises(ValueError, match="sampling factors"):
        jpeg.parse_jpeg(enc.tobytes())


def test_rejects_adobe_rgb_and_keeps_adobe_ycc():
    blob = _pil(_rgb(), quality=90)
    with pytest.raises(ValueError, match="RGB-coded"):
        jpeg.parse_jpeg(_adobe(blob, 0))
    assert jpeg.parse_jpeg(_adobe(blob, 1)).ncomp == 3


def test_rejects_multi_scan():
    b = _pil(_rgb())
    i = b.index(b"\xff\xda")
    L = struct.unpack(">H", b[i + 2:i + 4])[0]
    first_scan = b"\xff\xda\x00\x08\x01\x01\x00\x00\x3f\x00"     # a first scan of component 1 alone
    with pytest.raises(ValueError, match="multi-scan"):
        jpeg.parse_jpeg(b[:i] + first_scan + b[i + 2 + L:])


def test_rejects_truncated():
    blob = _pil(_rgb())
    with pytest.raises(ValueError, match="truncated"):
        jpeg.parse_jpeg(blob[:100])
    with pytest.raises(ValueError, match="truncated"):
        oracle_jpeg.decode(blob[:len(blob) // 2])
    with pytest.raises(ValueError, match="MCU count|truncated|Huffman"):
        oracle_jpeg.decode(blob[:len(blob) // 2] + b"\xff\xd9")


def test_rejects_not_a_jpeg():
    with pytest.raises(ValueError, match="no SOI"):
        jpeg.parse_jpeg(b"\x89PNG\r\n\x1a\n" + bytes(40))


def test_pack_batch_names_the_image():
    good = CASES[0]["blob"]
    with pytest.raises(ValueError, match=r"^image 2: progressive"):
        jpeg.pack_batch([good, good, _set_sof(good, 0xC2)])


def test_pack_batch_layout():
    sel = [c for c in CASES if c["name"] in ("cv2_17x33_q75_420", "pil_16x16_q50_gray", "cv2_7x9_q95_440")]
    pk = jpeg.pack_batch([c["blob"] for c in sel])
    assert pk["shapes"].tolist() == [list(c["shape"]) for c in sel]
    sizes = 3 * pk["shapes"][:, 0] * pk["shapes"][:, 1]
    assert pk["offsets"].tolist() == [0, int(sizes[0]), int(sizes[0] + sizes[1])]
    assert pk["out_bytes"] == int(sizes.sum())
    d = pk["desc"]
    for s, c in enumerate(sel):
        hd = jpeg.parse_jpeg(c["blob"])
        assert d[s, 1] == len(c["blob"]) - hd.scan
        assert bytes(pk["data"][d[s, 0]:d[s, 0] + d[s, 1]]) == c["blob"][hd.scan:]
    assert pk["huff"].shape == (3, 6, jpeg.HUFF_WORDS) and pk["quant"].shape == (3, 3, 64)


def test_device_huff_table_decodes_every_code():
    """The 9-bit lookahead plus the per-length maxcode / valoff walk finds each code's symbol."""
    hd = jpeg.parse_jpeg(next(c for c in CASES if c["name"] == "pil_17x33_optimize")["blob"])
    for table in (hd.comps[0]["dc"], hd.comps[0]["ac"], hd.comps[1]["ac"]):
        t = jpeg.device_huff_table(*table)
        lut = t[:256].view(np.uint16)
        maxcode, valoff, vals = t[256:274], t[274:292], t[292:].view(np.uint8)
        for length, code, sym in jpeg.huff_codes(*table):
            p16 = code << (16 - length)
            e = int(lut[p16 >> 7])
            if e:
                got = (e >> 8, e & 255)
            else:
                got = next((l, int(vals[(p16 >> (16 - l)) + valoff[l]])) for l in range(10, 17)
                           if (p16 >> (16 - l)) <= maxcode[l])
            assert got == (length, sym)
