"""CPU checks of the PNG decoder's host side: the oracle (oracle_png) against OpenCV's decisions and pixels in
tests/golden/png_small.npz, png.py's header checks and packing, and the stdlib writer the GPU tests and the benchmark
draw their frames from."""
import hashlib
import os
import struct
import zlib

import numpy as np
import pytest

import oracle_png
from deepi2p_b200 import png, synthetic

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "png_small.npz")


def golden():
    g = np.load(GOLDEN)
    so = np.concatenate([[0], np.cumsum(g["stream_lens"])])
    po = np.concatenate([[0], np.cumsum(g["pixel_lens"])])
    out = []
    for i, name in enumerate(g["names"]):
        h, w = g["shapes"][i]
        px = g["pixels"][po[i]:po[i + 1]].reshape(h, w, 3) if g["pixel_lens"][i] else None
        out.append(dict(name=str(name), blob=g["streams"][so[i]:so[i + 1]].tobytes(), cv2_ok=bool(g["cv2_ok"][i]),
                        reject=bool(g["reject"][i]), shape=(int(h), int(w)), pixels=px, digest=str(g["digests"][i])))
    return out


CASES = golden()


def test_fixture_covers_the_cases():
    names = {c["name"] for c in CASES}
    for n in ("cv2_c0", "cv2_c9", "cv2_strategy_rle", "cv2_strategy_fixed", "cv2_strategy_huffman_only",
              "pil_optimize", "zlib_wbits8", "zlib_wbits15", "zlib_full_flush", "zlib_level0", "zlib_idat_1byte",
              "zlib_idat_empty", "zlib_paeth_ties", "size_1x1", "kitti_376x1241", "kitti_375x1242", "kitti_370x1226",
              "bad_adler", "no_adler", "short_one_byte", "idat_crc", "ihdr_crc", "no_iend", "filter5",
              "deflate_lit_incomplete", "deflate_single_code", "dist_beyond_window", "zlib_fdict"):
        assert n in names
    assert os.path.getsize(GOLDEN) < 500_000


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_oracle_follows_opencv(case):
    """Never accept what OpenCV rejects; on what both accept, OpenCV's pixels exactly."""
    try:
        img = oracle_png.decode(case["blob"])
    except ValueError:
        assert case["reject"], f"{case['name']}: the oracle rejects a stream OpenCV accepts"
        return
    assert case["cv2_ok"] and not case["reject"], case["name"]
    assert img.shape[:2] == case["shape"]
    assert hashlib.sha256(np.ascontiguousarray(img).tobytes()).hexdigest() == case["digest"]
    if case["pixels"] is not None:
        assert np.array_equal(img, case["pixels"])


def _stream(ihdr=None, chunks=(), idat=None):
    img = np.zeros((5, 7, 3), np.uint8)
    z = zlib.compress(synthetic.png_filter(img, 0)) if idat is None else idat
    ih = ihdr if ihdr is not None else struct.pack(">IIBBBBB", 7, 5, 8, 2, 0, 0, 0)
    return (png.SIGNATURE + synthetic.png_chunk(b"IHDR", ih) + b"".join(chunks) + synthetic.png_chunk(b"IDAT", z) +
            synthetic.png_chunk(b"IEND", b""))


@pytest.mark.parametrize("ctype,depth,interlace,reason", [
    (6, 8, 0, "unsupported colour type 6"), (2, 16, 0, "unsupported colour type 2 with bit depth 16"),
    (0, 8, 0, "unsupported colour type 0"), (3, 8, 0, "unsupported colour type 3"), (4, 8, 0, "unsupported"),
    (2, 8, 1, "unsupported interlace"), (2, 4, 0, "invalid colour type 2 with bit depth 4"),
    (7, 8, 0, "invalid colour type 7")])
def test_parse_rejects_unsupported_headers(ctype, depth, interlace, reason):
    with pytest.raises(ValueError, match=reason):
        png.parse_png(_stream(struct.pack(">IIBBBBB", 7, 5, depth, ctype, 0, 0, interlace)))


def test_parse_rejects_bad_structure():
    good = _stream()
    assert png.parse_png(good).W == 7
    with pytest.raises(ValueError, match="bad signature"):
        png.parse_png(b"\x89PNG\r\n\x1a\x0b" + good[8:])
    with pytest.raises(ValueError, match="incomplete"):
        png.parse_png(good[:-12])
    with pytest.raises(ValueError, match="IHDR: CRC error"):
        png.parse_png(good[:29] + bytes([good[29] ^ 1]) + good[30:])
    with pytest.raises(ValueError, match="size 0 x 5"):
        png.parse_png(_stream(struct.pack(">IIBBBBB", 0, 5, 8, 2, 0, 0, 0)))
    with pytest.raises(ValueError, match="exceeds OpenCV's limits"):
        png.parse_png(_stream(struct.pack(">IIBBBBB", (1 << 20) + 1, 1, 8, 2, 0, 0, 0)))
    with pytest.raises(ValueError, match="unknown critical chunk"):
        png.parse_png(_stream(chunks=[synthetic.png_chunk(b"ABCD", b"x")]))
    split = good.index(b"IEND") - 4
    text = synthetic.png_chunk(b"tEXt", b"a\0b")
    two = _stream(idat=b"")[:split - 12] + synthetic.png_chunk(b"IDAT", zlib.compress(b"\0" * 110)) + text + \
        synthetic.png_chunk(b"IDAT", b"") + synthetic.png_chunk(b"IEND", b"")
    with pytest.raises(ValueError, match="not consecutive"):
        png.parse_png(two)
    with pytest.raises(ValueError, match="incorrect header check"):
        png.parse_png(_stream(idat=b"\x78\x02" + zlib.compress(b"")[2:]))
    with pytest.raises(ValueError, match="truncated zlib header"):
        png.parse_png(_stream(idat=b"\x78"))
    # An ancillary chunk with a bad CRC is skipped, as libpng does.
    bad_text = text[:-1] + bytes([text[-1] ^ 1])
    assert png.parse_png(_stream(chunks=[bad_text])).H == 5


def test_pack_batch_layout():
    a = synthetic.encode_png(np.arange(5 * 7 * 3, dtype=np.uint8).reshape(5, 7, 3), idat=[3, 0, 4])
    b = b"not a png"
    c = synthetic.encode_png(np.zeros((2, 3, 3), np.uint8))
    pk = png.pack_batch([a, b, c])
    assert pk["errors"] == {1: "not a PNG stream (bad signature)"}
    assert pk["desc"][1, 7] == 1 and pk["shapes"][1].tolist() == [0, 0]
    assert pk["offsets"].tolist() == [0, 105, 105] and pk["out_bytes"] == 105 + 18
    d0, d2 = pk["desc"][0], pk["desc"][2]
    assert d0[0] % png.ALIGN == 0 and d2[0] % png.ALIGN == 0 and d2[0] >= d0[0] + d0[1] + png.ALIGN
    ch = pk["chunks"]
    assert ch[:, 0].tolist() == [0, 0, 0, 0, 2] and ch[:4, 2].sum() == d0[1] and d0[9] == 4 and d2[5] == 4
    hd = png.parse_png(a)
    z = b"".join(a[o:o + n] for o, n, _ in hd.idat)
    assert pk["data"][d0[0]:d0[0] + d0[1]].tobytes() == z
    assert [int(x) for x in ch[:4, 3]] == [zlib.crc32(b"IDAT" + a[o:o + n]) for o, n, _ in hd.idat]
    assert d0[6] == 15


@pytest.mark.parametrize("shape,filters", [((1, 1), 0), ((6, 11), 4), ((9, 5), [0, 1, 2, 3, 4, 4, 3, 2, 1])])
def test_writer_round_trips_through_the_oracle(shape, filters):
    img = np.random.default_rng(shape[1]).integers(0, 256, shape + (3,), dtype=np.uint8)
    assert np.array_equal(oracle_png.decode(synthetic.encode_png(img, filters=filters, idat=7)), img)


def test_writer_streams_decode_in_opencv():
    cv2 = pytest.importorskip("cv2")
    for wbits, level in ((9, 1), (15, 9)):
        img = np.random.default_rng(wbits).integers(0, 256, (37, 53, 3), dtype=np.uint8)
        s = synthetic.encode_png(img, filters=np.arange(37) % 5, level=level, wbits=wbits)
        out = cv2.imdecode(np.frombuffer(s, np.uint8), cv2.IMREAD_COLOR)
        assert np.array_equal(out[:, :, ::-1], img)


def test_kitti_image_folder_choice(tmp_path):
    from deepi2p_b200 import kitti
    root = str(tmp_path)
    with pytest.raises(FileNotFoundError, match="neither .*data_odometry_color_npy.*image_2 nor "
                                                ".*data_odometry_color/sequences/04/image_2"):
        kitti.image_dir(root, 4, "P2")
    png_dir = tmp_path / "data_odometry_color" / "sequences" / "04" / "image_2"
    png_dir.mkdir(parents=True)
    (png_dir / "000000.png").write_bytes(b"")
    assert kitti.image_path(root, 4, "P2", 3) == str(png_dir / "000003.png")
    assert kitti.sequence_length(root, 4) == 1
    npy_dir = tmp_path / "data_odometry_color_npy" / "sequences" / "04" / "image_2"
    npy_dir.mkdir(parents=True)
    assert kitti.image_path(root, 4, "P2", 3) == str(npy_dir / "000003.npy")


def _adler_by_threads(data, threads):
    """csrc/png.cu's Adler-32: thread t sums the bytes i = t, t + threads, ... as a = sum d_i and b = sum (n - i) d_i,
    exact in 64 bits, reduces both mod 65521, and the block adds the residues."""
    d = np.frombuffer(data, np.uint8).astype(np.uint64)
    n = d.size
    w = (n - np.arange(n, dtype=np.uint64)) * d
    s1 = s2 = 0
    for t in range(threads):
        a, b = int(d[t::threads].sum()), int(w[t::threads].sum())
        assert b < 1 << 64
        s1, s2 = s1 + a % 65521, s2 + b % 65521
    return (((n + s2) % 65521) << 16) | ((1 + s1) % 65521)


@pytest.mark.parametrize("n", [1, 767, 769, 200_003])
def test_adler_decomposition_equals_zlib(n):
    data = np.random.default_rng(n).integers(0, 256, n, dtype=np.uint8).tobytes()
    assert _adler_by_threads(data, 768) == zlib.adler32(data)
    assert _adler_by_threads(b"\xff" * n, 768) == zlib.adler32(b"\xff" * n)


def test_adler_partial_sums_fit_at_the_largest_image():
    """At OpenCV's largest image (2^30 pixels, 2^20 per side) one thread's position-weighted sum of all-0xFF bytes,
    the largest it can be, stays below 2^64, so the kernel's per-thread sums are exact."""
    n = 3 * (1 << 30) + (1 << 20)                      # h (1 + 3 w) at w h = 2^30, h = 2^20
    per = -(-n // 768)
    worst = sum(255 * (n - i) for i in range(0, per * 768, 768))   # thread 0 holds the largest weights
    assert worst < 1 << 62
    assert 255 * per * n < 1 << 62
