"""GPU PNG decoding (csrc/png.cu through imageprep.decode_png_batch) against OpenCV's decode stored in
tests/golden/png_small.npz: every case in one mixed batch and alone, seeded KITTI-sized frames from the stdlib writer
in batches of 1 and 64, repeatability across runs and streams, every rejected case naming its image, and the decode
feeding assemble_images."""
import hashlib
import os

import numpy as np
import pytest
import torch

from deepi2p_b200 import imageprep, synthetic

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "png_small.npz")


def golden():
    g = np.load(GOLDEN)
    so = np.concatenate([[0], np.cumsum(g["stream_lens"])])
    po = np.concatenate([[0], np.cumsum(g["pixel_lens"])])
    out = []
    for i, name in enumerate(g["names"]):
        h, w = g["shapes"][i]
        px = g["pixels"][po[i]:po[i + 1]].reshape(h, w, 3) if g["pixel_lens"][i] else None
        out.append(dict(name=str(name), blob=g["streams"][so[i]:so[i + 1]].tobytes(), reject=bool(g["reject"][i]),
                        shape=(int(h), int(w)), pixels=px, digest=str(g["digests"][i])))
    return out


CASES = golden()
GOOD = [c for c in CASES if not c["reject"]]
BAD = [c for c in CASES if c["reject"]]
KITTI_HW = ((376, 1241), (375, 1242), (370, 1226))


def images(out):
    data = out["data"].cpu().numpy()
    return [data[o:o + 3 * h * w].reshape(h, w, 3) for o, (h, w) in zip(out["offsets"], out["shapes"])]


def matches(img, case):
    if img.shape[:2] != case["shape"]:
        return False
    if case["pixels"] is not None:
        return np.array_equal(img, case["pixels"])
    return hashlib.sha256(np.ascontiguousarray(img).tobytes()).hexdigest() == case["digest"]


def kitti_frames(n, seed, first=0):
    """Seeded KITTI-shaped frames (smooth gradients plus noise, the three frame sizes in turn) and their PNG streams
    from the stdlib writer, the rows cycling through the five filters."""
    rng = np.random.default_rng(seed)
    imgs, blobs = [], []
    for k in range(first, first + n):
        h, w = KITTI_HW[k % 3]
        yy, xx = np.mgrid[0:h, 0:w]
        img = np.stack([(xx * (3 + k) + yy) % 256, (yy * (2 + k)) % 256, (xx + 7 * yy * k) % 256], -1)
        img = (img + rng.integers(0, 24, img.shape)).clip(0, 255).astype(np.uint8)
        imgs.append(img)
        blobs.append(synthetic.encode_png(img, filters=np.arange(h) % 5, level=1 + k % 9))
    return imgs, blobs


def test_mixed_batch_bit_exact(cuda):
    out = imageprep.decode_png_batch([c["blob"] for c in GOOD])
    assert out["data"].device.type == "cuda" and out["data"].dtype == torch.uint8
    bad = [c["name"] for img, c in zip(images(out), GOOD) if not matches(img, c)]
    assert not bad, bad


@pytest.mark.parametrize("case", GOOD, ids=[c["name"] for c in GOOD])
def test_each_case_alone(cuda, case):
    assert matches(images(imageprep.decode_png_batch([case["blob"]]))[0], case)


@pytest.mark.parametrize("S,first", [(1, 0), (1, 1), (1, 2), (64, 0)])
def test_kitti_sized_frames(cuda, S, first):
    imgs, blobs = kitti_frames(S, 7 + S, first)
    assert {img.shape[:2] for img in imgs} == ({KITTI_HW[first]} if S == 1 else set(KITTI_HW))
    got = images(imageprep.decode_png_batch(blobs))
    assert all(np.array_equal(a, b) for a, b in zip(got, imgs))


def test_repeatable_across_runs_and_streams(cuda):
    _, blobs = kitti_frames(6, 3)
    blobs += [c["blob"] for c in GOOD]
    a = imageprep.decode_png_batch(blobs)["data"].clone()
    b = imageprep.decode_png_batch(blobs)["data"].clone()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        c = imageprep.decode_png_batch(blobs, stream=s)["data"]
    s.synchronize()
    assert torch.equal(a, b) and torch.equal(a, c.to(a.device))


# The reason each rejected fixture case must be reported with: png.parse_png's on the host, png.STATUS's (the
# DIB_PNG_* codes) on the device.
REASONS = {
    "extra_inflated": "more inflated data than the image holds",
    "bad_adler": r"incorrect data check \(Adler-32\)",
    "no_adler": "Adler-32 missing",
    "short_one_byte": "not enough image data",
    "idat_crc": "IDAT: CRC error",
    "ihdr_crc": "IHDR: CRC error",
    "no_iend": "no IEND chunk",
    "filter5": "bad adaptive filter value",
    "truncated": "truncated zlib stream",
    "zlib_cm7": "unknown compression method",
    "zlib_cinfo8": "invalid window size",
    "zlib_fcheck": "incorrect header check",
    "zlib_fdict": "preset dictionary",
    "deflate_btype3": "invalid block type",
    "deflate_stored_nlen": "invalid stored block lengths",
    "deflate_clen_oversub": "invalid code lengths set",
    "deflate_clen_incomplete": "invalid code lengths set",
    "deflate_lit_oversub": "invalid code lengths set",
    "deflate_lit_incomplete": "invalid code lengths set",
    "deflate_no_eob": "missing end-of-block",
    "deflate_repeat_first": "no previous length",
    "deflate_lens_overrun": r"past HLIT \+ HDIST",
    "deflate_hlit287": "too many length or distance symbols",
    "deflate_sym286": "invalid literal/length code",
    "deflate_dist30": "invalid distance code",
    "deflate_dist_before_start": "before the start of the output",
    "dist_beyond_window": "beyond the declared window",
    "dist_beyond_window_same_row": "beyond the declared window",
    "unsupported_rgba": "unsupported colour type 6",
    "unsupported_rgb16": "unsupported colour type 2 with bit depth 16",
    "unsupported_gray": "unsupported colour type 0",
    "unsupported_palette": "unsupported colour type 3",
    "unsupported_adam7": "unsupported interlace method",
}


def test_every_rejected_case_has_a_reason():
    assert sorted(REASONS) == sorted(c["name"] for c in BAD)


@pytest.mark.parametrize("case", BAD, ids=[c["name"] for c in BAD])
def test_rejected_stream_names_the_image(cuda, case):
    good = [c["blob"] for c in GOOD[:3]]
    for pos in (0, 2):
        blobs = good[:pos] + [case["blob"]] + good[pos:]
        with pytest.raises(ValueError, match=f"^image {pos}: .*{REASONS[case['name']]}"):
            imageprep.decode_png_batch(blobs)
    # The first bad image is named, whichever of two is caught on the host and which on the device.
    with pytest.raises(ValueError, match="^image 1: "):
        imageprep.decode_png_batch(good[:1] + [case["blob"], b"not a png"] + good[1:])


def test_empty_batch(cuda):
    out = imageprep.decode_png_batch([])
    assert out["data"].numel() == 0 and out["shapes"].shape == (0, 2)


def test_read_png_batch(cuda, tmp_path):
    imgs, blobs = kitti_frames(2, 1)
    paths = []
    for k, b in enumerate(blobs):
        paths.append(str(tmp_path / f"{k:06d}.png"))
        with open(paths[-1], "wb") as f:
            f.write(b)
    got = images(imageprep.read_png_batch(paths))
    assert all(np.array_equal(a, b) for a, b in zip(got, imgs))


def test_feeds_assemble_images(cuda):
    """decode_png_batch -> assemble_images equals pack_images(the frames) -> assemble_images, bit for bit."""
    imgs, blobs = kitti_frames(3, 9)
    dec = imageprep.decode_png_batch(blobs)
    K = np.tile(np.array([[718.856, 0.0, 607.19], [0.0, 718.856, 185.22], [0.0, 0.0, 1.0]]), (3, 1, 1))
    a = imageprep.assemble_images(dec, K, "val", **imageprep.kitti_image_args())
    b = imageprep.assemble_images(imageprep.pack_images(imgs), K, "val", **imageprep.kitti_image_args())
    assert a["img"].shape == (3, 3, 160, 512)
    assert torch.equal(a["img"], b["img"]) and np.array_equal(a["K64"], b["K64"])


def test_unpadded_data_decodes_through_the_c_abi(cuda):
    """The C ABI needs only 16-byte-aligned starts: an image whose IDAT data ends inside the buffer's last partial
    16-byte vector, with no padding after it, decodes (its Adler-32 trailer is in that vector)."""
    from deepi2p_b200 import _native, png
    from deepi2p_b200._native import _workspace
    lib = _native.load()
    for case in (GOOD[0], next(c for c in GOOD if c["name"] == "zlib_idat_1byte")):
        pk = png.pack_batch([case["blob"]])
        n = int(pk["desc"][0, 1])
        assert n % 16 and pk["desc"][0, 0] == 0
        data = torch.from_numpy(pk["data"][:n].copy()).cuda()
        desc, chunks = np.ascontiguousarray(pk["desc"]), np.ascontiguousarray(pk["chunks"])
        out = torch.empty(pk["out_bytes"], dtype=torch.uint8, device="cuda")
        status = torch.empty((1, 4), dtype=torch.int32, device="cuda")
        sp = torch.cuda.current_stream().cuda_stream
        nws = lib.png_decode_workspace_bytes(desc.ctypes.data, 1, chunks.ctypes.data, len(chunks), n)
        ws = _workspace({}, nws, torch.device("cuda"))
        rc = lib.png_decode_batch_u8(data.data_ptr(), n, desc.ctypes.data, 1, chunks.ctypes.data, len(chunks),
                                     out.data_ptr(), out.numel(), status.data_ptr(), ws.data_ptr(), ws.numel(), sp)
        assert rc == 0
        assert status.cpu().numpy().tolist() == [[0, 0, 0, 0]], case["name"]
        h, w = case["shape"]
        assert matches(out.cpu().numpy().reshape(h, w, 3), case)
