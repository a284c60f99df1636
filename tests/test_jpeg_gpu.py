"""GPU JPEG decoding (csrc/jpeg.cu through imageprep.decode_jpeg_batch) against Pillow's decode stored in
tests/golden/jpeg_small.npz: every case in one mixed batch and alone, the full-size frames in batches of 1 and 64,
forced synchronisation over small windows, repeatability across runs and streams, corrupt streams, and the decode
feeding assemble_images."""
import hashlib
import os

import numpy as np
import pytest
import torch

from deepi2p_b200 import imageprep

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_small.npz")


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
FULL = [c for c in CASES if c["name"].startswith(("oxford", "nuscenes"))]


def images(out):
    data = out["data"].cpu().numpy()
    return [data[o:o + 3 * h * w].reshape(h, w, 3) for o, (h, w) in zip(out["offsets"], out["shapes"])]


def matches(img, case):
    if img.shape != case["shape"] + (3,):
        return False
    if case["pixels"] is not None:
        return np.array_equal(img, case["pixels"])
    return hashlib.sha256(np.ascontiguousarray(img).tobytes()).hexdigest() == case["digest"]


def test_mixed_batch_bit_exact(cuda):
    out = imageprep.decode_jpeg_batch([c["blob"] for c in CASES])
    bad = [c["name"] for img, c in zip(images(out), CASES) if not matches(img, c)]
    assert not bad, bad


def test_each_case_alone(cuda):
    bad = [c["name"] for c in CASES if not matches(images(imageprep.decode_jpeg_batch([c["blob"]]))[0], c)]
    assert not bad, bad


@pytest.mark.parametrize("window_bits", [32, 33, 64, 301, 4096])
def test_small_windows_synchronise(cuda, window_bits):
    """Windows of a few symbols: the no-restart path must synchronise across many windows (the full-size frame only
    from 64 bits on, to keep the run short)."""
    sel = [c for c in CASES if "rst" not in c["name"]][::3] + (FULL[:1] if window_bits >= 64 else [])
    out = imageprep.decode_jpeg_batch([c["blob"] for c in sel], _window_bits=window_bits)
    bad = [c["name"] for img, c in zip(images(out), sel) if not matches(img, c)]
    assert not bad, bad
    assert imageprep.decode_jpeg_batch.last_rounds.max() >= 1


@pytest.mark.parametrize("S", [1, 64])
def test_full_size_frames(cuda, S):
    for case in FULL:
        out = imageprep.decode_jpeg_batch([case["blob"]] * S)
        assert all(matches(img, case) for img in images(out)), case["name"]


def test_repeatable_across_runs_and_streams(cuda):
    blobs = [c["blob"] for c in CASES[::5]] + [f["blob"] for f in FULL]
    ref = imageprep.decode_jpeg_batch(blobs)["data"].clone()
    again = imageprep.decode_jpeg_batch(blobs)["data"]
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        other = imageprep.decode_jpeg_batch(blobs, stream=side)["data"]
    side.synchronize()
    assert torch.equal(ref, again) and torch.equal(ref, other)


def corrupt_cases():
    ox = FULL[0]["blob"]
    small = next(c["blob"] for c in CASES if c["name"] == "cv2_17x33_q75_420")
    rst = next(c["blob"] for c in CASES if c["name"] == "pil_17x33_rst1")
    sos = ox.index(b"\xff\xda")
    cut = ox[:len(ox) // 2]                                  # truncated: no EOI
    early_eoi = ox[:len(ox) // 2] + b"\xff\xd9"              # EOI before the last MCU
    garbage = bytearray(ox)
    garbage[sos + 2000:sos + 2064] = b"\xff\x00" * 32        # runs of ones: no Huffman code is all ones
    r = rst.index(b"\xff\xd3", rst.index(b"\xff\xda"))
    no_rst = rst[:r] + rst[r + 2:]                           # a restart marker removed
    second_scan = small[:-2] + b"\xff\xda\x00\x08\x01\x01\x00\x00\x3f\x00" + b"\x00" * 4 + b"\xff\xd9"
    return [("truncated", cut), ("early EOI", early_eoi), ("bad code", bytes(garbage)), ("restarts", no_rst),
            ("second scan", second_scan)]


@pytest.mark.parametrize("kind,blob", corrupt_cases(), ids=[k for k, _ in corrupt_cases()])
def test_corrupt_stream_names_the_image(cuda, kind, blob):
    good = [c["blob"] for c in CASES[:3]]
    with pytest.raises(ValueError, match=r"^image 3: "):
        imageprep.decode_jpeg_batch(good + [blob] + good)
    # the other images still decode on their own
    out = imageprep.decode_jpeg_batch(good)
    assert all(matches(img, c) for img, c in zip(images(out), CASES[:3]))


def test_unsupported_stream_names_the_image(cuda):
    with pytest.raises(ValueError, match=r"^image 1: progressive"):
        blob = bytearray(CASES[0]["blob"])
        i = blob.index(b"\xff\xc0")
        blob[i + 1] = 0xC2
        imageprep.decode_jpeg_batch([CASES[0]["blob"], bytes(blob)])


def test_empty_batch(cuda):
    out = imageprep.decode_jpeg_batch([])
    ref = imageprep.pack_images([])
    assert out["data"].numel() == 0 and out["offsets"].shape == (0,) and out["shapes"].shape == (0, 2)
    assert ref["data"].numel() == 0


def test_feeds_assemble_images(cuda):
    """decode_jpeg_batch -> assemble_images equals pack_images(Pillow's frames) -> assemble_images, bit for bit."""
    frames = [FULL[0]] * 3
    dec = imageprep.decode_jpeg_batch([f["blob"] for f in frames])
    host = [img.copy() for img in images(dec)]
    assert all(matches(img, f) for img, f in zip(host, frames))
    K = np.array([[983.0, 0.0, 640.0], [0.0, 983.0, 480.0], [0.0, 0.0, 1.0]])
    a = imageprep.assemble_images(dec, K, "val", **imageprep.oxford_image_args())
    b = imageprep.assemble_images(imageprep.pack_images(host), K, "val", **imageprep.oxford_image_args())
    assert a["img"].shape == (3, 3, 384, 640)
    assert torch.equal(a["img"], b["img"]) and np.array_equal(a["K64"], b["K64"])
