"""Write tests/golden/jpeg_small.npz: JPEG streams encoded by Pillow and cv2 (libjpeg-turbo) from seeded textured
frames, with Pillow's decode np.asarray(Image.open(BytesIO(b)).convert("RGB")) -- the pixels for the small cases,
a SHA-256 digest for the large ones.  The large frames are smooth apart from their edges and one noise band, so the
file stays under 512 KB.  Needs cv2 and Pillow; the tests only read the file.

    python tests/golden/make_jpeg_golden.py
"""
import hashlib
import io
import os
import struct

import cv2
import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "jpeg_small.npz")
SMALL = [(1, 1), (7, 9), (8, 8), (15, 17), (16, 16), (17, 33)]
QUALITIES = (1, 50, 75, 95, 100)
CV2_SAMPLING = (("444", cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444), ("422", cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422),
                ("420", cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420), ("440", cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440))
PIXELS_UP_TO = 64 * 64            # larger cases store a digest of the pixels instead


def frame(h, w, seed):
    """Gradients, a checkerboard of edges, a saturated white block, a zeroed channel and Gaussian noise."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    img = np.zeros((h, w, 3), np.float64)
    img[..., 0] = 255 * x / max(w - 1, 1)
    img[..., 1] = 255 * y / max(h - 1, 1)
    img[..., 2] = np.where((x // 7 + y // 5) % 2, 250, 5)
    img += rng.normal(0, 30.0, img.shape)
    img[:h // 4, :w // 4] = 255
    img[h // 2:, w // 2:, 0] = 0
    return np.clip(img, 0, 255).astype(np.uint8)


def large_frame(h, w, seed):
    """A full-size frame that stays small once encoded: slow colour waves, large saturated edges and blocks, and one
    16-row band of Gaussian noise, so the entropy-coded data still mixes long and short codes."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    img = np.zeros((h, w, 3), np.float64)
    img[..., 0] = 128 + 60 * np.sin(x / 800.0 + y / 1100.0)
    img[..., 1] = 128 + 60 * np.cos(y / 700.0 - x / 1300.0)
    img[..., 2] = np.where((x // 160 + y // 96) % 2, 240, 20)
    img[:h // 5, :w // 5] = 255
    img[h // 2:, w // 2:, 0] = 0
    r0 = int(h * 0.45)
    img[r0:r0 + 16] += rng.normal(0, 30, (16, w, 3))
    return np.clip(img, 0, 255).astype(np.uint8)


def cv2_jpeg(rgb, *params):
    ok, enc = cv2.imencode(".jpg", np.ascontiguousarray(rgb[..., ::-1]), list(params))
    assert ok
    return enc.tobytes()


def pil_jpeg(arr, **kw):
    bio = io.BytesIO()
    Image.fromarray(arr).save(bio, "JPEG", **kw)
    return bio.getvalue()


def segments(b):
    """(marker, start, end) of each header segment up to SOS."""
    out, i = [], 2
    while True:
        m = b[i + 1]
        L = struct.unpack(">H", b[i + 2:i + 4])[0]
        out.append((m, i, i + 2 + L))
        if m == 0xDA:
            return out
        i += 2 + L


def dqt16(b):
    """Rewrite every 8-bit DQT table as a 16-bit one with the same values."""
    out, last = bytearray(), 0
    for m, s, e in segments(b):
        if m != 0xDB:
            continue
        out += b[last:s]
        seg, p, body = b[s + 4:e], 0, bytearray()
        while p < len(seg):
            pq, tq = seg[p] >> 4, seg[p] & 15
            assert pq == 0
            body.append(0x10 | tq)
            body += np.frombuffer(seg[p + 1:p + 65], np.uint8).astype(">u2").tobytes()
            p += 65
        out += b"\xff\xdb" + struct.pack(">H", len(body) + 2) + body
        last = e
    return bytes(out + b[last:])


def with_extras(b):
    """COM and APP segments after SOI, fill bytes before DQT and SOS, trailing bytes after EOI."""
    com = b"\xff\xfe" + struct.pack(">H", 2 + 13) + b"a comment 123"
    app = b"\xff\xe5" + struct.pack(">H", 2 + 6) + b"APP5!!"
    out = bytearray(b[:2] + com + app)
    last = 2
    for m, s, e in segments(b):
        if m in (0xDB, 0xDA):
            out += b[last:s] + b"\xff\xff\xff"
            last = s
    out += b[last:]
    return bytes(out) + b"\x00\x11trailing junk\xff\xd9\x00"


def exif_jpeg(rgb):
    im = Image.fromarray(rgb)
    ex = Image.Exif()
    ex[0x0112] = 6                           # orientation: Pillow's Image.open does not apply it
    ex[0x010F] = "synthetic"
    bio = io.BytesIO()
    im.save(bio, "JPEG", quality=90, exif=ex.tobytes())
    return bio.getvalue()


def cases():
    """[(name, stream)] of the fixture, in order."""
    out = []
    for h, w in SMALL + [(376, 1241)]:
        big = h >= 100
        rgb = large_frame(h, w, 1000 + 31 * h + w) if big else frame(h, w, 1000 + 31 * h + w)
        for q in (50, 95) if big else QUALITIES:
            for name, sf in CV2_SAMPLING:
                if big and q == 95 and name != "420":
                    continue
                out.append((f"cv2_{h}x{w}_q{q}_{name}", cv2_jpeg(rgb, cv2.IMWRITE_JPEG_QUALITY, q,
                                                                    cv2.IMWRITE_JPEG_SAMPLING_FACTOR, sf)))
            if not big or q == 95:
                out.append((f"pil_{h}x{w}_q{q}_gray", pil_jpeg(rgb[..., 1], quality=q)))
            if h < 100:
                out.append((f"pil_{h}x{w}_q{q}_420", pil_jpeg(rgb, quality=q, subsampling=2)))
        if h < 100:
            for rb in (1, 4):
                out.append((f"pil_{h}x{w}_rst{rb}", pil_jpeg(rgb, quality=90, restart_marker_blocks=rb)))
            out.append((f"cv2_{h}x{w}_rst2", cv2_jpeg(rgb, cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_RST_INTERVAL,
                                                      2)))
            out.append((f"pil_{h}x{w}_optimize", pil_jpeg(rgb, quality=85, optimize=True, subsampling=1)))
            out.append((f"pil_{h}x{w}_dqt16", dqt16(pil_jpeg(rgb, quality=80))))
            out.append((f"pil_{h}x{w}_extras", with_extras(pil_jpeg(rgb, quality=80))))
            out.append((f"pil_{h}x{w}_exif", exif_jpeg(rgb)))
    sat = np.zeros((40, 56, 3), np.uint8)           # saturated primaries and hard edges at quality 100
    sat[:, ::2] = 255
    sat[::3, :, 1] = 255
    sat[20:, :28] = [255, 0, 0]
    out.append(("cv2_saturated_q100_444", cv2_jpeg(sat, cv2.IMWRITE_JPEG_QUALITY, 100,
                                                   cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444)))
    out.append(("cv2_saturated_q100_420", cv2_jpeg(sat, cv2.IMWRITE_JPEG_QUALITY, 100)))
    out.append(("cv2_376x1241_rst8", cv2_jpeg(large_frame(376, 1241, 7), cv2.IMWRITE_JPEG_QUALITY, 90,
                                              cv2.IMWRITE_JPEG_RST_INTERVAL, 8)))
    out.extend(full_size())
    return out


def full_size():
    """The two loaders' frame shapes as the Oxford build script writes them (cv2.imwrite defaults: q95, 4:2:0, no
    restart markers)."""
    return [("oxford_960x1280_q95_420", cv2_jpeg(large_frame(960, 1280, 11), cv2.IMWRITE_JPEG_QUALITY, 95)),
            ("nuscenes_900x1600_q95_420", cv2_jpeg(large_frame(900, 1600, 12), cv2.IMWRITE_JPEG_QUALITY, 95))]


def pillow_decode(b):
    return np.asarray(Image.open(io.BytesIO(b)).convert("RGB"))


def build():
    names, streams, shapes, digests, pix = [], [], [], [], []
    for name, b in cases():
        px = pillow_decode(b)
        names.append(name)
        streams.append(np.frombuffer(b, np.uint8))
        shapes.append(px.shape[:2])
        digests.append(hashlib.sha256(np.ascontiguousarray(px).tobytes()).hexdigest())
        pix.append(px.reshape(-1) if px.shape[0] * px.shape[1] <= PIXELS_UP_TO else np.zeros(0, np.uint8))
    lens = np.array([len(s) for s in streams], np.int64)
    plens = np.array([len(p) for p in pix], np.int64)
    return dict(names=np.array(names), streams=np.concatenate(streams), stream_lens=lens,
                shapes=np.array(shapes, np.int64), digests=np.array(digests), pixels=np.concatenate(pix),
                pixel_lens=plens)


if __name__ == "__main__":
    np.savez_compressed(OUT, **build())
    print(OUT, os.path.getsize(OUT))
