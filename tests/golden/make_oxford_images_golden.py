"""Make tests/golden/oxford_images_small.npz: the Oxford stereo-centre image conversion and the JPEG encoder's
expected outputs, from the RobotCar SDK's pipeline restated over scipy (oracle_oxford_images.sdk_load_image), OpenCV
4.13's cv2.imencode and Pillow.  Needs cv2, scipy and Pillow; run from the repository root:

    python tests/golden/make_oxford_images_golden.py

Contents (i indexes each group):
  dm_mosaic_i, dm_lut_i, dm_rgb_i     grey mosaic, LUT (x, y) and the SDK pipeline's uint8 RGB
  full_seeds, full_rgb_sha_i          two 1280 x 960 frames (synthetic.oxford_mosaic / oxford_distortion_lut by seed)
                                      and the sha256 of their RGB
  enc_spec_i, enc_shape_i, enc_q_i    an encoder case: the image (oracle_oxford_images.fixture_image, 'dm:<j>' for
                                      dm_rgb_j, 'full:<k>' for full frame k), its (h, w) and the quality
  enc_jpg_i / enc_sha_i               cv2.imencode(".jpg", rgb[:, :, ::-1]) bytes, or their sha256 for large images
  enc_pil_i / enc_pilsha_i            np.asarray(Image.open(stream).convert("RGB")), or its sha256
  png_blob_i, png_pix_i               grey PNG streams (PIL, cv2, and each of the five filter types) and Pillow's pixels
"""
import hashlib
import io
import os
import sys

import cv2
import numpy as np
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import oracle_oxford_images as o  # noqa: E402
from deepi2p_b200 import synthetic  # noqa: E402

FULL = (960, 1280)
FULL_SEEDS = (11, 12)


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes() if isinstance(a, np.ndarray) else a).hexdigest()


def full_frame(k):
    seed = FULL_SEEDS[k]
    mosaic = synthetic.oxford_mosaic(FULL, seed)
    return mosaic, synthetic.oxford_distortion_lut(*FULL, seed)


def main():
    out = {}
    rng = np.random.default_rng(20261017)
    dm = []
    for (h, w), kind in [((8, 8), "identity"), ((7, 5), "radial"), ((17, 33), "special"), ((48, 64), "radial"),
                         ((24, 40), "radial"), ((6, 10), "random"), ((2, 2), "special"), ((33, 18), "special")]:
        if len(dm) % 2:
            mosaic = rng.integers(0, 256, (h, w), dtype=np.uint8)
        else:
            mosaic = synthetic.oxford_mosaic((h, w), len(dm))
        if kind == "identity":
            lut = o.identity_lut(h, w)
        elif kind == "radial":
            lut = synthetic.oxford_distortion_lut(h, w, len(dm))
        elif kind == "special":
            lut = o.special_lut(h, w)
        else:
            lut = np.stack([rng.uniform(-2, w + 1, h * w), rng.uniform(-2, h + 1, h * w)], 1)
        rgb = o.sdk_load_image(mosaic, lut)
        out[f"dm_mosaic_{len(dm)}"], out[f"dm_lut_{len(dm)}"], out[f"dm_rgb_{len(dm)}"] = mosaic, lut, rgb
        dm.append(rgb)
    full = []
    for k in range(len(FULL_SEEDS)):
        rgb = o.sdk_load_image(*full_frame(k))
        out[f"full_rgb_sha_{k}"] = np.array(sha(rgb))
        full.append(rgb)
    out["full_seeds"] = np.array(FULL_SEEDS)

    cases = []
    for q in (1, 50, 95, 100):
        for (h, w) in [(1, 1), (7, 5), (17, 33), (8, 16), (16, 8), (31, 47)]:
            for spec in ("rand:1", "sat:2", "flat:255", "grad"):
                cases.append((spec, h, w, q))
    for j, rgb in enumerate(dm):
        cases.append((f"dm:{j}", *rgb.shape[:2], 95))
    for spec in ("rand:3", "sat:4", "grad"):
        cases.append((spec, 961, 1281, 95))
    cases.append(("flat:0", 961, 1281, 50))
    for k in range(len(full)):
        cases.append((f"full:{k}", *FULL, 95))
    for i, (spec, h, w, q) in enumerate(cases):
        if spec.startswith("dm:"):
            rgb = dm[int(spec[3:])]
        elif spec.startswith("full:"):
            rgb = full[int(spec[5:])]
        else:
            rgb = o.fixture_image(spec, h, w)
        jpg = cv2.imencode(".jpg", np.ascontiguousarray(rgb[:, :, ::-1]), [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes()
        pil = np.asarray(Image.open(io.BytesIO(jpg)).convert("RGB"))
        out[f"enc_spec_{i}"], out[f"enc_shape_{i}"], out[f"enc_q_{i}"] = np.array(spec), np.array([h, w]), np.array(q)
        if h * w > 200 * 200:
            out[f"enc_sha_{i}"], out[f"enc_pilsha_{i}"] = np.array(sha(jpg)), np.array(sha(pil))
        else:
            out[f"enc_jpg_{i}"], out[f"enc_pil_{i}"] = np.frombuffer(jpg, np.uint8), pil
    out["enc_n"] = np.array(len(cases))
    out["dm_n"] = np.array(len(dm))

    blobs = []
    for (h, w) in [(1, 1), (5, 7), (40, 64), (96, 128)]:
        g = synthetic.oxford_mosaic((h, w), h * 1000 + w)
        for f in range(5):
            blobs.append(synthetic.encode_png(g, filters=f))
        blobs.append(synthetic.encode_png(g, filters=[r % 5 for r in range(h)], level=9, idat=100))
        blobs.append(cv2.imencode(".png", g)[1].tobytes())
        b = io.BytesIO()
        Image.fromarray(g, "L").save(b, "PNG")
        blobs.append(b.getvalue())
    for i, b in enumerate(blobs):
        out[f"png_blob_{i}"] = np.frombuffer(b, np.uint8)
        out[f"png_pix_{i}"] = np.asarray(Image.open(io.BytesIO(b)))
    out["png_n"] = np.array(len(blobs))
    path = os.path.join(ROOT, "tests", "golden", "oxford_images_small.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes,", len(cases), "encoder cases")


if __name__ == "__main__":
    main()
