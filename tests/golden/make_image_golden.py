"""Write tests/golden/image_small.npz: the loaders' image side computed by the real libraries -- cv2.resize
(INTER_LINEAR), numpy crop and flip, torchvision.transforms.functional.adjust_* on PIL images -- for seeded synthetic
frames and explicit per-sample parameters.  Needs cv2, Pillow and torchvision; the tests only read the file.

    python tests/golden/make_image_golden.py
"""
import os

import cv2
import numpy as np
import torchvision.transforms.functional as F
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
H, W = 20, 36
# (h, w, row0, rows, scale, flip, jitter, order, (brightness, contrast, saturation, hue))
CASES = [
    (44, 76, 4, 40, 0.6, 0, 1, (0, 1, 2, 3), (1.2, 0.8, 1.2, -0.1)),
    (45, 79, 0, 42, 0.5, 1, 1, (3, 2, 1, 0), (0.8, 1.2, 0.8, 0.1)),
    (41, 72, 0, 41, 0.5, 0, 1, (2, 0, 3, 1), (1.05, 1.13, 0.91, -0.037)),
    (40, 72, 0, 40, 0.5, 1, 0, (0, 1, 2, 3), (1.0, 1.0, 1.0, 0.0)),
    (52, 90, 6, 46, 0.45, 1, 1, (1, 3, 0, 2), (0.93, 0.8, 1.2, 0.0)),
    (38, 80, 0, 38, 0.55, 0, 1, (3, 0, 1, 2), (1.2, 1.2, 1.2, -0.1)),
]


def frame(rng, h, w, adversarial):
    """Smooth colour gradients plus noise; the adversarial frame adds grey rows, max-channel ties and primaries."""
    y, x = np.mgrid[0:h, 0:w]
    base = np.stack([255 * x / w, 255 * y / h, 255 * (x + y) / (w + h)], -1)
    img = np.clip(base + rng.normal(0, 40, (h, w, 3)), 0, 255).astype(np.uint8)
    if adversarial:
        lv = np.arange(256, dtype=np.uint8)
        img[0] = lv[np.arange(w) * 255 // (w - 1)][:, None]
        img[1, :, :] = [250, 250, 3]
        img[2, :, :] = [3, 250, 250]
        img[3, :, :] = [255, 0, 0]
        img[4, :, :] = [0, 0, 255]
        img[5:9] = rng.integers(0, 2, (4, w, 3), dtype=np.uint8) * 255
    return img


def main():
    rng = np.random.default_rng(2026)
    imgs, shapes, params, factors, out, Ks, Kout = [], [], [], [], [], [], []
    for i, (h, w, row0, rows, s, flip, jitter, order, fac) in enumerate(CASES):
        raw = frame(rng, h, w, adversarial=i == 0)
        dh, dw = int(round(rows * s)), int(round(w * s))
        dy, dx = int(rng.integers(0, dh - H + 1)), int(rng.integers(0, dw - W + 1))
        img = cv2.resize(raw[row0:row0 + rows], (dw, dh), interpolation=cv2.INTER_LINEAR)[dy:dy + H, dx:dx + W]
        fac = np.float32(fac)
        if jitter:
            pil = Image.fromarray(np.ascontiguousarray(img))
            steps = (F.adjust_brightness, F.adjust_contrast, F.adjust_saturation, F.adjust_hue)
            for op in order:
                pil = steps[op](pil, float(fac[op]))
            img = np.array(pil)
        if flip:
            img = np.flip(img, 1)
        K = np.array([[100.0 + i, 0.0, w / 2 + 0.25], [0.0, 101.0 - i, h / 2 - 0.5], [0.0, 0.0, 1.0]])
        Kc = K.copy()
        Kc[1, 2] -= row0                          # camera_matrix_cropping, camera_matrix_scaling, cropping
        Kc = s * Kc
        Kc[2, 2] = 1
        Kc[0, 2] -= dx
        Kc[1, 2] -= dy
        imgs.append(raw.reshape(-1))
        shapes.append((h, w))
        params.append((row0, rows, dh, dw, dy, dx, flip, jitter, *order))
        factors.append(fac)
        out.append(np.ascontiguousarray(img.transpose(2, 0, 1)))
        Ks.append(K)
        Kout.append(Kc)
    np.savez_compressed(os.path.join(HERE, "image_small.npz"), frames=np.concatenate(imgs),
                        shapes=np.array(shapes, np.int64), params=np.array(params, np.int64),
                        factors=np.stack(factors), scale=np.array([c[4] for c in CASES]), img=np.stack(out),
                        K=np.stack(Ks), K_out=np.stack(Kout), img_HW=np.array([H, W]),
                        versions=np.array([cv2.__version__, Image.__version__]))


if __name__ == "__main__":
    main()
