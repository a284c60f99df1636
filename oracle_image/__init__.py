"""numpy oracle of the loaders' image side -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and the benchmark scripts may import this package; deepi2p_b200.imageprep never
does.  It restates DESIGN.md 4.13 one operation at a time: cv2.resize(INTER_LINEAR) on uint8 images by OpenCV's
fixed-point path (11-bit weights, the SIMD vertical pass), and torchvision's ColorJitter steps on PIL images by
Pillow's arithmetic (ImagingBlend with a float32 factor, the L24 luma, Convert.c's rgb2hsv / hsv2rgb with their mix of
float and double).  float32 / float64 numpy operations round once each and never contract a multiply-add, like the C
code they restate.
"""
import numpy as np

BRIGHTNESS, CONTRAST, SATURATION, HUE = 0, 1, 2, 3     # torchvision ColorJitter's fn_idx numbering


def resize_dims(h, w, s):
    """The loaders' cv2.resize target (dh, dw) = (int(round(h s)), int(round(w s))), Python's ties-to-even round."""
    return int(round(h * s)), int(round(w * s))


def axis_coeffs(n_src, n_dst):
    """cv2's linear source index and int16 weights along one axis: (sx, a0, a1) for d in [0, n_dst)."""
    scale = 1.0 / (float(n_dst) / n_src)
    d = np.arange(n_dst, dtype=np.float64)
    f = ((d + 0.5) * scale - 0.5).astype(np.float32)
    sx = np.floor(f).astype(np.int64)
    f = f - sx.astype(np.float32)
    lo, hi = sx < 0, sx >= n_src - 1
    sx = np.where(lo, 0, np.where(hi, n_src - 1, sx))
    f = np.where(lo | hi, np.float32(0), f).astype(np.float32)
    a0 = np.rint((np.float32(1) - f) * np.float32(2048)).astype(np.int64)
    a1 = np.rint(f * np.float32(2048)).astype(np.int64)
    return sx, a0, a1


def resize_window(img, dh, dw, y0=0, x0=0, H=None, W=None):
    """Rows [y0, y0+H) and columns [x0, x0+W) of cv2.resize(img, (dw, dh), INTER_LINEAR) for uint8 img [h,w,C]."""
    img = np.asarray(img)
    h, w = img.shape[:2]
    H = dh if H is None else H
    W = dw if W is None else W
    sx, a0, a1 = (v[x0:x0 + W] for v in axis_coeffs(w, dw))
    sy, b0, b1 = (v[y0:y0 + H] for v in axis_coeffs(h, dh))
    sx1 = np.minimum(sx + 1, w - 1)
    sy1 = np.minimum(sy + 1, h - 1)
    S = img.astype(np.int64)

    def row(ys):
        return S[ys][:, sx] * a0[None, :, None] + S[ys][:, sx1] * a1[None, :, None]

    r0, r1 = row(sy), row(sy1)
    v = (((r0 >> 4) * b0[:, None, None]) >> 16) + (((r1 >> 4) * b1[:, None, None]) >> 16)
    return np.clip((v + 2) >> 2, 0, 255).astype(np.uint8)


def luma(img):
    """Pillow's RGB -> L: (19595 R + 38470 G + 7471 B + 0x8000) >> 16, as int64 [H,W]."""
    x = np.asarray(img).astype(np.int64)
    return (19595 * x[..., 0] + 38470 * x[..., 1] + 7471 * x[..., 2] + 0x8000) >> 16


def blend(deg, img, a):
    """ImagingBlend(deg, img, a): t = (float) deg + a (img - deg) in float32; 0 <= a <= 1 truncates, any other a
    clips to [0, 255] first."""
    a = np.float32(a)
    deg = np.asarray(deg).astype(np.int64)
    x = np.asarray(img).astype(np.int64)
    t = deg.astype(np.float32) + a * (x - deg).astype(np.float32)
    if 0 <= a <= 1:
        return t.astype(np.int64).astype(np.uint8)
    return np.where(t <= 0, 0, np.where(t >= 255, 255, np.clip(t, 0, 255).astype(np.int64))).astype(np.uint8)


def adjust_brightness(img, a):
    return blend(np.zeros_like(img), img, a)


def contrast_degenerate(luma_sum, n):
    """ImageEnhance.Contrast's grey level: int(mean(L) + 0.5), the mean an exact integer sum over n pixels."""
    return int(float(luma_sum) / float(n) + 0.5)


def adjust_contrast(img, a):
    m = contrast_degenerate(int(luma(img).sum()), luma(img).size)
    return blend(np.full_like(img, m), img, a)


def adjust_saturation(img, a):
    return blend(np.repeat(luma(img)[..., None], 3, axis=-1), img, a)


def hue_shift(hue):
    """torchvision's np.int32(hue * 255).astype(np.uint8): truncation toward zero, then modulo 256."""
    return int(np.int32(hue * 255)) & 255


def rgb2hsv(img):
    """Pillow Convert.c rgb2hsv: float cr, s, rc, gc, bc; the 2.0 / 4.0 / 6.0 / 1.0 / 255.0 steps in double."""
    x = np.asarray(img).astype(np.int64)
    r, g, b = x[..., 0], x[..., 1], x[..., 2]
    mx, mn = x.max(-1), x.min(-1)
    grey = mx == mn
    f32 = np.float32
    with np.errstate(divide="ignore", invalid="ignore"):
        cr = (mx - mn).astype(f32)
        s = cr / mx.astype(f32)
        rc = (mx - r).astype(f32) / cr
        gc = (mx - g).astype(f32) / cr
        bc = (mx - b).astype(f32) / cr
        h = np.where(r == mx, (bc - gc).astype(np.float64),
                     np.where(g == mx, ((2.0 + rc.astype(np.float64)) - bc.astype(np.float64)).astype(f32),
                              ((4.0 + gc.astype(np.float64)) - rc.astype(np.float64)).astype(f32)))
        h = h.astype(f32).astype(np.float64)
        h = np.fmod(h / 6.0 + 1.0, 1.0).astype(f32)
        uh = np.clip(np.trunc(h.astype(np.float64) * 255.0), 0, 255)
        us = np.clip(np.trunc(s.astype(np.float64) * 255.0), 0, 255)
    uh = np.where(grey, 0, uh).astype(np.int64)
    us = np.where(grey, 0, us).astype(np.int64)
    return uh, us, mx


def _round_away(x):
    """C round(): halves away from zero (x >= 0 here)."""
    f = np.floor(x)
    return np.where(x - f >= 0.5, f + 1.0, f)


def hsv2rgb(h, s, v):
    """Pillow Convert.c hsv2rgb: double i and f (f stored as float), float fs; s == 0 gives v."""
    h = np.asarray(h).astype(np.int64)
    s = np.asarray(s).astype(np.int64)
    v = np.asarray(v).astype(np.int64)
    hd = h.astype(np.float32).astype(np.float64) * 6.0 / 255.0
    i = np.floor(hd)
    f = (hd - i).astype(np.float32)
    fs = (s.astype(np.float32).astype(np.float64) / 255.0).astype(np.float32)
    vd = v.astype(np.float64)
    p = _round_away(vd * (1.0 - fs.astype(np.float64)))
    q = _round_away(vd * (1.0 - (fs * f).astype(np.float64)))
    t = _round_away(vd * (1.0 - fs.astype(np.float64) * (1.0 - f.astype(np.float64))))
    p, q, t = (np.clip(a, 0, 255).astype(np.int64) for a in (p, q, t))
    k = i.astype(np.int64) % 6
    table = [(v, t, p), (q, v, p), (p, v, t), (p, q, v), (t, p, v), (v, p, q)]
    out = np.zeros(h.shape + (3,), np.int64)
    for c in range(3):
        ch = np.select([k == j for j in range(6)], [table[j][c] for j in range(6)])
        out[..., c] = np.where(s == 0, v, ch)
    return out.astype(np.uint8)


def adjust_hue(img, shift):
    """torchvision adjust_hue on a PIL RGB image, with the uint8 shift of hue_shift()."""
    h, s, v = rgb2hsv(img)
    return hsv2rgb((h + int(shift)) & 255, s, v)


def color_jitter(img, order, factors, shift=None):
    """ColorJitter's steps in `order` (fn_idx: 0 brightness, 1 contrast, 2 saturation, 3 hue) with factors (b, c, s,
    hue); shift overrides hue_shift(factors[3])."""
    shift = hue_shift(factors[3]) if shift is None else shift
    out = np.asarray(img, dtype=np.uint8)
    for op in order:
        op = int(op)
        if op == BRIGHTNESS:
            out = adjust_brightness(out, factors[0])
        elif op == CONTRAST:
            out = adjust_contrast(out, factors[1])
        elif op == SATURATION:
            out = adjust_saturation(out, factors[2])
        elif op == HUE:
            out = adjust_hue(out, shift)
        else:
            raise ValueError(f"order entries are 0..3 (got {op})")
    return out


def camera_K(K, row_cut_top, s, dx, dy):
    """camera_matrix_cropping(dy=row_cut_top), camera_matrix_scaling(s), camera_matrix_cropping(dx, dy) in fp64."""
    K = np.array(K, dtype=np.float64)
    K[1, 2] -= row_cut_top
    K = s * K
    K[2, 2] = 1
    K[0, 2] -= dx
    K[1, 2] -= dy
    return K


def assemble_image(raw, K, row0, rows, dh, dw, dy, dx, H, W, flip=False, jitter=False, order=(0, 1, 2, 3),
                   factors=(1.0, 1.0, 1.0, 0.0), shift=None, img_scale=None):
    """One sample's image side: rows [row0, row0 + rows) of raw [h,w,3] uint8, resized to (dh, dw), the H x W window
    at (dy, dx), the jitter, a column flip.  Returns (img [3,H,W] float32, K float64 or None)."""
    view = np.asarray(raw)[row0:row0 + rows]
    img = resize_window(view, dh, dw, dy, dx, H, W)
    if jitter:
        img = color_jitter(img, order, factors, shift)
    if flip:
        img = img[:, ::-1]
    Kout = None if K is None else camera_K(K, row0, img_scale, dx, dy)
    return np.ascontiguousarray(img.transpose(2, 0, 1)).astype(np.float32), Kout
