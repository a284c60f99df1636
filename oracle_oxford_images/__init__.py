"""CPU restatements of the Oxford stereo-centre image conversion (csrc/oxford_images.cu) and the baseline JPEG encoder
(csrc/jpeg_encode.cu), for tests and for checking the rules before any GPU run (DESIGN.md 4.25).

sdk_load_image is the RobotCar SDK's load_image(path, CameraModel) for the stereo camera, glued together here over
scipy's own convolve and map_coordinates: colour_demosaicing's demosaicing_CFA_Bayer_bilinear(CFA, 'GBRG') in
float64, then CameraModel.undistort (map_coordinates(channel, lut[:, 1::-1].T.reshape(2, H, W), order=1) per
channel), then np.array(img).astype(np.uint8).  debayer_undistort restates the same result in the kernel's
arithmetic: the demosaiced values as integer tap sums times 0.25, and map_coordinates_order1, scipy's order-1
'constant'-mode interpolation step by step.

encode_jpeg restates libjpeg-turbo's baseline 4:2:0 compression as OpenCV drives it (jccolor.c rgb_ycc_convert,
jcsample.c h2v2_downsample, jcprepct.c / jcsample.c edge expansion, jfdctint.c jpeg_fdct_islow, jcdctmgr.c
quantisation, jccoefct.c dummy blocks, jchuff.c encode_one_block), with deepi2p_b200.jpeg_encode's markers.
"""
import numpy as np

from deepi2p_b200 import jpeg_encode as je
from deepi2p_b200.jpeg import ZIGZAG

# ------------------------------------------------------------------------------------------------ the SDK pipeline
H_G = np.array([[0, 1, 0], [1, 4, 1], [0, 1, 0]], np.float64) / 4
H_RB = np.array([[1, 2, 1], [2, 4, 2], [1, 2, 1]], np.float64) / 4


def bayer_masks(shape, pattern="gbrg"):
    """colour_demosaicing masks_CFA_Bayer: (R, G, B) boolean masks of the 2 x 2 pattern."""
    ch = {c: np.zeros(shape, bool) for c in "RGB"}
    for c, (y, x) in zip(pattern.upper(), [(0, 0), (0, 1), (1, 0), (1, 1)]):
        ch[c][y::2, x::2] = True
    return ch["R"], ch["G"], ch["B"]


def sdk_demosaic(cfa, pattern="gbrg"):
    """demosaicing_CFA_Bayer_bilinear(CFA, pattern): float64 [H, W, 3]."""
    from scipy.ndimage import convolve
    cfa = np.asarray(cfa, np.float64)
    r, g, b = bayer_masks(cfa.shape, pattern)
    return np.stack([convolve(cfa * r, H_RB), convolve(cfa * g, H_G), convolve(cfa * b, H_RB)], -1)


def lut_coords(lut, h, w):
    """CameraModel.undistort's coordinates: lut [h w, 2] (x, y) -> [2, h, w] (row, column)."""
    lut = np.asarray(lut, np.float64)
    if lut.shape != (h * w, 2):
        raise ValueError("Incorrect image size for camera model")
    return lut[:, 1::-1].T.reshape(2, h, w)


def sdk_load_image(cfa, lut, pattern="gbrg"):
    """load_image(path, model) on a grey mosaic already read as uint8 [H, W]: uint8 [H, W, 3] RGB."""
    from scipy.ndimage import map_coordinates
    img = sdk_demosaic(cfa, pattern)
    coords = lut_coords(lut, *img.shape[:2])
    und = np.rollaxis(np.array([map_coordinates(img[:, :, c], coords, order=1) for c in range(3)]), 0, 3)
    return np.array(und.astype(img.dtype)).astype(np.uint8)


def map_coordinates_order1(channel, coords):
    """scipy.ndimage.map_coordinates(channel, coords, order=1) (mode 'constant', cval 0) for a float64 [H, W] array
    with H, W >= 2, step by step: a coordinate below 0 or above n - 1 on either axis gives 0; otherwise, per axis,
    f = floor(c), t = c - f, weights w0 = 1 - t and w1 = 1 - w0, and the four taps (f0, f1), (f0, f1 + 1),
    (f0 + 1, f1), (f0 + 1, f1 + 1) accumulate (v w_row) w_col into a sum that starts at 0.0, in that order.  A tap
    past the last row or column has weight 0 and contributes 0."""
    ch = np.asarray(channel, np.float64)
    H, W = ch.shape
    y = np.asarray(coords[0], np.float64)
    x = np.asarray(coords[1], np.float64)
    out_y = (y < 0) | (y > H - 1)
    out_x = (x < 0) | (x > W - 1)
    inside = ~(out_y | out_x)
    yy = np.where(inside, y, 0.0)
    xx = np.where(inside, x, 0.0)
    fy, fx = np.floor(yy), np.floor(xx)
    ty, tx = yy - fy, xx - fx
    wy0 = 1.0 - ty
    wy1 = 1.0 - wy0
    wx0 = 1.0 - tx
    wx1 = 1.0 - wx0
    iy, ix = fy.astype(np.int64), fx.astype(np.int64)
    iy1, ix1 = np.minimum(iy + 1, H - 1), np.minimum(ix + 1, W - 1)
    acc = np.zeros(y.shape, np.float64)
    for r, wr in ((iy, wy0), (iy1, wy1)):
        for c, wc in ((ix, wx0), (ix1, wx1)):
            acc = acc + (ch[r, c] * wr) * wc
    return np.where(inside, acc, 0.0)


def demosaic_sums(cfa, pattern="gbrg"):
    """The demosaiced values as integers: 4 x the float64 result, the masked 3 x 3 tap sums with the integer kernel
    weights and reflected borders (index -1 -> 0, n -> n - 1).  int64 [H, W, 3]."""
    cfa = np.asarray(cfa, np.int64)
    H, W = cfa.shape
    masks = bayer_masks(cfa.shape, pattern)
    kern = (H_RB * 4, H_G * 4, H_RB * 4)
    ry = np.clip(np.arange(-1, H + 1), 0, H - 1)
    rx = np.clip(np.arange(-1, W + 1), 0, W - 1)
    out = np.zeros((H, W, 3), np.int64)
    for c in range(3):
        m = (cfa * masks[c])[np.ix_(ry, rx)]
        k = kern[c].astype(np.int64)
        for dy in range(3):
            for dx in range(3):
                out[:, :, c] += k[dy, dx] * m[dy:dy + H, dx:dx + W]
    return out


def debayer_undistort(cfa, lut, pattern="gbrg"):
    """sdk_load_image in the kernel's arithmetic: uint8 [H, W, 3]."""
    cfa = np.asarray(cfa, np.uint8)
    H, W = cfa.shape
    coords = lut_coords(lut, H, W)
    rgb = demosaic_sums(cfa, pattern).astype(np.float64) * 0.25
    out = np.stack([map_coordinates_order1(rgb[:, :, c], coords) for c in range(3)], -1)
    return out.astype(np.uint8)


# ------------------------------------------------------------------------------------------------ the JPEG encoder
def rgb_to_ycc(rgb):
    """jccolor.c rgb_ycc_convert: int64 [H, W, 3] (Y, Cb, Cr) of uint8 RGB, 16-bit fixed point."""
    fix = lambda v: int(v * 65536 + 0.5)                       # noqa: E731
    r, g, b = (np.asarray(rgb, np.int64)[:, :, i] for i in range(3))
    half, off = 1 << 15, 128 << 16
    y = (fix(0.29900) * r + fix(0.58700) * g + fix(0.11400) * b + half) >> 16
    cb = (-fix(0.16874) * r - fix(0.33126) * g + fix(0.5) * b + off + half - 1) >> 16
    cr = (fix(0.5) * r - fix(0.41869) * g - fix(0.08131) * b + off + half - 1) >> 16
    return np.stack([y, cb, cr], -1)


def planes(rgb):
    """The three component planes libjpeg's preprocessing hands to the DCT: Y [8 yby, 16 mcux] (the last row and
    column replicated), Cb and Cr [8 mcuy, 8 mcux] (full-resolution rows padded to an even count and columns to
    16 mcux by replication, h2v2_downsample with the bias 1, 2, 1, 2, ... along each row, then the last downsampled
    row replicated to the iMCU height)."""
    H, W = rgb.shape[:2]
    g = je.geometry(H, W)
    ycc = rgb_to_ycc(rgb)
    rows = np.minimum(np.arange(16 * g["mcuy"]), H - 1)
    cols = np.minimum(np.arange(16 * g["mcux"]), W - 1)
    y = ycc[:, :, 0][np.ix_(rows, cols)]
    crow = -(-H // 2)
    full_rows = np.minimum(np.arange(2 * crow), H - 1)
    out = [y]
    bias = np.tile([1, 2], 4 * g["mcux"])
    for c in (1, 2):
        p = ycc[:, :, c][np.ix_(full_rows, cols)]
        d = (p[0::2, 0::2] + p[0::2, 1::2] + p[1::2, 0::2] + p[1::2, 1::2] + bias) >> 2
        d = d[np.minimum(np.arange(8 * g["mcuy"]), crow - 1)]
        out.append(d)
    return out


_C = dict(c0_298=2446, c0_390=3196, c0_541=4433, c0_765=6270, c0_899=7373, c1_175=9633, c1_501=12299,
          c1_847=15137, c1_961=16069, c2_053=16819, c2_562=20995, c3_072=25172)


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _fdct_1d(d, last):
    """One pass of jfdctint.c over axis -1 of int64 [..., 8] (CONST_BITS 13, PASS1_BITS 2)."""
    c = _C
    t0, t7 = d[..., 0] + d[..., 7], d[..., 0] - d[..., 7]
    t1, t6 = d[..., 1] + d[..., 6], d[..., 1] - d[..., 6]
    t2, t5 = d[..., 2] + d[..., 5], d[..., 2] - d[..., 5]
    t3, t4 = d[..., 3] + d[..., 4], d[..., 3] - d[..., 4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    sh = 13 + 2 if last else 13 - 2
    o = [None] * 8
    if last:
        o[0], o[4] = _descale(t10 + t11, 2), _descale(t10 - t11, 2)
    else:
        o[0], o[4] = (t10 + t11) << 2, (t10 - t11) << 2
    z1 = (t12 + t13) * c["c0_541"]
    o[2] = _descale(z1 + t13 * c["c0_765"], sh)
    o[6] = _descale(z1 + t12 * -c["c1_847"], sh)
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * c["c1_175"]
    t4, t5, t6, t7 = t4 * c["c0_298"], t5 * c["c2_053"], t6 * c["c3_072"], t7 * c["c1_501"]
    z1, z2 = z1 * -c["c0_899"], z2 * -c["c2_562"]
    z3, z4 = z3 * -c["c1_961"] + z5, z4 * -c["c0_390"] + z5
    o[7] = _descale(t4 + z1 + z3, sh)
    o[5] = _descale(t5 + z2 + z4, sh)
    o[3] = _descale(t6 + z2 + z3, sh)
    o[1] = _descale(t7 + z1 + z4, sh)
    return np.stack(o, -1)


def fdct_islow(blocks):
    """jpeg_fdct_islow of int64 [..., 8, 8] level-shifted samples: rows, then columns (output scaled by 8)."""
    rows = _fdct_1d(np.asarray(blocks, np.int64), False)
    return np.swapaxes(_fdct_1d(np.swapaxes(rows, -1, -2), True), -1, -2)


def quantize(coef, q):
    """jcdctmgr.c quantize: |c| rounded-divided by 8 q (floor((|c| + 4 q) / (8 q))) with the sign restored."""
    d = 8 * np.asarray(q, np.int64)
    a = np.abs(coef)
    return np.sign(coef) * ((a + (d >> 1)) // d)


def _blocks(plane):
    h, w = plane.shape
    return plane.reshape(h // 8, 8, w // 8, 8).swapaxes(1, 2)


def coefficients(rgb, quality=95):
    """The quantised blocks in coding order: int64 [mcuy, mcux, 6, 64] (natural order), dummy blocks included (AC
    zero, DC copied as jccoefct.c does)."""
    H, W = rgb.shape[:2]
    g = je.geometry(H, W)
    qt = je.quant_tables(quality)
    ys, cb, cr = planes(rgb)
    out = np.zeros((g["mcuy"], g["mcux"], 6, 64), np.int64)
    yq = quantize(fdct_islow(_blocks(ys - 128)).reshape(2 * g["mcuy"], 2 * g["mcux"], 64), qt[0])
    for k in range(4):
        out[:, :, k] = yq[k // 2::2, k % 2::2]
    out[:, :, 4] = quantize(fdct_islow(_blocks(cb - 128)).reshape(g["mcuy"], g["mcux"], 64), qt[1])
    out[:, :, 5] = quantize(fdct_islow(_blocks(cr - 128)).reshape(g["mcuy"], g["mcux"], 64), qt[1])
    # Dummy blocks: luma blocks past ceil(W / 8) or ceil(H / 8) in the last MCU column or row.
    right = g["ybx"] % 2 == 1
    bottom = g["yby"] % 2 == 1
    last = out[:, -1] if right else None
    if right:
        for k in (1, 3):
            last[:, k] = 0
            last[:, k, 0] = last[:, k - 1, 0]
    if bottom:
        row = out[-1]
        for k in (2, 3):
            row[:, k] = 0
            row[:, k, 0] = row[:, 1, 0]
    return out


def _nbits(v):
    return int(abs(int(v))).bit_length()


class _BitWriter:
    def __init__(self):
        self.bits = []

    def put(self, code, n):
        self.bits.extend((code >> (n - 1 - i)) & 1 for i in range(n))

    def data(self):
        pad = (-len(self.bits)) % 8
        bits = np.array(self.bits + [1] * pad, np.uint8)
        return np.packbits(bits).tobytes() if bits.size else b""


def entropy_code(coefs):
    """jchuff.c encode_one_block over the blocks of coefficients() in MCU order (DC predicted per component), padded
    with 1 bits to a byte and with 0xFF bytes stuffed: the entropy-coded segment."""
    tabs = [je.derived_table(*t) for t in (je.DC_LUMA, je.AC_LUMA, je.DC_CHROMA, je.AC_CHROMA)]
    bw = _BitWriter()
    last = [0, 0, 0]
    for mcu in coefs.reshape(-1, 6, 64):
        for k in range(6):
            comp = 0 if k < 4 else k - 3
            dc_t, ac_t = (tabs[0], tabs[1]) if comp == 0 else (tabs[2], tabs[3])
            blk = mcu[k][ZIGZAG]
            diff = int(blk[0]) - last[comp]
            last[comp] = int(blk[0])
            n = _nbits(diff)
            bw.put(dc_t[n][1], dc_t[n][0])
            if n:
                bw.put((diff if diff >= 0 else diff - 1) & ((1 << n) - 1), n)
            run = 0
            for kk in range(1, 64):
                v = int(blk[kk])
                if v == 0:
                    run += 1
                    continue
                while run > 15:
                    bw.put(ac_t[0xF0][1], ac_t[0xF0][0])
                    run -= 16
                n = _nbits(v)
                sym = (run << 4) + n
                bw.put(ac_t[sym][1], ac_t[sym][0])
                bw.put((v if v >= 0 else v - 1) & ((1 << n) - 1), n)
                run = 0
            if run:
                bw.put(ac_t[0][1], ac_t[0][0])
    return bw.data().replace(b"\xFF", b"\xFF\x00")


def encode_jpeg(rgb, quality=95):
    """cv2.imencode(".jpg", rgb[:, :, ::-1], [IMWRITE_JPEG_QUALITY, quality]) restated: bytes."""
    rgb = np.asarray(rgb, np.uint8)
    H, W = rgb.shape[:2]
    return je.header(H, W, quality) + entropy_code(coefficients(rgb, quality)) + je.EOI


# ------------------------------------------------------------------------------------------------ fixture inputs
def special_lut(h, w):
    """A LUT whose coordinates sit on the interpolation's edges: integers, n - 1 exactly, the largest double below
    n - 1, -0.0, 1e-9 outside either edge and far outside, cycled over the pixels; float64 [h w, 2]."""
    ys = [0.0, -0.0, 1.0, h - 1.0, np.nextafter(h - 1.0, 0.0), -1e-9, h - 1 + 1e-9, -5.0, h + 7.5, 0.5, h / 2.0]
    xs = [0.0, w - 1.0, -0.0, np.nextafter(w - 1.0, 0.0), 2.0, w - 1 + 1e-9, -1e-9, w + 3.0, -40.0, 0.25, w / 3.0]
    n = h * w
    y = np.array([ys[i % len(ys)] for i in range(n)])
    x = np.array([xs[(i // len(ys)) % len(xs)] for i in range(n)])
    return np.stack([x, y], 1)


def identity_lut(h, w):
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    return np.stack([xx.ravel(), yy.ravel()], 1)


def fixture_image(spec, h, w):
    """The encoder fixture's RGB inputs by name: 'rand:<seed>' uniform noise, 'sat:<seed>' black and white pixels
    (long runs of 0xFF bytes in the stream), 'flat:<v>' one grey level (EOB-only blocks), 'grad' smooth gradients."""
    kind, _, arg = spec.partition(":")
    if kind == "rand":
        return np.random.default_rng(int(arg)).integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "sat":
        m = np.random.default_rng(int(arg)).random((h, w, 1)) < 0.5
        return np.repeat(np.where(m, 255, 0).astype(np.uint8), 3, 2)
    if kind == "flat":
        return np.full((h, w, 3), int(arg), np.uint8)
    if kind == "grad":
        yy, xx = np.mgrid[0:h, 0:w]
        return np.stack([(yy * 7 + xx * 3) % 256, (xx * 5) % 256, (yy * 11) % 256], -1).astype(np.uint8)
    raise ValueError(f"unknown test image {spec!r}")
