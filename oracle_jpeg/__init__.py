"""CPU restatement of the batched JPEG decoder (csrc/jpeg.cu), checked bit for bit against Pillow 12.2 /
libjpeg-turbo.  It decodes the way libjpeg does -- one stream, one MCU after the other -- and shares only the marker
parser (deepi2p_b200/jpeg.py) with the product; the entropy decoding, DC prediction, islow IDCT, fancy upsampling and
YCbCr -> RGB conversion are written out here independently of the kernels, with every integer step of
libjpeg-turbo's jdhuff.c, jidctint.c, jdsample.c and jdcolor.c.  DESIGN.md 4.19 states the contract.

    decode(blob)              -> h x w x 3 uint8, equal to np.asarray(Image.open(BytesIO(blob)).convert("RGB"))
    decode(blob, stages=True) -> dict(rgb, coef (per component [bh, bw, 64] int16, natural order, DC resolved),
                                      planes (per component [bh*8, bw*8] uint8 IDCT output), header)
"""
import numpy as np

from deepi2p_b200.jpeg import ZIGZAG, huff_codes, image_geometry, parse_jpeg

# jpeg_natural_order with libjpeg's 16 guard entries: a corrupt run length past k = 63 writes coefficient 63.
NATURAL = np.concatenate([ZIGZAG, np.full(16, 63, np.int64)]).tolist()


def entropy_segments(b, start):
    """Unstuff the entropy-coded data after SOS: FF 00 is one FF data byte, FF fill bytes before a marker are dropped,
    RST0..7 split restart intervals, any other marker ends the scan.  Returns (list of interval bytes, the ending
    marker code); raises when no marker ends the data."""
    segs, seg, i, n = [], bytearray(), start, len(b)
    while True:
        j = b.find(b"\xff", i)
        if j < 0:
            raise ValueError("truncated stream (the scan has no ending marker)")
        seg += b[i:j]
        k = j
        while k < n and b[k] == 0xFF:
            k += 1
        if k >= n:
            raise ValueError("truncated stream (the scan has no ending marker)")
        m = b[k]
        if m == 0x00:
            seg.append(0xFF)
        elif 0xD0 <= m <= 0xD7:
            segs.append(bytes(seg))
            seg = bytearray()
        else:
            segs.append(bytes(seg))
            return segs, m
        i = k + 1


def _lut16(table):
    """16-bit lookahead: peek -> (length << 8 | symbol), 0 where no code of <= 16 bits is a prefix."""
    lut = np.zeros(65536, np.int32)
    for length, code, sym in huff_codes(*table):
        lut[code << (16 - length):(code + 1) << (16 - length)] = (length << 8) | sym
    return lut.tolist()


def _int32(x):
    return ((x + 0x80000000) & 0xFFFFFFFF) - 0x80000000


def _int16(x):
    return ((x + 0x8000) & 0xFFFF) - 0x8000


def decode_coefficients(hd, segs):
    """jdhuff.c decode_mcu for every MCU: per component [bh, bw, 64] int16 coefficients in natural order with the DC
    prediction applied (int32 accumulation, stored as JCOEF), reset at each restart interval."""
    mcux, mcuy, geo = image_geometry(hd)
    nc = hd.ncomp
    coef = [np.zeros((g["bh"], g["bw"], 64), np.int16) for g in geo]
    if nc == 1:
        units = [(0, by, bx) for by in range(geo[0]["bh"]) for bx in range(geo[0]["bw"])]
        mcus = [[u] for u in units]
    else:
        mcus = []
        for my in range(mcuy):
            for mx in range(mcux):
                mcus.append([(c, my * g["v"] + y, mx * g["h"] + x) for c, g in enumerate(geo)
                             for y in range(g["v"]) for x in range(g["h"])])
    n_mcu = len(mcus)
    Ri = hd.Ri
    expect = -(-n_mcu // Ri) if Ri else 1
    if len(segs) != expect:
        raise ValueError(f"restart interval count mismatch ({len(segs)} intervals, {expect} expected)")
    dc = [_lut16(c["dc"]) for c in hd.comps]
    ac = [_lut16(c["ac"]) for c in hd.comps]
    m = 0
    for seg in segs:
        n_here = min(Ri, n_mcu - m) if Ri else n_mcu
        a = np.frombuffer(seg + b"\0\0\0\0", np.uint8).astype(np.uint32)
        w = ((a[:-3] << 24) | (a[1:-2] << 16) | (a[2:-1] << 8) | a[3:]).tolist()
        nb = len(seg) * 8
        pos = 0
        pred = [0] * nc
        for _ in range(n_here):
            for c, by, bx in mcus[m]:
                blk = coef[c][by, bx]
                vals = {}
                # DC difference
                e = dc[c][(w[pos >> 3] >> (16 - (pos & 7))) & 0xFFFF]
                if e == 0:
                    raise ValueError("invalid Huffman code" if nb - pos >= 16 else "truncated stream")
                length, s = e >> 8, e & 255
                if pos + length + s > nb:
                    raise ValueError("truncated stream")
                pos += length
                v = 0
                if s:
                    r = (w[pos >> 3] >> (32 - (pos & 7) - s)) & ((1 << s) - 1)
                    pos += s
                    v = r if r >> (s - 1) else r - (1 << s) + 1
                pred[c] = _int32(pred[c] + v)
                vals[0] = _int16(pred[c])
                k = 1
                table = ac[c]
                while k < 64:
                    e = table[(w[pos >> 3] >> (16 - (pos & 7))) & 0xFFFF]
                    if e == 0:
                        raise ValueError("invalid Huffman code" if nb - pos >= 16 else "truncated stream")
                    length, rs = e >> 8, e & 255
                    r, s = rs >> 4, rs & 15
                    if pos + length + s > nb:
                        raise ValueError("truncated stream")
                    pos += length
                    if s:
                        k += r
                        x = (w[pos >> 3] >> (32 - (pos & 7) - s)) & ((1 << s) - 1)
                        pos += s
                        vals[NATURAL[k]] = x if x >> (s - 1) else x - (1 << s) + 1
                        k += 1
                    elif r == 15:
                        k += 16
                    else:
                        break
                for idx, x in vals.items():
                    blk[idx] = x
            m += 1
        # The interval must end here: a further complete symbol is data the MCU count does not account for.
        e = dc[mcus[m % n_mcu][0][0]][(w[pos >> 3] >> (16 - (pos & 7))) & 0xFFFF] if pos < nb else 0
        if e and pos + (e >> 8) + (e & 255) <= nb:
            raise ValueError("MCU count mismatch (data after the last MCU of an interval)")
        if e == 0 and nb - pos >= 16:
            raise ValueError("invalid Huffman code")
    return coef


# jidctint.c constants (CONST_BITS 13)
F0298, F0390, F0541, F0765, F0899, F1175 = 2446, 3196, 4433, 6270, 7373, 9633
F1501, F1847, F1961, F2053, F2562, F3072 = 12299, 15137, 16069, 16819, 20995, 25172
CONST_BITS, PASS1_BITS = 13, 2


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _idct_1d(i0, i1, i2, i3, i4, i5, i6, i7):
    """One jidctint.c butterfly on int64 arrays; returns (tmp10, tmp11, tmp12, tmp13, tmp0, tmp1, tmp2, tmp3)."""
    z2, z3 = i2, i6
    z1 = (z2 + z3) * F0541
    tmp2 = z1 + z3 * -F1847
    tmp3 = z1 + z2 * F0765
    tmp0 = (i0 + i4) << CONST_BITS
    tmp1 = (i0 - i4) << CONST_BITS
    tmp10, tmp13 = tmp0 + tmp3, tmp0 - tmp3
    tmp11, tmp12 = tmp1 + tmp2, tmp1 - tmp2
    t0, t1, t2, t3 = i7, i5, i3, i1
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * F1175
    t0, t1, t2, t3 = t0 * F0298, t1 * F2053, t2 * F3072, t3 * F1501
    z1, z2, z3, z4 = z1 * -F0899, z2 * -F2562, z3 * -F1961, z4 * -F0390
    z3 += z5
    z4 += z5
    t0 += z1 + z3
    t1 += z2 + z4
    t2 += z2 + z3
    t3 += z1 + z4
    return tmp10, tmp11, tmp12, tmp13, t0, t1, t2, t3


def idct_islow(coef, q):
    """jpeg_idct_islow for [N,64] natural-order coefficients and their quantisers: [N,8,8] uint8.  Dequantisation
    multiplies as ISLOW_MULT_TYPE (the quantiser cast to int16); the output indexes the post-IDCT range_limit table
    with x & RANGE_MASK (1023), which clamps [-128-512, 127+384] and wraps beyond."""
    c = coef.astype(np.int64).reshape(-1, 8, 8) * q.astype(np.int16).astype(np.int64).reshape(1, 8, 8)
    # pass 1: columns (the all-zero-AC shortcut gives the same value as the full butterfly)
    t10, t11, t12, t13, t0, t1, t2, t3 = _idct_1d(*(c[:, r, :] for r in range(8)))
    n = CONST_BITS - PASS1_BITS
    ws = np.stack([_descale(t10 + t3, n), _descale(t11 + t2, n), _descale(t12 + t1, n), _descale(t13 + t0, n),
                   _descale(t13 - t0, n), _descale(t12 - t1, n), _descale(t11 - t2, n), _descale(t10 - t3, n)], 1)
    ws = ws.astype(np.int32).astype(np.int64)       # the int workspace
    # pass 2: rows
    t10, t11, t12, t13, t0, t1, t2, t3 = _idct_1d(*(ws[:, :, k] for k in range(8)))
    n = CONST_BITS + PASS1_BITS + 3
    out = np.stack([_descale(t10 + t3, n), _descale(t11 + t2, n), _descale(t12 + t1, n), _descale(t13 + t0, n),
                    _descale(t13 - t0, n), _descale(t12 - t1, n), _descale(t11 - t2, n), _descale(t10 - t3, n)], 2)
    return range_limit(out)


def range_limit(x):
    """IDCT_range_limit[x & RANGE_MASK]: the 10-bit wrap of x, then clamp of x + 128 to [0, 255]."""
    t = (x.astype(np.int64) & 1023)
    s = np.where(t >= 512, t - 1024, t)
    return np.clip(s + 128, 0, 255).astype(np.uint8)


def component_planes(hd, coef):
    """The IDCT output of every block: per component a [bh*8, bw*8] uint8 plane."""
    planes = []
    for c, comp in zip(coef, hd.comps):
        bh, bw = c.shape[:2]
        px = idct_islow(c.reshape(-1, 64), comp["q"]).reshape(bh, bw, 8, 8)
        planes.append(np.ascontiguousarray(px.transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8)))
    return planes


def upsample(plane, dw, dh, rh, rv, W, H):
    """jdsample.c for one component of downsampled size dw x dh and ratios (rh, rv): fullsize, fancy h2v1 / h2v2
    (when dw > 2, else box replication) or fancy h1v2; context rows above the first and below the last row duplicate
    them.  Returns [H, W] int64."""
    p = plane[:dh, :dw].astype(np.int64)
    if rh == 1 and rv == 1:
        return p[:H, :W]
    if rh == 2 and dw <= 2:                     # h2v1 / h2v2 without fancy upsampling: box replication
        out = np.repeat(np.repeat(p, rh, 1), rv, 0)
        return out[:H, :W]
    if rv == 2:                                 # vertical: nearer row x 3 + further row (above for even rows)
        up = np.concatenate([p[:1], p[:-1]], 0)
        dn = np.concatenate([p[1:], p[-1:]], 0)
        colsum = np.empty((2 * dh, dw), np.int64)
        colsum[0::2] = 3 * p + up
        colsum[1::2] = 3 * p + dn
    else:
        colsum = p
    if rh == 1:                                 # h1v2
        out = colsum.copy()
        out[0::2] = (colsum[0::2] + 1) >> 2
        out[1::2] = (colsum[1::2] + 2) >> 2
        return out[:H, :W]
    left = np.concatenate([colsum[:, :1], colsum[:, :-1]], 1)
    right = np.concatenate([colsum[:, 1:], colsum[:, -1:]], 1)
    out = np.empty((colsum.shape[0], 2 * dw), np.int64)
    if rv == 2:                                 # h2v2
        out[:, 0::2] = (3 * colsum + left + 8) >> 4
        out[:, 1::2] = (3 * colsum + right + 7) >> 4
        out[:, 0] = (4 * colsum[:, 0] + 8) >> 4
        out[:, -1] = (4 * colsum[:, -1] + 7) >> 4
    else:                                       # h2v1
        out[:, 0::2] = (3 * colsum + left + 1) >> 2
        out[:, 1::2] = (3 * colsum + right + 2) >> 2
        out[:, 0] = colsum[:, 0]
        out[:, -1] = colsum[:, -1]
    return out[:H, :W]


SCALEBITS, ONE_HALF = 16, 1 << 15


def _fix(x):
    return int(x * (1 << SCALEBITS) + 0.5)


def ycc_to_rgb(y, cb, cr):
    """jdcolor.c ycc_rgb_convert with build_ycc_rgb_table's tables."""
    x = np.arange(256, dtype=np.int64) - 128
    cr_r = (_fix(1.40200) * x + ONE_HALF) >> SCALEBITS
    cb_b = (_fix(1.77200) * x + ONE_HALF) >> SCALEBITS
    cr_g = -_fix(0.71414) * x
    cb_g = -_fix(0.34414) * x + ONE_HALF
    r = y + cr_r[cr]
    g = y + ((cb_g[cb] + cr_g[cr]) >> SCALEBITS)
    b = y + cb_b[cb]
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def decode(blob, stages=False):
    """Decode one JPEG stream to h x w x 3 uint8 RGB (grey replicated).  Raises ValueError where the GPU decoder
    does: an unsupported stream, a missing ending marker or EOI, a bad Huffman code, truncation, or an interval or MCU
    count that does not match."""
    b = bytes(blob)
    hd = parse_jpeg(b)
    segs, marker = entropy_segments(b, hd.scan)
    if marker != 0xD9:
        raise ValueError(f"unexpected marker 0xFF{marker:02X} after the scan (only one scan and EOI are supported)")
    if not hd.Ri and len(segs) > 1:
        raise ValueError("restart interval count mismatch (RST markers without a DRI)")
    coef = decode_coefficients(hd, segs)
    planes = component_planes(hd, coef)
    W, H = hd.W, hd.H
    _, _, geo = image_geometry(hd)
    if hd.ncomp == 1:
        yy = planes[0][:H, :W]
        rgb = np.repeat(yy[:, :, None], 3, 2)
    else:
        full = [upsample(pl, g["dw"], g["dh"], hd.hmax // g["h"], hd.vmax // g["v"], W, H)
                for pl, g in zip(planes, geo)]
        rgb = ycc_to_rgb(*full)
    if stages:
        return dict(rgb=rgb, coef=coef, planes=planes, header=hd)
    return rgb
