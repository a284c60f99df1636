"""Host side of the batched JPEG decoder (csrc/jpeg.cu): the marker parser and the packing of the device tables.

parse_jpeg reads one stream's headers (SOI .. SOS) the way libjpeg-turbo's jdmarker.c / jdapimin.c do for the inputs
DESIGN.md 4.19 supports -- 8-bit baseline or extended sequential Huffman, one interleaved scan of 1 or 3 components,
sampling ratios of 1 or 2 per axis -- and raises ValueError with the reason for anything else.  It needs only numpy,
so oracle_jpeg/ and the CPU tests use it without the CUDA library.  imageprep.decode_jpeg_batch is the public entry.
"""
import numpy as np

# jpeg_natural_order: zig-zag index -> natural (row-major) index.
ZIGZAG = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
    28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
    54, 47, 55, 62, 63], dtype=np.int64)

_SOF_NAMES = {0xC2: "progressive", 0xC3: "lossless", 0xC5: "differential sequential (hierarchical)",
              0xC6: "differential progressive (hierarchical)", 0xC7: "differential lossless (hierarchical)",
              0xC9: "arithmetic-coded sequential", 0xCA: "arithmetic-coded progressive",
              0xCB: "arithmetic-coded lossless", 0xCD: "arithmetic-coded differential sequential",
              0xCE: "arithmetic-coded differential progressive", 0xCF: "arithmetic-coded differential lossless"}

HUFF_WORDS = 356          # one device Huffman table: lut u16[512], maxcode i32[18], valoff i32[18], vals u8[256]
DESC = 48                 # int64 slots of one image descriptor (the slot enum at the top of csrc/jpeg.cu)


class JpegHeader(dict):
    """Attribute view of parse_jpeg's result."""
    __getattr__ = dict.__getitem__


def _u16(b, i):
    if i + 2 > len(b):
        raise ValueError("truncated stream (inside a marker segment)")
    return (b[i] << 8) | b[i + 1]


def huff_codes(bits, vals):
    """Canonical codes of a DHT table (jdhuff.c jpeg_make_d_derived_tbl): a list of (length, code, symbol); raises on
    a table whose codes overflow their length."""
    out, code, p = [], 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            out.append((length, code, vals[p]))
            code += 1
            p += 1
        if code >= (1 << length):
            raise ValueError("bad Huffman table (codes overflow their length)")
        code <<= 1
    return out


def parse_jpeg(blob):
    """Headers of one JPEG stream.  Returns a JpegHeader with W, H, ncomp, comps (list of dicts: id, h, v, q (64
    int64 quantisers, natural order), dc and ac (bits[16], vals) tables), Ri (restart interval in MCUs, 0 = none),
    scan (byte offset of the entropy-coded data), hmax, vmax.  Raises ValueError naming the reason for a stream
    outside the supported set."""
    b = bytes(blob)
    if len(b) < 4 or b[0] != 0xFF or b[1] != 0xD8:
        raise ValueError("not a JPEG stream (no SOI marker)")
    i = 2
    qt, dht = {}, {}
    frame = None
    Ri = 0
    jfif = adobe = False
    adobe_transform = None
    while True:
        if i >= len(b):
            raise ValueError("truncated stream (no SOS marker)")
        if b[i] != 0xFF:
            raise ValueError(f"corrupt stream (byte 0x{b[i]:02X} where a marker was expected at {i})")
        while i < len(b) and b[i] == 0xFF:   # fill bytes before a marker
            i += 1
        if i >= len(b):
            raise ValueError("truncated stream (no SOS marker)")
        m = b[i]
        i += 1
        if m == 0xD9:
            raise ValueError("stream has no scan (EOI before SOS)")
        if 0xD0 <= m <= 0xD7 or m == 0x01:
            continue
        if m == 0xD8:
            raise ValueError("corrupt stream (a second SOI marker)")
        L = _u16(b, i)
        if L < 2 or i + L > len(b):
            raise ValueError("truncated stream (inside a marker segment)")
        seg = b[i + 2:i + L]
        if m in (0xC0, 0xC1):
            if frame is not None:
                raise ValueError("corrupt stream (two SOF markers)")
            if len(seg) < 6:
                raise ValueError("corrupt SOF segment")
            P, H, W, nf = seg[0], _u16(seg, 1), _u16(seg, 3), seg[5]
            if P != 8:
                raise ValueError(f"{P}-bit precision is not supported (only 8-bit)")
            if H == 0:
                raise ValueError("a DNL-defined height (SOF height 0) is not supported")
            if W == 0:
                raise ValueError("corrupt SOF segment (width 0)")
            if len(seg) != 6 + 3 * nf:
                raise ValueError("corrupt SOF segment (length does not match its components)")
            comps = []
            for c in range(nf):
                cid, hv, tq = seg[6 + 3 * c], seg[7 + 3 * c], seg[8 + 3 * c]
                h, v = hv >> 4, hv & 15
                if not (1 <= h <= 4 and 1 <= v <= 4) or tq > 3:
                    raise ValueError("corrupt SOF segment (sampling factor or table index)")
                comps.append(dict(id=cid, h=h, v=v, tq=tq))
            frame = dict(W=W, H=H, comps=comps)
        elif m in _SOF_NAMES:
            raise ValueError(f"{_SOF_NAMES[m]} JPEG (SOF{m - 0xC0}) is not supported")
        elif m == 0xCC:
            raise ValueError("arithmetic-coded JPEG (DAC marker) is not supported")
        elif m == 0xC4:
            p = 0
            while p < len(seg):
                if p + 17 > len(seg):
                    raise ValueError("corrupt DHT segment")
                tc, th = seg[p] >> 4, seg[p] & 15
                bits = list(seg[p + 1:p + 17])
                n = sum(bits)
                if tc > 1 or th > 3 or n > 256 or p + 17 + n > len(seg):
                    raise ValueError("corrupt DHT segment")
                vals = list(seg[p + 17:p + 17 + n])
                huff_codes(bits, vals)
                dht[(tc, th)] = (bits, vals)
                p += 17 + n
        elif m == 0xDB:
            p = 0
            while p < len(seg):
                pq, tq = seg[p] >> 4, seg[p] & 15
                n = 128 if pq else 64
                if pq > 1 or tq > 3 or p + 1 + n > len(seg):
                    raise ValueError("corrupt DQT segment")
                raw = np.frombuffer(seg[p + 1:p + 1 + n], dtype=">u2" if pq else np.uint8).astype(np.int64)
                q = np.zeros(64, np.int64)
                q[ZIGZAG] = raw
                qt[tq] = q
                p += 1 + n
        elif m == 0xDD:
            if len(seg) != 2:
                raise ValueError("corrupt DRI segment")
            Ri = _u16(seg, 0)
        elif m == 0xE0:
            if len(seg) >= 14 and seg[:5] == b"JFIF\0":
                jfif = True
        elif m == 0xEE:
            if len(seg) >= 12 and seg[:5] == b"Adobe":
                adobe, adobe_transform = True, seg[11]
        elif 0xE1 <= m <= 0xEF or m == 0xFE:
            pass
        elif m == 0xDA:
            break
        else:
            raise ValueError(f"unsupported marker 0xFF{m:02X} before the scan")
        i += L
    # SOS
    if frame is None:
        raise ValueError("corrupt stream (SOS before SOF)")
    ns = seg[0] if len(seg) else 0
    if len(seg) != 4 + 2 * ns or ns < 1:
        raise ValueError("corrupt SOS segment")
    comps = frame["comps"]
    nf = len(comps)
    if nf == 4:
        raise ValueError("4-component (CMYK / YCCK) JPEG is not supported")
    if nf not in (1, 3):
        raise ValueError(f"{nf}-component JPEG is not supported (only 1 or 3)")
    if ns != nf:
        raise ValueError(f"multi-scan JPEG is not supported (the first scan has {ns} of {nf} components)")
    ss, se, ahal = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]
    if ss != 0 or se != 63 or ahal != 0:
        raise ValueError("corrupt SOS segment (spectral selection of a sequential scan)")
    for c in range(ns):
        cs, tdta = seg[1 + 2 * c], seg[2 + 2 * c]
        if cs != comps[c]["id"]:
            raise ValueError("the scan's component order differs from the frame's")
        comps[c]["td"], comps[c]["ta"] = tdta >> 4, tdta & 15
    if nf == 3:
        ids = tuple(c["id"] for c in comps)
        if jfif:
            rgb = False
        elif adobe:
            rgb = adobe_transform == 0
        else:
            rgb = ids == (82, 71, 66)
        if rgb:
            raise ValueError("RGB-coded JPEG (Adobe transform 0 or component ids 'RGB') is not supported")
    hmax = max(c["h"] for c in comps)
    vmax = max(c["v"] for c in comps)
    for c in comps:
        if nf == 3 and (hmax % c["h"] or vmax % c["v"] or hmax // c["h"] > 2 or vmax // c["v"] > 2):
            fac = "x".join(f"{d['h']}x{d['v']}" for d in comps)
            raise ValueError(f"sampling factors {fac} are not supported (4:4:4, 4:2:2, 4:2:0 and 4:4:0 are)")
        if c["tq"] not in qt:
            raise ValueError(f"quantisation table {c['tq']} is not defined")
        for kind, key in (("DC", (0, c["td"])), ("AC", (1, c["ta"]))):
            if key not in dht:
                raise ValueError(f"{kind} Huffman table {key[1]} is not defined")
        if any(v > 15 for v in dht[(0, c["td"])][1]):
            raise ValueError("bad Huffman table (a DC symbol above 15)")
        c["q"] = qt[c["tq"]].copy()
        c["dc"], c["ac"] = dht[(0, c["td"])], dht[(1, c["ta"])]
    if nf == 3 and sum(c["h"] * c["v"] for c in comps) > 10:
        raise ValueError("corrupt SOF segment (more than 10 blocks per MCU)")
    if nf == 1:                       # a non-interleaved scan: one block per MCU whatever the SOF says
        comps[0]["h"] = comps[0]["v"] = 1
        hmax = vmax = 1
    return JpegHeader(W=frame["W"], H=frame["H"], ncomp=nf, comps=comps, Ri=Ri, scan=i + L, hmax=hmax, vmax=vmax)


def device_huff_table(bits, vals):
    """One Huffman table as the decoder reads it (HUFF_WORDS int32): a 9-bit lookahead table of (length << 8 |
    symbol) (0 = longer code), then per length 1..16 the largest code (-1 if none) and the offset from a code to its
    symbol's index, then the symbols."""
    lut = np.zeros(512, np.uint16)
    maxcode = np.full(18, -1, np.int32)
    valoff = np.zeros(18, np.int32)
    codes = huff_codes(bits, vals)
    p = 0
    for length in range(1, 17):
        n = bits[length - 1]
        if n:
            first = codes[p][1]
            valoff[length] = p - first
            maxcode[length] = codes[p + n - 1][1]
            if length <= 9:
                for j in range(n):
                    c = codes[p + j][1]
                    lut[c << (9 - length):(c + 1) << (9 - length)] = (length << 8) | codes[p + j][2]
        p += n
    v = np.zeros(256, np.uint8)
    v[:len(vals)] = vals
    return np.concatenate([lut.view(np.int32), maxcode, valoff, v.view(np.int32)])


def image_geometry(hd):
    """Per-component block grids and plane sizes of a parsed header: a list of dicts (h, v, bw, bh, dw, dh) where
    bw x bh is the component's block grid in the scan and dw x dh its downsampled size (jdinput.c)."""
    W, H, hmax, vmax = hd.W, hd.H, hd.hmax, hd.vmax
    mcux, mcuy = -(-W // (8 * hmax)), -(-H // (8 * vmax))
    out = []
    for c in hd.comps:
        dw, dh = -(-W * c["h"] // hmax), -(-H * c["v"] // vmax)
        if hd.ncomp == 1:
            bw, bh = -(-dw // 8), -(-dh // 8)
        else:
            bw, bh = mcux * c["h"], mcuy * c["v"]
        out.append(dict(h=c["h"], v=c["v"], bw=bw, bh=bh, dw=dw, dh=dh))
    return mcux, mcuy, out


def pack_batch(blobs):
    """Parse S streams and pack the decoder's inputs: dict(data uint8 (each image's entropy-coded data, back to
    back), desc int64 [S, DESC], huff int32 [S, 6, HUFF_WORDS], quant int32 [S, 3, 64], offsets int64 [S] (output
    byte offsets), shapes int64 [S, 2] (h, w), out_bytes).  Raises ValueError("image i: <reason>")."""
    S = len(blobs)
    desc = np.zeros((S, DESC), np.int64)
    huff = np.zeros((S, 6, HUFF_WORDS), np.int32)
    quant = np.zeros((S, 3, 64), np.int32)
    shapes = np.zeros((S, 2), np.int64)
    parts, pos, out = [], 0, 0
    for s, blob in enumerate(blobs):
        mv = memoryview(blob).cast("B")
        try:
            hd = parse_jpeg(mv)
        except ValueError as e:
            raise ValueError(f"image {s}: {e}") from None
        mcux, mcuy, geo = image_geometry(hd)
        d = desc[s]
        d[0], d[1], d[2] = pos, len(mv) - hd.scan, out
        d[3], d[4], d[5], d[6] = hd.W, hd.H, hd.ncomp, hd.Ri
        d[7], d[8] = mcux, mcuy
        d[9] = 1 if hd.ncomp == 1 else sum(g["h"] * g["v"] for g in geo)
        d[10] = sum(g["bw"] * g["bh"] for g in geo)
        d[11], d[12] = hd.hmax, hd.vmax
        first, comp_of, blk = 0, 0, 0
        for c, (g, comp) in enumerate(zip(geo, hd.comps)):
            d[16 + 8 * c:16 + 8 * c + 8] = [g["h"], g["v"], g["bw"], g["bh"], g["dw"], g["dh"], 0, first]
            first += g["bw"] * g["bh"]
            for _ in range(g["h"] * g["v"] if hd.ncomp == 3 else 1):
                comp_of |= c << (4 * blk)
                blk += 1
            huff[s, 2 * c] = device_huff_table(*comp["dc"])
            huff[s, 2 * c + 1] = device_huff_table(*comp["ac"])
            quant[s, c] = comp["q"].astype(np.int16)           # ISLOW_MULT_TYPE
        d[45] = comp_of
        parts.append(mv[hd.scan:])
        pos += len(mv) - hd.scan
        shapes[s] = hd.H, hd.W
        out += 3 * hd.H * hd.W
    data = np.empty(pos, np.uint8)
    p = 0
    for part in parts:
        data[p:p + len(part)] = np.frombuffer(part, np.uint8)
        p += len(part)
    offsets = np.concatenate([[0], np.cumsum(3 * shapes[:, 0] * shapes[:, 1])[:-1]]).astype(np.int64) if S else \
        np.zeros(0, np.int64)
    return dict(data=data, desc=desc, huff=huff, quant=quant, offsets=offsets, shapes=shapes, out_bytes=out)


STATUS = {1: "truncated stream (the entropy-coded data has no ending marker)",
          2: "unexpected marker after the scan (only one scan and EOI are supported)",
          3: "restart marker count does not match the restart interval",
          4: "invalid Huffman code",
          5: "MCU count mismatch (truncated or corrupt entropy-coded data)"}
