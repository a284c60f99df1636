"""Writes tests/golden/png_small.npz: PNG streams with OpenCV 4.13's decision on each and its pixels.

Run from the repository root with opencv-python-headless 4.13 and Pillow installed:
    python tests/golden/make_png_golden.py

Arrays: names [N] str; streams uint8 (all streams back to back) with stream_lens int64 [N]; cv2_ok bool [N]
(cv2.imdecode returned an image); reject bool [N] (the decoder must reject: OpenCV rejects, the format is outside
the supported set, or the case is one of DESIGN.md 4.23's deliberate deviations); shapes int64 [N, 2] (h, w, 0 when rejected); pixels uint8 (the HWC RGB
images of the small accepted cases back to back, cv2.imdecode(..)[:, :, ::-1]) with pixel_lens int64 [N] (0 for
rejected and large cases); digests [N] str (SHA-256 of every accepted image's pixels).
"""
import hashlib
import io
import os
import struct
import sys
import zlib

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))

from deepi2p_b200.synthetic import encode_png, png_chunk, png_filter  # noqa: E402

LARGE = 1 << 16           # images with more pixels are stored as digests only
# Streams OpenCV accepts that the decoder rejects on purpose (DESIGN.md 4.23): inflated data longer than the image
# (libpng warns), and a distance beyond the declared window whose source lies in the row being inflated.
DEVIATIONS = ("extra_inflated", "dist_beyond_window_same_row")


def image(h, w, seed, smooth=False):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    img = np.stack([(xx * 3 + yy) % 256, (yy * 5 + 17) % 256, (xx * yy) % 256], -1).astype(np.int64)
    if smooth:
        img = np.stack([xx * 255 // max(w - 1, 1), yy * 255 // max(h - 1, 1), (xx + yy) * 127 // max(w + h, 1)], -1)
        band = slice(h // 2, h // 2 + 4)
        img[band] = rng.integers(0, 256, img[band].shape)
    else:
        img = img + rng.integers(0, 40, img.shape)
    return np.clip(img, 0, 255).astype(np.uint8)


class Bits:
    """A Deflate bit writer: values LSB first, Huffman codes MSB first."""

    def __init__(self):
        self.v, self.n = 0, 0

    def put(self, value, n):
        self.v |= (value & ((1 << n) - 1)) << self.n
        self.n += n

    def code(self, code, n):
        self.put(int(format(code, f"0{n}b")[::-1], 2), n)

    def align(self):
        self.n += -self.n % 8

    def bytes(self):
        return self.v.to_bytes((self.n + 7) // 8, "little")


def canonical(lens):
    """Deflate's canonical codes for a list of code lengths."""
    count = [0] * 16
    for l in lens:
        count[l] += 1
    count[0] = 0
    code, nxt = 0, [0] * 16
    for l in range(1, 16):
        code = (code + count[l - 1]) << 1
        nxt[l] = code
    out = []
    for l in lens:
        out.append(nxt[l] if l else None)
        if l:
            nxt[l] += 1
    return out


CLEN_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
CLEN_DEFAULT = [4] * 15 + [5, 5, 0, 0]          # complete: 15 / 16 + 2 / 32


def dynamic_header(bw, lit, dist, final=1, clen=CLEN_DEFAULT, seq=None, hlit=None):
    """A dynamic block header; seq is the list of code-length symbols (sym, extra, extra_bits), the plain lengths by
    default."""
    bw.put(final, 1)
    bw.put(2, 2)
    bw.put((hlit or len(lit)) - 257, 5)
    bw.put(len(dist) - 1, 5)
    bw.put(15, 4)
    for s in CLEN_ORDER:
        bw.put(clen[s], 3)
    codes = canonical(clen)
    for s, e, n in (seq if seq is not None else [(l, 0, 0) for l in list(lit) + list(dist)]):
        bw.code(codes[s], clen[s])
        if n:
            bw.put(e, n)


def fixed_lit(bw, sym):
    if sym < 144:
        bw.code(0x30 + sym, 8)
    elif sym < 256:
        bw.code(0x190 + sym - 144, 9)
    elif sym < 280:
        bw.code(sym - 256, 7)
    else:
        bw.code(0xC0 + sym - 280, 8)


def zwrap(deflate, raw, cmf=0x78, flg=0x01):
    return bytes([cmf, flg]) + deflate + struct.pack(">I", zlib.adler32(raw))


def png_of(w, h, zdata, **kw):
    return encode_png(np.zeros((h, w, 3), np.uint8), zdata=zdata, **kw)


def cases():
    out = []
    small = image(5, 7, 1)
    raw = png_filter(small, 0)

    import cv2
    base = image(23, 37, 2)
    for level in range(10):
        out.append((f"cv2_c{level}", cv2.imencode(".png", base[:, :, ::-1], [cv2.IMWRITE_PNG_COMPRESSION, level])[1].tobytes()))
    for sname in ("DEFAULT", "FILTERED", "HUFFMAN_ONLY", "RLE", "FIXED"):
        st = getattr(cv2, "IMWRITE_PNG_STRATEGY_" + sname)
        out.append((f"cv2_strategy_{sname.lower()}", cv2.imencode(".png", base[:, :, ::-1], [cv2.IMWRITE_PNG_STRATEGY, st])[1].tobytes()))
    from PIL import Image
    for kw, tag in (({}, "default"), ({"optimize": True}, "optimize"), ({"compress_level": 0}, "c0"),
                    ({"compress_level": 1}, "c1"), ({"compress_level": 9}, "c9")):
        buf = io.BytesIO()
        Image.fromarray(image(31, 45, 3)).save(buf, "PNG", **kw)
        out.append(("pil_" + tag, buf.getvalue()))
    rep = np.tile(image(20, 9, 4), (1, 5, 1))            # repeats 27 bytes apart and further
    for wbits in range(9, 16):
        out.append((f"zlib_wbits{wbits}", encode_png(rep, filters=0, level=9, wbits=wbits)))
    # zlib writes CINFO 1 for wbits 8 (a 256-byte window needs the 512-byte setting to encode); declare 8 by hand.
    z = zlib.compressobj(9, zlib.DEFLATED, 9)
    zd = z.compress(png_filter(rep[:, :8], 0)) + z.flush()
    out.append(("zlib_wbits8", encode_png(rep[:, :8], zdata=bytes([0x08, 0x1D]) + zd[2:])))
    z = zlib.compressobj(6)
    rows = png_filter(base, 1)
    zd = z.compress(rows[:300]) + z.flush(zlib.Z_FULL_FLUSH) + z.flush(zlib.Z_FULL_FLUSH) + z.compress(rows[300:]) + z.flush()
    out.append(("zlib_full_flush", encode_png(base, zdata=zd)))
    out.append(("zlib_level0", encode_png(base, filters=2, level=0)))
    out.append(("zlib_idat_1byte", encode_png(small, idat=1)))
    out.append(("zlib_idat_empty", encode_png(base, idat=[0, 5, 0, 0, 17, 0])))
    for f in range(5):
        out.append((f"zlib_filter{f}", encode_png(base, filters=f)))
    out.append(("zlib_filters_mixed", encode_png(base, filters=np.arange(23) % 5)))
    ties = np.zeros((9, 11, 3), np.uint8)
    ties[::2] = 7
    ties[:, ::3] = 200
    out.append(("zlib_paeth_ties", encode_png(ties, filters=4)))
    out.append(("zlib_paeth_flat", encode_png(np.full((6, 6, 3), 9, np.uint8), filters=4)))
    for h, w in ((1, 1), (1, 17), (17, 1), (3, 5), (2, 255), (33, 3)):
        out.append((f"size_{h}x{w}", encode_png(image(h, w, h * 100 + w), filters=np.arange(h) % 5)))
        out.append((f"cv2_size_{h}x{w}", cv2.imencode(".png", image(h, w, w)[:, :, ::-1])[1].tobytes()))
    for h, w in ((376, 1241), (375, 1242), (370, 1226)):
        out.append((f"kitti_{h}x{w}", cv2.imencode(".png", image(h, w, w, smooth=True)[:, :, ::-1])[1].tobytes()))
    # A stored block with all the data, then a dynamic block whose only code is end-of-block, of length 1 (an
    # incomplete set zlib accepts), and no distance code.
    bw = Bits()
    bw.put(0, 1)
    bw.put(0, 2)
    bw.align()
    bw.put(len(raw), 16)
    bw.put(~len(raw) & 0xFFFF, 16)
    pre = bw.bytes() + raw
    bw = Bits()
    lit = [0] * 256 + [1]
    dynamic_header(bw, lit, [0])
    bw.code(0, 1)
    out.append(("deflate_single_code", png_of(7, 5, zwrap(pre + bw.bytes(), raw))))
    # Accepted by OpenCV: bytes after the zlib stream, a bad ancillary CRC, extra inflated bytes.
    out.append(("after_stream_bytes", png_of(7, 5, zlib.compress(raw) + b"\x00\x11junk")))
    good = encode_png(small)
    i = good.index(b"tEXt") + 4 + len(b"Software\0deepi2p_b200")
    out.append(("ancillary_crc", good[:i] + bytes([good[i] ^ 1]) + good[i + 1:]))
    out.append(("extra_inflated", png_of(7, 5, zlib.compress(raw + b"\x00" * 5))))

    # Rejected by OpenCV.
    z = zlib.compress(raw)
    out.append(("bad_adler", png_of(7, 5, z[:-1] + bytes([z[-1] ^ 1]))))
    out.append(("no_adler", png_of(7, 5, z[:-4])))
    out.append(("short_one_byte", png_of(7, 5, zlib.compress(raw[:-1]))))
    i = good.index(b"IDAT")
    n = struct.unpack(">I", good[i - 4:i])[0]
    out.append(("idat_crc", good[:i + 4 + n] + bytes([good[i + 4 + n] ^ 1]) + good[i + 5 + n:]))
    out.append(("ihdr_crc", good[:29] + bytes([good[29] ^ 1]) + good[30:]))
    out.append(("no_iend", good[:-12]))
    out.append(("filter5", png_of(7, 5, zlib.compress(bytes([5]) + raw[1:]))))
    out.append(("truncated", png_of(7, 5, z[:len(z) // 2])))
    out.append(("zlib_cm7", png_of(7, 5, bytes([0x77, 0x09]) + z[2:])))
    out.append(("zlib_cinfo8", png_of(7, 5, bytes([0x88, 0x1C]) + z[2:])))
    out.append(("zlib_fcheck", png_of(7, 5, bytes([0x78, 0x02]) + z[2:])))
    out.append(("zlib_fdict", png_of(7, 5, bytes([0x78, 0x20]) + b"\0\0\0\1" + z[2:])))

    def block(fn):
        bw = Bits()
        fn(bw)
        return png_of(7, 5, zwrap(bw.bytes() + b"\0" * 8, raw))

    out.append(("deflate_btype3", block(lambda bw: (bw.put(1, 1), bw.put(3, 2)))))

    def stored_nlen(bw):
        bw.put(1, 1)
        bw.put(0, 2)
        bw.align()
        bw.put(len(raw), 16)
        bw.put(len(raw), 16)
    out.append(("deflate_stored_nlen", png_of(7, 5, zwrap(Bits.bytes(_run(stored_nlen)) + raw, raw))))
    eight = [8] * 256 + [8] + [0] * 29        # over-subscribed: 257 codes of length 8
    lit_ok = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 6
    out.append(("deflate_clen_oversub", block(lambda bw: dynamic_header(bw, lit_ok, [5] * 30, clen=[1] * 19))))
    out.append(("deflate_clen_incomplete", block(lambda bw: dynamic_header(
        bw, lit_ok, [5] * 30, clen=[4] * 15 + [6, 6, 0, 0], seq=[]))))
    out.append(("deflate_lit_oversub", block(lambda bw: dynamic_header(bw, eight, [5] * 30))))
    out.append(("deflate_lit_incomplete", block(lambda bw: dynamic_header(bw, [2] + [0] * 255 + [2], [1]))))
    out.append(("deflate_no_eob", block(lambda bw: dynamic_header(bw, [8] * 256 + [0], [1]))))
    out.append(("deflate_repeat_first", block(lambda bw: dynamic_header(bw, lit_ok, [5] * 30, seq=[(16, 0, 2)]))))
    out.append(("deflate_lens_overrun", block(lambda bw: dynamic_header(
        bw, [8] * 256 + [8], [1], seq=[(8, 0, 0)] * 255 + [(16, 3, 2)]))))
    out.append(("deflate_hlit287", block(lambda bw: dynamic_header(bw, lit_ok, [5] * 30, hlit=287, seq=[]))))

    def fixed(bw, syms):
        bw.put(1, 1)
        bw.put(1, 2)
        for kind, v, extra in syms:
            if kind == "lit":
                fixed_lit(bw, v)
            else:
                bw.code(v, 5)
            if extra:
                bw.put(*extra)
    out.append(("deflate_sym286", block(lambda bw: fixed(bw, [("lit", 0, None), ("lit", 286, None)]))))
    out.append(("deflate_dist30", block(lambda bw: fixed(bw, [("lit", 0, None), ("lit", 257, None),
                                                             ("dist", 30, None)]))))
    out.append(("deflate_dist_before_start", block(lambda bw: fixed(bw, [("lit", 0, None), ("lit", 257, None),
                                                                        ("dist", 4, (0, 1))]))))
    # A distance of 300 with a 256-byte window declared (CINFO 0): a 30 x 10 image of filter-0 rows.
    big = np.random.default_rng(5).integers(0, 256, (10, 91), dtype=np.uint8)
    big[:, 0] = 0
    big = big.reshape(-1)
    big[400:410] = big[100:110]
    bw = Bits()
    syms = [("lit", int(v), None) for v in big[:400]] + [("lit", 264, None), ("dist", 16, (43, 7))] + \
           [("lit", int(v), None) for v in big[410:]] + [("lit", 256, None)]
    fixed(bw, syms)
    out.append(("dist_beyond_window", png_of(30, 10, zwrap(bw.bytes(), big.tobytes(), 0x08, 0x1D))))
    # The same distance with its source in the row being inflated: a 1241 x 2 image of filter-0 rows, 10 bytes at
    # 1000 copied from 700.  libpng inflates one row per call and zlib checks a distance against its window plus the
    # current call's output, so OpenCV's decision here can differ from the case above.
    row = np.random.default_rng(6).integers(0, 256, (2, 1 + 3 * 1241), dtype=np.uint8)
    row[:, 0] = 0
    row = row.reshape(-1)
    row[1000:1010] = row[700:710]
    bw = Bits()
    syms = [("lit", int(v), None) for v in row[:1000]] + [("lit", 264, None), ("dist", 16, (43, 7))] + \
           [("lit", int(v), None) for v in row[1010:]] + [("lit", 256, None)]
    fixed(bw, syms)
    out.append(("dist_beyond_window_same_row", png_of(1241, 2, zwrap(bw.bytes(), row.tobytes(), 0x08, 0x1D))))
    # Unsupported headers.
    for tag, ctype, depth, il in (("rgba", 6, 8, 0), ("rgb16", 2, 16, 0), ("gray", 0, 8, 0), ("palette", 3, 8, 0),
                                  ("adam7", 2, 8, 1)):
        ihdr = struct.pack(">IIBBBBB", 7, 5, depth, ctype, 0, 0, il)
        s = b"\x89PNG\r\n\x1a\n" + png_chunk(b"IHDR", ihdr)
        if ctype == 3:
            s += png_chunk(b"PLTE", bytes(range(48)))
        s += png_chunk(b"IDAT", zlib.compress(b"\0" * 200)) + png_chunk(b"IEND", b"")
        out.append(("unsupported_" + tag, s))
    return out


def _run(fn):
    bw = Bits()
    fn(bw)
    return bw


def main():
    import cv2
    assert cv2.__version__.startswith("4.13"), cv2.__version__
    names, streams, lens, ok, reject, shapes, pixels, plens, digests = [], [], [], [], [], [], [], [], []
    for name, s in cases():
        img = cv2.imdecode(np.frombuffer(s, np.uint8), cv2.IMREAD_COLOR)
        good = img is not None
        names.append(name)
        streams.append(np.frombuffer(s, np.uint8))
        lens.append(len(s))
        ok.append(good)
        reject.append(not good or name in DEVIATIONS or name.startswith("unsupported_"))
        if good:
            rgb = np.ascontiguousarray(img[:, :, ::-1])
            shapes.append(rgb.shape[:2])
            digests.append(hashlib.sha256(rgb.tobytes()).hexdigest())
            keep = rgb.shape[0] * rgb.shape[1] <= LARGE
            pixels.append(rgb.reshape(-1) if keep else np.zeros(0, np.uint8))
            plens.append(rgb.size if keep else 0)
        else:
            shapes.append((0, 0))
            digests.append("")
            plens.append(0)
        print(f"{name:28s} {len(s):8d} B  cv2 {'accepts' if good else 'rejects'}")
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "png_small.npz")
    np.savez_compressed(path, names=np.array(names), streams=np.concatenate(streams),
                        stream_lens=np.array(lens, np.int64), cv2_ok=np.array(ok), reject=np.array(reject),
                        shapes=np.array(shapes, np.int64), pixels=np.concatenate(pixels) if pixels else
                        np.zeros(0, np.uint8), pixel_lens=np.array(plens, np.int64), digests=np.array(digests))
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
