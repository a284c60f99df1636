"""CPU restatement of the batched PNG decoder (csrc/png.cu, DESIGN.md 4.23): deepi2p_b200/png.py's chunk walk, zlib
(the library libpng itself inflates with) for the inflate and the Adler-32, zlib.crc32 for the IDAT chunk CRCs, and
the five row filters undone in plain Python / numpy.  decode(blob) returns the HWC uint8 RGB image or raises
ValueError naming the reason, following the decoder's policy: never accept a stream OpenCV rejects, and also reject
inflated data longer than the image."""
import zlib

import numpy as np

from deepi2p_b200 import png as _png


def inflate(blob):
    """The parsed header and the inflated IDAT data of one stream (the chunk walk, the IDAT CRCs, inflate and
    Adler-32)."""
    hd = _png.parse_png(blob)
    b = memoryview(blob).cast("B")
    for off, n, crc in hd.idat:
        if zlib.crc32(b[off:off + n], zlib.crc32(b"IDAT")) != crc:
            raise ValueError("IDAT: CRC error")
    z = b"".join(bytes(b[off:off + n]) for off, n, _ in hd.idat)
    d = zlib.decompressobj(0)                     # the window the zlib header declares
    try:
        if hd.window == 32768:                    # no Deflate distance reaches beyond 32 KB
            raw = d.decompress(z)
        else:
            # zlib checks a distance against its window plus the output of the current call, so a call that yields
            # one byte makes it check against the declared window alone.
            raw, buf = bytearray(), z
            while not d.eof and len(raw) <= hd.H * (1 + 3 * hd.W):
                out = d.decompress(buf, 1)
                buf = d.unconsumed_tail
                raw += out
                if not out and not buf:
                    break
    except zlib.error as e:
        raise ValueError(f"IDAT: {e}") from None
    need = hd.H * (1 + 3 * hd.W)
    if len(raw) > need:
        raise ValueError("IDAT: more inflated data than the image holds")
    if len(raw) < need:
        raise ValueError("IDAT: not enough image data")
    if not d.eof:
        raise ValueError("IDAT: truncated zlib stream (Adler-32 missing)")
    return hd, raw


def unfilter(raw, h, w):
    """The filtered scanlines (h x (1 + 3 w) bytes) to HWC uint8 RGB: None, Sub, Up, Average and Paeth with 3 bytes
    per pixel, mod 256, the row above the first row and the pixel left of the first column being zero."""
    n = 3 * w
    rows = np.frombuffer(raw, np.uint8).reshape(h, n + 1)
    if (rows[:, 0] > 4).any():
        raise ValueError("bad adaptive filter value")
    out = np.zeros((h, n), np.uint8)
    prev = np.zeros(n, np.int64)
    for r in range(h):
        f, cur = int(rows[r, 0]), rows[r, 1:].astype(np.int64)
        if f == 0:
            line = cur
        elif f == 2:
            line = (cur + prev) & 255
        elif f == 1:
            line = cur.copy()
            for c in range(3):
                line[c::3] = np.cumsum(cur[c::3]) & 255
        else:
            line, up, x = [0] * n, prev.tolist(), cur.tolist()
            for i in range(n):
                a = line[i - 3] if i >= 3 else 0
                b = up[i]
                if f == 3:
                    p = (a + b) >> 1
                else:
                    c = up[i - 3] if i >= 3 else 0
                    q = a + b - c
                    pa, pb, pc = abs(q - a), abs(q - b), abs(q - c)
                    p = a if pa <= pb and pa <= pc else b if pb <= pc else c
                line[i] = (x[i] + p) & 255
            line = np.array(line, np.int64)
        out[r] = line
        prev = line
    return out.reshape(h, w, 3)


def decode(blob):
    hd, raw = inflate(blob)
    return unfilter(raw, hd.H, hd.W)
