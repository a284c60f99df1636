"""Host side of the batched PNG decoder (csrc/png.cu): the chunk walk, the header checks and the packing of the
concatenated IDAT payloads.

parse_png walks one stream's chunks the way libpng does for the inputs DESIGN.md 4.23 supports -- 8-bit truecolour
(colour type 2), not interlaced -- and raises ValueError with the reason for anything else.  It checks the CRC-32 of
the small critical chunks (IHDR, PLTE, IEND) itself; the IDAT CRCs and the Adler-32 of the inflated data are checked
on the device, so the bulk of the stream is never read twice on the host.  It needs only numpy and zlib, so
oracle_png/ and the CPU tests use it without the CUDA library.  imageprep.decode_png_batch is the public entry.
"""
import struct
import zlib

import numpy as np

SIGNATURE = b"\x89PNG\r\n\x1a\n"
DESC = 12                 # int64 slots of one image descriptor (the slot enum at the top of csrc/png.cu)
BPP_SLOT = 10             # descriptor slot of the bytes per pixel: 0 (RGB) or 1 (grey)
CHUNK = 4                 # int64 slots of one IDAT chunk record: image, data offset, length, expected CRC-32
ALIGN = 16                # each image's IDAT payload starts at a multiple of ALIGN in the packed data
MAX_SIDE = 1 << 20        # OpenCV's CV_IO_MAX_IMAGE_WIDTH / HEIGHT
MAX_PIXELS = 1 << 30      # OpenCV's CV_IO_MAX_IMAGE_PIXELS

# Bit depths PNG allows per colour type; every valid combination other than (2, 8) is "unsupported".
_DEPTHS = {0: (1, 2, 4, 8, 16), 2: (8, 16), 3: (1, 2, 4, 8), 4: (8, 16), 6: (8, 16)}
_KNOWN_CRITICAL = (b"IHDR", b"PLTE", b"IDAT", b"IEND")


class PngHeader(dict):
    """Attribute view of parse_png's result."""
    __getattr__ = dict.__getitem__


def parse_png(blob, grey=False):
    """Chunk structure of one PNG stream.  With grey=True the supported colour type is 8-bit greyscale (0) instead of
    8-bit truecolour (2).  Returns a PngHeader with W, H, window (the LZ77 window the zlib header
    declares, in bytes) and idat (a list of (payload offset in blob, payload length, expected CRC-32) of the IDAT
    chunks, in order).  Raises ValueError naming the reason for a stream outside the supported set or one libpng
    rejects before inflating: a bad signature, a truncated chunk, a bad IHDR, PLTE or IEND CRC, an unknown critical
    chunk, chunks out of order, IDAT chunks that are not consecutive, no IEND, or a bad zlib header."""
    b = memoryview(blob).cast("B")
    n = len(b)
    if n < 8 or bytes(b[:8]) != SIGNATURE:
        raise ValueError("not a PNG stream (bad signature)")
    i, hdr, idat, seen_idat, after_idat, seen_plte = 8, None, [], False, False, False
    while True:
        if i + 8 > n:
            raise ValueError("PNG input buffer is incomplete (no IEND chunk)")
        length, ctype = struct.unpack(">I4s", b[i:i + 8])
        if length > 0x7FFFFFFF:
            raise ValueError("chunk length exceeds 2^31 - 1")
        if i + 12 + length > n:
            raise ValueError("PNG input buffer is incomplete (truncated chunk)")
        data_off = i + 8
        crc = struct.unpack(">I", b[data_off + length:data_off + length + 4])[0]
        if not all(65 <= c <= 90 or 97 <= c <= 122 for c in ctype):
            raise ValueError(f"invalid chunk type {bytes(ctype)!r}")
        critical = ctype[0] & 0x20 == 0
        if hdr is None and ctype != b"IHDR":
            raise ValueError("missing IHDR before " + ctype.decode("latin-1"))
        if ctype == b"IDAT":
            if after_idat:
                raise ValueError("IDAT chunks are not consecutive")
            seen_idat = True
            idat.append((data_off, length, crc))
        else:
            after_idat = seen_idat
            if critical:
                if ctype not in _KNOWN_CRITICAL:
                    raise ValueError(f"unknown critical chunk {ctype.decode('latin-1')}")
                if zlib.crc32(b[i + 4:data_off + length]) != crc:
                    raise ValueError(f"{ctype.decode('latin-1')}: CRC error")
            if ctype == b"IHDR":
                if hdr is not None:
                    raise ValueError("IHDR: out of place")
                hdr = _ihdr(bytes(b[data_off:data_off + length]), grey)
            elif ctype == b"PLTE":
                if seen_idat or seen_plte or length % 3 or length == 0 or length > 768:
                    raise ValueError("PLTE: invalid or out of place")
                seen_plte = True
            elif ctype == b"IEND":
                if length:
                    raise ValueError("IEND: invalid length")
                break
        i = data_off + length + 4
    if not seen_idat:
        raise ValueError("no IDAT chunk")
    total = sum(l for _, l, _ in idat)
    head = bytearray()
    for off, l, _ in idat:
        head += b[off:off + min(l, 2 - len(head))]
        if len(head) == 2:
            break
    if len(head) < 2:
        raise ValueError("IDAT: truncated zlib header")
    cmf, flg = head
    if cmf & 15 != 8:
        raise ValueError("IDAT: unknown compression method")
    if cmf >> 4 > 7:
        raise ValueError("IDAT: invalid window size")
    if (cmf * 256 + flg) % 31:
        raise ValueError("IDAT: incorrect header check")
    if flg & 0x20:
        raise ValueError("IDAT: preset dictionary not supported")
    return PngHeader(W=hdr[0], H=hdr[1], window=1 << ((cmf >> 4) + 8), idat=idat, idat_bytes=total)


def _ihdr(d, grey=False):
    if len(d) != 13:
        raise ValueError("IHDR: invalid length")
    w, h, depth, ctype, comp, filt, interlace = struct.unpack(">IIBBBBB", d)
    if not (1 <= w <= 0x7FFFFFFF and 1 <= h <= 0x7FFFFFFF):
        raise ValueError(f"IHDR: invalid image size {w} x {h}")
    if depth not in _DEPTHS.get(ctype, ()):
        raise ValueError(f"IHDR: invalid colour type {ctype} with bit depth {depth}")
    if comp != 0 or filt != 0 or interlace > 1:
        raise ValueError("IHDR: invalid compression, filter or interlace method")
    if grey and (ctype, depth) != (0, 8):
        raise ValueError(f"unsupported colour type {ctype} with bit depth {depth} (only 8-bit grey is decoded here)")
    if not grey and (ctype, depth) != (2, 8):
        raise ValueError(f"unsupported colour type {ctype} with bit depth {depth} (only 8-bit RGB is decoded)")
    if interlace:
        raise ValueError("unsupported interlace method (Adam7)")
    if w > MAX_SIDE or h > MAX_SIDE or w * h > MAX_PIXELS:
        raise ValueError(f"image size {w} x {h} exceeds OpenCV's limits")
    return w, h


def pack_batch(blobs, grey=False):
    """Parse S streams (8-bit greyscale ones with grey=True, one output byte per pixel) and pack the decoder's inputs: dict(data uint8 (each image's concatenated IDAT payloads,
    ALIGN-aligned and zero-padded), desc int64 [S, DESC], chunks int64 [C, CHUNK], offsets int64 [S] (output byte
    offsets), shapes int64 [S, 2] (h, w), out_bytes, errors (a dict image -> reason of the streams the host already
    rejected; those images get empty descriptors and no output bytes))."""
    S = len(blobs)
    desc = np.zeros((S, DESC), np.int64)
    shapes = np.zeros((S, 2), np.int64)
    chunks, parts, errors, pos = [], [], {}, 0
    for s, blob in enumerate(blobs):
        mv = memoryview(blob).cast("B")
        try:
            hd = parse_png(mv, grey)
        except ValueError as e:
            errors[s] = str(e)
            desc[s, 7] = 1
            continue
        d = desc[s]
        d[0], d[1], d[3], d[4], d[6] = pos, hd.idat_bytes, hd.W, hd.H, hd.window.bit_length() - 1
        d[5], d[9], d[BPP_SLOT] = len(chunks), len(hd.idat), 1 if grey else 0
        p = pos
        for off, l, crc in hd.idat:
            chunks.append((s, p, l, crc))
            parts.append((p, mv[off:off + l]))
            p += l
        d[7] = 0
        shapes[s] = hd.H, hd.W
        pos += -(-(hd.idat_bytes + ALIGN) // ALIGN) * ALIGN          # at least ALIGN zero bytes of padding
    data = np.zeros(max(pos, ALIGN), np.uint8)
    for p, part in parts:
        data[p:p + len(part)] = np.frombuffer(part, np.uint8)
    sizes = (1 if grey else 3) * shapes[:, 0] * shapes[:, 1]
    offsets = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64) if S else np.zeros(0, np.int64)
    desc[:, 2] = offsets
    chunks = np.array(chunks, np.int64).reshape(-1, CHUNK)
    return dict(data=data, desc=desc, chunks=chunks, offsets=offsets, shapes=shapes, out_bytes=int(sizes.sum()),
                errors=errors)


# Per-image device status (csrc/png.cu, DIB_PNG_*), in the order the library reports them.
STATUS = {1: "IDAT: truncated zlib stream (not enough compressed data)",
          2: "IDAT: invalid block type",
          3: "IDAT: invalid stored block lengths",
          4: "IDAT: invalid code lengths set (over-subscribed or incomplete)",
          5: "IDAT: invalid code -- missing end-of-block",
          6: "IDAT: invalid bit length repeat (no previous length)",
          7: "IDAT: invalid bit length repeat (past HLIT + HDIST)",
          8: "IDAT: too many length or distance symbols",
          9: "IDAT: invalid literal/length code",
          10: "IDAT: invalid distance code",
          11: "IDAT: invalid distance too far back (before the start of the output)",
          12: "IDAT: invalid distance too far back (beyond the declared window)",
          13: "IDAT: more inflated data than the image holds",
          14: "IDAT: not enough image data",
          15: "IDAT: Adler-32 missing (truncated zlib trailer)",
          16: "IDAT: incorrect data check (Adler-32)",
          17: "IDAT: CRC error",
          18: "bad adaptive filter value"}
