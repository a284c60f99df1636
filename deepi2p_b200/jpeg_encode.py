"""Host side of the batched baseline JPEG encoder (csrc/jpeg_encode.cu): the quantisation and Huffman tables, the
image geometry and the marker segments around the entropy-coded data.

The stream is what OpenCV 4.13's cv2.imencode(".jpg", bgr, [IMWRITE_JPEG_QUALITY, q]) writes through libjpeg-turbo
3.1 with its defaults: SOI, APP0 JFIF 1.01 (density 1:1, no unit), DQT 0 and DQT 1 (each its own marker, 8-bit
entries in zig-zag order), SOF0 (Y 2x2 on table 0, Cb and Cr 1x1 on table 1: 4:2:0), DHT DC0, AC0, DC1, AC1 (the
Annex K.3 tables), SOS, the entropy-coded data, EOI.  No restart markers, no optimised Huffman tables.  It needs only
numpy, so oracle_oxford_images/ and the CPU tests use it without the CUDA library.  imageprep.encode_jpeg_batch is
the public entry.
"""
import struct

import numpy as np

from .jpeg import ZIGZAG

# Annex K.1 tables in natural (row-major) order (jcparam.c std_luminance_quant_tbl / std_chrominance_quant_tbl).
STD_LUMA_Q = np.array([
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
    14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99], dtype=np.int64)
STD_CHROMA_Q = np.array([
    17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
    47, 66, 99, 99, 99, 99, 99, 99] + [99] * 32, dtype=np.int64)

# Annex K.3 Huffman tables (jstdhuff.c): bits[1..16] and the symbols in code order.
DC_LUMA = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12)))
DC_CHROMA = ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))
AC_LUMA = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7D], [
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07,
    0x22, 0x71, 0x14, 0x32, 0x81, 0x91, 0xA1, 0x08, 0x23, 0x42, 0xB1, 0xC1, 0x15, 0x52, 0xD1, 0xF0,
    0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0A, 0x16, 0x17, 0x18, 0x19, 0x1A, 0x25, 0x26, 0x27, 0x28,
    0x29, 0x2A, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3A, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49,
    0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5A, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69,
    0x6A, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7A, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89,
    0x8A, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9A, 0xA2, 0xA3, 0xA4, 0xA5, 0xA6, 0xA7,
    0xA8, 0xA9, 0xAA, 0xB2, 0xB3, 0xB4, 0xB5, 0xB6, 0xB7, 0xB8, 0xB9, 0xBA, 0xC2, 0xC3, 0xC4, 0xC5,
    0xC6, 0xC7, 0xC8, 0xC9, 0xCA, 0xD2, 0xD3, 0xD4, 0xD5, 0xD6, 0xD7, 0xD8, 0xD9, 0xDA, 0xE1, 0xE2,
    0xE3, 0xE4, 0xE5, 0xE6, 0xE7, 0xE8, 0xE9, 0xEA, 0xF1, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8,
    0xF9, 0xFA])
AC_CHROMA = ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77], [
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71,
    0x13, 0x22, 0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xA1, 0xB1, 0xC1, 0x09, 0x23, 0x33, 0x52, 0xF0,
    0x15, 0x62, 0x72, 0xD1, 0x0A, 0x16, 0x24, 0x34, 0xE1, 0x25, 0xF1, 0x17, 0x18, 0x19, 0x1A, 0x26,
    0x27, 0x28, 0x29, 0x2A, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3A, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
    0x49, 0x4A, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5A, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68,
    0x69, 0x6A, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7A, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87,
    0x88, 0x89, 0x8A, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9A, 0xA2, 0xA3, 0xA4, 0xA5,
    0xA6, 0xA7, 0xA8, 0xA9, 0xAA, 0xB2, 0xB3, 0xB4, 0xB5, 0xB6, 0xB7, 0xB8, 0xB9, 0xBA, 0xC2, 0xC3,
    0xC4, 0xC5, 0xC6, 0xC7, 0xC8, 0xC9, 0xCA, 0xD2, 0xD3, 0xD4, 0xD5, 0xD6, 0xD7, 0xD8, 0xD9, 0xDA,
    0xE2, 0xE3, 0xE4, 0xE5, 0xE6, 0xE7, 0xE8, 0xE9, 0xEA, 0xF2, 0xF3, 0xF4, 0xF5, 0xF6, 0xF7, 0xF8,
    0xF9, 0xFA])

MAX_SIDE = 65500          # libjpeg's JPEG_MAX_DIMENSION
BLOCKS_PER_MCU = 6        # 4:2:0: four Y blocks, then Cb, then Cr
MAX_BLOCK_BYTES = 208     # an upper bound of one block's entropy-coded bytes before stuffing (max_block_bits / 8)


def max_block_bits():
    """The longest code a block can take with the standard tables: an 11-bit DC category and 63 AC coefficients of
    category 10 with the longest run-0 / size-10 code, both on the longer of the two tables."""
    dc = max(l for t in (DC_LUMA, DC_CHROMA) for l, _ in derived_table(*t).values()) + 11
    ac = max(l for t in (AC_LUMA, AC_CHROMA) for l, _ in derived_table(*t).values()) + 10
    return dc + 63 * ac


def quality_scaling(quality):
    """jcparam.c jpeg_quality_scaling: 1..100 -> the percentage the Annex K tables are scaled by."""
    q = int(quality)
    q = 1 if q <= 0 else 100 if q > 100 else q
    return 5000 // q if q < 50 else 200 - 2 * q


def quant_tables(quality):
    """jpeg_set_quality(cinfo, quality, force_baseline=TRUE): the two tables (natural order, int64 [2, 64]), each
    entry (basic * scale + 50) / 100 clamped to 1..255."""
    scale = quality_scaling(quality)
    out = []
    for basic in (STD_LUMA_Q, STD_CHROMA_Q):
        t = (basic * scale + 50) // 100
        out.append(np.clip(t, 1, 255))
    return np.stack(out).astype(np.int64)


def derived_table(bits, vals):
    """jchuff.c jpeg_make_c_derived_tbl: symbol -> (code length, code)."""
    out, code, p = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            out[vals[p]] = (length, code)
            code += 1
            p += 1
        code <<= 1
    return out


def device_tables():
    """The encoder's Huffman tables as one int32 array [4, 256] of (length << 16) | code per symbol (0: no code), in
    the order DC luma, AC luma, DC chroma, AC chroma."""
    t = np.zeros((4, 256), np.int32)
    for i, spec in enumerate((DC_LUMA, AC_LUMA, DC_CHROMA, AC_CHROMA)):
        for sym, (l, c) in derived_table(*spec).items():
            t[i, sym] = (l << 16) | c
    return t


def geometry(h, w):
    """Block geometry of an h x w 4:2:0 image: MCU columns and rows (16 x 16 pixels each), luma blocks per row and
    column (ceil(w / 8), ceil(h / 8)) and the number of coded blocks (six per MCU, dummy blocks included)."""
    mx, my = -(-w // 16), -(-h // 16)
    return dict(mcux=mx, mcuy=my, ybx=-(-w // 8), yby=-(-h // 8), blocks=BLOCKS_PER_MCU * mx * my)


def check_shape(h, w, what):
    if not (1 <= h <= MAX_SIDE and 1 <= w <= MAX_SIDE):
        raise ValueError(f"{what}: size {h} x {w} is outside 1..{MAX_SIDE} per side")


def _segment(marker, payload):
    return struct.pack(">BBH", 0xFF, marker, len(payload) + 2) + payload


def header(h, w, quality):
    """SOI .. SOS of the stream for an h x w image at `quality`."""
    q = quant_tables(quality)
    parts = [b"\xFF\xD8", _segment(0xE0, b"JFIF\x00\x01\x01\x00" + struct.pack(">HH", 1, 1) + b"\x00\x00")]
    for i in range(2):
        parts.append(_segment(0xDB, bytes([i]) + bytes(int(v) for v in q[i][ZIGZAG])))
    parts.append(_segment(0xC0, struct.pack(">BHHB", 8, h, w, 3) + bytes([1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1])))
    for cls_id, (bits, vals) in ((0x00, DC_LUMA), (0x10, AC_LUMA), (0x01, DC_CHROMA), (0x11, AC_CHROMA)):
        parts.append(_segment(0xC4, bytes([cls_id]) + bytes(bits) + bytes(vals)))
    parts.append(_segment(0xDA, bytes([3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0])))
    return b"".join(parts)


EOI = b"\xFF\xD9"
