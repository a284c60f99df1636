"""The image side of classifier batches on the GPU: the loaders' row cut, cv2.resize(INTER_LINEAR), crop, torchvision
ColorJitter on a PIL image, column flip, CHW float conversion and the K updates (data/kitti_pc_img_pose_loader.py:
326-349,360-362,439-440, data/oxford_pc_img_pose_loader.py:238-259,300-301,368, and the same steps of the nuScenes
loader), for S samples at once and bit for bit against cv2 and Pillow.

pack_images packs ragged HWC uint8 frames into one device buffer, and decode_jpeg_batch / read_jpeg_batch decode the
loaders' JPEG frames (Image.open(path).convert("RGB"), bit for bit; csrc/jpeg.cu, DESIGN.md 4.19) into the same
buffer on the device, and decode_png_batch / read_png_batch do the same for KITTI's official PNG frames
(cv2.imread(path)[:, :, ::-1], bit for bit; csrc/png.cu, DESIGN.md 4.23); decode_grey_png_batch decodes 8-bit grey
PNGs (the RobotCar Bayer mosaics) and encode_jpeg_batch encodes pack_images' frames as baseline JPEG, bit for bit with
cv2.imencode (csrc/jpeg_encode.cu, DESIGN.md 4.25); image_params draws the per-sample crop offsets and
jitter on the host; assemble_images runs csrc/imageprep.cu and composes K in fp64.  kitti_image_args /
oxford_image_args / nuscenes_image_args are the loaders' options (nuScenes: crop_top_rows=100, img_scale=0.2, 160 x
320, jitter_prob=0.5).  augment_img is a host drop-in for the loaders' augment_img that works on current torchvision.
DESIGN.md 4.13 states the contract.  There is no CPU fallback.
"""
import numpy as np
import torch

from . import _native
from . import jpeg as _jpeg
from . import jpeg_encode as _jpege
from . import png as _png
from .assemble import MODES
from ._native import _ptr, _require_cuda, _stream_ptr, _workspace
from .frustum import _ws_cache

_JPEGE_DESC = 8                   # include/deepi2p_b200.h DIB_JPEGE_DESC
IMAGE_PARAMS = 16                 # include/deepi2p_b200.h DIB_IMAGE_PARAMS and the DIB_IMG_* slots below
_H, _W, _ROW0, _ROWS, _DH, _DW, _DY, _DX, _FLIP, _JITTER, _ORDER, _SHIFT = 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 14
JITTER_RANGES = dict(brightness=(0.8, 1.2), contrast=(0.8, 1.2), saturation=(0.8, 1.2), hue=(-0.1, 0.1))


def kitti_image_args():
    """kitti/options.py: cut 50 top rows, scale 0.5, 160 x 512; every train sample is jittered."""
    return dict(img_H=160, img_W=512, img_scale=0.5, crop_top_rows=50, crop_bottom_rows=0, jitter_prob=1.0)


def oxford_image_args():
    """oxford/options.py: no row cut, scale 0.5, 384 x 640; a train sample is jittered with probability 1/2."""
    return dict(img_H=384, img_W=640, img_scale=0.5, crop_top_rows=0, crop_bottom_rows=0, jitter_prob=0.5)


def nuscenes_image_args():
    """nuscenes_t/options.py: cut 100 top rows, scale 0.2, 160 x 320; a train sample is jittered with probability
    1/2."""
    return dict(img_H=160, img_W=320, img_scale=0.2, crop_top_rows=100, crop_bottom_rows=0, jitter_prob=0.5)


def resize_dims(h, w, s):
    """The loaders' cv2.resize target (dh, dw) = (int(round(h s)), int(round(w s))) (Python's ties-to-even round)."""
    return int(round(h * s)), int(round(w * s))


def hue_shift(hue):
    """torchvision adjust_hue's uint8 shift np.int32(hue * 255).astype(np.uint8): -0.1 -> 231, 0.1 -> 25."""
    return int(np.int32(hue * 255)) & 255


def _rng(rng):
    return rng if isinstance(rng, np.random.Generator) else np.random.default_rng(rng)


def _draw_jitter(rng, S, brightness, contrast, saturation, hue):
    """ColorJitter.get_params for S samples: a random order of the four steps and float32 factors (b, c, s, hue)."""
    order = np.stack([rng.permutation(4) for _ in range(S)]) if S else np.zeros((0, 4), np.int64)
    cols = [rng.uniform(lo, hi, S) for lo, hi in (brightness, contrast, saturation, hue)]
    return order.astype(np.int32), np.stack(cols, -1).astype(np.float32).reshape(S, 4)


def pack_images(images, device="cuda"):
    """Host frames -> assemble_images' `images`: a list of h x w x 3 uint8 arrays (h, w may differ).  Returns dict(data
    uint8 [bytes] on `device`, offsets int64 [S], shapes int64 [S,2] (h, w) on the host)."""
    arrs = [np.ascontiguousarray(a) for a in images]
    for s, a in enumerate(arrs):
        if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3 or a.shape[0] < 1 or a.shape[1] < 1:
            raise ValueError(f"image {s} must be an h x w x 3 uint8 array (got {a.dtype} {a.shape})")
    sizes = np.array([a.size for a in arrs], dtype=np.int64)
    offsets = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64) if len(arrs) else np.zeros(0, np.int64)
    flat = np.concatenate([a.reshape(-1) for a in arrs]) if arrs else np.zeros(0, np.uint8)
    return dict(data=torch.from_numpy(flat).to(torch.device(device)), offsets=offsets,
                shapes=np.array([a.shape[:2] for a in arrs], dtype=np.int64).reshape(-1, 2))


JPEG_WINDOW_BITS = 8192          # bit length of the windows the Huffman decoder synchronises (csrc/jpeg.cu)


def decode_jpeg_batch(blobs, device="cuda", stream=None, *, _window_bits=None):
    """Decode S JPEG streams (bytes-like) on the GPU into pack_images' dict: data uint8 [sum 3 h w] on `device`
    (HWC RGB, each image equal to np.asarray(PIL.Image.open(BytesIO(b)).convert("RGB")) on Pillow 12.2 /
    libjpeg-turbo), offsets int64 [S], shapes int64 [S,2] (h, w), so assemble_images takes it as it is.

    Supported: 8-bit baseline / extended sequential Huffman, one scan of 1 (grey, replicated to RGB) or 3 (YCbCr)
    components, 4:4:4 / 4:2:2 / 4:2:0 / 4:4:0, any Huffman tables, restart intervals, any size.  Anything else --
    progressive, arithmetic, lossless, 12-bit, multi-scan, CMYK / YCCK, RGB-coded, other sampling factors -- and a
    truncated or corrupt entropy-coded segment raise ValueError("image i: <reason>"); the whole call raises, and no
    output is returned for any image.  Corrupt data that still decodes validly is not detected.  The call waits for
    the decode to finish (the per-image status is read back).  _window_bits is a test hook: the synchronisation
    window length in bits."""
    _require_cuda()
    lib = _native.load()
    dev = torch.device(device)
    S = len(blobs)
    pk = _jpeg.pack_batch(blobs)
    with torch.cuda.device(dev), torch.cuda.stream(stream):
        out = torch.empty(pk["out_bytes"], dtype=torch.uint8, device=dev)
        if S:
            wb = int(_window_bits) if _window_bits is not None else JPEG_WINDOW_BITS
            sp = _stream_ptr(stream)
            data = torch.from_numpy(pk["data"]).to(dev) if pk["data"].size else torch.zeros(1, dtype=torch.uint8, device=dev)
            huff = torch.from_numpy(pk["huff"]).to(dev, non_blocking=True)
            quant = torch.from_numpy(pk["quant"]).to(dev, non_blocking=True)
            status = torch.zeros((S, 2), dtype=torch.int32, device=dev)
            desc = np.ascontiguousarray(pk["desc"])
            nws = lib.jpeg_decode_workspace_bytes(desc.ctypes.data, S, pk["data"].size, wb)
            if nws == 0:
                raise _native.NativeError("jpeg_decode_workspace_bytes rejected the batch")
            ws = _workspace(_ws_cache, nws, dev, stream)
            rc = lib.jpeg_decode_batch_u8(_ptr(data), pk["data"].size, desc.ctypes.data, _ptr(huff), _ptr(quant), S, wb,
                                          _ptr(out), out.numel(), _ptr(status), _ptr(ws), ws.numel(), sp)
            _native.check(rc, "jpeg_decode")
            st = status.cpu().numpy()
            bad = np.flatnonzero(st[:, 0])
            if bad.size:
                i = int(bad[0])
                raise ValueError(f"image {i}: {_jpeg.STATUS.get(int(st[i, 0]), f'status {int(st[i, 0])}')}")
            decode_jpeg_batch.last_rounds = st[:, 1].copy()
    return dict(data=out, offsets=pk["offsets"], shapes=pk["shapes"])


decode_jpeg_batch.last_rounds = np.zeros(0, np.int32)


def read_jpeg_batch(paths, device="cuda", stream=None):
    """The loaders' Image.open(path).convert("RGB") for S JPEG files: reads the files on the host and decodes them
    with decode_jpeg_batch."""
    blobs = []
    for p in paths:
        with open(p, "rb") as f:
            blobs.append(f.read())
    return decode_jpeg_batch(blobs, device=device, stream=stream)


def decode_png_batch(blobs, device="cuda", stream=None):
    """Decode S PNG streams (bytes-like) on the GPU into pack_images' dict: data uint8 [sum 3 h w] on `device` (HWC
    RGB, each image equal to cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)[:, :, ::-1] on OpenCV 4.13),
    offsets int64 [S], shapes int64 [S,2] (h, w), so assemble_images takes it as it is.

    Supported: 8-bit truecolour (colour type 2), not interlaced, from 1 x 1 up to OpenCV's limits (2^20 per side,
    2^30 pixels); the zlib stream split over any number of IDAT chunks (empty ones included), stored, fixed and
    dynamic Deflate blocks, any declared window, all five row filters; ancillary chunks are skipped (a bad CRC on one is ignored, as libpng does).  Other colour types,
    bit depths and Adam7 raise ValueError("image i: unsupported ...").  Every stream OpenCV rejects raises too: a bad
    signature, chunk structure or critical-chunk CRC, a bad zlib header, corrupt or truncated Deflate data, a bad
    Adler-32, too little image data or a filter byte above 4.  Beyond OpenCV, a stream whose inflated data is longer
    than the image or that uses a distance beyond its declared window is rejected (DESIGN.md 4.23).  The error names
    the first bad image, ValueError("image i: <reason>"), and no output is returned for any image.  The call waits for
    the decode to finish (the per-image status is read back)."""
    return _decode_png(blobs, device, stream, grey=False)


def decode_grey_png_batch(blobs, device="cuda", stream=None):
    """Decode S 8-bit greyscale PNG streams (bytes-like; the RobotCar stereo Bayer mosaics) on the GPU: dict(data
    uint8 [sum h w] on `device` (image s is h x w, row-major, at offsets[s] and equal to
    np.asarray(PIL.Image.open(BytesIO(b))), mode "L"), offsets int64 [S], shapes int64 [S,2] (h, w)).  Supported:
    colour type 0 with bit depth 8, not interlaced, with everything else decode_png_batch accepts about the chunks,
    the zlib stream and the filters; any other colour type or depth, and every stream decode_png_batch would reject,
    raise ValueError("image i: <reason>") for the first bad image.  The call waits for the decode to finish."""
    return _decode_png(blobs, device, stream, grey=True)


def _decode_png(blobs, device, stream, grey):
    _require_cuda()
    lib = _native.load()
    dev = torch.device(device)
    S = len(blobs)
    pk = _png.pack_batch(blobs, grey=grey)
    bad = dict(pk["errors"])
    with torch.cuda.device(dev), torch.cuda.stream(stream):
        out = torch.empty(pk["out_bytes"], dtype=torch.uint8, device=dev)
        if S and len(bad) < S:
            sp = _stream_ptr(stream)
            data = torch.from_numpy(pk["data"]).to(dev)
            status = torch.empty((S, 4), dtype=torch.int32, device=dev)
            desc = np.ascontiguousarray(pk["desc"])
            chunks = np.ascontiguousarray(pk["chunks"])
            nws = lib.png_decode_workspace_bytes(desc.ctypes.data, S, chunks.ctypes.data, len(chunks), data.numel())
            if nws == 0:
                raise _native.NativeError("png_decode_workspace_bytes rejected the batch")
            ws = _workspace(_ws_cache, nws, dev, stream)
            rc = lib.png_decode_batch_u8(_ptr(data), data.numel(), desc.ctypes.data, S, chunks.ctypes.data,
                                         len(chunks), _ptr(out), out.numel(), _ptr(status), _ptr(ws), ws.numel(), sp)
            _native.check(rc, "png_decode")
            st = status.cpu().numpy()
            for i in np.flatnonzero(st.any(1)):
                code = int(st[i][np.flatnonzero(st[i])[0]])
                bad.setdefault(int(i), _png.STATUS.get(code, f"status {code}"))
    if bad:
        i = min(bad)
        raise ValueError(f"image {i}: {bad[i]}")
    return dict(data=out, offsets=pk["offsets"], shapes=pk["shapes"])


def read_png_batch(paths, device="cuda", stream=None):
    """cv2.imread(path)[:, :, ::-1] for S PNG files (the frames kitti_png_to_npy.py converts): reads the files on the
    host and decodes them with decode_png_batch."""
    blobs = []
    for p in paths:
        with open(p, "rb") as f:
            blobs.append(f.read())
    return decode_png_batch(blobs, device=device, stream=stream)


def encode_jpeg_batch(images, quality=95, stream=None):
    """Encode pack_images' frames (dict: data uint8 on a CUDA device, HWC RGB, offsets, shapes) as baseline JPEG on the
    GPU.  Returns a list of S bytes objects, item s equal to cv2.imencode(".jpg", rgb_s[:, :, ::-1],
    [cv2.IMWRITE_JPEG_QUALITY, quality])[1].tobytes() on OpenCV 4.13 / libjpeg-turbo 3.1: 4:2:0, islow DCT, the Annex K
    tables scaled to `quality` (1..100, baseline-clamped), standard Huffman tables, no restart markers, any size from
    1 x 1 to 65500 per side (DESIGN.md 4.25).  The call waits: the per-image sizes are read back once before the
    stuffed bytes are packed, then the bytes are copied to the host."""
    _require_cuda()
    lib = _native.load()
    q = int(quality)
    if not 1 <= q <= 100:
        raise ValueError(f"quality must be in 1..100 (got {quality})")
    data = images["data"]
    if not (isinstance(data, torch.Tensor) and data.is_cuda and data.dtype == torch.uint8 and data.dim() == 1):
        raise ValueError("images['data'] must be a 1-D uint8 CUDA tensor (pack_images)")
    shapes = np.asarray(images["shapes"], dtype=np.int64).reshape(-1, 2)
    offsets = np.asarray(images["offsets"], dtype=np.int64).reshape(-1)
    S = shapes.shape[0]
    if offsets.shape != (S,):
        raise ValueError("images needs one offset per shape")
    for s in range(S):
        _jpege.check_shape(int(shapes[s, 0]), int(shapes[s, 1]), f"image {s}")
        if offsets[s] < 0 or offsets[s] + 3 * shapes[s, 0] * shapes[s, 1] > data.numel():
            raise ValueError(f"image {s}: lies outside images['data']")
    if S == 0:
        return []
    desc = np.zeros((S, _JPEGE_DESC), np.int64)
    desc[:, 0], desc[:, 1], desc[:, 2] = offsets, shapes[:, 0], shapes[:, 1]
    quant = np.ascontiguousarray(_jpege.quant_tables(q), dtype=np.int32)
    huff = np.ascontiguousarray(_jpege.device_tables())
    dev = data.device
    with torch.cuda.device(dev), torch.cuda.stream(stream):
        sp = _stream_ptr(stream)
        nws = lib.jpeg_encode_workspace_bytes(desc.ctypes.data, S)
        if nws == 0:
            raise _native.NativeError("jpeg_encode_workspace_bytes rejected the batch")
        ws = _workspace(_ws_cache, nws, dev, stream)
        counts = torch.empty((S, 2), dtype=torch.int64, device=dev)
        rc = lib.jpeg_encode_entropy_u8(_ptr(data), data.numel(), desc.ctypes.data, S, quant.ctypes.data,
                                        huff.ctypes.data, _ptr(counts), _ptr(ws), ws.numel(), sp)
        _native.check(rc, "jpeg_encode_entropy")
        n = counts.cpu().numpy()
        sizes = n[:, 0] + n[:, 1]
        out_off = np.ascontiguousarray(np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64))
        out = torch.empty(max(int(sizes.sum()), 1), dtype=torch.uint8, device=dev)
        rc = lib.jpeg_encode_stuff_u8(desc.ctypes.data, S, out_off.ctypes.data, _ptr(out), out.numel(), _ptr(ws),
                                      ws.numel(), sp)
        _native.check(rc, "jpeg_encode_stuff")
        host = out.cpu().numpy()
    headers = {}
    for h, w in shapes:
        if (h, w) not in headers:
            headers[h, w] = _jpege.header(int(h), int(w), q)
    return [b"".join((headers[h, w], host[o:o + z].data, _jpege.EOI)) for (h, w), o, z in zip(shapes, out_off, sizes)]


def image_params(shapes, mode, rng=None, img_H=160, img_W=512, img_scale=0.5, crop_top_rows=0, crop_bottom_rows=0,
                 jitter_prob=1.0, **ranges):
    """The loaders' per-sample image draws for frames of `shapes` ([S,2] (h, w)): `train` crops at dx ~ U{0..dw-W},
    dy ~ U{0..dh-H} and jitters with probability jitter_prob (order and factors as ColorJitter.get_params draws them
    from JITTER_RANGES, overridable by brightness= / contrast= / saturation= / hue=); other modes crop centred and do
    not jitter.  rng: a numpy Generator or a seed; the draws match the loaders in distribution.  Returns dict(row0,
    rows, dh, dw, dy, dx [S] int64, jitter [S] bool, order [S,4] int32, factors [S,4] float32 (b, c, s, hue), scale,
    img_H, img_W)."""
    if mode not in MODES:
        raise ValueError(f"mode must be one of {MODES} (got {mode!r})")
    bad = set(ranges) - set(JITTER_RANGES)
    if bad:
        raise TypeError(f"unknown jitter ranges {sorted(bad)}")
    rg = {**JITTER_RANGES, **ranges}
    s = float(img_scale)
    if not 0.0 < s <= 1.0:
        raise ValueError(f"img_scale must be in (0, 1] (got {img_scale}); upscaling is not supported")
    H, W = int(img_H), int(img_W)
    if H < 1 or W < 1:
        raise ValueError(f"img_H and img_W must be positive (got {img_H}, {img_W})")
    if not 0.0 <= jitter_prob <= 1.0:
        raise ValueError(f"jitter_prob must be in [0, 1] (got {jitter_prob})")
    shapes = np.asarray(shapes, dtype=np.int64).reshape(-1, 2)
    S = shapes.shape[0]
    top, bottom = int(crop_top_rows), int(crop_bottom_rows)
    if top < 0 or bottom < 0:
        raise ValueError("crop_top_rows and crop_bottom_rows must be >= 0")
    rows = shapes[:, 0] - top - bottom
    if S and rows.min() < 1:
        raise ValueError(f"the row cut ({top} top, {bottom} bottom) leaves no row of a {shapes[rows.argmin(), 0]}-row "
                         "frame")
    dims = np.array([resize_dims(r, w, s) for r, w in zip(rows, shapes[:, 1])], dtype=np.int64).reshape(S, 2)
    small = (dims[:, 0] < H) | (dims[:, 1] < W)
    if small.any():
        i = int(np.argmax(small))
        raise ValueError(f"sample {i}: the resized image {dims[i, 0]} x {dims[i, 1]} is smaller than the {H} x {W} "
                         "output")
    rng = _rng(rng)
    if mode == "train":
        dx = np.array([rng.integers(0, dw - W + 1) for dw in dims[:, 1]], dtype=np.int64).reshape(S)
        dy = np.array([rng.integers(0, dh - H + 1) for dh in dims[:, 0]], dtype=np.int64).reshape(S)
        jitter = rng.random(S) < jitter_prob
        order, factors = _draw_jitter(rng, S, rg["brightness"], rg["contrast"], rg["saturation"], rg["hue"])
    else:
        dx = (dims[:, 1] - W) // 2
        dy = (dims[:, 0] - H) // 2
        jitter = np.zeros(S, dtype=bool)
        order = np.tile(np.arange(4, dtype=np.int32), (S, 1))
        factors = np.tile(np.array([1, 1, 1, 0], np.float32), (S, 1))
    return dict(row0=np.full(S, top, np.int64), rows=rows, dh=dims[:, 0], dw=dims[:, 1], dy=dy, dx=dx,
                jitter=jitter, order=order, factors=factors, scale=s, img_H=H, img_W=W)


def camera_K(K, row0, scale, dx, dy):
    """The loaders' K updates in fp64 for [S,3,3] K: camera_matrix_cropping(dy=row0), camera_matrix_scaling(scale),
    camera_matrix_cropping(dx, dy); scale is one value or one per sample."""
    K = np.array(K, dtype=np.float64)
    K[:, 1, 2] -= np.asarray(row0, dtype=np.float64)
    K = np.asarray(scale, dtype=np.float64).reshape(-1, 1, 1) * K
    K[:, 2, 2] = 1.0
    K[:, 0, 2] -= np.asarray(dx, dtype=np.float64)
    K[:, 1, 2] -= np.asarray(dy, dtype=np.float64)
    return K


def _pack_params(shapes, p, flip):
    S = shapes.shape[0]
    P = np.zeros((S, IMAGE_PARAMS), dtype=np.int32)
    P[:, _H], P[:, _W] = shapes[:, 0], shapes[:, 1]
    for slot, key in ((_ROW0, "row0"), (_ROWS, "rows"), (_DH, "dh"), (_DW, "dw"), (_DY, "dy"), (_DX, "dx")):
        v = np.asarray(p[key], dtype=np.int64).reshape(-1)
        if v.shape != (S,):
            raise ValueError(f"params[{key!r}] needs one entry per image ({S})")
        P[:, slot] = v
    P[:, _FLIP] = flip
    P[:, _JITTER] = np.asarray(p["jitter"], dtype=bool).reshape(S)
    order = np.asarray(p["order"], dtype=np.int64).reshape(S, 4)
    factors = np.asarray(p["factors"], dtype=np.float32).reshape(S, 4)
    P[:, _ORDER:_ORDER + 4] = order
    P[:, _SHIFT] = [hue_shift(float(h)) for h in factors[:, 3]]
    H, W = int(p["img_H"]), int(p["img_W"])
    checks = [
        (P[:, _ROW0] >= 0) & (P[:, _ROWS] >= 1) & (P[:, _ROW0] + P[:, _ROWS] <= P[:, _H]), "the row cut leaves the frame",
        (P[:, _DH] >= 1) & (P[:, _DH] <= P[:, _ROWS]) & (P[:, _DW] >= 1) & (P[:, _DW] <= P[:, _W]),
        "the resize is not a downscale",
        (P[:, _DH] >= H) & (P[:, _DW] >= W), f"the resized image is smaller than the {H} x {W} output",
        (P[:, _DY] >= 0) & (P[:, _DY] <= P[:, _DH] - H) & (P[:, _DX] >= 0) & (P[:, _DX] <= P[:, _DW] - W),
        "the crop offset is outside the resized image",
        ~P[:, _JITTER].astype(bool) | (np.sort(order, 1) == np.arange(4)).all(1),
        "the jitter order is not a permutation of 0..3",
        ~P[:, _JITTER].astype(bool) | np.isfinite(factors).all(1), "a jitter factor is not finite",
    ]
    for i in range(0, len(checks), 2):
        ok = np.asarray(checks[i])
        if not ok.all():
            raise ValueError(f"sample {int(np.argmin(ok))}: {checks[i + 1]}")
    return P, np.ascontiguousarray(factors[:, :3])


def assemble_images(images, K, mode="train", params=None, rng=None, flip=None, out_dtype=torch.float32, stream=None,
                    **geometry):
    """The loaders' image side for S samples.  images: pack_images' dict (device buffer + host offsets and shapes);
    K [3,3] or [S,3,3] intrinsics of the raw frames.  params: image_params' dict, or None to draw it with
    image_params(shapes, mode, rng, **geometry) (kitti_image_args() / oxford_image_args() give the geometry).  flip:
    [S] bool (assemble_batch's out["flip"]; numpy or torch) or None.  Returns dict(img [S,3,img_H,img_W] out_dtype on
    the device (float32 holding integers, or uint8), K [S,3,3] float32 (host), K64 [S,3,3] float64, params)."""
    _require_cuda()
    lib = _native.load()
    data = images["data"]
    if not (isinstance(data, torch.Tensor) and data.is_cuda and data.dtype == torch.uint8 and data.dim() == 1):
        raise ValueError("images['data'] must be a 1-D uint8 CUDA tensor (pack_images)")
    if out_dtype not in (torch.float32, torch.uint8):
        raise ValueError(f"out_dtype must be torch.float32 or torch.uint8 (got {out_dtype})")
    shapes = np.asarray(images["shapes"], dtype=np.int64).reshape(-1, 2)
    offsets = np.ascontiguousarray(images["offsets"], dtype=np.int64).reshape(-1)
    S = shapes.shape[0]
    if offsets.shape != (S,):
        raise ValueError("images needs one offset per shape")
    if S and (offsets.min() < 0 or (offsets + 3 * shapes[:, 0] * shapes[:, 1]).max() > data.numel()):
        raise ValueError("an image lies outside images['data']")
    K = np.asarray(K, dtype=np.float64)
    K = np.broadcast_to(K, (S, 3, 3)) if K.shape == (3, 3) else K
    if K.shape != (S, 3, 3) or not np.isfinite(K).all():
        raise ValueError(f"K must be [3,3] or [{S},3,3] finite")
    if params is None:
        params = image_params(shapes, mode, rng, **geometry)
    elif geometry:
        raise TypeError("pass either params or the geometry arguments, not both")
    if flip is None:
        fl = np.zeros(S, dtype=bool)
    else:
        fl = (flip.cpu().numpy() if isinstance(flip, torch.Tensor) else np.asarray(flip)).astype(bool).reshape(-1)
        if fl.shape != (S,):
            raise ValueError(f"flip needs one entry per sample ({S})")
    P, factors = _pack_params(shapes, params, fl)
    H, W = int(params["img_H"]), int(params["img_W"])
    dev = data.device
    K64 = camera_K(K, params["row0"], params["scale"], params["dx"], params["dy"])
    with torch.cuda.device(dev), torch.cuda.stream(stream):
        img = torch.empty((S, 3, H, W), dtype=out_dtype, device=dev)
        if S:
            sp = _stream_ptr(stream)
            ws = _workspace(_ws_cache, lib.image_assemble_workspace_bytes(S, H, W), dev, stream)
            fn = lib.image_assemble_f32 if out_dtype == torch.float32 else lib.image_assemble_u8
            rc = fn(_ptr(data), data.numel(), offsets.ctypes.data, P.ctypes.data, factors.ctypes.data, S, H, W,
                    _ptr(img), _ptr(ws), ws.numel(), sp)
            _native.check(rc, "image_assemble")
    return dict(img=img, K=torch.from_numpy(K64.astype(np.float32)), K64=K64, params=params)


def augment_img(img_np, rng=None, **ranges):
    """Host drop-in for the loaders' augment_img (HxWx3 uint8 in and out) that works on current torchvision: the
    order and factors are drawn from rng (a numpy Generator or a seed) as ColorJitter.get_params draws them, then
    torchvision.transforms.functional's adjust_* run on a PIL image in that order.  Needs Pillow and torchvision."""
    from PIL import Image
    import torchvision.transforms.functional as F
    rg = {**JITTER_RANGES, **ranges}
    order, factors = _draw_jitter(_rng(rng), 1, rg["brightness"], rg["contrast"], rg["saturation"], rg["hue"])
    steps = (F.adjust_brightness, F.adjust_contrast, F.adjust_saturation, F.adjust_hue)
    img = Image.fromarray(np.ascontiguousarray(img_np, dtype=np.uint8))
    for op in order[0]:
        img = steps[op](img, float(factors[0, op]))
    return np.array(img)
