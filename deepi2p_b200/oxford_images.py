"""Oxford RobotCar stereo-centre frames on the GPU: the raw 8-bit Bayer PNGs to the loaders' undistorted RGB JPEGs,
bit for bit with data/oxford/build_dataset.py's conversion (the SDK's load_image(path, CameraModel), then
cv2.imwrite(jpg, cv2.cvtColor(image, cv2.COLOR_BGR2RGB)) at OpenCV's default quality 95).  DESIGN.md 4.25 states the
contract.

read_distortion_lut reads the SDK's models/stereo_narrow_left_distortion_lut.bin; decode_grey_png_batch
(imageprep) decodes the mosaics; debayer_undistort_batch runs csrc/oxford_images.cu (GBRG bilinear demosaicing and
the LUT undistortion, fused); encode_jpeg_batch (imageprep) encodes; convert_frames chains the four over files.
There is no CPU fallback.
"""
import os
import re

import numpy as np
import torch

from . import _native
from .frustum import _ptr, _require_cuda, _stream_ptr, _workspace
from .imageprep import decode_grey_png_batch, encode_jpeg_batch

LUT_FILE = "stereo_narrow_left_distortion_lut.bin"    # <sdk>/models/, the stereo centre camera's undistortion LUT
PATTERN = "gbrg"                                       # the SDK's BAYER_STEREO
_DESC = 8                                              # include/deepi2p_b200.h DIB_OXIMG_DESC


def read_distortion_lut(path, h, w):
    """CameraModel's bilinear_lut: np.fromfile(path, np.float64).reshape(2, -1).T, float64 [h w, 2] of (x, y) =
    (column, row) source coordinates per output pixel.  Raises ValueError when the table does not hold h w pairs
    (the SDK's "Incorrect image size for camera model") or holds a non-finite coordinate."""
    raw = np.fromfile(path, dtype=np.float64)
    if raw.size % 2 or raw.size // 2 != h * w:
        raise ValueError(f"Incorrect image size for camera model: {path} holds {raw.size} values, {h} x {w} images "
                         f"need {2 * h * w}")
    lut = np.ascontiguousarray(raw.reshape(2, -1).T)
    if not np.isfinite(lut).all():
        raise ValueError(f"{path}: the LUT holds a non-finite coordinate")
    return lut


def _lut_tensor(lut, dev):
    if isinstance(lut, torch.Tensor):
        t = lut.to(dev, torch.float64)
        if not bool(torch.isfinite(t).all()):
            raise ValueError("the LUT holds a non-finite coordinate")
    else:
        a = np.asarray(lut, dtype=np.float64)
        if not np.isfinite(a).all():
            raise ValueError("the LUT holds a non-finite coordinate")
        t = torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    if t.dim() != 2 or t.shape[1] != 2:
        raise ValueError(f"a LUT must be [h w, 2] (x, y) pairs (got {tuple(t.shape)})")
    return t.contiguous()


def debayer_undistort_batch(grey, lut, pattern=PATTERN, stream=None):
    """The SDK's load_image for S stereo-centre mosaics: grey is decode_grey_png_batch's dict (data uint8 on a CUDA
    device, offsets, shapes); lut is one table for every image (read_distortion_lut's [h w, 2], numpy or a CUDA
    tensor, uploaded once per call) or a list of S tables.  Returns pack_images' dict (HWC RGB uint8 on the same
    device, offsets, shapes), image s equal to np.array(model.undistort(demosaic(mosaic_s, 'gbrg'))).astype(np.uint8)
    bit for bit.  Only the stereo camera's 'gbrg' pattern is supported.  Raises ValueError("image i: ...") for a
    mosaic smaller than 2 x 2 or a LUT of the wrong size."""
    _require_cuda()
    if str(pattern).lower() != PATTERN:
        raise ValueError(f"unsupported Bayer pattern {pattern!r} (only the stereo camera's 'gbrg')")
    lib = _native.load()
    data = grey["data"]
    if not (isinstance(data, torch.Tensor) and data.is_cuda and data.dtype == torch.uint8 and data.dim() == 1):
        raise ValueError("grey['data'] must be a 1-D uint8 CUDA tensor (decode_grey_png_batch)")
    shapes = np.asarray(grey["shapes"], dtype=np.int64).reshape(-1, 2)
    offsets = np.asarray(grey["offsets"], dtype=np.int64).reshape(-1)
    S = shapes.shape[0]
    if offsets.shape != (S,):
        raise ValueError("grey needs one offset per shape")
    dev = data.device
    per_image = isinstance(lut, (list, tuple))
    if per_image and len(lut) != S:
        raise ValueError(f"one LUT per image is needed ({S}, got {len(lut)})")
    with torch.cuda.device(dev), torch.cuda.stream(stream):
        tabs = [_lut_tensor(t, dev) for t in lut] if per_image else [_lut_tensor(lut, dev)]
        lut_off = np.zeros(S, np.int64)
        if per_image:
            lut_off = np.concatenate([[0], np.cumsum([t.shape[0] for t in tabs])[:-1]]).astype(np.int64)
        for s in range(S):
            h, w = int(shapes[s, 0]), int(shapes[s, 1])
            if h < 2 or w < 2:
                raise ValueError(f"image {s}: a {h} x {w} mosaic is smaller than one 2 x 2 Bayer cell")
            if offsets[s] < 0 or offsets[s] + h * w > data.numel():
                raise ValueError(f"image {s}: lies outside grey['data']")
            n = tabs[s if per_image else 0].shape[0]
            if n != h * w:
                raise ValueError(f"image {s}: Incorrect image size for camera model (a {h} x {w} image, a LUT of "
                                 f"{n} entries)")
        table = tabs[0] if len(tabs) == 1 else torch.cat(tabs)
        sizes = 3 * shapes[:, 0] * shapes[:, 1]
        out_off = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64) if S else np.zeros(0, np.int64)
        out = torch.empty(int(sizes.sum()), dtype=torch.uint8, device=dev)
        if S:
            desc = np.zeros((S, _DESC), np.int64)
            desc[:, 0], desc[:, 1], desc[:, 2], desc[:, 3], desc[:, 4] = offsets, out_off, shapes[:, 0], \
                shapes[:, 1], lut_off
            sp = _stream_ptr(stream)
            ws = _workspace(lib.oxford_debayer_workspace_bytes(S), dev, sp)
            rc = lib.oxford_debayer_undistort_u8(_ptr(data), data.numel(), _ptr(table), table.shape[0],
                                                 desc.ctypes.data, S, _ptr(out), out.numel(), _ptr(ws), ws.numel(),
                                                 sp)
            _native.check(rc, "oxford_debayer_undistort")
    return dict(data=out, offsets=out_off, shapes=shapes.copy())


def convert_frames(png_paths, jpg_paths, lut, batch=64, quality=95, device="cuda", stream=None):
    """build_dataset.py's image conversion for the frames png_paths -> jpg_paths (same length): read the mosaics,
    decode, demosaic and undistort with `lut` (one table for every frame), encode at `quality` and write each JPEG,
    `batch` frames per device pass.  The LUT is uploaded once.  Returns the number of frames written."""
    if len(png_paths) != len(jpg_paths):
        raise ValueError(f"{len(png_paths)} PNG paths but {len(jpg_paths)} JPEG paths")
    if int(batch) < 1:
        raise ValueError(f"batch must be positive (got {batch})")
    if not png_paths:
        return 0
    _require_cuda()
    dev = torch.device(device)
    with torch.cuda.device(dev), torch.cuda.stream(stream):
        table = _lut_tensor(lut, dev)
    for i in range(0, len(png_paths), int(batch)):
        blobs = []
        for p in png_paths[i:i + int(batch)]:
            with open(p, "rb") as f:
                blobs.append(f.read())
        try:
            grey = decode_grey_png_batch(blobs, device=dev, stream=stream)
        except ValueError as e:                       # name the file rather than its place in the batch
            m = re.match(r"image (\d+): (.*)", str(e), re.S)
            if not m:
                raise
            raise ValueError(f"{png_paths[i + int(m.group(1))]}: {m.group(2)}") from None
        rgb = debayer_undistort_batch(grey, table, stream=stream)
        for p, b in zip(jpg_paths[i:i + int(batch)], encode_jpeg_batch(rgb, quality=quality, stream=stream)):
            d = os.path.dirname(p)
            if d:
                os.makedirs(d, exist_ok=True)
            with open(p, "wb") as f:
                f.write(b)
    return len(png_paths)
