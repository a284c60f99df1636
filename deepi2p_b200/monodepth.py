"""Monodepth depth clouds for the ICP baseline (evaluation/icp/save_depth_map.py) on the GPU.

The reference makes the target cloud of registration_icp.py one frame at a time: Pillow's Lanczos resize of
<id>_img.png to the network's feed size, ToTensor, monodepth2's ResNet-18 encoder and depth decoder, a bilinear
upsample of ("disp", 0) back to the image size, its reciprocal, and a numpy back-projection through K^-1.  Here a
batch goes through:

  resize_normalise  csrc/monodepth.cu: Pillow's 8-bit Lanczos resize, bit for bit, fused with ToTensor and the
                    encoder's (x - 0.45) / 0.225 as torch computes them on the device
  DepthNet          monodepth2's ResnetEncoder(18) + DepthDecoder(scales=range(4)) as torch modules with monodepth2's
                    state_dict keys; the convolutions are cuDNN's and follow torch's TF32 flags
  depth_clouds      the two above, then csrc/monodepth.cu: torch's bilinear upsample and reciprocal, bit for bit, and
                    the fp64 back-projection, written as save_depth_map.py's float64 [3, H*W] cloud or, scaled on the
                    device by the ground-truth calibration of registration_icp.py:215-218, as icp_register_batch's
                    float32 target

load_monodepth reads monodepth2's encoder.pth / depth.pth unchanged.  The architecture is restated from monodepth2's
published code and pinned by seeded checkpoints in that layout (oracle_monodepth); DESIGN.md 4.31 states the contract.
There is no CPU fallback.
"""
import functools
import math
import os

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _native
from ._native import _ptr, _require_cuda, _stream_ptr, _workspace
from .frustum import _ws_cache
from .network import _BasicBlock

PRECISION_BITS = 22                      # Pillow's Resample.c, 8 bits per channel
FEED_SUB = np.float32(0.45)              # ResnetEncoder.forward: (x - 0.45) / 0.225; torch's CUDA division by a CPU
FEED_MUL = np.float32(1.0) / np.float32(0.225)   # scalar multiplies by the float32 reciprocal
NON_TENSOR_KEYS = ("height", "width", "use_stereo")
ENC_CHANNELS = (64, 64, 128, 256, 512)
DEC_CHANNELS = (16, 32, 64, 128, 256)


# ---------------------------------------------------------------------------------------------------------------------
# the network

class _Conv3x3(nn.Module):
    """monodepth2's Conv3x3: ReflectionPad2d(1), then a 3x3 convolution with bias."""

    def __init__(self, c_in, c_out):
        super().__init__()
        self.pad = nn.ReflectionPad2d(1)
        self.conv = nn.Conv2d(c_in, c_out, 3)

    def forward(self, x):
        return self.conv(self.pad(x))


class _ConvBlock(nn.Module):
    """monodepth2's ConvBlock: Conv3x3, then ELU."""

    def __init__(self, c_in, c_out):
        super().__init__()
        self.conv = _Conv3x3(c_in, c_out)
        self.nonlin = nn.ELU(inplace=True)

    def forward(self, x):
        return self.nonlin(self.conv(x))


class _ResNet18(nn.Module):
    """torchvision's ResNet-18 parameters (monodepth2's ResnetEncoder.encoder); forward returns the five features
    relu(bn1(conv1(x))), layer1(maxpool(.)), layer2, layer3, layer4.  fc is unused but part of the checkpoint."""

    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 64, 7, 2, 3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(3, 2, 1)
        c_in = 64
        for i, c in enumerate(ENC_CHANNELS[1:]):
            s = 1 if i == 0 else 2
            setattr(self, f"layer{i + 1}", nn.Sequential(_BasicBlock(c_in, c, s), _BasicBlock(c, c, 1)))
            c_in = c
        self.fc = nn.Linear(512, 1000)

    def forward(self, x):
        feats = [self.relu(self.bn1(self.conv1(x)))]
        feats.append(self.layer1(self.maxpool(feats[-1])))
        for layer in (self.layer2, self.layer3, self.layer4):
            feats.append(layer(feats[-1]))
        return feats


class DepthNet(nn.Module):
    """monodepth2's ResnetEncoder(18) under "encoder." and DepthDecoder(num_ch_enc, scales=range(4)) under "decoder."
    (nn.ModuleList in insertion order: upconv(4,0), upconv(4,1), ..., upconv(0,1), then dispconv(0..3)), so
    encoder.pth and depth.pth load with their own keys.  forward takes the normalised input ((x - 0.45) / 0.225, NCHW,
    sides multiples of 32) and returns ("disp", 0) [S,1,h,w]; dispconv(1..3) are loaded but not run (their outputs
    are unused).  feed_height / feed_width: the checkpoint's training size."""

    def __init__(self, feed_height=192, feed_width=640):
        super().__init__()
        self.feed_height, self.feed_width = int(feed_height), int(feed_width)
        self.encoder = _ResNet18()
        convs = []
        for i in range(4, -1, -1):
            convs.append(_ConvBlock(ENC_CHANNELS[-1] if i == 4 else DEC_CHANNELS[i + 1], DEC_CHANNELS[i]))
            convs.append(_ConvBlock(DEC_CHANNELS[i] + (ENC_CHANNELS[i - 1] if i > 0 else 0), DEC_CHANNELS[i]))
        convs += [_Conv3x3(DEC_CHANNELS[s], 1) for s in range(4)]
        self.decoder = nn.ModuleList(convs)

    def forward(self, x):
        feats = self.encoder(x)
        y = feats[-1]
        for i in range(4, -1, -1):
            j = 2 * (4 - i)
            y = F.interpolate(self.decoder[j](y), scale_factor=2, mode="nearest")
            if i > 0:
                y = torch.cat([y, feats[i - 1]], 1)
            y = self.decoder[j + 1](y)
        return torch.sigmoid(self.decoder[10](y))


def load_monodepth(model_dir, device="cuda"):
    """monodepth2's <model_dir>/encoder.pth and depth.pth (e.g. mono+stereo_640x192) -> a DepthNet in eval mode on
    `device` whose feed_height / feed_width are the encoder checkpoint's height / width.  The non-tensor entries
    height, width and use_stereo are dropped and the rest loads strictly: a missing or unexpected key raises, and so
    does a feed size that is not a positive multiple of 32."""
    enc = torch.load(os.path.join(model_dir, "encoder.pth"), map_location="cpu", weights_only=True)
    dec = torch.load(os.path.join(model_dir, "depth.pth"), map_location="cpu", weights_only=True)
    for k in ("height", "width"):
        if k not in enc:
            raise ValueError(f"encoder.pth has no {k!r} entry (the feed size)")
    fh, fw = int(enc["height"]), int(enc["width"])
    if fh < 32 or fw < 32 or fh % 32 or fw % 32:
        raise ValueError(f"the feed size must be a positive multiple of 32, got {fh} x {fw}")
    sd = {k: v for k, v in enc.items() if k not in NON_TENSOR_KEYS}
    overlap = sorted(set(sd) & set(dec))
    if overlap:
        raise ValueError(f"encoder.pth and depth.pth share keys: {overlap[:4]}")
    sd.update(dec)
    model = DepthNet(fh, fw)
    model.load_state_dict(sd, strict=True)
    return model.to(device).eval()


# ---------------------------------------------------------------------------------------------------------------------
# the device passes

@functools.lru_cache(maxsize=32)
def lanczos_table(in_size, out_size):
    """Pillow's precompute_coeffs + normalize_coeffs_8bpc for one axis with the Lanczos filter, in float64 with the C
    library's sin (math.sin): int32 [out_size, 2 + ksize] rows of (first input index, tap count, coefficients in 2^-22
    units rounded half away from zero), ksize = 2 ceil(3 max(in / out, 1)) + 1."""
    scale = float(in_size) / out_size
    fscale = max(scale, 1.0)
    support = 3.0 * fscale
    ksize = int(math.ceil(support)) * 2 + 1
    tab = np.zeros((out_size, 2 + ksize), np.int32)

    def lanczos(x):
        if not -3.0 <= x < 3.0:
            return 0.0
        a = 1.0 if x == 0.0 else math.sin(x * math.pi) / (x * math.pi)
        b = 1.0 if x == 0.0 else math.sin(x / 3 * math.pi) / (x / 3 * math.pi)
        return a * b

    for i in range(out_size):
        center = (i + 0.5) * scale
        lo = max(int(center - support + 0.5), 0)
        n = min(int(center + support + 0.5), in_size) - lo
        w = [lanczos((j + lo - center + 0.5) * (1.0 / fscale)) for j in range(n)]
        total = 0.0
        for v in w:
            total += v
        if total != 0.0:
            w = [v / total for v in w]
        tab[i, 0], tab[i, 1] = lo, n
        tab[i, 2:2 + n] = [int(v * (1 << PRECISION_BITS) + (-0.5 if v < 0 else 0.5)) for v in w]
    tab.setflags(write=False)
    return tab


def _frames(images):
    data = images["data"]
    if not (isinstance(data, torch.Tensor) and data.is_cuda and data.dtype == torch.uint8 and data.dim() == 1):
        raise ValueError("images['data'] must be a 1-D uint8 CUDA tensor (imageprep.pack_images)")
    shapes = np.asarray(images["shapes"], dtype=np.int64).reshape(-1, 2)
    offsets = np.asarray(images["offsets"], dtype=np.int64).reshape(-1)
    S = shapes.shape[0]
    if S < 1 or offsets.shape != (S,):
        raise ValueError("images needs at least one frame and one offset per shape")
    if (shapes != shapes[0]).any():
        raise ValueError("the frames of one call must share one size (got %s)" % sorted({tuple(s) for s in shapes}))
    h, w = int(shapes[0, 0]), int(shapes[0, 1])
    if (offsets < 0).any() or (offsets + 3 * h * w > data.numel()).any():
        raise ValueError("a frame lies outside images['data']")
    return data, offsets, S, h, w


def resize_normalise(images, feed_height, feed_width, stream=None):
    """The encoder's input for pack_images' frames (one size h x w per call, HWC RGB uint8 on a CUDA device):
    (ToTensor(Image.resize((feed_width, feed_height), LANCZOS)) - 0.45) / 0.225 as float32 [S,3,feed_height,
    feed_width], the resize bit for bit with Pillow and the arithmetic torch's on the device."""
    _require_cuda()
    lib = _native.load()
    data, offsets, S, h, w = _frames(images)
    dev = data.device
    with torch.cuda.device(dev), torch.cuda.stream(stream):
        sp = _stream_ptr(stream)
        off = torch.from_numpy(offsets).to(dev)
        tx = torch.from_numpy(np.array(lanczos_table(w, feed_width))).to(dev) if w != feed_width else None
        ty = torch.from_numpy(np.array(lanczos_table(h, feed_height))).to(dev) if h != feed_height else None
        out = torch.empty((S, 3, feed_height, feed_width), dtype=torch.float32, device=dev)
        tmp = None
        if tx is not None and ty is not None:
            tmp = _workspace(_ws_cache, S * h * feed_width * 3, dev, stream)
        rc = lib.monodepth_resize_f32(_ptr(data), _ptr(off), S, h, w, feed_height, feed_width, _ptr(tx),
                                      0 if tx is None else tx.shape[1] - 2, _ptr(ty),
                                      0 if ty is None else ty.shape[1] - 2, float(FEED_SUB), float(FEED_MUL),
                                      _ptr(tmp), 0 if tmp is None else tmp.numel(), _ptr(out), sp)
    _native.check(rc, "monodepth_resize")
    return out


def k_inverse(K):
    """save_depth_map.py's np.linalg.inv(K_np) per frame, in K's own dtype (the reference's _K.npy files hold
    float32), upcast to float64 as the script's product does: [S,3,3] (or [3,3]) -> [S,9] float64."""
    K = np.asarray(K)
    K = K.reshape((-1, 3, 3))
    return np.stack([np.linalg.inv(k) for k in K]).astype(np.float64).reshape(-1, 9)


def _dev_f64(a, shape, dev, name):
    t = torch.as_tensor(a, dtype=torch.float64)
    if t.numel() != int(np.prod(shape)):
        raise ValueError(f"{name} must hold {list(shape)} values")
    return t.reshape(shape).to(dev).contiguous()


def depth_clouds(model, images, K_inv, *, src=None, n_pts=None, P_gt=None, K=None, cloud64=True, depth=False,
                 stream=None):
    """save_depth_map.py for a batch: pack_images' frames (one size H x W per call) -> resize_normalise -> model
    (a DepthNet on the frames' device, eval mode) -> depth at H x W (torch's bilinear upsample and reciprocal, bit for
    bit) -> the cloud K^-1 (d x, d y, d) in fp64, point y W + x.  K_inv: [S,9] or [S,3,3] float64 (k_inverse).

    Returns a dict with
      pc     [S,3,H*W] float64, the unscaled <id>_pc.npy contents (with cloud64)
      depth  [S,H,W] float32 (with depth)
    and, when the LiDAR side is given (src [S,3,Ns] f32 and n_pts [S] int32 or None on the device, P_gt [S,4,4] and K
    [S,3,3] float64), the ground-truth calibration of registration_icp.py:215-218 on the device:
      scale  [S] float64 = mean z of the LiDAR points inside the image under P_gt / mean z of the cloud
      tgt    [S,3,H*W] float32 = float32(pc * scale), icp_register_batch's target
    All outputs stay on the device; nothing is read back."""
    _require_cuda()
    lib = _native.load()
    if model.training:
        raise ValueError("the depth network must be in eval mode")
    data, _, S, H, W = _frames(images)
    dev = data.device
    x = resize_normalise(images, model.feed_height, model.feed_width, stream=stream)
    with torch.cuda.device(dev), torch.cuda.stream(stream), torch.no_grad():
        disp = model(x).float().contiguous()
        if tuple(disp.shape) != (S, 1, model.feed_height, model.feed_width):
            raise ValueError(f"the network returned {tuple(disp.shape)}")
        sp = _stream_ptr(stream)
        ki = _dev_f64(K_inv, (S, 9), dev, "K_inv")
        res = {}
        if cloud64:
            res["pc"] = torch.empty((S, 3, H * W), dtype=torch.float64, device=dev)
        if depth:
            res["depth"] = torch.empty((S, H, W), dtype=torch.float32, device=dev)
        ws = None
        Ns, P_d, K_d = 0, None, None
        if src is not None:
            if not (isinstance(src, torch.Tensor) and src.is_cuda and src.dtype == torch.float32 and src.dim() == 3
                    and src.shape[0] == S and src.shape[1] == 3 and src.is_contiguous() and src.device == dev):
                raise ValueError("src must be a contiguous float32 [S,3,Ns] tensor on the frames' device")
            if n_pts is not None and not (isinstance(n_pts, torch.Tensor) and n_pts.dtype == torch.int32
                                          and tuple(n_pts.shape) == (S,) and n_pts.device == dev):
                raise ValueError("n_pts must be an int32 [S] tensor on the frames' device")
            if P_gt is None or K is None:
                raise ValueError("the scale needs P_gt and K")
            Ns = src.shape[2]
            P_d = _dev_f64(P_gt, (S, 16), dev, "P_gt")
            K_d = _dev_f64(K, (S, 9), dev, "K")
            res["scale"] = torch.empty((S,), dtype=torch.float64, device=dev)
            res["tgt"] = torch.empty((S, 3, H * W), dtype=torch.float32, device=dev)
            ws = _workspace(_ws_cache, lib.monodepth_cloud_workspace_bytes(S, H, W), dev, stream)
        if not res:
            raise ValueError("no output requested")
        rc = lib.monodepth_cloud_f32(_ptr(disp), S, disp.shape[2], disp.shape[3], H, W, _ptr(ki),
                                     _ptr(res.get("depth")), _ptr(res.get("pc")), _ptr(src), _ptr(n_pts), Ns, _ptr(P_d), _ptr(K_d),
                                     _ptr(res.get("scale")), _ptr(res.get("tgt")), _ptr(ws),
                                     0 if ws is None else ws.numel(), sp)
    _native.check(rc, "monodepth_cloud")
    return res


def images_from_batch(img):
    """A classifier batch's float image [S,3,H,W] on the device -> pack_images' dict, rounded as
    visualize_and_save_data.py:130 writes <id>_img.png (img.round().to(uint8), HWC RGB), so a kitti_batch /
    oxford_batch batch goes to depth_clouds without a PNG."""
    if not (isinstance(img, torch.Tensor) and img.is_cuda and img.dim() == 4 and img.shape[1] == 3):
        raise ValueError("img must be a [S,3,H,W] CUDA tensor")
    S, _, H, W = img.shape
    data = img.detach().round().to(torch.uint8).permute(0, 2, 3, 1).contiguous().reshape(-1)
    return dict(data=data, offsets=np.arange(S, dtype=np.int64) * (3 * H * W),
                shapes=np.tile(np.array([[H, W]], np.int64), (S, 1)))
