"""Fused TF32 inference of the classifier's ResNet-34 image encoder (csrc/resnet.cu, DESIGN.md 4.30).

Every convolution runs with its eval-mode BatchNorm folded into the weights (network.fold_resnet34) as one implicit
GEMM on the tensor cores, with the bias, the block's residual and the ReLU applied in the epilogue; activations stay
NHWC float32 between layers and each is written once.  A block's 1x1 stride-2 downsample runs as extra K columns of its
second convolution.  The stem reads the [B,3,H,W] image directly; the stride-16 and stride-32 maps are written
channel-major by the epilogues that end layer3 and layer4, and img_global is a float64 mean of the stride-32 map
rounded once.  Inference only: there is no backward.

    packed = resnet.pack_resnet34(network.fold_resnet34(model.img_encoder.backbone))
    s16, s32, img_global = resnet.resnet34_features(img, packed)     # [B,256,P16], [B,512,P32], [B,512]

Operands are rounded to TF32 (nearest, ties away from zero: the weights once when packed, the activations as they are
read), accumulation is float32, so results differ from the float64 module at rounding level; oracle_resnet states the
per-layer bound.
"""
import torch

from . import _native
from ._native import _ptr, _stream_ptr

STAGES = ((64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2))     # (channels, blocks, first stride) of layers 1-4
MIN_IMAGE = 32                                                     # the smallest H and W resnet34_features takes


class PackedConv:
    """One folded convolution on the device: `packed` (weights [C_out][K] rounded to TF32, K = kernel^2 C_in + c_short,
    rows zero-padded to a multiple of 32) and `bias` [C_out] float32.  c_short > 0 marks a fused 1x1 shortcut
    (a block's downsample): its C_in columns follow the main ones and its bias is already added to `bias`."""

    def __init__(self, packed, bias, kernel, c_in, c_out, c_short=0):
        self.packed, self.bias = packed, bias
        self.kernel, self.pad, self.c_in, self.c_out, self.c_short = kernel, kernel // 2, c_in, c_out, c_short


class PackedResNet34:
    """pack_resnet34's result: `stem` (PackedConv of conv1) and `blocks` [(stride, conv1, conv2)] in forward order,
    16 blocks; `stage_ends` are the indices of the last block of layer3 and layer4."""

    def __init__(self, stem, blocks):
        self.stem, self.blocks = stem, blocks
        ends = [sum(n for _, n, _ in STAGES[:s + 1]) - 1 for s in range(4)]
        self.stage_ends = (ends[2], ends[3])

    @property
    def device(self):
        return self.stem.packed.device


def _check_tensor(t, name, device=None):
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a torch.Tensor")
    if t.dtype != torch.float32:
        raise TypeError(f"{name} must be float32, got {t.dtype}")
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor")
    if device is not None and t.device != device:
        raise RuntimeError(f"{name} is on {t.device}, the layers are on {device}")
    if not t.is_contiguous():
        raise RuntimeError(f"{name} must be contiguous")


def pack_conv(W, b, shortcut=None):
    """Pack one folded convolution: W [C_out, k, k, C_in] and b [C_out] float32 CUDA (fold_resnet34's pair);
    shortcut = (Wd [C_out, 1, 1, C2], bd) fuses a 1x1 shortcut convolution as extra K columns, with the bias b + bd."""
    if not isinstance(W, torch.Tensor) or W.dim() != 4 or W.shape[1] != W.shape[2]:
        raise ValueError("W must be [C_out, k, k, C_in]")
    C_out, k, _, C_in = W.shape
    if C_out % 8 or not 1 <= k <= 7:
        raise ValueError(f"need C_out a multiple of 8 and 1 <= k <= 7, got C_out = {C_out}, k = {k}")
    if not isinstance(b, torch.Tensor) or tuple(b.shape) != (C_out,):
        raise ValueError(f"b must be [{C_out}]")
    for t, name in ((W, "W"), (b, "b")):
        _check_tensor(t.contiguous(), name, W.device)
    w = W.detach().reshape(C_out, -1)
    bias = b.detach()
    c_short = 0
    if shortcut is not None:
        Wd, bd = shortcut
        if not isinstance(Wd, torch.Tensor) or Wd.dim() != 4 or tuple(Wd.shape[:3]) != (C_out, 1, 1):
            raise ValueError(f"the shortcut's W must be [{C_out}, 1, 1, C2]")
        if (k * k * C_in) % 32 or Wd.shape[3] % 32:
            raise ValueError("a fused shortcut needs k^2 C_in and C2 multiples of 32")
        for t, name in ((Wd, "shortcut W"), (bd, "shortcut b")):
            _check_tensor(t.contiguous(), name, W.device)
        c_short = int(Wd.shape[3])
        w = torch.cat((w, Wd.detach().reshape(C_out, -1)), dim=1)
        bias = bias + bd.detach()                  # one float32 addition: the correctly rounded b + bd
    w, K = w.contiguous(), w.shape[1]
    lib = _native.load()
    need = lib.resnet_conv_packed_bytes(C_out, K)
    with torch.cuda.device(W.device):
        packed = torch.empty(need // 4, dtype=torch.float32, device=W.device)
        rc = lib.resnet_conv_pack_f32(w.data_ptr(), C_out, K, packed.data_ptr(), need, _stream_ptr())
    _native.check(rc, "resnet_conv_pack_f32")
    return PackedConv(packed, bias.contiguous(), int(k), int(C_in), int(C_out), c_short)


def pack_resnet34(folded):
    """Device-resident packed weights from network.fold_resnet34's dict (float32 CUDA tensors): the stem, and each
    block's two convolutions with the downsample fused into the second.  Returns a PackedResNet34."""
    if not isinstance(folded, dict) or "conv1" not in folded:
        raise ValueError("folded: need network.fold_resnet34's dict")
    if torch.is_grad_enabled() and any(t.requires_grad for pair in folded.values() for t in pair):
        raise RuntimeError("resnet34 has no backward: pack under torch.no_grad() or detach the folded weights")
    stem = pack_conv(*folded["conv1"])
    blocks = []
    for s, (C, n, first) in enumerate(STAGES, 1):
        for j in range(n):
            key = f"layer{s}.{j}"
            try:
                c1, c2 = folded[key + ".conv1"], folded[key + ".conv2"]
            except KeyError:
                raise ValueError(f"folded: missing {key}.conv1 / {key}.conv2") from None
            down = folded.get(key + ".downsample")
            stride = first if j == 0 else 1
            if (stride != 1) != (down is not None):
                raise ValueError(f"folded: {key} needs a downsample exactly when its stride is 2")
            blocks.append((stride, pack_conv(*c1), pack_conv(*c2, shortcut=down)))
    return PackedResNet34(stem, blocks)


def _out_size(n, k, stride, pad):
    return (n + 2 * pad - k) // stride + 1


def conv2d_fused(x, layer, stride, residual=None, relu=True, shortcut=None, shortcut_stride=2, nchw_input=False,
                 channel_major=False, nhwc=True):
    """One folded convolution (a PackedConv): relu?(conv(x) + bias + residual), padding kernel // 2.

    x: [B,H,W,C_in] NHWC float32 CUDA contiguous, or with nchw_input=True [B,C_in,H,W] (the stem reads the image).
    residual: NHWC [B,H_out,W_out,C_out] or None.  shortcut: the block input [B,H2,W2,C2] NHWC for a layer packed
    with a fused 1x1 shortcut, read at shortcut_stride: (H2 - 1) // shortcut_stride + 1 == H_out.
    Returns the NHWC output [B,H_out,W_out,C_out]; with channel_major=True (out_nhwc, out_cm [B,C_out,H_out*W_out]),
    where nhwc=False skips the NHWC store (out_nhwc is then None)."""
    if not isinstance(layer, PackedConv):
        raise TypeError("layer must be a resnet.PackedConv (pack_conv / pack_resnet34)")
    if stride not in (1, 2) or shortcut_stride not in (1, 2):
        raise ValueError(f"stride and shortcut_stride must be 1 or 2, got {stride} and {shortcut_stride}")
    dev = layer.packed.device
    if not isinstance(x, torch.Tensor) or x.dim() != 4:
        raise ValueError("x must be a 4-D tensor")
    if nchw_input:
        B, C, H, W = x.shape
    else:
        B, H, W, C = x.shape
    if C != layer.c_in:
        raise ValueError(f"x has {C} channels, the layer takes {layer.c_in}")
    if not nchw_input and C % 32:
        raise ValueError(f"an NHWC input needs a multiple of 32 channels, got {C}")
    if not 1 <= B <= 65535:
        raise ValueError(f"need 1 <= B <= 65535, got {B}")
    _check_tensor(x, "x", dev)
    k, pad = layer.kernel, layer.pad
    if H + 2 * pad < k or W + 2 * pad < k:
        raise ValueError(f"a {H} x {W} input is smaller than the {k} x {k} kernel")
    Ho, Wo = _out_size(H, k, stride, pad), _out_size(W, k, stride, pad)
    C_out = layer.c_out
    if (shortcut is None) != (layer.c_short == 0):
        raise ValueError("shortcut must be given exactly when the layer was packed with one")
    H2 = W2 = C2 = 0
    if shortcut is not None:
        _check_tensor(shortcut, "shortcut", dev)
        if shortcut.dim() != 4 or shortcut.shape[0] != B or shortcut.shape[3] != layer.c_short:
            raise ValueError(f"shortcut must be [{B}, H2, W2, {layer.c_short}]")
        _, H2, W2, C2 = shortcut.shape
        if ((H2 - 1) // shortcut_stride + 1, (W2 - 1) // shortcut_stride + 1) != (Ho, Wo):
            raise ValueError(f"a {H2} x {W2} shortcut at stride {shortcut_stride} does not give the {Ho} x {Wo} "
                             f"output")
    if residual is not None:
        _check_tensor(residual, "residual", dev)
        if tuple(residual.shape) != (B, Ho, Wo, C_out):
            raise ValueError(f"residual must be [{B}, {Ho}, {Wo}, {C_out}], got {tuple(residual.shape)}")
    if not (nhwc or channel_major):
        raise ValueError("at least one of nhwc and channel_major must be True")
    out = torch.empty((B, Ho, Wo, C_out), dtype=torch.float32, device=dev) if nhwc else None
    cm = torch.empty((B, C_out, Ho * Wo), dtype=torch.float32, device=dev) if channel_major else None
    lib = _native.load()
    with torch.cuda.device(dev):
        rc = lib.resnet_conv_f32(x.data_ptr(), int(nchw_input), B, H, W, C, k, stride, pad, _ptr(shortcut), H2, W2, C2,
                                 shortcut_stride, layer.packed.data_ptr(), layer.packed.numel() * 4, layer.bias.data_ptr(),
                                 _ptr(residual), int(bool(relu)), C_out, _ptr(out), _ptr(cm), _stream_ptr())
    _native.check(rc, "resnet_conv_f32")
    return (out, cm) if channel_major else out


def max_pool_3x3s2(x):
    """torch.nn.MaxPool2d(3, 2, 1) over NHWC x [B,H,W,C] float32 CUDA -> [B,(H-1)//2+1,(W-1)//2+1,C]; a NaN in a
    window gives NaN."""
    _check_tensor(x, "x")
    if x.dim() != 4:
        raise ValueError(f"x must be [B,H,W,C], got {tuple(x.shape)}")
    B, H, W, C = x.shape
    out = torch.empty((B, (H - 1) // 2 + 1, (W - 1) // 2 + 1, C), dtype=torch.float32, device=x.device)
    if out.numel() == 0:
        return out
    lib = _native.load()
    with torch.cuda.device(x.device):
        rc = lib.resnet_maxpool_f32(x.data_ptr(), B, H, W, C, out.data_ptr(), _stream_ptr())
    _native.check(rc, "resnet_maxpool_f32")
    return out


def stem(img, packed):
    """conv1 + bn1 + relu + maxpool of the backbone: img [B,3,H,W] float32 CUDA -> NHWC [B,H/4,W/4,64] (rounded up)."""
    return max_pool_3x3s2(conv2d_fused(img, packed.stem, 2, nchw_input=True))


def channel_mean(x):
    """The mean over the last axis of x [B,C,P] float32 CUDA contiguous -> [B,C]: a float64 sum in a fixed order,
    rounded once, so it is the same bits on every run."""
    _check_tensor(x, "x")
    if x.dim() != 3 or x.shape[2] < 1:
        raise ValueError(f"x must be [B,C,P] with P >= 1, got {tuple(x.shape)}")
    out = torch.empty(x.shape[:2], dtype=torch.float32, device=x.device)
    if out.numel() == 0:
        return out
    lib = _native.load()
    with torch.cuda.device(x.device):
        rc = lib.resnet_mean_f32(x.data_ptr(), x.shape[0] * x.shape[1], x.shape[2], out.data_ptr(), _stream_ptr())
    _native.check(rc, "resnet_mean_f32")
    return out


def resnet34_features(img, packed):
    """The image encoder's outputs from the assembled image: img [B,3,H,W] float32 CUDA contiguous (H, W >= 32) ->
    (s16 [B,256,P16], s32 [B,512,P32], img_global [B,512]), s16 and s32 channel-major (the end of layer3 and layer4,
    P = h * w of the map), img_global the mean of s32 over P: what point_ops.attention_fusion and point_ops.node_mlp
    take.  packed: pack_resnet34's result.  Inference only."""
    if not isinstance(packed, PackedResNet34):
        raise TypeError("packed must be a resnet.PackedResNet34 (pack_resnet34)")
    if not isinstance(img, torch.Tensor) or img.dim() != 4 or img.shape[1] != 3:
        raise ValueError(f"img must be a [B,3,H,W] tensor, got {getattr(img, 'shape', type(img))}")
    if img.shape[2] < MIN_IMAGE or img.shape[3] < MIN_IMAGE:
        raise ValueError(f"a {img.shape[2]} x {img.shape[3]} image is too small: the stride-32 map needs H and W "
                         f">= {MIN_IMAGE}")
    _check_tensor(img, "img", packed.device)
    if torch.is_grad_enabled() and img.requires_grad:
        raise RuntimeError("resnet34_features has no backward: call it under torch.no_grad()")
    x = stem(img, packed)
    s16 = s32 = None
    for i, (stride, c1, c2) in enumerate(packed.blocks):
        y = conv2d_fused(x, c1, stride)
        # the block input is the residual, or with a downsample the fused shortcut read at the block's stride
        kw = dict(residual=x) if c2.c_short == 0 else dict(shortcut=x, shortcut_stride=stride)
        if i == packed.stage_ends[0]:
            x, s16 = conv2d_fused(y, c2, 1, channel_major=True, **kw)
        elif i == packed.stage_ends[1]:
            _, s32 = conv2d_fused(y, c2, 1, channel_major=True, nhwc=False, **kw)
        else:
            x = conv2d_fused(y, c2, 1, **kw)
        del y
    return s16, s32, channel_mean(s32)
