"""Independent restatements for the monodepth depth clouds (deepi2p_b200/monodepth.py, csrc/monodepth.cu, DESIGN.md
4.31): Pillow's 8-bit Lanczos resize in numpy, a float64 CPU composition of monodepth2's ResNet-18 encoder and depth
decoder written with torch.nn.functional only, save_depth_map.py's convert_depth_to_pointcloud line for line, and a
writer for seeded checkpoints in monodepth2's encoder.pth / depth.pth layout.  Tests and the benchmark use this module,
nothing else does.

The architecture is restated from monodepth2's published code (networks/resnet_encoder.py, networks/depth_decoder.py,
layers.py); it has not been checked against a monodepth2 checkout.
"""
import math
import os

import numpy as np

PRECISION_BITS = 22                   # Pillow's Resample.c, 8 bits per channel
ENC_CHANNELS = (64, 64, 128, 256, 512)
DEC_CHANNELS = (16, 32, 64, 128, 256)


# ---------------------------------------------------------------------------------------------------------------------
# Pillow's Image.resize(size, Image.LANCZOS) on an RGB uint8 image (Resample.c: precompute_coeffs,
# normalize_coeffs_8bpc, ImagingResampleHorizontal_8bpc / Vertical_8bpc)

def _lanczos(x):
    def sinc(v):
        if v == 0.0:
            return 1.0
        v = v * math.pi
        return math.sin(v) / v
    if -3.0 <= x < 3.0:
        return sinc(x) * sinc(x / 3)
    return 0.0


def lanczos_coeffs(in_size, out_size):
    """One axis: (xmin [out] int64, xsize [out] int64, coefficients [out, ksize] int32 in 2^-22 units)."""
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = 3.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    xmin_all = np.zeros(out_size, np.int64)
    xsize_all = np.zeros(out_size, np.int64)
    kk = np.zeros((out_size, ksize), np.int32)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        ss = 1.0 / filterscale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = [_lanczos((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for v in w:
            ww += v
        if ww != 0.0:
            w = [v / ww for v in w]
        for x, v in enumerate(w):
            kk[xx, x] = int(-0.5 + v * (1 << PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << PRECISION_BITS))
        xmin_all[xx], xsize_all[xx] = xmin, xmax
    return xmin_all, xsize_all, kk


def _pass(img, axis, out_size):
    """One separable pass over axis 1 (horizontal) or 0 (vertical) of an [h, w, 3] uint8 image."""
    xmin, xsize, kk = lanczos_coeffs(img.shape[axis], out_size)
    src = np.moveaxis(img.astype(np.int64), axis, 0)
    out = np.empty((out_size,) + src.shape[1:], np.uint8)
    for i in range(out_size):
        acc = np.full(src.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
        for j in range(int(xsize[i])):
            acc += src[xmin[i] + j] * int(kk[i, j])
        out[i] = np.clip(acc >> PRECISION_BITS, 0, 255)
    return np.moveaxis(out, 0, axis)


def lanczos_resize(img, width, height):
    """PIL.Image.fromarray(img).resize((width, height), Image.LANCZOS) for an [h, w, 3] uint8 array: the horizontal
    pass first, each pass skipped when its axis keeps its size, a uint8 intermediate."""
    img = np.ascontiguousarray(img, np.uint8)
    if img.shape[1] != width:
        img = _pass(img, 1, width)
    if img.shape[0] != height:
        img = _pass(img, 0, height)
    return np.ascontiguousarray(img)


# ---------------------------------------------------------------------------------------------------------------------
# monodepth2's ResnetEncoder(18) + DepthDecoder(scales=range(4)) in float64, from a state_dict

def _bn(x, sd, p):
    import torch.nn.functional as F
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"],
                        False, 0.0, 1e-5)


def _block(x, sd, p, stride):
    import torch.nn.functional as F
    y = F.relu(_bn(F.conv2d(x, sd[p + ".conv1.weight"], None, stride, 1), sd, p + ".bn1"))
    y = _bn(F.conv2d(y, sd[p + ".conv2.weight"], None, 1, 1), sd, p + ".bn2")
    if p + ".downsample.0.weight" in sd:
        x = _bn(F.conv2d(x, sd[p + ".downsample.0.weight"], None, stride, 0), sd, p + ".downsample.1")
    return F.relu(y + x)


def _pad_conv(x, sd, p):
    import torch.nn.functional as F
    return F.conv2d(F.pad(x, (1, 1, 1, 1), mode="reflect"), sd[p + ".weight"], sd[p + ".bias"])


def depth_net(state_dict, x):
    """disp0 [S,1,h,w] for the normalised input x [S,3,h,w], in float64 on the CPU.  state_dict: the encoder.pth and
    depth.pth tensors under their own keys (any dtype; cast to float64 here)."""
    import torch
    import torch.nn.functional as F
    sd = {k: torch.as_tensor(v).to(torch.float64) for k, v in state_dict.items() if torch.is_tensor(v)}
    x = torch.as_tensor(x).to(torch.float64)
    f0 = F.relu(_bn(F.conv2d(x, sd["encoder.conv1.weight"], None, 2, 3), sd, "encoder.bn1"))
    feats = [f0]
    y = F.max_pool2d(f0, 3, 2, 1)
    for li in range(4):
        for bi in range(2):
            y = _block(y, sd, f"encoder.layer{li + 1}.{bi}", 2 if (li > 0 and bi == 0) else 1)
        feats.append(y)
    y = feats[-1]
    for i in range(4, -1, -1):
        j = 2 * (4 - i)                          # ModuleList index of upconv(i, 0); upconv(i, 1) follows
        y = F.elu(_pad_conv(y, sd, f"decoder.{j}.conv.conv"))
        y = F.interpolate(y, scale_factor=2, mode="nearest")
        if i > 0:
            y = torch.cat([y, feats[i - 1]], 1)
        y = F.elu(_pad_conv(y, sd, f"decoder.{j + 1}.conv.conv"))
    return torch.sigmoid(_pad_conv(y, sd, "decoder.10.conv"))


def checkpoint_shapes():
    """(encoder tensor shapes, decoder tensor shapes) by key, as monodepth2's ResnetEncoder(18) / DepthDecoder
    state_dicts name them (torchvision ResNet-18 under "encoder.", nn.ModuleList under "decoder.")."""
    enc = {"encoder.conv1.weight": (64, 3, 7, 7)}

    def bn(p, c):
        enc.update({p + ".weight": (c,), p + ".bias": (c,), p + ".running_mean": (c,), p + ".running_var": (c,),
                    p + ".num_batches_tracked": ()})
    bn("encoder.bn1", 64)
    c_in = 64
    for li, c in enumerate((64, 128, 256, 512)):
        for bi in range(2):
            p = f"encoder.layer{li + 1}.{bi}"
            cin = c_in if bi == 0 else c
            enc[p + ".conv1.weight"] = (c, cin, 3, 3)
            bn(p + ".bn1", c)
            enc[p + ".conv2.weight"] = (c, c, 3, 3)
            bn(p + ".bn2", c)
            if bi == 0 and li > 0:
                enc[p + ".downsample.0.weight"] = (c, cin, 1, 1)
                bn(p + ".downsample.1", c)
        c_in = c
    enc["encoder.fc.weight"], enc["encoder.fc.bias"] = (1000, 512), (1000,)
    dec = {}
    j = 0
    for i in range(4, -1, -1):
        cin = ENC_CHANNELS[-1] if i == 4 else DEC_CHANNELS[i + 1]
        for cin_, cout in ((cin, DEC_CHANNELS[i]), (DEC_CHANNELS[i] + (ENC_CHANNELS[i - 1] if i > 0 else 0),
                                                    DEC_CHANNELS[i])):
            dec[f"decoder.{j}.conv.conv.weight"], dec[f"decoder.{j}.conv.conv.bias"] = (cout, cin_, 3, 3), (cout,)
            j += 1
    for s in range(4):
        dec[f"decoder.{10 + s}.conv.weight"], dec[f"decoder.{10 + s}.conv.bias"] = (1, DEC_CHANNELS[s], 3, 3), (1,)
    return enc, dec


def seeded_checkpoint(seed, height=192, width=640):
    """(encoder dict, decoder dict) of CPU float32 tensors drawn from numpy.random.default_rng(seed) in sorted key
    order: convolution and linear weights N(0, 1 / fan_in), norm weights 1 + N(0, 0.1^2), biases and running means
    N(0, 0.1^2), running variances U(0.5, 1.5), num_batches_tracked 0 (int64).  The encoder dict also holds the
    non-tensor entries monodepth2's trainer saves: height, width and use_stereo."""
    import torch
    rng = np.random.default_rng(seed)
    enc_s, dec_s = checkpoint_shapes()
    out = []
    for shapes in (enc_s, dec_s):
        d = {}
        for k in sorted(shapes):
            shp = shapes[k]
            if k.endswith("num_batches_tracked"):
                d[k] = torch.tensor(0, dtype=torch.int64)
                continue
            if k.endswith("running_var"):
                v = rng.uniform(0.5, 1.5, shp)
            elif k.endswith("running_mean") or k.endswith("bias"):
                v = rng.normal(0.0, 0.1, shp)
            elif len(shp) >= 2:
                v = rng.normal(0.0, 1.0 / math.sqrt(int(np.prod(shp[1:]))), shp)
            else:
                v = 1.0 + rng.normal(0.0, 0.1, shp)
            d[k] = torch.from_numpy(v.astype(np.float32))
        out.append(d)
    enc, dec = out
    enc.update(height=int(height), width=int(width), use_stereo=True)
    return enc, dec


def write_checkpoint(model_dir, seed, height=192, width=640):
    """seeded_checkpoint written as <model_dir>/encoder.pth and depth.pth with torch.save.  Returns model_dir."""
    import torch
    os.makedirs(model_dir, exist_ok=True)
    enc, dec = seeded_checkpoint(seed, height, width)
    torch.save(enc, os.path.join(model_dir, "encoder.pth"))
    torch.save(dec, os.path.join(model_dir, "depth.pth"))
    return model_dir


# ---------------------------------------------------------------------------------------------------------------------
# save_depth_map.py:84-102

def grid_generation(H, W):
    x = np.linspace(0, W - 1, W)
    y = np.linspace(0, H - 1, H)
    xv, yv = np.meshgrid(x, y)  # HxW
    meshgrid_np = np.stack((xv, yv, np.ones_like(xv)), axis=2)
    return meshgrid_np


def convert_depth_to_pointcloud(depth_np, K_np):
    """depth_np [H, W, 1] (float32 as the script has it), K_np [3, 3] in its stored dtype -> [3, H*W] float64."""
    H, W, _ = depth_np.shape
    K_inv_np = np.linalg.inv(K_np)  # 3x3
    meshgrid_np = grid_generation(H, W)  # HxWx1
    xyz_homo = depth_np * meshgrid_np
    xyz_homo = np.transpose(np.resize(xyz_homo, (H * W, 3)))
    pc_np = np.dot(K_inv_np, xyz_homo)
    return pc_np
