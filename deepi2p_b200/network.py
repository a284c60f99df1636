"""DeepI2P's classifier network (models/networks_united.py:14-210, KeypointDetector) built on the project's ops.

The parameters and buffers are exactly the reference's `KeypointDetector(opt).state_dict()`, so a checkpoint written
by MMClassifer.save_network loads with `load_checkpoint`.  Every non-convolution step of the forward is a project op
(DESIGN.md 4.18): cluster_assign_forward for the clustering and the interpolation searches, cluster_max_pool,
knn_group, upsample_by_interpolation and attention_fusion.  No B x N x M or B x C x P x M tensor is built.  What
stays in torch is the convolutions and norms (cuDNN), torch.cat, the two max over the K neighbours of the node kNN
module and the global max over the nodes; their backwards write distinct indices, so they use no float atomics.

The image branch is a ResNet-34 (the reference's models/resnet.py) returning the stride-16 and stride-32 maps; its
global feature is the mean over H and W, which equals AdaptiveAvgPool2d((1, 1)) but has a deterministic CUDA
backward.  ResNet weights come only from an optional local file with torchvision's key layout; constructing the model
touches neither CUDA nor the network.

    model = network.KeypointDetector(**network.SHAPES["kitti"]).cuda()
    network.load_checkpoint(model, "checkpoints/best.pth")
    coarse, fine = model(pc, intensity, sn, node_a, node_b, img)
    coarse_pred, fine_pred = network.predict(coarse, fine)
"""
import math
import os
import types

import torch
import torch.nn as nn

from . import classifier, frustum, point_ops

# the image sizes of the shipped option sets (kitti/options.py, oxford/options.py, nuscenes_t/options.py); all three
# use fine_scale 32, 20480 points, 128 / 128 nodes, k_ab 16, k = 3, BatchNorm and ReLU
SHAPES = {"kitti": dict(img_H=160, img_W=512), "oxford": dict(img_H=384, img_W=640),
          "nuscenes": dict(img_H=160, img_W=320)}

# forward chunk of classify_and_register: at the Oxford shape (20480 points, 384 x 640) one chunk of 64 samples peaks
# at 13.5 GB above the inputs on an H100 (BENCH_E2E.json, DESIGN.md 4.18)
DEFAULT_CHUNK = 64


def _check_menu(normalization, activation):
    if normalization != "batch":
        raise ValueError(f"normalization must be 'batch' (every shipped option set uses it), got {normalization!r}")
    if activation != "relu":
        raise ValueError(f"activation must be 'relu' (every shipped option set uses it), got {activation!r}")


def _point_init(conv):
    """The reference's point-layer rule (layers_pc.py:157-175, :304-322): weights N(0, sqrt(2 / n)) with n = kernel
    area x in_channels, biases 0.  Norm layers keep torch's weight 1, bias 0."""
    n = conv.in_channels
    for k in conv.kernel_size:
        n *= k
    nn.init.normal_(conv.weight, 0.0, math.sqrt(2.0 / n))
    if conv.bias is not None:
        nn.init.zeros_(conv.bias)


class _PointLayer(nn.Module):
    """1x1 convolution (Conv1d over [B,C,N] or Conv2d over [B,C,M,K]), then BatchNorm, ReLU and Dropout where asked:
    the reference's EquivariantLayer (layers_pc.py:259-342) and MyConv2d (:110-190) with their shipped menu."""

    def __init__(self, c_in, c_out, norm_act, momentum=0.1, dropout=None, dims=1):
        super().__init__()
        Conv, Norm = (nn.Conv1d, nn.BatchNorm1d) if dims == 1 else (nn.Conv2d, nn.BatchNorm2d)
        self.conv = Conv(c_in, c_out, kernel_size=1)
        self.norm = Norm(c_out, momentum=momentum) if norm_act else None
        self.act = nn.ReLU() if norm_act else None
        self.dropout = nn.Dropout(p=dropout) if dropout is not None and 0 < dropout < 1 else None
        _point_init(self.conv)

    def forward(self, x):
        x = self.conv(x)
        if self.norm is not None:
            x = self.act(self.norm(x))
        if self.dropout is not None:
            x = self.dropout(x)
        return x


class _PointNet(nn.Module):
    """A chain of _PointLayer (layers_pc.py:345-408): BatchNorm + ReLU on every layer, on the last one only with
    norm_act_at_last."""

    def __init__(self, c_in, c_outs, norm_act_at_last, momentum=0.1, dropouts=None):
        super().__init__()
        dropouts = dropouts or [None] * len(c_outs)
        self.layers = nn.ModuleList()
        for i, c in enumerate(c_outs):
            last = i == len(c_outs) - 1
            self.layers.append(_PointLayer(c_in, c, norm_act_at_last or not last, momentum, dropouts[i]))
            c_in = c

    def forward(self, x):
        for layer in self.layers:
            x = layer(x)
        return x


class _KnnFusion(nn.Module):
    """The node kNN module (GeneralKNNFusionModule, layers_pc.py:756-818): group the K nearest database nodes of each
    query (point_ops.knn_group), 1x1 convolutions, max over K, concatenate the max back, convolutions, max over K."""

    def __init__(self, c_in, c_before, c_after, momentum=0.1):
        super().__init__()
        self.layers_before = nn.ModuleList()
        for c in c_before:
            self.layers_before.append(_PointLayer(c_in, c, True, momentum, dims=2))
            c_in = c
        c_in *= 2
        self.layers_after = nn.ModuleList()
        for c in c_after:
            self.layers_after.append(_PointLayer(c_in, c, True, momentum, dims=2))
            c_in = c

    def forward(self, query, database, database_features, K):
        _, x = point_ops.knn_group(query, database, database_features, K)      # [B,3+C,M,K]
        for layer in self.layers_before:
            x = layer(x)
        pooled = torch.max(x, dim=3, keepdim=True)[0]
        y = torch.cat((pooled.expand_as(x), x), dim=1)
        for layer in self.layers_after:
            y = layer(y)
        return torch.max(y, dim=3)[0]                                           # [B,C,M]


class _PCEncoder(nn.Module):
    """Parameters of PCEncoder (networks_pc.py:15-45, Ca 64, Cb 256, Cg 512); KeypointDetector.forward runs it."""

    def __init__(self, momentum=0.1, Ca=64, Cb=256, Cg=512):
        super().__init__()
        self.first_pointnet = _PointNet(3 + 1 + 3, [Ca // 2] * 3, True, momentum)
        self.second_pointnet = _PointNet(Ca, [Ca, Ca], True, momentum)
        self.knnlayer = _KnnFusion(3 + Ca, (Cb, Cb), (Cb * 2, Cb), momentum)
        self.final_pointnet = _PointNet(3 + Cb, [Cg // 2, Cg], True, momentum)


class _BasicBlock(nn.Module):
    def __init__(self, c_in, c_out, stride):
        super().__init__()
        self.conv1 = nn.Conv2d(c_in, c_out, 3, stride, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(c_out)
        self.relu = nn.ReLU(inplace=True)
        self.conv2 = nn.Conv2d(c_out, c_out, 3, 1, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(c_out)
        self.downsample = None
        if stride != 1 or c_in != c_out:
            self.downsample = nn.Sequential(nn.Conv2d(c_in, c_out, 1, stride, bias=False), nn.BatchNorm2d(c_out))

    def forward(self, x):
        y = self.relu(self.bn1(self.conv1(x)))
        y = self.bn2(self.conv2(y))
        return self.relu(y + (x if self.downsample is None else self.downsample(x)))


class _ResNet34(nn.Module):
    """ResNet-34 with torchvision's parameter names (the reference's models/resnet.py), returning the stride-16 and
    stride-32 maps.  fc is unused but kept: it is part of the reference's state_dict."""

    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 64, 7, 2, 3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(3, 2, 1)
        c_in = 64
        for i, (c, n, s) in enumerate(((64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2))):
            setattr(self, f"layer{i + 1}", nn.Sequential(*[_BasicBlock(c_in if j == 0 else c, c, s if j == 0 else 1)
                                                           for j in range(n)]))
            c_in = c
        self.fc = nn.Linear(512, 1000)
        for m in self.modules():                    # the reference's ResNet rule (models/resnet.py:154-159)
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")

    def forward(self, x):
        x = self.maxpool(self.relu(self.bn1(self.conv1(x))))
        s16 = self.layer3(self.layer2(self.layer1(x)))
        return s16, self.layer4(s16)


class _ImageEncoder(nn.Module):
    def __init__(self):
        super().__init__()
        self.backbone = _ResNet34()


def _resnet_map_size(H, W, stride):
    """(h, w) of ResNet-34's stride-16 or stride-32 map for an H x W image: conv1 and the max-pool, then one stride-2
    3x3 convolution per stage after the first."""
    def down(n, k, p):
        return (n + 2 * p - k) // 2 + 1
    h, w = down(down(H, 7, 3), 3, 1), down(down(W, 7, 3), 3, 1)
    for _ in range({16: 2, 32: 3}[stride]):
        h, w = down(h, 3, 1), down(w, 3, 1)
    return h, w


class KeypointDetector(nn.Module):
    """The classifier network: (pc [B,3,N], intensity [B,1,N], sn [B,3,N], node_a [B,3,Ma], node_b [B,3,Mb],
    img [B,3,H,W]) float32 CUDA -> coarse scores [B,2,N] and, with fine=True, fine scores [B,L,N], L = H_f * W_f.
    Both are channel slices of one [B,2+L,N] tensor, which classifier.classifier_loss reads without a copy.

    The stride-32 map must have H_f x W_f = round(H / fine_scale) x round(W / fine_scale) pixels and the stride-16 map
    four times as many, because the attention PointNets give one weight per pixel; the shipped sizes do.  Only
    normalization='batch' and activation='relu' are supported.  resnet_weights: optional path of a torchvision-layout
    ResNet-34 state_dict (e.g. resnet34-333f7ec4.pth) for the image backbone; without it the backbone starts from the
    reference's initialisation.  Construction runs on the CPU and reads nothing but that file."""

    def __init__(self, img_H=160, img_W=512, fine_scale=32, fine=True, node_a_num=128, node_b_num=128, k_ab=16,
                 k_interp_ab=3, k_interp_point_a=3, k_interp_point_b=3, normalization="batch", activation="relu",
                 norm_momentum=0.1, resnet_weights=None):
        super().__init__()
        _check_menu(normalization, activation)
        H_f, W_f = classifier.fine_grid(img_H, img_W, fine_scale)
        L = H_f * W_f
        s32, s16 = _resnet_map_size(img_H, img_W, 32), _resnet_map_size(img_H, img_W, 16)
        if L < 1 or s32[0] * s32[1] != L or s16[0] * s16[1] != 4 * L:
            raise ValueError(f"a {img_H} x {img_W} image gives {s32[0]} x {s32[1]} stride-32 and {s16[0]} x {s16[1]} "
                             f"stride-16 maps, but the fine grid of scale {fine_scale} is {H_f} x {W_f}: the "
                             f"stride-32 map must have H_f * W_f pixels and the stride-16 map four times as many")
        self.img_H, self.img_W, self.fine_scale, self.fine = int(img_H), int(img_W), fine_scale, bool(fine)
        self.node_a_num, self.node_b_num = int(node_a_num), int(node_b_num)
        self.k_ab, self.k_interp_ab = int(k_ab), int(k_interp_ab)
        self.k_interp_point_a, self.k_interp_point_b = int(k_interp_point_a), int(k_interp_point_b)
        m = norm_momentum

        self.pc_encoder = _PCEncoder(m)
        self.img_encoder = _ImageEncoder()
        self.node_b_attention_pn = _PointNet(256 + 512, [256, L], False, m)
        self.node_b_pn = _PointNet(256 + 512 + 512 + 512, [1024, 512, 512], False, m)
        self.node_a_attention_pn = _PointNet(64 + 512, [256, 4 * L], False, m)
        self.node_a_pn = _PointNet(64 + 256 + 512, [512, 128, 128], False, m)
        head = [256, 256, 2 + L] if self.fine else [128, 128, 2]
        self.per_point_pn = _PointNet(32 + 64 + 128 + 512, head, False, m, dropouts=[0.5, 0.5, 0])
        if resnet_weights is not None:
            sd = torch.load(os.fspath(resnet_weights), map_location="cpu", weights_only=True)
            self.img_encoder.backbone.load_state_dict(sd, strict=True)

    def forward(self, pc, intensity, sn, node_a, node_b, img):
        B, Ma, Mb = pc.shape[0], node_a.shape[2], node_b.shape[2]
        # the coordinates get no gradient in the reference (every use is detached); the ops require that
        pc, node_a, node_b = (t.detach().contiguous() for t in (pc, node_a, node_b))
        enc = self.pc_encoder

        # point encoder (networks_pc.py:58-115)
        ca = point_ops.cluster_assign_forward(pc, node_a, k=self.k_interp_point_a)
        min_idx = ca["min_idx"]
        first_pn_out = enc.first_pointnet(torch.cat((ca["pc_decentered"], intensity, sn), dim=1))
        _, scattered = point_ops.cluster_max_pool(first_pn_out, min_idx, Ma, broadcast=True)
        second_pn_out = enc.second_pointnet(torch.cat((first_pn_out, scattered), dim=1))
        node_a_features = point_ops.cluster_max_pool(second_pn_out, min_idx, Ma)
        node_b_features = enc.knnlayer(node_b, ca["cluster_mean"], node_a_features, self.k_ab)
        final_pn_out = enc.final_pointnet(torch.cat((node_b, node_b_features), dim=1))
        global_feature = torch.max(final_pn_out, dim=2, keepdim=True)[0]            # [B,Cg,1]

        # image encoder: the global feature is the mean over H and W (= AdaptiveAvgPool2d((1, 1)))
        s16, s32 = self.img_encoder.backbone(img)
        img_global = s32.mean(dim=(2, 3))                                           # [B,C_img]
        C_img = img_global.shape[1]
        s16 = s16.reshape(B, s16.shape[1], -1).contiguous()
        s32 = s32.reshape(B, C_img, -1).contiguous()
        img_global_a = img_global.unsqueeze(2).expand(B, C_img, Ma)
        img_global_b = img_global.unsqueeze(2).expand(B, C_img, Mb)

        # node_b: attention over the stride-32 map, then the node_b PointNet (networks_united.py:147-155)
        att_b = self.node_b_attention_pn(torch.cat((node_b_features, img_global_b), dim=1))
        weighted_s32 = point_ops.attention_fusion(s32, att_b)
        up_node_b_features = self.node_b_pn(torch.cat((node_b_features, global_feature.expand(B, -1, Mb),
                                                       weighted_s32, img_global_b), dim=1))

        # decoder (networks_united.py:158-197)
        pb_idx = point_ops.cluster_assign_forward(pc, node_b, k=self.k_interp_point_b, want_centers=False)["min_k_idx"]
        pb = point_ops.upsample_by_interpolation(pb_idx, pc, node_b, up_node_b_features)
        att_a = self.node_a_attention_pn(torch.cat((node_a_features, img_global_a), dim=1))
        weighted_s16 = point_ops.attention_fusion(s16, att_a)
        ab_idx = point_ops.cluster_assign_forward(node_a, node_b, k=self.k_interp_ab, want_centers=False)["min_k_idx"]
        ab = point_ops.upsample_by_interpolation(ab_idx, node_a, node_b, up_node_b_features)
        up_node_a_features = self.node_a_pn(torch.cat((node_a_features, ab, weighted_s16), dim=1))
        pa = point_ops.upsample_by_interpolation(ca["min_k_idx"], pc, node_a, up_node_a_features)
        scores = self.per_point_pn(torch.cat((pa, pb, first_pn_out, second_pn_out), dim=1))
        if self.fine:
            return scores[:, 0:2, :], scores[:, 2:, :]
        return scores[:, 0:2, :]


def load_checkpoint(model, path_or_dict):
    """Load what MMClassifer.save_network wrote (torch.save of the detector's state_dict, with the `module.` prefix
    when it was trained under DataParallel) into `model`, strictly.  A missing or unexpected key raises KeyError
    naming the keys; a shape mismatch raises torch's RuntimeError.  Returns the model."""
    if isinstance(path_or_dict, (str, os.PathLike)):
        sd = torch.load(os.fspath(path_or_dict), map_location="cpu", weights_only=True)
    else:
        sd = path_or_dict
    if sd and all(k.startswith("module.") for k in sd):                  # util/pytorch_helper.py:5-33
        sd = {k[len("module."):]: v for k, v in sd.items()}
    want = set(model.state_dict())
    missing, unexpected = sorted(want - set(sd)), sorted(set(sd) - want)
    if missing or unexpected:
        raise KeyError(f"checkpoint does not match the model: missing keys {missing}, unexpected keys {unexpected}")
    model.load_state_dict(sd, strict=True)
    return model


def predict(coarse, fine=None):
    """Per-point predictions by torch.max's rule (first maximal index, NaN maximal), the rule classifier_loss applies:
    coarse [B,2,N] -> int8 [B,N] (1 = inside the image), fine [B,L,N] -> int32 [B,N] (the cell), or None.  These are
    the dtypes frustum.register_batch and pnp.pnp_ransac_batch take."""
    coarse_pred = torch.argmax(coarse, dim=1).to(torch.int8)
    fine_pred = torch.argmax(fine, dim=1).to(torch.int32) if fine is not None else None
    return coarse_pred, fine_pred


def fold_pointnet(pointnet, dtype=torch.float32):
    """The layers of a _PointNet as plain affine maps for inference: [(W [C_out,C_in], b [C_out], relu)] with each
    layer's eval-mode BatchNorm folded in float64, W' = W * gamma / sqrt(var + eps) per output row and b' = (b - mean)
    * gamma / sqrt(var + eps) + beta, then rounded once to `dtype`.  Dropout is the identity in eval mode.  The
    tensors are new (detached) and live on the pointnet's device: what point_ops.pointwise_mlp takes."""
    out = []
    for layer in pointnet.layers:
        conv, norm = layer.conv, layer.norm
        W = conv.weight.detach().double().reshape(conv.out_channels, conv.in_channels)
        b = conv.bias.detach().double() if conv.bias is not None else W.new_zeros(conv.out_channels)
        if norm is not None:
            scale = norm.weight.detach().double() / torch.sqrt(norm.running_var.detach().double() + norm.eps)
            W = W * scale.unsqueeze(1)
            b = (b - norm.running_mean.detach().double()) * scale + norm.bias.detach().double()
        out.append((W.to(dtype).contiguous(), b.to(dtype).contiguous(), layer.act is not None))
    return out


def fold_knn_fusion(module, dtype=torch.float32):
    """The layers of a _KnnFusion as plain affine maps for inference: (before, after), each [(W [C_out,C_in], b
    [C_out], relu)] folded as fold_pointnet does (eval-mode BatchNorm in float64, rounded once to `dtype`).  The first
    after layer keeps its 2 C_b input columns, the per-node max first: what point_ops.knn_fusion takes."""
    return (fold_pointnet(types.SimpleNamespace(layers=module.layers_before), dtype),
            fold_pointnet(types.SimpleNamespace(layers=module.layers_after), dtype))


class FusedInference:
    """Inference through KeypointDetector with its per-point layers fused (DESIGN.md 4.21): first_pointnet,
    second_pointnet and the decoder's two per-point interpolations + concatenation + per_point_pn + predict each run
    as one point_ops.pointwise_mlp call, so no [B,C,N] tensor wider than 64 channels is built.  Everything else (the
    node-level layers, ResNet, and with the default encoder="torch" the kNN module and final_pointnet) is the model's
    own code.  encoder="fused" also runs the point encoder's kNN module as one point_ops.knn_fusion call and
    final_pointnet + the max over the nodes as one point_ops.pointwise_mlp_max call (DESIGN.md 4.26), so no
    [B,C,Mb,K] tensor and no [B,512,Mb] tensor is built.  decoder="fused" runs the decoder's four node-level
    PointNets (node_b_attention_pn, node_b_pn, node_a_attention_pn, node_a_pn) as one point_ops.node_mlp call each
    (DESIGN.md 4.27): the per-sample inputs (img_global, global_feature) are projected once per sample instead of
    being expanded and concatenated.  attention_fusion and the ab interpolation stay the project's exact ops.

    The fused layers compute in TF32 whatever torch's TF32 flags say, with BatchNorm folded into the weights, so the
    scores differ from model.forward's at rounding level and a prediction can differ where the top two scores nearly
    tie.  Inference only: classify raises under grad mode.  The folded layers are cached and rebuilt when a parameter
    or buffer they were read from has changed (load_state_dict, an optimizer step, .to())."""

    _CHAINS = (("first", lambda m: m.pc_encoder.first_pointnet, ((3, 0, 0), (1, 0, 0), (3, 0, 0))),
               ("second", lambda m: m.pc_encoder.second_pointnet, ((32, 0, 0), (32, 0, 0))),
               ("head", lambda m: m.per_point_pn, None))

    ENCODERS = ("torch", "fused")
    DECODERS = ("torch", "fused")

    # node-level PointNets of the decoder: the (channels, per sample) of their input rows, in torch.cat's order
    _NODE_CHAINS = {"att_b": (lambda m: m.node_b_attention_pn, ((256, False), (512, True))),
                    "node_b": (lambda m: m.node_b_pn, ((256, False), (512, True), (512, False), (512, True))),
                    "att_a": (lambda m: m.node_a_attention_pn, ((64, False), (512, True))),
                    "node_a": (lambda m: m.node_a_pn, ((64, False), (512, False), (256, False)))}

    def __init__(self, model, encoder="torch", decoder="torch"):
        if not isinstance(model, KeypointDetector):
            raise TypeError("FusedInference wraps a network.KeypointDetector")
        if encoder not in self.ENCODERS:
            raise ValueError(f"encoder must be one of {self.ENCODERS}, got {encoder!r}")
        if decoder not in self.DECODERS:
            raise ValueError(f"decoder must be one of {self.DECODERS}, got {decoder!r}")
        self.model, self.encoder, self.decoder = model, encoder, decoder
        self._packed, self._stamp = {}, {}

    def _cached(self, name, module, pack):
        tensors = list(module.parameters()) + list(module.buffers())
        stamp = tuple((t.data_ptr(), t._version) for t in tensors)
        if self._stamp.get(name) != stamp:
            self._packed[name] = pack()
            self._stamp[name] = stamp
        return self._packed[name]

    def _chain(self, name):
        model = self.model
        enc = model.pc_encoder
        if name == "knn":
            C = enc.knnlayer.layers_before[0].conv.in_channels - 3
            return self._cached(name, enc.knnlayer,
                                lambda: point_ops.pack_knn_fusion(C, *fold_knn_fusion(enc.knnlayer)))
        if name == "final":
            pn = enc.final_pointnet
            return self._cached(name, pn, lambda: point_ops.pack_pointwise_mlp_max(pn.layers[0].conv.in_channels,
                                                                                     fold_pointnet(pn)))
        if name in self._NODE_CHAINS:
            get, spec = self._NODE_CHAINS[name]
            pn = get(model)
            return self._cached(name, pn, lambda: point_ops.pack_node_mlp(spec, fold_pointnet(pn)))
        _, get, spec = next(c for c in self._CHAINS if c[0] == name)
        if spec is None:
            spec = ((128, model.node_a_num, model.k_interp_point_a), (512, model.node_b_num, model.k_interp_point_b),
                    (32, 0, 0), (64, 0, 0))
        pn = get(model)
        return self._cached(name, pn, lambda: point_ops.pack_pointwise_mlp(spec, fold_pointnet(pn)))

    def classify(self, pc, intensity, sn, node_a, node_b, img, return_scores=False):
        """(pc [B,3,N], intensity [B,1,N], sn [B,3,N], node_a [B,3,Ma], node_b [B,3,Mb], img [B,3,H,W]) float32 CUDA ->
        (coarse_pred int8 [B,N], fine_pred int32 [B,N] or None for a coarse-only model), the dtypes
        frustum.register_batch and pnp.pnp_ransac_batch take; with return_scores=True the scores [B,2+L,N] come third.
        Runs the model's layers in eval mode (the training flag is restored) under no_grad."""
        if torch.is_grad_enabled():
            raise RuntimeError("FusedInference.classify is inference only: call it under torch.no_grad()")
        model = self.model
        was_training = model.training
        model.eval()
        try:
            return self._classify(pc, intensity, sn, node_a, node_b, img, return_scores)
        finally:
            model.train(was_training)

    def _classify(self, pc, intensity, sn, node_a, node_b, img, return_scores):
        model, enc = self.model, self.model.pc_encoder
        B, Ma, Mb = pc.shape[0], node_a.shape[2], node_b.shape[2]
        if (Ma, Mb) != (model.node_a_num, model.node_b_num):
            raise ValueError(f"node_a / node_b have {Ma} / {Mb} nodes, the model was built for {model.node_a_num} / "
                             f"{model.node_b_num}")
        pc, node_a, node_b = (t.detach().contiguous() for t in (pc, node_a, node_b))
        ca = point_ops.cluster_assign_forward(pc, node_a, k=model.k_interp_point_a)
        min_idx = ca["min_idx"]
        first_pn_out = point_ops.pointwise_mlp([ca["pc_decentered"], intensity, sn], self._chain("first"))
        _, scattered = point_ops.cluster_max_pool(first_pn_out, min_idx, Ma, broadcast=True)
        second_pn_out = point_ops.pointwise_mlp([first_pn_out, scattered], self._chain("second"))
        del scattered
        node_a_features = point_ops.cluster_max_pool(second_pn_out, min_idx, Ma)
        if self.encoder == "fused":
            node_b_features = point_ops.knn_fusion(node_b, ca["cluster_mean"], node_a_features, model.k_ab,
                                                   self._chain("knn"))
            global_feature = point_ops.pointwise_mlp_max([node_b, node_b_features], self._chain("final"))
        else:
            node_b_features = enc.knnlayer(node_b, ca["cluster_mean"], node_a_features, model.k_ab)
            final_pn_out = enc.final_pointnet(torch.cat((node_b, node_b_features), dim=1))
            global_feature = torch.max(final_pn_out, dim=2, keepdim=True)[0]

        s16, s32 = model.img_encoder.backbone(img)
        img_global = s32.mean(dim=(2, 3))
        C_img = img_global.shape[1]
        s16 = s16.reshape(B, s16.shape[1], -1).contiguous()
        s32 = s32.reshape(B, C_img, -1).contiguous()
        img_global_a = img_global.unsqueeze(2).expand(B, C_img, Ma)
        img_global_b = img_global.unsqueeze(2).expand(B, C_img, Mb)

        if self.decoder == "fused":
            node = lambda name, sources: point_ops.node_mlp(sources, self._chain(name))
            g = global_feature[:, :, 0]
            att_b = node("att_b", [node_b_features, img_global])
            weighted_s32 = point_ops.attention_fusion(s32, att_b)
            up_node_b_features = node("node_b", [node_b_features, g, weighted_s32, img_global])
        else:
            att_b = model.node_b_attention_pn(torch.cat((node_b_features, img_global_b), dim=1))
            weighted_s32 = point_ops.attention_fusion(s32, att_b)
            up_node_b_features = model.node_b_pn(torch.cat((node_b_features, global_feature.expand(B, -1, Mb),
                                                            weighted_s32, img_global_b), dim=1))
        pb_idx = point_ops.cluster_assign_forward(pc, node_b, k=model.k_interp_point_b,
                                                  want_centers=False)["min_k_idx"]
        if self.decoder == "fused":
            att_a = node("att_a", [node_a_features, img_global])
        else:
            att_a = model.node_a_attention_pn(torch.cat((node_a_features, img_global_a), dim=1))
        weighted_s16 = point_ops.attention_fusion(s16, att_a)
        ab_idx = point_ops.cluster_assign_forward(node_a, node_b, k=model.k_interp_ab,
                                                  want_centers=False)["min_k_idx"]
        ab = point_ops.upsample_by_interpolation(ab_idx, node_a, node_b, up_node_b_features)
        if self.decoder == "fused":
            up_node_a_features = node("node_a", [node_a_features, ab, weighted_s16])
        else:
            up_node_a_features = model.node_a_pn(torch.cat((node_a_features, ab, weighted_s16), dim=1))

        # the decoder's per-point half in one call: rows (pa, pb, first_pn_out, second_pn_out) of per_point_pn's input
        wa, ia = point_ops.interpolation_weights(ca["min_k_idx"], pc, node_a)
        wb, ib = point_ops.interpolation_weights(pb_idx, pc, node_b)
        return point_ops.pointwise_mlp([(up_node_a_features, wa, ia), (up_node_b_features, wb, ib), first_pn_out,
                                        second_pn_out], self._chain("head"), output="argmax", c_split=2,
                                       return_scores=return_scores)


HEADS = ("torch", "fused", "fused_encoder", "fused_all")


def classify_and_register(model, pc, intensity, sn, node_a, node_b, img, K, chunk=DEFAULT_CHUNK, n_inits=60, seed=0,
                          t_lb=frustum.DEFAULT_T_LB, t_ub=frustum.DEFAULT_T_UB, head="torch"):
    """Classify an assembled batch and register every sample: visualize_and_save_data.py's forward and
    registration_lsq.py's solve in one call, with nothing going to the host or to files.

    pc [S,3,N] (N a multiple of 16, as the loaders' 20480), intensity [S,1,N], sn [S,3,N], node_a [S,3,Ma],
    node_b [S,3,Mb], img [S,3,H,W] float32 CUDA (assemble.assemble_batch / imageprep.assemble_images outputs) and K
    [S,3,3] or [3,3].  The forward runs in eval mode under no_grad over chunks of `chunk` samples (BatchNorm uses its
    running statistics, so chunking does not change the maths; cuDNN may pick other algorithms per chunk size, which
    changes rounding only); the model's training flag is restored afterwards.  The coarse predictions go to
    frustum.register_batch with registration_lsq.py's settings (n_inits starts, 2-D, the t bounds of :340).

    head selects a numeric contract, not a tuning.  "torch" (the default) is model.forward and network.predict: the
    convolutions are cuDNN's and honour torch's TF32 flags.  "fused" is FusedInference.classify per chunk: the
    per-point layers run as fused TF32 tensor-core kernels whatever the flags say, so predictions can differ from
    "torch" at points whose top two scores nearly tie.  "fused_encoder" is FusedInference(model, encoder="fused")
    per chunk: the point encoder's kNN module and final_pointnet + max run fused in TF32 too.  "fused_all" is
    FusedInference(model, encoder="fused", decoder="fused") per chunk: the decoder's node-level PointNets run fused in
    TF32 as well, so only ResNet keeps separate convolution / BatchNorm / ReLU kernels.

    Returns dict(P [S,4,4] f64, cost [S] f64, coarse_pred int8 [S,N], fine_pred int32 [S,N] or None, degenerate
    int32 [S]); a sample with no point predicted inside gets P = I, cost 1e4 and degenerate = 1."""
    S, N = pc.shape[0], pc.shape[2]
    chunk = int(chunk)
    if chunk < 1:
        raise ValueError(f"chunk must be >= 1, got {chunk}")
    if head not in HEADS:
        raise ValueError(f"head must be one of {HEADS}, got {head!r}")
    fused = FusedInference(model, encoder="fused" if head in ("fused_encoder", "fused_all") else "torch",
                           decoder="fused" if head == "fused_all" else "torch") if head != "torch" else None
    for t, name in ((intensity, "intensity"), (sn, "sn"), (node_a, "node_a"), (node_b, "node_b"), (img, "img")):
        if t.shape[0] != S:
            raise ValueError(f"{name} has {t.shape[0]} samples, pc has {S}")
    H, W = img.shape[2], img.shape[3]
    was_training = model.training
    model.eval()
    try:
        with torch.no_grad():
            coarse_pred = torch.empty((S, N), dtype=torch.int8, device=pc.device)
            fine_pred = torch.empty((S, N), dtype=torch.int32, device=pc.device) if model.fine else None
            for a in range(0, S, chunk):
                b = min(a + chunk, S)
                args = (pc[a:b], intensity[a:b], sn[a:b], node_a[a:b], node_b[a:b], img[a:b])
                if fused is not None:
                    out = None
                    c, f = fused.classify(*args)
                else:
                    out = model(*args)
                    c, f = predict(*out) if model.fine else predict(out)
                coarse_pred[a:b] = c
                if fine_pred is not None:
                    fine_pred[a:b] = f
                del out
    finally:
        model.train(was_training)
    reg = frustum.register_batch(pc.contiguous(), coarse_pred, N, K, H, W, n_inits=n_inits, seed=seed, t_lb=t_lb,
                                 t_ub=t_ub, is_2d=True)
    return dict(P=reg["P"], cost=reg["cost"], coarse_pred=coarse_pred, fine_pred=fine_pred,
                degenerate=reg["degenerate"])
