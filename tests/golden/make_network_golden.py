"""Writes tests/golden/network_small.npz: the REFERENCE's own KeypointDetector (models/networks_united.py), imported
by path from a DeepI2P checkout and run on the CPU, on seeded weights and inputs.  Needs the checkout and the
reference's index_max extension built into oracle/_ref/ (oracle/build_ref.py); no GPU, no network:

    python oracle/build_ref.py && python tests/golden/make_network_golden.py [OUT.npz] [--reference DIR]

How the reference runs here without edits:
  - opt.device = cpu; `torch.cuda.device(-1)`, which networks_pc.py enters around index_max, is a no-op;
  - `index_max.forward_cuda_shared_mem` is the reference's own `forward_cpu` (on float32 data in the float64 run);
  - models/resnet.py imports `torchvision.models.utils.load_state_dict_from_url`, which current torchvision lacks: a
    stub module returns the state_dict of a freshly built ResNet-34 (the seeded weights replace it anyway), and every
    socket connect raises, so no code path can reach a URL.

Stored (the inputs are not: synthetic.make_network_inputs(INPUT_SEED, ...) regenerates them, and `input_sums` holds
the float64 sum of each input and loss weight so that a change of the generator is caught):
  keys_<shape>_<head>   "key:d0,d1,..." for every state_dict entry, at the kitti / oxford / nuscenes sizes and the
                        fine / coarse heads (20480 points, 128 / 128 nodes, k_ab 16, k 3, scale 32);
  at the small shape (B 2, N 2048, 128 / 128 nodes, a 64 x 128 image: L = 8, the s16 map is 4 x 8 = 4L), from the
  reference in float64, with spread_<name> = max|ref32 - ref64| over the same entries from its float32 run:
    eval_coarse, eval_fine       eval-mode scores (BatchNorm on the seeded running statistics);
    train_coarse, train_fine     train-mode scores (BatchNorm on batch statistics, Dropout in eval mode);
    grad_<i>                     train-mode gradients of sum(coarse * lw_coarse) + sum(fine * lw_fine) with respect to
                                 GRAD_KEYS[i].
  The scores are kept at every point_stride-th point ([..., ::point_stride]) and the gradients at every
  grad_stride[i]-th entry of the flattened tensor (at most GRAD_ENTRIES of them): the forward and backward still run
  over all 2048 points, and every point feeds every gradient entry, so the kept entries see every step of the path.
The float64 run (index_max's arg-max still on float32 data) is the reference the GPU test measures against; the
float32 run's distance from it sets the GPU test's tolerance.  Weights: synthetic.seeded_state_dict(model, WEIGHT_SEED).
Data are continuous random values, so no kNN, arg-min or arg-max ties occur (the maker checks the kNN margins).
"""
import copy
import os
import socket
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import build_ref  # noqa: E402
from deepi2p_b200 import synthetic as syn  # noqa: E402

SHAPES = {"kitti": (160, 512), "oxford": (384, 640), "nuscenes": (160, 320)}
SMALL = dict(B=2, N=2048, Ma=128, Mb=128, H=64, W=128)
WEIGHT_SEED = 20261016
INPUT_SEED = 7
POINT_STRIDE = 8
GRAD_ENTRIES = 2048
GRAD_KEYS = ("img_encoder.backbone.conv1.weight", "pc_encoder.first_pointnet.layers.0.conv.weight",
             "pc_encoder.knnlayer.layers_before.0.conv.weight", "node_b_attention_pn.layers.1.conv.weight",
             "node_a_attention_pn.layers.1.conv.weight", "per_point_pn.layers.2.conv.weight")


def _no_network(*args, **kwargs):
    raise RuntimeError("make_network_golden: network access attempted")


def import_reference(ref_dir):
    socket.socket.connect = _no_network
    socket.socket.connect_ex = _no_network
    socket.create_connection = _no_network
    import torchvision.models

    def load_state_dict_from_url(url, progress=True, **kwargs):
        return torchvision.models.resnet34(weights=None).state_dict()

    stub = types.ModuleType("torchvision.models.utils")
    stub.load_state_dict_from_url = load_state_dict_from_url
    sys.modules["torchvision.models.utils"] = stub
    ref_im = build_ref.load("index_max")
    im = types.ModuleType("index_max")
    im.forward_cuda_shared_mem = lambda data, index, K: ref_im.forward_cpu(data.float().contiguous(), index, K)
    sys.modules["index_max"] = im
    sys.path.insert(0, ref_dir)
    from models import networks_united
    return networks_united


class Opt:
    def __init__(self, H, W, fine, N=20480, Ma=128, Mb=128, B=8):
        self.device = torch.device("cpu")
        self.img_H, self.img_W, self.img_fine_resolution_scale = H, W, 32
        self.is_fine_resolution = fine
        self.input_pt_num, self.node_a_num, self.node_b_num = N, Ma, Mb
        self.k_ab, self.k_interp_ab, self.k_interp_point_a, self.k_interp_point_b = 16, 3, 3, 3
        self.batch_size = B
        self.normalization, self.norm_momentum, self.activation = "batch", 0.1, "relu"


def key_list(model):
    return np.array([k + ":" + ",".join(str(d) for d in v.shape) for k, v in model.state_dict().items()])


def knn_margin(q, d, k):
    """Smallest relative gap between the k-th and (k+1)-th nearest distances (and within the first k) over all
    queries: the searches are unambiguous when it is far above float32 rounding."""
    dist = np.sqrt(((q[:, :, :, None].astype(np.float64) - d[:, :, None, :]) ** 2).sum(1))
    s = np.sort(dist, axis=2)[:, :, :k + 1]
    return float((np.diff(s, axis=2) / s[:, :, 1:]).min())


def run(model, inputs, lw, dtype, train):
    model = copy.deepcopy(model).to(dtype)
    model.train(train)
    for m in model.modules():
        if isinstance(m, torch.nn.Dropout):
            m.eval()
    x = [torch.from_numpy(inputs[k]).to(dtype) for k in ("pc", "intensity", "sn", "node_a", "node_b", "img")]
    coarse, fine = model(*x)
    out = dict(coarse=coarse.detach().numpy(), fine=fine.detach().numpy())
    if train:
        loss = (coarse * torch.from_numpy(lw[0]).to(dtype)).sum() + (fine * torch.from_numpy(lw[1]).to(dtype)).sum()
        loss.backward()
        params = dict(model.named_parameters())
        out["grads"] = [params[k].grad.numpy() for k in GRAD_KEYS]
    return out


def main(out_path, ref_dir):
    torch.manual_seed(0)
    nu = import_reference(ref_dir)
    blob = {}
    for name, (H, W) in SHAPES.items():
        for fine in (True, False):
            blob[f"keys_{name}_{'fine' if fine else 'coarse'}"] = key_list(nu.KeypointDetector(Opt(H, W, fine)))
    s = SMALL
    model = nu.KeypointDetector(Opt(s["H"], s["W"], True, s["N"], s["Ma"], s["Mb"], s["B"]))
    model.load_state_dict(syn.seeded_state_dict(model, WEIGHT_SEED), strict=True)
    L = (s["H"] // 32) * (s["W"] // 32)
    inputs = syn.make_network_inputs(INPUT_SEED, s["B"], s["N"], s["Ma"], s["Mb"], s["H"], s["W"], L)
    margins = dict(pc_a=knn_margin(inputs["pc"], inputs["node_a"], 3), pc_b=knn_margin(inputs["pc"], inputs["node_b"], 3),
                   a_b=knn_margin(inputs["node_a"], inputs["node_b"], 3))
    print("kNN margins", margins)
    assert min(margins.values()) > 1e-6, "an input seed lands within 8 float32 ulps of a kNN tie: take another"
    lw = (inputs["lw_coarse"], inputs["lw_fine"])
    blob.update(input_seed=np.int64(INPUT_SEED), weight_seed=np.int64(WEIGHT_SEED), grad_keys=np.array(GRAD_KEYS),
                input_names=np.array(sorted(inputs)),
                input_sums=np.array([inputs[k].astype(np.float64).sum() for k in sorted(inputs)]))
    res = {}
    for dtype, p in ((torch.float32, 32), (torch.float64, 64)):
        ev = run(model, inputs, lw, dtype, False)
        tr = run(model, inputs, lw, dtype, True)
        res[p] = dict(eval_coarse=ev["coarse"], eval_fine=ev["fine"], train_coarse=tr["coarse"], train_fine=tr["fine"],
                      **{f"grad_{i}": g for i, g in enumerate(tr["grads"])})
    strides = [max(1, -(-res[64][f"grad_{i}"].size // GRAD_ENTRIES)) for i in range(len(GRAD_KEYS))]
    blob.update(point_stride=np.int64(POINT_STRIDE), grad_stride=np.array(strides, dtype=np.int64))

    def kept(name, a):
        if name.startswith("grad_"):
            return a.reshape(-1)[::strides[int(name[5:])]]
        return a[..., ::POINT_STRIDE]
    for name in res[64]:
        r64, r32 = kept(name, res[64][name]), kept(name, res[32][name]).astype(np.float64)
        blob[name] = r64
        blob["spread_" + name] = np.float64(np.abs(r32 - r64).max())
        full = np.abs(res[32][name].astype(np.float64) - res[64][name]).max()
        print(f"{name:14s} kept {r64.size:6d}  max|ref64| {np.abs(r64).max():.3e}  max|ref32 - ref64| kept "
              f"{blob['spread_' + name]:.3e}, all entries {full:.3e}")
    np.savez_compressed(out_path, **blob)
    print("wrote", out_path)


if __name__ == "__main__":
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    ref = sys.argv[sys.argv.index("--reference") + 1] if "--reference" in sys.argv else build_ref.REF
    if ref in args:
        args.remove(ref)
    main(args[0] if args else os.path.join(HERE, "network_small.npz"), ref)
