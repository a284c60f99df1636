"""End-to-end classify-then-register (BASELINE config 5) and one KITTI training step of the classifier network
(network.KeypointDetector, DESIGN.md 4.18).

    python scripts/bench_e2e.py [--samples 1024] [--chunk 64] [--reps 3] [--out BENCH_E2E.json]
    python scripts/bench_e2e.py --profile [--out BENCH_E2E.json]       # the torch.profiler breakdown, a separate run

Config 5 on one GPU: `--samples` Oxford-shaped samples (synthetic.make_sample(..., shape="oxford") clouds of 20480
points, node sets drawn from each cloud, seeded 384 x 640 images, intensities and normals) through the network with
seeded, untrained weights:
- forward: eval mode under no_grad in chunks of `--chunk`; per-chunk and whole-batch time and the peak allocation of
  one chunk above the resident inputs;
- registration: frustum.register_batch (60 inits, 2-D) on the same clouds with the synthetic labels (ground truth +
  5 % flips, as bench.py uses), since untrained predictions mean nothing to the solver;
- config 5 = forward + registration; and one whole network.classify_and_register call on the untrained predictions,
  labelled as such.
KITTI training step: B = 8 at 160 x 512: forward (train mode), classifier.classifier_loss, backward and Adam.
Every shape is warmed up first; times are CUDA events, median over --reps.  --profile runs torch.profiler over
forward chunks and splits the forward's device time into convolution / norm (cuDNN), the project's kernels and other
torch ops.  Prints one JSON line with the GPU name and power limit read in the same run; --out merges it into the
file.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from deepi2p_b200 import classifier, frustum, network, synthetic  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_prep import _power_limit  # noqa: E402

ARGS = ("pc", "intensity", "sn", "node_a", "node_b", "img")
# the project's kernels live in namespace dib (csrc/*.cu); the CNN layers are cuDNN / cuBLAS convolutions, their
# layout transposes, BatchNorm and ResNet's max-pool; everything else (ReLU, the residual adds, torch.cat, the max
# reductions, copies) is "other_torch".  Matched as substrings of the profiler's kernel names.
PROJECT_KERNELS = ("dib::",)
CONV_KERNELS = ("conv", "cudnn", "xmma", "implicit", "gemm", "winograd", "fft", "bn_", "batch_norm", "batchnorm",
                "nchwToNhwc", "nhwcToNchw", "cutlass", "max_pool")


def _time(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def batch(S, shape, seed, dev):
    """S seeded samples of `shape` on the device; labels = synthetic predictions (ground truth + 5 % flips)."""
    H, W = (384, 640) if shape == "oxford" else (160, 512)
    smps = [synthetic.make_sample(seed + s, 20480, shape) for s in range(S)]
    pc = torch.from_numpy(np.stack([s["points"] for s in smps])).to(dev)
    gen = torch.Generator(device=dev).manual_seed(seed)
    idx = torch.argsort(torch.rand(S, 20480, device=dev, generator=gen), dim=1)[:, :256]
    nodes = torch.gather(pc, 2, idx.unsqueeze(1).expand(S, 3, 256))
    out = dict(pc=pc, intensity=torch.rand(S, 1, 20480, device=dev, generator=gen),
               sn=torch.nn.functional.normalize(torch.randn(S, 3, 20480, device=dev, generator=gen), dim=1),
               node_a=nodes[:, :, :128].contiguous(), node_b=nodes[:, :, 128:].contiguous(),
               img=torch.rand(S, 3, H, W, device=dev, generator=gen),
               label=torch.from_numpy(np.stack([s["pred"] for s in smps]).astype(np.int8)).to(dev),
               K=torch.from_numpy(np.stack([s["K"] for s in smps])).float().to(dev),
               P=torch.from_numpy(np.stack([s["P_gt"][:3] for s in smps])).float().to(dev), H=H, W=W)
    return out


def model_for(shape, dev):
    model = network.KeypointDetector(**network.SHAPES[shape])
    model.load_state_dict(synthetic.seeded_state_dict(model, 1))
    return model.to(dev)


def config5(a, dev):
    S, chunk = a.samples, a.chunk
    b = batch(S, "oxford", 1000, dev)
    model = model_for("oxford", dev).eval()
    chunks = [(i, min(i + chunk, S)) for i in range(0, S, chunk)]

    def forward_chunk(i, j):
        with torch.no_grad():
            return network.predict(*model(*(b[k][i:j] for k in ARGS)))

    def forward_all():
        for i, j in chunks:
            forward_chunk(i, j)
    for i, j in {(i, j) for i, j in chunks if j - i in {chunk, chunks[-1][1] - chunks[-1][0]}}:
        forward_chunk(i, j)                                 # warm up every chunk shape
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    forward_chunk(*chunks[0])
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    chunk_ms = _time(lambda: forward_chunk(*chunks[0]), a.reps * 3)
    fwd_ms = _time(forward_all, a.reps)

    def register():
        frustum.register_batch(b["pc"], b["label"], 20480, b["K"], b["H"], b["W"])
    register()
    reg_ms = _time(register, a.reps)

    def whole():
        network.classify_and_register(model, *(b[k] for k in ARGS), b["K"], chunk=chunk)
    whole()
    whole_ms = _time(whole, a.reps)
    return {"samples": S, "points": 20480, "image": [384, 640], "chunk": chunk, "n_inits": 60,
            "forward_ms_per_chunk": chunk_ms, "forward_ms_batch": fwd_ms, "forward_samples_per_s": S / fwd_ms * 1e3,
            "forward_peak_bytes_above_inputs": peak - base, "forward_peak_bytes": peak,
            "inputs_bytes": base, "register_ms_synthetic_labels": reg_ms,
            "config5_forward_plus_register_ms": fwd_ms + reg_ms,
            "config5_samples_per_s": S / (fwd_ms + reg_ms) * 1e3,
            "classify_and_register_ms_untrained_predictions": whole_ms,
            "note": "seeded untrained weights: the whole-call time registers meaningless predictions",
            "gpus_8": "not measured"}


def train_step(a, dev):
    b = batch(8, "kitti", 2000, dev)
    model = model_for("kitti", dev).train()
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)

    def step():
        coarse, fine = model(*(b[k] for k in ARGS))
        out = classifier.classifier_loss(coarse, fine, b["pc"], b["P"], b["K"], 160, 512)
        opt.zero_grad(set_to_none=True)
        out["loss"].backward()
        opt.step()
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    ms = _time(step, a.reps * 3)
    return {"B": 8, "points": 20480, "image": [160, 512], "step_ms": ms, "peak_bytes": torch.cuda.max_memory_allocated()}


def profile(a, dev):
    from torch.profiler import ProfilerActivity, profile as tprofile
    S = a.chunk
    b = batch(S, "oxford", 1000, dev)
    model = model_for("oxford", dev).eval()

    def fwd():
        with torch.no_grad():
            model(*(b[k] for k in ARGS))
    for _ in range(3):
        fwd()
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.reps):
            fwd()
        torch.cuda.synchronize()
    share = {"convolution_and_norm": 0.0, "project_kernels": 0.0, "other_torch": 0.0}
    top = []
    for e in prof.key_averages():
        t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        if t <= 0 or e.key.startswith("cuda") or e.key.startswith("Memcpy") or e.key.startswith("Memset"):
            continue
        name = e.key
        low = name.lower()
        if any(p.lower() in low for p in PROJECT_KERNELS):
            cls = "project_kernels"
        elif any(p.lower() in low for p in CONV_KERNELS):
            cls = "convolution_and_norm"
        else:
            cls = "other_torch"
        share[cls] += t
        top.append((t, cls, name[:120]))
    total = sum(share.values())
    top.sort(reverse=True)
    return {"shape": "oxford", "chunk": S, "forwards": a.reps, "device_us_per_forward": total / a.reps,
            "share": {k: v / total for k, v in share.items()},
            "top_kernels": [{"us_per_forward": t / a.reps, "class": c, "name": n} for t, c, n in top[:25]]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=1024)
    ap.add_argument("--chunk", type=int, default=network.DEFAULT_CHUNK)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_e2e.py needs a CUDA device")
    dev = torch.device("cuda:0")
    head = {"gpu": torch.cuda.get_device_name(0), "power_limit": _power_limit(),
            "tf32": [torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32]}
    if a.profile:
        res = {"e2e_profile": dict(head, **profile(a, dev))}
    else:
        res = {"e2e": dict(head, reps=a.reps, config5=config5(a, dev))}
        torch.cuda.empty_cache()
        res["e2e"]["kitti_train_step"] = train_step(a, dev)
    print(json.dumps(res))
    if a.out:
        old = {}
        if os.path.exists(a.out):
            with open(a.out) as f:
                old = json.loads(f.read() or "{}")
        old.update(res)
        with open(a.out, "w") as f:
            f.write(json.dumps(old) + "\n")


if __name__ == "__main__":
    main()
