"""Image-attention fusion (point_ops.attention_fusion, DESIGN.md 4.17) against the reference's torch formulation and
against torch.bmm.

    python scripts/bench_fusion.py [--reps 50] [--out BENCH_FUSION.json]

Shapes: the two calls of KeypointDetector.forward (networks_united.py:149-150 on the s32 map with node_b, C = 512;
:172-174 on the s16 map with node_a, C = 256; Ma = Mb = 128) at the shipped KITTI (B = 8, 160 x 512), Oxford (B = 8,
384 x 640) and nuScenes (B = 12, 160 x 320) options, P = H/32 W/32 or H/16 W/16.  Three implementations:
- op: point_ops.attention_fusion;
- formulation: torch.mean(F.unsqueeze(3) * A.unsqueeze(1), dim=2), the reference's lines;
- bmm: torch.bmm(F, A) / P with torch.backends.cuda.matmul.allow_tf32 off (full float32 cuBLAS).
Each is timed as forward and as forward + backward (gradients of both inputs, a fixed output gradient), CUDA events
around each whole call after a warm-up, median over --reps.  Memory: torch.cuda.max_memory_allocated minus the
allocation before the call.  max_abs_diff_* compares the op's and bmm's outputs and gradients with the formulation's.
Prints one JSON line with the GPU name and power limit read in the same run.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from deepi2p_b200 import point_ops  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_encoder import _measure  # noqa: E402
from bench_prep import _power_limit  # noqa: E402

M_NODES = 128
# (dataset, B, image H, W)
DATASETS = (("kitti", 8, 160, 512), ("oxford", 8, 384, 640), ("nuscenes", 12, 160, 320))


def formulation(F, A):
    return torch.mean(F.unsqueeze(3) * A.unsqueeze(1), dim=2)


def bmm(F, A):
    return torch.bmm(F, A) / F.shape[2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fusion.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    result = {"gpu": torch.cuda.get_device_name(0), "power_limit": _power_limit(), "reps": a.reps,
              "bmm_allow_tf32": torch.backends.cuda.matmul.allow_tf32, "calls": {}}
    impls = (("op", point_ops.attention_fusion), ("formulation", formulation), ("bmm", bmm))
    for name, B, H, W in DATASETS:
        for scale, C in ((32, 512), (16, 256)):
            P = (H // scale) * (W // scale)
            F = torch.randn(B, C, P, device=dev, generator=gen)
            A = torch.randn(B, P, M_NODES, device=dev, generator=gen)
            g = torch.randn(B, C, M_NODES, device=dev, generator=gen)
            Fr, Ar = F.clone().requires_grad_(True), A.clone().requires_grad_(True)
            row = {"B": B, "C": C, "P": P, "M": M_NODES, "product_tensor_bytes": 4 * B * C * P * M_NODES}
            results = {}
            for label, fn in impls:
                def fwd(fn=fn):
                    with torch.no_grad():
                        return fn(F, A)

                def fwd_bwd(fn=fn):
                    Fr.grad = Ar.grad = None
                    fn(Fr, Ar).backward(g)
                    return Fr.grad, Ar.grad
                out = fwd()
                gF, gA = (t.clone() for t in fwd_bwd())
                results[label] = (out, gF, gA)
                row[label] = _measure(fwd, fwd_bwd, a.reps)
                Fr.grad = Ar.grad = None
                torch.cuda.empty_cache()
            ref = results["formulation"]
            for label in ("op", "bmm"):
                for part, x, r in zip(("forward", "grad_features", "grad_attention"), results[label], ref):
                    row[f"max_abs_diff_{part}_{label}"] = float((x - r).abs().max())
            result["calls"][f"{name}_s{scale}"] = row
            del F, A, g, Fr, Ar, results, ref
            torch.cuda.empty_cache()
    line = json.dumps({"fusion": result})
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
