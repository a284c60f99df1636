"""Decoder interpolation (point_ops.upsample_by_interpolation, DESIGN.md 4.12) against the reference's formulation.

    python scripts/bench_interp.py [--reps 20] [--out FILE.json]

Shapes: the three calls of KeypointDetector.forward with the shipped KITTI / Oxford options (B = 8, k = 3, 128 nodes
per set, N = 20480): points <- node_b (C = 512), node_a <- node_b (C = 512), points <- node_a (C = 128).  Indices
are the k nearest nodes (cluster_assign_forward), int64 as torch.topk returns them.  Each call is timed as forward
and as forward + backward (the backward gets a fixed gradient of the output's shape), CUDA events around each
repetition after a warm-up, median over --reps.  The formulation is a torch restatement of the reference's gather /
norm / weight / sum (written for this script).  For the first call the index search is timed too: torch.norm of the
B x 3 x N x M difference + torch.topk against cluster_assign_forward.  Algorithmic bytes: the tensors each direction
must read and write once (indices, coordinates, features, output; in the backward the output gradient, the saved
weights and indices, the feature gradient); their share of the H100 SXM data-sheet 3.35 TB/s is
bytes / 3.35e12 / time.  Memory: torch.cuda.max_memory_allocated minus the allocation before the call.  Prints one
JSON line with the GPU name and power limit read in the same run.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepi2p_b200 import point_ops  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_prep import _power_limit, _time  # noqa: E402

HBM_BPS = 3.35e12
CALLS = [("points_from_node_b", 8, 20480, 128, 512, 3), ("node_a_from_node_b", 8, 128, 128, 512, 3),
         ("points_from_node_a", 8, 20480, 128, 128, 3)]


def formulation(idx, query, node, features):
    B, Nq, k = idx.shape
    C, M = features.shape[1], features.shape[2]
    nodes_k = torch.gather(node.unsqueeze(3).expand(B, 3, M, k), 2, idx.unsqueeze(1).expand(B, 3, Nq, k))
    dist = torch.norm(query.unsqueeze(3) - nodes_k, p=2, dim=1)
    weight = 1 - dist / torch.sum(dist, dim=2, keepdim=True)
    feats_k = torch.gather(features.unsqueeze(3).expand(B, C, M, k), 2, idx.unsqueeze(1).expand(B, C, Nq, k))
    return torch.sum(weight.unsqueeze(1) * feats_k, dim=3)


def _peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    r = fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del r
    return int(peak)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_interp.py needs a CUDA device")
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    result = {"gpu": torch.cuda.get_device_name(0), "power_limit": _power_limit(), "reps": a.reps, "calls": {}}
    for name, B, Nq, M, C, k in CALLS:
        q = torch.rand(B, 3, Nq, device=dev, generator=gen) * 40 - 20
        nd = torch.rand(B, 3, M, device=dev, generator=gen) * 40 - 20
        F = torch.randn(B, C, M, device=dev, generator=gen)
        g = torch.randn(B, C, Nq, device=dev, generator=gen)
        idx = point_ops.cluster_assign_forward(q, nd, k=k, want_centers=False)["min_k_idx"].long()
        Fr = F.clone().requires_grad_(True)

        def fwd(fn):
            with torch.no_grad():
                return fn(idx, q, nd, F)

        def fwd_bwd(fn):
            Fr.grad = None
            fn(idx, q, nd, Fr).backward(g)
            return Fr.grad

        row = {"B": B, "Nq": Nq, "M": M, "C": C, "k": k}
        op, ref = point_ops.upsample_by_interpolation, formulation
        row["max_abs_diff_forward"] = float((fwd(op) - fwd(ref)).abs().max())
        row["max_abs_diff_grad"] = float((fwd_bwd(op) - fwd_bwd(ref)).abs().max())
        for label, fn in (("op", op), ("formulation", ref)):
            for _ in range(3):
                fwd_bwd(fn)
            row[label] = {"forward_ms": _time(lambda: fwd(fn), a.reps) * 1e3,
                          "forward_backward_ms": _time(lambda: fwd_bwd(fn), a.reps) * 1e3,
                          "forward_peak_bytes": _peak(lambda: fwd(fn)),
                          "forward_backward_peak_bytes": _peak(lambda: fwd_bwd(fn))}
        fwd_bytes = B * Nq * k * 8 + B * 3 * (Nq + M) * 4 + B * C * M * 4 + B * C * Nq * 4 + B * Nq * k * 8
        bwd_bytes = B * C * Nq * 4 + B * Nq * k * 8 + B * C * M * 4
        t_f = row["op"]["forward_ms"] * 1e-3
        t_b = row["op"]["forward_backward_ms"] * 1e-3 - t_f
        row["algorithmic_bytes"] = {"forward": fwd_bytes, "backward": bwd_bytes}
        row["op_share_of_3_35_TBps"] = {"forward": fwd_bytes / HBM_BPS / t_f,
                                         "backward_by_difference": bwd_bytes / HBM_BPS / max(t_b, 1e-9)}
        if name == "points_from_node_b":
            def search_ref():
                d = torch.norm(q.unsqueeze(3) - nd.unsqueeze(2), p=2, dim=1)
                return torch.topk(d, k=k, dim=2, largest=False, sorted=True)[1]

            def search_op():
                return point_ops.cluster_assign_forward(q, nd, k=k, want_centers=False)["min_k_idx"]

            row["index_search_ms"] = {"cluster_assign": _time(search_op, a.reps) * 1e3,
                                      "norm_topk": _time(search_ref, a.reps) * 1e3}
        result["calls"][name] = row
        del q, nd, F, g, idx, Fr
        torch.cuda.empty_cache()
    line = json.dumps({"interp": result})
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
