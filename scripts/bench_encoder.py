"""Encoder cluster max-pool and node kNN grouping (point_ops.cluster_max_pool / knn_group, DESIGN.md 4.16) against the
reference's torch formulation.

    python scripts/bench_encoder.py [--reps 50] [--out BENCH_ENCODER.json]

Shapes: the three calls of PCEncoder.forward with the shipped KITTI / Oxford options (B = 8, N = 20480, Ma = Mb = 128,
k_ab = 16): the first pool (C = 32, with its broadcast back to the points; only the broadcast feeds the network, so
the backward gets a gradient of `scattered` alone), the second pool (C = 64, no broadcast, a gradient of `pooled`)
and the kNN grouping of the 128 node_b queries over the 128 cluster means (C = 64).  The segment ids come from
cluster_assign_forward on a uniform cloud.  The pool formulation is networks_pc.py:88-104 with this project's
index_max_forward and, where oracle/_ref holds the reference's compiled index_max, with that one too; its
mask_row_max is computed once outside the timed call, as the reference shares it between both pools.  The kNN
formulation is layers_pc.py:793-807.  Each call is timed as forward and as forward + backward (a fixed gradient of
the outputs' shape), CUDA events around each repetition after a warm-up, median over --reps.  Memory:
torch.cuda.max_memory_allocated minus the allocation before the call.  Prints one JSON line with the GPU name and
power limit read in the same run.
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
from bench_prep import _power_limit, _time  # noqa: E402

B, N, MA, MB, K_AB = 8, 20480, 128, 128, 16


def pool_formulation(index_max):
    def run(F, min_idx, M, mask_row_max, broadcast):
        sel = index_max(F.detach(), min_idx, M).long()
        pooled = F.gather(dim=2, index=sel) * mask_row_max
        if not broadcast:
            return pooled
        return pooled, torch.gather(pooled, dim=2, index=min_idx.long().unsqueeze(1).expand(F.shape[0], F.shape[1],
                                                                                             F.shape[2]))
    return run


def knn_formulation(query, database, features, K):
    Bq, M, Nd, C = query.size(0), query.size(2), database.size(2), features.size(1)
    q = query.detach().unsqueeze(3)
    norm = torch.norm(q - database.detach().unsqueeze(2), dim=1, keepdim=False)
    _, knn_I = torch.topk(norm, k=K, dim=2, largest=False, sorted=True)
    I3 = knn_I.unsqueeze(1).expand(Bq, 3, M, K).contiguous().view(Bq, 3, M * K)
    IC = knn_I.unsqueeze(1).expand(Bq, C, M, K).contiguous().view(Bq, C, M * K)
    coord = torch.gather(database, dim=2, index=I3).view(Bq, 3, M, K)
    feat = torch.gather(features, dim=2, index=IC).view(Bq, C, M, K)
    return torch.cat(((coord - q).detach(), feat), dim=1)


def _peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    r = fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del r
    return int(peak)


def _measure(fwd, fwd_bwd, reps):
    for _ in range(3):
        fwd_bwd()
    return {"forward_ms": _time(fwd, reps) * 1e3, "forward_backward_ms": _time(fwd_bwd, reps) * 1e3,
            "forward_peak_bytes": _peak(fwd), "forward_backward_peak_bytes": _peak(fwd_bwd)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_encoder.py needs a CUDA device")
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    result = {"gpu": torch.cuda.get_device_name(0), "power_limit": _power_limit(), "reps": a.reps, "calls": {}}
    pc = torch.rand(B, 3, N, device=dev, generator=gen) * 40 - 20
    node_a = torch.rand(B, 3, MA, device=dev, generator=gen) * 40 - 20
    node_b = torch.rand(B, 3, MB, device=dev, generator=gen) * 40 - 20
    ca = point_ops.cluster_assign_forward(pc, node_a, k=1, want_centers=False)
    min_idx, cluster_mean = ca["min_idx"], ca["cluster_mean"]
    mask_row_max = (ca["count"] > 0).float().unsqueeze(1)

    formulations = {"formulation": pool_formulation(point_ops.index_max_forward)}
    try:
        sys.path.insert(0, os.path.join(ROOT, "oracle"))
        import build_ref
        if build_ref.built("index_max"):
            ref_im = build_ref.load("index_max")
            formulations["formulation_reference_index_max"] = pool_formulation(
                lambda d, i, m: ref_im.forward_cuda_shared_mem(d, i, m))
        else:
            result["reference_index_max"] = "not built"
    except Exception as e:  # noqa: BLE001
        result["reference_index_max"] = "unavailable: %s" % e

    for name, C, broadcast in (("first_pool", 32, True), ("second_pool", 64, False)):
        F = torch.randn(B, C, N, device=dev, generator=gen)
        Fr = F.clone().requires_grad_(True)
        g = torch.randn(B, C, N if broadcast else MA, device=dev, generator=gen)

        def op(X):
            out = point_ops.cluster_max_pool(X, min_idx, MA, broadcast=broadcast)
            return out[1] if broadcast else out

        def make(fn):
            def fwd():
                with torch.no_grad():
                    return fn(F)

            def fwd_bwd():
                Fr.grad = None
                fn(Fr).backward(g)
                return Fr.grad
            return fwd, fwd_bwd

        row = {"B": B, "C": C, "N": N, "M": MA, "broadcast": broadcast}
        fo, fbo = make(op)
        row["op"] = _measure(fo, fbo, a.reps)
        for label, form in formulations.items():
            def ref(X, form=form):
                out = form(X, min_idx, MA, mask_row_max, broadcast)
                return out[1] if broadcast else out
            fr, fbr = make(ref)
            row["max_abs_diff_forward_" + label] = float((fo() - fr()).abs().max())
            row["max_abs_diff_grad_" + label] = float((fbo().clone() - fbr()).abs().max())
            row[label] = _measure(fr, fbr, a.reps)
        result["calls"][name] = row
        del F, Fr, g
        torch.cuda.empty_cache()

    C = 64
    F = torch.randn(B, C, MA, device=dev, generator=gen)
    Fr = F.clone().requires_grad_(True)
    g = torch.randn(B, 3 + C, MB, K_AB, device=dev, generator=gen)

    def op(X):
        return point_ops.knn_group(node_b, cluster_mean, X, K_AB)[1]

    def ref(X):
        return knn_formulation(node_b, cluster_mean, X, K_AB)

    row = {"B": B, "C": C, "M": MB, "N": MA, "K": K_AB}
    for label, fn in (("op", op), ("formulation", ref)):
        def fwd(fn=fn):
            with torch.no_grad():
                return fn(F)

        def fwd_bwd(fn=fn):
            Fr.grad = None
            fn(Fr).backward(g)
            return Fr.grad
        row[label] = _measure(fwd, fwd_bwd, a.reps)
    with torch.no_grad():
        row["max_abs_diff_forward"] = float((op(F) - ref(F)).abs().max())
    result["calls"]["knn_group"] = row
    line = json.dumps({"encoder": result})
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
