"""Classifier training targets and losses (classifier.classifier_loss, DESIGN.md 4.15) against the reference's tail.

    python scripts/bench_classifier_loss.py [--reps 30] [--out FILE.json]

Shapes: the shipped classifier options, N = 20480 points: KITTI (B = 8, 160 x 512 -> L = 80), Oxford (B = 8,
384 x 640 -> L = 240) and nuScenes (B = 12, 160 x 320 -> L = 50), cells of 32 px.  The formulation is a torch
restatement of MMClassifer.foraward_pass's tail (models/multimodal_classifier.py:135-191, written for this script):
two fp32 matmuls, the label rule, .item() on the inside count, the sort of the mask, the fine-label range checks
(.item() twice), the gather of the inside rows from a permuted copy, kornia's focal loss, nn.CrossEntropyLoss and the
three argmaxes.  Each side is timed as forward and as forward + backward of `loss`, CUDA events around each
repetition after a warm-up, median over --reps.  Algorithmic bytes: the logits and coordinates read once, labels and
predictions written once (forward); the logits read and both gradients written once (backward).  Their share of the
H100 SXM data-sheet 3.35 TB/s is bytes / 3.35e12 / time.  Memory: torch.cuda.max_memory_allocated minus the
allocation before the call.  Prints one JSON line with the GPU name and power limit read in the same run.
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepi2p_b200 import classifier  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_prep import _power_limit, _time  # noqa: E402

HBM_BPS = 3.35e12
SHAPES = [("kitti", 8, 20480, 160, 512), ("oxford", 8, 20480, 384, 640), ("nuscenes", 12, 20480, 160, 320)]
SCALE = 32


def focal_loss(input, target, alpha=0.5, gamma=2.0, eps=1e-6):
    soft = F.softmax(input, dim=1) + eps
    one_hot = torch.zeros_like(soft).scatter_(1, target.unsqueeze(1), 1.0) + eps
    focal = -alpha * torch.pow(-soft + 1.0, gamma) * torch.log(soft)
    return torch.mean(torch.sum(one_hot * focal, dim=1))


def formulation(coarse_scores, fine_scores, pc, P, K, H, W, coarse_loss_alpha=50.0):
    B, L, N = fine_scores.shape
    W_f = int(round(W / SCALE))
    pc_homo = torch.cat((pc, torch.ones((B, 1, N), dtype=torch.float32, device=pc.device)), dim=1)
    P_pc_homo = torch.matmul(P, pc_homo)
    KP_pc_homo = torch.matmul(K, P_pc_homo)
    KP_pc_pxpy = KP_pc_homo[:, 0:2, :] / KP_pc_homo[:, 2:3, :]
    x_in = (KP_pc_pxpy[:, 0:1, :] >= 0) & (KP_pc_pxpy[:, 0:1, :] <= W - 1)
    y_in = (KP_pc_pxpy[:, 1:2, :] >= 0) & (KP_pc_pxpy[:, 1:2, :] <= H - 1)
    z_in = KP_pc_homo[:, 2:3, :] > 0.1
    inside_mask = (x_in & y_in & z_in).squeeze(1)
    scaled = torch.floor(KP_pc_pxpy / SCALE).to(dtype=torch.long)
    index = scaled[:, 0, :] + scaled[:, 1, :] * W_f
    coarse_labels = inside_mask.to(dtype=torch.long)
    mask_int = inside_mask.reshape(B * N).to(dtype=torch.int32)
    insider_num = int(torch.sum(mask_int).item())
    _, idx = torch.sort(mask_int, descending=True)
    insider_idx = idx[0:insider_num]
    index_insider = torch.gather(index.view(B * N), dim=0, index=insider_idx)
    assert torch.min(index_insider).item() >= 0
    assert torch.max(index_insider).item() <= L - 1
    fine_BnL = fine_scores.permute(0, 2, 1).reshape(B * N, L).contiguous()
    fine_insider = torch.gather(fine_BnL, dim=0, index=insider_idx.unsqueeze(1).expand(insider_num, L))
    coarse_loss = focal_loss(coarse_scores, coarse_labels) * coarse_loss_alpha
    fine_loss = F.cross_entropy(fine_insider, index_insider)
    loss = coarse_loss + fine_loss
    _, coarse_pred = torch.max(coarse_scores, dim=1)
    coarse_acc = torch.sum(torch.eq(coarse_labels, coarse_pred).to(dtype=torch.float)) / (B * N)
    _, fine_pred_in = torch.max(fine_insider, dim=1)
    fine_acc = torch.sum(torch.eq(index_insider, fine_pred_in).to(dtype=torch.float)) / insider_num
    _, fine_pred = torch.max(fine_scores, dim=1)
    return dict(loss=loss, coarse=coarse_loss, fine=fine_loss, coarse_accuracy=coarse_acc, fine_accuracy=fine_acc,
                coarse_predictions=coarse_pred, fine_predictions=fine_pred)


def make_inputs(B, N, H, W, gen, dev):
    L = int(round(H / SCALE)) * int(round(W / SCALE))
    pc = torch.stack([torch.rand(B, N, device=dev, generator=gen) * 60 - 30,
                      torch.rand(B, N, device=dev, generator=gen) * 12 - 6,
                      torch.rand(B, N, device=dev, generator=gen) * 80 - 20], dim=1)
    P = torch.eye(4, device=dev).repeat(B, 1, 1)[:, :3, :].contiguous()
    P[:, :3, 3] = torch.rand(B, 3, device=dev, generator=gen) * 2 - 1
    K = torch.tensor([[0.74 * W, 0.0, W / 2], [0.0, 0.74 * W, H / 2], [0.0, 0.0, 1.0]], device=dev).repeat(B, 1, 1)
    coarse = torch.randn(B, 2, N, device=dev, generator=gen) * 3
    fine = torch.randn(B, L, N, device=dev, generator=gen) * 3
    return coarse, fine, pc, P, K


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
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_classifier_loss.py needs a CUDA device")
    dev = torch.device("cuda:0")
    gen = torch.Generator(device=dev).manual_seed(0)
    result = {"gpu": torch.cuda.get_device_name(0), "power_limit": _power_limit(), "reps": a.reps, "shapes": {}}
    for name, B, N, H, W in SHAPES:
        coarse, fine, pc, P, K = make_inputs(B, N, H, W, gen, dev)
        L = fine.shape[1]
        cr, fr = coarse.clone().requires_grad_(True), fine.clone().requires_grad_(True)

        def op(c, f):
            return classifier.classifier_loss(c, f, pc, P, K, H, W, fine_scale=SCALE)

        def ref(c, f):
            return formulation(c, f, pc, P, K, H, W)

        def fwd(fn):
            with torch.no_grad():
                return fn(coarse, fine)

        def fwd_bwd(fn):
            cr.grad = fr.grad = None
            fn(cr, fr)["loss"].backward()
            return cr.grad, fr.grad

        o, r = fwd(op), fwd(ref)
        row = {"B": B, "N": N, "H": H, "W": W, "L": L, "n_inside": int(o["n_inside"].sum()),
               "loss": [float(o["loss"]), float(r["loss"])],
               "prediction_mismatches": int((o["fine_predictions"].long() != r["fine_predictions"]).sum())}
        go, gr = fwd_bwd(op), fwd_bwd(ref)
        row["max_abs_diff_grad"] = [float((go[0] - gr[0]).abs().max()), float((go[1] - gr[1]).abs().max())]
        for label, fn in (("op", op), ("formulation", ref)):
            for _ in range(3):
                fwd_bwd(fn)
            row[label] = {"forward_ms": _time(lambda: fwd(fn), a.reps) * 1e3,
                          "forward_backward_ms": _time(lambda: fwd_bwd(fn), a.reps) * 1e3,
                          "forward_peak_bytes": _peak(lambda: fwd(fn)),
                          "forward_backward_peak_bytes": _peak(lambda: fwd_bwd(fn))}
        logits = B * (2 + L) * N * 4
        fwd_bytes = logits + B * 3 * N * 4 + B * N * (1 + 4 + 1 + 4 + 4)      # + labels, predictions, log-sum-exp
        bwd_bytes = logits + B * N * (1 + 4 + 4) + logits                       # logits, labels, lse, gradients
        t_f = row["op"]["forward_ms"] * 1e-3
        t_fb = row["op"]["forward_backward_ms"] * 1e-3
        row["algorithmic_bytes"] = {"forward": fwd_bytes, "backward": bwd_bytes}
        row["op_share_of_3_35_TBps"] = {"forward": fwd_bytes / HBM_BPS / t_f,
                                         "forward_backward": (fwd_bytes + bwd_bytes) / HBM_BPS / t_fb}
        row["speedup"] = {"forward": row["formulation"]["forward_ms"] / row["op"]["forward_ms"],
                          "forward_backward": row["formulation"]["forward_backward_ms"] / row["op"]["forward_backward_ms"]}
        result["shapes"][name] = row
        del coarse, fine, pc, P, K, cr, fr, o, r, go, gr
        torch.cuda.empty_cache()
    line = json.dumps({"classifier_loss": result})
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
