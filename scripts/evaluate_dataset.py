"""Evaluate a classifier checkpoint on a KITTI, Oxford or nuScenes root, end to end on the GPU: val_random_Ry batches
(kitti.kitti_batch / oxford.oxford_batch / nuscenes.nuscenes_batch), network.classify_and_register, and
frustum.pose_error_batch, with registration_result_analysis.py's summary line and register_dir.py's
P_pred_all_np.npy / P_gt_all_np.npy / cost_all_np.npy.

    python scripts/evaluate_dataset.py --dataset {kitti,oxford,nuscenes} --root R --checkpoint C
        [--head torch|fused|fused_encoder|fused_all|fused_image] [--every k] [--batch B] [--seed S] [--inits I] [--version v1.0-trainval] [--out DIR]

The checkpoint is what the reference's training saved (network.load_checkpoint).  Every k-th entry of the val list is
taken (registration_lsq.py uses 30).  The per-sample draws (image pairing, Pr) come from numpy Generators seeded by
--seed, so a run is repeatable.
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from deepi2p_b200 import frustum, handoff, kitti, network, nuscenes, oxford  # noqa: E402

MODE = "val_random_Ry"


def batches(dataset, root, version):
    """(entry count, fn(items, seed, rng) -> the loader's tuple) for the val list of `dataset` at `root`."""
    if dataset == "kitti":
        ds = kitti.KittiDataset(root, MODE)
        return len(ds), lambda items, seed, rng: kitti.kitti_batch(ds, items, MODE, seed, rng=rng)
    if dataset == "oxford":
        ds = oxford.OxfordDataset(root, MODE)
        return len(ds), lambda items, seed, rng: oxford.oxford_batch(ds, items, MODE, seed, rng=rng)
    tables = nuscenes.Tables(root, version)
    info = nuscenes.load_dataset_info(os.path.join(root, "dataset_info.list"))
    return len(info), lambda items, seed, rng: nuscenes.nuscenes_batch(tables, [info[i] for i in items], MODE, seed,
                                                                        rng=rng)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--dataset", required=True, choices=("kitti", "oxford", "nuscenes"))
    ap.add_argument("--root", required=True)
    ap.add_argument("--checkpoint", required=True)
    ap.add_argument("--head", default="torch", choices=network.HEADS)
    ap.add_argument("--every", type=int, default=1)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--inits", type=int, default=60)
    ap.add_argument("--version", default="v1.0-trainval", help="nuScenes table version")
    ap.add_argument("--out", default=None, help="where to write P_pred_all_np.npy / P_gt_all_np.npy / cost_all_np.npy")
    a = ap.parse_args(argv)
    if a.every < 1 or a.batch < 1:
        ap.error("--every and --batch must be >= 1")
    if not torch.cuda.is_available():
        raise SystemExit("evaluate_dataset.py needs a CUDA device")
    model = network.KeypointDetector(**network.SHAPES[a.dataset])
    network.load_checkpoint(model, a.checkpoint)
    model = model.cuda()
    n, make = batches(a.dataset, a.root, a.version)
    items = list(range(0, n, a.every))
    rng = np.random.default_rng(a.seed)
    P_pred, P_gt, cost = [], [], []
    for b in range(0, len(items), a.batch):
        pc, inten, sn, na, nb, P, img, K, _ = make(items[b:b + a.batch], a.seed * 100003 + b, rng)
        res = network.classify_and_register(model, pc, inten, sn, na, nb, img, K.numpy(), n_inits=a.inits,
                                            seed=a.seed, head=a.head)
        gt = np.tile(np.eye(4), (P.shape[0], 1, 1))
        gt[:, :3] = P.cpu().numpy().astype(np.float64)
        P_pred.append(res["P"].cpu().numpy())
        P_gt.append(gt)
        cost.append(res["cost"].cpu().numpy())
    P_pred, P_gt, cost = np.concatenate(P_pred), np.concatenate(P_gt), np.concatenate(cost)
    err = frustum.pose_error_batch(P_pred, P_gt)
    t_err, r_err, ok = (err[k].cpu().numpy() for k in ("t_err", "r_err", "success"))
    for i, it in enumerate(items):
        print("%06d - cost: %.1f, T: %.1f, R:%.1f" % (it, cost[i], t_err[i], r_err[i]))
    s = handoff.summarize(t_err, r_err, cost, ok)
    print("RTE %.2f +- %.2f, RRE %.2f +- %.2f, success rate %.2f" % (s["rte_mean"], s["rte_sigma"], s["rre_mean"],
                                                                     s["rre_sigma"], s["success_rate"] * 100))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        np.save(os.path.join(a.out, "P_pred_all_np.npy"), P_pred)
        np.save(os.path.join(a.out, "P_gt_all_np.npy"), P_gt)
        np.save(os.path.join(a.out, "cost_all_np.npy"), cost)
    return s


if __name__ == "__main__":
    main()
