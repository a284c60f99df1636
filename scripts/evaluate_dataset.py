"""Evaluate a classifier checkpoint on a KITTI, Oxford or nuScenes root, end to end on the GPU: val_random_Ry batches
(kitti.kitti_batch / oxford.oxford_batch / nuscenes.nuscenes_batch), network.classify_batch once per batch, then one
of the paper's three registration methods, with registration_result_analysis.py's summary line and register_dir.py's
P_pred_all_np.npy / P_gt_all_np.npy / cost_all_np.npy.

    python scripts/evaluate_dataset.py --dataset {kitti,oxford,nuscenes} --root R --checkpoint C
        [--method lsq|pnp|icp] [--is-3d] [--fine-scale 0.03125] [--depth-model DIR] [--accuracy]
        [--head torch|fused|fused_encoder|fused_all|fused_image] [--every k] [--batch B] [--seed S] [--inits I]
        [--version v1.0-trainval] [--out DIR]

The methods are register_dir.py's, with the same option names and meanings (DESIGN.md 4.35):
  lsq  frustum classification + inverse camera projection (registration_lsq.py): frustum.register_batch on the coarse
       predictions with classify_and_register's settings, 2-D unless --is-3d; cost = the solver's.
  pnp  grid classification + PnP-RANSAC (registration_pnp.py): pnp.pnp_ransac_batch on the coarse and fine
       predictions (500 iterations, 0.6 px, confidence 0.99, --fine-scale), seed --seed + the batch's first position;
       cost = outlier ratio.  Needs a checkpoint with a fine head.
  icp  monodepth cloud + multi-start ICP (icp/registration_icp.py): the batch image rounded as save_depth_map.py reads
       <id>_img.png, the depth cloud of the monodepth2 checkpoint in --depth-model scaled with the ground truth, and
       icp.register_images from icp.random_inits(S, --inits, --seed + the batch's first position); cost = fitness.
With --accuracy, visualize_and_save_data.py's "Overall coarse accuracy, fine accuracy" line is printed and both values
join the returned summary (classifier.prediction_accuracy per batch, the counts read back once at the end).

The checkpoint is what the reference's training saved (network.load_checkpoint); a coarse-only one (no fine head) is
recognised by its head.  Every k-th entry of the val list is taken (registration_lsq.py uses 30).  The per-sample
draws (image pairing, Pr) come from numpy Generators seeded by --seed, so a run is repeatable.
"""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from deepi2p_b200 import (classifier, frustum, handoff, icp, kitti, monodepth, network, nuscenes, oxford,  # noqa: E402
                          pnp)

MODE = "val_random_Ry"
PNP = dict(iterations=500, reproj_err=0.6, confidence=0.99)      # registration_pnp.py's solvePnPRansac arguments
ICP_T_THRESH, ICP_R_THRESH = 2.0, 5.0                            # registration_icp.py's success thresholds
LINE = {"lsq": "%06d - cost: %.1f, T: %.1f, R:%.1f", "pnp": "%06d - cost: %.2f, T: %.1f, R:%.1f",
        "icp": "%06d - fitness: %.1f, T: %.1f, R:%.1f"}


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


def load_model(dataset, checkpoint):
    """The detector of `dataset`'s shapes with the checkpoint's weights, on the GPU.  A checkpoint whose head ends in
    two channels is the coarse-only classifier (MMClassiferCoarse)."""
    sd = torch.load(checkpoint, map_location="cpu", weights_only=True)
    last = [v for k, v in sd.items() if k.endswith("per_point_pn.layers.2.conv.weight")]
    fine = not (len(last) == 1 and last[0].shape[0] == 2)
    model = network.KeypointDetector(**network.SHAPES[dataset], fine=fine)
    network.load_checkpoint(model, sd)
    return model.cuda()


def register(method, model, batch, seed, first, head="torch", inits=60, is_3d=False, fine_scale=1 / 32.0,
             depth_model=None):
    """Classify one loader batch once and register its samples by `method`.  `first` is the batch's position in the
    evaluated list (the pnp and icp seeds add it, as register_dir.py does).  Returns (P_pred [S,4,4] f64, P_gt [S,4,4]
    f64, cost [S] f64) on the host and the predictions (coarse int8 [S,N], fine int32 [S,N] or None) on the device."""
    pc, inten, sn, na, nb, P, img, K, _ = batch
    coarse, fine = network.classify_batch(model, pc, inten, sn, na, nb, img, head=head)
    S, N, H, W = pc.shape[0], pc.shape[2], img.shape[2], img.shape[3]
    gt = np.tile(np.eye(4), (P.shape[0], 1, 1))
    gt[:, :3] = P.cpu().numpy().astype(np.float64)
    if method == "lsq":
        out = frustum.register_batch(pc.contiguous(), coarse, N, K.numpy(), H, W, n_inits=inits, seed=seed,
                                     is_2d=not is_3d)
        P_pred, cost = out["P"], out["cost"]
    elif method == "pnp":
        out = pnp.pnp_ransac_batch(pc.contiguous(), coarse, fine, None, K.numpy(), H, W, scale=fine_scale,
                                   seed=seed + first, **PNP)
        P_pred, cost = out["P"], out["outlier_ratio"]
    else:
        n = torch.full((S,), N, dtype=torch.int32, device=pc.device)
        init = torch.from_numpy(icp.random_inits(S, inits, seed + first)).to(pc.device)
        out = icp.register_images(pc.contiguous(), n, monodepth.images_from_batch(img), K.numpy(), gt, init,
                                  depth_model)
        P_pred, cost = out["P"], out["fitness"]
    return P_pred.cpu().numpy(), gt, cost.cpu().numpy(), coarse, fine


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--dataset", required=True, choices=("kitti", "oxford", "nuscenes"))
    ap.add_argument("--root", required=True)
    ap.add_argument("--checkpoint", required=True)
    ap.add_argument("--method", default="lsq", choices=("lsq", "pnp", "icp"),
                    help="lsq: frustum classification + inverse camera projection (registration_lsq.py); "
                         "pnp: grid classification + PnP-RANSAC (registration_pnp.py); "
                         "icp: monodepth cloud + multi-start ICP (icp/registration_icp.py)")
    ap.add_argument("--is-3d", action="store_true", help="lsq only: the 6-DoF solve")
    ap.add_argument("--fine-scale", type=float, default=None,
                    help="pnp only: fine grid resolution relative to the image (default 1/32, registration_pnp.py:163)")
    ap.add_argument("--depth-model", default=None,
                    help="icp only (required): monodepth2 checkpoint directory (encoder.pth, depth.pth)")
    ap.add_argument("--accuracy", action="store_true",
                    help="print and return the overall coarse and fine classification accuracy")
    ap.add_argument("--head", default="torch", choices=network.HEADS)
    ap.add_argument("--every", type=int, default=1)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--inits", type=int, default=60, help="lsq and icp: multi-start inits per sample")
    ap.add_argument("--version", default="v1.0-trainval", help="nuScenes table version")
    ap.add_argument("--out", default=None, help="where to write P_pred_all_np.npy / P_gt_all_np.npy / cost_all_np.npy")
    a = ap.parse_args(argv)
    if a.every < 1 or a.batch < 1:
        ap.error("--every and --batch must be >= 1")
    if a.method == "icp" and a.depth_model is None:
        ap.error("--method icp needs --depth-model DIR (a monodepth2 checkpoint)")
    if a.method != "icp" and a.depth_model is not None:
        ap.error("--depth-model is only used by --method icp")
    if a.method != "pnp" and a.fine_scale is not None:
        ap.error("--fine-scale is only used by --method pnp")
    if a.method != "lsq" and a.is_3d:
        ap.error("--is-3d is only used by --method lsq")
    fine_scale = 1 / 32.0 if a.fine_scale is None else a.fine_scale
    if not torch.cuda.is_available():
        raise SystemExit("evaluate_dataset.py needs a CUDA device")
    model = load_model(a.dataset, a.checkpoint)
    if a.method == "pnp" and not model.fine:
        raise SystemExit("--method pnp needs fine predictions, and %s is a coarse-only checkpoint" % a.checkpoint)
    depth_model = monodepth.load_monodepth(a.depth_model) if a.method == "icp" else None
    n, make = batches(a.dataset, a.root, a.version)
    items = list(range(0, n, a.every))
    rng = np.random.default_rng(a.seed)
    P_pred, P_gt, cost, counts = [], [], [], []
    for b in range(0, len(items), a.batch):
        batch = make(items[b:b + a.batch], a.seed * 100003 + b, rng)
        pp, gt, c, coarse, fine = register(a.method, model, batch, a.seed, b, head=a.head, inits=a.inits,
                                           is_3d=a.is_3d, fine_scale=fine_scale, depth_model=depth_model)
        P_pred.append(pp)
        P_gt.append(gt)
        cost.append(c)
        if a.accuracy:
            pc, P, img, K = batch[0], batch[5], batch[6], batch[7]
            acc = classifier.prediction_accuracy(pc, P.to(pc.device), K.to(pc.device), img.shape[2], img.shape[3],
                                                 coarse, fine, fine_scale=model.fine_scale)
            counts.append(torch.stack([acc["n_inside"], acc["coarse_correct"],
                                       acc["fine_correct"] if fine is not None else acc["coarse_correct"]]))
    P_pred, P_gt, cost = np.concatenate(P_pred), np.concatenate(P_gt), np.concatenate(cost)
    if a.method == "icp":
        t_err, r_err = handoff.get_p_diff(P_pred, P_gt)
        ok = ((t_err < ICP_T_THRESH) & (r_err < ICP_R_THRESH)).astype(np.int32)
    else:
        err = frustum.pose_error_batch(P_pred, P_gt)
        t_err, r_err, ok = (err[k].cpu().numpy() for k in ("t_err", "r_err", "success"))
    for i, it in enumerate(items):
        print(LINE[a.method] % (it, cost[i], t_err[i], r_err[i]))
    s = handoff.summarize(t_err, r_err, cost, ok)
    print("RTE %.2f +- %.2f, RRE %.2f +- %.2f, success rate %.2f" % (s["rte_mean"], s["rte_sigma"], s["rre_mean"],
                                                                     s["rre_sigma"], s["success_rate"] * 100))
    if a.accuracy:
        n_inside, coarse_ok, fine_ok = torch.cat(counts, dim=1).cpu().numpy()       # [3, samples], read once
        s["coarse_accuracy"], s["fine_accuracy"] = classifier.overall_accuracy(
            n_inside, coarse_ok, fine_ok if model.fine else None, batch[0].shape[2])
        print("Overall coarse accuracy %.4f, fine accuracy %.4f" % (s["coarse_accuracy"], s["fine_accuracy"]))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        np.save(os.path.join(a.out, "P_pred_all_np.npy"), P_pred)
        np.save(os.path.join(a.out, "P_gt_all_np.npy"), P_gt)
        np.save(os.path.join(a.out, "cost_all_np.npy"), cost)
    return s


if __name__ == "__main__":
    main()
