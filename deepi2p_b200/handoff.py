"""Hand-off between the classifier and the registration solver (SURVEY.md 8(f) N2).

The reference passes data through a triple of files per frame, written by
evaluation/visualize_and_save_data.py:174-186 and read back by evaluation/registration_lsq.py:291-302:

    <id>_pc_label.npy   float array [7, N]: rows 0-2 xyz, 3 coarse prediction, 4 coarse label,
                        5 fine prediction, 6 fine label (labels stored as floats)
    <id>_K.npy          [3, 3] intrinsics
    <id>_P.npy          [3, 4] or [4, 4] ground-truth pose

with <id> = '%06d_%02d' (9 characters, registration_lsq.py:273).  The batched contract of this
framework is the C ABI's device record: (xyz f32 [S,3,Ns], label int8 [S,Ns], n_pts int32 [S],
K f64 [S,9]).  This module converts between the two on the host (file I/O only -- no compute path
lives here) and drives a whole directory through frustum.register_batch.
"""
import math
import os

import numpy as np

ROW_COARSE_PREDICTION = 3
ROW_COARSE_LABEL = 4
ROW_FINE_PREDICTION = 5
ROW_FINE_LABEL = 6
LABEL_ROWS = {"coarse_prediction": ROW_COARSE_PREDICTION, "coarse_label": ROW_COARSE_LABEL,
              "fine_prediction": ROW_FINE_PREDICTION, "fine_label": ROW_FINE_LABEL}
SUFFIXES = ("_pc_label.npy", "_K.npy", "_P.npy")

# registration_lsq.py:236-247: nuScenes clouds are east-north-up; camera axes are x right, y down, z forward.
ENU2CAM = np.array([[1.0, 0.0, 0.0, 0.0], [0.0, 0.0, -1.0, 0.0], [0.0, 1.0, 0.0, 0.0], [0.0, 0.0, 0.0, 1.0]])


def list_records(data_dir):
    """Frame ids present in a legacy directory: first 9 characters of every file name, unique, sorted
    (registration_lsq.py:273-275; the reference then shuffles them, which only changes print order)."""
    names = {f[0:9] for f in os.listdir(data_dir) if os.path.isfile(os.path.join(data_dir, f)) and f.endswith(".npy")
             and f.endswith(SUFFIXES)}
    return sorted(names)


def save_record(data_dir, name, pc, coarse_prediction, coarse_label, fine_prediction, fine_label, K, P):
    """Write one frame in the reference's layout (visualize_and_save_data.py:174-186)."""
    pc = np.asarray(pc, dtype=np.float32)
    rows = [np.asarray(r, dtype=np.float32)[None, :] for r in (coarse_prediction, coarse_label, fine_prediction,
                                                               fine_label)]
    out = np.concatenate([pc] + rows, axis=0)
    os.makedirs(data_dir, exist_ok=True)
    np.save(os.path.join(data_dir, name + "_pc_label.npy"), out)
    np.save(os.path.join(data_dir, name + "_K.npy"), np.asarray(K))
    np.save(os.path.join(data_dir, name + "_P.npy"), np.asarray(P))


def load_record(data_dir, name, which="coarse_prediction", enu2cam=False):
    """One frame -> (pc [3,N] float, label [N] int64, K [3,3] f64, P_gt [4,4] f64), as
    registration_lsq.py:291-304 reads it."""
    data = np.load(os.path.join(data_dir, name + "_pc_label.npy"))
    if data.ndim != 2 or data.shape[0] < 4:
        raise ValueError("%s_pc_label.npy: expected [>=4, N], got %s" % (name, data.shape))
    row = LABEL_ROWS[which]
    if row >= data.shape[0]:
        raise ValueError("%s_pc_label.npy has no row %d (%s)" % (name, row, which))
    pc = data[0:3, :]
    label = data[row, :].astype(np.int64)
    K = np.load(os.path.join(data_dir, name + "_K.npy")).astype(np.float64)
    P = np.load(os.path.join(data_dir, name + "_P.npy")).astype(np.float64)
    if P.shape[0] == 3:
        P = np.concatenate((P, np.identity(4)[3:4, :]), axis=0)
    if enu2cam:
        pc = (ENU2CAM[0:3, 0:3].astype(pc.dtype) @ pc)
        P = P @ np.linalg.inv(ENU2CAM)
    return pc, label, K, P


def load_batch(data_dir, names=None, which="coarse_prediction", enu2cam=False):
    """Legacy directory -> host arrays of the batched contract.

    Returns dict(names, xyz f32 [S,3,Nmax], label int8 [S,Nmax] (-1 = padding), n_pts int32 [S],
    K f64 [S,9], P_gt f64 [S,4,4]).  Coordinates are float32: that is what the loaders produced
    before the .npy detour promoted them (data/kitti_pc_img_pose_loader.py:431)."""
    if names is None:
        names = list_records(data_dir)
    recs = [load_record(data_dir, n, which, enu2cam) for n in names]
    S = len(recs)
    n_max = max((r[0].shape[1] for r in recs), default=0)
    xyz = np.zeros((S, 3, n_max), dtype=np.float32)
    label = np.full((S, n_max), -1, dtype=np.int8)
    n_pts = np.zeros((S,), dtype=np.int32)
    K = np.zeros((S, 9), dtype=np.float64)
    P = np.zeros((S, 4, 4), dtype=np.float64)
    for s, (pc, lab, k, p) in enumerate(recs):
        n = pc.shape[1]
        pc32 = pc.astype(np.float32)
        if pc.dtype != np.float32 and not np.array_equal(pc32.astype(pc.dtype), pc):
            raise ValueError("%s: coordinates are not float32-representable; use frustum.pack_clouds" % names[s])
        xyz[s, :, :n] = pc32
        label[s, :n] = np.where(lab == 1, 1, np.where(lab == 0, 0, -1)).astype(np.int8)
        n_pts[s] = n
        K[s] = k.reshape(9)
        P[s] = p
    return dict(names=list(names), xyz=xyz, label=label, n_pts=n_pts, K=K, P_gt=P)


def load_batch_fine(data_dir, names=None, coarse="coarse_prediction", fine="fine_prediction", enu2cam=False):
    """Legacy directory -> host arrays for the PnP path (registration_pnp.py:185-196 reads the same rows).

    Returns dict(names, xyz f32 [S,3,Nmax], coarse int8 [S,Nmax] (1 = predicted inside, 0 otherwise and on padding),
    fine int32 [S,Nmax] (grid cell), n_pts int32 [S], K f64 [S,9], P_gt f64 [S,4,4])."""
    if names is None:
        names = list_records(data_dir)
    rec = load_batch(data_dir, names, coarse, enu2cam)
    S, n_max = rec["label"].shape
    fine_rows = np.zeros((S, n_max), dtype=np.int32)
    for s, name in enumerate(names):
        _, f, _, _ = load_record(data_dir, name, fine, enu2cam)
        if f.size and (f.min() < -2 ** 31 or f.max() >= 2 ** 31):
            raise ValueError("%s: fine cell indices do not fit int32" % name)
        fine_rows[s, :f.shape[0]] = f
    coarse_rows = (rec["label"] == 1).astype(np.int8)
    return dict(names=rec["names"], xyz=rec["xyz"], coarse=coarse_rows, fine=fine_rows, n_pts=rec["n_pts"],
                K=rec["K"], P_gt=rec["P_gt"])


def register_directory_pnp(data_dir, H, W, fine_scale=1 / 32.0, iterations=500, reproj_err=0.6, confidence=0.99,
                           seed=0, enu2cam=False, batch=512, names=None, device="cuda", out_dir=None):
    """The __main__ of evaluation/registration_pnp.py:151-259 as one function: every frame of a legacy directory
    through pnp.pnp_ransac_batch (the GPU path), errors by frustum.pose_error_batch, and the P_pred_all_np /
    P_gt_all_np / cost_all_np files (cost = outlier ratio) the analysis script expects (:257-259)."""
    import torch
    from . import frustum, pnp

    if names is None:
        names = list_records(data_dir)
    P_pred = np.zeros((len(names), 4, 4))
    P_gt = np.zeros((len(names), 4, 4))
    cost = np.zeros((len(names),))
    for a in range(0, len(names), batch):
        rec = load_batch_fine(data_dir, names[a:a + batch], enu2cam=enu2cam)
        S, n_in = rec["coarse"].shape
        ns = frustum.round_up(max(n_in, 1), 16)
        dev = torch.device(device)
        xyz = torch.zeros((S, 3, ns), dtype=torch.float32, device=dev)
        c8 = torch.zeros((S, ns), dtype=torch.int8, device=dev)
        f32 = torch.zeros((S, ns), dtype=torch.int32, device=dev)
        xyz[:, :, :n_in] = torch.from_numpy(rec["xyz"]).to(dev)
        c8[:, :n_in] = torch.from_numpy(rec["coarse"]).to(dev)
        f32[:, :n_in] = torch.from_numpy(rec["fine"]).to(dev)
        n_pts = torch.from_numpy(rec["n_pts"]).to(dev)
        out = pnp.pnp_ransac_batch(xyz, c8, f32, n_pts, rec["K"], H, W, scale=fine_scale, iterations=iterations,
                                   reproj_err=reproj_err, confidence=confidence, seed=seed + a)
        P_pred[a:a + batch] = out["P"].cpu().numpy()
        cost[a:a + batch] = out["outlier_ratio"].cpu().numpy()
        P_gt[a:a + batch] = rec["P_gt"]
    err = frustum.pose_error_batch(P_pred, P_gt)
    t_err, r_err, ok = err["t_err"].cpu().numpy(), err["r_err"].cpu().numpy(), err["success"].cpu().numpy()
    if out_dir is not None:
        os.makedirs(out_dir, exist_ok=True)
        np.save(os.path.join(out_dir, "P_pred_all_np.npy"), P_pred)
        np.save(os.path.join(out_dir, "P_gt_all_np.npy"), P_gt)
        np.save(os.path.join(out_dir, "cost_all_np.npy"), cost)
    return dict(names=names, P_pred=P_pred, P_gt=P_gt, cost=cost, t_err=t_err, r_err=r_err, success=ok,
                summary=summarize(t_err, r_err, cost, ok))


def get_p_diff(P_pred, P_gt):
    """get_P_diff of evaluation/icp/registration_icp.py:57-65 with the fold of :224-225, on the host: P_diff =
    np.linalg.inv(P_pred) P_gt, t = |P_diff[:3,3]|, r = sum |euler 'xzy'| in degrees (scipy), r > 180 -> 360 - r.
    The ICP poses carry the 2-D forcing, which is not a rigid transform, so the rigid inverse of pose_error_batch
    does not apply.  Returns (t_err [S], r_err [S])."""
    from scipy.spatial.transform import Rotation
    P_pred = np.asarray(P_pred, dtype=np.float64).reshape(-1, 4, 4)
    P_gt = np.asarray(P_gt, dtype=np.float64).reshape(-1, 4, 4)
    t_err = np.zeros(len(P_pred))
    r_err = np.zeros(len(P_pred))
    for s in range(len(P_pred)):
        D = np.dot(np.linalg.inv(P_pred[s]), P_gt[s])
        t_err[s] = np.linalg.norm(D[0:3, 3])
        r = np.sum(np.abs(Rotation.from_matrix(D[0:3, 0:3]).as_euler("xzy", degrees=True)))
        r_err[s] = 360 - r if r > 180 else r
    return t_err, r_err


def register_directory_icp(data_dir, monodepth_dir, H, W, n_inits=60, seed=0, max_corr_dist=1.0, max_iteration=30,
                           enu2cam=False, batch=64, names=None, device="cuda", out_dir=None, t_thresh=2.0,
                           r_thresh=5.0):
    """The __main__ of evaluation/icp/registration_icp.py:165-245 as one function: every frame of a legacy directory
    and its <monodepth_dir>/<id>_pc.npy depth cloud, scale-calibrated with the ground truth (icp.calibrate_scale),
    through icp.icp_register_batch (the GPU path, random_inits(S, n_inits, seed + first frame of the batch)), errors
    by get_p_diff, and the P_pred_all_np / P_gt_all_np / cost_all_np files (cost = fitness, :241-243)."""
    import torch
    from . import icp

    if names is None:
        names = list_records(data_dir)
    P_pred = np.zeros((len(names), 4, 4))
    P_gt = np.zeros((len(names), 4, 4))
    cost = np.zeros((len(names),))
    for a in range(0, len(names), batch):
        srcs, tgts = [], []
        for s, name in enumerate(names[a:a + batch]):
            pc, _, K, P = load_record(data_dir, name, enu2cam=enu2cam)
            depth = np.load(os.path.join(monodepth_dir, name + "_pc.npy")).astype(np.float64)
            if depth.ndim != 2 or depth.shape[0] != 3:
                raise ValueError("%s_pc.npy: expected [3, N], got %s" % (name, depth.shape))
            depth = depth * icp.calibrate_scale(pc, P, K, H, W, depth)
            srcs.append(pc)
            tgts.append(depth)
            P_gt[a + s] = P
        src, n = icp.pack_clouds(srcs, device)
        tgt, m = icp.pack_clouds(tgts, device)
        init = torch.from_numpy(icp.random_inits(len(srcs), n_inits, seed + a)).to(src.device)
        out = icp.icp_register_batch(src, n, tgt, m, init, max_corr_dist=max_corr_dist, max_iteration=max_iteration)
        P_pred[a:a + batch] = out["P"].cpu().numpy()
        cost[a:a + batch] = out["fitness"].cpu().numpy()
    t_err, r_err = get_p_diff(P_pred, P_gt)
    ok = ((t_err < t_thresh) & (r_err < r_thresh)).astype(np.int32)
    if out_dir is not None:
        os.makedirs(out_dir, exist_ok=True)
        np.save(os.path.join(out_dir, "P_pred_all_np.npy"), P_pred)
        np.save(os.path.join(out_dir, "P_gt_all_np.npy"), P_gt)
        np.save(os.path.join(out_dir, "cost_all_np.npy"), cost)
    return dict(names=names, P_pred=P_pred, P_gt=P_gt, cost=cost, t_err=t_err, r_err=r_err, success=ok,
                summary=summarize(t_err, r_err, cost, ok))


def summarize(t_err, r_err, cost, ok):
    """registration_result_analysis.py:19-47 on the per-frame errors: frames with cost <= 1e-6 are dropped,
    RTE/RRE mean and sigma, success rate over the kept frames."""
    t_err, r_err, cost, ok = (np.asarray(a) for a in (t_err, r_err, cost, ok))
    valid = cost > 1e-6
    t, r, s = t_err[valid], r_err[valid], ok[valid]
    n = int(valid.sum())
    if n == 0:
        return dict(n=0, rte_mean=math.nan, rte_sigma=math.nan, rre_mean=math.nan, rre_sigma=math.nan,
                    success_rate=math.nan)
    return dict(n=n, rte_mean=float(t.mean()), rte_sigma=float(math.sqrt(t.var())), rre_mean=float(r.mean()),
                rre_sigma=float(math.sqrt(r.var())), success_rate=float(s.astype(np.float64).mean()))


def register_directory(data_dir, H, W, which="coarse_prediction", enu2cam=False, n_inits=60, seed=0, is_2d=True,
                       batch=512, names=None, device="cuda", out_dir=None):
    """The __main__ of evaluation/registration_lsq.py:250-398 as one function: every frame of a legacy
    directory through frustum.register_batch (the GPU path), errors by frustum.pose_error_batch, and the
    P_pred_all_np / P_gt_all_np / cost_all_np files the analysis script expects (:396-398)."""
    import torch
    from . import frustum

    if names is None:
        names = list_records(data_dir)
    P_pred = np.zeros((len(names), 4, 4))
    P_gt = np.zeros((len(names), 4, 4))
    cost = np.zeros((len(names),))
    for a in range(0, len(names), batch):
        rec = load_batch(data_dir, names[a:a + batch], which, enu2cam)
        n_in = rec["xyz"].shape[2]
        ns = frustum.round_up(max(n_in, 1), 16)
        xyz = torch.zeros((len(rec["names"]), 3, ns), dtype=torch.float32, device=device)
        pred = torch.full((len(rec["names"]), ns), -1, dtype=torch.int8, device=device)
        xyz[:, :, :n_in] = torch.from_numpy(rec["xyz"]).to(device)
        pred[:, :n_in] = torch.from_numpy(rec["label"]).to(device)
        out = frustum.register_batch(xyz, pred, n_in, rec["K"], H, W, n_inits=n_inits, seed=seed + a, is_2d=is_2d)
        P_pred[a:a + batch] = out["P"].cpu().numpy()
        cost[a:a + batch] = out["cost"].cpu().numpy()
        P_gt[a:a + batch] = rec["P_gt"]
    err = frustum.pose_error_batch(P_pred, P_gt)
    t_err, r_err, ok = err["t_err"].cpu().numpy(), err["r_err"].cpu().numpy(), err["success"].cpu().numpy()
    if out_dir is not None:
        os.makedirs(out_dir, exist_ok=True)
        np.save(os.path.join(out_dir, "P_pred_all_np.npy"), P_pred)
        np.save(os.path.join(out_dir, "P_gt_all_np.npy"), P_gt)
        np.save(os.path.join(out_dir, "cost_all_np.npy"), cost)
    return dict(names=names, P_pred=P_pred, P_gt=P_gt, cost=cost, t_err=t_err, r_err=r_err, success=ok,
                summary=summarize(t_err, r_err, cost, ok))
