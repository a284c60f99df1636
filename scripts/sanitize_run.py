"""Small invocations of every kernel, for compute-sanitizer (memcheck / racecheck)."""
import sys, os
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deepi2p_b200 import frustum, point_ops, synthetic as syn

which = sys.argv[1] if len(sys.argv) > 1 else "all"
S, n, I = 2, 6000, 3        # 6 rounds of 1024 points = 2 slices per pass: the 6 problems run on 6 CTAs whose other warps HELP
smps = [syn.make_sample(40 + s, n) for s in range(S)]
xyz_in, pred_in, _ = frustum.pack_clouds(np.stack([s["points"] for s in smps]), np.stack([s["pred"] for s in smps]))
if which in ("all", "solver"):
    for is_2d in (True, False):
        out = frustum.register_batch(xyz_in, pred_in, n, smps[0]["K"], smps[0]["H"], smps[0]["W"], n_inits=I, seed=3,
                                     is_2d=is_2d, return_all=True)
        print("register_batch", is_2d, out["cost"].cpu().numpy())
    tr = frustum.solve_batch(*[frustum.prepare_batch(xyz_in, pred_in, n, I, seed=3)[k] for k in ("xyz", "label", "n_pts")],
                             smps[0]["K"], frustum.prepare_batch(xyz_in, pred_in, n, I, seed=3)["init"], smps[0]["H"], smps[0]["W"],
                             return_all=True, trace_cap=64)
    print("traced", int((tr["trace"][..., 15] > 0).sum()))
    x = np.zeros((S, 6)); x[:, 0] = 0.1; x[:, 3] = 1.0
    prep = frustum.prepare_batch(xyz_in, pred_in, n, I, seed=3, sort=False)
    c, g, A = frustum.evaluate_batch(prep["xyz"], prep["label"], prep["n_pts"], smps[0]["K"], x, smps[0]["H"], smps[0]["W"], True)
    r = frustum.residuals(prep["xyz"][0], prep["label"][0], int(prep["n_pts"][0]), smps[0]["K"], x[0, :4], smps[0]["H"], smps[0]["W"], True)
    m = frustum.inside_mask_batch(xyz_in, None, np.stack([s["P_gt"] for s in smps]), smps[0]["K"], smps[0]["H"], smps[0]["W"])
    e = frustum.pose_error_batch(out["P"], np.stack([s["P_gt"] for s in smps]))
    print("evaluate", c.cpu().numpy(), r.shape, int(m.sum()), e["t_err"].cpu().numpy())
    # f64 record
    pts64 = smps[0]["points"].astype(np.float64) + 1e-9
    xyz64, lab64, n64 = frustum.pack_clouds(pts64, smps[0]["pred"])
    o64 = frustum.solve_batch(xyz64, lab64, n64, smps[0]["K"], np.array([[[0.1, 0, 0, 1.0]]]), smps[0]["H"], smps[0]["W"])
    print("f64", o64["cost"].cpu().numpy())
    sx, sl, sn = frustum.sort_clouds(*frustum.pack_clouds(np.stack([s["points"] for s in smps]), np.stack([s["pred"] for s in smps]))[:2], n)
    print("sort_clouds", sn.tolist(), int((sl >= 0).sum()))
if which in ("all", "ops"):
    data, index = syn.make_index_max_inputs(1, 2, 6, 1030, 16)
    print("index_max", point_ops.index_max_forward(torch.from_numpy(data).cuda(), torch.from_numpy(index).cuda(), 16).sum().item())
    data, index = syn.make_index_max_inputs(1, 2, 8, 4096, 32)
    print("index_max vec", point_ops.index_max_forward(torch.from_numpy(data).cuda(), torch.from_numpy(index).cuda(), 32).sum().item())
    dist, radius = syn.make_ball_query_inputs(2, 2, 6, 5000, 16)
    print("ball_query split", point_ops.ball_query_forward(torch.from_numpy(dist).cuda(), radius, 16).sum().item())
    dist, radius = syn.make_ball_query_inputs(2, 2, 6, 8192, 16)
    print("ball_query split, 128-bit path", point_ops.ball_query_forward(torch.from_numpy(dist).cuda(), radius, 16).sum().item())
    dist, radius = syn.make_ball_query_inputs(2, 2, 6, 700, 16)
    print("ball_query warp", point_ops.ball_query_forward(torch.from_numpy(dist).cuda(), radius, 16).sum().item())
    rng = np.random.default_rng(0)
    pts = rng.uniform(0, 10, (2, 3, 3000)).astype(np.float32); nodes = rng.uniform(0, 10, (2, 3, 9)).astype(np.float32)
    print("ball_query_xyz", point_ops.ball_query_xyz_forward(torch.from_numpy(pts).cuda(), torch.from_numpy(nodes).cuda(), 1.5, 12).sum().item())
    ca = point_ops.cluster_assign_forward(torch.from_numpy(pts).cuda(), torch.from_numpy(nodes).cuda(), 3)
    print("cluster_assign", ca["count"].sum().item(), ca["pc_decentered"].abs().sum().item())
if which in ("all", "pnp"):
    from deepi2p_b200 import pnp
    fines = [syn.make_fine_labels(s, seed=i) for i, s in enumerate(smps)]
    pts = [s["points"] for s in smps] + [smps[0]["points"][:, :40]]          # a ragged third frame
    pred = [s["pred"] for s in smps] + [np.ones(40, np.int32)]
    args = pnp.pack_frames(pts, pred, fines + [fines[0][:40]])
    o = pnp.pnp_ransac_batch(*args, smps[0]["K"], smps[0]["H"], smps[0]["W"], iterations=150, return_all=True)
    print("pnp_ransac", o["inliers"].cpu().tolist(), o["hyp_used"].cpu().tolist())
    rng = np.random.default_rng(1)
    print("epnp", pnp.epnp_batch([(rng.uniform(1, 9, (n_, 3)), rng.uniform(0, 16, (n_, 2))) for n_ in (5, 40)],
                                 np.eye(3))[1].tolist())
torch.cuda.synchronize()
print("done")
