#!/usr/bin/env python
"""Register every frame of a legacy hand-off directory on the GPU.

Replaces `python evaluation/registration_lsq.py` + `registration_result_analysis.py` of the reference
(registration_lsq.py:250-398, registration_result_analysis.py:13-47) for directories written by
visualize_and_save_data.py:174-186, and, with --method pnp, `python evaluation/registration_pnp.py`
(registration_pnp.py:151-259: grid classification + PnP-RANSAC, cost = outlier ratio) and, with --method icp,
`python evaluation/icp/registration_icp.py` (registration_icp.py:165-245: monodepth cloud + multi-start ICP,
cost = fitness; the depth clouds <id>_pc.npy come from --monodepth, or are made on the GPU from the
<id>_img.png frames of the sibling visualization/ directory by the monodepth2 checkpoint in --depth-model, as
save_depth_map.py would).  Examples:

    python scripts/register_dir.py /data/kitti/save/run/data --H 160 --W 512 --out /data/kitti/save/run
    python scripts/register_dir.py /data/kitti/save/run/data --H 160 --W 512 --method pnp --fine-scale 0.03125
    python scripts/register_dir.py /data/oxford/run/data --H 384 --W 640 --method icp --monodepth /data/oxford/run/monodepth
    python scripts/register_dir.py run/data --H 384 --W 640 --method icp --depth-model models/mono+stereo_640x192
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from deepi2p_b200 import handoff  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("data_dir")
    ap.add_argument("--H", type=float, required=True, help="image height (kitti 160, oxford 384, nuscenes 160)")
    ap.add_argument("--W", type=float, required=True, help="image width (kitti 512, oxford 640, nuscenes 320)")
    ap.add_argument("--method", default="lsq", choices=("lsq", "pnp", "icp"),
                    help="lsq: frustum classification + inverse camera projection (registration_lsq.py); "
                         "pnp: grid classification + PnP-RANSAC (registration_pnp.py); "
                         "icp: monodepth cloud + multi-start ICP (icp/registration_icp.py)")
    ap.add_argument("--monodepth", default=None,
                    help="icp only (this or --depth-model): directory of the <id>_pc.npy depth clouds "
                         "(save_depth_map.py)")
    ap.add_argument("--depth-model", default=None,
                    help="icp only (this or --monodepth): monodepth2 checkpoint directory (encoder.pth, "
                         "depth.pth); the depth clouds are made on the GPU from the <id>_img.png frames in "
                         "visualization/ beside data_dir")
    ap.add_argument("--labels", default="coarse_prediction", choices=sorted(handoff.LABEL_ROWS),
                    help="lsq only: the in/out-of-frustum row the solver reads")
    ap.add_argument("--fine-scale", type=float, default=1 / 32.0,
                    help="pnp only: fine grid resolution relative to the image (registration_pnp.py:163)")
    ap.add_argument("--iterations", type=int, default=500, help="pnp only: RANSAC iterations (iterationsCount)")
    ap.add_argument("--enu2cam", action="store_true", help="nuScenes axis convention (registration_lsq.py:236-247)")
    ap.add_argument("--inits", type=int, default=60, help="lsq and icp: multi-start inits per frame")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--is-3d", action="store_true")
    ap.add_argument("--every", type=int, default=1, help="take every n-th frame (the reference uses 30, :285)")
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--out", default=None, help="where to write P_pred_all_np.npy / P_gt_all_np.npy / cost_all_np.npy")
    args = ap.parse_args()

    if args.method == "lsq" and args.labels.startswith("fine_"):
        ap.error("--labels %s holds grid cell indices, not in/out-of-frustum labels; use --method pnp" % args.labels)
    if args.method == "icp" and args.monodepth is None and args.depth_model is None:
        ap.error("--method icp needs --monodepth DIR (the <id>_pc.npy depth clouds) or --depth-model DIR")
    if args.method == "icp" and args.monodepth is not None and args.depth_model is not None:
        ap.error("--monodepth and --depth-model are alternatives; give one")
    if args.method != "icp" and args.monodepth is not None:
        ap.error("--monodepth is only used by --method icp")
    if args.method != "icp" and args.depth_model is not None:
        ap.error("--depth-model is only used by --method icp")
    names = handoff.list_records(args.data_dir)[::args.every]
    if args.method == "icp":
        model = None
        if args.depth_model is not None:
            from deepi2p_b200 import monodepth
            model = monodepth.load_monodepth(args.depth_model)
        res = handoff.register_directory_icp(args.data_dir, args.monodepth, args.H, args.W, n_inits=args.inits,
                                             seed=args.seed, enu2cam=args.enu2cam, batch=args.batch,
                                             names=names, out_dir=args.out, depth_model=model)
    elif args.method == "pnp":
        res = handoff.register_directory_pnp(args.data_dir, args.H, args.W, fine_scale=args.fine_scale,
                                             iterations=args.iterations, seed=args.seed, enu2cam=args.enu2cam,
                                             batch=args.batch, names=names, out_dir=args.out)
    else:
        res = handoff.register_directory(args.data_dir, args.H, args.W, which=args.labels, enu2cam=args.enu2cam,
                                         n_inits=args.inits, seed=args.seed, is_2d=not args.is_3d, batch=args.batch,
                                         names=names, out_dir=args.out)
    for i, n in enumerate(res["names"]):
        fmt = {"pnp": "%s - cost: %.2f, T: %.1f, R:%.1f", "icp": "%s - fitness: %.1f, T: %.1f, R:%.1f"}.get(
            args.method, "%s - cost: %.1f, T: %.1f, R:%.1f")
        print(fmt % (n, res["cost"][i], res["t_err"][i], res["r_err"][i]))
    s = res["summary"]
    print("RTE %.2f +- %.2f, RRE %.2f +- %.2f, success rate %.2f" % (s["rte_mean"], s["rte_sigma"], s["rre_mean"],
                                                                     s["rre_sigma"], s["success_rate"] * 100))
    print(json.dumps(s))


if __name__ == "__main__":
    main()
