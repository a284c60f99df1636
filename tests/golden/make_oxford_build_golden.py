"""Write tests/golden/oxford_build_small.npz: the reference's own Oxford build (data/oxford/build_dataset.py) on a small
seeded raw traversal (synthetic.write_oxford_raw with RAW_ARGS), run on the CPU.  No GPU, no network:

    python tests/golden/make_oxford_build_golden.py [OUT.npz] [--reference DIR]

The reference runs unedited: VOManager, my_build_pointcloud, downsample and save_pc_img_for_traversal (images on,
plotting off).  Its imports are stubbed:
  - the RobotCar SDK: build_se3_transform and interpolate_poses are deepi2p_b200.oxford_build's restatement (DESIGN.md
    4.24), returned as np.matrix so that the reference's window-local chain `abs * rel` multiplies matrices;
  - CameraModel reads G_camera_image from the model file; load_image returns a tiny frame (cv2 writes it);
  - open3d's voxel_down_sample is oracle_nuscenes.voxel_downsample64 (the project's restatement of Open3D, 4.10);
  - matplotlib, mpl_toolkits and util.vis_tools are empty modules;
  - np.int / np.float, removed from numpy 2, are int / float for the reference's table writes.

Stored: the records of every built cloud, the four tables, the kept / skipped / missing scan counts per cloud and the
reference's window-local relative poses of three clouds' scans (for the global-chain bound of the CPU tests).
"""
import importlib.util
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

TRAVERSAL = "2014-05-19-13-20-57"
RAW_ARGS = dict(seconds=26.0, zero_reflectance_after=19.0, n_returns=8, seed=3)
BUILD_ARGS = dict(pc_sample_distance=2.0, min_vehicle_velocity=3.0, accumulation_distance=20.0,
                  ignore_first_n_second=2, voxel_grid_downsample_size=0.1, remove_ground_threshold=0.1)


def import_reference(ref_dir):
    from deepi2p_b200 import oxford_build as ob
    import oracle_nuscenes

    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    class CameraModel:
        def __init__(self, models_dir, images_dir):
            self.camera = "stereo"
            self.G_camera_image = ob.read_camera_model(os.path.join(models_dir, ob.CAMERA_MODEL))

    def interpolate_poses(pose_timestamps, abs_poses, requested_timestamps, origin_timestamp):
        out = ob.interpolate_poses(pose_timestamps, np.stack([np.asarray(p) for p in abs_poses]),
                                   list(requested_timestamps), origin_timestamp)
        return [np.matrix(p) for p in out]

    sdk = "data.oxford.robotcar_dataset_sdk.python"
    for name in ("data", "data.oxford", "data.oxford.robotcar_dataset_sdk", sdk):
        mod(name, __path__=[])
    mod(sdk + ".build_pointcloud", build_pointcloud=None)
    mod(sdk + ".transform", build_se3_transform=lambda v: np.matrix(ob.se3(v)))
    mod(sdk + ".image", load_image=lambda path, model: np.zeros((2, 2, 3), dtype=np.uint8))
    mod(sdk + ".camera_model", CameraModel=CameraModel)
    mod(sdk + ".interpolate_poses", interpolate_poses=interpolate_poses, interpolate_vo_poses=None)

    class PointCloud:
        def voxel_down_sample(self, voxel_size):
            p = np.asarray(self.points, dtype=np.float64).T
            c = np.asarray(self.colors, dtype=np.float64).T
            px, A = oracle_nuscenes.voxel_downsample64(p, voxel_size, c)
            out = PointCloud()
            out.points, out.colors = px.T, A.T
            return out

    mod("open3d", geometry=types.SimpleNamespace(PointCloud=PointCloud),
        utility=types.SimpleNamespace(Vector3dVector=lambda a: np.array(a, dtype=np.float64)))
    mod("matplotlib", use=lambda *a, **k: None)
    mod("matplotlib.pyplot")
    mod("matplotlib.cm")
    mod("mpl_toolkits", __path__=[])
    mod("mpl_toolkits.mplot3d", Axes3D=None)
    mod("util", __path__=[])
    mod("util.vis_tools")
    np.int, np.float = int, float
    spec = importlib.util.spec_from_file_location("build_dataset", os.path.join(ref_dir, "data", "oxford",
                                                                                "build_dataset.py"))
    bd = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bd)
    return bd


def make(out_path, ref_dir):
    from deepi2p_b200 import synthetic as syn
    bd = import_reference(ref_dir)
    with tempfile.TemporaryDirectory() as tmp:
        raw, lms, sdk, out = (os.path.join(tmp, d) for d in ("raw", "lms", "sdk", "out"))
        syn.write_oxford_raw(raw, lms, sdk, **RAW_ARGS)
        calls, windows = [], {}
        build = bd.my_build_pointcloud

        def my_build_pointcloud(G, lidar_dir, vo_manager, timestamps, origin_time, **kw):
            pc, refl, skip = build(G, lidar_dir, vo_manager, timestamps, origin_time, **kw)
            missing = sum(not os.path.isfile(os.path.join(lidar_dir, "%d.bin" % t)) for t in timestamps)
            calls.append((origin_time, len(timestamps), skip, missing))
            windows[origin_time] = (list(timestamps), np.stack([np.asarray(p) for p in
                                                                vo_manager.interpolate_vo_poses(timestamps,
                                                                                                origin_time)]))
            return pc, refl, skip

        bd.my_build_pointcloud = my_build_pointcloud
        a = BUILD_ARGS
        bd.save_pc_img_for_traversal(TRAVERSAL, lms, raw, out, os.path.join(sdk, "models"),
                                     os.path.join(sdk, "extrinsics"), True, a["remove_ground_threshold"], True,
                                     False, False, a["pc_sample_distance"], a["min_vehicle_velocity"],
                                     a["accumulation_distance"], a["ignore_first_n_second"],
                                     a["voxel_grid_downsample_size"])
        d = os.path.join(out, TRAVERSAL)
        pc_ts = np.load(os.path.join(d, "pc_timestamps.npy"))
        recs = [np.load(os.path.join(d, "lms_front_foreground", "%d.npy" % t)) for t in pc_ts]
        sel = [int(pc_ts[0]), int(pc_ts[len(pc_ts) // 2]), int(pc_ts[-1])]
        res = dict(
            traversal=np.array(TRAVERSAL), raw_args=np.array(repr(RAW_ARGS)), build_args=np.array(repr(BUILD_ARGS)),
            pc_timestamps=pc_ts, pc_poses=np.load(os.path.join(d, "pc_poses.npy")),
            camera_timestamps=np.load(os.path.join(d, "camera_timestamps.npy")),
            camera_poses=np.load(os.path.join(d, "camera_poses.npy")),
            m_pts=np.array([r.shape[1] for r in recs], dtype=np.int64),
            records=np.concatenate(recs, 1) if recs else np.zeros((4, 0), np.float32),
            window_len=np.array([c[1] for c in calls]), n_skipped=np.array([c[2] for c in calls]),
            n_missing=np.array([c[3] for c in calls]),
            n_kept=np.array([c[1] - c[2] - c[3] for c in calls]),
            pose_centres=np.array(sel, dtype=np.int64),
            pose_lms_ts=np.concatenate([windows[c][0] for c in sel]).astype(np.int64),
            pose_lens=np.array([len(windows[c][0]) for c in sel]),
            pose_rel=np.concatenate([windows[c][1] for c in sel]))
    np.savez_compressed(out_path, **res)
    print(f"wrote {out_path}: {len(pc_ts)} clouds, {res['records'].shape[1]} points, "
          f"{os.path.getsize(out_path)} bytes")


if __name__ == "__main__":
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    from oracle import build_ref
    ref = sys.argv[sys.argv.index("--reference") + 1] if "--reference" in sys.argv else build_ref.REF
    if "--reference" in sys.argv:
        args = [a for a in args if a != ref]
    make(args[0] if args else os.path.join(HERE, "oxford_build_small.npz"), ref)
