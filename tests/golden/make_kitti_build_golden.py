"""Write tests/golden/kitti_build_small.npz: the KITTI accumulated-frame records of a small seeded root
(synthetic.write_kitti_root with ROOT_ARGS, one sequence), computed by oracle_kitti_build on the CPU.  No GPU, no
network:

    python tests/golden/make_kitti_build_golden.py [OUT.npz] [--reference DIR]

BUILD_ARGS give accumulate_frames = round(10 / 4) = round(2.5) = 2 (Python rounds the half to even), so every window
but the ones at the sequence ends holds five stride frames.  Two frames have all their intensities set to zero
(ZERO_INTENSITY, the last two stride frames), so the last frame, whose window holds only those two, carries a NaN
intensity row as numpy's 0 / 0 gives the reference.

With --reference DIR the generator also runs the reference's own accumulate_sequence (data/kitti/frame_accumulation.py,
unedited) on the same root, with open3d's voxel_down_sample stubbed by oracle_nuscenes.voxel_downsample64 (the
project's restatement of Open3D, DESIGN.md 4.10) and matplotlib, util.vis_tools and data.kitti_helper by empty
modules, and reports how its records compare with the oracle's.  Only np.dot's BLAS order of the transform differs.

Stored: the stride list, the windows, every frame's P_transform stack, the records (concatenated, with m_pts) and the
parameters.
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

SEQ = 3
ROOT_ARGS = dict(seqs=(SEQ,), n_frames=20, seed=5, n_rings=8, n_azimuth=48, image_hw=(8, 8), n_images=1)
BUILD_ARGS = dict(frame_stride_dist=4, accumulate_radius=10, voxel_size=0.4)
ZERO_INTENSITY = (13, 18)


def write_root(root):
    """The seeded root: write_kitti_root, then the frames of ZERO_INTENSITY with intensity 0."""
    from deepi2p_b200 import kitti, synthetic as syn
    syn.write_kitti_root(root, **ROOT_ARGS)
    for i in ZERO_INTENSITY:
        p = kitti.record_path(root, SEQ, i)
        r = np.load(p)
        r[3] = 0.0
        np.save(p, r)
    return root


def compute(root):
    import oracle_kitti_build as okb
    from deepi2p_b200 import kitti
    Tr = kitti.read_calib(root, SEQ)["Tr"]
    res = okb.accumulate_sequence(root, SEQ, Tr, **BUILD_ARGS)
    n = res["sample_num"]
    recs = [res["records"][i] for i in range(n)]
    return dict(seq=np.array(SEQ), root_args=np.array(repr(ROOT_ARGS)), build_args=np.array(repr(BUILD_ARGS)),
                zero_intensity=np.array(ZERO_INTENSITY, dtype=np.int64),
                strides=np.array(res["strides"], dtype=np.int64), acc=np.array(res["acc"]),
                windows=np.array(res["windows"], dtype=np.int64),
                window_strides=np.concatenate([[j for j, _ in res["transforms"][i]] for i in range(n)]).astype(np.int64),
                P=np.concatenate([np.stack([P for _, P in res["transforms"][i]]) for i in range(n)]),
                m_pts=np.array([r.shape[1] for r in recs], dtype=np.int64), records=np.concatenate(recs, 1))


def run_reference(ref_dir, root):
    """The reference's accumulate_sequence on `root` with the stubs above; returns {frame: record}."""
    import oracle_nuscenes
    from deepi2p_b200 import kitti

    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    class PointCloud:
        def voxel_down_sample(self, voxel_size):
            p = np.asarray(self.points, dtype=np.float64).T
            A = np.concatenate([np.asarray(self.colors, dtype=np.float64).T, np.asarray(self.normals).T])
            px, m = oracle_nuscenes.voxel_downsample64(p, voxel_size, A)
            out = PointCloud()
            out.points, out.colors, out.normals = px.T, m[0:3].T, m[3:6].T
            return out

    mod("open3d", geometry=types.SimpleNamespace(PointCloud=PointCloud),
        utility=types.SimpleNamespace(Vector3dVector=lambda a: np.array(a, dtype=np.float64)))
    mod("matplotlib", use=lambda *a, **k: None)
    mod("matplotlib.pyplot")
    mod("matplotlib.cm")
    mod("mpl_toolkits", __path__=[])
    mod("mpl_toolkits.mplot3d", Axes3D=None)
    mod("util", __path__=[], vis_tools=mod("util.vis_tools"))
    mod("data", __path__=[], kitti_helper=mod("data.kitti_helper"))
    spec = importlib.util.spec_from_file_location("frame_accumulation", os.path.join(ref_dir, "data", "kitti",
                                                                                     "frame_accumulation.py"))
    fa = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(fa)
    a = BUILD_ARGS
    Tr = kitti.read_calib(root, SEQ)["Tr"]
    with np.errstate(divide="ignore", invalid="ignore"):
        fa.accumulate_sequence(root, SEQ, Tr, a["frame_stride_dist"], a["accumulate_radius"], a["voxel_size"],
                               is_plot=False)
    d = os.path.join(root, "data_odometry_velodyne_NWU", "sequences", "%02d" % SEQ,
                     "stride%d-acc%d-voxel%.1f" % (a["frame_stride_dist"], a["accumulate_radius"], a["voxel_size"]))
    return {int(f[:6]): np.load(os.path.join(d, f)) for f in sorted(os.listdir(d))}


def make(out_path, ref_dir=None):
    with tempfile.TemporaryDirectory() as tmp:
        root = write_root(os.path.join(tmp, "kitti"))
        res = compute(root)
        if ref_dir is not None:
            ref = run_reference(ref_dir, root)
            off = np.concatenate([[0], np.cumsum(res["m_pts"])])
            same, worst = 0, 0
            for i, r in ref.items():
                o = res["records"][:, off[i]:off[i + 1]]
                if r.shape == o.shape and np.array_equal(r, o, equal_nan=True):
                    same += 1
                elif r.shape == o.shape:
                    d = np.abs(r.view(np.int32).astype(np.int64) - o.view(np.int32).astype(np.int64))
                    worst = max(worst, int(d[np.isfinite(r) & np.isfinite(o)].max(initial=0)))
                else:
                    worst = -1
            print(f"reference: {same} of {len(ref)} records bit-identical to the oracle's; "
                  f"largest difference elsewhere {worst} float32 ulps (-1: a count differs)")
    np.savez_compressed(out_path, **res)
    print(f"wrote {out_path}: {len(res['m_pts'])} records, {res['records'].shape[1]} points, "
          f"{os.path.getsize(out_path)} bytes")


if __name__ == "__main__":
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    ref = sys.argv[sys.argv.index("--reference") + 1] if "--reference" in sys.argv else None
    if ref is not None:
        args = [a for a in args if a != ref]
    make(args[0] if args else os.path.join(HERE, "kitti_build_small.npz"), ref)
