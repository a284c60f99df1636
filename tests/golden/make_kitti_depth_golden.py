"""Write tests/golden/kitti_depth_small.npz: the KITTI camera-frame records and depth maps of a small seeded root
(synthetic.write_kitti_velodyne_root, one sequence, both cameras), computed by oracle_kitti_depth on the CPU.  No
GPU, no network:

    python tests/golden/make_kitti_depth_golden.py [OUT.npz] [--reference DIR]

The root's five scans:
  0, 1  seeded make_lidar_scan scans;
  2     scan 1 plus planted points: on the P2 camera (Pc = Tr, K = (16, 16, 20, 6), all exact at Z = 8) pixel
        coordinates of exactly -0.5 and W - 0.5 = 40.5 in x and -0.5 and H - 0.5 = 12.5 in y (which round to the
        border pixels, halves to even), points on one ray at Z = 8 and 16 (one pixel, equal d, different depth),
        and the first DUPLICATES points of the scan appended again (equal d: the later copy wins only where d rounds
        up to float32);
  3     scan 0 without its points with x > -1: no point lands in either image;
  4     scan 0 with images of another size (12 x 40), so a batch splits there.

With --reference DIR the generator also runs the reference's own process_kitti
(data/kitti/kitti_pc_bin_to_npy_in_img_frame.py, unedited) on the same root, with open3d replaced by the oracle's
restatements (oracle_prep), matplotlib and util.vis_tools by empty modules and np.bool = bool, and reports how many
records and maps are bit-identical to the oracle's.

Stored: the parameters, the sizes, the records (concatenated along points, with m_pts) and the maps (flattened, in
(frame, camera) order).
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

SEQ = 4
K = (16.0, 16.0, 20.0, 6.0)
HW = (13, 41)
SIZES = [HW, HW, HW, HW, (12, 40)]
SCAN_ARGS = dict(n_rings=16, n_azimuth=256)
DUPLICATES = 400
BUILD_ARGS = dict(voxel_size=0.1, sn_radius=0.6, sn_max_nn=30)


def planted_points():
    """[4, n] float32 velodyne points (x = Z, y = -X, z = -Y of the P2 camera) at the halves and on one ray."""
    Z = 8.0
    cam = [(-10.25, 0.0), (10.25, 0.0), (0.0, -3.25), (0.0, 3.25), (10.75, 0.0), (-10.25, -3.25), (10.25, 3.25),
           (1.3, 0.7), (-4.1, 1.9)]
    pts = [(Z, -X, -Y) for X, Y in cam]
    pts += [(2 * Z, -2 * np.float32(X), -2 * np.float32(Y)) for X, Y in cam[-2:]]    # the same rays, twice as far
    p = np.array(pts, dtype=np.float32).T
    return np.concatenate([p, np.full((1, p.shape[1]), 0.5, dtype=np.float32)])


def scans():
    from deepi2p_b200 import synthetic as syn
    base = []
    for k in range(2):
        sc = syn.make_lidar_scan(100 + k, **SCAN_ARGS)
        base.append(np.concatenate([sc["xyz"], sc["intensity"][None]]).astype(np.float32))
    planted = np.concatenate([base[1], planted_points(), base[1][:, :DUPLICATES]], 1)
    behind = base[0][:, base[0][0] <= -1.0]
    return [base[0], base[1], planted, behind, base[0]]


def write_root(tmp):
    from deepi2p_b200 import synthetic as syn
    root, vel = os.path.join(tmp, "kitti"), os.path.join(tmp, "velodyne")
    syn.write_kitti_velodyne_root(root, vel, SEQ, scans(), SIZES, K)
    return root, vel


def compute(root, vel):
    import oracle_kitti_depth as okd
    from deepi2p_b200 import kitti
    calib = kitti.read_calib(root, SEQ)
    Pc = {k: kitti.camera_Pc(calib, k) for k in okd.CAMERAS}
    Kk = {k: calib[k + "_K"] for k in okd.CAMERAS}
    sizes = {k: SIZES for k in okd.CAMERAS}
    records, maps = okd.process_sequence(root, vel, SEQ, Pc, Kk, sizes, **BUILD_ARGS)
    keys = sorted(records)
    return dict(seq=np.array(SEQ), K=np.array(K), sizes=np.array(SIZES, dtype=np.int64),
                build_args=np.array(repr(BUILD_ARGS)), duplicates=np.array(DUPLICATES),
                Pc=np.stack([Pc[k] for k in okd.CAMERAS]),
                m_pts=np.array([records[k].shape[1] for k in keys], dtype=np.int64),
                records=np.concatenate([records[k] for k in keys], 1),
                maps=np.concatenate([maps[k].reshape(-1) for k in keys]))


def unpack(z):
    """{(frame, key): record} and {(frame, key): map} of a stored file (z: a dict or an NpzFile)."""
    sizes = [tuple(s) for s in z["sizes"]]
    keys = [(i, k) for i in range(len(sizes)) for k in ("P2", "P3")]
    off = np.concatenate([[0], np.cumsum(z["m_pts"])])
    records = {key: z["records"][:, off[j]:off[j + 1]] for j, key in enumerate(keys)}
    maps, o = {}, 0
    for i, k in keys:
        H, W = sizes[i]
        maps[(i, k)] = z["maps"][o:o + 2 * H * W].reshape(2, H, W)
        o += 2 * H * W
    return records, maps


def run_reference(ref_dir, root, vel):
    """The reference's process_kitti on the root with the stubs above; returns (records, maps) as unpack does."""
    import oracle_prep

    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    class PointCloud:
        points = normals = None

    def voxel_down_sample(pcd, voxel_size):
        out = PointCloud()
        out.points = oracle_prep.voxel_downsample(np.asarray(pcd.points).T, voxel_size)[0].T
        return out

    def estimate_normals(pcd, search_param):
        pcd.normals = oracle_prep.estimate_normals(np.asarray(pcd.points).T.astype(np.float32), search_param.radius,
                                                   search_param.max_nn)[0].T

    mod("open3d", geometry=types.SimpleNamespace(
        PointCloud=PointCloud, voxel_down_sample=voxel_down_sample, estimate_normals=estimate_normals,
        orient_normals_to_align_with_direction=lambda pcd, d: None,
        KDTreeSearchParamHybrid=lambda radius, max_nn: types.SimpleNamespace(radius=radius, max_nn=max_nn)),
        utility=types.SimpleNamespace(Vector3dVector=lambda a: np.array(a, dtype=np.float64)))
    mod("matplotlib", use=lambda *a, **k: None)
    mod("matplotlib.pyplot")
    mod("util", __path__=[], vis_tools=mod("util.vis_tools"))
    if ref_dir not in sys.path:
        sys.path.insert(0, ref_dir)
    import scipy.ndimage  # noqa: F401 - imported before np.bool exists: numpy.ma breaks when it does
    import scipy.spatial  # noqa: F401
    np.bool = bool
    spec = importlib.util.spec_from_file_location(
        "kitti_pc_bin_to_npy_in_img_frame",
        os.path.join(ref_dir, "data", "kitti", "kitti_pc_bin_to_npy_in_img_frame.py"))
    ref = importlib.util.module_from_spec(spec)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)
        spec.loader.exec_module(ref)
    import contextlib
    import io
    with contextlib.redirect_stdout(io.StringIO()):
        ref.process_kitti(root, vel, [SEQ], BUILD_ARGS["voxel_size"], BUILD_ARGS["sn_radius"], BUILD_ARGS["sn_max_nn"])
    records, maps = {}, {}
    for i in range(len(SIZES)):
        for k in ("P2", "P3"):
            records[(i, k)] = np.load(os.path.join(root, "data_odometry_velodyne_%s_npy" % k, "sequences",
                                                   "%02d" % SEQ, "voxel0.1-SNr0.6", "%06d.npy" % i))
            maps[(i, k)] = np.load(os.path.join(root, "data_odometry_color_depth_npy", "sequences", "%02d" % SEQ,
                                                "image_" + k[1], "%06d.npy" % i))
    return records, maps


def make(out_path, ref_dir=None):
    with tempfile.TemporaryDirectory() as tmp:
        root, vel = write_root(tmp)
        res = compute(root, vel)
        if ref_dir is not None:
            rr, rm = run_reference(ref_dir, root, vel)
            orr, om = unpack(res)
            for what, a, b in (("records", rr, orr), ("maps", rm, om)):
                same = [k for k in a if a[k].shape == b[k].shape and np.array_equal(a[k], b[k])]
                print(f"reference: {len(same)} of {len(a)} {what} bit-identical to the oracle's")
                for k in sorted(set(a) - set(same)):
                    if a[k].shape != b[k].shape:
                        print(f"  {k}: shape {a[k].shape} against {b[k].shape}")
                        continue
                    d = a[k] != b[k]
                    at = [tuple(int(v) for v in w) for w in np.argwhere(d)[:6]]
                    print(f"  {k}: {int(d.sum())} values differ, at {at}")
    np.savez_compressed(out_path, **res)
    print(f"wrote {out_path}: {len(res['m_pts'])} records ({res['records'].shape[1]} points) and maps, "
          f"{os.path.getsize(out_path)} bytes")


if __name__ == "__main__":
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    ref = sys.argv[sys.argv.index("--reference") + 1] if "--reference" in sys.argv else None
    if ref is not None:
        args = [a for a in args if a != ref]
    make(args[0] if args else os.path.join(HERE, "kitti_depth_small.npz"), ref)
