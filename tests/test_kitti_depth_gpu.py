"""KITTI camera-frame records and depth maps on the GPU (deepi2p_b200.kitti_depth) against the golden file and the
numpy oracle (oracle_kitti_depth), bit for bit."""
import importlib.util
import os

import numpy as np
import pytest
import torch

import oracle_kitti_depth as okd
from deepi2p_b200 import kitti, kitti_depth, synthetic as syn
from deepi2p_b200.icp import pack_clouds

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _mk():
    spec = importlib.util.spec_from_file_location("mk_kitti_depth",
                                                  os.path.join(ROOT, "tests", "golden", "make_kitti_depth_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    return mk


@pytest.fixture(scope="module")
def golden_root(tmp_path_factory):
    mk = _mk()
    root, vel = mk.write_root(str(tmp_path_factory.mktemp("kd")))
    with np.load(os.path.join(ROOT, "tests", "golden", "kitti_depth_small.npz")) as z:
        records, maps = mk.unpack(dict(z))
    return mk, root, vel, records, maps


def _gpu_map(p, Pc, K, H, W):
    xyz, n = pack_clouds([p])
    return kitti_depth.depth_maps(xyz, n, Pc[None], K[None], H, W)[0].cpu().numpy()


def test_every_map_and_record_against_the_fixture(golden_root):
    mk, root, vel, records, maps = golden_root
    plan = kitti_depth.plan_sequence(root, vel, mk.SEQ)
    res = kitti_depth.build_frames(plan, list(range(plan["n"])))
    for key, r in records.items():
        assert np.array_equal(res["records"][key], r), key
        assert np.array_equal(res["maps"][key], maps[key]), key


def test_fixture_frames_against_the_oracle(golden_root):
    mk, root, vel, records, maps = golden_root
    plan = kitti_depth.plan_sequence(root, vel, mk.SEQ)
    scan = kitti_depth.read_scan(kitti_depth.velodyne_path(vel, mk.SEQ, 2))
    for k in okd.CAMERAS:
        H, W = plan["sizes"][k][2]
        assert np.array_equal(_gpu_map(scan[:3], plan["Pc"][k], plan["K"][k], H, W),
                              okd.depth_map(scan[:3], plan["Pc"][k], plan["K"][k], H, W))


@pytest.mark.parametrize("batch", [1, 3, 64])
def test_batches_give_the_same_bytes(golden_root, batch):
    mk, root, vel, records, maps = golden_root
    plan = kitti_depth.plan_sequence(root, vel, mk.SEQ)
    n = plan["n"]
    for s in range(0, n, batch):
        res = kitti_depth.build_frames(plan, list(range(s, min(s + batch, n))))
        for key, m in res["maps"].items():
            assert np.array_equal(m, maps[key]), key
            assert np.array_equal(res["records"][key], records[key]), key


def test_second_stream(golden_root):
    mk, root, vel, records, maps = golden_root
    plan = kitti_depth.plan_sequence(root, vel, mk.SEQ)
    scans = [kitti_depth.read_scan(kitti_depth.velodyne_path(vel, mk.SEQ, i)) for i in (0, 1, 2)]
    xyz, n = pack_clouds([s[:3] for s in scans])
    Pc = np.stack([plan["Pc"][k] for _ in scans for k in okd.CAMERAS])
    K = np.stack([plan["K"][k] for _ in scans for k in okd.CAMERAS])
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        out = kitti_depth.depth_maps(xyz, n, Pc, K, *mk.HW, stream=st)
    st.synchronize()
    out = out.cpu().numpy()
    for s in range(3):
        for c, k in enumerate(okd.CAMERAS):
            assert np.array_equal(out[2 * s + c], maps[(s, k)])


# Constructed cases under a pure-axis Pc (camera = velodyne axes) and K = (4, 4, 3, 2) on a 5 x 7 image: u / w =
# 4 X / Z + 3, v / w = 4 Y / Z + 2, all exact for the coordinates below.
AXIS_K = np.array([[4, 0, 3], [0, 4, 2], [0, 0, 1]], dtype=np.float32)
H5, W7 = 5, 7


def _axis(points, tz=0.0):
    Pc = np.eye(4)
    Pc[2, 3] = tz
    p = np.asarray(points, dtype=np.float32).T
    return p, Pc


def _both(p, Pc, K=AXIS_K, H=H5, W=W7):
    g = _gpu_map(p, Pc, K, H, W)
    o = okd.depth_map(p, Pc, K, H, W)
    assert np.array_equal(g, o)
    return g


def test_depth_of_exactly_point_one_is_not_projected():
    # Z = 0 + 0.1 (the translation) is exactly 0.1: not > 0.1 (it would land on (2, 4)); a point just beyond counts
    p, Pc = _axis([(0.025, 0.0, 0.0), (0.0, 0.0, 1e-7)], tz=0.1)
    g = _both(p, Pc)
    assert [tuple(v) for v in np.argwhere(g[1] < 0.75)] == [(2, 3)]


def test_halves_at_both_borders_round_to_even():
    # u / w = -0.5 -> 0 (inside), W - 0.5 = 6.5 -> 6 (inside), 7.5 -> 8 (outside); v / w = -0.5 -> 0, 4.5 -> 4
    p, Pc = _axis([(-0.875, 0.0, 1.0), (0.875, 0.0, 1.0), (1.125, 0.0, 1.0), (0.0, -0.625, 1.0), (0.0, 0.625, 1.0)])
    g = _both(p, Pc)
    filled = np.argwhere(g[1] < 0.75)
    assert sorted(map(tuple, filled)) == [(0, 3), (2, 0), (2, 6), (4, 3)]
    assert np.all(g[1][g[1] < 0.75] == 0.5)


def test_duplicates_on_one_ray_keep_the_last_when_d_rounds_up_and_the_first_otherwise():
    # Points on one ray share the pixel and d exactly, with different Z.  d = sqrt(dx^2 + dy^2) either rounds up to
    # float32 (the later point wins: d < (double) float32(d)) or down / exactly (the first one stays).
    rng = np.random.default_rng(3)
    up = down = 0
    for _ in range(64):
        X, Y = rng.uniform(-0.1, 0.1, 2).astype(np.float32)
        pts = [(X * z, Y * z, z) for z in (1.0, 2.0, 4.0)]
        p, Pc = _axis(pts)
        g = _both(p, Pc)
        d = okd.project_loop(p, Pc, AXIS_K, H5, W7)
        px = 4.0 * np.float64(X) + 3
        py = 4.0 * np.float64(Y) + 2
        dd = np.sqrt((px - np.rint(px)) ** 2 + (py - np.rint(py)) ** 2)
        pix = (int(np.rint(py)), int(np.rint(px)))
        if dd < np.float64(np.float32(dd)):
            up += 1
            assert g[0][pix] == 4.0
        else:
            down += 1
            assert g[0][pix] == 1.0
        assert d[0][pix] == g[0][pix]
    assert up and down


def test_empty_image_reads_the_bottom_left_pixel():
    p, Pc = _axis([(0.0, 0.0, -1.0), (1.0, 1.0, 0.05)])
    g = _both(p, Pc)
    r, c = np.mgrid[0:H5, 0:W7]
    assert np.all(g[0] == 0)
    assert np.array_equal(g[1], np.sqrt(((r + 1) ** 2 + c ** 2).astype(np.float64)).astype(np.float32))


def test_scan_sized_maps_against_the_oracle():
    sc = syn.make_lidar_scan(11, n_rings=32, n_azimuth=512)
    Pc = np.array([[0, -1, 0, 0.06], [0, 0, -1, -0.08], [1, 0, 0, -0.27], [0, 0, 0, 1]], dtype=np.float64)
    K = np.array([[95.3, 0, 80.1], [0, 95.3, 24.7], [0, 0, 1]], dtype=np.float32)
    _both(sc["xyz"], Pc, K, 50, 161)


def _write(tmp_path, n=4, sizes=None):
    mk = _mk()
    root, vel = str(tmp_path / "kitti"), str(tmp_path / "vel")
    syn.write_kitti_velodyne_root(root, vel, 1, mk.scans()[:n], sizes or [mk.HW] * n, mk.K)
    return root, vel


def test_build_sequence_files_to_files(tmp_path):
    root, vel = _write(tmp_path)
    mk = _mk()
    assert kitti_depth.build_sequence(root, vel, 1, batch=3) == 4
    plan = kitti_depth.plan_sequence(root, vel, 1)
    recs, maps = okd.process_sequence(root, vel, 1, plan["Pc"], plan["K"], plan["sizes"])
    for (i, k), r in recs.items():
        assert np.array_equal(np.load(os.path.join(kitti_depth.record_dir(root, 1, k), "%06d.npy" % i)), r)
        assert np.array_equal(np.load(os.path.join(kitti_depth.depth_dir(root, 1, k), "%06d.npy" % i)), maps[(i, k)])
    assert not any(os.path.exists(d + ".partial") for d in kitti_depth.output_dirs(root, 1))
    logs = []
    assert kitti_depth.build_sequence(root, vel, 1, log=logs.append) == 0       # the folders exist: skipped
    assert "skip" in logs[0]
    assert kitti_depth.build_root(root, vel, seqs=(1,)) == {1: 0}
    del mk


def test_build_sequence_errors(tmp_path):
    root, vel = _write(tmp_path)
    os.remove(kitti.image_path(root, 1, "P3", 2))
    with pytest.raises(FileNotFoundError):
        kitti_depth.build_sequence(root, vel, 1)
    root2, vel2 = _write(tmp_path / "b")
    with open(kitti_depth.velodyne_path(vel2, 1, 1), "ab") as f:
        f.write(b"\0" * 4)
    with pytest.raises(ValueError, match="whole number"):
        kitti_depth.build_sequence(root2, vel2, 1)
    xyz, n = pack_clouds([np.zeros((3, 4), np.float32)])
    with pytest.raises(ValueError, match="Pc"):
        kitti_depth.depth_maps(xyz, n, np.eye(4)[None, :3], AXIS_K[None], 5, 7)
    with pytest.raises(ValueError, match="K"):
        kitti_depth.depth_maps(xyz, n, np.eye(4)[None], AXIS_K[None, :2], 5, 7)
    with pytest.raises(ValueError, match="H and W"):
        kitti_depth.depth_maps(xyz, n, np.eye(4)[None], AXIS_K[None], 0, 7)
    os.makedirs(kitti_depth.output_dirs(root2, 1)[0])
    with pytest.raises(FileExistsError):
        kitti_depth.build_sequence(root2, vel2, 1)


def test_prepare_scans_unchanged_by_the_shared_chain():
    from deepi2p_b200 import pointprep
    import oracle_prep
    sc = syn.make_lidar_scan(5, n_rings=16, n_azimuth=256)
    xyz, n = pack_clouds([sc["xyz"]])
    inten = torch.zeros((1, xyz.shape[2]), dtype=torch.float32)
    inten[0, :sc["xyz"].shape[1]] = torch.from_numpy(sc["intensity"])
    rec, m = pointprep.prepare_scans(xyz, inten.cuda(), n)
    ref = oracle_prep.prepare_scan(sc["xyz"], sc["intensity"])
    assert np.array_equal(rec[0, :, :int(m[0])].cpu().numpy(), ref)
