"""KITTI camera-frame records and depth maps, host side: the oracle's winner rule against the reference's literal
loop, the oracle's distance transform against scipy, the host plan (paths, sample_num, image sizes, calibration) and
the golden file."""
import importlib.util
import os
import warnings

import numpy as np
import pytest

import oracle_kitti_depth as okd
from deepi2p_b200 import kitti, kitti_depth, synthetic as syn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _golden_module():
    spec = importlib.util.spec_from_file_location("mk_kitti_depth",
                                                  os.path.join(ROOT, "tests", "golden", "make_kitti_depth_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    return mk


def _scipy_edt(mask_inv):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)
        from scipy.ndimage import distance_transform_edt
    return distance_transform_edt(mask_inv, return_indices=True, return_distances=True)


def _adversarial(seed, n=60):
    """Points crowded into few pixels of a 5 x 7 image under an axis Pc: duplicates, one-ray copies and halves."""
    rng = np.random.default_rng(seed)
    Pc = np.eye(4)
    K = np.array([[4, 0, 3], [0, 4, 2], [0, 0, 1]], dtype=np.float32)
    X = rng.integers(-2, 3, n) / 8 + rng.choice([0.0, 1 / 16, 1e-7], n) * rng.choice([-1, 1], n)
    Y = rng.integers(-1, 2, n) / 8 + rng.choice([0.0, 1 / 16, 3e-8], n)
    Z = rng.choice([1.0, 2.0, 4.0, 0.1], n)
    p = np.stack([X * Z, Y * Z, Z]).astype(np.float32)
    dup = rng.integers(0, n, n // 3)
    p = np.concatenate([p, p[:, dup]], 1)
    return p[:, rng.permutation(p.shape[1])], Pc, K


@pytest.mark.parametrize("seed", range(40))
def test_winner_rule_matches_the_literal_loop(seed):
    p, Pc, K = _adversarial(seed)
    a = okd.project_loop(p, Pc, K, 5, 7)
    b = okd.project_rule(p, Pc, K, 5, 7)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def test_winner_rule_on_a_scan():
    sc = syn.make_lidar_scan(3, n_rings=16, n_azimuth=512)
    Pc = np.array([[0, -1, 0, 0.1], [0, 0, -1, -0.05], [1, 0, 0, -0.3], [0, 0, 0, 1]], dtype=np.float64)
    K = np.array([[30.1, 0, 20.3], [0, 29.7, 6.2], [0, 0, 1]], dtype=np.float32)
    a = okd.project_loop(sc["xyz"], Pc, K, 13, 41)
    b = okd.project_rule(sc["xyz"], Pc, K, 13, 41)
    assert a[2].sum() > 100
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def _masks():
    rng = np.random.default_rng(7)
    out = {"sparse": rng.random((37, 53)) < 0.02, "dense": rng.random((37, 53)) < 0.6,
           "single": np.zeros((20, 31), bool), "full": np.ones((9, 12), bool), "empty": np.zeros((11, 17), bool),
           "one_row": np.zeros((1, 40), bool), "one_column": np.zeros((25, 1), bool)}
    out["single"][13, 4] = True
    out["one_row"][0, [3, 17, 18, 30]] = True
    out["one_column"][[0, 12, 24], 0] = True
    lines = np.zeros((60, 90), bool)                  # scan-line-like: sparse rows of points, many ties
    for r in range(30, 60, 3):
        lines[r, rng.integers(0, 90, 25)] = True
    out["lines"] = lines
    return out


@pytest.mark.parametrize("name", sorted(_masks()))
def test_edt_matches_scipy(name):
    filled = _masks()[name]
    val, idx = okd.edt(~filled)
    sval, sidx = _scipy_edt(~filled)
    assert np.array_equal(idx, sidx)
    assert np.array_equal(val, sval)


def test_depth_map_of_an_empty_image_reads_the_bottom_left_pixel():
    p = np.array([[-1.0, -2.0], [0.0, 0.5], [0.0, 0.1]], dtype=np.float32)     # behind the camera
    m = okd.depth_map(p, np.eye(4), np.eye(3, dtype=np.float32), 4, 6)
    r, c = np.mgrid[0:4, 0:6]
    assert np.array_equal(m[0], np.zeros((4, 6), np.float32))
    assert np.array_equal(m[1], np.sqrt(((r + 1) ** 2 + c ** 2).astype(np.float64)).astype(np.float32))


def test_host_plan(tmp_path):
    root, vel = str(tmp_path / "kitti"), str(tmp_path / "vel")
    scans = [np.zeros((4, 5), np.float32)] * 3
    syn.write_kitti_velodyne_root(root, vel, 7, scans, [(13, 41), ((12, 40), (11, 40)), (13, 41)], K=(16, 16, 20, 6))
    plan = kitti_depth.plan_sequence(root, vel, 7)
    assert plan["n"] == 3 == kitti_depth.sample_num(vel, 7)
    assert plan["sizes"]["P2"] == [(13, 41), (12, 40), (13, 41)]
    assert plan["sizes"]["P3"] == [(13, 41), (11, 40), (13, 41)]
    calib = kitti.read_calib(root, 7)
    assert np.array_equal(plan["Pc"]["P2"], np.dot(calib["P2"], calib["Tr"]))
    assert np.array_equal(plan["K"]["P3"], calib["P3_K"])
    assert kitti_depth.record_dir(root, 7, "P3") == os.path.join(root, "data_odometry_velodyne_P3_npy", "sequences",
                                                                 "07", "voxel0.1-SNr0.6")
    assert kitti_depth.depth_dir(root, 7, "P2") == os.path.join(root, "data_odometry_color_depth_npy", "sequences",
                                                                "07", "image_2")
    assert kitti_depth.velodyne_path(vel, 7, 2) == os.path.join(vel, "sequences", "07", "velodyne", "000002.bin")
    runs = kitti_depth._size_runs(plan, [0, 1, 2])
    assert runs == [([0], ("P2", "P3"), (13, 41)), ([1], ("P2",), (12, 40)), ([1], ("P3",), (11, 40)),
                    ([2], ("P2", "P3"), (13, 41))]
    # sample_num counts every entry of the velodyne folder, as os.listdir does
    open(os.path.join(kitti_depth.velodyne_dir(vel, 7), "notes.txt"), "w").close()
    assert kitti_depth.sample_num(vel, 7) == 4


def test_image_size_from_npy_header_and_png(tmp_path):
    a = tmp_path / "a.npy"
    np.save(a, np.zeros((17, 23, 3), np.uint8))
    assert kitti_depth.image_size(str(a)) == (17, 23)
    b = tmp_path / "b.png"
    b.write_bytes(syn.encode_png(np.zeros((9, 31), np.uint8)))
    assert kitti_depth.image_size(str(b)) == (9, 31)
    c = tmp_path / "c.png"
    c.write_bytes(b"not a png at all, not at all")
    with pytest.raises(ValueError):
        kitti_depth.image_size(str(c))
    with pytest.raises(FileNotFoundError):
        kitti_depth.image_size(str(tmp_path / "missing.npy"))


def test_png_only_root_reads_png_sizes(tmp_path):
    root, vel = str(tmp_path / "kitti"), str(tmp_path / "vel")
    syn.write_kitti_velodyne_root(root, vel, 0, [np.zeros((4, 3), np.float32)] * 2, [(5, 9), (6, 10)], images="png")
    assert kitti_depth.plan_sequence(root, vel, 0)["sizes"]["P3"] == [(5, 9), (6, 10)]


def test_read_scan_rejects_a_truncated_file(tmp_path):
    p = tmp_path / "000000.bin"
    p.write_bytes(np.zeros(7, np.float32).tobytes())
    with pytest.raises(ValueError, match="whole number"):
        kitti_depth.read_scan(str(p))


def test_golden_regenerates_bit_for_bit(tmp_path):
    mk = _golden_module()
    out = tmp_path / "kd.npz"
    mk.make(str(out))
    with np.load(out) as a, np.load(os.path.join(ROOT, "tests", "golden", "kitti_depth_small.npz")) as b:
        assert sorted(a.files) == sorted(b.files)
        for k in a.files:
            assert np.array_equal(a[k], b[k]), k


def test_golden_covers_its_cases():
    mk = _golden_module()
    with np.load(os.path.join(ROOT, "tests", "golden", "kitti_depth_small.npz")) as z:
        records, maps = mk.unpack(z)
    H, W = mk.HW
    for k in ("P2", "P3"):
        assert maps[(3, k)][0].max() == 0            # no point lands: every depth is img_depth[-1, 0] = 0
        assert maps[(4, k)].shape == (2, 12, 40)
    m = maps[(2, "P2")]
    filled = m[1] < 0.75
    for r, c in ((0, 0), (H - 1, W - 1), (6, 0), (6, W - 1), (0, 20), (H - 1, 20)):   # the planted halves
        assert filled[r, c], (r, c)
    assert records[(0, "P2")].shape[0] == 7
