"""The scan-preparation oracle (oracle_prep) against independent numpy / scipy restatements, the synthetic scans, the
Python-side validation of deepi2p_b200.pointprep and the .bin reader.  No GPU needed."""
import os
import struct

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

import oracle_prep
from deepi2p_b200 import pointprep, synthetic

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pointprep_small.npz")


def _voxel_numpy(xyz, v, attr=None):
    """np.unique grouping of floor((p - min_bound) / v), sequential sums in ascending point index."""
    p = xyz.astype(np.float64)
    mb = p.min(1, keepdims=True) - 0.5 * v
    key = np.floor((p - mb) / v).astype(np.int64).T
    uniq, inv = np.unique(key, axis=0, return_inverse=True)
    inv = inv.reshape(-1)
    rows = p if attr is None else np.concatenate([p, attr])
    out = np.zeros((rows.shape[0], len(uniq)))
    cnt = np.zeros(len(uniq))
    for j in range(p.shape[1]):              # sequential, ascending index
        out[:, inv[j]] += rows[:, j]
        cnt[inv[j]] += 1
    return out / cnt


@pytest.mark.parametrize("v", [0.1, 0.3, 0.25])
def test_voxel_against_numpy(v):
    sc = synthetic.make_lidar_scan(3, n_rings=16, n_azimuth=512)
    attr = np.random.default_rng(1).standard_normal((2, sc["xyz"].shape[1]))
    rx, ra = oracle_prep.voxel_downsample(sc["xyz"], v, attr)
    ref = _voxel_numpy(sc["xyz"], v, attr)
    assert np.array_equal(rx, ref[:3]) and np.array_equal(ra, ref[3:])


def test_voxel_limit():
    c = np.array([[0.0, 3000.0], [0.0, 0.0], [0.0, 0.0]], np.float32)
    with pytest.raises(ValueError):
        oracle_prep.voxel_downsample(c, 1e-3)
    assert oracle_prep.voxel_downsample(c, 2e-3)[0].shape == (3, 2)


def _neighbours_numpy(xyz, r, max_nn):
    p = xyz.astype(np.float64).T
    tree = cKDTree(p)
    out = []
    for i, cand in enumerate(tree.query_ball_point(p, r * (1 + 1e-9))):
        cand = np.array(sorted(cand), dtype=np.int64)
        d = p[i] - p[cand]
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        keep = d2 < r * r
        cand, d2 = cand[keep], d2[keep]
        order = np.lexsort((cand, d2))
        out.append(cand[order][:max_nn])
    return out


@pytest.mark.parametrize("max_nn", [1, 7, 30, 64])
def test_neighbours_against_ckdtree(max_nn):
    sc = synthetic.make_lidar_scan(4, n_rings=16, n_azimuth=512)
    down = oracle_prep.voxel_downsample(sc["xyz"], 0.2)[0].astype(np.float32)
    g = np.arange(5, dtype=np.float32)                      # plus a lattice with equidistant shells
    lat = np.stack(np.meshgrid(g, g, g, indexing="ij")).reshape(3, -1) + np.float32(100)
    cloud = np.concatenate([down, lat], 1)
    _, cnt, nbr = oracle_prep.estimate_normals(cloud, 1.8, max_nn, neighbours=True)
    ref = _neighbours_numpy(cloud, 1.8, max_nn)
    for i, r in enumerate(ref):
        assert cnt[i] == len(r) and np.array_equal(nbr[i, :cnt[i]], r), i


def test_normals_against_eigh():
    sc = synthetic.make_lidar_scan(5, n_rings=32, n_azimuth=1024)
    down = oracle_prep.voxel_downsample(sc["xyz"], 0.1)[0].astype(np.float32)
    nrm, cnt, nbr = oracle_prep.estimate_normals(down, 0.6, 30, neighbours=True)
    p = down.astype(np.float64)
    checked = 0
    for i in range(0, p.shape[1], 7):
        if cnt[i] < 3:
            assert np.array_equal(nrm[:, i], [0.0, 0.0, 1.0])
            continue
        d = p[:, nbr[i, :cnt[i]]] - p[:, i:i + 1]
        C = d @ d.T / cnt[i] - np.outer(d.mean(1), d.mean(1))
        w, V = np.linalg.eigh(C)
        if w[1] - w[0] < 1e-3 * max(w[2], 1e-300):
            continue                                           # nearly degenerate: the eigenvector is ill-posed
        e = V[:, 0] * (1.0 if V[2, 0] >= 0 else -1.0)
        if e[2] == 0:
            continue
        ang = float(np.linalg.norm(np.cross(e, nrm[:, i])))      # sin of the angle, exact near 0
        assert ang < 1e-9 and nrm[2, i] >= 0, (i, ang)
        checked += 1
    assert checked > 1000


def test_noise_free_ground_normals():
    sc = synthetic.make_lidar_scan(6, noise=0.0)
    g = sc["xyz"][:, sc["ground"]]
    far = np.hypot(g[0], g[1]) > 3.0
    nrm, cnt = oracle_prep.estimate_normals(g[:, far][:, ::5].copy(), 0.6, 30)
    ok = cnt >= 3
    assert ok.mean() > 0.9
    assert np.abs(nrm[:, ok] - np.array([[0.0], [0.0], [1.0]])).max() < 1e-9


def test_lidar_scan_shape():
    a, b = synthetic.make_lidar_scan(0), synthetic.make_lidar_scan(0)
    assert a["xyz"].shape == (3, 131072) and a["xyz"].dtype == np.float32
    assert a["intensity"].dtype == np.float32 and 0 <= a["intensity"].min() and a["intensity"].max() < 1
    assert np.array_equal(a["xyz"], b["xyz"]) and np.array_equal(a["intensity"], b["intensity"])


def test_golden_oracle():
    import importlib.util
    spec = importlib.util.spec_from_file_location(
        "mk", os.path.join(os.path.dirname(GOLDEN), "make_pointprep_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    g = np.load(GOLDEN)
    for k, v in mk.compute().items():
        assert np.array_equal(g[k], v), k


def test_python_rejects_bad_arguments():
    xyz = torch.zeros((1, 3, 16))
    for v in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError):
            pointprep.voxel_downsample(xyz, None, v)
        with pytest.raises(ValueError):
            pointprep.estimate_normals(xyz, None, radius=v)
        with pytest.raises(ValueError):
            pointprep.downsample_with_reflectance(np.zeros((3, 4)), np.ones(4), v)
    for k in (0, 65, 2.5):
        with pytest.raises(ValueError):
            pointprep.estimate_normals(xyz, None, max_nn=k)
        with pytest.raises(ValueError):
            pointprep.prepare_scans(xyz, None, None, sn_max_nn=k)
    with pytest.raises(ValueError):
        pointprep.estimate_normals(xyz, None, orient=(0.0, float("nan"), 1.0))
    bad = np.zeros((3, 4))
    bad[1, 2] = np.nan
    with pytest.raises(ValueError):
        pointprep.downsample_with_intensity_sn(bad, np.ones((1, 4)), np.zeros((3, 4)), 0.1)
    bad[1, 2] = np.inf
    with pytest.raises(ValueError):
        pointprep.downsample_with_reflectance(bad, np.ones(4), 0.1)


def test_read_velodyne_bin(tmp_path):
    rng = np.random.default_rng(2)
    data = rng.standard_normal((1000, 4)).astype(np.float32)
    path = str(tmp_path / "000000.bin")
    with open(path, "wb") as f:
        for row in data:
            f.write(struct.pack("<ffff", *row))
    # the reference's reader (kitti_pc_bin_to_npy_with_downsample_sn.py:18-29), restated
    with open(path, "rb") as f:
        ref = np.asarray([list(p) for p in struct.iter_unpack("ffff", f.read())], dtype=np.float32).T
    got = pointprep.read_velodyne_bin(path)
    assert got.dtype == np.float32 and got.shape == (4, 1000) and np.array_equal(got, ref)
