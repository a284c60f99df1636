"""Scan preparation on the GPU (deepi2p_b200.pointprep) against the CPU oracle (oracle_prep) and the stored golden
results.

The oracle restates the kernels' arithmetic (no FMA, the same summation orders, the same Jacobi eigensolver) and
finds the same neighbour sets with a different search (a uniform grid, and oracle_icp's k-d tree for the nearest
point), so voxel counts, coordinates, attributes, normals, neighbour counts and nearest indices must be
bit-identical."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import oracle_prep
from deepi2p_b200 import pointprep, synthetic
from deepi2p_b200.icp import pack_clouds

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "pointprep_small.npz")


def _pad(rows, N, dtype=np.float64):
    a = np.zeros((len(rows), rows[0].shape[0] if rows else 0, N), dtype=dtype)
    for s, r in enumerate(rows):
        a[s, :, :r.shape[1]] = r
    return a


def _check_voxel(clouds, v, attrs=None, stream=None):
    xyz, n = pack_clouds(clouds)
    A = None if attrs is None else torch.from_numpy(_pad(attrs, xyz.shape[2])).cuda()
    out = pointprep.voxel_downsample(xyz, n, v, attr=A, stream=stream)
    torch.cuda.synchronize()
    m = out["m_pts"].cpu().numpy()
    for s, c in enumerate(clouds):
        rx, ra = oracle_prep.voxel_downsample(c, v, None if attrs is None else attrs[s])
        assert m[s] == rx.shape[1], s
        assert np.array_equal(out["xyz"][s, :, :m[s]].cpu().numpy(), rx), s
        assert not out["xyz"][s, :, m[s]:].any()
        if attrs is not None:
            assert np.array_equal(out["attr"][s, :, :m[s]].cpu().numpy(), ra), s
    return out


def _check_normals(clouds, r, max_nn, orient=(0.0, 0.0, 1.0), stream=None):
    xyz, m = pack_clouds(clouds)
    nrm, cnt = pointprep.estimate_normals(xyz, m, r, max_nn, orient, counts=True, stream=stream)
    torch.cuda.synchronize()
    for s, c in enumerate(clouds):
        rn, rc = oracle_prep.estimate_normals(c, r, max_nn, orient)
        k = c.shape[1]
        assert np.array_equal(cnt[s, :k].cpu().numpy(), rc), s
        assert np.array_equal(nrm[s, :, :k].cpu().numpy(), rn), s
    return nrm, cnt


def _check_nearest(clouds, queries):
    xyz, m = pack_clouds(clouds)
    Q = max(16, -(-max(q.shape[1] for q in queries) // 16) * 16)
    q = torch.from_numpy(_pad(queries, Q)).cuda()
    qn = torch.tensor([x.shape[1] for x in queries], dtype=torch.int32, device="cuda")
    idx = pointprep.nearest(q, qn, xyz, m).cpu().numpy()
    for s, c in enumerate(clouds):
        k = queries[s].shape[1]
        assert np.array_equal(idx[s, :k], oracle_prep.nearest(c, queries[s])), s
        assert (idx[s, k:] == -1).all()


def test_full_scans_at_kitti_parameters():
    scans = [synthetic.make_lidar_scan(s) for s in (1, 2)]
    downs = [oracle_prep.voxel_downsample(sc["xyz"], 0.1)[0] for sc in scans]
    _check_voxel([sc["xyz"] for sc in scans], 0.1)
    nrm, cnt = _check_normals([d.astype(np.float32) for d in downs], 0.6, 30)
    assert 10 < float(cnt.sum()) / sum(d.shape[1] for d in downs) <= 30
    _check_nearest([sc["xyz"] for sc in scans], downs)
    xyz, n = pack_clouds([sc["xyz"] for sc in scans])
    inten = torch.from_numpy(np.stack([sc["intensity"] for sc in scans])).cuda()
    rec, m = pointprep.prepare_scans(xyz, inten, n)
    rec, m = rec.cpu().numpy(), m.cpu().numpy()
    for s, sc in enumerate(scans):
        ref = oracle_prep.prepare_scan(sc["xyz"], sc["intensity"])
        assert m[s] == ref.shape[1]
        assert np.array_equal(rec[s, :, :m[s]], ref), s
        assert not rec[s, :, m[s]:].any()


def test_ragged_batch_with_attributes():
    scans = [synthetic.make_lidar_scan(10 + s, n_rings=16, n_azimuth=256 + 64 * s)["xyz"][:, :3000 + 777 * s]
             for s in range(3)]
    rng = np.random.default_rng(5)
    attrs = [rng.standard_normal((4, c.shape[1])) for c in scans]
    _check_voxel(scans, 0.3, attrs)
    _check_voxel(scans[:1] + [np.zeros((3, 0), np.float32)] + scans[2:], 0.3)       # an empty cloud in the middle
    _check_normals(scans, 0.9, 20)
    _check_nearest(scans, [c[:, ::3].astype(np.float64) + 0.01 for c in scans])


def test_tiny_clouds():
    one = np.array([[1.5], [-2.0], [0.25]], np.float32)
    two = np.array([[0.0, 0.05], [0.0, 0.0], [0.0, -0.05]], np.float32)
    _check_voxel([one, two], 0.1, [np.ones((2, 1)), np.arange(4.0).reshape(2, 2)])
    nrm, cnt = _check_normals([one, two], 1.0, 30)
    assert (cnt[0, :1] == 1).all() and (cnt[1, :2] == 2).all()
    assert np.array_equal(nrm[:, :, 0].cpu().numpy(), [[0, 0, 1], [0, 0, 1]])       # fewer than 3 neighbours
    _check_nearest([one, two], [np.array([[9.0], [9.0], [9.0]]), np.array([[0.0], [0.0], [0.0]])])


def test_one_voxel_and_duplicates():
    rng = np.random.default_rng(3)
    blob = (rng.random((3, 500)) * 0.04).astype(np.float32)   # min_bound sits 0.05 below the minimum: one voxel
    dup = np.repeat(np.array([[1.0], [2.0], [3.0]], np.float32), 40, axis=1)
    dup[:, 20:] = np.array([[1.5], [2.0], [3.0]], np.float32)
    out = _check_voxel([blob, dup], 0.1, [rng.standard_normal((1, 500)), rng.standard_normal((1, 40))])
    assert out["m_pts"].cpu().tolist() == [1, 2]
    nrm, cnt = _check_normals([dup], 0.1, 30)              # zero covariance: the normal becomes the orientation
    assert np.array_equal(nrm[0, :, :40].cpu().numpy(), np.repeat([[0.0], [0.0], [1.0]], 40, axis=1))
    _check_normals([dup], 0.1, 30, orient=(0.0, 1.0, 0.0))
    _check_nearest([dup], [np.array([[1.0, 1.5, 1.25], [2.0, 2.0, 2.0], [3.0, 3.0, 3.0]])])   # ties -> lowest index


def test_voxel_boundaries():
    # v = 0.25 and integer-multiple coordinates: (p - min_bound) / v lands exactly on integers + 0.5 and the mins on
    # exact boundaries; negative and positive coordinates, and a point shared by 8 voxel corners.
    g = np.arange(-4, 5, dtype=np.float32) * 0.125
    x, y, z = np.meshgrid(g, g, g, indexing="ij")
    lat = np.stack([x.ravel(), y.ravel(), z.ravel()])
    _check_voxel([lat, lat[:, ::-1].copy()], 0.25, [np.arange(lat.shape[1], dtype=np.float64)[None]] * 2)
    _check_voxel([lat], 0.125)


@pytest.mark.parametrize("max_nn", [1, 3, 16, 30, 64])
def test_lattice_ties_at_the_cut(max_nn):
    # A unit lattice: every interior point has 6 neighbours at d2 = 1, 12 at 2, 8 at 3, 6 at 4 ... so the cut at
    # max_nn falls inside a shell of equal distances, decided by index.
    g = np.arange(7, dtype=np.float32)
    x, y, z = np.meshgrid(g, g, g, indexing="ij")
    lat = np.stack([x.ravel(), y.ravel(), z.ravel()]).astype(np.float32)
    perm = np.random.default_rng(max_nn).permutation(lat.shape[1])
    _, cnt = _check_normals([lat, lat[:, perm].copy()], 2.5, max_nn)
    assert int(cnt.max()) == max_nn


def test_drop_ins():
    rng = np.random.default_rng(11)
    sc = synthetic.make_lidar_scan(20, n_rings=32, n_azimuth=512)
    pc = sc["xyz"]
    inten = (sc["intensity"] * 255).astype(np.float32)[None]
    sn = rng.standard_normal((3, pc.shape[1])).astype(np.float32)
    p, i, n = pointprep.downsample_with_intensity_sn(pc, inten, sn, 0.3)
    imax = np.max(inten)
    attr = np.concatenate([(inten.T / imax).T.astype(np.float64), sn.astype(np.float64)])
    rx, ra = oracle_prep.voxel_downsample(pc, 0.3, attr)
    assert p.dtype == i.dtype == n.dtype == np.float64
    assert p.shape == (3, rx.shape[1]) and i.shape == (1, rx.shape[1]) and n.shape == (3, rx.shape[1])
    assert np.array_equal(p, rx) and np.array_equal(i, ra[0:1] * imax) and np.array_equal(n, ra[1:4])
    refl = sc["intensity"]
    p2, r2 = pointprep.downsample_with_reflectance(pc, refl, 0.2)
    rx, ra = oracle_prep.voxel_downsample(pc, 0.2, (refl / np.max(refl)).astype(np.float64)[None])
    assert r2.shape == (rx.shape[1],) and np.array_equal(p2, rx) and np.array_equal(r2, ra[0] * np.max(refl))


def test_prepare_scans_script(tmp_path):
    vel, out = tmp_path / "velodyne", tmp_path / "out"
    vel.mkdir()
    scans = [synthetic.make_lidar_scan(30 + s, n_rings=32, n_azimuth=1024 - 96 * s) for s in range(3)]
    for s, sc in enumerate(scans):
        np.concatenate([sc["xyz"], sc["intensity"][None]]).T.astype("<f4").tofile(str(vel / ("%06d.bin" % s)))
    subprocess.check_call([sys.executable, os.path.join(ROOT, "scripts", "prepare_scans.py"), str(vel), str(out),
                           "--batch", "2"])
    for s, sc in enumerate(scans):
        got = np.load(str(out / ("%06d.npy" % s)))
        ref = oracle_prep.prepare_scan(sc["xyz"], sc["intensity"])
        assert got.dtype == np.float32 and np.array_equal(got, ref), s


def test_second_stream():
    scans = [synthetic.make_lidar_scan(50 + s, n_rings=16, n_azimuth=512)["xyz"] for s in range(2)]
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        _check_voxel(scans, 0.2, stream=st)
        _check_normals(scans, 0.6, 30, stream=st)
    xyz, n = pack_clouds(scans)
    inten = torch.rand((2, xyz.shape[2]), device="cuda")
    a, ma = pointprep.prepare_scans(xyz, inten, n, stream=st)
    st.synchronize()
    b, mb = pointprep.prepare_scans(xyz, inten, n)
    torch.cuda.synchronize()
    assert torch.equal(ma, mb) and torch.equal(a, b)


def test_golden():
    g = np.load(GOLDEN)
    import importlib.util
    spec = importlib.util.spec_from_file_location("mk", os.path.join(ROOT, "tests", "golden", "make_pointprep_golden.py"))
    mk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mk)
    scans = mk.scans()
    xyz, n = pack_clouds([sc["xyz"] for sc in scans])
    out = pointprep.voxel_downsample(xyz, n, mk.VOXEL)
    m = out["m_pts"].cpu().numpy()
    downs = [out["xyz"][s, :, :m[s]].cpu().numpy() for s in range(2)]
    d32, dm = pack_clouds([d.astype(np.float32) for d in downs])
    nrm, cnt = pointprep.estimate_normals(d32, dm, mk.RADIUS, mk.MAX_NN, counts=True)
    q = torch.from_numpy(_pad(downs, d32.shape[2])).cuda()
    idx = pointprep.nearest(q, dm, xyz, n).cpu().numpy()
    for s in range(2):
        assert np.array_equal(downs[s], g[f"down{s}"])
        assert np.array_equal(nrm[s, :, :m[s]].cpu().numpy(), g[f"normals{s}"])
        assert np.array_equal(cnt[s, :m[s]].cpu().numpy(), g[f"count{s}"])
        assert np.array_equal(idx[s, :m[s]], g[f"nearest{s}"])


def test_voxel_limit_is_rejected_on_the_host():
    c = np.array([[0.0, 3000.0], [0.0, 0.0], [0.0, 0.0]], np.float32)
    xyz, n = pack_clouds([c])
    with pytest.raises(ValueError, match="2\\^21"):
        pointprep.voxel_downsample(xyz, n, 1e-3)           # 3e6 voxels along x
    out = pointprep.voxel_downsample(xyz, n, 2e-3)         # 1.5e6: admitted
    assert int(out["m_pts"][0]) == 2
