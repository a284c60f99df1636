"""The nuScenes records, poses and sweep walk without the devkit (deepi2p_b200.nuscenes), the oracle's ego-box mask
and fp64 accumulation (oracle_nuscenes), and the host checks of the nuScenes keywords.  Every fixture is written by
the tests from seeds."""
import ctypes
import math

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import oracle_nuscenes as onu
from deepi2p_b200 import assemble, imageprep, nuscenes, synthetic


def _tables(tmp_path, chains, sweeps=False, **kw):
    items = synthetic.write_nuscenes_dataroot(str(tmp_path), chains, sweeps=sweeps, **kw)
    return nuscenes.Tables(str(tmp_path), "v1.0-mini"), items


@pytest.mark.parametrize("links", [0, 1, 2, 3, 4, 5, 7, 8, 11, 12, 13, 20])
def test_sweep_walk_offsets_and_scene_ends(tmp_path, links):
    """Offsets 4, 8, 12 along next, then along prev; a direction stops at its first empty link, so `links` sweeps on
    one side give the multiples of 4 up to min(links, 12)."""
    tab, _ = _tables(tmp_path, [(2 * links + 1, links), (links + 1, 0), (links + 1, links)])
    want = [4 * k for k in (1, 2, 3) if 4 * k <= links]
    walk = nuscenes.sweep_walk(tab, f"lidar-0-{links}")
    assert [o for _, o in walk] == [0] + want + [-o for o in want]
    assert [sd["token"] for sd, _ in walk] == [f"lidar-0-{links + o}" for _, o in walk]
    assert [o for _, o in nuscenes.sweep_walk(tab, "lidar-1-0")] == [0] + want       # nothing before the scene start
    assert [o for _, o in nuscenes.sweep_walk(tab, f"lidar-2-{links}")] == [0] + [-o for o in want]


def test_tables_and_dataset_info(tmp_path):
    tab, items = _tables(tmp_path, [(5, 2), (3, 0)])
    assert nuscenes.load_dataset_info(str(tmp_path / "dataset_info.list")) == items
    assert [it[0] for it in items] == ["lidar-0-2", "lidar-1-0"]
    assert set(items[0][1]) == set(nuscenes.CAMERAS)
    sd = tab.get("sample_data", "lidar-0-2")
    assert sd["next"] == "lidar-0-3" and sd["prev"] == "lidar-0-1"
    assert tab.get("ego_pose", sd["ego_pose_token"])["token"] == "ego-0-2"
    cam = tab.get("sample_data", items[0][1]["CAM_BACK"][0])
    assert nuscenes.camera_K(tab, cam).dtype == np.float32 and nuscenes.camera_K(tab, cam).shape == (3, 3)
    with pytest.raises(KeyError):
        tab.get("sample_data", "nope")
    with pytest.raises(ValueError):
        tab.get("sample", "lidar-0-2")


def _f32_ulps(a, b):
    a32, b32 = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.abs(a32.view(np.int32).astype(np.int64) - b32.view(np.int32).astype(np.int64))


def test_rotation_matrix_against_scipy():
    rng = np.random.default_rng(3)
    q = rng.normal(size=(500, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    for w in q:
        R = nuscenes.rotation_matrix(w)
        ref = Rotation.from_quat([w[1], w[2], w[3], w[0]]).as_matrix()
        assert ((_f32_ulps(R, ref) <= 1) | (np.abs(R - ref) < 1e-15)).all()      # 1e-15: entries near 0
    assert np.array_equal(nuscenes.rotation_matrix([1, 0, 0, 0]), np.eye(3))
    for axis in range(3):                                           # half-turns about x, y, z are exact
        w = np.zeros(4)
        w[1 + axis] = 1.0
        want = -np.eye(3)
        want[axis, axis] = 1.0
        assert np.array_equal(nuscenes.rotation_matrix(w), want)
    w = np.array([0.9, 0.1, -0.2, 0.3])
    assert np.allclose(nuscenes.rotation_matrix(3.0 * w), nuscenes.rotation_matrix(w / np.linalg.norm(w)),
                       atol=1e-15)
    R = nuscenes.rotation_matrix(3.0 * w)
    assert np.allclose(R @ R.T, np.eye(3), atol=1e-14)
    for bad in ([0, 0, 0, 0], [1, 0, 0], [np.nan, 0, 0, 1]):
        with pytest.raises(ValueError):
            nuscenes.rotation_matrix(bad)


def _loader_P(rec):
    """get_P_from_Rt(Quaternion(rotation).rotation_matrix.astype(f32), translation.astype(f32)), written out."""
    a, b, c, d = np.asarray(rec["rotation"], dtype=np.float64) / np.linalg.norm(rec["rotation"])
    R = np.array([[a * a + b * b - c * c - d * d, 2 * (b * c - a * d), 2 * (b * d + a * c)],
                  [2 * (b * c + a * d), a * a - b * b + c * c - d * d, 2 * (c * d - a * b)],
                  [2 * (b * d - a * c), 2 * (c * d + a * b), a * a - b * b - c * c + d * d]])
    P = np.identity(4)
    P[:3, :3] = R.astype(np.float32)
    P[:3, 3] = np.asarray(rec["translation"]).astype(np.float32)
    return P


def test_pose_chain_equals_the_loaders_composition(tmp_path):
    tab, items = _tables(tmp_path, [(30, 14)], seed=5)
    walk = nuscenes.sweep_walk(tab, items[0][0])
    assert len(walk) == 7
    anchor = walk[0][0]
    pose = lambda sd: nuscenes.ego_pose_P(tab, sd)
    calib = lambda sd: nuscenes.calibration_P(tab, sd)
    for sd in (w[0] for w in walk):
        P = pose(sd)
        ref = _loader_P(tab.get("ego_pose", sd["ego_pose_token"]))
        assert np.array_equal(P[3], [0, 0, 0, 1]) and np.array_equal(P[:3, 3], ref[:3, 3])
        assert _f32_ulps(P[:3, :3], ref[:3, :3]).max() <= 1
        assert np.array_equal(P[:3, :3].astype(np.float32).astype(np.float64), P[:3, :3])
    # data/nuscenes_pc_img_pose_loader.py:242-267: P_io = inv(P_oi), P_ij_trans = (P_lv (P_io P_oj)) P_vl
    P_io = np.linalg.inv(pose(anchor))
    P_vl = calib(anchor)
    P_lv = np.linalg.inv(P_vl)
    FT = nuscenes.sweep_transforms(tab, walk)
    assert np.array_equal(FT[0], np.eye(4))
    for t, (sd, _) in enumerate(walk[1:], 1):
        assert np.array_equal(FT[t], np.dot(np.dot(P_lv, np.dot(P_io, pose(sd))), P_vl))
    # :351-356: P_cam_pc = inv(cam_calib) (inv(cam_pose) (lidar_pose lidar_calib)), t_ij = P_cam_pc[:3, 3]
    cam = tab.get("sample_data", items[0][1]["CAM_FRONT_LEFT"][0])
    P_cam_pc, t_ij = nuscenes.pose_chain(tab, anchor, cam)
    ref = np.dot(np.linalg.inv(calib(cam)), np.dot(np.linalg.inv(pose(cam)), np.dot(pose(anchor), calib(anchor))))
    assert np.array_equal(P_cam_pc, ref) and np.array_equal(t_ij, ref[:3, 3])


def test_read_sweep(tmp_path):
    r = synthetic.make_nuscenes_sweep(4, n_rings=4, n_azimuth=64)
    r.tofile(str(tmp_path / "s.pcd.bin"))
    got = nuscenes.read_sweep(str(tmp_path / "s.pcd.bin"))
    assert got.dtype == np.float32 and np.array_equal(got, r[:, :4])


def test_oracle_mask_equals_the_loaders():
    f32 = np.float32
    edge = np.array([-0.8, 0.8, -2.7, 2.7], dtype=f32)
    vals_x = np.concatenate([edge[:2], np.nextafter(edge[:2], f32(0)), np.nextafter(edge[:2], f32(10) * edge[:2]),
                             np.array([0.0, 0.5, -1.5], f32)])
    vals_y = np.concatenate([edge[2:], np.nextafter(edge[2:], f32(0)), np.nextafter(edge[2:], f32(10) * edge[2:]),
                             np.array([0.0, 2.0, 3.5], f32)])
    X, Y = np.meshgrid(vals_x, vals_y)
    pts = np.stack([X.ravel(), Y.ravel(), np.zeros(X.size, f32)]).astype(f32)
    pts = np.concatenate([pts, synthetic.make_nuscenes_sweep(1, n_rings=4, n_azimuth=256)[:, :3].T], 1)
    # data/nuscenes_pc_img_pose_loader.py:200-206, float32 arrays against Python floats
    x_inside = np.logical_and(pts[0, :] < 0.8, pts[0, :] > -0.8)
    y_inside = np.logical_and(pts[1, :] < 2.7, pts[1, :] > -2.7)
    want = np.logical_not(np.logical_and(x_inside, y_inside))
    keep = onu.ego_mask(pts)
    assert np.array_equal(keep, want)
    assert 0 < (~keep).sum() < keep.size
    on_edge = np.isin(pts[0], edge[:2]) | np.isin(pts[1], edge[2:])
    assert keep[on_edge].all()                                    # strict compares keep the box's edges


def test_oracle_accumulation_within_two_ulps_of_np_dot(tmp_path):
    smp = synthetic.make_nuscenes_sample(2, n_sweeps=4, n_rings=8, n_azimuth=256)
    x, it = onu.accumulate(smp["frames"], smp["frame_T"])
    assert x.dtype == np.float64 and it.dtype == np.float32
    xs, mags = [], []
    for (p, _, _), M in zip(smp["frames"], smp["frame_T"]):
        p = p[:, onu.ego_mask(p)]
        hom = np.concatenate([p, np.ones((1, p.shape[1]), dtype=p.dtype)], 0)
        xs.append(np.dot(M, hom)[:3])                             # transform_pc_np
        mags.append(np.dot(np.abs(M), np.abs(hom.astype(np.float64)))[:3])
    ref = np.concatenate(xs, 1)
    assert ref.shape == x.shape
    # ulps of the sum of the terms' magnitudes: the two differ only in the order the four products are added
    assert (np.abs(x - ref) <= 2 * np.spacing(np.concatenate(mags, 1))).all()
    n0 = int(onu.ego_mask(smp["frames"][0][0]).sum())
    assert np.array_equal(x[:, :n0], ref[:, :n0])                 # the anchor is not moved


def test_oracle_voxel_grid_on_float32_clouds_equals_oracle_prep():
    import oracle_prep
    p = synthetic.make_nuscenes_sweep(6, n_rings=16, n_azimuth=512)
    xyz, refl = p[:, :3].T, p[:, 3]
    attr = (refl / refl.max()).astype(np.float64)[None]
    a, A = onu.voxel_downsample64(xyz.astype(np.float64), 0.2, attr)
    b, B = oracle_prep.voxel_downsample(xyz, 0.2, attr)
    assert np.array_equal(a, b) and np.array_equal(A, B)


def test_presets():
    P = np.eye(4)
    a = assemble.nuscenes_args(P)
    assert a["voxel_size"] == 0.2 and a["range_max"] is None and a["flip"] is False and a["accumulate_f64"] is True
    assert a["exclude_box"] == (-0.8, 0.8, -2.7, 2.7) and a["jitter"] == ("pc", "intensity")
    assert a["amplitudes"] == a["val_amplitudes"] == (0.0, 0.0, 0.0, 0.0, 0.0, 2.0 * math.pi)
    assert np.array_equal(a["pre"], np.eye(4))
    assert imageprep.nuscenes_image_args() == dict(img_H=160, img_W=320, img_scale=0.2, crop_top_rows=100,
                                                   crop_bottom_rows=0, jitter_prob=0.5)
    for mode in ("train", "val_random_Ry"):
        Pr, flip = assemble.random_transforms(64, mode, a["amplitudes"], rng=1, flip=False,
                                              val_amplitudes=a["val_amplitudes"])
        assert not flip.any()
        assert np.array_equal(Pr[:, 2], np.tile([0.0, 0.0, 1.0, 0.0], (64, 1)))        # a rotation about z
        assert np.array_equal(Pr[:, :3, 3], np.zeros((64, 3)))
        ang = np.arctan2(Pr[:, 1, 0], Pr[:, 0, 0])
        assert np.ptp(ang) > 3.0
    # without val_amplitudes, val_random_Ry keeps its rotation about y
    Pr, _ = assemble.random_transforms(8, "val_random_Ry", rng=0)
    assert np.allclose(Pr[:, 1], [0, 1, 0, 0])


def test_bad_arguments(tmp_path):
    with pytest.raises(ValueError):
        assemble.random_transforms(3, "val_random_Ry", val_amplitudes=(0, 0, 0))
    with pytest.raises(ValueError):
        assemble.random_transforms(3, "val_random_Ry", val_amplitudes=(0, 0, 0, 0, 0, np.inf))
    for kw in (dict(exclude_box=(0.8, -0.8, -2.7, 2.7), accumulate_f64=True),
               dict(exclude_box=(0, 1, 2), accumulate_f64=True),
               dict(exclude_box=(-0.8, 0.8, -2.7, np.nan), accumulate_f64=True),
               dict(exclude_box=(-0.8, 0.8, -2.7, 2.7)),                       # the box needs the fp64 path
               dict(accumulate_f64="yes"),
               dict(val_amplitudes=(1, 2))):
        with pytest.raises(ValueError):
            assemble.assemble_batch({}, "train", 0, **kw)
    with pytest.raises(ValueError):
        nuscenes.sweep_walk(None, "x", frame_skip=0)
    tab, items = _tables(tmp_path, [(3, 1)])
    with pytest.raises(ValueError):
        nuscenes.nuscenes_batch(tab, items, "bogus", 0)
    with pytest.raises(ValueError):
        nuscenes.nuscenes_batch(tab, [], "train", 0)
    from deepi2p_b200 import _native
    lib = _native.load()
    buf = ctypes.create_string_buffer(1024)
    a = ctypes.addressof(buf)
    ws = lib.assemble_accumulate_f64_workspace_bytes(1, 16, 1)
    assert ws == lib.assemble_accumulate_workspace_bytes(1, 16, 1) > 0
    box = (ctypes.c_float * 4)(0.8, -0.8, -2.7, 2.7)
    assert lib.assemble_accumulate_f64(a, a, None, 16, 1, a, a, 1, 0.0, ctypes.addressof(box), a, a, 16, a, a, ws,
                                       None) == -22
    assert b"exclude_box" in lib.dib_last_error()
    assert lib.assemble_accumulate_f64(a, a, None, 16, 1, a, a, 1, 0.0, None, None, a, 16, a, a, ws, None) == -22
    assert lib.assemble_accumulate_f64(a, a, None, 16, 1, a, a, 1, 0.0, None, a, a, 16, a, a, 16, None) == -22
    assert b"workspace" in lib.dib_last_error()
    assert lib.voxel_downsample_batch_f64(a, None, 17, 1, None, 0, 0.2, a, None, a, a, 1024, None) == -22
