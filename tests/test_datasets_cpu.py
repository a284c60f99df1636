"""The KITTI and Oxford readers' host code (deepi2p_b200.kitti / deepi2p_b200.oxford) against oracle_datasets, the
loaders' host computation worked out independently in numpy: calibration, dataset lists, the accumulation walk and its
transforms, the image and camera pairing draws, the Oxford conjugation, the scan store's layout and a batch's record deduplication, and the
error messages.  No GPU is needed."""
import os

import numpy as np
import pytest

import oracle_datasets as od
from deepi2p_b200 import assemble, kitti, oxford, synthetic


@pytest.fixture(scope="module")
def kitti_root(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("kitti"))
    synthetic.write_kitti_root(root, seqs=(0, 9, 10), n_frames=90, n_images=2, image_hw=(8, 8))
    return root


@pytest.fixture(scope="module")
def oxford_root(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("oxford"))
    synthetic.write_oxford_root(root, n_images=2, image_hw=(16, 16))
    return root


CALIB = """P0: 7.188560000000e+02 0.000000000000e+00 6.071928000000e+02 0.000000000000e+00 0.000000000000e+00 7.188560000000e+02 1.852157000000e+02 0.000000000000e+00 0.000000000000e+00 0.000000000000e+00 1.000000000000e+00 0.000000000000e+00
P2: 7.188560000000e+02 0.000000000000e+00 6.071928000000e+02 4.538225000000e+01 0.000000000000e+00 7.188560000000e+02 1.852157000000e+02 -1.130887000000e-01 0.000000000000e+00 0.000000000000e+00 1.000000000000e+00 3.779761000000e-03
Tr: 4.276802385584e-04 -9.999672484946e-01 -8.084491683471e-03 -1.198459927713e-02 -7.210626507497e-03 8.081198471645e-03 -9.999413164504e-01 -5.403984729748e-02 9.999738645903e-01 4.859485810390e-04 -7.206933692422e-03 -2.921968648686e-01
"""


def test_calibration_parse_against_hand_computed_values():
    c = kitti.parse_calib(CALIB)
    f32 = np.float32
    fx, cx, fy, cy = f32(718.856), f32(607.1928), f32(718.856), f32(185.2157)
    tz = f32(3.779761e-03)
    tx = (f32(45.38225) - cx * tz) / fx          # float32 arithmetic, as KittiCalibHelper does it
    ty = (f32(-0.1130887) - cy * tz) / fy
    assert c["P2"].dtype == np.float64 and c["P2_K"].dtype == np.float32
    assert np.array_equal(c["P2"][:3, 3], np.array([tx, ty, tz], dtype=np.float64))
    assert np.array_equal(c["P2"][:3, :3], np.eye(3)) and np.array_equal(c["P2"][3], [0, 0, 0, 1])
    assert abs(float(tx) - 0.0599386) < 1e-6 and abs(float(ty) + 1.13117e-3) < 1e-7
    assert np.array_equal(c["P2_K"], np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], dtype=np.float32))
    assert np.array_equal(c["P0"], np.eye(4))
    tr = np.array([float(v) for v in CALIB.splitlines()[2][4:].split()], dtype=np.float32).reshape(3, 4)
    assert c["Tr"].shape == (4, 4) and np.array_equal(c["Tr"][:3], tr.astype(np.float64))
    assert np.array_equal(c["Tr"][3], [0, 0, 0, 1])
    assert np.array_equal(kitti.camera_Pc(c, "P2"), np.dot(c["P2"], c["Tr"]))


def test_calibration_matches_the_oracle(kitti_root):
    for seq in (0, 9, 10):
        got, ref = kitti.read_calib(kitti_root, seq), od.calibration(kitti_root, seq)
        assert set(got) == set(ref)
        for k in got:
            assert got[k].dtype == ref[k].dtype and np.array_equal(got[k], ref[k]), (seq, k)


def test_dataset_lists(kitti_root):
    ds = kitti.KittiDataset(kitti_root, "val_random_Ry")
    assert ds.entries == od.kitti_list(kitti_root, (9, 10))
    assert len(ds) == 2 * 2 * (90 - 80)
    assert {e[0] for e in ds.entries} == {9, 10}
    assert ds.entries[0] == (9, 40, 90, "P2") and ds.entries[1] == (9, 40, 90, "P3") and ds.entries[2][1] == 41
    assert max(e[1] for e in ds.entries) == 49
    tr = kitti.make_dataset(kitti_root, "train", seqs=(0,))
    assert tr == od.kitti_list(kitti_root, (0,))
    assert kitti.mode_seqs("train") == tuple(range(9)) and kitti.mode_seqs("val") == (9, 10)


@pytest.mark.parametrize("i,n", [(0, 100), (5, 100), (12, 100), (17, 100), (18, 100), (50, 100), (81, 100),
                                 (82, 100), (93, 100), (94, 100), (99, 100), (0, 1), (3, 7)])
def test_walk_at_both_sequence_ends(i, n):
    walk = kitti.accumulation_walk(i, n)
    prev = [i - 6 * c for c in (1, 2, 3) if i - 6 * c >= 0]
    nxt = [i + 6 * c for c in (1, 2, 3) if i + 6 * c < n]
    assert walk == [i] + prev + nxt


def test_walk_and_transforms_match_the_oracle(kitti_root):
    ds = kitti.KittiDataset(kitti_root, "train", seqs=(0,))
    ref_list = od.kitti_list(kitti_root, (0,))
    for it in (0, 1, 9, 19):
        seq, i, n, key = ds.entries[it]
        Pc = kitti.camera_Pc(ds.calib(seq), key)
        walk = kitti.accumulation_walk(i, n)
        FT = ds.frame_transforms(seq, walk, Pc)
        ref = od.kitti_expected(kitti_root, ref_list[it], np.random.default_rng(0), limit=-1)
        assert walk == ref["walk"]
        assert np.array_equal(Pc, ref["Pc"]) and np.array_equal(FT, ref["frame_T"])
    # the walk near a sequence end, on transforms too: i = 3 has no frame before it, i = 88 none after
    assert od.neighbours(88, 90) == kitti.accumulation_walk(88, 90)[1:] == [82, 76, 70]
    assert od.neighbours(3, 90) == kitti.accumulation_walk(3, 90)[1:] == [9, 15, 21]
    FT = ds.frame_transforms(0, kitti.accumulation_walk(3, 90), Pc)
    anchor = od.kitti_pose(kitti_root, 0, 3)
    ref = [od.frame_transform(Pc, anchor, od.kitti_pose(kitti_root, 0, j)) for j in (9, 15, 21)]
    assert np.array_equal(FT[1:], np.stack(ref))


@pytest.mark.parametrize("i", [40, 45, 49])
@pytest.mark.parametrize("tmax", [10.0, 2.5, 0.5])
def test_sequence_j_matches_the_oracle(kitti_root, i, tmax):
    ds = kitti.KittiDataset(kitti_root, "train", seqs=(0,))
    a, b = np.random.default_rng(i), np.random.default_rng(i)
    for _ in range(5):
        j, Pji, t = ds.sequence_j(a, 0, i, 90, 40, tmax)
        rj, rP = od.draw_pair(b, lambda k: od.kitti_pose(kitti_root, 0, k), i, 90, 40, tmax)
        assert j == rj and Pji.dtype == np.float32 and np.array_equal(Pji, rP) and np.array_equal(t, rP[:3, 3])
        assert np.linalg.norm(t) < tmax and abs(j - i) <= 40
    assert a.integers(1 << 30) == b.integers(1 << 30)       # both consumed the same draws


def test_sequence_j_window_edges_and_identity_branch(kitti_root):
    ds = kitti.KittiDataset(kitti_root, "train", seqs=(0,))
    rng = np.random.default_rng(3)
    js = {ds.sequence_j(rng, 0, 2, 90, 3, 1e9)[0] for _ in range(200)}
    assert js == set(range(0, 6))                             # clipped at 0, i + 3 inclusive
    js = {ds.sequence_j(rng, 0, 88, 90, 3, 1e9)[0] for _ in range(200)}
    assert js == set(range(85, 90))                           # clipped at n - 1
    j, P, t = ds.sequence_j(rng, 0, 44, 90, 40, -1.0)
    assert j == 44 and P.dtype == np.float64 and np.array_equal(P, np.identity(4)) and not t.any()
    before = rng.bit_generator.state
    ds.sequence_j(rng, 0, 44, 90, 40, -5.0)
    assert rng.bit_generator.state == before                 # the identity branch draws nothing
    with pytest.raises(ValueError, match="no frame j in \\[4, 84\\] lies within translation_max=0.0"):
        ds.sequence_j(rng, 0, 44, 90, 40, 0.0)


def test_oxford_conjugation_and_lists(oxford_root):
    entries, tables = od.oxford_tables(oxford_root, "val")
    ds = oxford.OxfordDataset(oxford_root, "val")
    assert ds.entries == entries
    for t, tr in ds.traversals.items():
        assert tr.pc_poses.dtype == np.float32 and np.array_equal(tr.pc_poses, tables[t]["pc_P"])
        assert np.array_equal(tr.camera_poses, tables[t]["cam_P"])
        assert tr.camera_timestamps == tables[t]["cam_ts"].tolist()
    raw = np.load(os.path.join(oxford_root, ds.entries[0][0], "pc_poses.npy"))[0]
    Pc = np.array([[0, 1, 0, 0], [0, 0, 1, 0], [1, 0, 0, 0], [0, 0, 0, 1]], dtype=np.float32)
    hand = Pc @ raw.astype(np.float32) @ Pc.T                 # P_convert is a permutation: exact
    assert np.array_equal(oxford.convert_poses(raw[None])[0], hand)
    assert oxford.read_split(oxford_root, "train") == ["2014-05-19-13-20-57", "2014-06-26-08-53-56"]


@pytest.mark.parametrize("mode", ["train", "val"])
def test_camera_timestamp_matches_the_oracle(oxford_root, mode):
    ds = oxford.OxfordDataset(oxford_root, mode)
    _, tables = od.oxford_tables(oxford_root, mode)
    a, b = np.random.default_rng(7), np.random.default_rng(7)
    for it in (0, 1, 11, 23, len(ds) - 1):
        t, _, i, n = ds.entries[it]
        for tm in (10.0, 3.0):
            c, P = oxford.camera_index(a, ds.traversals[t], i, tm)
            rc, rP = od.draw_camera(b, tables[t], i, tm)
            assert c == rc and P.dtype == np.float32 and np.array_equal(P, rP), (it, tm)
    assert a.integers(1 << 30) == b.integers(1 << 30)


def test_camera_window_edges(oxford_root):
    ds = oxford.OxfordDataset(oxford_root, "val")
    tr = next(iter(ds.traversals.values()))
    rng = np.random.default_rng(1)
    n = len(tr.pc_timestamps)
    # ceil(1e9 / 2e8) = 5 clouds either side (every camera within 1e9 m), bisect_left into the camera timestamps,
    # clipped at both ends of the traversal
    for i, lo_pc, hi_pc in ((0, 0, 5), (n - 1, n - 6, n - 1)):
        lo = np.searchsorted(tr.camera_timestamps, tr.pc_timestamps[lo_pc], "left")
        hi = np.searchsorted(tr.camera_timestamps, tr.pc_timestamps[hi_pc], "left")
        got = {oxford.camera_index(rng, tr, i, 1e9, pc_build_interval=2e8)[0] for _ in range(400)}
        assert got == set(range(lo, min(hi, len(tr.camera_timestamps) - 1) + 1)), i
    # 1.5 m -> ceil(1.5 / 2) = 1 cloud either side
    lo = np.searchsorted(tr.camera_timestamps, tr.pc_timestamps[9], "left")
    hi = np.searchsorted(tr.camera_timestamps, tr.pc_timestamps[11], "left")
    assert {oxford.camera_index(rng, tr, 10, 1.5)[0] for _ in range(200)} <= set(range(lo, hi + 1))
    with pytest.raises(ValueError, match="no camera frame in .* translation_max=0.0"):
        oxford.camera_index(rng, tr, 3, 0.0)


def test_store_layout_and_deduplication():
    rows, off, cnt = assemble.store_layout([(7, 5), (7, 0), (7, 3), (7, 2**20)])
    assert rows == 7 and off.dtype == np.int64 and cnt.dtype == np.int32
    assert off.tolist() == [0, 5, 5, 8] and cnt.tolist() == [5, 0, 3, 2**20]
    assert assemble.store_layout([(4, 1)])[0] == 4
    big = assemble.store_layout([(4, 2**31 - 1), (4, 2**31 - 1), (4, 7)])[1]
    assert big.tolist() == [0, 2**31 - 1, 2**32 - 2]          # offsets past 2^31 stay exact
    keys = [(0, 40), (0, 34), (0, 46), (0, 41), (0, 35), (0, 47), (0, 40), (0, 34)]
    uniq, ids = assemble.unique_records(keys)
    assert uniq == [(0, 40), (0, 34), (0, 46), (0, 41), (0, 35), (0, 47)]
    assert ids.tolist() == [0, 1, 2, 3, 4, 5, 0, 1] and [uniq[k] for k in ids] == keys


def test_batch_records_are_deduplicated(kitti_root):
    ds = kitti.KittiDataset(kitti_root, "train", seqs=(0,))
    plan = kitti.plan_batch(ds, [0, 1, 2, 3], "val", np.random.default_rng(0))
    keys = [(p["seq"], j) for p in plan for j in p["walk"]]
    uniq, ids = assemble.unique_records(keys)
    assert len(keys) == 28 and len(uniq) == 14                 # P2 / P3 of frames 40 and 41 share all 7 records


def test_error_messages(kitti_root, oxford_root, tmp_path):
    with pytest.raises(ValueError, match="every record must be \\[4, n\\]"):
        assemble.store_layout([(7, 3), (4, 3)])
    with pytest.raises(ValueError, match="at least one record"):
        assemble.store_layout([])
    with pytest.raises(ValueError, match="2\\^31 or more points"):
        assemble.store_layout([(4, 2**31)])
    with pytest.raises(ValueError, match="KITTI has train and val\\* modes"):
        kitti.make_dataset(kitti_root, "test")
    with pytest.raises(FileNotFoundError, match="KITTI image folder not found: .*sequences/01/image_2"):
        kitti.KittiDataset(kitti_root, "train")
    empty = tmp_path / "k" / "data_odometry_color_npy" / "sequences" / "03" / "image_2"
    empty.mkdir(parents=True)
    with pytest.raises(ValueError, match="KITTI sequence 03 is empty: no frame in .*03/image_2"):
        kitti.make_dataset(str(tmp_path / "k"), "train", seqs=(3,))
    short = tmp_path / "k" / "data_odometry_color_npy" / "sequences" / "04" / "image_2"
    short.mkdir(parents=True)
    (short / "000000.npy").write_bytes(b"")
    with pytest.raises(ValueError, match="the KITTI train list of .* is empty"):
        kitti.make_dataset(str(tmp_path / "k"), "train", seqs=(4,))
    with pytest.raises(FileNotFoundError, match="KITTI calibration not found: .*calib/05/calib.txt"):
        kitti.read_calib(kitti_root, 5)
    ds = kitti.KittiDataset(kitti_root, "train", seqs=(0,))
    with pytest.raises(FileNotFoundError, match="KITTI pose not found: .*poses/00/000090.npz"):
        ds.pose(0, 90)
    with pytest.raises(FileNotFoundError, match="KITTI scan record not found: .*voxel0.1-SNr0.6/000095.npy"):
        kitti.read_record(kitti.record_path(kitti_root, 0, 95))
    with pytest.raises(FileNotFoundError, match="KITTI scan record folder not found: .*sequences/07/voxel0.1-SNr0.6"):
        kitti.store_nbytes(kitti_root, (7,))
    with pytest.raises(ValueError, match="a KITTI scan record is \\[7, n\\]"):
        bad = tmp_path / "bad.npy"
        np.save(bad, np.zeros((4, 3), np.float32))
        kitti.read_record(str(bad))
    with pytest.raises(ValueError, match="expected 'KEY: 12 numbers'"):
        kitti.parse_calib("P2: 1 2 3\n")
    with pytest.raises(KeyError, match="calibration has no 'P3' entry"):
        kitti.camera_Pc(kitti.parse_calib(CALIB), "P3")
    with pytest.raises(IndexError, match="item 20 is outside the KITTI train list of 20 entries"):
        kitti.plan_batch(ds, [20], "train", np.random.default_rng(0))
    with pytest.raises(ValueError, match="mode must be one of"):
        kitti.plan_batch(ds, [0], "eval", np.random.default_rng(0))
    with pytest.raises(FileNotFoundError, match="Oxford split file not found: .*val.txt"):
        oxford.read_split(str(tmp_path), "val")
    with pytest.raises(ValueError, match="Oxford has train and val\\* modes"):
        oxford.read_split(oxford_root, "test")
    with pytest.raises(FileNotFoundError, match="Oxford timestamps not found: .*nowhere/pc_timestamps.npy"):
        oxford.OxfordDataset(oxford_root, "val", traversals=["nowhere"])
    (tmp_path / "o").mkdir()
    (tmp_path / "o" / "val.txt").write_text("\n")
    with pytest.raises(ValueError, match="the Oxford val split of .* lists no traversal"):
        oxford.OxfordDataset(str(tmp_path / "o"), "val")
    t = tmp_path / "o" / "t0"
    t.mkdir()
    for name in ("pc_timestamps", "camera_timestamps"):
        np.save(t / (name + ".npy"), np.zeros(0, np.int64))
    for name in ("pc_poses", "camera_poses"):
        np.save(t / (name + ".npy"), np.zeros((0, 4, 4)))
    with pytest.raises(ValueError, match="Oxford traversal t0 is empty"):
        oxford.OxfordDataset(str(tmp_path / "o"), "val", traversals=["t0"])
    with pytest.raises(FileNotFoundError, match="Oxford scan record not found: .*lms_front/1.npy"):
        oxford.read_record(oxford.record_path(oxford_root, "x", 1))
    ods = oxford.OxfordDataset(oxford_root, "val")
    with pytest.raises(IndexError, match="item 24 is outside the Oxford val list of 24 entries"):
        oxford.plan_batch(ods, [24], "val", np.random.default_rng(0))
