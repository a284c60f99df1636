"""The KITTI accumulated-frame build's host half (deepi2p_b200.kitti_build: the stride walk, the windows and the
transforms) against oracle_kitti_build on synthetic pose chains, the ego box against the reference's numpy
expression, the golden file against its generator, and the readers' record_dir argument."""
import os
import sys

import numpy as np
import pytest

import oracle_kitti_build as okb
from deepi2p_b200 import kitti, kitti_build as kb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_kitti_build_golden as mg  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "kitti_build_small.npz")


def _pose(t, yaw=0.0):
    P = np.eye(4)
    c, s = np.cos(yaw), np.sin(yaw)
    P[0, 0], P[0, 2], P[2, 0], P[2, 2] = c, s, -s, c
    P[:3, 3] = t
    return P


def _write_chain(root, seq, poses, records=True):
    """poses/<seq>/%06d.npz and, with records, one tiny [7, 1] record per frame (the build plan reads the poses and
    counts the record folder)."""
    pdir = os.path.join(root, "poses", "%02d" % seq)
    rdir = kitti.record_dir(root, seq)
    os.makedirs(pdir, exist_ok=True)
    os.makedirs(rdir, exist_ok=True)
    for i, P in enumerate(poses):
        np.savez(os.path.join(pdir, "%06d.npz" % i), pose=P)
        if records:
            np.save(os.path.join(rdir, "%06d.npy" % i), np.ones((7, 1), np.float32))


TR = np.array([[0.0, -1.0, 0.0, 0.01], [0.0, 0.0, -1.0, -0.07], [1.0, 0.0, 0.0, -0.27], [0.0, 0.0, 0.0, 1.0]])


def _chains():
    rng = np.random.default_rng(7)
    # steps along z that are exact in float64: 4.0 from the last kept frame is not kept (the test is strict),
    # 4 + 2^-48 is; 8.5 is 4.0 from the kept 4.5 but 3.5 from the frame before it, so P_prev moves only on a keep
    exact = [_pose([0.0, 0.0, z]) for z in (0, 1, 2, 3, 4, 4.5, 8.5, 8.5 + 2.0 ** -48, 12, 13)]
    drive, yaw, p = [], 0.3, np.zeros(3)
    for _ in range(60):
        yaw += rng.normal(0.0, 0.05)
        p = p + np.array([np.sin(yaw), rng.normal(0.0, 0.01), np.cos(yaw)]) * rng.uniform(0.0, 2.5)
        drive.append(_pose(p, yaw))
    f32 = [P.astype(np.float32) for P in drive[:30]]          # poses stored in float32 keep their dtype
    return dict(exact=exact, drive=drive, short=drive[:5], one=drive[:1], f32=f32)


@pytest.mark.parametrize("name", ["exact", "drive", "short", "one", "f32"])
@pytest.mark.parametrize("stride,radius", [(4, 50), (4, 10), (4, 14), (4, 1), (2.5, 5), (4, 2)])
def test_plan_equals_oracle(tmp_path, name, stride, radius):
    poses = _chains()[name]
    root = str(tmp_path)
    _write_chain(root, 0, poses)
    o = okb.plan(root, 0, stride, radius)
    p = kb.plan_sequence(root, 0, stride, radius, Tr=TR)
    assert p["n"] == o["sample_num"] == len(poses)
    assert p["strides"] == o["strides"]
    assert p["acc"] == o["acc"]
    assert [tuple(w) for w in p["windows"].tolist()] == o["windows"]
    frames = [i for i in range(p["n"]) if o["windows"][i][0] <= o["windows"][i][1]]
    if not frames:
        return
    strides, first, P = kb.frame_pairs(p, frames)
    for k, i in enumerate(frames):
        ref = okb.transforms(root, 0, TR, o["strides"], o["windows"][i], i)
        assert strides[first[k]:first[k + 1]] == [j for j, _ in ref]
        got = P[first[k]:first[k + 1]]
        assert got.dtype == np.float64
        assert np.array_equal(got, np.stack([M for _, M in ref]))


def test_stride_walk_edges(tmp_path):
    ch = _chains()
    # a step of exactly frame_stride_dist is not kept; the first frame always is; P_prev moves only on a kept frame
    assert kb.stride_list(ch["exact"], 4) == [0, 5, 7, 9]
    assert kb.stride_list(ch["one"], 4) == [0]
    assert kb.stride_list(ch["exact"], 100) == [0]


def test_round_half_to_even_and_windows():
    assert [kb.accumulate_frames(4, r) for r in (10, 14, 18, 2, 6, 50)] == [2, 4, 4, 0, 2, 12]
    assert kb.accumulate_frames(2.5, 5) == 2
    strides = [0, 5, 7, 8, 9]
    w = kb.windows(strides, 12, 1)
    # first frame, a stride frame, a frame between strides, frames past the last stride (clamped to the list)
    assert w[0].tolist() == [0, 1] and w[5].tolist() == [0, 2] and w[6].tolist() == [1, 3]
    assert w[9].tolist() == [3, 4] and w[10].tolist() == [4, 4] and w[11].tolist() == [4, 4]
    # a window wider than the sequence covers the whole list
    assert kb.windows(strides, 12, 12)[6].tolist() == [0, 4]
    # accumulate_frames 0 past the last stride frame: an empty window, refused by frame_pairs
    e = kb.windows(strides, 12, 0)
    assert e[10].tolist() == [5, 4]


def test_empty_window_raises(tmp_path):
    root = str(tmp_path)
    _write_chain(root, 0, _chains()["exact"][:7])
    p = kb.plan_sequence(root, 0, 4, 1, Tr=TR)
    assert p["acc"] == 0 and p["strides"] == [0, 5]             # frame 6 lies past the last stride frame
    kb.frame_pairs(p, [0, 1, 5])
    with pytest.raises(ValueError, match="frame 6: its window of stride frames is empty"):
        kb.frame_pairs(p, [5, 6])


def test_ego_box_matches_the_reference_expression():
    """The kernel compares float32 coordinates against the float32-rounded borders; the reference's numpy expression
    on the float32 record does the same, so the borders themselves are kept and one ulp inside is dropped."""
    b = np.array(kb.EGO_BOX, dtype=np.float64).astype(np.float32)
    assert b.tolist() == [np.float32(-2.025), np.float32(2.7), np.float32(-0.8), np.float32(0.8)]
    xs = [b[0], b[1], np.nextafter(b[0], np.float32(0)), np.nextafter(b[1], np.float32(0)), np.float32(0),
          np.nextafter(b[0], np.float32(-9)), np.nextafter(b[1], np.float32(9))]
    ys = [b[2], b[3], np.nextafter(b[2], np.float32(0)), np.nextafter(b[3], np.float32(0)), np.float32(0)]
    X, Y = np.meshgrid(np.array(xs, np.float32), np.array(ys, np.float32))
    d = np.stack([X.ravel(), Y.ravel()]).astype(np.float32)
    x_inside = np.logical_and(d[0, :] < 2.7, d[0, :] > -2.7 * 0.75)
    y_inside = np.logical_and(d[1, :] < 0.8, d[1, :] > -0.8)
    ref_keep = np.logical_not(np.logical_and(x_inside, y_inside))
    ours = np.logical_not((d[0] < b[1]) & (d[0] > b[0]) & (d[1] < b[3]) & (d[1] > b[2]))
    assert np.array_equal(ref_keep, ours)
    inside = (np.abs(d[0]) < 2) & (np.abs(d[1]) < 0.7)
    assert not ref_keep[inside].any() and ref_keep[~inside & ((d[0] == b[1]) | (d[1] == b[3]))].all()


def test_golden_regenerates_bit_for_bit(tmp_path):
    out = str(tmp_path / "g.npz")
    mg.make(out)
    a, b = np.load(out), np.load(GOLDEN)
    assert sorted(a.files) == sorted(b.files)
    for k in a.files:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, k
        assert np.array_equal(a[k], b[k], equal_nan=a[k].dtype.kind == "f"), k
    assert np.isnan(b["records"][3]).any()


def test_golden_plan_equals_host_plan(tmp_path):
    g = np.load(GOLDEN)
    root = mg.write_root(str(tmp_path / "kitti"))
    p = kb.plan_sequence(root, mg.SEQ, mg.BUILD_ARGS["frame_stride_dist"], mg.BUILD_ARGS["accumulate_radius"])
    assert p["strides"] == g["strides"].tolist() and p["acc"] == int(g["acc"]) == 2
    assert np.array_equal(p["windows"], g["windows"])
    strides, first, P = kb.frame_pairs(p, range(p["n"]))
    assert strides == g["window_strides"].tolist() and np.array_equal(P, g["P"])


def test_output_folder_and_record_dir_defaults(tmp_path):
    assert kb.output_folder() == "stride4-acc50-voxel0.4"
    assert kb.output_folder(4, 50, 0.2) == "stride4-acc50-voxel0.2"
    root = str(tmp_path)
    assert kitti.record_dir(root, 3) == os.path.join(root, "data_odometry_velodyne_NWU", "sequences", "03",
                                                     "voxel0.1-SNr0.6")
    assert kitti.record_path(root, 3, 7).endswith(os.path.join("03", "voxel0.1-SNr0.6", "000007.npy"))
    acc = kitti.record_path(root, 3, 7, record_dir="stride4-acc50-voxel0.4")
    assert acc.endswith(os.path.join("03", "stride4-acc50-voxel0.4", "000007.npy"))
    assert kb.output_dir(root, 3) == kitti.record_dir(root, 3, "stride4-acc50-voxel0.4")


def test_store_nbytes_reads_the_named_folder(tmp_path):
    root = str(tmp_path)
    for folder, n in (("voxel0.1-SNr0.6", 3), ("stride4-acc50-voxel0.4", 5)):
        d = kitti.record_dir(root, 0, folder)
        os.makedirs(d)
        for i in range(2):
            np.save(os.path.join(d, "%06d.npy" % i), np.zeros((7, n), np.float32))
    assert kitti.store_nbytes(root, [0]) == 2 * 28 * 3
    assert kitti.store_nbytes(root, [0], record_dir="stride4-acc50-voxel0.4") == 2 * 28 * 5
    with pytest.raises(FileNotFoundError):
        kitti.store_nbytes(root, [0], record_dir="missing")


def test_build_frames_validates_before_the_device():
    with pytest.raises(ValueError):
        kb._box((1.0, 0.0, 0.0, 1.0))
    with pytest.raises(ValueError):
        kb._box((0.0, 1.0, 0.0))
