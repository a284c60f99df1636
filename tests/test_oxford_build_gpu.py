"""The Oxford RobotCar cloud build on the device (csrc/oxford_build.cu via deepi2p_b200.oxford_build) against
oracle_oxford_build bit for bit, against the reference's own run (tests/golden/oxford_build_small.npz), and end to
end through oxford_batch."""
import ast
import os

import numpy as np
import pytest
import torch

import oracle_oxford_build as oo
from deepi2p_b200 import oxford, oxford_build as ob, synthetic as syn

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "oxford_build_small.npz"))
RAW_ARGS = ast.literal_eval(str(GOLDEN["raw_args"]))
BUILD_ARGS = ast.literal_eval(str(GOLDEN["build_args"]))
T = str(GOLDEN["traversal"])
FULL_RAW = dict(seconds=60.0, speed=10.0, stops=((30.0, 31.0),), curve=(35.0, 45.0), n_returns=541, seed=11)


def _raw(tmp_path_factory, name, raw_args):
    d = tmp_path_factory.mktemp(name)
    raw, lms, sdk, out = (str(d / x) for x in ("raw", "lms", "sdk", "out"))
    syn.write_oxford_raw(raw, lms, sdk, **raw_args)
    return raw, lms, sdk, out


@pytest.fixture(scope="module")
def small(tmp_path_factory, cuda):
    raw, lms, sdk, out = _raw(tmp_path_factory, "oxsmall", RAW_ARGS)
    plan = ob.plan_traversal(raw, lms, out, T, sdk, **BUILD_ARGS)
    oracle = [oo.build_cloud(plan, c) for c in range(len(plan["centres"]))]
    return (raw, lms, sdk, out), plan, ob.RawScanStore(plan), oracle


def _check(res, oracle, ids):
    rec = res["records"].cpu().numpy()
    m = res["m_pts"].cpu().numpy()
    for k, c in enumerate(ids):
        o = oracle[c]
        assert m[k] == o["record"].shape[1], c
        assert np.array_equal(rec[k, :, :m[k]], o["record"], equal_nan=True), c
        assert not rec[k, :, m[k]:].any(), c
        assert (res["n_kept"][k], res["n_skipped"][k], res["n_pts"][k]) == (o["n_kept"], o["n_skipped"], o["n_pts"]), c


def test_small_traversal_equals_oracle_and_reference(small):
    _, plan, store, oracle = small
    ids = list(range(len(plan["centres"])))
    res = ob.build_clouds(store, plan, ids)
    _check(res, oracle, ids)
    rec, m = res["records"].cpu().numpy(), res["m_pts"].cpu().numpy()
    assert np.array_equal(m, GOLDEN["m_pts"]) and np.array_equal(res["n_kept"], GOLDEN["n_kept"])
    assert np.array_equal(res["n_skipped"], GOLDEN["n_skipped"])
    off = np.concatenate([[0], np.cumsum(GOLDEN["m_pts"])])
    for k in ids:
        ref = GOLDEN["records"][:, off[k]:off[k + 1]]
        assert np.array_equal(rec[k, 3, :m[k]], ref[3], equal_nan=True), k
        ulp = np.spacing(np.abs(ref[:3])).astype(np.float64)
        assert np.all(np.abs(rec[k, :3, :m[k]].astype(np.float64) - ref[:3]) <= ulp), k


@pytest.mark.parametrize("split", [[1], [3, 1, 4], [7, 2, 9, 0]])
def test_ragged_batches_and_splits(small, split):
    _, plan, store, oracle = small
    n = len(plan["centres"])
    rng = np.random.default_rng(len(split))
    order = rng.permutation(n).tolist()
    pos = 0
    for size in split + [n]:
        ids = order[pos:pos + max(size, 1)]
        if not ids:
            break
        _check(ob.build_clouds(store, plan, ids), oracle, ids)
        pos += len(ids)


def test_second_stream(small):
    _, plan, store, oracle = small
    s = torch.cuda.Stream()
    ids = [5, 0, 19, 12, 24]
    with torch.cuda.stream(s):
        res = ob.build_clouds(store, plan, ids, stream=s)
    s.synchronize()
    _check(res, oracle, ids)


def test_stream_not_current(small):
    """stream=s without making s current: every step and read-back still runs on s."""
    _, plan, store, oracle = small
    s = torch.cuda.Stream()
    ids = [24, 3, 17, 8, 0, 11]
    res = ob.build_clouds(store, plan, ids, stream=s)
    s.synchronize()
    _check(res, oracle, ids)


def test_vo_sourced_at_camera_frames_on_a_second_stream(tmp_path_factory, cuda):
    """The RobotCar layout (VO rows sourced at the camera frames, the last frame the last VO row) built end to end
    through build_traversal on a stream that is not current, against the oracle."""
    raw, lms, sdk, out = _raw(tmp_path_factory, "oxvocam", dict(RAW_ARGS, vo_on_cameras=True))
    plan = ob.plan_traversal(raw, lms, out, T, sdk, **BUILD_ARGS)
    s = torch.cuda.Stream()
    summary = ob.build_traversal(raw, lms, out, T, sdk, batch=6, stream=s, **BUILD_ARGS)
    assert summary["cameras_outside_vo"] == 1 and summary["clouds_built"] == len(plan["centres"]) > 0
    for c, (ts, *_) in enumerate(plan["centres"]):
        got = np.load(os.path.join(out, T, "lms_front_foreground", "%d.npy" % ts))
        o = oo.build_cloud(plan, c)
        assert np.array_equal(got, o["record"], equal_nan=True), c
        assert (summary["n_kept"][c], summary["n_skipped"][c]) == (o["n_kept"], o["n_skipped"]), c
    assert np.array_equal(np.load(os.path.join(out, T, "camera_timestamps.npy")), plan["camera_timestamps"])


def test_errors(small):
    _, plan, store, _ = small
    high = ob.RawScanStore(plan)
    high.xyr[0].fill_(5.0)                          # every return above the 0.1 m ground threshold
    with pytest.raises(ValueError, match="no point of the scans in .* is left after the ground mask"):
        ob.build_clouds(high, plan, [0])
    with pytest.raises(ValueError, match="clouds is empty"):
        ob.build_clouds(store, plan, [])


def test_missing_window_raises(tmp_path_factory, cuda):
    raw, lms, sdk, out = _raw(tmp_path_factory, "oxmissing", dict(RAW_ARGS, missing_scans=0.0))
    plan = ob.plan_traversal(raw, lms, out, T, sdk, **BUILD_ARGS)
    _, lo, hi, _ = plan["centres"][0]
    for ts in plan["lms_ts"][lo:hi]:
        os.remove(os.path.join(plan["lidar_dir"], "%d.bin" % ts))
    with pytest.raises(FileNotFoundError, match="no scan file of centre .* window in"):
        ob.build_clouds(ob.RawScanStore(plan), plan, [0])


def test_full_size_segment(tmp_path_factory, cuda):
    raw, lms, sdk, out = _raw(tmp_path_factory, "oxfull", FULL_RAW)
    plan = ob.plan_traversal(raw, lms, out, T, sdk)
    n = len(plan["centres"])
    assert n >= 64
    store = ob.RawScanStore(plan)
    ids = list(range(64))
    res = ob.build_clouds(store, plan, ids)
    assert min(hi - lo for _, lo, hi, _ in plan["centres"][:64]) > 400
    sub = [0, 21, 42, 63]
    oracle = {c: oo.build_cloud(plan, c) for c in sub}
    for c in sub:
        _check(dict(records=res["records"][c:c + 1], m_pts=res["m_pts"][c:c + 1], n_kept=res["n_kept"][c:c + 1],
                    n_skipped=res["n_skipped"][c:c + 1], n_pts=res["n_pts"][c:c + 1]), {c: oracle[c]}, [c])


def test_build_traversal_end_to_end(tmp_path_factory, cuda):
    from PIL import Image
    raw, lms, sdk, out = _raw(tmp_path_factory, "oxe2e", RAW_ARGS)
    plan = ob.plan_traversal(raw, lms, out, T, sdk, **BUILD_ARGS)
    jpg = os.path.join(out, "frame.jpg")
    os.makedirs(out, exist_ok=True)
    Image.fromarray(np.random.default_rng(0).integers(0, 256, (960, 1280, 3), dtype=np.uint8)).save(jpg, quality=90)
    os.makedirs(os.path.join(out, T, "stereo", "centre"), exist_ok=True)
    for c in plan["camera_timestamps"]:
        os.link(jpg, os.path.join(out, T, "stereo", "centre", "%d.jpg" % c))
    summary = ob.build_traversal(raw, lms, out, T, sdk, batch=7, **BUILD_ARGS)
    assert summary["clouds_built"] == len(GOLDEN["pc_timestamps"]) and summary["clouds_skipped_velocity"] == 10
    assert summary["scans_skipped"] == int(GOLDEN["n_skipped"].sum())
    missing = {x for _, lo, hi, _ in plan["centres"] for x in plan["lms_ts"][lo:hi]
               if not os.path.isfile(os.path.join(plan["lidar_dir"], "%d.bin" % x))}
    assert 0 < summary["scans_missing"] == len(missing) < int(GOLDEN["n_missing"].sum())
    assert os.path.isfile(os.path.join(out, T, "tags.csv"))
    for name in ("val.txt", "train.txt"):
        with open(os.path.join(out, name), "w") as f:
            f.write(T + "\n")
    # the same root with the oracle's records
    ref = str(tmp_path_factory.mktemp("oxe2e_ref"))
    os.makedirs(os.path.join(ref, T, "lms_front_foreground"))
    for name in ("val.txt", "train.txt"):
        os.link(os.path.join(out, name), os.path.join(ref, name))
    for name in ("pc_timestamps.npy", "pc_poses.npy", "camera_timestamps.npy", "camera_poses.npy", "stereo"):
        os.symlink(os.path.join(out, T, name), os.path.join(ref, T, name))
    for c, (ts, *_) in enumerate(plan["centres"]):
        np.save(os.path.join(ref, T, "lms_front_foreground", "%d.npy" % ts), oo.build_cloud(plan, c)["record"])
    got_ds = oxford.OxfordDataset(out, "train")
    assert len(got_ds) == len(GOLDEN["pc_timestamps"])
    for mode in ("train", "val", "val_random_Ry"):
        items = [0, 3, 11, 17]
        a, b = (oxford.oxford_batch(r, items, mode, seed=5, rng=9, input_pt_num=1024, node_a_num=16, node_b_num=16,
                                    remove_ground=True) for r in (out, ref))
        for x, y in zip(a, b):
            x = x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)
            y = y.cpu().numpy() if isinstance(y, torch.Tensor) else np.asarray(y)
            assert np.array_equal(x, y, equal_nan=True), mode
