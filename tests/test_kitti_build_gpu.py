"""The KITTI accumulated-frame build on the device (csrc/kitti_build.cu via deepi2p_b200.kitti_build) against
oracle_kitti_build and tests/golden/kitti_build_small.npz bit for bit, at the ego box's borders and the range radius,
across batch sizes, and read back through kitti_batch(record_dir=...)."""
import os
import sys

import numpy as np
import pytest
import torch

import oracle_kitti_build as okb
from deepi2p_b200 import assemble, kitti, kitti_build as kb, synthetic as syn

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_kitti_build_golden as mg  # noqa: E402

GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "kitti_build_small.npz"))


def _golden_records():
    off = np.concatenate([[0], np.cumsum(GOLDEN["m_pts"])])
    return [GOLDEN["records"][:, off[i]:off[i + 1]] for i in range(len(GOLDEN["m_pts"]))]


@pytest.fixture(scope="module")
def small(tmp_path_factory, cuda):
    root = mg.write_root(str(tmp_path_factory.mktemp("kbsmall") / "kitti"))
    a = mg.BUILD_ARGS
    plan = kb.plan_sequence(root, mg.SEQ, a["frame_stride_dist"], a["accumulate_radius"])
    return root, plan, kb.stride_store(plan)


def _same_bits(a, b):
    """Bit-identical floats, except that a NaN may be any NaN (numpy's 0 / 0 and the device's differ in sign)."""
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a.view(np.uint32)[~na],
                                                                             b.view(np.uint32)[~nb])


def _records(res):
    rec = res["records"].cpu().numpy()
    return [rec[k, :, :m] for k, m in enumerate(res["m_host"])], rec, res["m_host"]


def test_small_sequence_equals_golden_and_oracle(small):
    root, plan, store = small
    res = kb.build_plan_frames(store, plan, range(plan["n"]), mg.BUILD_ARGS["voxel_size"])
    got, rec, m = _records(res)
    gold = _golden_records()
    assert len(got) == len(gold)
    for i, (g, r) in enumerate(zip(got, gold)):
        assert g.shape == r.shape, i
        assert _same_bits(g, r), i                                           # bit for bit, NaN where NaN
        assert not rec[i, :, m[i]:].any(), i
    # the all-zero-intensity window: a NaN intensity row, every other row finite
    last = got[-1]
    assert np.isnan(last[3]).all() and np.isfinite(last[[0, 1, 2, 4, 5, 6]]).all()
    assert res["imax"][-1] == 0.0
    o = okb.accumulate_sequence(root, mg.SEQ, kitti.read_calib(root, mg.SEQ)["Tr"], **mg.BUILD_ARGS, frames=[0, 9])
    for i in (0, 9):
        assert _same_bits(got[i], o["records"][i]), i


def test_batch_sizes_give_the_same_bytes(small):
    _, plan, store = small
    v = mg.BUILD_ARGS["voxel_size"]
    whole, _, _ = _records(kb.build_plan_frames(store, plan, range(plan["n"]), v))
    for size in (1, 3, 64):
        parts = []
        for s in range(0, plan["n"], size):
            parts += _records(kb.build_plan_frames(store, plan, range(s, min(s + size, plan["n"])), v))[0]
        assert all(a.tobytes() == b.tobytes() for a, b in zip(whole, parts)), size


def test_pinned_store_and_a_second_stream(small):
    _, plan, store = small
    v = mg.BUILD_ARGS["voxel_size"]
    ref, _, _ = _records(kb.build_plan_frames(store, plan, range(plan["n"]), v))
    s = torch.cuda.Stream()
    got, _, _ = _records(kb.build_plan_frames(store.to("pinned"), plan, range(plan["n"]), v, stream=s))
    assert all(a.tobytes() == b.tobytes() for a, b in zip(ref, got))


def _edge_record():
    """Points at the float32-rounded ego borders, one ulp inside and outside, and at ranges around 5: (3, 4) is
    exactly 5 from the sensor, its neighbours one float32 ulp in y either side."""
    b = np.array(kb.EGO_BOX, dtype=np.float64).astype(np.float32)
    inward = lambda v: np.nextafter(v, np.float32(0))           # noqa: E731
    pts = [(b[1], 0.0), (b[0], 0.0), (0.5, b[3]), (0.5, b[2]),                  # on the borders: kept
           (inward(b[1]), 0.0), (inward(b[0]), 0.0), (0.5, inward(b[3])), (0.5, inward(b[2])),   # inside: dropped
           (b[1], b[3]), (b[0], b[2]), (-3.0, 0.3), (1.0, -1.5),                   # corners and outside: kept
           (3.0, 4.0), (3.0, np.nextafter(np.float32(4), np.float32(0))), (3.0, np.nextafter(np.float32(4),
                                                                                       np.float32(9))),
           (-4.0, 3.0), (0.0, 5.0), (0.0, 7.0)]
    xy = np.array(pts, dtype=np.float32).T
    n = xy.shape[1]
    rec = np.zeros((7, n), np.float32)
    rec[0:2] = xy
    rec[2] = np.arange(n, dtype=np.float32) * 0.25 - 1.0
    rec[3] = np.linspace(0.1, 0.9, n, dtype=np.float32)
    rec[4:7] = np.array([[0.0], [0.6], [0.8]], np.float32)
    return rec


def test_ego_borders_kept_and_radius_dropped(cuda):
    rec = _edge_record()
    store = assemble.ScanStore([rec])
    P = np.eye(4)[None]
    res = kb.build_frames(store, [0], [0, 1], P, voxel_size=0.01, accumulate_radius=5.0)
    got = res["records"][0, :, :res["m_host"][0]].cpu().numpy()
    ref = okb.accumulate_frame([rec], [P[0]], 0.01, 5.0)
    assert _same_bits(got, ref)
    assert res["n_pts"][0] == rec.shape[1] - 4                   # the four points one ulp inside the box
    keep = {(float(x), float(y)) for x, y in got[0:2].T}
    for x, y in [(2.7, 0.0), (-2.025, 0.0), (0.5, 0.8), (0.5, -0.8), (2.7, 0.8), (-2.025, -0.8)]:
        assert (float(np.float32(x)), float(np.float32(y))) in keep, (x, y)
    ys = {y for x, y in keep if x == 3.0}
    assert float(np.nextafter(np.float32(4), np.float32(0))) in ys
    assert 4.0 not in ys and float(np.nextafter(np.float32(4), np.float32(9))) not in ys
    assert (-4.0, 3.0) not in keep and (0.0, 5.0) not in keep and (0.0, 7.0) not in keep
    # intensity rides through as colour = intensity / max and back; normals pass through the identity
    assert np.array_equal(got[4:7], np.repeat(np.array([[0.0], [0.6], [0.8]], np.float32), got.shape[1], 1))


def test_normals_take_the_translation_and_errors(cuda):
    rec = _edge_record()[:, 10:12]
    store = assemble.ScanStore([rec])
    P = np.eye(4)
    P[:3, 3] = (1.0, -2.0, 0.5)
    res = kb.build_frames(store, [0], [0, 1], P[None], voxel_size=0.01, accumulate_radius=50.0)
    got = res["records"][0, :, :res["m_host"][0]].cpu().numpy()
    ref = okb.accumulate_frame([rec], [P], 0.01, 50.0)
    assert np.array_equal(got, ref)
    assert np.allclose(got[4:7], rec[4:7] + np.array([[1.0], [-2.0], [0.5]], np.float32))
    inside = np.zeros((7, 3), np.float32)
    with pytest.raises(ValueError, match="no point outside the ego box"):
        kb.build_frames(assemble.ScanStore([inside]), [0], [0, 1], np.eye(4)[None])
    with pytest.raises(ValueError, match="first"):
        kb.build_frames(store, [0], [0, 2], P[None])
    with pytest.raises(ValueError, match="P must be"):
        kb.build_frames(store, [0], [0, 1], np.full((1, 4, 4), np.nan))


def test_build_sequence_files_and_kitti_batch(tmp_path, cuda):
    root = str(tmp_path / "kitti")
    syn.write_kitti_root(root, seqs=(9, 10), n_frames=84, seed=2, n_rings=8, n_azimuth=128, n_images=2)
    logs = []
    assert kb.build_sequence(root, 9, batch=32, log=logs.append) == 84
    assert len(logs) == 3 and kb.build_sequence(root, 9, log=logs.append) == 0 and logs[-1].endswith("exists, skip")
    folder = "stride4-acc50-voxel0.4"
    d = kitti.record_dir(root, 9, folder)
    assert sorted(os.listdir(d)) == ["%06d.npy" % i for i in range(84)]
    plan = kb.plan_sequence(root, 9)
    o = okb.accumulate_sequence(root, 9, kitti.read_calib(root, 9)["Tr"], 4, 50, 0.4, frames=[0, 41, 83])
    for i in (0, 41, 83):
        assert np.array_equal(np.load(os.path.join(d, "%06d.npy" % i)), o["records"][i]), i
    assert o["strides"] == plan["strides"]
    # the readers: record_dir names the accumulated folder; without it they read voxel0.1-SNr0.6 as before
    items = [0, 3, 5]
    ds = kitti.KittiDataset(root, "val", record_dir=folder)
    recs = {(9, i): np.load(os.path.join(d, "%06d.npy" % i)) for i in range(84)}
    store = assemble.ScanStore(list(recs.values()), keys=list(recs))
    a = kitti.kitti_batch(ds, items, "val", seed=4, rng=11)
    b = kitti.kitti_batch(root, items, "val", seed=4, rng=11, record_dir=folder)
    c = kitti.kitti_batch(root, items, "val", seed=4, rng=11, store=store)
    assert kitti.store_nbytes(root, [9], record_dir=folder) == store.nbytes
    acc_store = kitti.scan_store(root, [9], record_dir=folder)
    e = kitti.kitti_batch(root, items, "val", seed=4, rng=11, store=acc_store)
    for x, y, z, w in zip(a, b, c, e):
        assert torch.equal(x.cpu(), y.cpu()) and torch.equal(x.cpu(), z.cpu()) and torch.equal(x.cpu(), w.cpu())
    base = {(9, i): np.load(kitti.record_path(root, 9, i)) for i in range(84)}
    f = kitti.kitti_batch(root, items, "val", seed=4, rng=11)
    g = kitti.kitti_batch(root, items, "val", seed=4, rng=11, store=assemble.ScanStore(list(base.values()),
                                                                                       keys=list(base)))
    h = kitti.kitti_batch(root, items, "val", seed=4, rng=11, record_dir="voxel0.1-SNr0.6")
    for x, y, z in zip(f, g, h):
        assert torch.equal(x.cpu(), y.cpu()) and torch.equal(x.cpu(), z.cpu())
    assert not torch.equal(a[0].cpu(), f[0].cpu())
