"""Accumulation from a ragged scan store (assemble_accumulate_gather_f32) against the padded entry, and the KITTI and
Oxford readers (kitti_batch, oxford_batch) on seeded roots against assemble_batch(pack_frames(...)) +
assemble_images on the frames, transforms and draws of oracle_datasets, bit for bit."""
import numpy as np
import pytest
import torch

import oracle_datasets as od
from deepi2p_b200 import assemble, imageprep, kitti, oxford, synthetic

pytestmark = pytest.mark.gpu


def _records(seed, sizes, rows=7):
    rng = np.random.default_rng(seed)
    out = []
    for n in sizes:
        r = rng.uniform(-40.0, 40.0, (rows, n)).astype(np.float32)
        r[3] = rng.random(n, dtype=np.float32)
        out.append(r)
    return out


def _rigid(rng):
    P = np.eye(4)
    a = rng.uniform(-0.3, 0.3, 3)
    c, s = np.cos(a), np.sin(a)
    P[:3, :3] = (np.array([[c[2], -s[2], 0], [s[2], c[2], 0], [0, 0, 1]]) @
                 np.array([[c[1], 0, s[1]], [0, 1, 0], [-s[1], 0, c[1]]]))
    P[:3, 3] = rng.uniform(-5, 5, 3)
    return P


@pytest.mark.parametrize("with_sn", [True, False])
@pytest.mark.parametrize("range_max", [None, 30.0])
@pytest.mark.parametrize("location", ["cuda", "pinned"])
def test_gather_equals_padded(cuda, with_sn, range_max, location):
    recs = _records(1, [700, 0, 1531, 16, 1, 2048, 333], rows=7 if with_sn else 4)
    store = assemble.ScanStore(recs, location)
    # out-of-order and repeated records, an empty record inside a sample and a sample made of it alone
    ids = np.array([2, 0, 2, 5, 1, 1, 6, 3, 4, 6, 0, 5, 5])
    fs = np.array([0, 0, 0, 0, 1, 2, 2, 2, 3, 3, 3, 3, 4])
    rng = np.random.default_rng(2)
    FT = np.stack([np.eye(4) if k == 0 or fs[k] != fs[k - 1] else _rigid(rng) for k in range(len(ids))])
    fr = assemble.store_frames(store, ids, fs, FT)
    got = assemble.accumulate_gather(fr, range_max)
    samples = [([(recs[i][:3], recs[i][3], recs[i][4:7] if with_sn else None) for i in ids[fs == s]], FT[fs == s])
               for s in range(fs[-1] + 1)]
    pk = assemble.pack_frames(samples)
    ref = assemble.accumulate(pk["xyz"], pk["intensity"], pk["sn"], pk["n_pts"], pk["frame_sample"], pk["frame_T"],
                              range_max)
    torch.cuda.synchronize()
    assert np.array_equal(got[4], ref[4]) and got[4][1] == 0
    assert (got[2] is None) == (ref[2] is None) == (not with_sn)
    for a, b in zip(got[:3], ref[:3]):
        if a is not None:
            assert a.shape == b.shape and torch.equal(a, b)
    n_in = sum(recs[i].shape[1] for i in ids)
    assert (ref[4].sum() < n_in) if range_max is not None else (ref[4].sum() == n_in)


def test_store_locations_and_per_batch_path_agree(cuda):
    recs = _records(3, [900, 1200, 640, 1100])
    ids, fs = np.array([0, 1, 2, 1, 3, 0]), np.array([0, 0, 0, 1, 1, 1])
    rng = np.random.default_rng(4)
    FT = np.stack([np.eye(4) if k in (0, 3) else _rigid(rng) for k in range(6)])
    dev = assemble.ScanStore(recs, "cuda")
    pin = assemble.ScanStore(recs, "pinned")
    assert dev.nbytes == pin.nbytes == 7 * 4 * sum(r.shape[1] for r in recs)
    assert dev.offsets.tolist() == [0, 900, 2100, 2740] and pin.counts.tolist() == [900, 1200, 640, 1100]
    outs = []
    for fr in (assemble.store_frames(dev, ids, fs, FT), assemble.store_frames(pin, ids, fs, FT),
               assemble.batch_frames(recs, ids, fs, FT), assemble.store_frames(pin.to("cuda"), ids, fs, FT)):
        outs.append(assemble.assemble_batch(fr, "train", 9, input_pt_num=1024, node_a_num=16, node_b_num=16, rng=5,
                                            **assemble.kitti_args(np.eye(4))))
    torch.cuda.synchronize()
    for o in outs[1:]:
        for k in ("pc", "intensity", "sn", "node_a", "node_b", "src_index", "n_before_resample"):
            assert torch.equal(o[k], outs[0][k]), k


def test_device_store_staging_across_transfers(cuda, monkeypatch):
    recs = _records(6, [700, 0, 2500, 16, 1, 999, 1000])
    pin = assemble.ScanStore(recs, "pinned")
    monkeypatch.setattr(assemble, "STAGE_POINTS", 1000)       # records split over transfers, one ends on a boundary
    dev = assemble.ScanStore(recs, "cuda")
    assert torch.equal(dev.data.cpu(), pin.data)
    assert torch.equal(pin.data[:, 3217:4216], torch.from_numpy(recs[5]))


def test_store_errors(cuda):
    with pytest.raises(ValueError, match="location must be one of"):
        assemble.ScanStore(_records(0, [4]), "cpu")
    bad = _records(0, [4])
    bad[0][1, 2] = np.nan
    with pytest.raises(ValueError, match="record 0 has a non-finite coordinate"):
        assemble.ScanStore(bad, "cuda")
    st = assemble.ScanStore(_records(0, [4, 5]), "cuda", keys=["a", "b"])
    assert st.index("b") == 1
    with pytest.raises(KeyError, match="no record 'c' in the scan store"):
        st.index("c")
    with pytest.raises(ValueError, match="record ids must be in \\[0, 2\\)"):
        assemble.store_frames(st, [0, 2], [0, 0], np.tile(np.eye(4), (2, 1, 1)))
    fr = assemble.store_frames(st, [0, 1], [0, 0], np.tile(np.eye(4), (2, 1, 1)))
    with pytest.raises(ValueError, match="store-backed frames take the float32 accumulation"):
        assemble.assemble_batch(fr, "test", 1, input_pt_num=8, node_a_num=1, node_b_num=1, accumulate_f64=True)
    # pageable host memory is refused by the kernel entry
    lib = __import__("deepi2p_b200._native", fromlist=["load"]).load()
    host = np.zeros((4, 8), np.float32)
    off = torch.zeros(1, dtype=torch.int64, device="cuda")
    n = torch.full((1,), 8, dtype=torch.int32, device="cuda")
    fsd = torch.zeros(1, dtype=torch.int32, device="cuda")
    T = torch.eye(4, dtype=torch.float64, device="cuda")
    out = torch.zeros((3, 16), device="cuda")
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    ws = torch.zeros(lib.assemble_accumulate_gather_workspace_bytes(1, 8, 1) + 256, dtype=torch.uint8, device="cuda")
    wp = (ws.data_ptr() + 255) // 256 * 256
    rc = lib.assemble_accumulate_gather_f32(host.ctypes.data, host.ctypes.data + 96, None, 8, off.data_ptr(),
                                            n.data_ptr(), 8, 1, fsd.data_ptr(), T.data_ptr(), 1, 0.0,
                                            out.data_ptr(), out[0].data_ptr(), None, 16, cnt.data_ptr(), wp,
                                            ws.numel() - 256, 0)
    assert rc != 0 and b"device or pinned host memory" in lib.dib_last_error()


@pytest.fixture(scope="module")
def kitti_root(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("kitti"))
    synthetic.write_kitti_root(root, seqs=(0, 9, 10), n_frames=90, seed=5)
    return root


@pytest.fixture(scope="module")
def oxford_root(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("oxford"))
    synthetic.write_oxford_root(root, seed=5)
    return root


KN, KM = 2048, 64
ON, OM = 512, 32


def _kitti_expected(root, mode, items, seed, rng_seed, seqs):
    rng = np.random.default_rng(rng_seed)
    lst = od.kitti_list(root, seqs)
    smps = [od.kitti_expected(root, lst[it], rng) for it in items]
    out = assemble.assemble_batch(assemble.pack_frames([(m["frames"], m["frame_T"]) for m in smps]), mode, seed,
                                  input_pt_num=KN, node_a_num=KM, node_b_num=KM, rng=rng,
                                  **assemble.kitti_args(np.stack([m["Pc"] for m in smps]),
                                                        np.stack([m["Pji"] for m in smps])))
    im = imageprep.assemble_images(imageprep.pack_images([m["img"] for m in smps]), np.stack([m["K"] for m in smps]),
                                   mode, rng=rng, flip=out["flip"], **imageprep.kitti_image_args())
    t = np.stack([np.asarray(m["t_ji"]) for m in smps]).astype(np.float32)
    return (out["pc"], out["intensity"], out["sn"], out["node_a"], out["node_b"], out["P"], im["img"], im["K"],
            torch.from_numpy(t))


def _equal(got, ref):
    names = ("pc", "intensity", "sn", "node_a", "node_b", "P", "img", "K", "t")
    for name, g, r in zip(names, got, ref):
        assert g.shape == r.shape and torch.equal(g.cpu(), r.cpu()), name


@pytest.mark.parametrize("mode", ["train", "val", "val_random_Ry"])
def test_kitti_batch_equals_the_oracle_frames(cuda, kitti_root, mode):
    seqs = (0,) if mode == "train" else (9, 10)
    ds = kitti.KittiDataset(kitti_root, mode, seqs=seqs)
    items = [0, 1, 3, 7, len(ds) - 1, 2]
    got = kitti.kitti_batch(ds, items, mode, 11, rng=21, input_pt_num=KN, node_a_num=KM, node_b_num=KM)
    ref = _kitti_expected(kitti_root, mode, items, 11, 21, seqs)
    torch.cuda.synchronize()
    _equal(got, ref)
    assert got[0].shape == (6, 3, KN) and got[6].shape == (6, 3, 160, 512) and got[2].abs().sum() > 0


def test_kitti_stores_runs_and_streams_agree(cuda, kitti_root):
    ds = kitti.KittiDataset(kitti_root, "val_random_Ry", seqs=(9, 10))
    items = list(range(0, len(ds), 3))
    dev = kitti.scan_store(kitti_root, (9, 10), "cuda")
    pin = kitti.scan_store(kitti_root, (9, 10), "pinned")
    assert dev.nbytes == kitti.store_nbytes(kitti_root, (9, 10)) and len(dev) == 180
    runs = [kitti.kitti_batch(ds, items, "val_random_Ry", 3, rng=8, store=s, input_pt_num=KN, node_a_num=KM,
                              node_b_num=KM) for s in (None, dev, pin, None)]
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        runs.append(kitti.kitti_batch(ds, items, "val_random_Ry", 3, rng=8, store=dev, input_pt_num=KN,
                                      node_a_num=KM, node_b_num=KM, stream=st))
    st.synchronize()
    torch.cuda.synchronize()
    for r in runs[1:]:
        _equal(r, runs[0])


def _oxford_expected(root, mode, items, seed, rng_seed):
    rng = np.random.default_rng(rng_seed)
    entries, tables = od.oxford_tables(root, mode)
    smps = [od.oxford_expected(root, tables, entries[it], rng) for it in items]
    P = np.stack([m["P_cam_pc"] for m in smps])
    out = assemble.assemble_batch(assemble.pack_frames([(m["frames"], m["frame_T"]) for m in smps]), mode, seed,
                                  input_pt_num=ON, node_a_num=OM, node_b_num=OM, rng=rng, **assemble.oxford_args(P))
    im = imageprep.assemble_images(imageprep.read_jpeg_batch([m["image_path"] for m in smps]), oxford.K_CENTRE, mode,
                                   rng=rng, **imageprep.oxford_image_args())
    return (out["pc"], out["intensity"], out["sn"], out["node_a"], out["node_b"], out["P"], im["img"], im["K"],
            torch.from_numpy(P[:, :3, 3].astype(np.float32)))


@pytest.mark.parametrize("mode", ["train", "val", "val_random_Ry"])
def test_oxford_batch_equals_the_oracle_frames(cuda, oxford_root, mode):
    ds = oxford.OxfordDataset(oxford_root, mode)
    items = [0, 5, 5, len(ds) - 1, 1]
    got = oxford.oxford_batch(ds, items, mode, 4, rng=13, input_pt_num=ON, node_a_num=OM, node_b_num=OM)
    ref = _oxford_expected(oxford_root, mode, items, 4, 13)
    torch.cuda.synchronize()
    _equal(got, ref)
    assert got[6].shape == (5, 3, 384, 640) and not got[2].any()


def test_oxford_stores_runs_and_streams_agree(cuda, oxford_root):
    ds = oxford.OxfordDataset(oxford_root, "train")
    names = list(ds.traversals)
    dev = oxford.scan_store(oxford_root, names, "cuda")
    pin = oxford.scan_store(oxford_root, names, "pinned")
    items = [0, 30, 2, 47, 2]
    runs = [oxford.oxford_batch(ds, items, "train", 6, rng=1, store=s, input_pt_num=ON, node_a_num=OM,
                                node_b_num=OM) for s in (None, dev, pin, None)]
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        runs.append(oxford.oxford_batch(ds, items, "train", 6, rng=1, store=pin, input_pt_num=ON, node_a_num=OM,
                                        node_b_num=OM, stream=st))
    st.synchronize()
    torch.cuda.synchronize()
    for r in runs[1:]:
        _equal(r, runs[0])


def test_evaluate_dataset_script_end_to_end(cuda, kitti_root, oxford_root, tmp_path, capsys):
    import importlib.util
    import os
    from deepi2p_b200 import network
    spec = importlib.util.spec_from_file_location(
        "evaluate_dataset", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts",
                                         "evaluate_dataset.py"))
    ev = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ev)
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_small.npz"))
    so = np.concatenate([[0], np.cumsum(g["stream_lens"])])
    i = int(np.nonzero((g["shapes"][:, 0] == 900) & (g["shapes"][:, 1] == 1600))[0][0])
    nu_root = str(tmp_path / "nuscenes")
    synthetic.write_nuscenes_dataroot(nu_root, [(14, 6), (9, 4)], seed=2,
                                      jpeg=g["streams"][so[i]:so[i + 1]].tobytes())
    for name, root, every in (("kitti", kitti_root, 10), ("oxford", oxford_root, 8), ("nuscenes", nu_root, 1)):
        ckpt = str(tmp_path / f"{name}.pth")
        torch.save(synthetic.seeded_state_dict(network.KeypointDetector(**network.SHAPES[name]), 3), ckpt)
        out = str(tmp_path / f"out_{name}")
        s = ev.main(["--dataset", name, "--root", root, "--checkpoint", ckpt, "--every", str(every), "--batch", "2",
                     "--inits", "8", "--version", "v1.0-mini", "--out", out, "--head", "fused"])
        text = capsys.readouterr().out
        assert "RTE " in text and "success rate" in text, name
        P = np.load(os.path.join(out, "P_pred_all_np.npy"))
        gt = np.load(os.path.join(out, "P_gt_all_np.npy"))
        cost = np.load(os.path.join(out, "cost_all_np.npy"))
        assert P.shape == gt.shape == (cost.shape[0], 4, 4) and cost.shape[0] >= 2, name
        assert np.isfinite(P).all() and np.isfinite(gt).all() and s["n"] <= cost.shape[0], name
