"""classifier.prediction_accuracy against oracle_cls labels and classifier_loss's counts, network.classify_batch under
classify_and_register, and scripts/evaluate_dataset.py's three methods against the same library calls composed by
hand on the same batches and seeds, bit for bit (DESIGN.md 4.35)."""
import importlib.util
import math
import os

import numpy as np
import pytest
import torch

import oracle_cls
import oracle_monodepth as om
from deepi2p_b200 import classifier, frustum, handoff, icp, monodepth, network, pnp, synthetic

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H, W = 160, 512


def _load_script():
    spec = importlib.util.spec_from_file_location("evaluate_dataset", os.path.join(ROOT, "scripts",
                                                                                   "evaluate_dataset.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


ev = _load_script()


def _cloud(seed, S, N, boundary=False):
    """pc [S,3,N] f32 around a 160 x 512 camera, P [S,4,4] and K [S,3,3] f64; with boundary, exact pixels on u = 0,
    u = W - 1, v = H - 1, z = float32(0.1), behind the camera and in the last fine cell."""
    rng = np.random.default_rng(seed)
    z = rng.uniform(0.05, 40.0, (S, N))
    u = rng.uniform(-60.0, W + 60.0, (S, N))
    v = rng.uniform(-60.0, H + 60.0, (S, N))
    K = np.tile(np.array([[300.0, 0.0, 255.5], [0.0, 300.0, 79.5], [0.0, 0.0, 1.0]]), (S, 1, 1))
    x, y = (u - 255.5) * z / 300.0, (v - 79.5) * z / 300.0
    if boundary:
        K = np.tile(np.eye(3), (S, 1, 1))
        x, y = u * z, v * z
        k = min(N, 12)
        pu = np.array([0.0, W - 1.0, 10.0, W - 1.0, 0.0, W - 1.0, 480.0, 100.0, 100.0, 5.0, W - 1.0, W])[:k]
        pv = np.array([0.0, 0.0, H - 1.0, H - 1.0, H - 1.0, 128.0, 159.0, 50.0, 50.0, 5.0, H, 5.0])[:k]
        pz = np.array([1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, np.float32(0.1), -1.0, 0.0, 1.0, 1.0])[:k]
        x[:, :k], y[:, :k], z[:, :k] = pu * pz, pv * pz, pz
    pc = np.stack([x, y, z], 1).astype(np.float32)
    P = np.tile(np.eye(4), (S, 1, 1))
    if not boundary:
        a = rng.uniform(-0.05, 0.05, S)
        P[:, 0, 0], P[:, 0, 2], P[:, 2, 0], P[:, 2, 2] = np.cos(a), np.sin(a), -np.sin(a), np.cos(a)
        P[:, :3, 3] = rng.uniform(-0.5, 0.5, (S, 3))
    return pc, P, K


def _preds(seed, coarse_lab, fine_lab):
    rng = np.random.default_rng(seed)
    c = np.where(rng.random(coarse_lab.shape) < 0.7, coarse_lab, 1 - coarse_lab).astype(np.int8)
    f = np.where(rng.random(fine_lab.shape) < 0.5, fine_lab, rng.integers(0, 80, fine_lab.shape)).astype(np.int32)
    return c, f


def _dev(*a):
    return [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in a]


@pytest.mark.parametrize("S, N, boundary, fine", [(3, 1000, False, True), (1, 513, False, True),
                                                  (2, 20480, False, True), (4, 12, True, True), (2, 777, True, False),
                                                  (1, 1, False, False)])
def test_counts_equal_the_oracle_labels(cuda, S, N, boundary, fine):
    pc, P, K = _cloud(10 + N, S, N, boundary)
    cl, fl = oracle_cls.labels(pc, P, K, H, W)
    cp, fp = _preds(N, cl, fl)
    tpc, tP, tK, tcp, tfp = _dev(pc, P, K, cp, fp)
    out = classifier.prediction_accuracy(tpc, tP, tK, H, W, tcp, tfp if fine else None, return_labels=True)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(out["coarse_labels"].cpu().numpy(), cl)
    np.testing.assert_array_equal(out["fine_labels"].cpu().numpy(), fl)
    np.testing.assert_array_equal(out["n_inside"].cpu().numpy(), cl.astype(np.int64).sum(1))
    np.testing.assert_array_equal(out["coarse_correct"].cpu().numpy(), (cp == cl).sum(1))
    if fine:
        np.testing.assert_array_equal(out["fine_correct"].cpu().numpy(), ((fp == fl) & (fl >= 0)).sum(1))
    else:
        assert out["fine_correct"] is None
    if boundary:
        assert cl[:, :8].all() and not cl[:, 8:12].any() and (fl[:, 6] == 79).all()
    # without labels, from [S,3,4] poses: the same counts
    again = classifier.prediction_accuracy(tpc, tP[:, :3], tK, H, W, tcp, tfp if fine else None)
    assert "coarse_labels" not in again
    for k in ("n_inside", "coarse_correct") + (("fine_correct",) if fine else ()):
        assert torch.equal(again[k], out[k]), k


@pytest.mark.parametrize("fine", [True, False])
def test_counts_equal_classifier_loss_on_scores_with_these_argmaxes(cuda, fine):
    S, N = 5, 3000
    pc, P, K = _cloud(3, S, N)
    g = torch.Generator().manual_seed(4)
    coarse = torch.randn((S, 2, N), generator=g).cuda()
    fine_s = torch.randn((S, 80, N), generator=g).cuda() if fine else None
    tpc, tP, tK = _dev(pc, P, K)
    ref = classifier.classifier_loss(coarse, fine_s, tpc, tP, tK, H, W)
    cp, fp = network.predict(coarse, fine_s)
    got = classifier.prediction_accuracy(tpc, tP, tK, H, W, cp, fp)
    for k in ("n_inside", "coarse_correct") + (("fine_correct",) if fine else ()):
        assert torch.equal(got[k], ref[k]), k
    assert torch.equal(cp, ref["coarse_predictions"])


def test_graph_capture_and_replay(cuda):
    S, N = 4, 4096
    pc, P, K = _cloud(5, S, N)
    cl, fl = oracle_cls.labels(pc, P, K, H, W)
    cp, fp = _preds(6, cl, fl)
    tpc, tP, tK, tcp, tfp = _dev(pc, P, K, cp, fp)
    eager = classifier.prediction_accuracy(tpc, tP, tK, H, W, tcp, tfp)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        classifier.prediction_accuracy(tpc, tP, tK, H, W, tcp, tfp)          # warm-up off the capture
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        cap = classifier.prediction_accuracy(tpc, tP, tK, H, W, tcp, tfp)
    graph.replay()
    torch.cuda.synchronize()
    for k in ("n_inside", "coarse_correct", "fine_correct"):
        assert torch.equal(cap[k], eager[k]), k
    # new predictions in the captured buffers: the replay counts them
    cp2, fp2 = _preds(7, cl, fl)
    tcp.copy_(torch.from_numpy(cp2))
    tfp.copy_(torch.from_numpy(fp2))
    graph.replay()
    torch.cuda.synchronize()
    assert np.array_equal(cap["coarse_correct"].cpu().numpy(), (cp2 == cl).sum(1))
    assert np.array_equal(cap["fine_correct"].cpu().numpy(), ((fp2 == fl) & (fl >= 0)).sum(1))


# --------------------------------------------------------------------------------------------------------------------
# the script on seeded roots

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


@pytest.fixture(scope="module")
def nuscenes_root(tmp_path_factory):
    g = np.load(os.path.join(ROOT, "tests", "golden", "jpeg_small.npz"))
    so = np.concatenate([[0], np.cumsum(g["stream_lens"])])
    i = int(np.nonzero((g["shapes"][:, 0] == 900) & (g["shapes"][:, 1] == 1600))[0][0])
    root = str(tmp_path_factory.mktemp("nuscenes"))
    synthetic.write_nuscenes_dataroot(root, [(14, 6), (9, 4)], seed=2, jpeg=g["streams"][so[i]:so[i + 1]].tobytes())
    return root


@pytest.fixture(scope="module")
def ckpts(tmp_path_factory):
    d = tmp_path_factory.mktemp("ckpt")
    out = {}
    for name in ("kitti", "oxford", "nuscenes"):
        out[name] = str(d / f"{name}.pth")
        torch.save(synthetic.seeded_state_dict(network.KeypointDetector(**network.SHAPES[name]), 3), out[name])
    out["kitti_coarse"] = str(d / "kitti_coarse.pth")
    torch.save(synthetic.seeded_state_dict(network.KeypointDetector(**network.SHAPES["kitti"], fine=False), 3),
               out["kitti_coarse"])
    return out


@pytest.fixture(scope="module")
def depth_dir(tmp_path_factory):
    return om.write_checkpoint(str(tmp_path_factory.mktemp("monodepth")), seed=7)


EVERY = {"kitti": 13, "oxford": 6, "nuscenes": 1}          # 4, 4 and 2 samples
BATCH = {"kitti": 2, "oxford": 3, "nuscenes": 1}
SEED, INITS = 3, 8


def _roots(request, dataset):
    return request.getfixturevalue(f"{dataset}_root")


def _by_hand(dataset, root, ckpt, method, head, is_3d=False, depth_dir=None):
    """The script's loop spelled out with the library calls register_dir.py's methods make."""
    model = network.KeypointDetector(**network.SHAPES[dataset])
    network.load_checkpoint(model, ckpt)
    model = model.cuda()
    dm = monodepth.load_monodepth(depth_dir) if method == "icp" else None
    n, make = ev.batches(dataset, root, "v1.0-mini")
    items = list(range(0, n, EVERY[dataset]))
    rng = np.random.default_rng(SEED)
    P_pred, P_gt, cost, preds = [], [], [], []
    for b in range(0, len(items), BATCH[dataset]):
        pc, inten, sn, na, nb, P, img, K, _ = make(items[b:b + BATCH[dataset]], SEED * 100003 + b, rng)
        S, N = pc.shape[0], pc.shape[2]
        gt = np.tile(np.eye(4), (S, 1, 1))
        gt[:, :3] = P.cpu().numpy().astype(np.float64)
        if method == "lsq" and not is_3d:
            res = network.classify_and_register(model, pc, inten, sn, na, nb, img, K.numpy(), n_inits=INITS,
                                                seed=SEED, head=head)
            P_pred.append(res["P"].cpu().numpy())
            cost.append(res["cost"].cpu().numpy())
            c, f = res["coarse_pred"], res["fine_pred"]
        else:
            c, f = network.classify_batch(model, pc, inten, sn, na, nb, img, head=head)
            if method == "lsq":
                out = frustum.register_batch(pc.contiguous(), c, N, K.numpy(), H=img.shape[2], W=img.shape[3],
                                             n_inits=INITS, seed=SEED, is_2d=False)
                P_pred.append(out["P"].cpu().numpy())
                cost.append(out["cost"].cpu().numpy())
            elif method == "pnp":
                out = pnp.pnp_ransac_batch(pc.contiguous(), c, f, None, K.numpy(), img.shape[2], img.shape[3],
                                           scale=1 / 32.0, iterations=500, reproj_err=0.6, confidence=0.99,
                                           seed=SEED + b)
                P_pred.append(out["P"].cpu().numpy())
                cost.append(out["outlier_ratio"].cpu().numpy())
            else:
                src, n_pts = icp.pack_clouds(list(pc.cpu().numpy()))
                init = torch.from_numpy(icp.random_inits(S, INITS, SEED + b)).cuda()
                out = icp.register_images(src, n_pts, monodepth.images_from_batch(img), K.numpy(), gt, init, dm,
                                          max_corr_dist=1.0, max_iteration=30)
                P_pred.append(out["P"].cpu().numpy())
                cost.append(out["fitness"].cpu().numpy())
        P_gt.append(gt)
        preds.append((pc.cpu().numpy(), P.cpu().numpy(), K.numpy(), c.cpu().numpy(),
                      None if f is None else f.cpu().numpy()))
    return np.concatenate(P_pred), np.concatenate(P_gt), np.concatenate(cost), items, preds


def _run(tmp_path, capsys, dataset, root, ckpt, *extra):
    out = str(tmp_path / ("out_" + "_".join(extra).replace("-", "").replace("/", "_")))
    s = ev.main(["--dataset", dataset, "--root", root, "--checkpoint", ckpt, "--every", str(EVERY[dataset]),
                 "--batch", str(BATCH[dataset]), "--seed", str(SEED), "--inits", str(INITS), "--version", "v1.0-mini",
                 "--out", out, *extra])
    text = capsys.readouterr().out
    files = [np.load(os.path.join(out, f + "_all_np.npy")) for f in ("P_pred", "P_gt", "cost")]
    return s, text, files


def _expected_text(method, items, P_pred, P_gt, cost):
    if method == "icp":
        t, r = handoff.get_p_diff(P_pred, P_gt)
        ok = ((t < 2.0) & (r < 5.0)).astype(np.int32)
    else:
        e = frustum.pose_error_batch(P_pred, P_gt)
        t, r, ok = (e[k].cpu().numpy() for k in ("t_err", "r_err", "success"))
    fmt = {"lsq": "%06d - cost: %.1f, T: %.1f, R:%.1f", "pnp": "%06d - cost: %.2f, T: %.1f, R:%.1f",
           "icp": "%06d - fitness: %.1f, T: %.1f, R:%.1f"}[method]
    lines = [fmt % (it, cost[i], t[i], r[i]) for i, it in enumerate(items)]
    s = handoff.summarize(t, r, cost, ok)
    lines.append("RTE %.2f +- %.2f, RRE %.2f +- %.2f, success rate %.2f" % (
        s["rte_mean"], s["rte_sigma"], s["rre_mean"], s["rre_sigma"], s["success_rate"] * 100))
    return "\n".join(lines) + "\n", s


def _check(got, want, method):
    s, text, files = got
    P_pred, P_gt, cost, items, _ = want
    for g, w, name in zip(files, (P_pred, P_gt, cost), ("P_pred", "P_gt", "cost")):
        assert g.dtype == np.float64 and g.shape == w.shape and np.array_equal(g, w, equal_nan=True), name
    want_text, want_s = _expected_text(method, items, P_pred, P_gt, cost)
    assert text == want_text
    assert s == want_s or all(s[k] == want_s[k] or (math.isnan(s[k]) and math.isnan(want_s[k])) for k in want_s)
    assert len(items) >= 2 and P_pred.shape == (len(items), 4, 4)


def test_classify_and_register_is_classify_batch_then_register_batch(cuda, kitti_root, ckpts):
    model = network.KeypointDetector(**network.SHAPES["kitti"])
    network.load_checkpoint(model, ckpts["kitti"])
    model = model.cuda().train()
    n, make = ev.batches("kitti", kitti_root, None)
    pc, inten, sn, na, nb, P, img, K, _ = make([0, 13, 39], 9, np.random.default_rng(1))
    for head in network.HEADS:
        res = network.classify_and_register(model, pc, inten, sn, na, nb, img, K.numpy(), chunk=2, n_inits=INITS,
                                            seed=4, head=head)
        assert model.training
        c, f = network.classify_batch(model, pc, inten, sn, na, nb, img, chunk=2, head=head)
        assert model.training
        reg = frustum.register_batch(pc.contiguous(), c, pc.shape[2], K.numpy(), 160, 512, n_inits=INITS, seed=4)
        assert torch.equal(res["coarse_pred"], c) and torch.equal(res["fine_pred"], f), head
        for k in ("P", "cost", "degenerate"):
            assert torch.equal(res[k], reg[k]), (head, k)
        if head == "torch":
            model.eval()
            with torch.no_grad():
                ref = network.predict(*model(pc, inten, sn, na, nb, img))
            model.train()
            assert torch.equal(ref[0], c) and torch.equal(ref[1], f)
    with pytest.raises(ValueError, match="head must be one of"):
        network.classify_batch(model, pc, inten, sn, na, nb, img, head="cuda")
    with pytest.raises(ValueError, match="chunk must be >= 1"):
        network.classify_batch(model, pc, inten, sn, na, nb, img, chunk=0)
    with pytest.raises(ValueError, match="sn has 2 samples, pc has 3"):
        network.classify_batch(model, pc, inten, sn[:2], na, nb, img)
    model.eval()
    cm = network.KeypointDetector(**network.SHAPES["kitti"], fine=False)
    network.load_checkpoint(cm, ckpts["kitti_coarse"])
    c, f = network.classify_batch(cm.cuda(), pc, inten, sn, na, nb, img)
    assert f is None and c.dtype == torch.int8 and c.shape == pc.shape[::2]


@pytest.mark.parametrize("dataset", ["kitti", "oxford"])
@pytest.mark.parametrize("head", ["torch", "fused"])
def test_default_lsq_writes_what_classify_and_register_gives(cuda, request, tmp_path, capsys, ckpts, dataset, head):
    root = _roots(request, dataset)
    want = _by_hand(dataset, root, ckpts[dataset], "lsq", head)
    _check(_run(tmp_path, capsys, dataset, root, ckpts[dataset], "--head", head), want, "lsq")


@pytest.mark.parametrize("dataset", ["kitti", "oxford"])
@pytest.mark.parametrize("head", ["torch", "fused"])
@pytest.mark.parametrize("method", ["lsq3d", "pnp", "icp"])
def test_methods_write_what_the_library_calls_give(cuda, request, tmp_path, capsys, ckpts, depth_dir, dataset, head,
                                                   method):
    root = _roots(request, dataset)
    extra = {"lsq3d": ["--is-3d"], "pnp": ["--method", "pnp"],
             "icp": ["--method", "icp", "--depth-model", depth_dir]}[method]
    m = "lsq" if method == "lsq3d" else method
    want = _by_hand(dataset, root, ckpts[dataset], m, head, is_3d=method == "lsq3d", depth_dir=depth_dir)
    _check(_run(tmp_path, capsys, dataset, root, ckpts[dataset], "--head", head, *extra), want, m)


def test_nuscenes_lsq_with_accuracy(cuda, tmp_path, capsys, nuscenes_root, ckpts):
    want = _by_hand("nuscenes", nuscenes_root, ckpts["nuscenes"], "lsq", "torch")
    s, text, files = _run(tmp_path, capsys, "nuscenes", nuscenes_root, ckpts["nuscenes"], "--accuracy")
    lines = text.splitlines()
    _check((s, "\n".join(lines[:-1]) + "\n", files), want, "lsq")
    # the accuracy from the oracle labels of the same batches, with the script's arithmetic
    c_sum = f_sum = 0.0
    n = 0
    for pc, P, K, c, f in want[4]:
        cl, fl = oracle_cls.labels(pc, P, K, 160, 320)
        for b in range(pc.shape[0]):
            c_sum += np.mean((c[b] == cl[b]).astype(np.float64))
            m = cl[b] == 1
            f_sum += np.mean((f[b][m] == fl[b][m]).astype(np.float64)) if m.any() else math.nan
            n += 1
    assert n == 2
    want_c, want_f = c_sum / n, f_sum / n
    assert s["coarse_accuracy"] == want_c
    assert s["fine_accuracy"] == want_f or (math.isnan(want_f) and math.isnan(s["fine_accuracy"]))
    assert lines[-1] == "Overall coarse accuracy %.4f, fine accuracy %.4f" % (want_c, want_f)


def test_accuracy_of_a_coarse_only_checkpoint_and_pnp_refusal(cuda, tmp_path, capsys, kitti_root, ckpts,
                                                              monkeypatch):
    s, text, _ = _run(tmp_path, capsys, "kitti", kitti_root, ckpts["kitti_coarse"], "--accuracy")
    assert 0 <= s["coarse_accuracy"] <= 1 and math.isnan(s["fine_accuracy"])
    assert text.splitlines()[-1].startswith("Overall coarse accuracy ") and text.endswith("fine accuracy nan\n")
    built = []
    real = ev.batches
    monkeypatch.setattr(ev, "batches", lambda *a: built.append(a) or real(*a))
    with pytest.raises(SystemExit, match="coarse-only checkpoint"):
        ev.main(["--dataset", "kitti", "--root", kitti_root, "--checkpoint", ckpts["kitti_coarse"], "--method", "pnp"])
    assert not built
