"""Training on the device (deepi2p_b200/train.py): the captured step against the eager INTEGRATION.md 4d loop bit for
bit, dropout's graph-safe draws against eager's, the overlapped trainer against a serial loop, no host
synchronisation in a captured step, resume, learning on a tiny KITTI root, and the checkpoint round trip through
network.load_checkpoint and scripts/evaluate_dataset.py."""
import os
import sys

import numpy as np
import pytest
import torch

from deepi2p_b200 import classifier, kitti, network, synthetic, train

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def deterministic():
    flags = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    yield
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = flags


@pytest.fixture(scope="module")
def kitti_root(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("kitti"))
    synthetic.write_kitti_root(root, seqs=(0, 9, 10), n_frames=90)
    return root


def _model(seed=1, fine=True):
    m = network.KeypointDetector(**network.SHAPES["kitti"], fine=fine)
    m.load_state_dict(synthetic.seeded_state_dict(m, seed))
    return m.cuda()


def _inputs(S, seed):
    rng = np.random.default_rng(seed)
    smps = [synthetic.make_sample(seed + s, 20480, "kitti") for s in range(S)]
    pc = torch.from_numpy(np.stack([s["points"] for s in smps])).cuda()
    idx = torch.from_numpy(np.stack([rng.permutation(20480)[:256] for _ in range(S)])).cuda()
    nodes = torch.gather(pc, 2, idx.unsqueeze(1).expand(S, 3, 256))
    return dict(pc=pc, intensity=torch.from_numpy(rng.random((S, 1, 20480), dtype=np.float32)).cuda(),
                sn=torch.from_numpy(rng.standard_normal((S, 3, 20480), dtype=np.float32)).cuda(),
                node_a=nodes[:, :, :128].contiguous(), node_b=nodes[:, :, 128:].contiguous(),
                img=torch.from_numpy(rng.random((S, 3, 160, 512), dtype=np.float32)).cuda(),
                K=torch.from_numpy(np.stack([s["K"] for s in smps])).float().cuda(),
                P=torch.from_numpy(np.stack([s["P_gt"][:3] for s in smps])).float().cuda())


def _state(model, opt):
    out = {("model", k): v.clone() for k, v in model.state_dict().items()}
    for i, p in enumerate(model.parameters()):
        for k, v in opt.state[p].items():
            out[("adam", i, k)] = v.clone()
    return out


def _assert_same(a, b):
    assert a.keys() == b.keys()
    bad = [k for k in a if not torch.equal(a[k], b[k])]
    assert not bad, f"{len(bad)} tensors differ, first {bad[:3]}"


@pytest.mark.parametrize("dropout", [True, False])
def test_captured_step_is_the_eager_loop_bit_for_bit(deterministic, dropout):
    batches = [_inputs(2, 100 + k) for k in range(7)]

    def run(capture):
        model = _model()
        if not dropout:
            model.per_point_pn.layers[0].dropout = model.per_point_pn.layers[1].dropout = None
        opt = train.make_optimizer(model)
        static = {k: torch.empty_like(v) for k, v in batches[0].items()}
        stats, losses = torch.zeros(5, device="cuda"), []
        torch.cuda.manual_seed(7)
        graph = None
        for k, b in enumerate(batches):
            for n, v in b.items():
                static[n].copy_(v)
            if not capture or k < train.WARMUP_STEPS:
                stats.copy_(train._stats(train.train_step(model, opt, static)))
            else:
                if graph is None:
                    opt.zero_grad(set_to_none=True)
                    graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graph):
                        stats.copy_(train._stats(train.train_step(model, opt, static)))
                graph.replay()
            losses.append(stats.clone())
        torch.cuda.synchronize()
        return _state(model, opt), torch.stack(losses)

    s_eager, l_eager = run(False)
    s_graph, l_graph = run(True)
    assert torch.equal(l_eager, l_graph)
    _assert_same(s_eager, s_graph)


def test_graph_dropout_draws_equal_eager():
    x = torch.ones(4, 256, 2048, device="cuda")
    drop = torch.nn.Dropout(0.5).train()
    torch.cuda.manual_seed(3)
    eager = [drop(x).clone() for _ in range(3)]
    torch.cuda.manual_seed(3)
    out = torch.empty_like(x)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out.copy_(drop(x))
    graph = []
    for _ in range(3):
        g.replay()
        graph.append(out.clone())
    for a, b in zip(eager, graph):
        assert torch.equal(a, b)
    assert not torch.equal(eager[0], eager[1])


def test_captured_step_does_not_synchronise(kitti_root, tmp_path):
    src = train.batch_source("kitti", kitti_root, "train", seqs=(0,))
    t = train.Trainer(_model(), src, src, "kitti", str(tmp_path), batch_size=2, log=lambda s: None)
    order = train.epoch_order(src[0], 2, 0, 0)
    for b in range(train.WARMUP_STEPS + 1):
        seed, rng = train.batch_draws(0, 0, b)
        t._take(t._load(order[b], seed, rng, src[1]))
        t._step()
    assert t.graph is not None
    seed, rng = train.batch_draws(0, 0, train.WARMUP_STEPS + 1)
    ready = t._load(order[train.WARMUP_STEPS + 1], seed, rng, src[1])    # the assembly reads counts on its stream
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        t._take(ready)
        t._step()
        t._step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_overlapped_epoch_equals_serial_loop(deterministic, kitti_root, tmp_path):
    src = train.batch_source("kitti", kitti_root, "train", seqs=(0,))
    torch.cuda.manual_seed(11)
    t = train.Trainer(_model(), src, src, "kitti", str(tmp_path), batch_size=2, log=lambda s: None)
    seen = []
    take = t._take

    def record(ready):
        take(ready)
        seen.append({k: v.clone() for k, v in t.inputs.items()})
    t._take = record
    t.train_epoch(0)
    torch.cuda.synchronize()

    torch.cuda.manual_seed(11)
    model = _model()
    opt = train.make_optimizer(model)
    order = train.epoch_order(src[0], 2, 0, 0)
    assert len(seen) == len(order) > train.WARMUP_STEPS
    for b, items in enumerate(order):
        seed, rng = train.batch_draws(0, 0, b)
        vals = src[1](items, seed, rng, None)
        inp = {k: v.to("cuda", torch.float32) for k, v in zip(train.INPUT_FIELDS, vals[:8])}
        for k in train.INPUT_FIELDS:
            assert torch.equal(inp[k], seen[b][k]), (b, k)
        train.train_step(model, opt, inp)
    _assert_same(_state(t.model, t.optimizer), _state(model, opt))


def test_resume_equals_uninterrupted_run(deterministic, kitti_root, tmp_path):
    tr = train.batch_source("kitti", kitti_root, "train", seqs=(0,))
    te = train.batch_source("kitti", kitti_root, "val")

    def trainer(out):
        return train.Trainer(_model(), tr, te, "kitti", str(out), batch_size=2, epochs=2, log=lambda s: None)
    torch.cuda.manual_seed(5)
    a = trainer(tmp_path / "a")
    last_a = a.run()
    torch.cuda.manual_seed(5)
    b = trainer(tmp_path / "b")
    b.run(1)
    torch.cuda.manual_seed(999)                      # the resume file restores the device RNG
    c = trainer(tmp_path / "b")
    c.resume(str(tmp_path / "b" / "resume.pth"))
    assert c.epoch == 1 and c.step_count == tr[0] // 2
    last_c = c.run()
    assert os.path.basename(last_a) == os.path.basename(last_c)
    sa, sc = torch.load(last_a, weights_only=True), torch.load(last_c, weights_only=True)
    _assert_same(sa, sc)
    ra, rc = train.load_resume(os.path.join(a.out_dir, "resume.pth")), train.load_resume(
        os.path.join(c.out_dir, "resume.pth"))
    assert (ra["epoch"], ra["step"], ra["lr"]) == (rc["epoch"], rc["step"], rc["lr"])


def test_it_learns_and_the_checkpoint_round_trips(kitti_root, tmp_path):
    """Train on sequence 9 and test on sequence 10 in "val" mode (the camera keeps its heading, so the frustum can be
    learned from geometry alone; the synthetic images carry no cue): held-out coarse accuracy ends clearly above the
    all-outside baseline."""
    def source(root, seq):
        ds = kitti.KittiDataset(root, "val", seqs=(seq,))
        return len(ds), lambda items, seed, rng, stream: kitti.kitti_batch(ds, items, "val", seed, rng=rng,
                                                                           stream=stream)
    root = str(tmp_path / "root")
    synthetic.write_kitti_root(root, seqs=(9, 10), n_frames=200, seed=4)
    tr, te = source(root, 9), source(root, 10)
    lines = []
    t = train.Trainer(_model(3), tr, te, "kitti", str(tmp_path / "out"), batch_size=4, epochs=6, log=lines.append)
    last = t.run()
    inside = []
    for items in train.test_batches(te[0], 4):
        vals = te[1](items, 0, 0, None)
        pc, P, K = vals[0], vals[5].cuda(), vals[7].cuda().float()
        z = torch.zeros(pc.shape[0], 2, pc.shape[2], device="cuda")
        inside.append(classifier.classifier_loss(z, None, pc, P, K, 160, 512)["coarse_labels"].float().mean().item())
    baseline = 1.0 - float(np.mean(inside))
    acc = float(os.path.basename(last)[:-4].split("-")[-1])
    print("held-out coarse accuracy", acc, "all-outside baseline", baseline, lines[-6:])
    assert acc > baseline + 0.04

    m = network.KeypointDetector(**network.SHAPES["kitti"])
    network.load_checkpoint(m, last)
    sys.path.insert(0, os.path.join(ROOT, "scripts"))
    import evaluate_dataset
    s = evaluate_dataset.main(["--dataset", "kitti", "--root", kitti_root, "--checkpoint", last, "--every", "10",
                               "--batch", "4", "--inits", "8"])
    assert np.isfinite(s["rte_mean"])
