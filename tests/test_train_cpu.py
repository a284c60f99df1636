"""The training loop's host logic (deepi2p_b200/train.py, scripts/train_classifier.py): the per-dataset defaults of
the three options.py files, the lr rule over 101 epochs, the epoch order, checkpoint names, the resume file, the test
pass's weighted means and the script's arguments.  No device needed."""
import os
import sys

import numpy as np
import pytest
import torch

from deepi2p_b200 import network, train

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import train_classifier  # noqa: E402


def test_defaults_are_the_options_files():
    # kitti/options.py, oxford/options.py, nuscenes_t/options.py; print intervals of each train_classifier.py
    assert train.DEFAULTS["kitti"] == dict(batch_size=8, lr_decay_step=20, print_interval=800, version="1.27")
    assert train.DEFAULTS["oxford"] == dict(batch_size=8, lr_decay_step=10, print_interval=600, version="0.1-fine")
    assert train.DEFAULTS["nuscenes"] == dict(batch_size=12, lr_decay_step=15, print_interval=1200, version="3.3")
    assert (train.LR, train.BETAS, train.WEIGHT_DECAY) == (0.001, (0.9, 0.999), 0.0)
    assert (train.LR_DECAY_SCALE, train.LR_CLIP, train.EPOCHS) == (0.5, 0.00001, 101)
    assert (train.coarse_loss_alpha(True), train.coarse_loss_alpha(False)) == (50.0, 1.0)
    assert set(train.DEFAULTS) == set(network.SHAPES)


def _reference_lrs(epochs, step):
    """train_classifier.py's loop with MMClassifer.update_learning_rate, line for line."""
    old_lr, out = 0.001, []
    for epoch in range(epochs):
        out.append(old_lr)
        if epoch % step == 0 and epoch > 0:
            lr = old_lr * 0.5
            if lr < 0.00001:
                lr = 0.00001
            old_lr = lr
    return out


@pytest.mark.parametrize("dataset", train.DATASETS)
def test_lr_schedule_is_the_reference_rule(dataset):
    step = train.DEFAULTS[dataset]["lr_decay_step"]
    got = train.lr_schedule(101, step)
    assert got == _reference_lrs(101, step)
    assert got[0] == got[step] == 0.001 and got[step + 1] == 0.0005


def test_lr_clip():
    got = train.lr_schedule(101, 5)
    assert got == _reference_lrs(101, 5)
    assert min(got) == 0.00001 and got[-1] == 0.00001
    assert train.decayed_lr(1.5e-5, 10, 5) == 0.00001
    assert train.decayed_lr(0.001, 0, 5) == 0.001


@pytest.mark.parametrize("n,B", [(20, 8), (16, 8), (7, 8), (100, 12), (1, 1)])
def test_epoch_order_is_a_seeded_permutation_with_drop_last(n, B):
    o = train.epoch_order(n, B, 3, 5)
    assert o.shape == (n // B, B)
    assert len(set(o.reshape(-1).tolist())) == o.size and (o.size == 0 or (o.min() >= 0 and o.max() < n))
    np.testing.assert_array_equal(o, train.epoch_order(n, B, 3, 5))
    np.testing.assert_array_equal(o.reshape(-1), np.random.default_rng([3, 5]).permutation(n)[:o.size])
    if n >= 8:
        assert not np.array_equal(train.epoch_order(n, B, 3, 6), o) or not np.array_equal(
            train.epoch_order(n, B, 4, 5), o)


def test_batch_draws_are_repeatable_and_distinct():
    s1, r1 = train.batch_draws(0, 1, 2)
    s2, r2 = train.batch_draws(0, 1, 2)
    assert s1 == s2 and r1.integers(1 << 30) == r2.integers(1 << 30)
    seeds = {train.batch_draws(0, e, b, t)[0] for e in range(3) for b in range(3) for t in (False, True)}
    assert len(seeds) == 18


def test_test_batches_keep_the_partial_last_batch():
    assert train.test_batches(10, 4) == [[0, 1, 2, 3], [4, 5, 6, 7], [8, 9]]
    assert train.test_batches(8, 4) == [[0, 1, 2, 3], [4, 5, 6, 7]]


def test_weighted_means_with_a_partial_batch():
    # batches of 4, 4 and 2 with per-batch means a, b, c: sum B * value / 10
    per_batch = [(4, 0.5), (4, 0.25), (2, 1.0)]
    sums = {"coarse_accuracy": sum(B * v for B, v in per_batch)}
    got = train.weighted_means(sums, sum(B for B, _ in per_batch))
    assert got["coarse_accuracy"] == pytest.approx((4 * 0.5 + 4 * 0.25 + 2 * 1.0) / 10)
    assert got["coarse_accuracy"] != pytest.approx(np.mean([v for _, v in per_batch]))


def test_checkpoint_name_is_the_reference_format():
    assert train.checkpoint_name("1.27", 1, 7, 0.8125) == "v1.27-gpu1-epoch7-0.812500.pth"
    assert train.checkpoint_name("0.1-fine", 0, 100, 1.0) == "v0.1-fine-gpu0-epoch100-1.000000.pth"


def test_format_losses():
    line = train.format_losses({"loss": 1.0, "coarse": 0.5, "fine": 0.5},
                               {"coarse_accuracy": 0.75, "fine_accuracy": 0.25}, 0.01)
    assert line == ("Per sample time: 0.0100 - loss: 1.0000, coarse: 0.5000, fine: 0.5000, coarse_accuracy: 0.7500, "
                    "fine_accuracy: 0.2500, ")
    assert train.format_losses({"loss": 1.0}, {"coarse_accuracy": 0.75}, 0.01, fine=False) == \
        "Per sample time: 0.010 - loss: 1.00, coarse_accuracy: 0.75, "


def test_resume_file_round_trips(tmp_path, monkeypatch):
    monkeypatch.setattr(torch.cuda, "get_rng_state", lambda dev=None: torch.arange(16, dtype=torch.uint8))
    model = torch.nn.Linear(3, 2)
    opt = torch.optim.Adam(model.parameters(), lr=0.001)
    model(torch.ones(4, 3)).sum().backward()
    opt.step()
    path = str(tmp_path / "resume.pth")
    train.save_resume(path, model, opt, 4, 123, 0.0005, 9, dict(best=0.5))
    st = train.load_resume(path)
    assert (st["epoch"], st["step"], st["lr"], st["seed"], st["extra"]) == (4, 123, 0.0005, 9, {"best": 0.5})
    assert torch.equal(st["cuda_rng"], torch.arange(16, dtype=torch.uint8))
    for k, v in model.state_dict().items():
        assert torch.equal(st["model"][k], v)
    opt2 = torch.optim.Adam(torch.nn.Linear(3, 2).parameters(), lr=0.001)
    opt2.load_state_dict(st["optimizer"])
    for a, b in zip(opt.state.values(), opt2.state.values()):
        for k in a:
            assert torch.equal(torch.as_tensor(a[k]), torch.as_tensor(b[k]))
    assert not os.path.exists(path + ".partial")


def test_script_arguments():
    a = train_classifier.parse_args(["--dataset", "kitti", "--root", "R", "--out", "O"])
    assert (a.dataset, a.root, a.out, a.epochs, a.batch, a.seed, a.version, a.coarse_only) == \
        ("kitti", "R", "O", 101, None, 0, None, False)
    assert (a.resnet_weights, a.record_dir, a.nuscenes_version, a.resume, a.store) == (None,) * 5
    a = train_classifier.parse_args(["--dataset", "kitti", "--root", "R", "--out", "O", "--epochs", "3", "--batch",
                                     "4", "--seed", "2", "--version", "x", "--coarse-only", "--resnet-weights", "w.pth",
                                     "--record-dir", "stride4-acc50-voxel0.4", "--resume", "O/resume.pth",
                                     "--store", "pinned"])
    assert (a.epochs, a.batch, a.seed, a.version, a.coarse_only, a.resnet_weights, a.record_dir, a.resume,
            a.store) == (3, 4, 2, "x", True, "w.pth", "stride4-acc50-voxel0.4", "O/resume.pth", "pinned")
    a = train_classifier.parse_args(["--dataset", "nuscenes", "--root", "R", "--out", "O", "--nuscenes-version",
                                     "v1.0-mini"])
    assert a.nuscenes_version == "v1.0-mini"
    for bad in (["--dataset", "oxford", "--record-dir", "x"], ["--dataset", "kitti", "--nuscenes-version", "v"],
                ["--dataset", "nuscenes", "--store", "cuda"], ["--dataset", "kitti", "--epochs", "0"],
                ["--dataset", "kitti", "--batch", "0"], ["--dataset", "waymo"], ["--dataset", "kitti", "--store", "x"]):
        with pytest.raises(SystemExit):
            train_classifier.parse_args(bad + ["--root", "R", "--out", "O"])


def test_batch_source_rejects_bad_settings(tmp_path):
    with pytest.raises(ValueError):
        train.batch_source("waymo", str(tmp_path), "train")
    with pytest.raises(ValueError):
        train.batch_source("kitti", str(tmp_path), "train", store="disk")
    with pytest.raises(ValueError):
        train.batch_source("oxford", str(tmp_path), "train", record_dir="x")
    with pytest.raises(ValueError):
        train.batch_source("nuscenes", str(tmp_path), "train", store="cuda")
