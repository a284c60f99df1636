"""scripts/evaluate_dataset.py without a GPU: the option rules of its registration methods, and the overall
classification accuracy of visualize_and_save_data.py (:137-147, 216-217) from per-sample counts
(classifier.overall_accuracy) against the script's own arithmetic on oracle_cls labels, at the label rule's edges."""
import importlib.util
import math
import os
import warnings

import numpy as np
import pytest
import torch

import oracle_cls
from deepi2p_b200 import classifier

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H, W, SCALE = 160, 512, 32
W_F = W // SCALE


@pytest.fixture(scope="module")
def ev():
    spec = importlib.util.spec_from_file_location("evaluate_dataset", os.path.join(ROOT, "scripts",
                                                                                   "evaluate_dataset.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


BASE = ["--dataset", "kitti", "--root", "/nonexistent", "--checkpoint", "/nonexistent.pth"]


@pytest.mark.parametrize("extra, message", [
    (["--method", "icp"], "--method icp needs --depth-model"),
    (["--method", "lsq", "--depth-model", "m"], "--depth-model is only used by --method icp"),
    (["--method", "pnp", "--depth-model", "m"], "--depth-model is only used by --method icp"),
    (["--fine-scale", "0.0625"], "--fine-scale is only used by --method pnp"),
    (["--method", "icp", "--depth-model", "m", "--fine-scale", "0.0625"], "--fine-scale is only used by --method pnp"),
    (["--method", "pnp", "--is-3d"], "--is-3d is only used by --method lsq"),
    (["--method", "icp", "--depth-model", "m", "--is-3d"], "--is-3d is only used by --method lsq"),
    (["--method", "ransac"], "invalid choice"),
])
def test_option_errors(ev, capsys, extra, message):
    with pytest.raises(SystemExit) as e:
        ev.main(BASE + extra)
    assert e.value.code == 2
    assert message in capsys.readouterr().err


def _cloud(rng, n):
    """Camera-frame points (P = I, K = I, so u = x / z and v = y / z) with planted edges: u = 0, u = W - 1 and
    v = H - 1 exactly, z = float32(0.1), points behind the camera and at z = 0, and points in the last fine column and
    row."""
    z = rng.uniform(2.0, 30.0, n)
    u = rng.uniform(-40.0, W + 40.0, n)
    v = rng.uniform(-40.0, H + 40.0, n)
    u[0:4], v[0:4] = 0.0, [0.0, 50.0, H - 1.0, 200.0]
    u[4:8], v[4:8] = W - 1.0, [0.0, H - 1.0, 80.0, -1.0]
    u[8:12], v[8:12] = [10.0, 300.0, W - 1.0, W - 32.0], H - 1.0
    u[12:16], v[12:16] = [W - 20.0, W - 1.0, W - 32.0, 480.0], [H - 20.0, 128.0, H - 32.0, 130.0]
    u[16:20], v[16:20] = 100.0, 50.0
    z[16:20] = np.float32(0.1)
    z[20:24] = [-1.0, -5.0, -0.05, 0.0]
    x, y = u * z, v * z
    x[:16], y[:16], z[:16] = u[:16], v[:16], 1.0      # exact pixels
    return np.stack([x, y, z]).astype(np.float32)


def _scene(seed=0, S=4, n=300):
    rng = np.random.default_rng(seed)
    pc = np.stack([_cloud(rng, n) for _ in range(S)])
    pc[2, 2] = -np.abs(pc[2, 2]) - 1.0              # sample 2: every point behind the camera
    P = np.tile(np.eye(4), (S, 1, 1))
    K = np.tile(np.eye(3), (S, 1, 1))
    coarse, fine = oracle_cls.labels(pc, P, K, H, W, SCALE)
    return rng, pc, coarse, fine


def _script_overall(cp, cl, fp, fl):
    """visualize_and_save_data.py:137-147, 216-217 written out."""
    coarse_sum = fine_sum = 0
    counter = 0
    for b in range(cp.shape[0]):
        cur_c = np.mean((cp[b] == cl[b]).astype(np.float64))
        m = cl[b] == 1
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)       # np.mean([]) warns and returns NaN
            cur_f = np.mean((fp[b][m] == fl[b][m]).astype(np.float64))
        coarse_sum += cur_c
        fine_sum += cur_f
        counter += 1
    return coarse_sum / counter, fine_sum / counter


def _same(a, b):
    return (math.isnan(a) and math.isnan(b)) or a == b


def test_planted_edges_have_the_labels_they_were_planted_for():
    _, pc, coarse, fine = _scene()
    c, f = coarse[0], fine[0]
    assert c[0:3].all() and not c[3] and c[4:7].all() and not c[7] and c[8:12].all()
    assert f[11] == (W - 1) // SCALE + ((H - 1) // SCALE) * W_F == W_F * (H // SCALE) - 1
    assert f[12] == f[13] == f[14] == f[15] == f[11] and f[4] == W_F - 1 and f[9] == 9 + 4 * W_F and f[1] == W_F
    assert not c[20:24].any() and (f[20:24] == -1).all()
    assert c[16:20].all()                                      # z = float32(0.1) > 0.1
    assert coarse[2].sum() == 0 and coarse[[0, 1, 3]].sum(axis=1).min() > 50


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_overall_accuracy_follows_the_script(seed):
    rng, pc, cl, fl = _scene(seed)
    S, N = cl.shape
    cp = np.where(rng.random((S, N)) < 0.8, cl, 1 - cl).astype(np.int8)
    fp = np.where(rng.random((S, N)) < 0.6, fl, rng.integers(0, 80, (S, N))).astype(np.int32)
    n_inside = cl.astype(np.int64).sum(axis=1)
    c_ok = (cp == cl).sum(axis=1)
    f_ok = ((fp == fl) & (fl >= 0)).sum(axis=1)
    got = classifier.overall_accuracy(n_inside, c_ok, f_ok, N)
    want = _script_overall(cp, cl, fp, fl)
    assert math.isnan(want[1]) and math.isnan(got[1])            # sample 2 has no inside point
    assert _same(got[0], want[0]) and not math.isnan(got[0])
    keep = [0, 1, 3]                                              # without the empty sample the fine mean is finite
    got = classifier.overall_accuracy(n_inside[keep], c_ok[keep], f_ok[keep], N)
    want = _script_overall(cp[keep], cl[keep], fp[keep], fl[keep])
    assert got == want and 0 < got[1] < 1
    # counts as CPU tensors, as the script reads them back
    t = classifier.overall_accuracy(*(torch.from_numpy(np.asarray(a, np.int32)) for a in (n_inside[keep], c_ok[keep],
                                                                                         f_ok[keep])), N)
    assert t == got


def test_overall_accuracy_sums_in_sample_order():
    # counts whose per-sample sevenths sum to another float64 in the script's loop than in np.sum or math.fsum
    N = 7
    c_ok = [5, 4, 4, 7, 2, 6, 5, 0, 3, 6, 4, 0, 6, 5, 6, 1]
    got = classifier.overall_accuracy([1] * len(c_ok), c_ok, None, N)
    acc = 0
    for c in c_ok:
        acc += np.mean(np.array([1.0] * c + [0.0] * (N - c)))
    per = [c / N for c in c_ok]
    assert acc != np.sum(per) and acc != math.fsum(per)
    assert got[0] == acc / len(c_ok) and math.isnan(got[1])


def test_overall_accuracy_errors():
    with pytest.raises(ValueError, match="at least one"):
        classifier.overall_accuracy([], [], None, 4)
    with pytest.raises(ValueError, match="same number"):
        classifier.overall_accuracy([1, 2], [1], None, 4)


def test_prediction_accuracy_argument_errors():
    pc = torch.zeros((2, 3, 8))
    P, K = torch.eye(4).repeat(2, 1, 1), torch.eye(3).repeat(2, 1, 1)
    c8, f32 = torch.zeros((2, 8), dtype=torch.int8), torch.zeros((2, 8), dtype=torch.int32)
    with pytest.raises(RuntimeError, match="coarse_pred must be an int8"):
        classifier.prediction_accuracy(pc, P, K, H, W, f32)
    with pytest.raises(RuntimeError, match="fine_pred must be an int32"):
        classifier.prediction_accuracy(pc, P, K, H, W, c8, c8)
    with pytest.raises(RuntimeError, match="pc must be a float32"):
        classifier.prediction_accuracy(pc.double(), P, K, H, W, c8)
    with pytest.raises(RuntimeError, match="K must be"):
        classifier.prediction_accuracy(pc, P, K[:1], H, W, c8)
    with pytest.raises(ValueError, match="falls outside"):
        classifier.prediction_accuracy(pc, P, K, 160, 500, c8, f32, fine_scale=40)
    with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
        classifier.prediction_accuracy(pc, P, K, H, W, c8, f32)
