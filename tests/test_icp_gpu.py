"""Batched ICP on the GPU (deepi2p_b200.icp) against the CPU oracle (oracle_icp) and the stored golden results.

The oracle restates the kernels' arithmetic (no FMA, the same summation order, the same Jacobi SVD) and finds the
same exact nearest neighbours with a different tree, so every per-problem output (T, fitness, rmse, update steps,
n_corr) and every per-frame output (P, fitness, best) must be bit-identical."""
import os

import numpy as np
import pytest
import torch

import oracle_icp
from deepi2p_b200 import icp, synthetic

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "icp_small.npz")


def _gpu(frames, max_iteration=30, stream=None, out=None, force_2d=True):
    src, n = icp.pack_clouds([f[0] for f in frames])
    tgt, m = icp.pack_clouds([f[1] for f in frames])
    init = torch.from_numpy(np.stack([f[2] for f in frames])).cuda()
    o = icp.icp_register_batch(src, n, tgt, m, init, max_iteration=max_iteration, return_all=True, stream=stream,
                               out=out, force_2d=force_2d)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in o.items()}


def _check(frames, g, max_iteration=30, force_2d=True):
    for s, (src, tgt, init) in enumerate(frames):
        r = oracle_icp.register_frame(src, tgt, init, max_iteration=max_iteration, force_2d=force_2d)
        np.testing.assert_array_equal(g["stats"][s], r["stats"], err_msg=f"frame {s}")
        np.testing.assert_array_equal(g["T"][s], r["T"], err_msg=f"frame {s}")
        np.testing.assert_array_equal(g["fitness_all"][s], r["fitness"])
        np.testing.assert_array_equal(g["rmse_all"][s], r["rmse"])
        np.testing.assert_array_equal(g["P"][s], r["P"])
        assert g["fitness"][s] == r["fitness_best"] and g["best"][s] == r["best"], s


def _frame(seed, shape, I, init_seed=0):
    f = synthetic.make_icp_frame(seed, shape)
    sc = icp.calibrate_scale(f["src"], f["P_gt"], f["K"], f["H"], f["W"], f["tgt"])
    init = np.concatenate([f["P_gt"][None], icp.random_inits(1, I - 1, seed=init_seed)[0]])
    return f["src"], (f["tgt"] * sc).astype(np.float32), init


def test_golden_ragged_batch():
    g = np.load(GOLDEN)
    frames = [(g["src"][f][:, :int(g["n"][f])], g["tgt"][f][:, :int(g["m"][f])], g["init"][f])
              for f in range(int(g["n_frames"]))]
    out = _gpu(frames, max_iteration=int(g["max_iteration"]))
    for k, gk in (("T", "T"), ("fitness_all", "fitness"), ("rmse_all", "rmse"), ("stats", "stats"), ("P", "P"),
                  ("best", "best")):
        np.testing.assert_array_equal(out[k], g[gk], err_msg=k)


@pytest.mark.parametrize("shape", ["kitti", "oxford"])
def test_full_clouds_reduced_inits_match_oracle(shape):
    frames = [_frame(40 + s, shape, 6, init_seed=s) for s in range(2)]
    g = _gpu(frames)
    _check(frames, g)
    assert (g["stats"][..., 1] > 0).all()


def test_no_init_reaches_the_floor_and_zero_correspondences():
    src, tgt, init = _frame(7, "kitti", 3)
    far = init.copy()
    far[:, 0, 3] += 500.0                                  # nothing within 1 m: every problem has 0 correspondences
    ragged = (src[:, :5000], tgt[:, :30000], init)
    frames = [(src, tgt, far), ragged]
    g = _gpu(frames)
    _check(frames, g)
    assert (g["stats"][0, :, 1] == 0).all() and (g["stats"][0, :, 0] == 1).all()
    assert g["best"][0] == -1 and g["fitness"][0] == 0.001
    np.testing.assert_array_equal(g["P"][0], np.eye(4))
    np.testing.assert_array_equal(g["T"][0], far)


def test_dense_patch_in_the_target():
    """50k target points inside one cubic metre that the source surfaces cross: the index must stay exact."""
    src, tgt, init = _frame(9, "kitti", 4)
    q = init[0, :3, :3] @ src[:, 4000].astype(np.float64) + init[0, :3, 3]
    rng = np.random.default_rng(0)
    patch = (q[:, None] + rng.uniform(-0.5, 0.5, (3, 50000))).astype(np.float32)
    dup = np.repeat(patch[:, :16], 4, axis=1)                # exact duplicates: the lowest index must win
    frames = [(src, np.concatenate([tgt, patch, dup], axis=1), init)]
    g = _gpu(frames)
    _check(frames, g)


def test_full_size_oxford_60_inits_match_oracle():
    frames = [_frame(60 + s, "oxford", 60, init_seed=100 + s) for s in range(2)]
    g = _gpu(frames)
    _check(frames, g)


def test_out_reuse_and_stream_give_identical_results():
    frames = [_frame(20 + s, "kitti", 5, init_seed=s) for s in range(3)]
    a = _gpu(frames)
    src, n = icp.pack_clouds([f[0] for f in frames])
    tgt, m = icp.pack_clouds([f[1] for f in frames])
    init = torch.from_numpy(np.stack([f[2] for f in frames])).cuda()
    o = icp.icp_register_batch(src, n, tgt, m, init, return_all=True)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        icp.icp_register_batch(src, n, tgt, m, init, return_all=True, stream=st, out=o)
    st.synchronize()
    for k in a:
        np.testing.assert_array_equal(o[k].cpu().numpy(), a[k], err_msg=k)


def test_dropin_matches_the_batched_call():
    f = synthetic.make_icp_frame(33, "kitti")
    sc = icp.calibrate_scale(f["src"], f["P_gt"], f["K"], f["H"], f["W"], f["tgt"])
    tgt = f["tgt"] * sc
    P, fit = icp.icp_random_init(f["src"].astype(np.float64), tgt, 12, False, seed=5)
    frames = [(f["src"], tgt.astype(np.float32), icp.random_inits(1, 12, seed=5)[0])]
    g = _gpu(frames)
    np.testing.assert_array_equal(P, g["P"][0])
    assert fit == g["fitness"][0]
    with pytest.raises(ValueError):
        icp.icp_random_init(f["src"], tgt, 2, True)


def test_eval_counter():
    frames = [_frame(5, "kitti", 2)]
    with icp.count_evals() as c:
        g = _gpu(frames)
    assert c["queries"] >= 20480 * 2 * (1 + g["stats"][0, :, 0].min())
    assert c["evals"] > 0


def test_register_directory_icp_matches_the_batched_call(tmp_path):
    from deepi2p_b200 import handoff
    d, md, od = str(tmp_path / "data"), str(tmp_path / "monodepth"), str(tmp_path / "out")
    frames = synthetic.write_icp_handoff(d, md, [71, 72, 73], "kitti")
    res = handoff.register_directory_icp(d, md, 160, 512, n_inits=6, seed=3, batch=2, out_dir=od)
    for a, names in ((0, res["names"][:2]), (2, res["names"][2:])):
        fr = [frames[nm] for nm in names]
        tg = [f["tgt"] * icp.calibrate_scale(f["src"], f["P_gt"], f["K"], 160, 512, f["tgt"]) for f in fr]
        g = _gpu([(f["src"], t.astype(np.float32), i) for f, t, i in zip(fr, tg, icp.random_inits(len(fr), 6, 3 + a))])
        np.testing.assert_array_equal(res["P_pred"][a:a + len(fr)], g["P"])
        np.testing.assert_array_equal(res["cost"][a:a + len(fr)], g["fitness"])
    for k in ("P_pred_all_np", "P_gt_all_np", "cost_all_np"):
        assert os.path.exists(os.path.join(od, k + ".npy"))
    assert np.isfinite(res["t_err"]).all() and res["summary"]["n"] == 3
