"""ICP on the GPU beyond the sizes of test_icp_gpu.py: a target deep enough for a 17-level index tree, and the
measurement entry points (explicit counters, the index build on its own).  Bit-exact against oracle_icp."""
import numpy as np
import pytest
import torch

import oracle_icp
from deepi2p_b200 import icp, synthetic

pytestmark = pytest.mark.gpu


def _frame(seed, shape, I, init_seed=0):
    f = synthetic.make_icp_frame(seed, shape)
    sc = icp.calibrate_scale(f["src"], f["P_gt"], f["K"], f["H"], f["W"], f["tgt"])
    init = np.concatenate([f["P_gt"][None], icp.random_inits(1, I - 1, seed=init_seed)[0]])
    return f["src"], (f["tgt"] * sc).astype(np.float32), init


def _gpu(frames, **kw):
    src, n = icp.pack_clouds([f[0] for f in frames])
    tgt, m = icp.pack_clouds([f[1] for f in frames])
    init = torch.from_numpy(np.stack([f[2] for f in frames])).cuda()
    o = icp.icp_register_batch(src, n, tgt, m, init, return_all=True, **kw)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in o.items()}, (src, n, tgt, m, init)


def test_large_target_deep_tree_matches_oracle():
    """More than 2^19 target points: the index tree has 17 levels (root level 16), next to a frame with a shallow tree
    in the same batch."""
    src, tgt, init = _frame(80, "oxford", 4)
    rng = np.random.default_rng(1)
    big = np.concatenate([tgt, (tgt + rng.normal(0, 0.01, tgt.shape)).astype(np.float32),
                          (tgt + rng.normal(0, 0.02, tgt.shape)).astype(np.float32)], axis=1)
    assert big.shape[1] > 1 << 19
    frames = [(src, big, init), _frame(81, "kitti", 4)]
    g, _ = _gpu(frames)
    for s, (sr, tg, ini) in enumerate(frames):
        r = oracle_icp.register_frame(sr, tg, ini)
        np.testing.assert_array_equal(g["stats"][s], r["stats"], err_msg=f"frame {s}")
        np.testing.assert_array_equal(g["T"][s], r["T"], err_msg=f"frame {s}")
        np.testing.assert_array_equal(g["fitness_all"][s], r["fitness"])
        np.testing.assert_array_equal(g["rmse_all"][s], r["rmse"])
        np.testing.assert_array_equal(g["P"][s], r["P"])
        assert g["fitness"][s] == r["fitness_best"] and g["best"][s] == r["best"], s
    assert (g["stats"][0, :, 1] > 0).any()


def test_explicit_counters_and_index_build():
    frames = [_frame(5, "kitti", 2)]
    a, (src, n, tgt, m, init) = _gpu(frames)
    cnt = torch.zeros(2, dtype=torch.int64, device="cuda")
    b, _ = _gpu(frames, counters=cnt)
    for k in a:
        np.testing.assert_array_equal(b[k], a[k], err_msg=k)
    queries, evals = cnt.cpu().tolist()
    assert queries == 20480 * int((a["stats"][0, :, 0] + 1).sum())
    assert evals > 0
    icp.build_index(tgt, m)
    torch.cuda.synchronize()
