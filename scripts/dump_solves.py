"""Solve a seeded 6-DoF batch (64 clouds x 8 inits) and the 4096 x 1 configuration and save every output array, so that
two builds of the library (DIB_LIB_OVERRIDE) can be compared bit for bit; bench.py --dump-outputs covers the 4-DoF
headline batch only.

    python scripts/dump_solves.py OUT_DIR            # writes OUT_DIR/{6dof,4096x1}_<array>.npy
    python scripts/dump_solves.py --compare A B      # exit 1 unless every array of A equals that of B
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def run(out_dir):
    import torch
    from deepi2p_b200 import frustum
    from deepi2p_b200 import synthetic as syn
    os.makedirs(out_dir, exist_ok=True)
    for name, S, I, is_2d, n in (("6dof", 64, 8, False, 20480), ("4096x1", 4096, 1, True, 20480)):
        base = [syn.make_sample(500 + s, n) for s in range(min(S, 64))]
        smps = [base[s % len(base)] for s in range(S)]
        pts = torch.as_tensor(np.stack([s["points"] for s in smps]).astype(np.float32), device="cuda").contiguous()
        pred = torch.as_tensor(np.stack([s["pred"] for s in smps]).astype(np.int8), device="cuda").contiguous()
        prep = frustum.prepare_batch(pts, pred, n, I, seed=3)
        K = np.stack([np.asarray(s["K"], dtype=np.float64).reshape(9) for s in smps])
        res = frustum.solve_batch(prep["xyz"], prep["label"], prep["n_pts"], K, prep["init"], smps[0]["H"],
                                  smps[0]["W"], is_2d=is_2d, return_all=True)
        torch.cuda.synchronize()
        for k, v in res.items():
            np.save(os.path.join(out_dir, "%s_%s.npy" % (name, k)), v.cpu().numpy())


def compare(a, b):
    names = sorted(f for f in os.listdir(a) if f.endswith(".npy"))
    assert names == sorted(f for f in os.listdir(b) if f.endswith(".npy")), "different array sets"
    bad = [f for f in names if not np.array_equal(np.load(os.path.join(a, f)), np.load(os.path.join(b, f)),
                                                  equal_nan=True)]
    print("%d arrays compared, %d differ %s" % (len(names), len(bad), bad))
    return 1 if bad else 0


if __name__ == "__main__":
    if sys.argv[1] == "--compare":
        sys.exit(compare(sys.argv[2], sys.argv[3]))
    run(sys.argv[1])
