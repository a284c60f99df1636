"""Write tests/golden/icp_small.npz: oracle_icp results on a few small ragged ICP frames.

    python tests/golden/make_icp_golden.py

Frames: make_icp_frame (KITTI shape) with the source subsampled to 2048 + 97 f points and the depth cloud to every
7th point, scale-calibrated by the true factor, 6 inits each (the first at the ground truth), max_iteration 12.
tests/test_icp_cpu.py checks that the oracle still reproduces them and tests/test_icp_gpu.py that the GPU does."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import oracle_icp  # noqa: E402
from deepi2p_b200 import icp, synthetic  # noqa: E402

N_FRAMES, I, MAX_IT = 3, 6, 12


def frames():
    out = []
    for f in range(N_FRAMES):
        fr = synthetic.make_icp_frame(300 + f, "kitti")
        src = fr["src"][:, ::10][:, :2048 + 97 * f]
        tgt = (fr["tgt"][:, ::7] / fr["scale"]).astype(np.float32)[:, :11000 + 513 * f]
        init = np.concatenate([fr["P_gt"][None], icp.random_inits(1, I - 1, seed=f)[0]])
        out.append((src, tgt, init))
    return out


def main():
    fs = frames()
    ns, ms = max(s.shape[1] for s, _, _ in fs), max(t.shape[1] for _, t, _ in fs)
    res = dict(n_frames=N_FRAMES, max_iteration=MAX_IT, n=np.array([s.shape[1] for s, _, _ in fs]),
               m=np.array([t.shape[1] for _, t, _ in fs]), src=np.zeros((N_FRAMES, 3, ns), np.float32),
               tgt=np.zeros((N_FRAMES, 3, ms), np.float32), init=np.stack([i for _, _, i in fs]),
               T=np.zeros((N_FRAMES, I, 4, 4)), fitness=np.zeros((N_FRAMES, I)), rmse=np.zeros((N_FRAMES, I)),
               stats=np.zeros((N_FRAMES, I, 2), np.int32), P=np.zeros((N_FRAMES, 4, 4)),
               best=np.zeros(N_FRAMES, np.int32))
    for f, (s, t, init) in enumerate(fs):
        res["src"][f, :, :s.shape[1]] = s
        res["tgt"][f, :, :t.shape[1]] = t
        r = oracle_icp.register_frame(s, t, init, max_iteration=MAX_IT, force_2d=True)
        for k in ("T", "fitness", "rmse", "stats", "P"):
            res[k][f] = r[k]
        res["best"][f] = r["best"]
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "icp_small.npz")
    np.savez_compressed(path, **res)
    print(path, res["best"], res["stats"][..., 0])


if __name__ == "__main__":
    main()
