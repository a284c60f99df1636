"""Writes tests/golden/ref_kernels.npz: the outputs of the REFERENCE's own CUDA kernels
index_max.forward_cuda_shared_mem and ball_query.forward_cuda_shared_mem (compiled unmodified by
oracle/build_ref.py into oracle/_ref/) on the seeded inputs of tests/test_ops_gpu.py::test_against_reference_kernels.
Needs a CUDA device and a built oracle/_ref/:

    python oracle/build_ref.py && python tests/golden/make_ref_kernels_golden.py [OUT.npz]

Only the outputs are stored; the inputs are regenerated from their seeds by deepi2p_b200.synthetic
(the stored ball_query radius pins that generator).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import build_ref  # noqa: E402
from deepi2p_b200 import synthetic as syn  # noqa: E402

IM_SHAPE = dict(seed=77, B=8, C=32, N=20480, K=128)     # shipped model shape, B <= 1024, B*K*4 <= 48 KB
BQ_SHAPE = dict(seed=78, B=8, M=64, N=16384, K=64)


def main(out_path):
    ref_im = build_ref.load("index_max")
    ref_bq = build_ref.load("ball_query")
    s = IM_SHAPE
    data, index = syn.make_index_max_inputs(s["seed"], s["B"], s["C"], s["N"], s["K"])
    im = ref_im.forward_cuda_shared_mem(torch.from_numpy(data).cuda(), torch.from_numpy(index).cuda(), s["K"])
    s = BQ_SHAPE
    dist, radius = syn.make_ball_query_inputs(s["seed"], s["B"], s["M"], s["N"], s["K"])
    bq = ref_bq.forward_cuda_shared_mem(torch.from_numpy(dist).cuda(), radius, s["K"])
    torch.cuda.synchronize()
    # int32 outputs, stored as int16 (every index is < N <= 20480) to keep the file small
    np.savez_compressed(out_path, index_max_out=im.cpu().numpy().astype(np.int16),
                        ball_query_out=bq.cpu().numpy().astype(np.int16),
                        ball_query_radius=np.float64(radius), device=np.str_(torch.cuda.get_device_name()))
    print("wrote", out_path, tuple(im.shape), tuple(bq.shape))


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "ref_kernels.npz"))
