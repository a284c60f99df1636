"""Drop-in for the reference's torch extension `index_max` (models/index_max_ext/index_max.cpp:154-159).

forward_cuda and forward_cuda_shared_mem run the sm_90a segmented-argmax kernel on CUDA tensors.  The reference's
CPU entry points (forward_cpu, forward_multi_thread_cpu; index_max.cpp:73-112) take and return CPU tensors; this
framework has no CPU compute path, so they keep that CONTRACT (CPU tensors in, int32 CPU tensor out, identical
indices) but compute on the GPU: host -> device copy, the same kernel, device -> host copy.  Without a CUDA device
they raise, like everything else here.
"""
import torch

from deepi2p_b200.point_ops import index_max_forward as _fwd


def forward_cuda(data, index, K):
    return _fwd(data, index, K)


def forward_cuda_shared_mem(data, index, K):
    return _fwd(data, index, K)


def _via_gpu(data, index, K):
    if data.is_cuda or index.is_cuda:
        raise RuntimeError("forward_cpu takes CPU tensors (index_max.cpp:75-76); use forward_cuda for CUDA tensors")
    if not torch.cuda.is_available():
        raise RuntimeError("deepi2p_b200 has no CPU compute path: forward_cpu needs a CUDA device to run the kernel on")
    out = _fwd(data.contiguous().cuda(), index.contiguous().cuda(), K)
    return out.cpu()


def forward_cpu(data, index, K):
    return _via_gpu(data, index, K)


def forward_multi_thread_cpu(data, index, K, thread_num):
    # thread_num only sized the reference's std::thread pool (index_max.cpp:37-71); the result does not depend on it
    return _via_gpu(data, index, K)
