"""Host side of index_max / ball_query: torch tensors in, torch tensors out, kernels via the C ABI.

Mirrors the reference's extension modules (models/index_max_ext/index_max.cpp:119-159,
models/ball_query_ext/ball_query.cpp:23-48): same argument checks (CUDA + contiguous ->
RuntimeError), output allocated on the input's device, int32 outputs.  Unlike the reference the
kernels are launched on torch's *current* stream of the tensor's device, not the legacy default
stream (SURVEY.md 8b).
"""
import torch

from . import _native
from ._native import _stream_ptr, _workspace


def _check_input(t, name, dtype):
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"{name} must be a torch.Tensor")
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor/variable")
    if not t.is_contiguous():
        raise RuntimeError(f"{name} must be contiguous")
    if t.dtype != dtype:
        raise RuntimeError(f"{name} must have dtype {dtype}")


def index_max_forward(data, index, K):
    """out[b,c,k] = lowest n with index[b,n]==k attaining max data[b,c,n] over that segment if
    that max > -1000, else 0 (index_max_cuda.cu:30-62)."""
    _check_input(data, "data", torch.float32)
    _check_input(index, "index", torch.int32)
    if data.dim() != 3 or index.dim() != 2 or index.shape[0] != data.shape[0] or index.shape[1] != data.shape[2]:
        raise RuntimeError("data must be [B,C,N] and index [B,N]")
    lib = _native.load()
    B, C, N = data.shape
    K = int(K)
    with torch.cuda.device(data.device):
        out = torch.empty((B, C, K), dtype=torch.int32, device=data.device)
        rc = lib.index_max_forward(data.data_ptr(), index.data_ptr(), out.data_ptr(), B, C, N, K, _stream_ptr())
    _native.check(rc, "index_max_forward")
    return out


def ball_query_forward(node_to_point_dist, radius, K):
    """out[b,m,:] = first K indices n (ascending) with dist[b,m,n] <= radius; none -> 0; fewer ->
    cyclic repeat (ball_query_cuda.cu:11-50)."""
    _check_input(node_to_point_dist, "node_to_point_dist", torch.float32)
    if node_to_point_dist.dim() != 3:
        raise RuntimeError("node_to_point_dist must be [B,M,N]")
    lib = _native.load()
    B, M, N = node_to_point_dist.shape
    K = int(K)
    with torch.cuda.device(node_to_point_dist.device):
        out = torch.empty((B, M, K), dtype=torch.int32, device=node_to_point_dist.device)
        rc = lib.ball_query_forward(node_to_point_dist.data_ptr(), float(radius), out.data_ptr(), B, M, N, K,
                                    _stream_ptr())
    _native.check(rc, "ball_query_forward")
    return out


_xyz_ws = {}


def ball_query_xyz_forward(points, nodes, radius, K):
    """Grid-hash radius search from coordinates: points [B,3,N], nodes [B,3,M] float32 CUDA -> int32 [B,M,K]
    with the ball_query contract (first K indices in ascending n within radius; none -> 0; fewer -> cyclic).
    The contract is on SQUARED float32 distances: hit <=> ((dx*dx + dy*dy) + dz*dz) <= radius*radius (no fma), which
    is what ball_query_forward gives on a matrix of those squared distances with radius^2.  The reference pipeline
    thresholds torch.norm (the rounded square root) against radius; the two can differ for a distance within one
    float32 ulp of the radius.  Points with a NaN coordinate never hit."""
    _check_input(points, "points", torch.float32)
    _check_input(nodes, "nodes", torch.float32)
    if points.dim() != 3 or nodes.dim() != 3 or points.shape[1] != 3 or nodes.shape[1] != 3 or points.shape[0] != nodes.shape[0]:
        raise RuntimeError("points must be [B,3,N] and nodes [B,3,M]")
    lib = _native.load()
    B, _, N = points.shape
    M = nodes.shape[2]
    K = int(K)
    dev = points.device
    with torch.cuda.device(dev):
        ws = _workspace(_xyz_ws, lib.ball_query_xyz_workspace_bytes(B, N), dev)
        out = torch.empty((B, M, K), dtype=torch.int32, device=dev)
        rc = lib.ball_query_xyz_forward(points.data_ptr(), nodes.data_ptr(), float(radius), out.data_ptr(), B, M, N, K,
                                        ws.data_ptr(), ws.numel(), _stream_ptr())
    _native.check(rc, "ball_query_xyz_forward")
    return out


_ca_ws = {}


def cluster_assign_forward(pc, node, k=1, want_centers=True):
    """Nearest-node clustering of models/networks_pc.py:60-85 without its B x N x Ma intermediates.

    pc [B,3,N], node [B,3,M] float32 CUDA.  Returns dict(min_k_idx int32 [B,N,k] (nearest first), min_idx int32
    [B,N] (feed it to index_max_forward), count int32 [B,M] (mask_row_max = count > 0), cluster_mean [B,3,M],
    pc_centers [B,3,N], pc_decentered [B,3,N]).  Forward only, like the reference (everything here is
    detached there: :76,:82)."""
    _check_input(pc, "pc", torch.float32)
    _check_input(node, "node", torch.float32)
    if pc.dim() != 3 or node.dim() != 3 or pc.shape[1] != 3 or node.shape[1] != 3 or pc.shape[0] != node.shape[0]:
        raise RuntimeError("pc must be [B,3,N] and node [B,3,M]")
    lib = _native.load()
    B, _, N = pc.shape
    M = node.shape[2]
    k = int(k)
    dev = pc.device
    with torch.cuda.device(dev):
        ws = _workspace(_ca_ws, lib.cluster_assign_workspace_bytes(B, M), dev, floor=1 << 16)
        topk = torch.empty((B, N, k), dtype=torch.int32, device=dev)
        min_idx = torch.empty((B, N), dtype=torch.int32, device=dev)
        count = torch.empty((B, M), dtype=torch.int32, device=dev)
        mean = torch.empty((B, 3, M), dtype=torch.float32, device=dev)
        centers = torch.empty((B, 3, N), dtype=torch.float32, device=dev) if want_centers else None
        dec = torch.empty((B, 3, N), dtype=torch.float32, device=dev) if want_centers else None
        rc = lib.cluster_assign_forward(pc.data_ptr(), node.data_ptr(), B, N, M, k, topk.data_ptr(), min_idx.data_ptr(),
                                        count.data_ptr(), mean.data_ptr(),
                                        centers.data_ptr() if want_centers else 0,
                                        dec.data_ptr() if want_centers else 0, ws.data_ptr(), ws.numel(), _stream_ptr())
    _native.check(rc, "cluster_assign_forward")
    return dict(min_k_idx=topk, min_idx=min_idx, count=count, cluster_mean=mean, pc_centers=centers,
                pc_decentered=dec)


INTERP_MAX_K = 8
INTERP_MAX_NODES = 2048
_backward_ws = {}


def _backward_workspace(dev, need):
    """The fp64 slice partials of the interpolation's and the encoder ops' backwards, for a launch on the current
    stream."""
    return _workspace(_backward_ws, need, dev, floor=1 << 16)


def _check_interp_args(topk_idx, query, node, features):
    """Shape, dtype, bound and autograd checks first (they need no device), then device and layout."""
    for t, name in ((topk_idx, "topk_idx"), (query, "query"), (node, "node"), (features, "features")):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{name} must be a torch.Tensor")
        if t.dim() != 3:
            raise RuntimeError(f"{name} must have 3 dimensions")
    if topk_idx.dtype not in (torch.int32, torch.int64):
        raise RuntimeError("topk_idx must have dtype torch.int32 or torch.int64")
    for t, name in ((query, "query"), (node, "node"), (features, "features")):
        if t.dtype != torch.float32:
            raise RuntimeError(f"{name} must have dtype {torch.float32}")
    B, Nq, k = topk_idx.shape
    M = node.shape[2]
    if (query.shape[0] != B or query.shape[1] != 3 or query.shape[2] != Nq or node.shape[0] != B or node.shape[1] != 3
            or features.shape[0] != B or features.shape[2] != M):
        raise RuntimeError("topk_idx must be [B,Nq,k], query [B,3,Nq], node [B,3,M] and features [B,C,M]")
    if not 1 <= k <= INTERP_MAX_K:
        raise RuntimeError(f"topk_idx: need 1 <= k <= {INTERP_MAX_K}, got {k}")
    if not 1 <= M <= INTERP_MAX_NODES:
        raise RuntimeError(f"node: need 1 <= M <= {INTERP_MAX_NODES}, got {M}")
    if query.requires_grad or node.requires_grad:
        raise RuntimeError("upsample_by_interpolation has no gradient with respect to query or node: detach them")
    for t, name in ((topk_idx, "topk_idx"), (query, "query"), (node, "node"), (features, "features")):
        if not t.is_cuda:
            raise RuntimeError(f"{name} must be a CUDA tensor/variable")
        if not t.is_contiguous():
            raise RuntimeError(f"{name} must be contiguous")
        if t.device != features.device:
            raise RuntimeError(f"{name} must be on {features.device}")


class _Interpolation(torch.autograd.Function):
    @staticmethod
    def forward(ctx, topk_idx, query, node, features):
        lib = _native.load()
        B, Nq, k = topk_idx.shape
        C, M = features.shape[1], features.shape[2]
        dev = features.device
        with torch.cuda.device(dev):
            w = torch.empty((B, Nq, k), dtype=torch.float32, device=dev)
            idx = torch.empty((B, Nq, k), dtype=torch.int32, device=dev)
            out = torch.empty((B, C, Nq), dtype=torch.float32, device=dev)
            if out.numel():
                stream = _stream_ptr()
                rc = lib.interp_weights_f32(topk_idx.data_ptr(), topk_idx.element_size(), query.data_ptr(),
                                            node.data_ptr(), B, Nq, M, k, w.data_ptr(), idx.data_ptr(), stream)
                _native.check(rc, "interp_weights_f32")
                rc = lib.interp_forward_f32(features.data_ptr(), w.data_ptr(), idx.data_ptr(), B, C, Nq, M, k,
                                            out.data_ptr(), stream)
                _native.check(rc, "interp_forward_f32")
        ctx.save_for_backward(w, idx)
        ctx.shape = (B, C, Nq, M, k)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        if not ctx.needs_input_grad[3]:
            return None, None, None, None
        w, idx = ctx.saved_tensors
        B, C, Nq, M, k = ctx.shape
        dev = w.device
        # the kernel takes any batch stride with (channel, point) strides (Nq, 1): a channel slice of a torch.cat
        # gradient needs no copy
        grad_out = grad_out.float()
        if (C > 1 and grad_out.stride(1) != Nq) or (Nq > 1 and grad_out.stride(2) != 1):
            grad_out = grad_out.contiguous()
        lib = _native.load()
        with torch.cuda.device(dev):
            gF = torch.empty((B, C, M), dtype=torch.float32, device=dev)
            if gF.numel():
                stream = _stream_ptr()
                ws = _backward_workspace(dev, lib.interp_backward_workspace_bytes(B, C, Nq, M))
                bstride = grad_out.stride(0) if B > 1 else 0
                rc = lib.interp_backward_f32(grad_out.data_ptr(), bstride, w.data_ptr(), idx.data_ptr(), B, C, Nq, M,
                                             k, gF.data_ptr(), ws.data_ptr(), ws.numel(), stream)
                _native.check(rc, "interp_backward_f32")
        return None, None, None, gF


def upsample_by_interpolation(topk_idx, query, node, features):
    """Inverse-distance interpolation of node features onto query points: KeypointDetector.upsample_by_interpolation
    (models/networks_united.py:90-103, the same argument order without `self`) without its B x C x Nq x k tensors.

    topk_idx [B,Nq,k] int32 / int64 (e.g. cluster_assign_forward(...)["min_k_idx"] or a torch.topk result), query
    [B,3,Nq], node [B,3,M], features [B,C,M] float32 CUDA; 1 <= k <= 8, 1 <= M <= 2048.  Returns out [B,C,Nq] with
    out[b,c,n] = sum_j w_j features[b,c,idx_j], d_j = |query_n - node_{idx_j}|, w_j = 1 - d_j / sum_j d_j (DESIGN.md
    4.12).  As in the reference the weights sum to k - 1, k = 1 gives weight 0 and a zero distance sum gives NaN; a
    query point with any index outside [0, M) gets NaN in all C channels and no share of the feature gradient.
    Differentiable with respect to `features` only, with a deterministic gradient; query and node must not require
    grad."""
    _check_interp_args(topk_idx, query, node, features)
    return _Interpolation.apply(topk_idx, query, node, features)


KNN_MAX_K = 32
KNN_MAX_NODES = 2048


def _check_device(tensors, device):
    for t, name in tensors:
        if not t.is_cuda:
            raise RuntimeError(f"{name} must be a CUDA tensor/variable")
        if not t.is_contiguous():
            raise RuntimeError(f"{name} must be contiguous")
        if t.device != device:
            raise RuntimeError(f"{name} must be on {device}")


def _check_pool_args(features, min_idx, M):
    """Shape, dtype and bound checks first (they need no device), then device and layout."""
    for t, name in ((features, "features"), (min_idx, "min_idx")):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{name} must be a torch.Tensor")
    if features.dtype != torch.float32:
        raise RuntimeError(f"features must have dtype {torch.float32}")
    if min_idx.dtype != torch.int32:
        raise RuntimeError(f"min_idx must have dtype {torch.int32}")
    if features.dim() != 3 or min_idx.dim() != 2 or min_idx.shape[0] != features.shape[0] \
            or min_idx.shape[1] != features.shape[2]:
        raise RuntimeError("features must be [B,C,N] and min_idx [B,N]")
    if features.shape[2] < 1:
        raise RuntimeError("features: need N >= 1")
    if isinstance(M, bool) or int(M) != M or M < 1:
        raise RuntimeError(f"M must be an integer >= 1, got {M}")
    _check_device(((features, "features"), (min_idx, "min_idx")), features.device)


class _ClusterMaxPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, features, min_idx, M, broadcast):
        lib = _native.load()
        B, C, N = features.shape
        dev = features.device
        with torch.cuda.device(dev):
            sel = torch.empty((B, C, M), dtype=torch.int32, device=dev)
            mask = torch.empty((B, M), dtype=torch.float32, device=dev)
            pooled = torch.empty((B, C, M), dtype=torch.float32, device=dev)
            scattered = torch.empty((B, C, N), dtype=torch.float32, device=dev) if broadcast else None
            if B:
                rc = lib.cluster_pool_forward_f32(features.data_ptr(), min_idx.data_ptr(), B, C, N, M, sel.data_ptr(),
                                                  mask.data_ptr(), pooled.data_ptr(),
                                                  scattered.data_ptr() if broadcast and scattered.numel() else None,
                                                  _stream_ptr())
                _native.check(rc, "cluster_pool_forward_f32")
        ctx.set_materialize_grads(False)           # a missing pooled or scattered gradient stays None
        ctx.save_for_backward(min_idx, sel, mask)
        ctx.shape = (B, C, N, M)
        return (pooled, scattered) if broadcast else pooled

    @staticmethod
    def backward(ctx, grad_pooled, grad_scattered=None):
        if not ctx.needs_input_grad[0] or (grad_pooled is None and grad_scattered is None):
            return None, None, None, None
        min_idx, sel, mask = ctx.saved_tensors
        B, C, N, M = ctx.shape
        dev = sel.device
        if grad_pooled is not None:
            grad_pooled = grad_pooled.float().contiguous()
        if grad_scattered is not None:
            # any batch stride with (channel, point) strides (N, 1): a channel slice of a torch.cat gradient needs
            # no copy
            grad_scattered = grad_scattered.float()
            if (C > 1 and grad_scattered.stride(1) != N) or (N > 1 and grad_scattered.stride(2) != 1):
                grad_scattered = grad_scattered.contiguous()
        lib = _native.load()
        with torch.cuda.device(dev):
            gF = torch.empty((B, C, N), dtype=torch.float32, device=dev)
            if gF.numel():
                stream = _stream_ptr()
                ws, ws_bytes = None, 0
                if grad_scattered is not None:
                    ws = _backward_workspace(dev, lib.cluster_pool_backward_workspace_bytes(B, C, N, M))
                    ws_bytes = ws.numel()
                gs_ptr = grad_scattered.data_ptr() if grad_scattered is not None else None
                bstride = grad_scattered.stride(0) if grad_scattered is not None and B > 1 else 0
                rc = lib.cluster_pool_backward_f32(grad_pooled.data_ptr() if grad_pooled is not None else None, gs_ptr,
                                                   bstride, min_idx.data_ptr(), sel.data_ptr(), mask.data_ptr(), B, C,
                                                   N, M, gF.data_ptr(), ws.data_ptr() if ws is not None else None,
                                                   ws_bytes, stream)
                _native.check(rc, "cluster_pool_backward_f32")
        return gF, None, None, None


def cluster_max_pool(features, min_idx, M, broadcast=False):
    """SO-Net masked max-pool of PCEncoder.forward (models/networks_pc.py:88-104) in one op, with a deterministic
    feature gradient (DESIGN.md 4.16).

    features [B,C,N] float32 and min_idx [B,N] int32 (cluster_assign_forward's) CUDA, M >= 1 segments.  Returns pooled
    [B,C,M] = features[b,c,sel] * mask[b,m], sel = index_max_forward(features, min_idx, M) and mask[b,m] = 1.0 where
    some point has min_idx == m (else 0.0: an empty segment gives features[b,c,0] * 0.0, -0.0 or NaN included).  With
    broadcast=True returns (pooled, scattered), scattered [B,C,N] = pooled[b,c,min_idx[b,n]].  A point whose min_idx
    is outside [0, M) joins no segment, gets NaN in every channel of scattered and no share of the gradient.
    Differentiable with respect to `features`: fp64 sums in an order fixed by the shape, no float atomics."""
    _check_pool_args(features, min_idx, M)
    return _ClusterMaxPool.apply(features, min_idx, int(M), bool(broadcast))


def _check_knn_args(query, database, features, K):
    """Shape, dtype, bound and autograd checks first (they need no device), then device and layout."""
    for t, name in ((query, "query"), (database, "database"), (features, "features")):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{name} must be a torch.Tensor")
        if t.dtype != torch.float32:
            raise RuntimeError(f"{name} must have dtype {torch.float32}")
        if t.dim() != 3:
            raise RuntimeError(f"{name} must have 3 dimensions")
    B, N = database.shape[0], database.shape[2]
    if query.shape[0] != B or query.shape[1] != 3 or database.shape[1] != 3 or features.shape[0] != B \
            or features.shape[2] != N:
        raise RuntimeError("query must be [B,3,M], database [B,3,N] and features [B,C,N]")
    if isinstance(K, bool) or int(K) != K or not 1 <= K <= KNN_MAX_K:
        raise RuntimeError(f"K: need 1 <= K <= {KNN_MAX_K}, got {K}")
    if not 1 <= N <= KNN_MAX_NODES:
        raise RuntimeError(f"database: need 1 <= N <= {KNN_MAX_NODES}, got {N}")
    if K > N:
        raise RuntimeError(f"K: need K <= N, got K = {K} and N = {N}")
    if query.requires_grad or database.requires_grad:
        raise RuntimeError("knn_group has no gradient with respect to query or database: detach them")
    _check_device(((query, "query"), (database, "database"), (features, "features")), features.device)


class _KnnGroup(torch.autograd.Function):
    @staticmethod
    def forward(ctx, query, database, features, K):
        lib = _native.load()
        B, C, N = features.shape
        M = query.shape[2]
        dev = features.device
        with torch.cuda.device(dev):
            idx = torch.empty((B, M, K), dtype=torch.int32, device=dev)
            grouped = torch.empty((B, 3 + C, M, K), dtype=torch.float32, device=dev)
            if idx.numel():
                rc = lib.knn_group_forward_f32(query.data_ptr(), database.data_ptr(), features.data_ptr(), B, C, M, N,
                                               K, idx.data_ptr(), grouped.data_ptr(), _stream_ptr())
                _native.check(rc, "knn_group_forward_f32")
        ctx.mark_non_differentiable(idx)
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(idx)
        ctx.shape = (B, C, M, N, K)
        return idx, grouped

    @staticmethod
    def backward(ctx, grad_idx, grad_grouped):
        if not ctx.needs_input_grad[2]:
            return None, None, None, None
        idx, = ctx.saved_tensors
        B, C, M, N, K = ctx.shape
        dev = idx.device
        if grad_grouped is None:                   # grouped took no part in the loss: a zero gradient, not materialised
            return None, None, None, None
        # any batch stride with (row, query, neighbour) strides (M * K, K, 1).  There are always 3 + C >= 3 rows, so the
        # row stride is checked whatever M and K are (at M = K = 1 a slice of a cat along dim 3 has row stride != 1)
        grad_grouped = grad_grouped.float()
        if grad_grouped.stride(1) != M * K or (M > 1 and grad_grouped.stride(2) != K) \
                or (K > 1 and grad_grouped.stride(3) != 1):
            grad_grouped = grad_grouped.contiguous()
        lib = _native.load()
        with torch.cuda.device(dev):
            gF = torch.empty((B, C, N), dtype=torch.float32, device=dev)
            if gF.numel():
                stream = _stream_ptr()
                ws = _backward_workspace(dev, lib.knn_group_backward_workspace_bytes(B, C, M, N, K))
                bstride = grad_grouped.stride(0) if B > 1 else 0
                rc = lib.knn_group_backward_f32(grad_grouped.data_ptr() if M else None, bstride, idx.data_ptr(), B, C,
                                                M, N, K, gF.data_ptr(), ws.data_ptr(), ws.numel(), stream)
                _native.check(rc, "knn_group_backward_f32")
        return None, None, gF, None


def knn_group(query, database, features, K):
    """Node kNN grouping of GeneralKNNFusionModule.forward (models/layers_pc.py:793-807) in one op, with a
    deterministic feature gradient (DESIGN.md 4.16).

    query [B,3,M], database [B,3,N], features [B,C,N] float32 CUDA; 1 <= K <= 32, K <= N <= 2048.  Returns (knn_idx
    [B,M,K] int32, grouped [B,3+C,M,K]): knn_idx holds the K nearest database nodes of each query, nearest first, by
    cluster_assign's key (f32 ((dx*dx + dy*dy) + dz*dz) without fma, ties -> lower index, +inf after finite keys, NaN
    after +inf); grouped rows 0-2 are database[idx] - query and rows 3 onward features[idx], the tensor
    layers_pc.py:807 concatenates.  Differentiable with respect to `features` only (fp64 sums in an order fixed by the
    shape, no float atomics); query and database must not require grad, as the reference detaches both."""
    _check_knn_args(query, database, features, K)
    return _KnnGroup.apply(query, database, features, int(K))


FUSION_MAX_BATCH = 65535
FUSION_MAX_ROWS = 32 * 65535      # C and P: 65535 row tiles of 32 in the kernel's grid


def _check_fusion_args(img_features, attention):
    """Type, dimension, dtype, shape and bound checks first (they need no device), then device and layout."""
    for t, name in ((img_features, "img_features"), (attention, "attention")):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{name} must be a torch.Tensor")
        if t.dim() != 3:
            raise RuntimeError(f"{name} must have 3 dimensions")
        if t.dtype != torch.float32:
            raise RuntimeError(f"{name} must have dtype {torch.float32}")
    B, C, P = img_features.shape
    M = attention.shape[2]
    if attention.shape[0] != B or attention.shape[1] != P:
        raise RuntimeError("img_features must be [B,C,P] and attention [B,P,M]")
    if not 1 <= B <= FUSION_MAX_BATCH:
        raise RuntimeError(f"img_features: need 1 <= B <= {FUSION_MAX_BATCH}, got {B}")
    if min(C, P, M) < 1:
        raise RuntimeError(f"need C, P, M >= 1, got C = {C}, P = {P}, M = {M}")
    if max(C, P) > FUSION_MAX_ROWS or M > 2 ** 31 - 1:
        raise RuntimeError(f"need C, P <= {FUSION_MAX_ROWS} and M < 2^31, got C = {C}, P = {P}, M = {M}")
    _check_device(((img_features, "img_features"), (attention, "attention")), img_features.device)


class _AttentionFusion(torch.autograd.Function):
    @staticmethod
    def forward(ctx, img_features, attention):
        lib = _native.load()
        B, C, P = img_features.shape
        M = attention.shape[2]
        dev = img_features.device
        with torch.cuda.device(dev):
            out = torch.empty((B, C, M), dtype=torch.float32, device=dev)
            rc = lib.attn_fusion_forward_f32(img_features.data_ptr(), attention.data_ptr(), B, C, P, M, out.data_ptr(),
                                             _stream_ptr())
        _native.check(rc, "attn_fusion_forward_f32")
        ctx.set_materialize_grads(False)           # a missing output gradient stays None
        ctx.save_for_backward(img_features, attention)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        need_F, need_A = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if grad_out is None or not (need_F or need_A):
            return None, None
        F, A = ctx.saved_tensors
        B, C, P = F.shape
        M = A.shape[2]
        dev = F.device
        # any batch stride with (channel, node) strides (M, 1): a channel slice of a torch.cat gradient needs no copy
        grad_out = grad_out.float()
        if (C > 1 and grad_out.stride(1) != M) or (M > 1 and grad_out.stride(2) != 1):
            grad_out = grad_out.contiguous()
        lib = _native.load()
        with torch.cuda.device(dev):
            gF = torch.empty((B, C, P), dtype=torch.float32, device=dev) if need_F else None
            gA = torch.empty((B, P, M), dtype=torch.float32, device=dev) if need_A else None
            bstride = grad_out.stride(0) if B > 1 else 0
            rc = lib.attn_fusion_backward_f32(grad_out.data_ptr(), bstride, F.data_ptr(), A.data_ptr(), B, C, P, M,
                                              gF.data_ptr() if need_F else None, gA.data_ptr() if need_A else None,
                                              _stream_ptr())
        _native.check(rc, "attn_fusion_backward_f32")
        return gF, gA


def attention_fusion(img_features, attention):
    """Attention-weighted image features of KeypointDetector.forward (models/networks_united.py:149-150,172-174,
    torch.mean(img_features.unsqueeze(3) * attention.unsqueeze(1), dim=2)) without its B x C x P x M product
    (DESIGN.md 4.17).

    img_features [B,C,P] (the feature map's .view(B, C, -1)) and attention [B,P,M] float32 CUDA, contiguous, on one
    device.  Returns out [B,C,M], out[b,c,m] = float((sum over p ascending of F[b,c,p] * A[b,p,m]) / P), one fp64
    accumulator per output over the exact products, so the result does not depend on tiling, batch composition or the
    TF32 flags.  Differentiable with respect to both inputs with the same rule (sums over m for img_features, over c
    for attention); an input that needs no gradient costs nothing in the backward."""
    _check_fusion_args(img_features, attention)
    return _AttentionFusion.apply(img_features, attention)


def interpolation_weights(topk_idx, query, node):
    """The weights half of upsample_by_interpolation: topk_idx [B,Nq,k], query [B,3,Nq], node [B,3,M] -> (w float32
    [B,Nq,k], idx int32 [B,Nq,k]) with w_j = 1 - d_j / sum_j d_j; a point with an index outside [0, M) gets w = NaN and
    idx = -1 in every slot.  pointwise_mlp takes these for an interpolated source.  No gradient."""
    _check_interp_args(topk_idx, query, node, query.new_empty((query.shape[0], 1, node.shape[2])))
    lib = _native.load()
    B, Nq, k = topk_idx.shape
    dev = query.device
    with torch.cuda.device(dev):
        w = torch.empty((B, Nq, k), dtype=torch.float32, device=dev)
        idx = torch.empty((B, Nq, k), dtype=torch.int32, device=dev)
        if w.numel():
            rc = lib.interp_weights_f32(topk_idx.data_ptr(), topk_idx.element_size(), query.data_ptr(),
                                        node.data_ptr(), B, Nq, node.shape[2], k, w.data_ptr(), idx.data_ptr(),
                                        _stream_ptr())
            _native.check(rc, "interp_weights_f32")
    return w, idx


MLP_MAX_SOURCES = 4
MLP_MAX_LAYERS = 3
MLP_MAX_WIDTH = 256
MLP_MAX_IN = 1024
MLP_MAX_BATCH = 65535
_MLP_SRC, _MLP_LAYER = 8, 4       # int64 slots per source / layer (DIB_MLP_SRC, DIB_MLP_LAYER)
_mlp_ws = {}


def _mlp_source_shapes(sources):
    """[(C, M, k)] per source (M = k = 0: dense) and (B, N), from shapes alone; ValueError on a mismatch."""
    if not isinstance(sources, (list, tuple)) or not 1 <= len(sources) <= MLP_MAX_SOURCES:
        raise ValueError(f"sources: need a list of 1 to {MLP_MAX_SOURCES} sources")
    spec, B, N = [], None, None
    for i, s in enumerate(sources):
        if isinstance(s, torch.Tensor):
            if s.dim() != 3:
                raise ValueError(f"sources[{i}]: a dense source must be [B,C,N]")
            b, C, n, M, k = s.shape[0], s.shape[1], s.shape[2], 0, 0
        else:
            if not isinstance(s, (list, tuple)) or len(s) != 3 or not all(isinstance(t, torch.Tensor) for t in s):
                raise ValueError(f"sources[{i}]: need a tensor [B,C,N] or a tuple (features [B,C,M], w, idx)")
            F, w, idx = s
            if F.dim() != 3 or w.dim() != 3 or idx.shape != w.shape or w.shape[0] != F.shape[0]:
                raise ValueError(f"sources[{i}]: need features [B,C,M] and w, idx [B,N,k]")
            b, C, M, n, k = F.shape[0], F.shape[1], F.shape[2], w.shape[1], w.shape[2]
            if not 1 <= k <= INTERP_MAX_K:
                raise ValueError(f"sources[{i}]: need 1 <= k <= {INTERP_MAX_K}, got {k}")
            if not 1 <= M <= INTERP_MAX_NODES:
                raise ValueError(f"sources[{i}]: need 1 <= M <= {INTERP_MAX_NODES}, got {M}")
        if C < 1:
            raise ValueError(f"sources[{i}]: need at least one channel")
        if B is None:
            B, N = b, n
        elif (b, n) != (B, N):
            raise ValueError(f"sources[{i}] has B, N = {b}, {n}; sources[0] has {B}, {N}")
        spec.append((C, M, k))
    if sum(c for c, _, _ in spec) > MLP_MAX_IN:
        raise ValueError(f"the concatenated input has {sum(c for c, _, _ in spec)} rows, more than {MLP_MAX_IN}")
    if N < 1 or not 1 <= B <= MLP_MAX_BATCH:
        raise ValueError(f"need N >= 1 and 1 <= B <= {MLP_MAX_BATCH}, got B = {B}, N = {N}")
    return spec, B, N


def _mlp_layer_widths(layers, c_in):
    """[(C_out, relu)] of a list of (W [C_out,C_in], b [C_out] or None, relu); ValueError on a bad width."""
    if not isinstance(layers, (list, tuple)) or not 1 <= len(layers) <= MLP_MAX_LAYERS:
        raise ValueError(f"layers: need a list of 1 to {MLP_MAX_LAYERS} layers")
    meta = []
    for i, layer in enumerate(layers):
        if not isinstance(layer, (list, tuple)) or len(layer) != 3:
            raise ValueError(f"layers[{i}]: need (W, b, relu)")
        W, b, relu = layer
        if not isinstance(W, torch.Tensor) or W.dim() != 2 or W.shape[1] != c_in:
            raise ValueError(f"layers[{i}]: W must be [C_out, {c_in}]")
        if not 1 <= W.shape[0] <= MLP_MAX_WIDTH:
            raise ValueError(f"layers[{i}]: need 1 <= C_out <= {MLP_MAX_WIDTH}, got {W.shape[0]}")
        if b is not None and (not isinstance(b, torch.Tensor) or tuple(b.shape) != (W.shape[0],)):
            raise ValueError(f"layers[{i}]: b must be [{W.shape[0]}] or None")
        c_in = W.shape[0]
        meta.append((c_in, bool(relu)))
    return meta


def _mlp_tables(spec, meta):
    import numpy as np
    src = np.zeros((len(spec), _MLP_SRC), dtype=np.int64)
    for i, (C, M, k) in enumerate(spec):
        src[i, 2], src[i, 3], src[i, 6] = C, M, k
    lay = np.zeros((len(meta), _MLP_LAYER), dtype=np.int64)
    for i, (C, relu) in enumerate(meta):
        lay[i, 2], lay[i, 3] = C, int(relu)
    return src, lay


class PackedPointwiseMLP:
    """The layers of one pointwise_mlp chain in the kernel's order on the device (weights rounded to TF32 once), for
    sources of the widths `spec` = [(C, M, k)] (M = k = 0 for a dense source).  pack_pointwise_mlp builds it."""

    def __init__(self, spec, meta, packed):
        self.spec, self.meta, self.packed = list(spec), list(meta), packed


def pack_pointwise_mlp(spec, layers):
    """Pack `layers` = [(W [C_out,C_in] float32 CUDA, b [C_out] or None, relu)] for sources of the widths `spec`
    (as PackedPointwiseMLP.spec); pointwise_mlp does this itself when given the raw layers."""
    spec = [tuple(int(v) for v in s) for s in spec]
    meta = _mlp_layer_widths(layers, sum(c for c, _, _ in spec))
    dev = layers[0][0].device
    keep = []
    for W, b, _ in layers:
        for t in (W, b):
            if t is None:
                continue
            if t.requires_grad and torch.is_grad_enabled():
                raise RuntimeError("pointwise_mlp has no backward: call it under torch.no_grad() or detach the layers")
            if not t.is_cuda or t.device != dev or t.dtype != torch.float32:
                raise RuntimeError("the layers must be float32 CUDA tensors on one device")
        keep.append((W.detach().contiguous(), None if b is None else b.detach().contiguous()))
    src, lay = _mlp_tables(spec, meta)
    for i, (W, b) in enumerate(keep):
        lay[i, 0], lay[i, 1] = W.data_ptr(), 0 if b is None else b.data_ptr()
    lib = _native.load()
    need = lib.pointwise_mlp_packed_bytes(src.ctypes.data, len(spec), lay.ctypes.data, len(meta))
    if need == 0:
        raise ValueError("pointwise_mlp: " + lib.dib_last_error().decode("utf-8", "replace"))
    with torch.cuda.device(dev):
        packed = torch.empty(need // 4, dtype=torch.float32, device=dev)
        rc = lib.pointwise_mlp_pack_f32(src.ctypes.data, len(spec), lay.ctypes.data, len(meta), packed.data_ptr(), need,
                                        _stream_ptr())
    _native.check(rc, "pointwise_mlp_pack_f32")
    return PackedPointwiseMLP(spec, meta, packed)


def pointwise_mlp(sources, layers, output="activations", c_split=None, return_scores=False):
    """A chain of one to three 1x1-convolution layers y = act(W x + b) over every point, in one kernel, for inference
    (DESIGN.md 4.21): the PointNets the classifier applies per point, with BatchNorm already folded into W and b
    (network.fold_pointnet) and the input concatenation never built.

    sources: 1 to 4 of, in the order of layer 1's input rows, a dense float32 CUDA tensor [B,C,N] (a channel slice of
    a wider contiguous tensor is read in place) or a tuple (features [B,C,M], w [B,N,k], idx [B,N,k]) whose rows are
    the interpolation upsample_by_interpolation computes (w, idx from interpolation_weights; k <= 8, M <= 2048, a
    point with idx = -1 has NaN rows).  At most 1024 rows in all.  layers: [(W [C_out,C_in], b [C_out] or None, relu)]
    with every C_out in [1, 256], or a PackedPointwiseMLP.

    output="activations" returns the last layer [B,C_out,N].  output="argmax" returns (int8 [B,N], int32 [B,N] or
    None): the arg-max over channels [0, c_split) and over [c_split, C_out) (None when that range is empty) by
    torch.max's rule, so c_split = 2 is network.predict; with return_scores=True the scores [B,C_out,N] come third.

    The products run on the tensor cores in TF32 with float32 accumulation whatever torch's TF32 flags say: weights,
    source values and the activations between layers are rounded to TF32 (nearest, ties away from zero); bias, ReLU
    (NaN stays NaN) and the arg-max are float32.  No backward: an input that requires grad raises RuntimeError unless
    grad mode is off.  Shape and bound errors raise ValueError before anything is launched."""
    spec, B, N = _mlp_source_shapes(sources)
    if isinstance(layers, PackedPointwiseMLP):
        if layers.spec != spec:
            raise ValueError(f"the layers were packed for sources {layers.spec}, got {spec}")
        packed = layers
    else:
        packed = None
    meta = packed.meta if packed is not None else _mlp_layer_widths(layers, sum(c for c, _, _ in spec))
    C_out = meta[-1][0]
    if output not in ("activations", "argmax"):
        raise ValueError(f"output must be 'activations' or 'argmax', got {output!r}")
    if output == "argmax":
        if c_split is None or isinstance(c_split, bool) or int(c_split) != c_split \
                or not 1 <= c_split <= min(C_out, 128):
            raise ValueError(f"c_split: need an integer in [1, min(C_out, 128)] with C_out = {C_out}, got {c_split}")
        c_split = int(c_split)
    elif c_split is not None or return_scores:
        raise ValueError("c_split and return_scores go with output='argmax'")
    flat = [t for s in sources for t in ((s,) if isinstance(s, torch.Tensor) else s)]
    dev = flat[0].device
    for t in flat:
        if t.requires_grad and torch.is_grad_enabled():
            raise RuntimeError("pointwise_mlp has no backward: call it under torch.no_grad() or detach the inputs")
        if not t.is_cuda:
            raise RuntimeError("pointwise_mlp: every source must be a CUDA tensor")
        if t.device != dev:
            raise RuntimeError(f"pointwise_mlp: every source must be on {dev}")
    src, lay = _mlp_tables(spec, meta)
    keep = []
    for i, s in enumerate(sources):
        if isinstance(s, torch.Tensor):
            if s.dtype != torch.float32:
                raise RuntimeError(f"sources[{i}] must have dtype {torch.float32}")
            C = s.shape[1]
            if (N > 1 and s.stride(2) != 1) or (C > 1 and s.stride(1) != N) or (B > 1 and s.stride(0) < C * N):
                s = s.contiguous()
            keep.append(s)
            src[i, 0], src[i, 1] = s.data_ptr(), s.stride(0) if B > 1 else C * N
        else:
            F, w, idx = s
            if F.dtype != torch.float32 or w.dtype != torch.float32 or idx.dtype != torch.int32:
                raise RuntimeError(f"sources[{i}] must be (float32 features, float32 w, int32 idx)")
            F, w, idx = F.contiguous(), w.contiguous(), idx.contiguous()
            keep.append((F, w, idx))
            src[i, 0], src[i, 1], src[i, 4], src[i, 5] = F.data_ptr(), F.shape[1] * F.shape[2], w.data_ptr(), \
                idx.data_ptr()
    if packed is None:
        packed = pack_pointwise_mlp(spec, layers)
    if packed.packed.device != dev:
        raise RuntimeError(f"the layers must be on {dev}")
    lib = _native.load()
    with torch.cuda.device(dev):
        stream = _stream_ptr()
        need = lib.pointwise_mlp_workspace_bytes(src.ctypes.data, len(spec), lay.ctypes.data, len(meta), B)
        ws = _workspace(_mlp_ws, need, dev, floor=0) if need else None
        want_out = output == "activations" or return_scores
        out = torch.empty((B, C_out, N), dtype=torch.float32, device=dev) if want_out else None
        pred_a = torch.empty((B, N), dtype=torch.int8, device=dev) if output == "argmax" else None
        pred_b = torch.empty((B, N), dtype=torch.int32, device=dev) if output == "argmax" and c_split < C_out else None
        rc = lib.pointwise_mlp_f32(src.ctypes.data, len(spec), lay.ctypes.data, len(meta), packed.packed.data_ptr(),
                                   packed.packed.numel() * 4, B, N, c_split or 0,
                                   out.data_ptr() if out is not None else None,
                                   pred_a.data_ptr() if pred_a is not None else None,
                                   pred_b.data_ptr() if pred_b is not None else None,
                                   ws.data_ptr() if ws is not None else None, ws.numel() if ws is not None else 0,
                                   stream)
    _native.check(rc, "pointwise_mlp_f32")
    del keep
    if output == "activations":
        return out
    return (pred_a, pred_b, out) if return_scores else (pred_a, pred_b)


KNN_FUSION_MAX_WIDTH = 512
KNN_FUSION_MAX_SIDE = 3
_mlp_max_ws = {}


def _chain_widths(layers, c_in, name, lo=1):
    """[(C_out, relu)] of lo to 3 layers (W [C_out,C_in], b [C_out] or None, relu), widths in [1, 512]; ValueError
    otherwise.  The first layer takes c_in rows."""
    if not isinstance(layers, (list, tuple)) or not lo <= len(layers) <= KNN_FUSION_MAX_SIDE:
        raise ValueError(f"{name}: need a list of {lo} to {KNN_FUSION_MAX_SIDE} layers")
    meta = []
    for i, layer in enumerate(layers):
        if not isinstance(layer, (list, tuple)) or len(layer) != 3:
            raise ValueError(f"{name}[{i}]: need (W, b, relu)")
        W, b, relu = layer
        if not isinstance(W, torch.Tensor) or W.dim() != 2 or W.shape[1] != c_in:
            raise ValueError(f"{name}[{i}]: W must be [C_out, {c_in}]")
        if not 1 <= W.shape[0] <= KNN_FUSION_MAX_WIDTH:
            raise ValueError(f"{name}[{i}]: need 1 <= C_out <= {KNN_FUSION_MAX_WIDTH}, got {W.shape[0]}")
        if b is not None and (not isinstance(b, torch.Tensor) or tuple(b.shape) != (W.shape[0],)):
            raise ValueError(f"{name}[{i}]: b must be [{W.shape[0]}] or None")
        c_in = W.shape[0]
        meta.append((c_in, bool(relu)))
    return meta


class PackedChain:
    """The layers of one knn_fusion or pointwise_mlp_max chain in the kernel's order on the device (weights rounded
    to TF32 once), for c_in input rows: meta = [(C_out, relu)] over every layer, n_before of them before the per-node
    max (all of them for pointwise_mlp_max).  pack_knn_fusion and pack_pointwise_mlp_max build it."""

    def __init__(self, kind, c_in, meta, n_before, packed):
        self.kind, self.c_in, self.meta, self.n_before, self.packed = kind, c_in, list(meta), n_before, packed


def _pack_chain(kind, c_in, layers, meta, n_before):
    dev = layers[0][0].device
    keep = []
    for W, b, _ in layers:
        for t in (W, b):
            if t is None:
                continue
            if t.requires_grad and torch.is_grad_enabled():
                raise RuntimeError(f"{kind} has no backward: call it under torch.no_grad() or detach the layers")
            if not t.is_cuda or t.device != dev or t.dtype != torch.float32:
                raise RuntimeError("the layers must be float32 CUDA tensors on one device")
        keep.append((W.detach().contiguous(), None if b is None else b.detach().contiguous()))
    _, lay = _mlp_tables([], meta)
    for i, (W, b) in enumerate(keep):
        lay[i, 0], lay[i, 1] = W.data_ptr(), 0 if b is None else b.data_ptr()
    lib = _native.load()
    if kind == "knn_fusion":
        args = (c_in, lay.ctypes.data, n_before, len(meta) - n_before)
        need = lib.knn_fusion_packed_bytes(*args)
    else:
        args = (c_in, lay.ctypes.data, len(meta))
        need = lib.pointwise_mlp_max_packed_bytes(*args)
    if need == 0:
        raise ValueError(f"{kind}: " + lib.dib_last_error().decode("utf-8", "replace"))
    with torch.cuda.device(dev):
        packed = torch.empty(need // 4, dtype=torch.float32, device=dev)
        stream = _stream_ptr()
        if kind == "knn_fusion":
            rc = lib.knn_fusion_pack_f32(*args, packed.data_ptr(), need, stream)
        else:
            rc = lib.pointwise_mlp_max_pack_f32(*args, packed.data_ptr(), need, stream)
    _native.check(rc, kind + "_pack_f32")
    del keep
    return PackedChain(kind, c_in, meta, n_before, packed)


def _knn_fusion_meta(C, before, after):
    if not isinstance(C, int) or not 1 <= C <= KNN_FUSION_MAX_WIDTH - 3:
        raise ValueError(f"knn_fusion: need 1 <= C <= {KNN_FUSION_MAX_WIDTH - 3} feature channels, got {C}")
    mb = _chain_widths(before, 3 + C, "before")
    ma = _chain_widths(after, 2 * mb[-1][0], "after")
    return mb + ma, len(mb)


def pack_knn_fusion(C, before, after):
    """Pack the folded layers of a kNN fusion module for C feature channels (network.fold_knn_fusion's lists) once;
    knn_fusion does this itself when given the raw layers."""
    meta, n_before = _knn_fusion_meta(int(C), before, after)
    return _pack_chain("knn_fusion", 3 + int(C), list(before) + list(after), meta, n_before)


def knn_fusion(query, database, features, K, layers, return_idx=False):
    """The node kNN module (GeneralKNNFusionModule.forward, layers_pc.py:793-818) in one kernel, for inference
    (DESIGN.md 4.26): group the K nearest database nodes of each query as knn_group does, the "before" layers, the max
    over the K neighbours, the "after" layers over the concatenation [max; x], the max over K again.  No [B,C,M,K]
    tensor is built: the max half of the first after layer is projected once per node and added like a bias.

    query [B,3,M], database [B,3,N], features [B,C,N] float32 CUDA; 1 <= K <= 32, K <= N <= 2048, 3 + C <= 512.
    layers: (before, after), each a list of 1 to 3 (W [C_out,C_in], b [C_out] or None, relu) with every C_out in
    [1, 512] (BatchNorm folded: network.fold_knn_fusion), the first after layer taking 2 C_b rows (max first), or a
    PackedChain from pack_knn_fusion.  Returns out [B,C_out,M], and knn_group's knn_idx [B,M,K] int32 with
    return_idx=True.

    TF32 tensor-core products with float32 accumulation whatever torch's TF32 flags say: weights, the grouped values
    and the activations between layers are rounded to TF32 (nearest, ties away from zero); bias, ReLU (NaN stays NaN)
    and both maxes are float32, a NaN among a node's K columns giving NaN.  No backward: an input that requires grad
    raises RuntimeError unless grad mode is off.  Shape and bound errors raise ValueError before anything is
    launched."""
    for t, name in ((query, "query"), (database, "database"), (features, "features")):
        if not isinstance(t, torch.Tensor) or t.dim() != 3:
            raise ValueError(f"{name} must be a 3-D tensor")
    B, C, N = features.shape
    M = query.shape[2]
    if query.shape[:2] != (B, 3) or database.shape != (B, 3, N):
        raise ValueError("query must be [B,3,M], database [B,3,N] and features [B,C,N]")
    if isinstance(K, bool) or int(K) != K or not 1 <= K <= KNN_MAX_K:
        raise ValueError(f"K: need 1 <= K <= {KNN_MAX_K}, got {K}")
    K = int(K)
    if not 1 <= N <= KNN_MAX_NODES or K > N:
        raise ValueError(f"database: need K <= N <= {KNN_MAX_NODES}, got K = {K}, N = {N}")
    if not 1 <= B <= MLP_MAX_BATCH or M < 1:
        raise ValueError(f"need 1 <= B <= {MLP_MAX_BATCH} and M >= 1, got B = {B}, M = {M}")
    if isinstance(layers, PackedChain):
        if layers.kind != "knn_fusion" or layers.c_in != 3 + C:
            raise ValueError(f"the layers were packed as {layers.kind} for {layers.c_in} input rows, need 3 + C = "
                             f"{3 + C}")
        packed = layers
        meta, n_before = packed.meta, packed.n_before
    else:
        if not isinstance(layers, (list, tuple)) or len(layers) != 2:
            raise ValueError("layers: need (before, after) or a PackedChain")
        meta, n_before = _knn_fusion_meta(C, *layers)
        packed = None
    for t in (query, database, features):
        if t.requires_grad and torch.is_grad_enabled():
            raise RuntimeError("knn_fusion has no backward: call it under torch.no_grad() or detach the inputs")
        if t.dtype != torch.float32:
            raise RuntimeError("query, database and features must be float32")
        if not t.is_cuda or t.device != features.device:
            raise RuntimeError("query, database and features must be CUDA tensors on one device")
    dev = features.device
    query, database, features = query.contiguous(), database.contiguous(), features.contiguous()
    if packed is None:
        packed = pack_knn_fusion(C, *layers)
    if packed.packed.device != dev:
        raise RuntimeError(f"the layers must be on {dev}")
    _, lay = _mlp_tables([], meta)
    lib = _native.load()
    with torch.cuda.device(dev):
        idx = torch.empty((B, M, K), dtype=torch.int32, device=dev)
        out = torch.empty((B, meta[-1][0], M), dtype=torch.float32, device=dev)
        rc = lib.knn_fusion_f32(query.data_ptr(), database.data_ptr(), features.data_ptr(), B, C, M, N, K,
                                lay.ctypes.data, n_before, len(meta) - n_before, packed.packed.data_ptr(),
                                packed.packed.numel() * 4, idx.data_ptr(), out.data_ptr(), _stream_ptr())
    _native.check(rc, "knn_fusion_f32")
    return (out, idx) if return_idx else out


def pack_pointwise_mlp_max(c_in, layers):
    """Pack `layers` = [(W [C_out,C_in] float32 CUDA, b [C_out] or None, relu)] for c_in input rows once;
    pointwise_mlp_max does this itself when given the raw layers."""
    c_in = int(c_in)
    if not 1 <= c_in <= KNN_FUSION_MAX_WIDTH:
        raise ValueError(f"pointwise_mlp_max: need 1 <= input rows <= {KNN_FUSION_MAX_WIDTH}, got {c_in}")
    return _pack_chain("pointwise_mlp_max", c_in, layers, _chain_widths(layers, c_in, "layers"), len(layers))


def pointwise_mlp_max(sources, layers):
    """A chain of one to three 1x1-convolution layers over the columns of each sample, then the max over all of them,
    in one kernel and a fixed-order reduction, for inference (DESIGN.md 4.26): final_pointnet + torch.max(dim=2) of
    the point encoder, with the input concatenation and the [B,C_out,N] activations never built.

    sources: 1 to 4 dense float32 CUDA tensors [B,C,N] (a channel slice of a wider contiguous tensor is read in
    place), at most 512 rows in all.  layers: [(W [C_out,C_in], b [C_out] or None, relu)], every C_out in [1, 512],
    or a PackedChain from pack_pointwise_mlp_max.  Returns [B,C_out,1] float32.  pointwise_mlp's TF32 rule; the max
    is float32 with torch.max's NaN rule.  No backward; shape and bound errors raise ValueError before any launch."""
    if not isinstance(sources, (list, tuple)) or not all(isinstance(s, torch.Tensor) for s in sources):
        raise ValueError("sources: need a list of dense [B,C,N] tensors")
    spec, B, N = _mlp_source_shapes(sources)
    c_in = sum(c for c, _, _ in spec)
    if c_in > KNN_FUSION_MAX_WIDTH:
        raise ValueError(f"the concatenated input has {c_in} rows, more than {KNN_FUSION_MAX_WIDTH}")
    if isinstance(layers, PackedChain):
        if layers.kind != "pointwise_mlp_max" or layers.c_in != c_in:
            raise ValueError(f"the layers were packed as {layers.kind} for {layers.c_in} input rows, got {c_in}")
        packed, meta = layers, layers.meta
    else:
        packed, meta = None, _chain_widths(layers, c_in, "layers")
    dev = sources[0].device
    for t in sources:
        if t.requires_grad and torch.is_grad_enabled():
            raise RuntimeError("pointwise_mlp_max has no backward: call it under torch.no_grad() or detach the inputs")
        if not t.is_cuda or t.device != dev:
            raise RuntimeError(f"pointwise_mlp_max: every source must be a CUDA tensor on {dev}")
        if t.dtype != torch.float32:
            raise RuntimeError("pointwise_mlp_max: every source must be float32")
    src, lay = _mlp_tables(spec, meta)
    keep = []
    for i, s in enumerate(sources):
        C = s.shape[1]
        if (N > 1 and s.stride(2) != 1) or (C > 1 and s.stride(1) != N) or (B > 1 and s.stride(0) < C * N):
            s = s.contiguous()
        keep.append(s)
        src[i, 0], src[i, 1] = s.data_ptr(), s.stride(0) if B > 1 else C * N
    if packed is None:
        packed = pack_pointwise_mlp_max(c_in, layers)
    if packed.packed.device != dev:
        raise RuntimeError(f"the layers must be on {dev}")
    C_out = meta[-1][0]
    lib = _native.load()
    with torch.cuda.device(dev):
        stream = _stream_ptr()
        need = lib.pointwise_mlp_max_workspace_bytes(C_out, B, N)
        ws = _workspace(_mlp_max_ws, need, dev, floor=0)
        out = torch.empty((B, C_out, 1), dtype=torch.float32, device=dev)
        rc = lib.pointwise_mlp_max_f32(src.ctypes.data, len(spec), lay.ctypes.data, len(meta), packed.packed.data_ptr(),
                                       packed.packed.numel() * 4, B, N, out.data_ptr(), ws.data_ptr(), ws.numel(),
                                       stream)
    _native.check(rc, "pointwise_mlp_max_f32")
    del keep
    return out


NODE_MLP_MAX_WIDTH = 1024         # dense input rows and every layer
NODE_MLP_MAX_DENSE = 4
NODE_MLP_MAX_PER_SAMPLE = 65536   # per-sample input rows
_node_mlp_ws = {}


def _node_mlp_source_shapes(sources, M):
    """[(C, bcast)] per source and (B, M), from shapes alone: a 3-D tensor [B,C,M] is dense, a 2-D tensor [B,C] is
    the same for every column of its sample; ValueError on a mismatch or a bound."""
    if not isinstance(sources, (list, tuple)) or not sources or not all(isinstance(s, torch.Tensor) for s in sources):
        raise ValueError("sources: need a non-empty list of tensors [B,C,M] (dense) or [B,C] (per sample)")
    spec, B = [], sources[0].shape[0]
    for i, s in enumerate(sources):
        if s.dim() not in (2, 3):
            raise ValueError(f"sources[{i}]: need [B,C,M] (dense) or [B,C] (per sample), got {tuple(s.shape)}")
        if s.shape[0] != B:
            raise ValueError(f"sources[{i}] has {s.shape[0]} samples, sources[0] has {B}")
        if s.shape[1] < 1:
            raise ValueError(f"sources[{i}]: need at least one channel")
        if s.dim() == 3:
            if M is None:
                M = s.shape[2]
            elif s.shape[2] != M:
                raise ValueError(f"sources[{i}] has {s.shape[2]} columns, expected {M}")
        spec.append((int(s.shape[1]), s.dim() == 2))
    if M is None:
        raise ValueError("M: give the number of columns when every source is per sample")
    _check_node_mlp_rows(spec)
    if not 1 <= B <= MLP_MAX_BATCH or M < 1:
        raise ValueError(f"need 1 <= B <= {MLP_MAX_BATCH} and M >= 1, got B = {B}, M = {M}")
    return spec, B, int(M)


def _check_node_mlp_rows(spec):
    dense = [c for c, bc in spec if not bc]
    if len(dense) > NODE_MLP_MAX_DENSE:
        raise ValueError(f"sources: at most {NODE_MLP_MAX_DENSE} dense sources")
    if sum(dense) > NODE_MLP_MAX_WIDTH:
        raise ValueError(f"the dense sources have {sum(dense)} rows, more than {NODE_MLP_MAX_WIDTH}")
    if sum(c for c, bc in spec if bc) > NODE_MLP_MAX_PER_SAMPLE:
        raise ValueError(f"the per-sample sources have more than {NODE_MLP_MAX_PER_SAMPLE} rows")


def _node_mlp_widths(layers, c_in):
    """[(C_out, relu)] of 1 to 3 layers (W [C_out,C_in], b [C_out] or None, relu), widths in [1, 1024]."""
    if not isinstance(layers, (list, tuple)) or not 1 <= len(layers) <= MLP_MAX_LAYERS:
        raise ValueError(f"layers: need a list of 1 to {MLP_MAX_LAYERS} layers")
    meta = []
    for i, layer in enumerate(layers):
        if not isinstance(layer, (list, tuple)) or len(layer) != 3:
            raise ValueError(f"layers[{i}]: need (W, b, relu)")
        W, b, relu = layer
        if not isinstance(W, torch.Tensor) or W.dim() != 2 or W.shape[1] != c_in:
            raise ValueError(f"layers[{i}]: W must be [C_out, {c_in}]")
        if not 1 <= W.shape[0] <= NODE_MLP_MAX_WIDTH:
            raise ValueError(f"layers[{i}]: need 1 <= C_out <= {NODE_MLP_MAX_WIDTH}, got {W.shape[0]}")
        if b is not None and (not isinstance(b, torch.Tensor) or tuple(b.shape) != (W.shape[0],)):
            raise ValueError(f"layers[{i}]: b must be [{W.shape[0]}] or None")
        c_in = W.shape[0]
        meta.append((c_in, bool(relu)))
    return meta


def _node_mlp_tables(spec, meta):
    import numpy as np
    src = np.zeros((len(spec), _MLP_SRC), dtype=np.int64)
    for i, (C, bcast) in enumerate(spec):
        src[i, 2], src[i, 7] = C, int(bcast)
    _, lay = _mlp_tables([], meta)
    return src, lay


class PackedNodeMLP:
    """The layers of one node_mlp chain in the kernel's order on the device (weights rounded to TF32 once, the per-
    sample sources' columns of W1 split off and transposed), for sources of the widths and kinds `spec` = [(C,
    per_sample)].  pack_node_mlp builds it."""

    def __init__(self, spec, meta, packed):
        self.spec, self.meta, self.packed = list(spec), list(meta), packed


def pack_node_mlp(spec, layers):
    """Pack `layers` = [(W [C_out,C_in] float32 CUDA, b [C_out] or None, relu)] (network.fold_pointnet's list) for
    sources of the widths and kinds `spec` = [(C, per_sample)] in input-row order; node_mlp does this itself when given
    the raw layers."""
    spec = [(int(c), bool(bc)) for c, bc in spec]
    if not spec or any(c < 1 for c, _ in spec):
        raise ValueError("spec: need a non-empty list of (C >= 1, per_sample)")
    _check_node_mlp_rows(spec)
    meta = _node_mlp_widths(layers, sum(c for c, _ in spec))
    dev = layers[0][0].device
    keep = []
    for W, b, _ in layers:
        for t in (W, b):
            if t is None:
                continue
            if t.requires_grad and torch.is_grad_enabled():
                raise RuntimeError("node_mlp has no backward: call it under torch.no_grad() or detach the layers")
            if not t.is_cuda or t.device != dev or t.dtype != torch.float32:
                raise RuntimeError("the layers must be float32 CUDA tensors on one device")
        keep.append((W.detach().contiguous(), None if b is None else b.detach().contiguous()))
    src, lay = _node_mlp_tables(spec, meta)
    for i, (W, b) in enumerate(keep):
        lay[i, 0], lay[i, 1] = W.data_ptr(), 0 if b is None else b.data_ptr()
    lib = _native.load()
    need = lib.node_mlp_packed_bytes(src.ctypes.data, len(spec), lay.ctypes.data, len(meta))
    if need == 0:
        raise ValueError("node_mlp: " + lib.dib_last_error().decode("utf-8", "replace"))
    with torch.cuda.device(dev):
        packed = torch.empty(need // 4, dtype=torch.float32, device=dev)
        rc = lib.node_mlp_pack_f32(src.ctypes.data, len(spec), lay.ctypes.data, len(meta), packed.data_ptr(), need,
                                   _stream_ptr())
    _native.check(rc, "node_mlp_pack_f32")
    del keep
    return PackedNodeMLP(spec, meta, packed)


def node_mlp(sources, layers, M=None):
    """A chain of one to three 1x1-convolution layers y = act(W x + b) over the M columns (nodes) of each sample, in
    one kernel, for inference (DESIGN.md 4.27): the decoder's node-level PointNets, with BatchNorm already folded into
    W and b (network.fold_pointnet) and the input concatenation never built.

    sources: in the order of layer 1's input rows, float32 CUDA tensors that are either dense [B,C,M] (at most 4 with
    at most 1024 rows in all; a channel slice of a wider contiguous tensor is read in place) or per sample [B,C] (any
    number, at most 65536 rows in all; a [B,C,1] tensor is passed as t[:, :, 0], with no copy).  M is needed only when every source is per sample.
    layers: [(W [C_out,C_in], b [C_out] or None, relu)] with every C_out in [1, 1024], or a PackedNodeMLP.  Returns
    the last layer [B,C_out,M] float32.

    The dense rows' products run on the tensor cores in TF32 with float32 accumulation whatever torch's TF32 flags
    say.  A per-sample source's block of W1 is applied once per sample and output row, as a float32 fma chain in
    ascending input row, and added to every column before the bias.  Weights, source values and the activations
    between layers are rounded to TF32 (nearest, ties away from zero); bias and ReLU (NaN stays NaN) are float32.  No
    backward: an input that requires grad raises RuntimeError unless grad mode is off.  Shape and bound errors raise
    ValueError before anything is launched."""
    spec, B, M = _node_mlp_source_shapes(sources, M)
    if isinstance(layers, PackedNodeMLP):
        if layers.spec != spec:
            raise ValueError(f"the layers were packed for sources {layers.spec}, got {spec}")
        packed, meta = layers, layers.meta
    else:
        packed, meta = None, _node_mlp_widths(layers, sum(c for c, _ in spec))
    dev = sources[0].device
    for t in sources:
        if t.requires_grad and torch.is_grad_enabled():
            raise RuntimeError("node_mlp has no backward: call it under torch.no_grad() or detach the inputs")
        if not t.is_cuda or t.device != dev:
            raise RuntimeError(f"node_mlp: every source must be a CUDA tensor on {dev}")
        if t.dtype != torch.float32:
            raise RuntimeError("node_mlp: every source must be float32")
    src, lay = _node_mlp_tables(spec, meta)
    keep = []
    for i, s in enumerate(sources):
        C = s.shape[1]
        if s.dim() == 3:
            if (M > 1 and s.stride(2) != 1) or (C > 1 and s.stride(1) != M) or (B > 1 and s.stride(0) < C * M):
                s = s.contiguous()
        elif (C > 1 and s.stride(1) != 1) or (B > 1 and s.stride(0) < C):
            s = s.contiguous()
        keep.append(s)
        src[i, 0], src[i, 1] = s.data_ptr(), s.stride(0) if B > 1 else C * (M if s.dim() == 3 else 1)
    if packed is None:
        packed = pack_node_mlp(spec, layers)
    if packed.packed.device != dev:
        raise RuntimeError(f"the layers must be on {dev}")
    lib = _native.load()
    with torch.cuda.device(dev):
        stream = _stream_ptr()
        need = lib.node_mlp_workspace_bytes(src.ctypes.data, len(spec), lay.ctypes.data, len(meta), B)
        ws = _workspace(_node_mlp_ws, need, dev, floor=0) if need else None
        out = torch.empty((B, meta[-1][0], M), dtype=torch.float32, device=dev)
        rc = lib.node_mlp_f32(src.ctypes.data, len(spec), lay.ctypes.data, len(meta), packed.packed.data_ptr(),
                              packed.packed.numel() * 4, B, M, out.data_ptr(),
                              ws.data_ptr() if ws is not None else None, ws.numel() if ws is not None else 0, stream)
    _native.check(rc, "node_mlp_f32")
    del keep
    return out
