"""Host side of index_max / ball_query: torch tensors in, torch tensors out, kernels via the C ABI.

Mirrors the reference's extension modules (models/index_max_ext/index_max.cpp:119-159,
models/ball_query_ext/ball_query.cpp:23-48): same argument checks (CUDA + contiguous ->
RuntimeError), output allocated on the input's device, int32 outputs.  Unlike the reference the
kernels are launched on torch's *current* stream of the tensor's device, not the legacy default
stream (SURVEY.md 8b).
"""
import torch

from . import _native
from ._native import _stream_ptr, _workspace, feature_dtype


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
    for t, name in ((query, "query"), (node, "node")):
        if t.dtype != torch.float32:
            raise RuntimeError(f"{name} must have dtype {torch.float32}")
    feature_dtype(((features, "features"),))
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
        dtype, sfx = feature_dtype(((features, "features"),))
        with torch.cuda.device(dev):
            w = torch.empty((B, Nq, k), dtype=torch.float32, device=dev)
            idx = torch.empty((B, Nq, k), dtype=torch.int32, device=dev)
            out = torch.empty((B, C, Nq), dtype=dtype, device=dev)
            if out.numel():
                stream = _stream_ptr()
                rc = lib.interp_weights_f32(topk_idx.data_ptr(), topk_idx.element_size(), query.data_ptr(),
                                            node.data_ptr(), B, Nq, M, k, w.data_ptr(), idx.data_ptr(), stream)
                _native.check(rc, "interp_weights_f32")
                rc = getattr(lib, f"interp_forward_{sfx}")(features.data_ptr(), w.data_ptr(), idx.data_ptr(), B, C,
                                                           Nq, M, k, out.data_ptr(), stream)
                _native.check(rc, f"interp_forward_{sfx}")
        ctx.save_for_backward(w, idx)
        ctx.shape = (B, C, Nq, M, k)
        ctx.dtype = (dtype, sfx)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        if not ctx.needs_input_grad[3]:
            return None, None, None, None
        w, idx = ctx.saved_tensors
        B, C, Nq, M, k = ctx.shape
        dtype, sfx = ctx.dtype
        dev = w.device
        # the kernel takes any batch stride with (channel, point) strides (Nq, 1): a channel slice of a torch.cat
        # gradient needs no copy
        grad_out = grad_out.to(dtype)
        if (C > 1 and grad_out.stride(1) != Nq) or (Nq > 1 and grad_out.stride(2) != 1):
            grad_out = grad_out.contiguous()
        lib = _native.load()
        with torch.cuda.device(dev):
            gF = torch.empty((B, C, M), dtype=dtype, device=dev)
            if gF.numel():
                stream = _stream_ptr()
                ws = _backward_workspace(dev, lib.interp_backward_workspace_bytes(B, C, Nq, M))
                bstride = grad_out.stride(0) if B > 1 else 0
                rc = getattr(lib, f"interp_backward_{sfx}")(grad_out.data_ptr(), bstride, w.data_ptr(), idx.data_ptr(),
                                                            B, C, Nq, M, k, gF.data_ptr(), ws.data_ptr(), ws.numel(),
                                                            stream)
                _native.check(rc, f"interp_backward_{sfx}")
        return None, None, None, gF


def upsample_by_interpolation(topk_idx, query, node, features):
    """Inverse-distance interpolation of node features onto query points: KeypointDetector.upsample_by_interpolation
    (models/networks_united.py:90-103, the same argument order without `self`) without its B x C x Nq x k tensors.

    topk_idx [B,Nq,k] int32 / int64 (e.g. cluster_assign_forward(...)["min_k_idx"] or a torch.topk result), query
    [B,3,Nq], node [B,3,M] float32 and features [B,C,M] float32 or bfloat16 CUDA; 1 <= k <= 8, 1 <= M <= 2048.
    Returns out [B,C,Nq] of the features' dtype with
    out[b,c,n] = sum_j w_j features[b,c,idx_j], d_j = |query_n - node_{idx_j}|, w_j = 1 - d_j / sum_j d_j (DESIGN.md
    4.12).  As in the reference the weights sum to k - 1, k = 1 gives weight 0 and a zero distance sum gives NaN; a
    query point with any index outside [0, M) gets NaN in all C channels and no share of the feature gradient.
    Differentiable with respect to `features` only, with a deterministic gradient; query and node must not require
    grad.  bfloat16 features give the float32 result on the widened features, rounded to bfloat16, and the same rule
    for the gradient (DESIGN.md 4.37)."""
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
    feature_dtype(((features, "features"),))
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
        dtype, sfx = feature_dtype(((features, "features"),))
        with torch.cuda.device(dev):
            sel = torch.empty((B, C, M), dtype=torch.int32, device=dev)
            mask = torch.empty((B, M), dtype=torch.float32, device=dev)
            pooled = torch.empty((B, C, M), dtype=dtype, device=dev)
            scattered = torch.empty((B, C, N), dtype=dtype, device=dev) if broadcast else None
            if B:
                rc = getattr(lib, f"cluster_pool_forward_{sfx}")(
                    features.data_ptr(), min_idx.data_ptr(), B, C, N, M, sel.data_ptr(), mask.data_ptr(),
                    pooled.data_ptr(), scattered.data_ptr() if broadcast and scattered.numel() else None,
                    _stream_ptr())
                _native.check(rc, f"cluster_pool_forward_{sfx}")
        ctx.set_materialize_grads(False)           # a missing pooled or scattered gradient stays None
        ctx.save_for_backward(min_idx, sel, mask)
        ctx.shape = (B, C, N, M)
        ctx.dtype = (dtype, sfx)
        return (pooled, scattered) if broadcast else pooled

    @staticmethod
    def backward(ctx, grad_pooled, grad_scattered=None):
        if not ctx.needs_input_grad[0] or (grad_pooled is None and grad_scattered is None):
            return None, None, None, None
        min_idx, sel, mask = ctx.saved_tensors
        B, C, N, M = ctx.shape
        dtype, sfx = ctx.dtype
        dev = sel.device
        if grad_pooled is not None:
            grad_pooled = grad_pooled.to(dtype).contiguous()
        if grad_scattered is not None:
            # any batch stride with (channel, point) strides (N, 1): a channel slice of a torch.cat gradient needs
            # no copy
            grad_scattered = grad_scattered.to(dtype)
            if (C > 1 and grad_scattered.stride(1) != N) or (N > 1 and grad_scattered.stride(2) != 1):
                grad_scattered = grad_scattered.contiguous()
        lib = _native.load()
        with torch.cuda.device(dev):
            gF = torch.empty((B, C, N), dtype=dtype, device=dev)
            if gF.numel():
                stream = _stream_ptr()
                ws, ws_bytes = None, 0
                if grad_scattered is not None:
                    ws = _backward_workspace(dev, lib.cluster_pool_backward_workspace_bytes(B, C, N, M))
                    ws_bytes = ws.numel()
                gs_ptr = grad_scattered.data_ptr() if grad_scattered is not None else None
                bstride = grad_scattered.stride(0) if grad_scattered is not None and B > 1 else 0
                rc = getattr(lib, f"cluster_pool_backward_{sfx}")(
                    grad_pooled.data_ptr() if grad_pooled is not None else None, gs_ptr, bstride, min_idx.data_ptr(),
                    sel.data_ptr(), mask.data_ptr(), B, C, N, M, gF.data_ptr(),
                    ws.data_ptr() if ws is not None else None, ws_bytes, stream)
                _native.check(rc, f"cluster_pool_backward_{sfx}")
        return gF, None, None, None


def cluster_max_pool(features, min_idx, M, broadcast=False):
    """SO-Net masked max-pool of PCEncoder.forward (models/networks_pc.py:88-104) in one op, with a deterministic
    feature gradient (DESIGN.md 4.16).

    features [B,C,N] float32 or bfloat16 and min_idx [B,N] int32 (cluster_assign_forward's) CUDA, M >= 1 segments.
    Returns pooled [B,C,M] (of the features' dtype, as scattered) = features[b,c,sel] * mask[b,m], sel = index_max_forward(features, min_idx, M) and mask[b,m] = 1.0 where
    some point has min_idx == m (else 0.0: an empty segment gives features[b,c,0] * 0.0, -0.0 or NaN included).  With
    broadcast=True returns (pooled, scattered), scattered [B,C,N] = pooled[b,c,min_idx[b,n]].  A point whose min_idx
    is outside [0, M) joins no segment, gets NaN in every channel of scattered and no share of the gradient.
    Differentiable with respect to `features`: fp64 sums in an order fixed by the shape, no float atomics.  bfloat16
    features give the float32 results on the widened features, rounded to bfloat16, and the same rule for the gradient
    (DESIGN.md 4.37)."""
    _check_pool_args(features, min_idx, M)
    return _ClusterMaxPool.apply(features, min_idx, int(M), bool(broadcast))


def _check_knn_args(query, database, features, K):
    """Shape, dtype, bound and autograd checks first (they need no device), then device and layout."""
    for t, name in ((query, "query"), (database, "database"), (features, "features")):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{name} must be a torch.Tensor")
        if t is features:
            feature_dtype(((features, "features"),))
        elif t.dtype != torch.float32:
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
        dtype, sfx = feature_dtype(((features, "features"),))
        with torch.cuda.device(dev):
            idx = torch.empty((B, M, K), dtype=torch.int32, device=dev)
            grouped = torch.empty((B, 3 + C, M, K), dtype=dtype, device=dev)
            if idx.numel():
                rc = getattr(lib, f"knn_group_forward_{sfx}")(query.data_ptr(), database.data_ptr(),
                                                              features.data_ptr(), B, C, M, N, K, idx.data_ptr(),
                                                              grouped.data_ptr(), _stream_ptr())
                _native.check(rc, f"knn_group_forward_{sfx}")
        ctx.mark_non_differentiable(idx)
        ctx.set_materialize_grads(False)
        ctx.save_for_backward(idx)
        ctx.shape = (B, C, M, N, K)
        ctx.dtype = (dtype, sfx)
        return idx, grouped

    @staticmethod
    def backward(ctx, grad_idx, grad_grouped):
        if not ctx.needs_input_grad[2]:
            return None, None, None, None
        idx, = ctx.saved_tensors
        B, C, M, N, K = ctx.shape
        dtype, sfx = ctx.dtype
        dev = idx.device
        if grad_grouped is None:                   # grouped took no part in the loss: a zero gradient, not materialised
            return None, None, None, None
        # any batch stride with (row, query, neighbour) strides (M * K, K, 1).  There are always 3 + C >= 3 rows, so the
        # row stride is checked whatever M and K are (at M = K = 1 a slice of a cat along dim 3 has row stride != 1)
        grad_grouped = grad_grouped.to(dtype)
        if grad_grouped.stride(1) != M * K or (M > 1 and grad_grouped.stride(2) != K) \
                or (K > 1 and grad_grouped.stride(3) != 1):
            grad_grouped = grad_grouped.contiguous()
        lib = _native.load()
        with torch.cuda.device(dev):
            gF = torch.empty((B, C, N), dtype=dtype, device=dev)
            if gF.numel():
                stream = _stream_ptr()
                ws = _backward_workspace(dev, lib.knn_group_backward_workspace_bytes(B, C, M, N, K))
                bstride = grad_grouped.stride(0) if B > 1 else 0
                rc = getattr(lib, f"knn_group_backward_{sfx}")(grad_grouped.data_ptr() if M else None, bstride,
                                                               idx.data_ptr(), B, C, M, N, K, gF.data_ptr(),
                                                               ws.data_ptr(), ws.numel(), stream)
                _native.check(rc, f"knn_group_backward_{sfx}")
        return None, None, gF, None


def knn_group(query, database, features, K):
    """Node kNN grouping of GeneralKNNFusionModule.forward (models/layers_pc.py:793-807) in one op, with a
    deterministic feature gradient (DESIGN.md 4.16).

    query [B,3,M], database [B,3,N] float32 and features [B,C,N] float32 or bfloat16 CUDA; 1 <= K <= 32, K <= N <=
    2048.  Returns (knn_idx [B,M,K] int32, grouped [B,3+C,M,K] of the features' dtype): knn_idx holds the K nearest database nodes of each query, nearest first, by
    cluster_assign's key (f32 ((dx*dx + dy*dy) + dz*dz) without fma, ties -> lower index, +inf after finite keys, NaN
    after +inf); grouped rows 0-2 are database[idx] - query and rows 3 onward features[idx], the tensor
    layers_pc.py:807 concatenates.  Differentiable with respect to `features` only (fp64 sums in an order fixed by the
    shape, no float atomics); query and database must not require grad, as the reference detaches both.  bfloat16
    features give the float32 result on the widened features rounded to bfloat16 (the coordinate rows too), and the
    same rule for the gradient (DESIGN.md 4.37)."""
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
    feature_dtype(((img_features, "img_features"), (attention, "attention")))
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
        dtype, sfx = feature_dtype(((img_features, "img_features"), (attention, "attention")))
        with torch.cuda.device(dev):
            out = torch.empty((B, C, M), dtype=dtype, device=dev)
            rc = getattr(lib, f"attn_fusion_forward_{sfx}")(img_features.data_ptr(), attention.data_ptr(), B, C, P, M,
                                                            out.data_ptr(), _stream_ptr())
        _native.check(rc, f"attn_fusion_forward_{sfx}")
        ctx.set_materialize_grads(False)           # a missing output gradient stays None
        ctx.save_for_backward(img_features, attention)
        ctx.dtype = (dtype, sfx)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        need_F, need_A = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if grad_out is None or not (need_F or need_A):
            return None, None
        F, A = ctx.saved_tensors
        B, C, P = F.shape
        M = A.shape[2]
        dtype, sfx = ctx.dtype
        dev = F.device
        # any batch stride with (channel, node) strides (M, 1): a channel slice of a torch.cat gradient needs no copy
        grad_out = grad_out.to(dtype)
        if (C > 1 and grad_out.stride(1) != M) or (M > 1 and grad_out.stride(2) != 1):
            grad_out = grad_out.contiguous()
        lib = _native.load()
        with torch.cuda.device(dev):
            gF = torch.empty((B, C, P), dtype=dtype, device=dev) if need_F else None
            gA = torch.empty((B, P, M), dtype=dtype, device=dev) if need_A else None
            bstride = grad_out.stride(0) if B > 1 else 0
            rc = getattr(lib, f"attn_fusion_backward_{sfx}")(grad_out.data_ptr(), bstride, F.data_ptr(), A.data_ptr(),
                                                             B, C, P, M, gF.data_ptr() if need_F else None,
                                                             gA.data_ptr() if need_A else None, _stream_ptr())
        _native.check(rc, f"attn_fusion_backward_{sfx}")
        return gF, gA


def attention_fusion(img_features, attention):
    """Attention-weighted image features of KeypointDetector.forward (models/networks_united.py:149-150,172-174,
    torch.mean(img_features.unsqueeze(3) * attention.unsqueeze(1), dim=2)) without its B x C x P x M product
    (DESIGN.md 4.17).

    img_features [B,C,P] (the feature map's .view(B, C, -1)) and attention [B,P,M] CUDA, contiguous, on one device,
    both float32 or both bfloat16.  Returns out [B,C,M] of their dtype, out[b,c,m] = float((sum over p ascending of F[b,c,p] * A[b,p,m]) / P), one fp64
    accumulator per output over the exact products, so the result does not depend on tiling, batch composition or the
    TF32 flags.  Differentiable with respect to both inputs with the same rule (sums over m for img_features, over c
    for attention); an input that needs no gradient costs nothing in the backward.  bfloat16 inputs give the float32
    result on the widened inputs, rounded to bfloat16, and the same rule for the gradients (DESIGN.md 4.37)."""
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


def _layer_widths(layers, c_in, max_width, name, lo, hi):
    """[(C_out, relu)] of lo to hi layers (W [C_out,C_in], b [C_out] or None, relu), widths in [1, max_width];
    ValueError otherwise.  The first layer takes c_in rows."""
    if not isinstance(layers, (list, tuple)) or not lo <= len(layers) <= hi:
        raise ValueError(f"{name}: need a list of {lo} to {hi} layers")
    meta = []
    for i, layer in enumerate(layers):
        if not isinstance(layer, (list, tuple)) or len(layer) != 3:
            raise ValueError(f"{name}[{i}]: need (W, b, relu)")
        W, b, relu = layer
        if not isinstance(W, torch.Tensor) or W.dim() != 2 or W.shape[1] != c_in:
            raise ValueError(f"{name}[{i}]: W must be [C_out, {c_in}]")
        if not 1 <= W.shape[0] <= max_width:
            raise ValueError(f"{name}[{i}]: need 1 <= C_out <= {max_width}, got {W.shape[0]}")
        if b is not None and (not isinstance(b, torch.Tensor) or tuple(b.shape) != (W.shape[0],)):
            raise ValueError(f"{name}[{i}]: b must be [{W.shape[0]}] or None")
        c_in = W.shape[0]
        meta.append((c_in, bool(relu)))
    return meta


def _mlp_tables(spec, meta, slots=(2, 3, 6)):
    """The int64 source and layer tables of the fused ops (DIB_MLP_SRC, DIB_MLP_LAYER rows): each entry of spec in
    the source slots `slots` (CHANNELS, NODES, K by default), (C_out, relu) per layer; the addresses are filled in by
    the caller."""
    import numpy as np
    src = np.zeros((len(spec), _MLP_SRC), dtype=np.int64)
    for i, row in enumerate(spec):
        for j, v in zip(slots, row):
            src[i, j] = v
    lay = np.zeros((len(meta), _MLP_LAYER), dtype=np.int64)
    for i, (C, relu) in enumerate(meta):
        lay[i, 2], lay[i, 3] = C, int(relu)
    return src, lay


class PackedLayers:
    """The layers of one fused chain in its kernel's order on the device (weights rounded to TF32 once), as
    pack_pointwise_mlp, pack_knn_fusion, pack_pointwise_mlp_max or pack_node_mlp built them: kind names the op, key
    the input they were packed for (the source spec of pointwise_mlp and node_mlp, the input rows of knn_fusion and
    pointwise_mlp_max), meta = [(C_out, relu)] over every layer, n_before of them before knn_fusion's per-node max
    (all of them for the other ops), packed the device buffer."""

    def __init__(self, kind, key, meta, n_before, packed):
        self.kind, self.key, self.meta, self.n_before, self.packed = kind, key, list(meta), n_before, packed


def _pack(kind, key, layers, meta, lay, args, n_before=None):
    """Pack `layers` (of the checked widths meta) with lib.<kind>_packed_bytes(*args) and lib.<kind>_pack_f32(*args,
    packed, bytes, stream), args naming the layer table lay, whose W and b addresses are filled in here."""
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
    for i, (W, b) in enumerate(keep):
        lay[i, 0], lay[i, 1] = W.data_ptr(), 0 if b is None else b.data_ptr()
    lib = _native.load()
    need = getattr(lib, kind + "_packed_bytes")(*args)
    if need == 0:
        raise ValueError(f"{kind}: " + lib.dib_last_error().decode("utf-8", "replace"))
    with torch.cuda.device(dev):
        packed = torch.empty(need // 4, dtype=torch.float32, device=dev)
        rc = getattr(lib, kind + "_pack_f32")(*args, packed.data_ptr(), need, _stream_ptr())
    _native.check(rc, kind + "_pack_f32")
    del keep
    return PackedLayers(kind, key, meta, len(meta) if n_before is None else n_before, packed)


def _prepacked(layers, kind, key):
    """layers if it is a PackedLayers that pack_<kind> built for `key`, None if it is not a PackedLayers; ValueError
    for layers packed for another op or input."""
    if not isinstance(layers, PackedLayers):
        return None
    if layers.kind != kind or layers.key != key:
        raise ValueError(f"the layers were packed as {layers.kind} for {layers.key}, need {kind} for {key}")
    return layers


def _check_sources(name, tensors):
    """RuntimeError unless every tensor is a float32 CUDA tensor on the first one's device, with no gradient to
    keep (the fused ops have no backward); returns that device."""
    dev = tensors[0].device
    for t in tensors:
        if t.requires_grad and torch.is_grad_enabled():
            raise RuntimeError(f"{name} has no backward: call it under torch.no_grad() or detach the inputs")
        if not t.is_cuda or t.device != dev:
            raise RuntimeError(f"{name}: every input must be a CUDA tensor on {dev}")
        if t.dtype != torch.float32:
            raise RuntimeError(f"{name}: every input must be float32")
    return dev


def _dense_source(s, B, N):
    """(s, batch stride) of a dense source [B,C,N] (or [B,C] with N = 1) as the kernels read it: rows of N contiguous
    columns C apart, so a channel slice of a wider contiguous tensor is read in place; any other layout is copied."""
    C = s.shape[1]
    if (N > 1 and s.stride(2) != 1) or (C > 1 and s.stride(1) != N) or (B > 1 and s.stride(0) < C * N):
        s = s.contiguous()
    return s, s.stride(0) if B > 1 else C * N


def pack_pointwise_mlp(spec, layers):
    """Pack `layers` = [(W [C_out,C_in] float32 CUDA, b [C_out] or None, relu)] for sources of the widths `spec` =
    [(C, M, k)] (M = k = 0 for a dense source) into a PackedLayers; pointwise_mlp does this itself when given the raw
    layers."""
    spec = [tuple(int(v) for v in s) for s in spec]
    meta = _layer_widths(layers, sum(c for c, _, _ in spec), MLP_MAX_WIDTH, "layers", 1, MLP_MAX_LAYERS)
    src, lay = _mlp_tables(spec, meta)
    return _pack("pointwise_mlp", spec, layers, meta, lay, (src.ctypes.data, len(spec), lay.ctypes.data, len(meta)))


def pointwise_mlp(sources, layers, output="activations", c_split=None, return_scores=False):
    """A chain of one to three 1x1-convolution layers y = act(W x + b) over every point, in one kernel, for inference
    (DESIGN.md 4.21): the PointNets the classifier applies per point, with BatchNorm already folded into W and b
    (network.fold_pointnet) and the input concatenation never built.

    sources: 1 to 4 of, in the order of layer 1's input rows, a dense float32 CUDA tensor [B,C,N] (a channel slice of
    a wider contiguous tensor is read in place) or a tuple (features [B,C,M], w [B,N,k], idx [B,N,k]) whose rows are
    the interpolation upsample_by_interpolation computes (w, idx from interpolation_weights; k <= 8, M <= 2048, a
    point with idx = -1 has NaN rows).  At most 1024 rows in all.  layers: [(W [C_out,C_in], b [C_out] or None, relu)]
    with every C_out in [1, 256], or a PackedLayers from pack_pointwise_mlp.

    output="activations" returns the last layer [B,C_out,N].  output="argmax" returns (int8 [B,N], int32 [B,N] or
    None): the arg-max over channels [0, c_split) and over [c_split, C_out) (None when that range is empty) by
    torch.max's rule, so c_split = 2 is network.predict; with return_scores=True the scores [B,C_out,N] come third.

    The products run on the tensor cores in TF32 with float32 accumulation whatever torch's TF32 flags say: weights,
    source values and the activations between layers are rounded to TF32 (nearest, ties away from zero); bias, ReLU
    (NaN stays NaN) and the arg-max are float32.  No backward: an input that requires grad raises RuntimeError unless
    grad mode is off.  Shape and bound errors raise ValueError before anything is launched."""
    spec, B, N = _mlp_source_shapes(sources)
    packed = _prepacked(layers, "pointwise_mlp", spec)
    meta = packed.meta if packed is not None else _layer_widths(layers, sum(c for c, _, _ in spec), MLP_MAX_WIDTH,
                                                                "layers", 1, MLP_MAX_LAYERS)
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
            s, src[i, 1] = _dense_source(s, B, N)
            keep.append(s)
            src[i, 0] = s.data_ptr()
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


def _knn_fusion_meta(C, before, after):
    if not isinstance(C, int) or not 1 <= C <= KNN_FUSION_MAX_WIDTH - 3:
        raise ValueError(f"knn_fusion: need 1 <= C <= {KNN_FUSION_MAX_WIDTH - 3} feature channels, got {C}")
    mb = _layer_widths(before, 3 + C, KNN_FUSION_MAX_WIDTH, "before", 1, KNN_FUSION_MAX_SIDE)
    ma = _layer_widths(after, 2 * mb[-1][0], KNN_FUSION_MAX_WIDTH, "after", 1, KNN_FUSION_MAX_SIDE)
    return mb + ma, len(mb)


def pack_knn_fusion(C, before, after):
    """Pack the folded layers of a kNN fusion module for C feature channels (network.fold_knn_fusion's lists) once
    into a PackedLayers; knn_fusion does this itself when given the raw layers."""
    meta, n_before = _knn_fusion_meta(int(C), before, after)
    c_in = 3 + int(C)
    _, lay = _mlp_tables([], meta)
    return _pack("knn_fusion", c_in, list(before) + list(after), meta, lay,
                 (c_in, lay.ctypes.data, n_before, len(meta) - n_before), n_before)


def knn_fusion(query, database, features, K, layers, return_idx=False):
    """The node kNN module (GeneralKNNFusionModule.forward, layers_pc.py:793-818) in one kernel, for inference
    (DESIGN.md 4.26): group the K nearest database nodes of each query as knn_group does, the "before" layers, the max
    over the K neighbours, the "after" layers over the concatenation [max; x], the max over K again.  No [B,C,M,K]
    tensor is built: the max half of the first after layer is projected once per node and added like a bias.

    query [B,3,M], database [B,3,N], features [B,C,N] float32 CUDA; 1 <= K <= 32, K <= N <= 2048, 3 + C <= 512.
    layers: (before, after), each a list of 1 to 3 (W [C_out,C_in], b [C_out] or None, relu) with every C_out in
    [1, 512] (BatchNorm folded: network.fold_knn_fusion), the first after layer taking 2 C_b rows (max first), or a
    PackedLayers from pack_knn_fusion.  Returns out [B,C_out,M], and knn_group's knn_idx [B,M,K] int32 with
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
    packed = _prepacked(layers, "knn_fusion", 3 + C)
    if packed is not None:
        meta, n_before = packed.meta, packed.n_before
    else:
        if not isinstance(layers, (list, tuple)) or len(layers) != 2:
            raise ValueError("layers: need (before, after) or a PackedLayers")
        meta, n_before = _knn_fusion_meta(C, *layers)
    dev = _check_sources("knn_fusion", (features, query, database))
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
    """Pack `layers` = [(W [C_out,C_in] float32 CUDA, b [C_out] or None, relu)] for c_in input rows once into a
    PackedLayers; pointwise_mlp_max does this itself when given the raw layers."""
    c_in = int(c_in)
    if not 1 <= c_in <= KNN_FUSION_MAX_WIDTH:
        raise ValueError(f"pointwise_mlp_max: need 1 <= input rows <= {KNN_FUSION_MAX_WIDTH}, got {c_in}")
    meta = _layer_widths(layers, c_in, KNN_FUSION_MAX_WIDTH, "layers", 1, KNN_FUSION_MAX_SIDE)
    _, lay = _mlp_tables([], meta)
    return _pack("pointwise_mlp_max", c_in, layers, meta, lay, (c_in, lay.ctypes.data, len(meta)))


def pointwise_mlp_max(sources, layers):
    """A chain of one to three 1x1-convolution layers over the columns of each sample, then the max over all of them,
    in one kernel and a fixed-order reduction, for inference (DESIGN.md 4.26): final_pointnet + torch.max(dim=2) of
    the point encoder, with the input concatenation and the [B,C_out,N] activations never built.

    sources: 1 to 4 dense float32 CUDA tensors [B,C,N] (a channel slice of a wider contiguous tensor is read in
    place), at most 512 rows in all.  layers: [(W [C_out,C_in], b [C_out] or None, relu)], every C_out in [1, 512],
    or a PackedLayers from pack_pointwise_mlp_max.  Returns [B,C_out,1] float32.  pointwise_mlp's TF32 rule; the max
    is float32 with torch.max's NaN rule.  No backward; shape and bound errors raise ValueError before any launch."""
    if not isinstance(sources, (list, tuple)) or not all(isinstance(s, torch.Tensor) for s in sources):
        raise ValueError("sources: need a list of dense [B,C,N] tensors")
    spec, B, N = _mlp_source_shapes(sources)
    c_in = sum(c for c, _, _ in spec)
    if c_in > KNN_FUSION_MAX_WIDTH:
        raise ValueError(f"the concatenated input has {c_in} rows, more than {KNN_FUSION_MAX_WIDTH}")
    packed = _prepacked(layers, "pointwise_mlp_max", c_in)
    meta = packed.meta if packed is not None else _layer_widths(layers, c_in, KNN_FUSION_MAX_WIDTH, "layers", 1,
                                                                KNN_FUSION_MAX_SIDE)
    dev = _check_sources("pointwise_mlp_max", sources)
    src, lay = _mlp_tables(spec, meta)
    keep = []
    for i, s in enumerate(sources):
        s, src[i, 1] = _dense_source(s, B, N)
        keep.append(s)
        src[i, 0] = s.data_ptr()
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
_NODE_SLOTS = (2, 7)              # node_mlp's source rows: CHANNELS, BCAST
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


def pack_node_mlp(spec, layers):
    """Pack `layers` = [(W [C_out,C_in] float32 CUDA, b [C_out] or None, relu)] (network.fold_pointnet's list) for
    sources of the widths and kinds `spec` = [(C, per_sample)] in input-row order into a PackedLayers (the per-sample
    sources' columns of W1 split off and transposed); node_mlp does this itself when given the raw layers."""
    spec = [(int(c), bool(bc)) for c, bc in spec]
    if not spec or any(c < 1 for c, _ in spec):
        raise ValueError("spec: need a non-empty list of (C >= 1, per_sample)")
    _check_node_mlp_rows(spec)
    meta = _layer_widths(layers, sum(c for c, _ in spec), NODE_MLP_MAX_WIDTH, "layers", 1, MLP_MAX_LAYERS)
    src, lay = _mlp_tables(spec, meta, _NODE_SLOTS)
    return _pack("node_mlp", spec, layers, meta, lay, (src.ctypes.data, len(spec), lay.ctypes.data, len(meta)))


def node_mlp(sources, layers, M=None):
    """A chain of one to three 1x1-convolution layers y = act(W x + b) over the M columns (nodes) of each sample, in
    one kernel, for inference (DESIGN.md 4.27): the decoder's node-level PointNets, with BatchNorm already folded into
    W and b (network.fold_pointnet) and the input concatenation never built.

    sources: in the order of layer 1's input rows, float32 CUDA tensors that are either dense [B,C,M] (at most 4 with
    at most 1024 rows in all; a channel slice of a wider contiguous tensor is read in place) or per sample [B,C] (any
    number, at most 65536 rows in all; a [B,C,1] tensor is passed as t[:, :, 0], with no copy).  M is needed only when every source is per sample.
    layers: [(W [C_out,C_in], b [C_out] or None, relu)] with every C_out in [1, 1024], or a PackedLayers from
    pack_node_mlp.  Returns
    the last layer [B,C_out,M] float32.

    The dense rows' products run on the tensor cores in TF32 with float32 accumulation whatever torch's TF32 flags
    say.  A per-sample source's block of W1 is applied once per sample and output row, as a float32 fma chain in
    ascending input row, and added to every column before the bias.  Weights, source values and the activations
    between layers are rounded to TF32 (nearest, ties away from zero); bias and ReLU (NaN stays NaN) are float32.  No
    backward: an input that requires grad raises RuntimeError unless grad mode is off.  Shape and bound errors raise
    ValueError before anything is launched."""
    spec, B, M = _node_mlp_source_shapes(sources, M)
    packed = _prepacked(layers, "node_mlp", spec)
    meta = packed.meta if packed is not None else _layer_widths(layers, sum(c for c, _ in spec), NODE_MLP_MAX_WIDTH,
                                                                "layers", 1, MLP_MAX_LAYERS)
    dev = _check_sources("node_mlp", sources)
    src, lay = _mlp_tables(spec, meta, _NODE_SLOTS)
    keep = []
    for i, s in enumerate(sources):
        s, src[i, 1] = _dense_source(s, B, M if s.dim() == 3 else 1)   # a per-sample source [B,C] is one column
        keep.append(s)
        src[i, 0] = s.data_ptr()
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


CHAIN_MAX_LAYERS = 3
CHAIN_MAX_WIDTH = 256
CHAIN_MAX_IN = 1024
CHAIN_MAX_SOURCES = 4
_PC_SRC, _PC_OP = 3, 6            # int64 slots per operand source / transform row (DIB_PC_SRC, DIB_PC_OP)
_OP_PLAIN, _OP_ACT, _OP_BN_GRAD, _OP_MAX_GRAD = 0, 1, 2, 3     # _OP_MAX_GRAD: DIB_PC_MODE_MAX_GRAD
BRANCH_MAX_WIDTH = 1024            # point_branch's layer widths (DIB_PC_MAX_WIDTH)
_EP_WRITE, _EP_STATS, _EP_ACT_GRAD = 0, 1, 2
_chain_part_ws, _chain_dw_ws = {}, {}


def _chain_operand(srcs, mode=_OP_PLAIN, stats=None, y=None, drop=None, layer=0):
    """The operand table of point_chain's kernels: dense [B,C,N] sources in row order, then the transform row.  drop:
    (state int64 [2], p) or None."""
    import numpy as np
    t = np.zeros(len(srcs) * _PC_SRC + _PC_OP, dtype=np.int64)
    for i, s in enumerate(srcs):
        t[i * _PC_SRC:(i + 1) * _PC_SRC] = (s.data_ptr(), s.stride(0) if s.shape[0] > 1 else s.shape[1] * s.shape[2],
                                            s.shape[1])
    h = len(srcs) * _PC_SRC
    t[h:h + _PC_OP] = (mode, 0 if stats is None else stats.data_ptr(), 0 if y is None else y.data_ptr(),
                       0 if drop is None else drop[0].data_ptr(), 0 if drop is None else round(drop[1] * 1e6), layer)
    return t


def _chain_act_row(stats, drop, layer):
    import numpy as np
    return np.array((stats.data_ptr(), 0, 0 if drop is None else drop[0].data_ptr(),
                     0 if drop is None else round(drop[1] * 1e6), layer), dtype=np.int64)


def _chain_pack(W, widths):
    """W [C_out, sum(widths)] packed by pointwise_mlp's packer for dense sources of those widths.  A layer wider than
    CHAIN_MAX_WIDTH is packed in blocks of that many rows whose weight parts are concatenated: the A-fragment layout is
    row-tile major, so that is the whole layer's layout, the one point_chain_gemm_group_f32's row blocks read."""
    spec = [(c, 0, 0) for c in widths]
    if W.shape[0] <= CHAIN_MAX_WIDTH:
        return pack_pointwise_mlp(spec, [(W.detach(), None, False)]).packed
    KT = (W.shape[1] + 7) // 8
    parts = []
    for r in range(0, W.shape[0], CHAIN_MAX_WIDTH):
        blk = W[r:r + CHAIN_MAX_WIDTH]
        rows = (blk.shape[0] + 15) // 16 * 16
        parts.append(pack_pointwise_mlp(spec, [(blk.detach(), None, False)]).packed[:rows * KT * 8])
    return torch.cat(parts)


def _chain_gemm(op, n_src, packed, bias, add, C, B, N, epilogue, act=None, act_y=None, add_group=1):
    lib = _native.load()
    dev = act_y.device if act_y is not None else torch.device("cuda", torch.cuda.current_device())
    out = torch.empty((B, C, N), dtype=torch.float32, device=dev)
    part = None
    if epilogue != _EP_WRITE:
        part = _workspace(_chain_part_ws, lib.point_chain_partial_bytes(B, N, C), dev, floor=0)
    args = (None if act is None else act.ctypes.data, None if act_y is None else act_y.data_ptr(), out.data_ptr(),
            None if part is None else part.data_ptr(), 0 if part is None else part.numel(), _stream_ptr())
    head = (op.ctypes.data, n_src, None if packed is None else packed.data_ptr(),
            None if bias is None else bias.data_ptr(), None if add is None else add.data_ptr())
    if C <= CHAIN_MAX_WIDTH and add_group == 1:
        rc, name = lib.point_chain_gemm_f32(*head, C, B, N, epilogue, *args), "point_chain_gemm_f32"
    else:
        rc = lib.point_chain_gemm_group_f32(*head, add_group, C, B, N, epilogue, *args)
        name = "point_chain_gemm_group_f32"
    _native.check(rc, name)
    return out, part


def _chain_max_grad_operand(g, idx, group):
    """The operand that reads a group max's gradient g [B,C,N/G] back over the group, at the indices idx."""
    import numpy as np
    return np.array((g.data_ptr(), g.shape[1] * g.shape[2], g.shape[1], _OP_MAX_GRAD, 0, idx.data_ptr(), 0, 0, group),
                    dtype=np.int64)


def _chain_group_max(op, B, N, C, group, want_act):
    lib = _native.load()
    dev = torch.device("cuda", torch.cuda.current_device())
    act = torch.empty((B, C, N), dtype=torch.float32, device=dev) if want_act else None
    mx = torch.empty((B, C, N // group), dtype=torch.float32, device=dev)
    idx = torch.empty((B, C, N // group), dtype=torch.int32, device=dev)
    rc = lib.point_chain_group_max_f32(op.ctypes.data, B, N, group, None if act is None else act.data_ptr(),
                                       mx.data_ptr(), idx.data_ptr(), _stream_ptr())
    _native.check(rc, "point_chain_group_max_f32")
    return act, mx, idx


def _chain_group_sum(op, B, N, C, group):
    lib = _native.load()
    out = torch.empty((B, C, N // group), dtype=torch.float32, device=torch.device("cuda", torch.cuda.current_device()))
    rc = lib.point_chain_group_sum_f32(op.ctypes.data, B, N, group, out.data_ptr(), _stream_ptr())
    _native.check(rc, "point_chain_group_sum_f32")
    return out


def _chain_bn(part, B, N, C, norm, stats, grad):
    lib = _native.load()
    dev = stats.device
    if grad:
        dgamma, dbeta = torch.empty(C, dtype=torch.float32, device=dev), torch.empty(C, dtype=torch.float32, device=dev)
        coef = torch.empty((3, C), dtype=torch.float32, device=dev)
        rc = lib.point_chain_bn_f32(part.data_ptr(), B, N, C, 1, norm.weight.data_ptr(), norm.bias.data_ptr(),
                                    float(norm.eps), 0.0, stats.data_ptr(), None, None, None, dgamma.data_ptr(),
                                    dbeta.data_ptr(), coef.data_ptr(), _stream_ptr())
        _native.check(rc, "point_chain_bn_f32")
        return dgamma, dbeta, coef
    nbt = norm.num_batches_tracked
    rc = lib.point_chain_bn_f32(part.data_ptr(), B, N, C, 0, norm.weight.data_ptr(), norm.bias.data_ptr(),
                                float(norm.eps), float(norm.momentum), stats.data_ptr(), norm.running_mean.data_ptr(),
                                norm.running_var.data_ptr(), None if nbt is None else nbt.data_ptr(), None, None, None,
                                _stream_ptr())
    _native.check(rc, "point_chain_bn_f32")


def _chain_dw(dy_op, x_op, n_src, B, N, C, K, want_db):
    lib = _native.load()
    dev = torch.device("cuda", torch.cuda.current_device())
    dW = torch.empty((C, K), dtype=torch.float32, device=dev)
    db = torch.empty(C, dtype=torch.float32, device=dev) if want_db else None
    ws = _workspace(_chain_dw_ws, lib.point_chain_dw_workspace_bytes(B, N, C, K), dev, floor=0)
    rc = lib.point_chain_dw_f32(dy_op.ctypes.data, x_op.ctypes.data, n_src, B, N, dW.data_ptr(),
                                None if db is None else db.data_ptr(), ws.data_ptr(), ws.numel(), _stream_ptr())
    _native.check(rc, "point_chain_dw_f32")
    return dW, db


def _chain_product(op, n_src, W, widths, B, N):
    """W [R, sum(widths)] . the operand, [B, R, N]: in blocks of CHAIN_MAX_WIDTH output rows, the kernel's limit."""
    R = W.shape[0]
    outs = [_chain_gemm(op, n_src, _chain_pack(W[r:r + CHAIN_MAX_WIDTH], widths), None, None,
                        min(CHAIN_MAX_WIDTH, R - r), B, N, _EP_WRITE)[0] for r in range(0, R, CHAIN_MAX_WIDTH)]
    return outs[0] if len(outs) == 1 else torch.cat(outs, dim=1)


def _gather_cols(W, cols, widths):
    """The columns of W [C, C_in] that sources of `widths` starting at layer columns `cols` feed, in source order."""
    if all(c == cols[0] + sum(widths[:i]) for i, c in enumerate(cols)):
        return W[:, cols[0]:cols[0] + sum(widths)]
    return torch.cat([W[:, c:c + w] for c, w in zip(cols, widths)], dim=1)


class _PointChain(torch.autograd.Function):
    """Inputs: (layers, drop_state, n_src, cols, add, add_group, max_group, output, *sources, *per-layer (W, b, gamma,
    beta)); gamma / beta are None for a layer without BatchNorm; cols: layer 1's first column of each source.  The BN
    buffers of `layers` are updated in place."""

    @staticmethod
    def forward(ctx, layers, drop_state, n_src, cols, add, add_group, max_group, output, *tensors):
        sources = list(tensors[:n_src])
        B, N = sources[0].shape[0], sources[0].shape[2]
        dev = sources[0].device
        # the masks of this call: a copy of (seed, offset) taken before the offset advances, so a replayed graph draws
        # new ones and the backward recomputes these
        drop = None
        if any(layer.dropout is not None for layer in layers):
            drop = drop_state.clone()
            drop_state[1:].add_(1)
        widths = [s.shape[1] for s in sources]
        op = _chain_operand(sources)
        ys, stats_all = [], []
        with torch.cuda.device(dev):
            for l, layer in enumerate(layers):
                conv, norm = layer.conv, layer.norm
                C = conv.out_channels
                W = conv.weight.detach().reshape(C, -1)
                packed = _chain_pack(_gather_cols(W, cols, widths) if l == 0 else W, widths)
                bias = None if conv.bias is None else conv.bias.detach()
                y, part = _chain_gemm(op, len(widths), packed, bias, add if l == 0 else None, C, B, N,
                                      _EP_STATS if norm is not None else _EP_WRITE, add_group=add_group)
                st = None
                if norm is not None:
                    st = torch.empty((4, C), dtype=torch.float32, device=dev)
                    with torch.no_grad():
                        _chain_bn(part, B, N, C, norm, st, grad=False)
                    d = None if layer.dropout is None else (drop, float(layer.dropout.p))
                    op = _chain_operand([y], _OP_ACT, st, drop=d, layer=l)
                else:
                    op = _chain_operand([y])
                ys.append(y)
                stats_all.append(st)
                widths = [C]
            last = layers[-1]
            idx = None
            if max_group is not None:            # the group max fused into the last layer's BN + ReLU pass
                act, mx, idx = _chain_group_max(op, B, N, last.conv.out_channels, max_group, output == "both")
                out = mx if output == "max" else (act, mx)
            elif last.norm is not None:
                out, _ = _chain_gemm(op, 1, None, None, None, last.conv.out_channels, B, N, _EP_WRITE)
            else:
                out = ys[-1]
        # the sources and the pre-norm outputs go through save_for_backward only: autograd then catches an in-place change
        # to a source before the backward, and the chain's output, which can be one of the outputs, is not held on ctx
        # (that would tie the autograd graph into a reference cycle)
        ctx.layers, ctx.n_src, ctx.cols, ctx.has_add = layers, n_src, cols, add is not None
        ctx.add_group, ctx.max_group, ctx.output = add_group, max_group, output
        ctx.stats, ctx.drop, ctx.shape = stats_all, drop, (B, N)
        ctx.save_for_backward(*sources, *ys, *(() if idx is None else (idx,)))
        return out

    @staticmethod
    def backward(ctx, *grad_outs):
        layers, (B, N), n_src = ctx.layers, ctx.shape, ctx.n_src
        saved = ctx.saved_tensors
        sources, ys = saved[:n_src], saved[n_src:n_src + len(layers)]
        grad_out = grad_outs[-1]                 # the activations', or the group max's
        g_dense = grad_outs[0].float().contiguous() if ctx.output == "both" else None
        dev = ys[0].device
        L = len(layers)
        grads = [None] * (4 * L)
        g_src = [None] * n_src
        g_add = None
        with torch.cuda.device(dev):
            G = grad_out.float().contiguous()
            dz = None
            for l in range(L - 1, -1, -1):
                layer = layers[l]
                conv, norm = layer.conv, layer.norm
                C = conv.out_channels
                y, st = ys[l], ctx.stats[l]
                d = None if layer.dropout is None else (ctx.drop, float(layer.dropout.p))
                if norm is not None:
                    if l == L - 1 and ctx.max_group is not None:
                        dz, part = _chain_gemm(_chain_max_grad_operand(G, saved[-1], ctx.max_group), 1, None, None,
                                               g_dense, C, B, N, _EP_ACT_GRAD, _chain_act_row(st, d, l), y)
                    elif l == L - 1:
                        dz, part = _chain_gemm(_chain_operand([G]), 1, None, None, None, C, B, N, _EP_ACT_GRAD,
                                               _chain_act_row(st, d, l), y)
                    dgamma, dbeta, coef = _chain_bn(part, B, N, C, norm, st, grad=True)
                    dy_op = _chain_operand([dz], _OP_BN_GRAD, coef, y)
                    grads[4 * l + 2], grads[4 * l + 3] = dgamma, dbeta
                else:
                    dy_op = _chain_operand([G])
                if l == 0:
                    x_op, nx = _chain_operand(sources), n_src
                else:
                    prev = layers[l - 1]
                    dp = None if prev.dropout is None else (ctx.drop, float(prev.dropout.p))
                    x_op, nx = _chain_operand([ys[l - 1]], _OP_ACT, ctx.stats[l - 1], drop=dp, layer=l - 1), 1
                widths = [s.shape[1] for s in sources]
                K = conv.in_channels if l > 0 else sum(widths)
                dW, db = _chain_dw(dy_op, x_op, nx, B, N, C, K, conv.bias is not None)
                # dW's columns are in source order: scatter them to the layer's columns unless the sources are its
                # columns 0 .. C_in in order (the rest, where `add` stands for them, get zero)
                if l == 0 and (K != conv.in_channels or
                               list(ctx.cols) != [sum(widths[:i]) for i in range(len(widths))]):
                    full = dW.new_zeros((C, conv.in_channels))
                    r = 0
                    for c0, w in zip(ctx.cols, widths):
                        full[:, c0:c0 + w] = dW[:, r:r + w]
                        r += w
                    dW = full
                grads[4 * l], grads[4 * l + 1] = dW.view_as(conv.weight), db
                W = conv.weight.detach().reshape(C, conv.in_channels)
                if l == 0:
                    W = _gather_cols(W, ctx.cols, widths)
                if l > 0:
                    prev = layers[l - 1]
                    dp = None if prev.dropout is None else (ctx.drop, float(prev.dropout.p))
                    dz, part = _chain_gemm(dy_op, 1, _chain_pack(W.t().contiguous(), [C]), None, None, K, B, N,
                                           _EP_ACT_GRAD, _chain_act_row(ctx.stats[l - 1], dp, l - 1), ys[l - 1])
                else:
                    if ctx.has_add and ctx.needs_input_grad[4]:
                        if ctx.add_group > 1:         # layer 1's dY summed over each group, in column order
                            g_add = _chain_group_sum(dy_op, B, N, C, ctx.add_group)
                        else:
                            g_add = G if norm is None else _chain_gemm(dy_op, 1, None, None, None, C, B, N,
                                                                       _EP_WRITE)[0]
                    if any(ctx.needs_input_grad[8:8 + n_src]):
                        gx = _chain_product(dy_op, 1, W.t(), [C], B, N)
                        r = 0
                        for i, s in enumerate(sources):
                            if ctx.needs_input_grad[8 + i]:
                                g_src[i] = gx[:, r:r + s.shape[1]]
                            r += s.shape[1]
        return (None, None, None, None, g_add, None, None, None, *g_src, *grads)


def _check_chain_args(sources, layers, drop_state, add, in_col, training):
    if not isinstance(layers, (list, tuple)) or not 1 <= len(layers) <= CHAIN_MAX_LAYERS:
        raise ValueError(f"layers: need a list of 1 to {CHAIN_MAX_LAYERS} point layers")
    if not isinstance(sources, (list, tuple)) or not 1 <= len(sources) <= CHAIN_MAX_SOURCES:
        raise ValueError(f"sources: need a list of 1 to {CHAIN_MAX_SOURCES} sources")
    c_in = 0
    for i, layer in enumerate(layers):
        conv = getattr(layer, "conv", None)
        if not isinstance(conv, torch.nn.Conv1d) or conv.kernel_size != (1,) or conv.groups != 1:
            raise TypeError(f"layers[{i}]: need a point layer with a 1x1 Conv1d `conv`")
        if not 1 <= conv.out_channels <= CHAIN_MAX_WIDTH:
            raise ValueError(f"layers[{i}]: need 1 <= C_out <= {CHAIN_MAX_WIDTH}, got {conv.out_channels}")
        if i > 0 and conv.in_channels != layers[i - 1].conv.out_channels:
            raise ValueError(f"layers[{i}]: has {conv.in_channels} input channels, layers[{i - 1}] gives "
                             f"{layers[i - 1].conv.out_channels}")
        if i < len(layers) - 1 and layer.norm is None:
            raise ValueError(f"layers[{i}]: only the last layer may go without BatchNorm + ReLU")
        if layer.norm is not None:
            if not isinstance(layer.norm, torch.nn.BatchNorm1d) or not layer.norm.affine \
                    or not layer.norm.track_running_stats:
                raise TypeError(f"layers[{i}]: the norm must be an affine BatchNorm1d with running statistics")
            if training and layer.norm.momentum is None:
                raise ValueError(f"layers[{i}]: a cumulative BatchNorm (momentum None) is not supported")
        if layer.dropout is not None and layer.norm is None:
            raise ValueError(f"layers[{i}]: dropout needs BatchNorm + ReLU on the same layer")
        if i == 0:
            c_in = conv.in_channels
    if c_in > CHAIN_MAX_IN:
        raise ValueError(f"layers[0]: more than {CHAIN_MAX_IN} input channels")
    rows, B, N, dev = 0, None, None, layers[0].conv.weight.device
    for i, s in enumerate(sources):
        if not isinstance(s, torch.Tensor):
            raise TypeError(f"sources[{i}] must be a torch.Tensor")
        if s.dim() != 3 or s.shape[1] < 1:
            raise ValueError(f"sources[{i}] must be [B,C,N] with C >= 1")
        if s.dtype != torch.float32:
            raise TypeError(f"sources[{i}] must have dtype torch.float32")
        if s.device != dev:
            raise ValueError(f"sources[{i}] must be on {dev}, the layers' device")
        if B is None:
            B, N = s.shape[0], s.shape[2]
        elif (s.shape[0], s.shape[2]) != (B, N):
            raise ValueError(f"sources[{i}] has B, N = {s.shape[0]}, {s.shape[2]}; sources[0] has {B}, {N}")
        rows += s.shape[1]
    if not isinstance(in_col, int) or isinstance(in_col, bool) or in_col < 0:
        raise TypeError(f"in_col must be a non-negative int, got {in_col!r}")
    if add is None and (in_col != 0 or rows != c_in):
        raise ValueError(f"sources: {rows} rows from column {in_col}; without `add` they must be all {c_in} columns "
                         f"of layers[0]")
    if in_col + rows > c_in:
        raise ValueError(f"sources: {rows} rows from column {in_col} exceed layers[0]'s {c_in} input columns")
    if not 1 <= B <= MLP_MAX_BATCH or N < 1:
        raise ValueError(f"sources: need 1 <= B <= {MLP_MAX_BATCH} and N >= 1, got B = {B}, N = {N}")
    if add is not None:
        if not isinstance(add, torch.Tensor):
            raise TypeError("add must be a torch.Tensor or None")
        if add.dtype != torch.float32:
            raise TypeError("add must have dtype torch.float32")
        if tuple(add.shape) != (B, layers[0].conv.out_channels, N) or add.device != dev:
            raise ValueError(f"add must be [{B}, {layers[0].conv.out_channels}, {N}] on {dev}")
    if training and any(layer.dropout is not None for layer in layers):
        if not isinstance(drop_state, torch.Tensor):
            raise TypeError("drop_state must be a torch.Tensor: int64 [2] (seed, offset) on the layers' device")
        if drop_state.dtype != torch.int64 or tuple(drop_state.shape) != (2,) or drop_state.device != dev \
                or not drop_state.is_contiguous():
            raise ValueError("drop_state must be a contiguous int64 [2] (seed, offset) on the layers' device")
    for i, layer in enumerate(layers):
        conv, norm = layer.conv, layer.norm
        for name, t in (("weight", conv.weight), ("bias", conv.bias)) + (
                (("norm.weight", norm.weight), ("norm.bias", norm.bias), ("norm.running_mean", norm.running_mean),
                 ("norm.running_var", norm.running_var)) if norm is not None else ()):
            if t is not None and (not t.is_cuda or t.dtype != torch.float32):
                raise TypeError(f"layers[{i}].{name} must be a float32 CUDA tensor")
    return B, N


def new_dropout_state(seed, device):
    """A point_chain dropout state: int64 [2] (seed, offset 0) on `device`."""
    return torch.tensor([int(seed) & 0x7FFFFFFFFFFFFFFF, 0], dtype=torch.int64, device=device)


def point_chain(sources, layers, training, drop_state=None, add=None, in_col=0):
    """A chain of one to three of the classifier's point layers (network._PointLayer: 1x1 Conv1d, then BatchNorm1d +
    ReLU and Dropout where the layer has them) over [B,C,N] points (DESIGN.md 4.34).

    sources: 1 to 4 float32 CUDA tensors [B,C_i,N] whose rows, in order, are layer 1's input (never concatenated).
    layers: the chain's _PointLayer modules as they are; only the last may lack BatchNorm + ReLU.

    training=True runs the layers in train mode as one differentiable op: products on the tensor cores in TF32 with
    float32 accumulation whatever torch's TF32 flags say; BatchNorm with the batch's statistics (fp64 per-tile sums
    reduced in a fixed order), the running statistics and num_batches_tracked updated as nn.BatchNorm1d does; dropout
    masks from counter-based Philox keyed by drop_state (int64 [2] (seed, offset) on the device, needed when a layer
    has dropout), whose offset the op advances on the device; add: an optional [B,C_1,N] term added to layer 1 before
    its BatchNorm, standing for the input columns the sources do not feed (the sources feed columns [in_col, in_col +
    their rows) of layer 1's weight, and layer 1's weight gradient is zero outside them).  Only each layer's pre-norm output is kept for the backward, which returns gradients for every
    parameter, every source and `add`, deterministically (no atomics, fixed summation orders).  The masks differ from
    torch's Dropout's.

    Up to 1024 source rows; every layer's C_out is at most 256.

    training=False is the eval-mode chain: fold_pointnet + pointwise_mlp, and `add` is not taken (give pointwise_mlp's
    interpolated sources instead).  It has no backward, so under grad mode a source or layer parameter that requires
    grad raises RuntimeError instead of returning an output cut off from autograd.  Errors name the argument: ValueError for shapes and widths,
    TypeError for types and dtypes."""
    if training:
        B, N = _check_chain_args(sources, layers, drop_state, add, in_col, True)
        flat = []
        for layer in layers:
            norm = layer.norm
            flat += [layer.conv.weight, layer.conv.bias, None if norm is None else norm.weight,
                     None if norm is None else norm.bias]
        srcs = []
        for s in sources:
            if (N > 1 and s.stride(2) != 1) or (s.shape[1] > 1 and s.stride(1) != N) \
                    or (B > 1 and s.stride(0) < s.shape[1] * N):
                s = s.contiguous()
            srcs.append(s)
        cols = [in_col + sum(s.shape[1] for s in srcs[:i]) for i in range(len(srcs))]
        return _PointChain.apply(list(layers), drop_state, len(srcs), cols, None if add is None else add.contiguous(),
                                 1, None, "activations", *srcs, *flat)
    if add is not None or in_col != 0:
        raise ValueError("add, in_col: the eval-mode chain takes interpolated sources instead of an additive term")
    if not isinstance(layers, (list, tuple)) or not 1 <= len(layers) <= CHAIN_MAX_LAYERS:
        raise ValueError(f"layers: need a list of 1 to {CHAIN_MAX_LAYERS} point layers")
    if torch.is_grad_enabled():
        flat = [t for s in sources for t in ((s,) if isinstance(s, torch.Tensor) else s)]
        if any(isinstance(t, torch.Tensor) and t.requires_grad for t in flat) or \
                any(p.requires_grad for layer in layers for p in layer.parameters()):
            raise RuntimeError("point_chain in eval mode (training=False) has no backward: call it under "
                               "torch.no_grad(), or detach the sources and freeze the layers")
    import types
    from .network import fold_pointnet
    return pointwise_mlp(list(sources), fold_pointnet(types.SimpleNamespace(layers=list(layers))))


def _check_branch_args(sources, layers, drop_state, cols, add, add_group, max_group, output):
    if not isinstance(layers, (list, tuple)) or not 1 <= len(layers) <= CHAIN_MAX_LAYERS:
        raise ValueError(f"layers: need a list of 1 to {CHAIN_MAX_LAYERS} point layers")
    if not isinstance(sources, (list, tuple)) or not 1 <= len(sources) <= CHAIN_MAX_SOURCES:
        raise ValueError(f"sources: need a list of 1 to {CHAIN_MAX_SOURCES} sources")
    for i, layer in enumerate(layers):
        conv, norm = getattr(layer, "conv", None), getattr(layer, "norm", None)
        if not isinstance(conv, (torch.nn.Conv1d, torch.nn.Conv2d)) or any(k != 1 for k in conv.kernel_size) \
                or conv.groups != 1:
            raise TypeError(f"layers[{i}]: need a point layer with a 1x1 Conv1d or Conv2d `conv`")
        if not 1 <= conv.out_channels <= BRANCH_MAX_WIDTH:
            raise ValueError(f"layers[{i}]: need 1 <= C_out <= {BRANCH_MAX_WIDTH}, got {conv.out_channels}")
        if i > 0 and conv.in_channels != layers[i - 1].conv.out_channels:
            raise ValueError(f"layers[{i}]: has {conv.in_channels} input channels, layers[{i - 1}] gives "
                             f"{layers[i - 1].conv.out_channels}")
        if i < len(layers) - 1 and norm is None:
            raise ValueError(f"layers[{i}]: only the last layer may go without BatchNorm + ReLU")
        if norm is not None and (not isinstance(norm, (torch.nn.BatchNorm1d, torch.nn.BatchNorm2d))
                                 or not norm.affine or not norm.track_running_stats or norm.momentum is None):
            raise TypeError(f"layers[{i}]: the norm must be an affine BatchNorm1d / 2d with running statistics and "
                            f"a momentum")
        if layer.dropout is not None and norm is None:
            raise ValueError(f"layers[{i}]: dropout needs BatchNorm + ReLU on the same layer")
    c_in, dev = layers[0].conv.in_channels, layers[0].conv.weight.device
    B = N = None
    for i, s in enumerate(sources):
        if not isinstance(s, torch.Tensor) or s.dtype != torch.float32:
            raise TypeError(f"sources[{i}] must be a float32 torch.Tensor")
        if s.dim() != 3 or s.shape[1] < 1 or s.device != dev:
            raise ValueError(f"sources[{i}] must be [B,C,N] with C >= 1 on {dev}, the layers' device")
        if B is None:
            B, N = s.shape[0], s.shape[2]
        elif (s.shape[0], s.shape[2]) != (B, N):
            raise ValueError(f"sources[{i}] has B, N = {s.shape[0]}, {s.shape[2]}; sources[0] has {B}, {N}")
    if not 1 <= B <= MLP_MAX_BATCH or N < 1:
        raise ValueError(f"sources: need 1 <= B <= {MLP_MAX_BATCH} and N >= 1, got B = {B}, N = {N}")
    if sum(s.shape[1] for s in sources) > CHAIN_MAX_IN:
        raise ValueError(f"sources: more than {CHAIN_MAX_IN} rows")
    if not isinstance(cols, (list, tuple)) or len(cols) != len(sources) or \
            any(not isinstance(c, int) or isinstance(c, bool) or c < 0 for c in cols):
        raise ValueError("cols: need one non-negative int per source, its first column of layers[0]")
    spans = sorted((c, c + s.shape[1]) for c, s in zip(cols, sources))
    if spans[-1][1] > c_in or any(a[1] > b[0] for a, b in zip(spans, spans[1:])):
        raise ValueError(f"cols: the sources' column ranges {spans} overlap or exceed layers[0]'s {c_in} columns")
    if add is None and sum(s.shape[1] for s in sources) != c_in:
        raise ValueError(f"sources: without `add` they must feed all {c_in} columns of layers[0]")
    for g, name in ((add_group, "add_group"), (max_group, "max_group")):
        if g is not None and (not isinstance(g, int) or isinstance(g, bool) or g < 1 or N % g):
            raise ValueError(f"{name} must be an int >= 1 that divides N = {N}, got {g!r}")
    if add is not None:
        if not isinstance(add, torch.Tensor) or add.dtype != torch.float32:
            raise TypeError("add must be a float32 torch.Tensor or None")
        C1 = layers[0].conv.out_channels
        if tuple(add.shape) != (B, C1, N // add_group) or add.device != dev:
            raise ValueError(f"add must be [{B}, {C1}, {N // add_group}] (N / add_group columns) on {dev}")
    if output not in ("activations", "max", "both"):
        raise ValueError(f"output must be 'activations', 'max' or 'both', got {output!r}")
    if (output != "activations") != (max_group is not None):
        raise ValueError("max_group: output 'max' and 'both' need it, 'activations' takes none")
    if max_group is not None and layers[-1].norm is None:
        raise ValueError("max_group: the group max is taken after the last layer's BatchNorm + ReLU")
    if any(layer.dropout is not None for layer in layers):
        if not isinstance(drop_state, torch.Tensor) or drop_state.dtype != torch.int64 \
                or tuple(drop_state.shape) != (2,) or drop_state.device != dev or not drop_state.is_contiguous():
            raise ValueError("drop_state must be a contiguous int64 [2] (seed, offset) on the layers' device")
    for i, layer in enumerate(layers):
        norm = layer.norm
        for t in list(layer.parameters()) + ([norm.running_mean, norm.running_var] if norm is not None else []):
            if not t.is_cuda or t.dtype != torch.float32:
                raise TypeError(f"layers[{i}]: every parameter and running statistic must be a float32 CUDA tensor")
    return B, N


def point_branch(sources, layers, drop_state=None, cols=None, add=None, add_group=1, max_group=None,
                 output="activations"):
    """point_chain in train mode, generalised to the point encoder's kNN module, final_pointnet and the decoder's
    node-level PointNets (DESIGN.md 4.36): the same kernels, rules and determinism, plus

    - 1x1 Conv2d + BatchNorm2d layers (the kNN module's): a [B,C,M,K] input is passed viewed as [B,C,M*K], and
      BatchNorm2d's statistics over B*M*K are the chain's over its columns;
    - layers up to BRANCH_MAX_WIDTH (1024) rows wide, run as row blocks into one pre-norm tensor;
    - cols: layer 1's first column of each source (default: the sources in order from column 0); the columns no
      source feeds stand for `add`, and layer 1's weight gradient is zero there;
    - add [B, C_1, N / add_group]: added to layer 1 at column n from entry n // add_group (a projected per-node max
      with add_group = K, a projected per-sample input with add_group = N); its gradient is layer 1's dY summed over
      each group in column order in fp64;
    - max_group: the max of the last layer's activations over groups of max_group consecutive columns by torch.max's
      rule (first maximal index; a NaN propagates), [B, C, N / max_group], fused into the BN + ReLU pass; the backward
      reads the compact gradient at the saved in-group index.  output "max" returns the max only (the activations are
      never written), "both" returns (activations, max).

    Train mode only; errors name the argument."""
    if cols is None and isinstance(sources, (list, tuple)):
        cols = [sum(s.shape[1] for s in sources[:i]) for i in range(len(sources))]
    B, N = _check_branch_args(sources, layers, drop_state, cols, add, add_group, max_group, output)
    flat = []
    for layer in layers:
        norm = layer.norm
        flat += [layer.conv.weight, layer.conv.bias, None if norm is None else norm.weight,
                 None if norm is None else norm.bias]
    srcs = [s.contiguous() if (N > 1 and s.stride(2) != 1) or (s.shape[1] > 1 and s.stride(1) != N)
            or (B > 1 and s.stride(0) < s.shape[1] * N) else s for s in sources]
    return _PointChain.apply(list(layers), drop_state, len(srcs), list(cols),
                             None if add is None else add.contiguous(), add_group, max_group, output, *srcs, *flat)


class _ChannelProduct(torch.autograd.Function):
    @staticmethod
    def forward(ctx, W, x):
        B, K, M = x.shape
        with torch.cuda.device(x.device):
            out = _chain_product(_chain_operand([x.detach()]), 1, W.detach(), [K], B, M)
        ctx.save_for_backward(W, x)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        W, x = ctx.saved_tensors
        B, K, M = x.shape
        C = W.shape[0]
        gW = gx = None
        with torch.cuda.device(x.device):
            G = grad_out.float().contiguous()
            g_op = _chain_operand([G])
            if ctx.needs_input_grad[0]:
                gW, _ = _chain_dw(g_op, _chain_operand([x.detach()]), 1, B, M, C, K, False)
            if ctx.needs_input_grad[1]:
                gx = _chain_product(g_op, 1, W.detach().t(), [C], B, M)
        return gW, gx


def channel_product(W, x):
    """W [C, K] . x [B, K, M] -> [B, C, M] float32: a 1x1 layer without bias over the M columns of each sample, on the
    chain kernels of point_chain (TF32 tensor-core products with float32 accumulation, the weight gradient summed over
    the columns in a fixed order), so it is deterministic without cuBLAS.  Differentiable in W and x; 1 <= K, C <=
    CHAIN_MAX_IN.  KeypointDetector(point_layers="fused") applies the head's pa / pb weight columns at the nodes with
    it."""
    for t, name in ((W, "W"), (x, "x")):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{name} must be a torch.Tensor")
        if t.dtype != torch.float32:
            raise TypeError(f"{name} must have dtype torch.float32")
    for t, name in ((W, "W"), (x, "x")):
        if not t.is_cuda:
            raise ValueError(f"{name} must be a CUDA tensor")
    if W.dim() != 2 or x.dim() != 3 or W.shape[1] != x.shape[1]:
        raise ValueError(f"W must be [C, K] and x [B, K, M] with the same K, got {tuple(W.shape)} and {tuple(x.shape)}")
    if not 1 <= W.shape[0] <= CHAIN_MAX_IN or not 1 <= W.shape[1] <= CHAIN_MAX_IN:
        raise ValueError(f"W: need 1 <= C, K <= {CHAIN_MAX_IN}, got {tuple(W.shape)}")
    if not 1 <= x.shape[0] <= MLP_MAX_BATCH or x.shape[2] < 1:
        raise ValueError(f"x: need 1 <= B <= {MLP_MAX_BATCH} and M >= 1, got {tuple(x.shape)}")
    if x.device != W.device:
        raise ValueError(f"x must be on {W.device}, W's device")
    return _ChannelProduct.apply(W, x.contiguous())


def point_chain_dropout_mask(drop_state, layer, p, B, C, N):
    """The keep bits point_chain draws for layer `layer` (0-based in its chain) of dropout probability p under
    drop_state (the (seed, offset) pair as it was when the call began): uint8 [B,C,N], 1 = kept.  For references that
    have to use the same mask."""
    if not isinstance(drop_state, torch.Tensor) or drop_state.dtype != torch.int64 or tuple(drop_state.shape) != (2,) \
            or not drop_state.is_cuda:
        raise ValueError("drop_state must be a CUDA int64 [2] (seed, offset)")
    if not 0 <= p < 1:
        raise ValueError(f"p: need 0 <= p < 1, got {p}")
    lib = _native.load()
    dev = drop_state.device
    with torch.cuda.device(dev):
        out = torch.empty((B, C, N), dtype=torch.uint8, device=dev)
        rc = lib.point_chain_dropout_mask(drop_state.contiguous().data_ptr(), int(layer), float(p), B, C, N,
                                          out.data_ptr(), _stream_ptr())
    _native.check(rc, "point_chain_dropout_mask")
    return out
