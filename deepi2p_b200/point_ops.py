"""Host side of index_max / ball_query: torch tensors in, torch tensors out, kernels via the C ABI.

Mirrors the reference's extension modules (models/index_max_ext/index_max.cpp:119-159,
models/ball_query_ext/ball_query.cpp:23-48): same argument checks (CUDA + contiguous ->
RuntimeError), output allocated on the input's device, int32 outputs.  Unlike the reference the
kernels are launched on torch's *current* stream of the tensor's device, not the legacy default
stream (SURVEY.md 8b).
"""
import torch

from . import _native


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
        rc = lib.index_max_forward(data.data_ptr(), index.data_ptr(), out.data_ptr(), B, C, N, K,
                                   torch.cuda.current_stream().cuda_stream)
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
                                    torch.cuda.current_stream().cuda_stream)
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
        need = lib.ball_query_xyz_workspace_bytes(B, N)
        key = (dev.index, torch.cuda.current_stream().cuda_stream)     # one scratch per stream: launches may overlap
        ws = _xyz_ws.get(key)
        if ws is None or ws.numel() < need:
            ws = torch.empty(max(need, 1 << 20), dtype=torch.uint8, device=dev)
            _xyz_ws[key] = ws
        out = torch.empty((B, M, K), dtype=torch.int32, device=dev)
        rc = lib.ball_query_xyz_forward(points.data_ptr(), nodes.data_ptr(), float(radius), out.data_ptr(), B, M, N, K,
                                        ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream)
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
        need = lib.cluster_assign_workspace_bytes(B, M)
        key = (dev.index, torch.cuda.current_stream().cuda_stream)
        ws = _ca_ws.get(key)
        if ws is None or ws.numel() < need:
            ws = torch.empty(max(need, 1 << 16), dtype=torch.uint8, device=dev)
            _ca_ws[key] = ws
        topk = torch.empty((B, N, k), dtype=torch.int32, device=dev)
        min_idx = torch.empty((B, N), dtype=torch.int32, device=dev)
        count = torch.empty((B, M), dtype=torch.int32, device=dev)
        mean = torch.empty((B, 3, M), dtype=torch.float32, device=dev)
        centers = torch.empty((B, 3, N), dtype=torch.float32, device=dev) if want_centers else None
        dec = torch.empty((B, 3, N), dtype=torch.float32, device=dev) if want_centers else None
        rc = lib.cluster_assign_forward(pc.data_ptr(), node.data_ptr(), B, N, M, k, topk.data_ptr(), min_idx.data_ptr(),
                                        count.data_ptr(), mean.data_ptr(),
                                        centers.data_ptr() if want_centers else 0,
                                        dec.data_ptr() if want_centers else 0, ws.data_ptr(), ws.numel(),
                                        torch.cuda.current_stream().cuda_stream)
    _native.check(rc, "cluster_assign_forward")
    return dict(min_k_idx=topk, min_idx=min_idx, count=count, cluster_mean=mean, pc_centers=centers,
                pc_decentered=dec)


INTERP_MAX_K = 8
INTERP_MAX_NODES = 2048
_interp_ws = {}


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
                stream = torch.cuda.current_stream().cuda_stream
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
                stream = torch.cuda.current_stream().cuda_stream
                need = lib.interp_backward_workspace_bytes(B, C, Nq, M)
                key = (dev.index, stream)
                ws = _interp_ws.get(key)
                if ws is None or ws.numel() < need:
                    ws = torch.empty(max(need, 1 << 16), dtype=torch.uint8, device=dev)
                    _interp_ws[key] = ws
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
