"""Host side of the registration path: thin Python over the C ABI (include/deepi2p_b200.h).

torch is used only for device memory, streams and pinned host buffers; every computation is a
hand-written sm_90a kernel reached through ctypes.  No CPU fallback exists: without a CUDA
device or without the compiled library every entry point raises.

Mirrors, in order of the reference's call stack (SURVEY.md 3.1):
  register_batch      <- the per-sample body of evaluation/registration_lsq.py:329-343
                         (get_initial_guess + solve_P_random_perturb), batched and on device
  solve_batch         <- the 60 x solvePGivenK loop of registration_lsq.py:142-186, one launch
  solve_p_given_k     <- FrustumRegistration.solvePGivenK (registration.cpp:9-186)
"""
import math

import numpy as np
import torch

from . import _native
from ._native import _ptr, _require_cuda, _stream_ptr, _workspace

DEFAULT_T_LB = (-5.0, -0.1, -10.0)      # registration_lsq.py:340
DEFAULT_T_UB = (5.0, 0.1, 10.0)
RY_SIGMA = 10.0 * math.pi / 180.0       # registration_lsq.py:339
T_AMPLITUDE = 10.0                      # registration_lsq.py:337
TERMINATION = ("gradient_tolerance", "parameter_tolerance", "function_tolerance", "max_iterations",
               "min_trust_region_radius", "invalid_steps", "infeasible_start")


def round_up(n, m):
    return (n + m - 1) // m * m


def pack_clouds(points, labels, device="cuda", n_pts=None, dtype=None):
    """Host clouds -> device record (xyz [S,3,Ns], label int8 [S,Ns], n_pts int32 [S]).

    points: array [S,3,N] (or [3,N]); labels: [S,N] ints (1 inside, 0 outside, anything else
    ignored).  Coordinates are stored as float32 when that is lossless (the loaders produce
    float32: data/kitti_pc_img_pose_loader.py:431), otherwise as float64.
    """
    pts = np.asarray(points)
    lab = np.asarray(labels)
    if pts.ndim == 2:
        pts, lab = pts[None], lab[None]
    S, three, N = pts.shape
    if three != 3 or lab.shape != (S, N):
        raise ValueError("points must be [S,3,N] and labels [S,N]")
    if dtype is None:
        if pts.dtype == np.float32:
            dtype = np.float32
        else:
            p32 = pts.astype(np.float32)
            dtype = np.float32 if np.array_equal(p32.astype(pts.dtype), pts) else np.float64
    Ns = round_up(max(N, 1), 16)
    xyz = np.zeros((S, 3, Ns), dtype=dtype)
    xyz[:, :, :N] = pts
    l8 = np.full((S, Ns), -1, dtype=np.int8)
    l8[:, :N] = np.where(lab == 1, 1, np.where(lab == 0, 0, -1))
    if n_pts is None:
        n_pts = np.full(S, N, dtype=np.int32)
    dev = torch.device(device)
    return (torch.from_numpy(xyz).to(dev), torch.from_numpy(l8).to(dev),
            torch.from_numpy(np.asarray(n_pts, dtype=np.int32)).to(dev))


def _as_K(K, S, device):
    K = torch.as_tensor(K, dtype=torch.float64)
    if K.numel() == 9:
        K = K.reshape(1, 9).expand(S, 9)
    K = K.reshape(S, 9).contiguous()
    return K.to(device)


def _check_cloud(xyz, label=None, n_pts=None, what="xyz", dtypes=(torch.float32, torch.float64)):
    """Shape / device / layout checks shared by every wrapper that hands raw pointers to the C ABI: a CPU tensor or a
    sliced view would otherwise be read as if it were a contiguous device array."""
    if not isinstance(xyz, torch.Tensor) or not xyz.is_cuda:
        raise ValueError(f"{what} must be a CUDA tensor")
    if xyz.dim() != 3 or xyz.shape[1] != 3:
        raise ValueError(f"{what} must be [S,3,Ns]")
    if xyz.dtype not in dtypes:
        raise ValueError(f"{what} must be one of {dtypes}")
    if not xyz.is_contiguous():
        raise ValueError(f"{what} must be contiguous (a sliced view would be read with the wrong stride)")
    S, _, Ns = xyz.shape
    if Ns % 16 != 0:
        raise ValueError("the point stride must be a multiple of 16 (pack_clouds pads)")
    if label is not None:
        if not (isinstance(label, torch.Tensor) and label.is_cuda and label.device == xyz.device):
            raise ValueError("label must be a CUDA tensor on the same device")
        if label.dtype != torch.int8 or tuple(label.shape) != (S, Ns) or not label.is_contiguous():
            raise ValueError("label must be a contiguous int8 [S,Ns] tensor")
    if n_pts is not None:
        if not (isinstance(n_pts, torch.Tensor) and n_pts.numel() == S):
            raise ValueError("n_pts must hold S entries")
    return S, Ns


_ws_cache = {}      # scratch of the solver, shared with the other wrappers that launch on its streams (1 MiB floor)


def last_solve_timeline(device=None, stream=None, register_shape=None):
    """(start_ns, queue_empty_ns, end_ns) of the most recent solve launched with this (device, stream)'s workspace, read
    from the timeline words the solver kernel writes next to its queue counter (globaltimer nanoseconds).  Benchmark
    aid: end - queue_empty is the end-of-kernel tail during which SMs run out of problems.
    register_shape = (S, I, n_in) when the last call was register_batch (the solver's block then sits behind the
    front-filtered clouds in the workspace)."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    key = (dev.index if dev.index is not None else torch.cuda.current_device(), int(_stream_ptr(stream)))
    buf = _ws_cache.get(key)
    if buf is None:
        return None
    off = 0
    if register_shape is not None:
        lib = _native.load()
        S, I, n_in = (int(v) for v in register_shape)
        off = lib.frustum_register_workspace_bytes(S, I, n_in) - lib.frustum_solve_workspace_bytes(S, I, round_up(n_in, 16))
    w = buf[off:off + 32].cpu().numpy().view(np.uint64)
    return int(w[1]), int(w[2]), int(w[3])


def last_solve_cta_end_times(device=None, stream=None, register_shape=None):
    """Exit time (globaltimer ns) of every CTA of the most recent solve, zeros removed -- with last_solve_timeline this
    shows whether the end-of-kernel tail is a few late SMs (imbalance) or all of them (critical path)."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    key = (dev.index if dev.index is not None else torch.cuda.current_device(), int(_stream_ptr(stream)))
    buf = _ws_cache.get(key)
    if buf is None:
        return None
    off = 0
    if register_shape is not None:
        lib = _native.load()
        S, I, n_in = (int(v) for v in register_shape)
        off = lib.frustum_register_workspace_bytes(S, I, n_in) - lib.frustum_solve_workspace_bytes(S, I, round_up(n_in, 16))
    w = buf[off + 256:off + 256 + 8192].cpu().numpy().view(np.uint64)
    return w[w > 0]


def solve_batch(xyz, label, n_pts, K, init, H, W, t_lb=DEFAULT_T_LB, t_ub=DEFAULT_T_UB, max_iter=500,
                is_2d=True, return_all=False, stream=None, out=None, trace_cap=0):
    """Batched multi-start solve, everything resident on the device.

    xyz [S,3,Ns] f32|f64 cuda, label [S,Ns] int8 cuda, n_pts [S] int32 cuda or None,
    K [S,9]|[9]|[3,3] f64, init [S,I,4] f64 = (init_y_angle, Tx, Ty, Tz) per problem.
    Returns dict(P [S,4,4], cost [S], best [S]) (+ params [S,I,6], costs [S,I], stats [S,I,4]
    = (LM iterations, cloud passes, line-search contractions, termination) if return_all).
    `out`: a dict returned by an earlier call with the same shapes; its tensors are overwritten in place
    (no allocation inside the call).
    trace_cap > 0 (float32 record only): additionally returns trace [S,I,trace_cap,16] f64, one record per cloud
    pass (layout: include/deepi2p_b200.h, frustum_solve_traced_f32) -- parity tooling.
    """
    _require_cuda()
    lib = _native.load()
    S, Ns = _check_cloud(xyz, label, n_pts)
    dev = xyz.device
    init = torch.as_tensor(init, dtype=torch.float64).to(dev).contiguous()
    if init.dim() != 3 or init.shape[0] != S or init.shape[2] != 4:
        raise ValueError("init must be [S,I,4]")
    I = init.shape[1]
    K9 = _as_K(K, S, dev)
    if n_pts is not None:
        n_pts = n_pts.to(dev, torch.int32).contiguous()
    lb = np.ascontiguousarray(np.asarray(t_lb, dtype=np.float64).reshape(3))
    ub = np.ascontiguousarray(np.asarray(t_ub, dtype=np.float64).reshape(3))
    with torch.cuda.device(dev):
        params = costs = stats = None
        if out is not None:
            P, cost, best = out["P"], out["cost"], out["best"]
            if tuple(P.shape) != (S, 4, 4) or P.device != dev:
                raise ValueError("out buffers do not match this batch")
            if return_all:
                params, costs, stats = out["params"], out["costs"], out["stats"]
                if tuple(params.shape) != (S, I, 6):
                    raise ValueError("out buffers do not match this batch")
        else:
            P = torch.empty((S, 4, 4), dtype=torch.float64, device=dev)
            cost = torch.empty((S,), dtype=torch.float64, device=dev)
            best = torch.empty((S,), dtype=torch.int32, device=dev)
            if return_all:
                params = torch.empty((S, I, 6), dtype=torch.float64, device=dev)
                costs = torch.empty((S, I), dtype=torch.float64, device=dev)
                stats = torch.empty((S, I, 4), dtype=torch.int32, device=dev)
        wsb = lib.frustum_solve_workspace_bytes(S, I, Ns)
        sp = _stream_ptr(stream)
        ws = _workspace(_ws_cache, wsb, dev, stream)
        trace = None
        if trace_cap > 0:
            if xyz.dtype != torch.float32:
                raise ValueError("the traced solve takes the float32 record")
            trace = torch.empty((S, I, int(trace_cap), 16), dtype=torch.float64, device=dev)
            rc = lib.frustum_solve_traced_f32(
                _ptr(xyz), _ptr(label), _ptr(n_pts), Ns, _ptr(K9), _ptr(init), lb.ctypes.data, ub.ctypes.data,
                float(H), float(W), int(max_iter), 1 if is_2d else 0, S, I, _ptr(P), _ptr(cost), _ptr(best),
                _ptr(params), _ptr(costs), _ptr(stats), _ptr(trace), int(trace_cap), _ptr(ws), ws.numel(), sp)
        else:
            fn = lib.frustum_solve_batch_f32 if xyz.dtype == torch.float32 else lib.frustum_solve_batch_f64
            rc = fn(_ptr(xyz), _ptr(label), _ptr(n_pts), Ns, _ptr(K9), _ptr(init), lb.ctypes.data, ub.ctypes.data,
                    float(H), float(W), int(max_iter), 1 if is_2d else 0, S, I, _ptr(P), _ptr(cost), _ptr(best),
                    _ptr(params), _ptr(costs), _ptr(stats), _ptr(ws), ws.numel(), sp)
    _native.check(rc, "frustum_solve_batch")
    res = dict(P=P, cost=cost, best=best)
    if trace is not None:
        res["trace"] = trace
    if return_all:
        res.update(params=params, costs=costs, stats=stats)
    return res


def evaluate_batch(xyz, label, n_pts, K, x, H, W, is_2d=True, stream=None, slice_rounds=4):
    """One cost / gradient / J^T J pass per sample at parameters x [S,6] (test hook).  slice_rounds: form the sums in
    slices of that many rounds of 1024 points (0 = in one piece) -- the solver uses frustum_solve_slice_rounds() from a
    problem's frustum_solve_slice_after()-th pass on and one piece before; the variants differ at rounding level, each
    reproduces the solver's own sums bit for bit."""
    _require_cuda()
    lib = _native.load()
    lib.dib_evaluate_sliced(int(slice_rounds))
    S, Ns = _check_cloud(xyz, label, n_pts)
    dev = xyz.device
    K9 = _as_K(K, S, dev)
    if n_pts is not None:
        n_pts = n_pts.to(dev, torch.int32).contiguous()
    x = torch.as_tensor(x, dtype=torch.float64).to(dev).contiguous().reshape(S, 6)
    with torch.cuda.device(dev):
        cost = torch.empty((S,), dtype=torch.float64, device=dev)
        grad = torch.empty((S, 6), dtype=torch.float64, device=dev)
        JtJ = torch.empty((S, 36), dtype=torch.float64, device=dev)
        sp = _stream_ptr(stream)
        ws = _workspace(_ws_cache, lib.frustum_evaluate_workspace_bytes(S, Ns), dev, stream)
        fn = lib.frustum_evaluate_f32 if xyz.dtype == torch.float32 else lib.frustum_evaluate_f64
        rc = fn(_ptr(xyz), _ptr(label), _ptr(n_pts), Ns, _ptr(K9), _ptr(x), float(H), float(W), 1 if is_2d else 0, S,
                _ptr(cost), _ptr(grad), _ptr(JtJ), _ptr(ws), ws.numel(), sp)
    _native.check(rc, "frustum_evaluate")
    P = 4 if is_2d else 6
    return cost, grad[:, :P], JtJ[:, :P * P].reshape(S, P, P)


def residuals(xyz, label, n, K, x, H, W, is_2d=True, stream=None, host_labels=None):
    """Loss-corrected residual vector of one cloud at x (registration.cpp:150-155).  host_labels: the labels as a host
    array if the caller still has them (the drop-in does) -- the row offsets are then a numpy prefix sum instead of four
    small torch kernels and a device->host read."""
    _require_cuda()
    lib = _native.load()
    dev = xyz.device
    Ns = xyz.shape[-1]
    if host_labels is not None:
        hl = np.asarray(host_labels).reshape(-1)[:n]
        rows = np.where(hl == 1, 3, np.where(hl == 0, 1, 0)).astype(np.int32)
        offs_h = np.cumsum(rows, dtype=np.int64) - rows
        total = int(rows.sum())
        offs = torch.from_numpy(offs_h.astype(np.int32)).to(dev)
    else:
        lab = label.reshape(-1)[:n]
        rows = torch.where(lab == 1, 3, torch.where(lab == 0, 1, 0)).to(torch.int32)
        offs = (torch.cumsum(rows, 0, dtype=torch.int32) - rows).contiguous()
        total = int(rows.sum().item())
    K9 = _as_K(K, 1, dev)
    xv = torch.as_tensor(x, dtype=torch.float64).reshape(-1)
    if xv.is_cuda and xv.numel() == 6:
        xx = xv.contiguous()
    else:
        xx = torch.zeros(6, dtype=torch.float64, device=dev)
        xx[:xv.numel()] = xv.to(dev)
    with torch.cuda.device(dev):
        res = torch.zeros((max(total, 1),), dtype=torch.float64, device=dev)
        fn = lib.frustum_residuals_f32 if xyz.dtype == torch.float32 else lib.frustum_residuals_f64
        rc = fn(_ptr(xyz), _ptr(label), int(n), Ns, _ptr(K9), _ptr(xx), float(H), float(W), 1 if is_2d else 0,
                _ptr(offs), _ptr(res), _stream_ptr(stream))
    _native.check(rc, "frustum_residuals")
    return res[:total]


def prepare_batch(xyz_in, pred, n_in, n_inits, seed=0, ry_sigma=RY_SIGMA, t_amp=T_AMPLITUDE, sort=True,
                  stream=None):
    """On-device get_initial_guess + init perturbation (registration_lsq.py:196-220, 163-164).

    xyz_in [S,3,Ns_in] f32 cuda, pred [S,Ns_in] int8 cuda.  sort=True additionally orders the kept
    points by (label, Morton cell) so that the solver's box culling bites.  Returns dict(xyz, label,
    n_pts, init, init_y_angle, degenerate) ready for solve_batch."""
    _require_cuda()
    lib = _native.load()
    S, Ns_in = _check_cloud(xyz_in, pred, what="xyz_in", dtypes=(torch.float32,))
    dev = xyz_in.device
    if not (0 <= int(n_in) <= Ns_in):
        raise ValueError("n_in must be within the point stride")
    Ns = round_up(int(n_in), 16)             # exactly the C side's n_out_stride ((n_in + 15) & ~15); 0 for an empty cloud
    with torch.cuda.device(dev):
        xyz = torch.empty((S, 3, Ns), dtype=torch.float32, device=dev)
        label = torch.empty((S, Ns), dtype=torch.int8, device=dev)
        n_pts = torch.empty((S,), dtype=torch.int32, device=dev)
        init = torch.empty((S, n_inits, 4), dtype=torch.float64, device=dev)
        ang = torch.empty((S,), dtype=torch.float64, device=dev)
        degen = torch.empty((S,), dtype=torch.int32, device=dev)
        rc = lib.frustum_prepare_batch_f32(_ptr(xyz_in), _ptr(pred), int(n_in), Ns_in, S, int(n_inits), int(seed),
                                           float(ry_sigma), float(t_amp), 1 if sort else 0, _ptr(xyz), _ptr(label),
                                           _ptr(n_pts),
                                           _ptr(init), _ptr(ang), _ptr(degen), 0, 0, _stream_ptr(stream))
    _native.check(rc, "frustum_prepare_batch")
    return dict(xyz=xyz, label=label, n_pts=n_pts, init=init, init_y_angle=ang, degenerate=degen)


def sort_clouds(xyz, label, n, stream=None):
    """Reorder clouds by (label, Morton cell of (x,z)) without filtering (frustum_sort_batch_f32): every point is kept,
    labels other than 0 / 1 sort last as ignored.  xyz [S,3,Ns] f32 cuda, label [S,Ns] int8, n valid points per cloud.
    Returns (xyz, label, n_pts) ready for solve_batch; the solver's sums do not depend on the order beyond rounding, its
    box cull does."""
    _require_cuda()
    lib = _native.load()
    S, Ns_in = _check_cloud(xyz, label, what="xyz", dtypes=(torch.float32,))
    dev = xyz.device
    if not (0 <= int(n) <= Ns_in):
        raise ValueError("n must be within the point stride")
    Ns = round_up(int(n), 16)
    with torch.cuda.device(dev):
        oxyz = torch.empty((S, 3, Ns), dtype=torch.float32, device=dev)
        olab = torch.empty((S, Ns), dtype=torch.int8, device=dev)
        n_pts = torch.empty((S,), dtype=torch.int32, device=dev)
        rc = lib.frustum_sort_batch_f32(_ptr(xyz), _ptr(label), int(n), Ns_in, S, _ptr(oxyz), _ptr(olab), _ptr(n_pts),
                                        _stream_ptr(stream))
    _native.check(rc, "frustum_sort_batch")
    return oxyz, olab, n_pts


def register_batch(xyz_in, pred, n_in, K, H, W, n_inits=60, seed=0, t_lb=DEFAULT_T_LB, t_ub=DEFAULT_T_UB,
                   max_iter=500, is_2d=True, return_all=False, stream=None, out=None):
    """Batched body of registration_lsq.py:329-343 in ONE C-ABI call (frustum_register_batch_f32): initial guess,
    front filter, n_inits perturbed starts, the multi-start solve, min-cost pose; degenerate samples (no
    predicted-inside point) get P = I, cost = 1e4.  This is the call that replaces the reference's
    fork-per-solve loop (registration_lsq.py:142-186).

    xyz_in [S,3,Ns_in] f32 cuda, pred [S,Ns_in] int8 cuda, n_in valid points per cloud.  Returns dict(P [S,4,4],
    cost [S], best [S], init_y_angle [S], n_pts [S], degenerate [S]) (+ init [S,I,4], params [S,I,6],
    costs [S,I], stats [S,I,4] if return_all).  `out`: the dict of an earlier call with the same shapes; its
    tensors are overwritten in place, so a steady-state loop allocates nothing."""
    _require_cuda()
    lib = _native.load()
    S, Ns_in = _check_cloud(xyz_in, pred, what="xyz_in", dtypes=(torch.float32,))
    dev = xyz_in.device
    n_in, I = int(n_in), int(n_inits)
    if not (0 <= n_in <= Ns_in) or I < 1:
        raise ValueError("bad n_in / n_inits")
    K9 = _as_K(K, S, dev)
    lb = np.ascontiguousarray(np.asarray(t_lb, dtype=np.float64).reshape(3))
    ub = np.ascontiguousarray(np.asarray(t_ub, dtype=np.float64).reshape(3))
    with torch.cuda.device(dev):
        if out is not None:
            res = out
            if tuple(res["P"].shape) != (S, 4, 4) or res["P"].device != dev or (return_all and "params" not in res):
                raise ValueError("out buffers do not match this batch")
            if return_all and tuple(res["params"].shape) != (S, I, 6):
                raise ValueError("out buffers do not match this batch")
        else:
            res = dict(P=torch.empty((S, 4, 4), dtype=torch.float64, device=dev),
                       cost=torch.empty((S,), dtype=torch.float64, device=dev),
                       best=torch.empty((S,), dtype=torch.int32, device=dev),
                       init_y_angle=torch.empty((S,), dtype=torch.float64, device=dev),
                       n_pts=torch.empty((S,), dtype=torch.int32, device=dev),
                       degenerate=torch.empty((S,), dtype=torch.int32, device=dev))
            if return_all:
                res.update(init=torch.empty((S, I, 4), dtype=torch.float64, device=dev),
                           params=torch.empty((S, I, 6), dtype=torch.float64, device=dev),
                           costs=torch.empty((S, I), dtype=torch.float64, device=dev),
                           stats=torch.empty((S, I, 4), dtype=torch.int32, device=dev))
        sp = _stream_ptr(stream)
        ws = _workspace(_ws_cache, lib.frustum_register_workspace_bytes(S, I, n_in), dev, stream)
        rc = lib.frustum_register_batch_f32(
            _ptr(xyz_in), _ptr(pred), n_in, Ns_in, S, I, int(seed), float(RY_SIGMA), float(T_AMPLITUDE), _ptr(K9),
            lb.ctypes.data, ub.ctypes.data, float(H), float(W), int(max_iter), 1 if is_2d else 0, _ptr(res["P"]),
            _ptr(res["cost"]), _ptr(res["best"]), _ptr(res["init_y_angle"]), _ptr(res["n_pts"]),
            _ptr(res["degenerate"]), _ptr(res.get("init") if return_all else None),
            _ptr(res.get("params") if return_all else None), _ptr(res.get("costs") if return_all else None),
            _ptr(res.get("stats") if return_all else None), _ptr(ws), ws.numel(), sp)
    _native.check(rc, "frustum_register_batch")
    return res


def solve_p_given_k(points, labels, K, init_y_angle, init_T, H, W, t_xyz_lower_bound, t_xyz_upper_bound,
                    max_iter, is_debug, is_2d):
    """Drop-in body of FrustumRegistration.solvePGivenK (registration.cpp:190-206): numpy in,
    (P 4x4 ndarray, final_cost float, residuals ndarray) out."""
    _require_cuda()
    pts = np.asarray(points, dtype=np.float64)
    if pts.ndim != 2 or pts.shape[0] != 3:
        raise TypeError("points must be a 3xN float array")
    lab = np.asarray(labels)
    if lab.ndim != 1 or lab.shape[0] != pts.shape[1]:
        raise TypeError("labels must be a length-N integer array")
    lb = list(t_xyz_lower_bound)
    ub = list(t_xyz_upper_bound)
    if len(lb) < 3 or len(ub) < 3:
        raise IndexError("bounds need 3 entries")       # std::out_of_range in the reference (:131-134)
    T = np.asarray(init_T, dtype=np.float64).reshape(3)
    xyz, l8, n_pts = pack_clouds(pts, lab)
    init = torch.tensor([[[float(init_y_angle), T[0], T[1], T[2]]]], dtype=torch.float64)
    # the solver reads a (label, Morton)-sorted copy (its box cull needs spatially compact groups; the sums do not depend
    # on the order beyond rounding); the residual vector below is formed from the caller's order
    sxyz, sl8, sn = sort_clouds(xyz, l8, pts.shape[1]) if xyz.dtype == torch.float32 and pts.shape[1] > 1 else (xyz, l8, n_pts)
    out = solve_batch(sxyz, sl8, sn, np.asarray(K, dtype=np.float64), init, H, W, lb[:3], ub[:3], int(max_iter),
                      bool(is_2d), return_all=True)
    x = out["params"][0, 0]                  # all six slots (unused ones are zero): goes to the kernel without a copy
    res = residuals(xyz[0], l8[0], pts.shape[1], np.asarray(K, dtype=np.float64), x, H, W, bool(is_2d),
                    host_labels=lab)
    if is_debug:
        st = out["stats"][0, 0].tolist()
        print("deepi2p_b200 solvePGivenK: iterations=%d evaluations=%d line_search_steps=%d termination=%s cost=%.6e"
              % (st[0], st[1], st[2], TERMINATION[st[3]] if 0 <= st[3] < len(TERMINATION) else st[3],
                 float(out["cost"][0])))
    return out["P"][0].cpu().numpy(), float(out["cost"][0].item()), res.cpu().numpy()


def inside_mask_batch(xyz, n_pts, P, K, H, W, stream=None):
    """Batched get_inside_img_mask (registration_lsq.py:67-84): int8 [S,Ns], 1 inside / 0 outside / -1 padding."""
    _require_cuda()
    lib = _native.load()
    S, Ns = _check_cloud(xyz, None, n_pts, dtypes=(torch.float32,))
    dev = xyz.device
    P16 = torch.as_tensor(P, dtype=torch.float64).to(dev).reshape(S, -1)
    if P16.shape[1] == 12:
        P16 = torch.cat([P16, torch.tensor([[0.0, 0.0, 0.0, 1.0]], dtype=torch.float64, device=dev).expand(S, 4)], 1)
    P16 = P16.contiguous()
    K9 = _as_K(K, S, dev)
    if n_pts is not None:
        n_pts = n_pts.to(dev, torch.int32).contiguous()
    with torch.cuda.device(dev):
        mask = torch.empty((S, Ns), dtype=torch.int8, device=dev)
        rc = lib.frustum_inside_mask_f32(_ptr(xyz), _ptr(n_pts), Ns, _ptr(P16), _ptr(K9), float(H), float(W), S,
                                         _ptr(mask), _stream_ptr(stream))
    _native.check(rc, "frustum_inside_mask")
    return mask


def pose_error_batch(P_pred, P_gt, t_thresh=2.0, r_thresh=5.0, stream=None):
    """Batched get_P_diff (registration_lsq.py:87-95) + the authors' success criterion
    (registration_result_analysis.py:37-38).  Returns dict(t_err [S] m, r_err [S] deg, success [S] int32,
    success_rate float tensor).

    P_pred is inverted as a general 4x4 matrix (as np.linalg.inv does), and r_err follows scipy's
    Rotation.from_matrix(...).as_euler('xzy') step for step, including its orthogonalisation of a non-rigid block and
    its gimbal-lock rule (DESIGN.md 4.14); oracle.pose_diff_restated reproduces the results bit for bit.  A rotation
    block with det <= 0 (where scipy raises) or a NaN gives r_err = NaN and success 0."""
    _require_cuda()
    lib = _native.load()
    Pp = torch.as_tensor(P_pred, dtype=torch.float64)
    dev = Pp.device if Pp.is_cuda else torch.device("cuda")
    Pp = Pp.to(dev).reshape(-1, 16).contiguous()
    Pg = torch.as_tensor(P_gt, dtype=torch.float64).to(dev).reshape(-1, 16).contiguous()
    S = Pp.shape[0]
    if Pg.shape[0] != S:
        raise ValueError("P_pred and P_gt must have the same batch size")
    with torch.cuda.device(dev):
        t_err = torch.empty((S,), dtype=torch.float64, device=dev)
        r_err = torch.empty((S,), dtype=torch.float64, device=dev)
        ok = torch.empty((S,), dtype=torch.int32, device=dev)
        rc = lib.pose_error_batch(_ptr(Pp), _ptr(Pg), S, float(t_thresh), float(r_thresh), _ptr(t_err), _ptr(r_err),
                                  _ptr(ok), _stream_ptr(stream))
    _native.check(rc, "pose_error_batch")
    return dict(t_err=t_err, r_err=r_err, success=ok, success_rate=ok.double().mean() if S else torch.tensor(0.0))
