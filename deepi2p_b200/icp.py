"""Monodepth + ICP baseline (evaluation/icp/registration_icp.py) on the GPU.

icp_register_batch runs many (frame, init) point-to-point ICP problems in one C-ABI call (icp_register_batch_f32,
csrc/icp.cu); icp_random_init is the reference's function of that name with its numpy signature.  DESIGN.md "ICP"
states the contract and where it deliberately differs from Open3D: points are transformed from the original source
by the composed pose at every pass, nearest-neighbour ties go to the lowest target index, the inits come from a
seeded generator, and the target is rounded once to float32 after scale calibration.  There is no CPU fallback.
"""
import contextlib
import math
import threading

import numpy as np
import torch

from . import _native, synthetic
from .frustum import _ptr, _require_cuda, _stream_ptr, _workspace, round_up

MAX_CORR_DIST = 1.0            # registration_icp.py:148
MAX_ITERATION = 30             # Open3D ICPConvergenceCriteria defaults
RELATIVE_FITNESS = 1e-6
RELATIVE_RMSE = 1e-6
T_AMPLITUDE = (5.0, 0.0, 10.0)            # registration_icp.py:116-117
RY_AMPLITUDE = 2.0 * math.pi


_counting = threading.local()      # count_evals(): the buffer of the innermost open context of this thread


def _check(t, name, dtype, shape, dev):
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == dtype and tuple(t.shape) == shape
            and t.is_contiguous() and (dev is None or t.device == dev)):
        raise ValueError(f"{name} must be a contiguous {dtype} {list(shape)} CUDA tensor on one device")


def icp_register_batch(src, n_pts, tgt, m_pts, init, max_corr_dist=MAX_CORR_DIST, max_iteration=MAX_ITERATION,
                       relative_fitness=RELATIVE_FITNESS, relative_rmse=RELATIVE_RMSE, force_2d=True,
                       return_all=False, stream=None, out=None, counters=None):
    """registration_icp.py's icp_random_init for S frames at once.

    src [S,3,Ns] f32 (LiDAR), n_pts [S] int32 or None (= Ns), tgt [S,3,Ms] f32 (depth cloud), m_pts [S] int32 or None,
    init [S,I,4,4] f64, all on one CUDA device; Ns and Ms multiples of 16 (pack_clouds pads).  Returns dict(P [S,4,4]
    f64 (2-D forced when force_2d), fitness [S] f64, best [S] i32 (-1: no init beat 0.001, P = I)) and, with
    return_all, T [S,I,4,4], fitness_all [S,I], rmse_all [S,I], stats [S,I,2] i32 (update steps, n_corr).
    `out`: the dict of an earlier call with the same shapes; its tensors are overwritten in place.
    `counters`: an int64 [2] CUDA tensor to which the call adds (nearest-neighbour queries, point distance
    evaluations); a measurement aid, the results do not change."""
    _require_cuda()
    lib = _native.load()
    if not (isinstance(src, torch.Tensor) and src.is_cuda and src.dim() == 3 and src.shape[1] == 3):
        raise ValueError("src must be a [S,3,Ns] CUDA tensor")
    S, _, Ns = src.shape
    dev = src.device
    _check(src, "src", torch.float32, (S, 3, Ns), dev)
    if not (isinstance(tgt, torch.Tensor) and tgt.dim() == 3):
        raise ValueError("tgt must be a [S,3,Ms] CUDA tensor")
    Ms = tgt.shape[2]
    _check(tgt, "tgt", torch.float32, (S, 3, Ms), dev)
    if not (isinstance(init, torch.Tensor) and init.dim() == 4):
        raise ValueError("init must be a [S,I,4,4] float64 CUDA tensor")
    I = init.shape[1]
    _check(init, "init", torch.float64, (S, I, 4, 4), dev)
    for t, name in ((n_pts, "n_pts"), (m_pts, "m_pts")):
        if t is not None:
            _check(t, name, torch.int32, (S,), dev)
    if counters is None:
        counters = getattr(_counting, "buf", None)
        if counters is not None and counters.device != dev:
            counters = None
    if counters is not None:
        _check(counters, "counters", torch.int64, (2,), dev)
    with torch.cuda.device(dev):
        shapes = dict(P=((S, 4, 4), torch.float64), fitness=((S,), torch.float64), best=((S,), torch.int32))
        if return_all:
            shapes.update(T=((S, I, 4, 4), torch.float64), fitness_all=((S, I), torch.float64),
                          rmse_all=((S, I), torch.float64), stats=((S, I, 2), torch.int32))
        if out is not None:
            for k, (shp, dt) in shapes.items():
                t = out.get(k)
                if t is None or tuple(t.shape) != shp or t.dtype != dt or t.device != dev:
                    raise ValueError("out buffers do not match this batch")
            res = out
        else:
            res = {k: torch.empty(shp, dtype=dt, device=dev) for k, (shp, dt) in shapes.items()}
        sp = _stream_ptr(stream)
        ws = _workspace(max(lib.icp_workspace_bytes(S, max(I, 1), Ns, max(Ms, 16)), 1), dev, sp)
        args = (_ptr(src), _ptr(n_pts), Ns, _ptr(tgt), _ptr(m_pts), Ms, S, _ptr(init), I, float(max_corr_dist),
                int(max_iteration), float(relative_fitness), float(relative_rmse), int(bool(force_2d)), _ptr(res["P"]),
                _ptr(res["fitness"]), _ptr(res["best"]), _ptr(res.get("T")), _ptr(res.get("fitness_all")),
                _ptr(res.get("rmse_all")), _ptr(res.get("stats")))
        if counters is None:
            rc = lib.icp_register_batch_f32(*args, _ptr(ws), ws.numel(), sp)
        else:
            rc = lib.icp_register_batch_counted_f32(*args, _ptr(counters), _ptr(ws), ws.numel(), sp)
    _native.check(rc, "icp_register_batch")
    return res


def pack_clouds(clouds, device="cuda"):
    """Host clouds (a list of [3,N_s] arrays, or one [3,N] array) -> (xyz [S,3,Ns] f32, n [S] int32) on `device`,
    Ns = round_up(max N_s, 16).  Coordinates are rounded to float32."""
    if isinstance(clouds, np.ndarray) and clouds.ndim == 2:
        clouds = [clouds]
    n = [int(np.asarray(c).shape[1]) for c in clouds]
    Ns = round_up(max(n + [1]), 16)
    xyz = np.zeros((len(clouds), 3, Ns), dtype=np.float32)
    for s, c in enumerate(clouds):
        c = np.asarray(c)
        if c.ndim != 2 or c.shape[0] != 3:
            raise ValueError("clouds are [3, N]")
        xyz[s, :, :n[s]] = c.astype(np.float32)
    dev = torch.device(device)
    return torch.from_numpy(xyz).to(dev), torch.tensor(n, dtype=torch.int32, device=dev)


def random_inits(S, I, seed=0):
    """generate_uniform_random_transform(5, 0, 10, 0, 2 pi, 0) of registration_icp.py:13-32 for S x I problems from
    numpy.random.default_rng(seed): t = (U(-5, 5), 0, U(-10, 10)), R = Ry(U(-2 pi, 2 pi)) (augmentation.py:14-25 with
    only the y angle non-zero).  Returns [S, I, 4, 4] float64."""
    rng = np.random.default_rng(seed)
    tx = rng.uniform(-T_AMPLITUDE[0], T_AMPLITUDE[0], (S, I))
    tz = rng.uniform(-T_AMPLITUDE[2], T_AMPLITUDE[2], (S, I))
    ry = rng.uniform(-RY_AMPLITUDE, RY_AMPLITUDE, (S, I))
    P = np.zeros((S, I, 4, 4))
    c, s = np.cos(ry), np.sin(ry)
    P[..., 0, 0], P[..., 0, 2], P[..., 1, 1], P[..., 2, 0], P[..., 2, 2] = c, s, 1.0, -s, c
    P[..., 0, 3], P[..., 2, 3], P[..., 3, 3] = tx, tz, 1.0
    return P


def calibrate_scale(pc, P_gt, K, H, W, depth_pc):
    """registration_icp.py:215-218: mean camera-frame z of the LiDAR points inside the image under the GROUND-TRUTH
    pose, over the mean z of the depth cloud.  The reference calibrates the depth scale with the ground truth; so does
    this baseline (the monodepth network's scale is otherwise unknown)."""
    pc = np.asarray(pc, dtype=np.float64)
    P_gt = np.asarray(P_gt, dtype=np.float64)
    mask = synthetic.inside_mask(pc, P_gt, np.asarray(K, dtype=np.float64), H, W)
    z = P_gt[2, :3] @ pc + P_gt[2, 3]
    return float(np.mean(z[mask]) / np.mean(np.asarray(depth_pc, dtype=np.float64)[2, :]))


def icp_random_init(pc_np, pc_monodepth_np, num_iterations, is_plot, seed=0):
    """Drop-in body of icp_random_init (registration_icp.py:115-139): numpy in, (P 4x4 ndarray, fitness float) out.
    Both clouds are rounded to float32; the inits are random_inits(1, num_iterations, seed)."""
    if is_plot:
        raise ValueError("is_plot=True needs Open3D's viewer, which this implementation does not have")
    src, n = pack_clouds(np.asarray(pc_np, dtype=np.float64))
    tgt, m = pack_clouds(np.asarray(pc_monodepth_np, dtype=np.float64))
    init = torch.from_numpy(random_inits(1, int(num_iterations), seed)).to(src.device)
    out = icp_register_batch(src, n, tgt, m, init)
    return out["P"][0].cpu().numpy(), float(out["fitness"][0])


def build_index(tgt, m_pts=None, stream=None):
    """Measurement aid: only the per-frame nearest-neighbour index build of an icp_register_batch call over tgt
    [S,3,Ms] f32 (icp_build_index_f32), enqueued on `stream`.  Nothing it computes is returned."""
    _require_cuda()
    lib = _native.load()
    if not (isinstance(tgt, torch.Tensor) and tgt.dim() == 3):
        raise ValueError("tgt must be a [S,3,Ms] CUDA tensor")
    S, _, Ms = tgt.shape
    _check(tgt, "tgt", torch.float32, (S, 3, Ms), None)
    if m_pts is not None:
        _check(m_pts, "m_pts", torch.int32, (S,), tgt.device)
    with torch.cuda.device(tgt.device):
        sp = _stream_ptr(stream)
        ws = _workspace(max(lib.icp_workspace_bytes(S, 1, 16, max(Ms, 16)), 1), tgt.device, sp)
        rc = lib.icp_build_index_f32(_ptr(tgt), _ptr(m_pts), Ms, S, _ptr(ws), ws.numel(), sp)
    _native.check(rc, "icp_build_index")


@contextlib.contextmanager
def count_evals(device="cuda"):
    """Measurement context: ``with count_evals() as c: ...`` then c["queries"], c["evals"] hold the nearest-neighbour
    queries and point distance evaluations of the icp_register_batch calls this thread makes inside on `device`.
    The context owns the counter buffer and passes it to each call explicitly (icp_register_batch_counted_f32); the
    library keeps no state between calls."""
    buf = torch.zeros(2, dtype=torch.int64, device=device)
    prev = getattr(_counting, "buf", None)
    _counting.buf = buf
    res = {}
    try:
        yield res
    finally:
        _counting.buf = prev
        torch.cuda.synchronize(buf.device)
        res["queries"], res["evals"] = (int(v) for v in buf.cpu().tolist())
