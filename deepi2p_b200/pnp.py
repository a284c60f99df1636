"""PnP-RANSAC registration from grid classifications (evaluation/registration_pnp.py:95-148) on the GPU.

pnp_ransac_batch runs many frames in one C-ABI call (pnp_ransac_batch_f32, csrc/pnp_ransac.cu); solve_pnp is the
reference's solve_PnP with its numpy signature.  DESIGN.md "PnP-RANSAC" states the contract, including where it
differs from cv2.solvePnPRansac: the minimal samples come from Philox4x32-10 rather than cv2's generator, and
frames with 4 or 5 selected points get EPnP on all of them.  There is no CPU fallback.
"""
import numpy as np
import torch

from . import _native
from ._native import _ptr, _require_cuda, _stream_ptr, _workspace
from .frustum import _as_K, _ws_cache, round_up

SOLVEPNP_EPNP = 1          # the value of cv2.SOLVEPNP_EPNP, the only method implemented


def _check_frames(xyz, coarse_pred, fine_pred, n_pts):
    if not isinstance(xyz, torch.Tensor) or not xyz.is_cuda:
        raise ValueError("xyz must be a CUDA tensor")
    if xyz.dim() != 3 or xyz.shape[1] != 3 or xyz.dtype != torch.float32 or not xyz.is_contiguous():
        raise ValueError("xyz must be a contiguous float32 [S,3,Ns] tensor")
    S, _, Ns = xyz.shape
    for t, dt, name in ((coarse_pred, torch.int8, "coarse_pred"), (fine_pred, torch.int32, "fine_pred")):
        if not (isinstance(t, torch.Tensor) and t.device == xyz.device and t.dtype == dt and tuple(t.shape) == (S, Ns)
                and t.is_contiguous()):
            raise ValueError(f"{name} must be a contiguous {dt} [S,Ns] tensor on the device of xyz")
    if n_pts is not None:
        if not (isinstance(n_pts, torch.Tensor) and n_pts.device == xyz.device and n_pts.dtype == torch.int32
                and n_pts.numel() == S and n_pts.is_contiguous()):
            raise ValueError("n_pts must be a contiguous int32 [S] tensor on the device of xyz")
    return S, Ns


def pnp_ransac_batch(xyz, coarse_pred, fine_pred, n_pts, K, H, W, scale=1 / 32.0, iterations=500, reproj_err=0.6,
                     confidence=0.99, seed=0, return_all=False, stream=None, out=None):
    """solve_PnP for S frames at once.

    xyz [S,3,Ns] f32, coarse_pred [S,Ns] int8 (1 = predicted inside the image), fine_pred [S,Ns] int32 (cell of the
    scale-W x scale-H grid), n_pts [S] int32 or None (= Ns), all on one CUDA device; K [3,3] or [S,3,3] (unscaled).
    Returns dict(P [S,4,4] f64, outlier_ratio [S] f64, inliers [S] i32, n_sel [S] i32, hyp_used [S] i32) and, with
    return_all, inlier_mask [S,Ns] u8, hyp_pose [S,iterations,12] f64 (R row-major | t), hyp_inliers [S,iterations]
    i32 (entries at h >= hyp_used unspecified: zero or a scored hypothesis past the stop in a new dict, kept from the
    earlier call with `out`).  `out`: the dict of an earlier call with the same shapes; its tensors are overwritten in
    place."""
    _require_cuda()
    lib = _native.load()
    S, Ns = _check_frames(xyz, coarse_pred, fine_pred, n_pts)
    dev = xyz.device
    iterations = int(iterations)
    K9 = _as_K(K, S, dev)
    with torch.cuda.device(dev):
        shapes = dict(P=((S, 4, 4), torch.float64), outlier_ratio=((S,), torch.float64),
                      inliers=((S,), torch.int32), n_sel=((S,), torch.int32), hyp_used=((S,), torch.int32))
        if return_all:
            shapes.update(inlier_mask=((S, Ns), torch.uint8), hyp_pose=((S, max(iterations, 1), 12), torch.float64),
                          hyp_inliers=((S, max(iterations, 1)), torch.int32))
        if out is not None:
            for k, (shp, dt) in shapes.items():
                t = out.get(k)
                if t is None or tuple(t.shape) != shp or t.dtype != dt or t.device != dev:
                    raise ValueError("out buffers do not match this batch")
            res = out
        else:
            res = {k: torch.empty(shp, dtype=dt, device=dev) for k, (shp, dt) in shapes.items()}
            if return_all:
                # a frame that stops early never writes the tail of its hypothesis rows; zeroed, it does not carry
                # whatever the allocator handed out, so two identical calls return identical arrays
                with torch.cuda.stream(stream):
                    res["hyp_pose"].zero_()
                    res["hyp_inliers"].zero_()
        sp = _stream_ptr(stream)
        ws = _workspace(_ws_cache, max(lib.pnp_ransac_workspace_bytes(S, Ns, max(iterations, 1)), 1), dev, stream)
        rc = lib.pnp_ransac_batch_f32(
            _ptr(xyz), _ptr(coarse_pred), _ptr(fine_pred), _ptr(n_pts), Ns, S, _ptr(K9), float(H), float(W),
            float(scale), iterations, float(reproj_err), float(confidence), int(seed) & 0xFFFFFFFFFFFFFFFF,
            _ptr(res["P"]), _ptr(res["outlier_ratio"]), _ptr(res["inliers"]), _ptr(res["n_sel"]),
            _ptr(res["hyp_used"]), _ptr(res.get("inlier_mask")), _ptr(res.get("hyp_pose")),
            _ptr(res.get("hyp_inliers")), _ptr(ws), ws.numel(), sp)
    _native.check(rc, "pnp_ransac_batch")
    return res


def pack_frames(points, coarse, fine, device="cuda"):
    """Host frames -> device tensors (xyz [S,3,Ns] f32, coarse int8 [S,Ns], fine int32 [S,Ns], n_pts int32 [S]).
    points: list of [3,N_s] arrays (or one [3,N] array), coarse / fine: matching [N_s] integer arrays."""
    if isinstance(points, np.ndarray) and points.ndim == 2:
        points, coarse, fine = [points], [coarse], [fine]
    S = len(points)
    n = [int(np.asarray(p).shape[1]) for p in points]
    Ns = round_up(max(n + [1]), 16)
    xyz = np.zeros((S, 3, Ns), dtype=np.float32)
    c8 = np.zeros((S, Ns), dtype=np.int8)
    f32 = np.zeros((S, Ns), dtype=np.int32)
    for s in range(S):
        p = np.asarray(points[s])
        p32 = p.astype(np.float32)
        if p.dtype != np.float32 and not np.array_equal(p32.astype(p.dtype), p):
            raise ValueError("coordinates are not float32-representable")
        xyz[s, :, :n[s]] = p32
        c8[s, :n[s]] = np.where(np.asarray(coarse[s]) == 1, 1, 0)
        f32[s, :n[s]] = np.asarray(fine[s]).astype(np.int64)
    dev = torch.device(device)
    return (torch.from_numpy(xyz).to(dev), torch.from_numpy(c8).to(dev), torch.from_numpy(f32).to(dev),
            torch.tensor(n, dtype=torch.int32, device=dev))


def solve_pnp(pc_np, coarse_predictions_np, fine_predictions_np, K_np, H, W, fine_resolution_scale, iterationsCount,
              method):
    """Drop-in body of solve_PnP (registration_pnp.py:95-148): numpy in, (P 4x4 ndarray, outlier_ratio float) out.
    method must be cv2.SOLVEPNP_EPNP (1).  Coordinates are rounded to float32, as the loaders produce them."""
    if int(method) != SOLVEPNP_EPNP:
        raise ValueError("only SOLVEPNP_EPNP (1) is implemented, got method=%r" % (method,))
    pc = np.asarray(pc_np, dtype=np.float64).astype(np.float32)
    if pc.ndim != 2 or pc.shape[0] != 3:
        raise ValueError("pc_np must be 3xN")
    xyz, c8, f32, n_pts = pack_frames(pc, np.asarray(coarse_predictions_np), np.asarray(fine_predictions_np))
    out = pnp_ransac_batch(xyz, c8, f32, n_pts, np.asarray(K_np, dtype=np.float64), H, W,
                           scale=fine_resolution_scale, iterations=iterationsCount)
    return out["P"][0].cpu().numpy(), float(out["outlier_ratio"][0])


def epnp_batch(sets, K):
    """Test hook: EPnP on each (xyz [n,3], uv [n,2]) of `sets` with intrinsics K [3,3] (used as given) or [B,3,3].
    Returns (pose [B,12] f64 = R row-major | t, ok [B] bool) as numpy."""
    _require_cuda()
    lib = _native.load()
    B = len(sets)
    offs = np.zeros(B + 1, dtype=np.int32)
    for b, (x, _) in enumerate(sets):
        offs[b + 1] = offs[b] + len(x)
    xyz = np.concatenate([np.asarray(x, dtype=np.float64).reshape(-1, 3) for x, _ in sets] + [np.zeros((0, 3))])
    uv = np.concatenate([np.asarray(u, dtype=np.float64).reshape(-1, 2) for _, u in sets] + [np.zeros((0, 2))])
    dev = torch.device("cuda")
    K9 = _as_K(K, B, dev) if B else torch.zeros((0, 9), dtype=torch.float64, device=dev)
    t_xyz = torch.from_numpy(np.ascontiguousarray(xyz)).to(dev)
    t_uv = torch.from_numpy(np.ascontiguousarray(uv)).to(dev)
    t_off = torch.from_numpy(offs).to(dev)
    pose = torch.zeros((B, 12), dtype=torch.float64, device=dev)
    ok = torch.zeros((B,), dtype=torch.int32, device=dev)
    rc = lib.epnp_batch_f64(_ptr(t_xyz), _ptr(t_uv), _ptr(t_off), B, _ptr(K9), _ptr(pose), _ptr(ok), _stream_ptr())
    _native.check(rc, "epnp_batch_f64")
    return pose.cpu().numpy(), ok.cpu().numpy().astype(bool)
