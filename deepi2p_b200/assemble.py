"""Classifier input batches on the GPU: the loaders' point side after the scan records are read (frame accumulation,
the voxel step, downsample_np, augmentation, the camera transform and the farthest-point node sets of
data/kitti_pc_img_pose_loader.py:199-446 and data/oxford_pc_img_pose_loader.py:262-352).

accumulate, resample, candidates and farthest_point_sample wrap the C-ABI calls of csrc/assemble.cu for S samples at
once; assemble_batch chains them (with pointprep.voxel_downsample for the voxel step) into the loader's point side;
random_transforms draws the per-sample augmentation on the host.  FarthestSampler / ProjectiveFarthestSampler are
drop-ins for data/kitti_helper.py's classes (numpy in, numpy out).  DESIGN.md "Batch assembly" states the contract and
where it deliberately differs from the loaders.  There is no CPU fallback.
"""
import math

import numpy as np
import torch

from . import _native
from .frustum import _ptr, _require_cuda, _stream_ptr, _workspace, round_up
from .icp import _check
from . import pointprep

INPUT_PT_NUM = 20480          # kitti/options.py, oxford/options.py
NODE_NUM = 128
FPS_MAX = 65536               # the largest set farthest_point_sample takes (a cluster of 8 CTAs x 8192 points)
SIGMA, CLIP = 0.01, 0.05      # augmentation.jitter_point_cloud
JITTER_BITS = {"pc": 1, "sn": 2, "intensity": 4}
MODES = ("train", "val_random_Ry", "val", "test")

# data/kitti_pc_img_pose_loader.py:374: NWU (x forward, y left, z up) -> camera (x right, y down, z forward)
P_CAM_NWU = np.array([[0, -1, 0, 0], [0, 0, -1, 0], [1, 0, 0, 0], [0, 0, 0, 1]], dtype=np.float64)
P_NWU_CAM = P_CAM_NWU.T.copy()


def compose(A, B):
    """A @ B for [...,4,4] float64 with a fixed association, ((a0 b0 + a1 b1) + a2 b2) + a3 b3, so that host and
    oracle agree bit for bit."""
    A = np.asarray(A, dtype=np.float64)
    B = np.asarray(B, dtype=np.float64)
    return ((A[..., :, 0, None] * B[..., None, 0, :] + A[..., :, 1, None] * B[..., None, 1, :])
            + A[..., :, 2, None] * B[..., None, 2, :]) + A[..., :, 3, None] * B[..., None, 3, :]


def rigid_inverse(P):
    """[R t; 0 1]^-1 = [R^T  -R^T t; 0 1] for [...,4,4]."""
    P = np.asarray(P, dtype=np.float64)
    out = np.zeros_like(P)
    Rt = np.swapaxes(P[..., :3, :3], -1, -2)
    out[..., :3, :3] = Rt
    out[..., :3, 3] = -np.einsum("...ij,...j->...i", Rt, P[..., :3, 3])
    out[..., 3, 3] = 1.0
    return out


def angles2rotation_matrix(angles):
    """augmentation.angles2rotation_matrix for [..., 3] angles (x, y, z): R = Rz (Ry Rx)."""
    a = np.asarray(angles, dtype=np.float64)
    c, s = np.cos(a), np.sin(a)
    z, o = np.zeros(a.shape[:-1]), np.ones(a.shape[:-1])
    Rx = np.stack([o, z, z, z, c[..., 0], -s[..., 0], z, s[..., 0], c[..., 0]], -1).reshape(a.shape[:-1] + (3, 3))
    Ry = np.stack([c[..., 1], z, s[..., 1], z, o, z, -s[..., 1], z, c[..., 1]], -1).reshape(a.shape[:-1] + (3, 3))
    Rz = np.stack([c[..., 2], -s[..., 2], z, s[..., 2], c[..., 2], z, z, z, o], -1).reshape(a.shape[:-1] + (3, 3))
    return Rz @ (Ry @ Rx)


def random_transforms(S, mode, amplitudes=(0.0, 0.0, 0.0, 0.0, 2.0 * math.pi, 0.0), rng=None, flip=True):
    """The loaders' Pr for S samples: `train` draws t ~ U(-a, a) and angles ~ U(-a, a) for amplitudes (tx, ty, tz,
    rx, ry, rz) (generate_random_transform) and, with `flip`, Pr <- Pr diag(-1, 1, 1, 1) with probability 1/2;
    `val_random_Ry` draws only ry ~ U(-2 pi, 2 pi); other modes give the identity.  rng: a numpy Generator or a seed.
    Returns (Pr [S,4,4] float64, flip [S] bool)."""
    if mode not in MODES:
        raise ValueError(f"mode must be one of {MODES} (got {mode!r})")
    rng = rng if isinstance(rng, np.random.Generator) else np.random.default_rng(rng)
    Pr = np.tile(np.eye(4), (S, 1, 1))
    flipped = np.zeros(S, dtype=bool)
    if mode == "train":
        a = np.asarray(amplitudes, dtype=np.float64).reshape(6)
        t = rng.uniform(-a[:3], a[:3], (S, 3))
        ang = rng.uniform(-a[3:], a[3:], (S, 3))
        Pr[:, :3, :3] = angles2rotation_matrix(ang)
        Pr[:, :3, 3] = t
        if flip:
            flipped = rng.random(S) > 0.5
            Pr[flipped, :, 0] *= -1.0
    elif mode == "val_random_Ry":
        ang = np.zeros((S, 3))
        ang[:, 1] = rng.uniform(-2.0 * math.pi, 2.0 * math.pi, S)
        Pr[:, :3, :3] = angles2rotation_matrix(ang)
    return Pr, flipped


def kitti_args(Pc, Pji=None):
    """assemble_batch arguments of the KITTI loader: points go to the camera frame by P_cam_nwu (pre), and
    P = Pji Pc P_nwu_cam Pr^-1; Pc [4,4] or [S,4,4] (camera <- velodyne), Pji [4,4] / [S,4,4] or None (identity)."""
    Pc = np.asarray(Pc, dtype=np.float64)
    Pji = np.eye(4) if Pji is None else np.asarray(Pji, dtype=np.float64)
    return dict(pre=P_CAM_NWU, P_base=compose(Pji, compose(Pc, P_NWU_CAM)), voxel_size=0.3, range_max=None,
                amplitudes=(0.0, 0.0, 0.0, 0.0, 2.0 * math.pi, 0.0), flip=True, jitter=("pc", "sn"))


def oxford_args(P_cam_pc, translation_max=10.0, pc_max_range=50.0):
    """assemble_batch arguments of the Oxford loader: pre = I, P = P_cam_pc Pr^-1, the x^2 + z^2 range mask, voxel 0.2,
    jitter on pc and intensity, no flip of the points."""
    tm = float(translation_max)
    return dict(pre=np.eye(4), P_base=np.asarray(P_cam_pc, dtype=np.float64), voxel_size=0.2, range_max=pc_max_range,
                amplitudes=(tm, 0.5 * tm, tm, 0.0, 2.0 * math.pi, 0.0), flip=False, jitter=("pc", "intensity"))


def _jitter_mask(jitter):
    m = 0
    for j in jitter:
        if j not in JITTER_BITS:
            raise ValueError(f"jitter entries are {tuple(JITTER_BITS)} (got {j!r})")
        m |= JITTER_BITS[j]
    return m


def _f32(t, name, shape, dev):
    _check(t, name, torch.float32, shape, dev)


def accumulate(xyz, intensity, sn, n_pts, frame_sample, frame_T, range_max=None, stream=None):
    """Frame accumulation for S samples.  xyz [T,3,n] f32, intensity [T,n] f32, sn [T,3,n] f32 or None (CUDA); n_pts
    [T] host ints; frame_sample [T] host ints, non-decreasing from 0 (sample of each frame, anchor frame first);
    frame_T [T,4,4] float64 (host).  Returns (xyz [S,3,A], intensity [S,A], sn [S,3,A] or None, count [S] int32 CUDA,
    count host numpy) with each sample's frames moved by frame_T and concatenated; range_max keeps x^2 + z^2 <
    range_max^2.  The counts are read back once."""
    _require_cuda()
    lib = _native.load()
    if not (isinstance(xyz, torch.Tensor) and xyz.is_cuda and xyz.dim() == 3 and xyz.shape[1] == 3):
        raise ValueError("xyz must be a [T,3,n] CUDA tensor")
    T, _, n = xyz.shape
    dev = xyz.device
    _f32(xyz, "xyz", (T, 3, n), None)
    _f32(intensity, "intensity", (T, n), dev)
    if sn is not None:
        _f32(sn, "sn", (T, 3, n), dev)
    npts = np.asarray(n_pts, dtype=np.int64).reshape(-1)
    fs = np.asarray(frame_sample, dtype=np.int64).reshape(-1)
    if npts.shape != (T,) or fs.shape != (T,) or T == 0:
        raise ValueError("n_pts and frame_sample need one entry per frame (T >= 1)")
    if npts.min() < 0 or npts.max() > n:
        raise ValueError(f"n_pts must be in [0, {n}]")
    if fs[0] != 0 or np.any(np.diff(fs) < 0) or np.any(np.diff(fs) > 1):
        raise ValueError("frame_sample must be non-decreasing from 0 without gaps")
    FT = np.ascontiguousarray(frame_T, dtype=np.float64)
    if FT.shape != (T, 4, 4) or not np.isfinite(FT).all():
        raise ValueError("frame_T must be [T,4,4] finite")
    if not bool(torch.isfinite(xyz).all()):
        raise ValueError("xyz has a non-finite coordinate")
    r = 0.0 if range_max is None else pointprep._positive(range_max, "range_max")
    S = int(fs[-1]) + 1
    A = round_up(max(int(np.bincount(fs, weights=npts).max()), 1), 16)
    with torch.cuda.device(dev), torch.cuda.stream(stream):
        fs_d = torch.from_numpy(fs.astype(np.int32)).to(dev)
        n_d = torch.from_numpy(npts.astype(np.int32)).to(dev)
        FT_d = torch.from_numpy(FT).to(dev)
        out_x = torch.zeros((S, 3, A), dtype=torch.float32, device=dev)
        out_i = torch.zeros((S, A), dtype=torch.float32, device=dev)
        out_n = torch.zeros((S, 3, A), dtype=torch.float32, device=dev) if sn is not None else None
        cnt = torch.zeros((S,), dtype=torch.int32, device=dev)
        sp = _stream_ptr(stream)
        ws = _workspace(lib.assemble_accumulate_workspace_bytes(T, n, S), dev, sp)
        rc = lib.assemble_accumulate_f32(_ptr(xyz), _ptr(intensity), _ptr(sn), _ptr(n_d), n, T, _ptr(fs_d), _ptr(FT_d),
                                         S, r, _ptr(out_x), _ptr(out_i), _ptr(out_n), A, _ptr(cnt), _ptr(ws),
                                         ws.numel(), sp)
        _native.check(rc, "assemble_accumulate")
        cnt_h = cnt.cpu().numpy()
    return out_x, out_i, out_n, cnt, cnt_h


def _voxel_step(xyz, inten, sn, cnt, cnt_h, N, voxel_size, stream):
    """The loaders' `if n > 2 N` branch: downsample_with_intensity_sn / downsample_with_reflectance on the samples that
    take it, with the drop-ins' arithmetic (intensity / max in float32, means in float64, times max, then float32)."""
    vox = np.nonzero(cnt_h > 2 * N)[0]
    if len(vox) == 0:
        return cnt, cnt_h
    dev = xyz.device
    sel = torch.from_numpy(vox).to(dev)
    A = xyz.shape[2]
    ns = cnt[sel].contiguous()
    valid = torch.arange(A, device=dev)[None] < ns[:, None]
    it = inten[sel]
    imax = it.masked_fill(~valid, -math.inf).amax(1)
    rows = [(it / imax[:, None]).double()]
    if sn is not None:
        rows += [sn[sel][:, a].double() for a in range(3)]
    attr = (torch.stack(rows, 1) * valid[:, None]).contiguous()
    out = pointprep.voxel_downsample(xyz[sel].contiguous(), ns, voxel_size, attr=attr, stream=stream)
    xyz[sel] = out["xyz"].to(torch.float32)
    inten[sel] = (out["attr"][:, 0] * imax.double()[:, None]).to(torch.float32)
    if sn is not None:
        sn[sel] = out["attr"][:, 1:4].to(torch.float32)
    cnt = cnt.clone()
    cnt[sel] = out["m_pts"]
    cnt_h = cnt_h.copy()
    cnt_h[vox] = out["m_pts"].cpu().numpy()
    return cnt, cnt_h


def resample(xyz, intensity, sn, n_pts, N, seed, M=None, jitter=(), sigma=SIGMA, clip=CLIP, stream=None):
    """downsample_np for S clouds, fused with the jitter and the transform.  xyz [S,3,A] f32, intensity [S,A] f32, sn
    [S,3,A] f32 or None, n_pts [S] int32 (CUDA); M [S,4,4] float64 (host; None = identity) moves the points (sn gets
    its rotation); jitter names the channels to jitter ("pc", "sn", "intensity").  Returns dict(pc [S,3,N],
    intensity [S,1,N], sn [S,3,N] (zeros without sn), src [S,N] int32 index into the input cloud)."""
    _require_cuda()
    lib = _native.load()
    if not (isinstance(xyz, torch.Tensor) and xyz.is_cuda and xyz.dim() == 3 and xyz.shape[1] == 3):
        raise ValueError("xyz must be a [S,3,A] CUDA tensor")
    S, _, A = xyz.shape
    dev = xyz.device
    _f32(xyz, "xyz", (S, 3, A), None)
    _f32(intensity, "intensity", (S, A), dev)
    if sn is not None:
        _f32(sn, "sn", (S, 3, A), dev)
    _check(n_pts, "n_pts", torch.int32, (S,), dev)
    if int(N) != N or N < 1:
        raise ValueError(f"input_pt_num must be a positive integer (got {N})")
    N = int(N)
    mask = _jitter_mask(jitter)
    if mask & JITTER_BITS["sn"] and sn is None:
        raise ValueError("sn jitter needs sn")
    M = np.tile(np.eye(4), (S, 1, 1)) if M is None else np.ascontiguousarray(M, dtype=np.float64)
    if M.shape != (S, 4, 4) or not np.isfinite(M).all():
        raise ValueError("M must be [S,4,4] finite")
    with torch.cuda.device(dev), torch.cuda.stream(stream):
        M_d = torch.from_numpy(M).to(dev)
        res = dict(pc=torch.empty((S, 3, N), dtype=torch.float32, device=dev),
                   intensity=torch.empty((S, 1, N), dtype=torch.float32, device=dev),
                   sn=torch.empty((S, 3, N), dtype=torch.float32, device=dev),
                   src=torch.empty((S, N), dtype=torch.int32, device=dev))
        sp = _stream_ptr(stream)
        ws = _workspace(lib.assemble_resample_workspace_bytes(S, A), dev, sp)
        rc = lib.assemble_resample_f32(_ptr(xyz), _ptr(intensity), _ptr(sn), _ptr(n_pts), A, S, N,
                                       int(seed) & (2**64 - 1), _ptr(M_d), float(sigma), float(clip), mask,
                                       _ptr(res["pc"]), _ptr(res["intensity"]), _ptr(res["sn"]), _ptr(res["src"]),
                                       _ptr(ws), ws.numel(), sp)
    _native.check(rc, "assemble_resample")
    return res


def candidates(pc, m, seed, node_set, stream=None):
    """The m smallest-key points of each sample of pc [S,3,N] f32 (node_set 0 = node_a, 1 = node_b): the loaders'
    np.random.choice(N, 8 M, replace=False).  Returns (idx [S,m] int32, xyz [S,3,m] f32)."""
    _require_cuda()
    lib = _native.load()
    if not (isinstance(pc, torch.Tensor) and pc.is_cuda and pc.dim() == 3 and pc.shape[1] == 3):
        raise ValueError("pc must be a [S,3,N] CUDA tensor")
    S, _, N = pc.shape
    _f32(pc, "pc", (S, 3, N), None)
    if not 1 <= m <= N:
        raise ValueError(f"8 * node_num ({m}) must be in [1, input_pt_num={N}]")
    dev = pc.device
    with torch.cuda.device(dev), torch.cuda.stream(stream):
        idx = torch.empty((S, m), dtype=torch.int32, device=dev)
        xyz = torch.empty((S, 3, m), dtype=torch.float32, device=dev)
        sp = _stream_ptr(stream)
        ws = _workspace(lib.assemble_candidates_workspace_bytes(S, N), dev, sp)
        rc = lib.assemble_candidates_f32(_ptr(pc), N, S, int(seed) & (2**64 - 1), int(node_set), int(m), _ptr(idx),
                                         _ptr(xyz), _ptr(ws), ws.numel(), sp)
    _native.check(rc, "assemble_candidates")
    return idx, xyz


def farthest_point_sample(xyz, n_pts, k, start=None, stream=None):
    """Farthest-point sampling of k points from each of S sets: xyz [S,3,n] or [S,2,n] (taken as z = 0), float32 or
    float64 CUDA; n_pts [S] int32 CUDA or None (= n); start [S] int32 CUDA or None (= 0).  Distances are fp64
    (dx dx + dy dy) + dz dz, ties go to the lowest index (data/kitti_helper.py FarthestSampler).  n <= 65536.
    Returns (idx [S,k] int32, nodes [S,D,k] in xyz's dtype)."""
    _require_cuda()
    lib = _native.load()
    if not (isinstance(xyz, torch.Tensor) and xyz.is_cuda and xyz.dim() == 3 and xyz.shape[1] in (2, 3)
            and xyz.dtype in (torch.float32, torch.float64)):
        raise ValueError("xyz must be a [S,3,n] or [S,2,n] float32 / float64 CUDA tensor")
    S, D, n = xyz.shape
    if n > FPS_MAX:
        raise ValueError(f"farthest_point_sample takes at most {FPS_MAX} points per set (got {n})")
    if int(k) != k or not 1 <= k <= n:
        raise ValueError(f"k must be an integer in [1, {n}] (got {k})")
    k = int(k)
    dev = xyz.device
    if n_pts is not None:
        _check(n_pts, "n_pts", torch.int32, (S,), dev)
        if S and int(n_pts.min()) < k:
            raise ValueError("every set needs at least k points")
    if start is not None:
        _check(start, "start", torch.int32, (S,), dev)
    with torch.cuda.device(dev), torch.cuda.stream(stream):
        x3 = xyz.contiguous() if D == 3 else torch.cat([xyz, torch.zeros_like(xyz[:, :1])], 1)
        idx = torch.empty((S, k), dtype=torch.int32, device=dev)
        nodes = torch.empty((S, 3, k), dtype=xyz.dtype, device=dev)
        fn = lib.fps_batch_f32 if xyz.dtype == torch.float32 else lib.fps_batch_f64
        rc = fn(_ptr(x3), _ptr(n_pts), n, S, k, _ptr(start), _ptr(idx), _ptr(nodes), _stream_ptr(stream))
    _native.check(rc, "fps_batch")
    return idx, nodes[:, :D]


def pack_frames(samples, device="cuda"):
    """Host samples -> assemble_batch's `frames`.  samples: a list of (frames, frame_T) with frames a list of (xyz
    [3,n], intensity [n] or [1,n], sn [3,n] or None) records, anchor frame first, and frame_T [T_s,4,4]; either every
    frame has sn or none has."""
    recs, Ts, fs = [], [], []
    for s, (frs, FT) in enumerate(samples):
        if len(frs) != len(FT):
            raise ValueError(f"sample {s}: one frame_T per frame")
        recs += frs
        Ts.append(np.asarray(FT, dtype=np.float64).reshape(-1, 4, 4))
        fs += [s] * len(frs)
    has_sn = {r[2] is not None for r in recs}
    if len(has_sn) != 1:
        raise ValueError("either every frame has sn or none has")
    n = [int(np.asarray(r[0]).shape[1]) for r in recs]
    ns = round_up(max(n + [1]), 16)
    X = np.zeros((len(recs), 3, ns), dtype=np.float32)
    I = np.zeros((len(recs), ns), dtype=np.float32)
    Nn = np.zeros((len(recs), 3, ns), dtype=np.float32) if has_sn == {True} else None
    for t, (x, it, sn) in enumerate(recs):
        X[t, :, :n[t]] = x
        I[t, :n[t]] = np.asarray(it).reshape(-1)
        if Nn is not None:
            Nn[t, :, :n[t]] = sn
    dev = torch.device(device)
    return dict(xyz=torch.from_numpy(X).to(dev), intensity=torch.from_numpy(I).to(dev),
                sn=None if Nn is None else torch.from_numpy(Nn).to(dev), n_pts=np.array(n),
                frame_sample=np.array(fs), frame_T=np.concatenate(Ts))


def assemble_batch(frames, mode, seed, input_pt_num=INPUT_PT_NUM, node_a_num=NODE_NUM, node_b_num=NODE_NUM,
                   voxel_size=0.3, range_max=None, pre=np.eye(4), P_base=np.eye(4),
                   amplitudes=(0.0, 0.0, 0.0, 0.0, 2.0 * math.pi, 0.0), flip=True, jitter=("pc", "sn"),
                   sigma=SIGMA, clip=CLIP, rng=None, stream=None):
    """The loaders' point side for S samples.  frames: dict(xyz [T,3,n] f32, intensity [T,n] f32, sn [T,3,n] f32 or
    None -- CUDA; n_pts [T], frame_sample [T] (non-decreasing from 0, anchor frame first) and frame_T [T,4,4] float64
    on the host).  kitti_args / oxford_args give pre, P_base and the rest as the two loaders compose them.  Steps:
    accumulate (range mask), the voxel step for clouds above 2 input_pt_num points, downsample_np, Pr from
    random_transforms(mode, amplitudes, rng) with jitter in train mode, points -> (Pr pre) p, and farthest-point
    node sets from 8 M candidates each.  Returns dict(pc [S,3,N], intensity [S,1,N], sn [S,3,N], node_a [S,3,Ma],
    node_b [S,3,Mb] f32, node_a_idx, node_b_idx (into pc) int32, Pr [S,4,4] f64, P [S,3,4] f32, P44 [S,4,4] f64,
    flip [S] bool, n_before_resample [S] int32)."""
    N = int(input_pt_num)
    if N < 1:
        raise ValueError(f"input_pt_num must be at least 1 (got {input_pt_num})")
    for m in (node_a_num, node_b_num):
        if int(m) != m or m < 1 or 8 * m > N:
            raise ValueError(f"8 * node_num ({8 * m}) must be in [8, input_pt_num={N}]")
    xyz, inten, sn, cnt, cnt_h = accumulate(frames["xyz"], frames["intensity"], frames.get("sn"), frames["n_pts"],
                                            frames["frame_sample"], frames["frame_T"], range_max, stream)
    if cnt_h.min() < 1:
        raise ValueError(f"sample {int(np.argmin(cnt_h))} has no point left to assemble")
    S = cnt_h.shape[0]
    with torch.cuda.device(xyz.device), torch.cuda.stream(stream):
        cnt, cnt_h = _voxel_step(xyz, inten, sn, cnt, cnt_h, N, pointprep._positive(voxel_size, "voxel_size"), stream)
        Pr, flipped = random_transforms(S, mode, amplitudes, rng, flip)
        pre = np.broadcast_to(np.asarray(pre, dtype=np.float64), (S, 4, 4))
        P44 = compose(np.broadcast_to(np.asarray(P_base, dtype=np.float64), (S, 4, 4)), rigid_inverse(Pr))
        out = resample(xyz, inten, sn, cnt, N, seed, M=compose(Pr, pre), jitter=jitter if mode == "train" else (),
                       sigma=sigma, clip=clip, stream=stream)
        res = dict(pc=out["pc"], intensity=out["intensity"], sn=out["sn"], src_index=out["src"],
                   Pr=Pr, P=torch.from_numpy(P44[:, :3].astype(np.float32)), P44=P44, flip=flipped,
                   n_before_resample=cnt)
        for name, m, node_set in (("node_a", node_a_num, 0), ("node_b", node_b_num, 1)):
            cidx, cxyz = candidates(out["pc"], 8 * m, seed, node_set, stream)
            fidx, nodes = farthest_point_sample(cxyz, None, m, stream=stream)
            res[name] = nodes
            res[name + "_idx"] = torch.gather(cidx, 1, fidx.long())
    return res


class FarthestSampler:
    """Drop-in for data/kitti_helper.py FarthestSampler: sample(pts [dim,n], k) -> (float64 [dim,k], int64 [k]).  The
    start index is np.random.randint(len(pts)) drawn on the host as the reference draws it (len(pts) = dim rows, so
    it is 0..dim-1), and the rounds run on the GPU; under the same np.random state the result is the reference's,
    bit for bit."""

    def __init__(self, dim=3):
        self.dim = dim

    def sample(self, pts, k):
        pts = np.asarray(pts)
        init_idx = np.random.randint(len(pts))
        if pts.ndim != 2 or pts.shape[0] != self.dim:
            raise ValueError(f"pts must be [{self.dim}, n]")
        n = pts.shape[1]
        if init_idx >= n:
            raise IndexError(f"index {init_idx} is out of bounds for a set of {n} points")
        x = torch.from_numpy(np.ascontiguousarray(pts, dtype=np.float64)[None]).cuda()
        start = torch.tensor([init_idx], dtype=torch.int32, device=x.device)
        idx, nodes = farthest_point_sample(x, None, k, start=start)
        return nodes[0].cpu().numpy(), idx[0].cpu().numpy().astype(np.int64)


class ProjectiveFarthestSampler:
    """Drop-in for data/kitti_helper.py ProjectiveFarthestSampler: the points are projected by projection_K on the host
    (np.dot, then x / z as the reference does) and sampled by the 2-D FarthestSampler.  Returns (pts[:, idx], idx)."""

    def __init__(self):
        self.fps_2d = FarthestSampler(dim=2)

    def sample(self, pts, k, projection_K):
        pts_2d = np.dot(projection_K, pts)
        pts_2d = pts_2d[0:2, :] / pts_2d[2:, :]
        _, nodes_idx = self.fps_2d.sample(pts_2d, k)
        return pts[:, nodes_idx], nodes_idx
