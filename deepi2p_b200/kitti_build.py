"""KITTI accumulated-frame records (data/kitti/frame_accumulation.py accumulate_sequence) without Open3D.

For every frame i of a sequence the reference concatenates the prepared scans (voxel0.1-SNr0.6) of the stride frames
around i, each without the points on the ego car and moved into frame i, voxelises the cloud with colours and normals
and keeps the voxels within accumulate_radius of the sensor, writing stride%d-acc%d-voxel%.1f/%06d.npy.

The host half (plan_sequence, frame_pairs) restates the stride walk, the windows and the transforms with the
reference's own numpy calls in its order, so they are its values bit for bit on the same numpy.  The device half
(build_frames) runs csrc/kitti_build.cu's count and scatter, pointprep.voxel_downsample (the Open3D restatement of
DESIGN.md 4.10) and the range compaction for many output frames per call, reading the stride records from an
assemble.ScanStore.  build_sequence and build_root go from files to files.  DESIGN.md 4.29 states the contract and
where it deliberately differs from the reference.  There is no CPU fallback.
"""
import bisect
import os
import shutil

import numpy as np
import torch

from . import _native, assemble, kitti, pointprep
from ._native import _ptr, _require_cuda, _stream_ptr, _workspace
from .frustum import _ws_cache, round_up

# frame_accumulation.py main(): the parameters the published records were written with
FRAME_STRIDE_DIST = 4
ACCUMULATE_RADIUS = 50
VOXEL_SIZE = 0.4
SEQS = tuple(range(11))
BATCH = 64
# The ego-car box of accumulate_sequence (x_lo, x_hi, y_lo, y_hi), both strict; -2.7 * 0.75 is formed in float64 and,
# like the other three, rounded to float32 when numpy compares the float32 record against it.
EGO_BOX = (-2.7 * 0.75, 2.7, -0.8, 0.8)


def output_folder(frame_stride_dist=FRAME_STRIDE_DIST, accumulate_radius=ACCUMULATE_RADIUS, voxel_size=VOXEL_SIZE):
    """The reference's output folder name, 'stride%d-acc%d-voxel%.1f'."""
    return "stride%d-acc%d-voxel%.1f" % (frame_stride_dist, accumulate_radius, voxel_size)


def accumulate_frames(frame_stride_dist, accumulate_radius):
    """int(round(accumulate_radius / frame_stride_dist)): Python's round, halves to even (12.5 -> 12)."""
    return int(round(accumulate_radius / frame_stride_dist))


def read_pose(root, seq, i):
    """np.load(poses/%02d/%06d.npz)['pose'] in its stored dtype, as accumulate_sequence reads it."""
    with np.load(kitti._require(kitti.pose_path(root, seq, i), "pose")) as z:
        return z["pose"]


def stride_list(poses, frame_stride_dist):
    """The greedy walk: frame 0, then every frame i whose translation from the last kept frame,
    norm(dot(inv(P_prev), P_i)[0:3, 3]), is strictly above frame_stride_dist."""
    out = [0]
    P_prev = poses[0]
    for i in range(1, len(poses)):
        P_prev_i = np.dot(np.linalg.inv(P_prev), poses[i])
        if np.linalg.norm(P_prev_i[0:3, 3]) > frame_stride_dist:
            out.append(i)
            P_prev = poses[i]
    return out


def windows(strides, n, acc):
    """[n, 2] int64: per frame i the inclusive range [lo, hi] of stride-list positions, the bisect_left position of i
    widened by acc on both sides and clamped to the list.  lo > hi marks an empty window (acc = 0 past the last
    stride frame)."""
    out = np.empty((n, 2), dtype=np.int64)
    for i in range(n):
        k = bisect.bisect_left(strides, i)
        out[i] = max(0, k - acc), min(len(strides) - 1, k + acc)
    return out


def plan_sequence(root, seq, frame_stride_dist=FRAME_STRIDE_DIST, accumulate_radius=ACCUMULATE_RADIUS,
                  record_dir=kitti.RECORD_DIR, Tr=None):
    """The host half of accumulate_sequence for one sequence: sample_num (the number of entries of the record
    folder), the poses, the stride list, accumulate_frames, the windows and Tr (the calibration's float64 4 x 4, or
    the one given).  Returns a dict."""
    folder = kitti._require(kitti.record_dir(root, seq, record_dir), "scan record folder")
    n = len(os.listdir(folder))
    if n == 0:
        raise ValueError(f"KITTI sequence {seq:02d} is empty: no scan record in {folder}")
    if Tr is None:
        Tr = kitti.read_calib(root, seq)["Tr"]
    poses = [read_pose(root, seq, i) for i in range(n)]
    strides = stride_list(poses, frame_stride_dist)
    acc = accumulate_frames(frame_stride_dist, accumulate_radius)
    return dict(root=root, seq=int(seq), n=n, poses=poses, strides=strides, acc=acc,
                windows=windows(strides, n, acc), Tr=np.asarray(Tr), Tr_inv=np.linalg.inv(Tr), record_dir=record_dir,
                frame_stride_dist=frame_stride_dist, accumulate_radius=accumulate_radius)


def frame_pairs(plan, frames):
    """The (frame, stride record) pairs of `frames`: returns (strides [T] frame numbers in window order, first
    [B + 1] int32 (frame k owns pairs first[k]:first[k+1]), P [T,4,4] float64 with P_transform =
    dot(Tr_inv, dot(dot(inv(P_i), P_j), Tr))).  Raises ValueError for an empty window."""
    strides, first, Ps = [], [0], []
    for i in frames:
        lo, hi = plan["windows"][i]
        if lo > hi:
            raise ValueError(f"KITTI sequence {plan['seq']:02d} frame {i}: its window of stride frames is empty "
                             f"(accumulate_frames = {plan['acc']}, past the last stride frame)")
        Pi_inv = np.linalg.inv(plan["poses"][i])
        for j in plan["strides"][lo:hi + 1]:
            Pij = np.dot(Pi_inv, plan["poses"][j])
            Ps.append(np.dot(plan["Tr_inv"], np.dot(Pij, plan["Tr"])))
            strides.append(j)
        first.append(len(strides))
    return strides, np.array(first, dtype=np.int32), np.stack(Ps).astype(np.float64)


def _box(box):
    b = np.asarray(box, dtype=np.float64).reshape(-1)
    if b.shape != (4,) or not np.isfinite(b).all() or b[0] > b[1] or b[2] > b[3]:
        raise ValueError(f"box must be four finite numbers (x_lo, x_hi, y_lo, y_hi), lo <= hi (got {box!r})")
    return np.ascontiguousarray(b.astype(np.float32))


def build_frames(store, ids, first, P, voxel_size=VOXEL_SIZE, accumulate_radius=ACCUMULATE_RADIUS, box=EGO_BOX,
                 stream=None):
    """The device half of accumulate_sequence's per-frame body for B = len(first) - 1 output frames: output k
    accumulates the store records ids[first[k]:first[k+1]] (a [7, n] ScanStore, device or pinned), each without its
    points strictly inside `box` and moved by P[t] (points and normals, in fp64), voxelises them at voxel_size with
    colour intensity / max and the normals as attributes, and keeps the voxels with |xy| < accumulate_radius.
    Returns dict(records [B,7,M_max] float32 and m_pts [B] int32 on the device (zeros past m_pts), m_host [B] numpy,
    n_pts [B] numpy (points before the voxel step), imax [B] numpy float32).  An output whose maximum intensity is 0
    gets a NaN intensity row, as numpy's 0 / 0 gives the reference.  Raises ValueError when an output has no point
    left after the ego mask (the reference's np.max of an empty array raises)."""
    _require_cuda()
    lib = _native.load()
    if not isinstance(store, assemble.ScanStore) or not store.has_sn:
        raise ValueError("store must be an assemble.ScanStore of [7, n] records")
    voxel_size = pointprep._positive(voxel_size, "voxel_size")
    radius = float(accumulate_radius)
    if not np.isfinite(radius):
        raise ValueError(f"accumulate_radius must be finite (got {accumulate_radius})")
    ids = np.asarray(ids, dtype=np.int64).reshape(-1)
    first = np.asarray(first, dtype=np.int64).reshape(-1)
    T, B = ids.shape[0], first.shape[0] - 1
    if B < 1 or first[0] != 0 or first[-1] != T or np.any(np.diff(first) < 0):
        raise ValueError("first must run from 0 to len(ids), non-decreasing, with at least one output")
    if T and (ids.min() < 0 or ids.max() >= len(store)):
        raise ValueError(f"record ids must be in [0, {len(store)})")
    P = np.ascontiguousarray(P, dtype=np.float64)
    if P.shape != (T, 4, 4) or not np.isfinite(P).all():
        raise ValueError("P must be [T,4,4] finite")
    b = _box(box)
    dev = store.device
    sp = _stream_ptr(stream)
    planes, ps = store.data.data_ptr(), store.data.stride(0)
    with torch.cuda.device(dev), torch.cuda.stream(stream):
        meta = torch.from_numpy(np.concatenate([store.offsets[ids], store.counts[ids]]).astype(np.int64)).to(dev)
        off_d = meta[:T]
        n_d = meta[T:].to(torch.int32)
        first_d = torch.from_numpy(first.astype(np.int32)).to(dev)
        pair_out = torch.from_numpy(np.repeat(np.arange(B, dtype=np.int32), np.diff(first))).to(dev)
        P_d = torch.from_numpy(P).to(dev)
        pos = torch.zeros((max(T, 1),), dtype=torch.int64, device=dev)
        n_pts = torch.zeros((B,), dtype=torch.int64, device=dev)
        imax = torch.zeros((B,), dtype=torch.float32, device=dev)
        ws = _workspace(_ws_cache, max(lib.kitti_build_count_workspace_bytes(T), 1), dev, stream)
        rc = lib.kitti_build_count_f32(planes, ps, _ptr(off_d), _ptr(n_d), T, _ptr(first_d), B,
                                       b.ctypes.data_as(_native._c.c_void_p), _ptr(pos), _ptr(n_pts), _ptr(imax),
                                       _ptr(ws), ws.numel(), sp)
        _native.check(rc, "kitti_build_count")
        n_host = n_pts.cpu().numpy()
        for k in np.nonzero(n_host == 0)[0]:
            raise ValueError(f"output frame {k} of the batch has no point outside the ego box")
        N = round_up(int(n_host.max()), 16)
        if B * 4 * N >= 2**31:
            raise ValueError(f"a batch of {B} frames of up to {int(n_host.max())} points is too large; use a smaller "
                             "batch")
        xyz = torch.zeros((B, 3, N), dtype=torch.float64, device=dev)
        attr = torch.zeros((B, 4, N), dtype=torch.float64, device=dev)
        rc = lib.kitti_build_scatter_f64(planes, ps, _ptr(off_d), _ptr(n_d), _ptr(pair_out), _ptr(P_d), T, B,
                                         b.ctypes.data_as(_native._c.c_void_p), _ptr(pos), _ptr(imax), N, _ptr(xyz),
                                         _ptr(attr), sp)
        _native.check(rc, "kitti_build_scatter")
        down = pointprep.voxel_downsample(xyz, n_pts.to(torch.int32), voxel_size, attr=attr, stream=stream)
        del xyz, attr
        M = round_up(max(int(down["m_pts"].max()), 1), 16)
        out = torch.empty((B, 7, M), dtype=torch.float32, device=dev)
        cnt = torch.zeros((B,), dtype=torch.int32, device=dev)
        rc = lib.kitti_build_finish_f32(_ptr(down["xyz"]), _ptr(down["attr"]), _ptr(down["m_pts"]), _ptr(imax), B,
                                        radius, N, M, _ptr(out), _ptr(cnt), sp)
        _native.check(rc, "kitti_build_finish")
        m_host = cnt.cpu().numpy()
        return dict(records=out, m_pts=cnt, m_host=m_host, n_pts=n_host, imax=imax.cpu().numpy())


def stride_store(plan, location="cuda", device=None):
    """A ScanStore of the sequence's stride records (the only records accumulate_sequence reads), keyed by frame."""
    recs = []
    for j in plan["strides"]:
        r = kitti.read_record(kitti.record_path(plan["root"], plan["seq"], j, plan["record_dir"]))
        if not np.isfinite(r).all():
            raise ValueError(f"{kitti.record_path(plan['root'], plan['seq'], j, plan['record_dir'])}: the record "
                             "has a non-finite value")
        recs.append(r)
    return assemble.ScanStore(recs, location, keys=list(plan["strides"]), device=device)


def build_plan_frames(store, plan, frames, voxel_size=VOXEL_SIZE, stream=None):
    """build_frames for frames of a plan_sequence plan, the records read from stride_store(plan)."""
    strides, first, P = frame_pairs(plan, frames)
    return build_frames(store, [store.index(j) for j in strides], first, P, voxel_size, plan["accumulate_radius"],
                        stream=stream)


def output_dir(root, seq, frame_stride_dist=FRAME_STRIDE_DIST, accumulate_radius=ACCUMULATE_RADIUS,
               voxel_size=VOXEL_SIZE):
    return kitti.record_dir(root, seq, output_folder(frame_stride_dist, accumulate_radius, voxel_size))


def build_sequence(root, seq, frame_stride_dist=FRAME_STRIDE_DIST, accumulate_radius=ACCUMULATE_RADIUS,
                   voxel_size=VOXEL_SIZE, batch=BATCH, record_dir=kitti.RECORD_DIR, location="cuda", device="cuda",
                   stream=None, log=print):
    """accumulate_sequence(root, seq, Tr, frame_stride_dist, accumulate_radius, voxel_size): writes every frame's
    record to output_dir(...)/%06d.npy, `batch` frames per device call, with one log line per batch.  A sequence
    whose output folder exists is skipped, as the reference skips it.  The records are written to a '.partial' sibling
    that is renamed once the sequence is complete, so an interrupted run is redone rather than skipped.  Returns the
    number of records written (0 when skipped)."""
    if int(batch) != batch or batch < 1:
        raise ValueError(f"batch must be a positive integer (got {batch})")
    out_dir = output_dir(root, seq, frame_stride_dist, accumulate_radius, voxel_size)
    if os.path.exists(out_dir):
        log(f"{out_dir} exists, skip")
        return 0
    plan = plan_sequence(root, seq, frame_stride_dist, accumulate_radius, record_dir)
    store = stride_store(plan, location, device)
    part = out_dir + ".partial"
    if os.path.isdir(part):
        shutil.rmtree(part)
    os.mkdir(part)
    n = plan["n"]
    for s in range(0, n, int(batch)):
        frames = list(range(s, min(s + int(batch), n)))
        res = build_plan_frames(store, plan, frames, voxel_size, stream)
        rec = res["records"].cpu().numpy()
        for k, i in enumerate(frames):
            np.save(os.path.join(part, "%06d.npy" % i), np.ascontiguousarray(rec[k, :, :res["m_host"][k]]))
        log(f"{seq:02d}: frames {frames[0]}-{frames[-1]} of {n} ({len(plan['strides'])} stride frames), "
            f"{int(res['n_pts'].sum())} points in, {int(res['m_host'].sum())} out")
    os.rename(part, out_dir)
    return n


def build_root(root, seqs=SEQS, frame_stride_dist=FRAME_STRIDE_DIST, accumulate_radius=ACCUMULATE_RADIUS,
               voxel_size=VOXEL_SIZE, batch=BATCH, record_dir=kitti.RECORD_DIR, log=print):
    """frame_accumulation.py main(): build_sequence for each sequence in turn, on one GPU."""
    return {int(seq): build_sequence(root, seq, frame_stride_dist, accumulate_radius, voxel_size, batch, record_dir,
                                     log=log) for seq in seqs}
