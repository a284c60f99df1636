"""KITTI camera-frame scan records and LiDAR depth maps (data/kitti/kitti_pc_bin_to_npy_in_img_frame.py) without
Open3D or scipy.

For every raw scan of a sequence and each colour camera (P2, P3) the reference writes two products:
  - data_odometry_velodyne_{P2,P3}_npy/sequences/%02d/voxel%.1f-SNr%.1f/%06d.npy, the voxel-downsampled scan with
    normals and nearest-point intensity moved into the camera frame: [7, M] float32 (x, y, z, intensity, nx, ny, nz);
  - data_odometry_color_depth_npy/sequences/%02d/image_{2,3}/%06d.npy, the raw scan projected through K, each pixel
    keeping its nearest point's depth, and every empty pixel filled with the depth of its nearest filled pixel and the
    distance to it: [2, H, W] float32 (depth, distance).

depth_maps and camera_records run csrc/kitti_depth.cu (and pointprep.downsample_scans, the chain prepare_scans also
uses) for many (scan, camera) pairs per call; build_sequence and build_root go from files to files.  DESIGN.md 4.33
states the contract and where it deliberately differs from the reference.  There is no CPU fallback.
"""
import os
import shutil
import struct

import numpy as np
import torch

from . import _native, kitti, pointprep
from ._native import _ptr, _require_cuda, _stream_ptr, _workspace
from .frustum import _ws_cache
from .icp import _check, pack_clouds

VOXEL_SIZE = pointprep.VOXEL_SIZE      # process_kitti's downsample_voxel_size, sn_radius, sn_max_nn
SN_RADIUS = pointprep.SN_RADIUS
SN_MAX_NN = pointprep.SN_MAX_NN
CAMERAS = ("P2", "P3")
SEQS = tuple(range(22))
BATCH = 32
MAX_SIDE = 32767


def velodyne_dir(velodyne_root, seq):
    return os.path.join(velodyne_root, "sequences", "%02d" % seq, "velodyne")


def velodyne_path(velodyne_root, seq, i):
    return os.path.join(velodyne_dir(velodyne_root, seq), "%06d.bin" % i)


def record_folder(voxel_size=VOXEL_SIZE, sn_radius=SN_RADIUS):
    """The reference's record folder name, 'voxel%.1f-SNr%.1f'."""
    return "voxel%.1f-SNr%.1f" % (voxel_size, sn_radius)


def record_dir(root, seq, key, voxel_size=VOXEL_SIZE, sn_radius=SN_RADIUS):
    return os.path.join(root, "data_odometry_velodyne_%s_npy" % key, "sequences", "%02d" % seq,
                        record_folder(voxel_size, sn_radius))


def depth_dir(root, seq, key):
    return os.path.join(root, "data_odometry_color_depth_npy", "sequences", "%02d" % seq, "image_" + key[1])


def output_dirs(root, seq, voxel_size=VOXEL_SIZE, sn_radius=SN_RADIUS):
    """The four folders a sequence writes: the P2 and P3 records, then the image_2 and image_3 depth maps."""
    return ([record_dir(root, seq, k, voxel_size, sn_radius) for k in CAMERAS] +
            [depth_dir(root, seq, k) for k in CAMERAS])


def sample_num(velodyne_root, seq):
    """The reference's sample_num: the number of entries of the sequence's velodyne folder."""
    d = kitti._require(velodyne_dir(velodyne_root, seq), "velodyne folder")
    n = len(os.listdir(d))
    if n == 0:
        raise ValueError(f"KITTI sequence {seq:02d} is empty: no scan in {d}")
    return n


def image_size(path):
    """(H, W) of a frame: from the .npy header (the array is not read) or from a PNG's IHDR chunk."""
    kitti._require(path, "image")
    with open(path, "rb") as f:
        if path.endswith(".npy"):
            try:
                version = np.lib.format.read_magic(f)
                read = np.lib.format.read_array_header_1_0 if version == (1, 0) else \
                    np.lib.format.read_array_header_2_0
                shape = read(f)[0]
            except ValueError as e:
                raise ValueError(f"{path}: not a .npy file ({e})") from None
            if len(shape) < 2:
                raise ValueError(f"{path}: an image has at least two dimensions (got shape {shape})")
            return int(shape[0]), int(shape[1])
        head = f.read(24)
    if len(head) < 24 or head[:8] != b"\x89PNG\r\n\x1a\n" or head[12:16] != b"IHDR":
        raise ValueError(f"{path}: not a PNG file with an IHDR chunk")
    w, h = struct.unpack(">II", head[16:24])
    return int(h), int(w)


def read_scan(path):
    """A velodyne scan [4, N] float32, as the reference's read_velodyne_bin returns it."""
    kitti._require(path, "velodyne scan")
    size = os.path.getsize(path)
    if size % 16:
        raise ValueError(f"{path}: {size} bytes is not a whole number of (x, y, z, reflectance) float32 records")
    scan = pointprep.read_velodyne_bin(path)
    if not np.isfinite(scan[:3]).all():
        raise ValueError(f"{path}: the scan has a non-finite coordinate")
    return scan


def plan_sequence(root, velodyne_root, seq):
    """The host half of process_kitti for one sequence: sample_num, the calibration's Pc = np.dot(P_key, Tr) and
    P_key_K per camera, and every frame's image size per camera.  Returns a dict."""
    n = sample_num(velodyne_root, seq)
    calib = kitti.read_calib(root, seq)
    Pc, K, sizes = {}, {}, {}
    for key in CAMERAS:
        Pc[key] = kitti.camera_Pc(calib, key)
        K[key] = np.asarray(calib[key + "_K"], dtype=np.float32)
        sizes[key] = [image_size(kitti.image_path(root, seq, key, i)) for i in range(n)]
    return dict(root=root, velodyne_root=velodyne_root, seq=int(seq), n=n, Pc=Pc, K=K, sizes=sizes)


def _pairs(xyz, n_pts, Pc, K):
    if not (isinstance(xyz, torch.Tensor) and xyz.is_cuda and xyz.dim() == 3 and xyz.shape[1] == 3):
        raise ValueError("xyz must be a [S,3,N] float32 CUDA tensor")
    S, _, N = xyz.shape
    _check(xyz, "xyz", torch.float32, (S, 3, N), None)
    if n_pts is None:
        n_pts = torch.full((S,), N, dtype=torch.int32, device=xyz.device)
    _check(n_pts, "n_pts", torch.int32, (S,), xyz.device)
    Pc = np.ascontiguousarray(Pc.cpu().numpy() if isinstance(Pc, torch.Tensor) else Pc, dtype=np.float64)
    if Pc.ndim != 3 or Pc.shape[1:] != (4, 4) or Pc.shape[0] < S or Pc.shape[0] % S or not np.isfinite(Pc).all():
        raise ValueError(f"Pc must be [T,4,4] finite with T a positive multiple of S = {S} (got {Pc.shape})")
    T = Pc.shape[0]
    if K is not None:
        K = np.ascontiguousarray(K.cpu().numpy() if isinstance(K, torch.Tensor) else K, dtype=np.float32)
        if K.shape != (T, 3, 3) or not np.isfinite(K).all():
            raise ValueError(f"K must be [T,3,3] = [{T},3,3] finite float32 (got {K.shape})")
    return S, N, T, n_pts, Pc, K


def depth_maps(xyz, n_pts, Pc, K, H, W, stream=None):
    """The reference's depth map for T (scan, camera) pairs of one image size: pair t projects scan t // (T // S) of
    xyz [S,3,N] f32 (n_pts [S] int32 or None = N) through Pc[t] [4,4] f64 and K[t] [3,3] float32 (numpy or tensors).
    Returns [T,2,H,W] float32 on xyz's device: plane 0 the depth, plane 1 the distance to the nearest projected point
    (DESIGN.md 4.33)."""
    _require_cuda()
    lib = _native.load()
    S, N, T, n_pts, Pc, K = _pairs(xyz, n_pts, Pc, K)
    H, W = int(H), int(W)
    if not (1 <= H <= MAX_SIDE and 1 <= W <= MAX_SIDE and (H - 1) ** 2 + (W - 1) ** 2 < 2**31):
        raise ValueError(f"H and W must be in [1, {MAX_SIDE}] with (H-1)^2 + (W-1)^2 < 2^31 (got {H} x {W})")
    if not bool(torch.isfinite(xyz).all()):
        raise ValueError("xyz has a non-finite coordinate")
    dev = xyz.device
    with torch.cuda.device(dev), torch.cuda.stream(stream):
        sp = _stream_ptr(stream)
        Pc_d = torch.from_numpy(Pc).to(dev)
        K_d = torch.from_numpy(K).to(dev)
        out = torch.empty((T, 2, H, W), dtype=torch.float32, device=dev)
        rc = lib.kitti_depth_project_f32(_ptr(xyz), N, _ptr(n_pts), S, _ptr(Pc_d), _ptr(K_d), T, H, W, _ptr(out), sp)
        _native.check(rc, "kitti_depth_project")
        ws = _workspace(_ws_cache, max(lib.kitti_depth_fill_workspace_bytes(T, H, W), 1), dev, stream)
        rc = lib.kitti_depth_fill_f32(_ptr(xyz), N, _ptr(n_pts), S, _ptr(Pc_d), _ptr(K_d), T, H, W, _ptr(out),
                                      _ptr(ws), ws.numel(), sp)
        _native.check(rc, "kitti_depth_fill")
    return out


def camera_records(xyz, intensity, n_pts, Pc, voxel_size=VOXEL_SIZE, sn_radius=SN_RADIUS, sn_max_nn=SN_MAX_NN,
                   stream=None):
    """The reference's camera-frame records for T (scan, camera) pairs: pointprep.downsample_scans of xyz [S,3,N] f32
    (intensity [S,N] f32, n_pts [S] int32 or None), then for pair t the fp64 centres of scan t // (T // S) moved by
    Pc[t] [4,4] f64, the intensity, and the normals mapped NWU -> camera (x <- -y, y <- -z, z <- x).  Returns
    (records [T,7,N] float32, zeros past m_pts; m_pts [S] int32)."""
    _require_cuda()
    lib = _native.load()
    S, N, T, n_pts, Pc, _ = _pairs(xyz, n_pts, Pc, None)
    d = pointprep.downsample_scans(xyz, intensity, n_pts, voxel_size, sn_radius, sn_max_nn, stream=stream)
    dev = xyz.device
    with torch.cuda.device(dev), torch.cuda.stream(stream):
        Pc_d = torch.from_numpy(Pc).to(dev)
        out = torch.empty((T, 7, N), dtype=torch.float32, device=dev)
        rc = lib.kitti_depth_records_f32(_ptr(d["xyz"]), _ptr(d["normals"]), _ptr(d["intensity"]), _ptr(d["m_pts"]),
                                         N, S, _ptr(Pc_d), T, _ptr(out), _stream_ptr(stream))
        _native.check(rc, "kitti_depth_records")
    return out, d["m_pts"]


def _size_runs(plan, frames):
    """Split `frames` where the image size changes: [(frames, keys, (H, W))], each run one depth_maps call.  A frame
    whose two cameras differ in size becomes one run per camera."""
    runs = []
    for i in frames:
        sz = [plan["sizes"][k][i] for k in CAMERAS]
        if sz[0] != sz[1]:
            runs += [([i], (k,), s) for k, s in zip(CAMERAS, sz)]
        elif runs and runs[-1][1] == CAMERAS and runs[-1][2] == sz[0]:
            runs[-1][0].append(i)
        else:
            runs.append(([i], CAMERAS, sz[0]))
    return runs


def build_frames(plan, frames, voxel_size=VOXEL_SIZE, sn_radius=SN_RADIUS, sn_max_nn=SN_MAX_NN, device="cuda",
                 stream=None):
    """process_kitti's per-scan body for `frames` of a plan_sequence plan.  Returns dict(records {(i, key): [7, M]
    float32}, maps {(i, key): [2, H, W] float32}) as numpy."""
    scans = [read_scan(velodyne_path(plan["velodyne_root"], plan["seq"], i)) for i in frames]
    xyz, n = pack_clouds([s[:3] for s in scans], device)
    inten = np.zeros((len(scans), xyz.shape[2]), dtype=np.float32)
    for s, scan in enumerate(scans):
        inten[s, :scan.shape[1]] = scan[3]
    Pc = np.stack([plan["Pc"][k] for _ in frames for k in CAMERAS])
    rec, m = camera_records(xyz, torch.from_numpy(inten).to(xyz.device), n, Pc, voxel_size, sn_radius, sn_max_nn,
                            stream)
    rec, m = rec.cpu().numpy(), m.cpu().numpy()
    out = dict(records={}, maps={})
    for s, i in enumerate(frames):
        for c, k in enumerate(CAMERAS):
            out["records"][(i, k)] = np.ascontiguousarray(rec[2 * s + c, :, :m[s]])
    pos = {i: s for s, i in enumerate(frames)}
    for run, keys, (H, W) in _size_runs(plan, frames):
        sel = [pos[i] for i in run]
        Pc = np.stack([plan["Pc"][k] for _ in run for k in keys])
        K = np.stack([plan["K"][k] for _ in run for k in keys])
        maps = depth_maps(xyz[sel].contiguous(), n[sel].contiguous(), Pc, K, H, W, stream).cpu().numpy()
        for s, i in enumerate(run):
            for c, k in enumerate(keys):
                out["maps"][(i, k)] = maps[len(keys) * s + c]
    return out


def build_sequence(root, velodyne_root, seq, voxel=VOXEL_SIZE, sn_radius=SN_RADIUS, sn_max_nn=SN_MAX_NN, batch=BATCH,
                   log=None):
    """process_kitti(root, velodyne_root, [seq], voxel, sn_radius, sn_max_nn): writes both cameras' records and depth
    maps of every scan, `batch` scans per device call, with one log line per batch.  A sequence whose four output
    folders exist is skipped.  The files go to '.partial' siblings that are renamed once the sequence is complete, so
    an interrupted run is redone rather than skipped.  Returns the number of scans written (0 when skipped)."""
    log = log or (lambda s: None)
    if int(batch) != batch or batch < 1:
        raise ValueError(f"batch must be a positive integer (got {batch})")
    dirs = output_dirs(root, seq, voxel, sn_radius)
    have = [d for d in dirs if os.path.exists(d)]
    if len(have) == len(dirs):
        log(f"{seq:02d}: output folders exist, skip")
        return 0
    if have:
        missing = sorted(set(dirs) - set(have))
        raise FileExistsError(f"KITTI sequence {seq:02d} is partly built: {have} exist but not {missing}; remove "
                              "them to rebuild")
    plan = plan_sequence(root, velodyne_root, seq)
    parts = [d + ".partial" for d in dirs]
    for p in parts:
        if os.path.isdir(p):
            shutil.rmtree(p)
        os.makedirs(p)
    n = plan["n"]
    for s in range(0, n, int(batch)):
        frames = list(range(s, min(s + int(batch), n)))
        res = build_frames(plan, frames, voxel, sn_radius, sn_max_nn)
        for i in frames:
            for c, k in enumerate(CAMERAS):
                np.save(os.path.join(parts[c], "%06d.npy" % i), res["records"][(i, k)])
                np.save(os.path.join(parts[2 + c], "%06d.npy" % i), res["maps"][(i, k)])
        log(f"{seq:02d}: scans {frames[0]}-{frames[-1]} of {n}, "
            f"{sum(r.shape[1] for (i, k), r in res['records'].items() if k == 'P2')} voxels")
    for p, d in zip(parts, dirs):
        os.rename(p, d)
    return n


def build_root(root, velodyne_root, seqs=SEQS, voxel=VOXEL_SIZE, sn_radius=SN_RADIUS, sn_max_nn=SN_MAX_NN,
               batch=BATCH, log=None):
    """process_kitti for each sequence in turn, on one GPU.  Returns {seq: scans written}."""
    return {int(seq): build_sequence(root, velodyne_root, seq, voxel, sn_radius, sn_max_nn, batch, log)
            for seq in seqs}
