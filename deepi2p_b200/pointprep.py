"""LiDAR scan preparation (data/kitti/kitti_pc_bin_to_npy_with_downsample_sn.py and the loaders' Open3D helpers) on
the GPU.

voxel_downsample, estimate_normals and nearest wrap the C-ABI calls of csrc/pointprep.cu for S clouds at once;
prepare_scans chains them into the per-scan body of the preparation script; downsample_with_intensity_sn and
downsample_with_reflectance are drop-ins for the loaders' functions of those names (numpy in, numpy out).  DESIGN.md
"Scan preparation" states the contract and where it deliberately differs from Open3D: voxels come out in ascending
(ix, iy, iz) order, the covariance is taken about each point, the eigenvectors come from a Jacobi solver, and
coordinates are float32.  There is no CPU fallback.
"""
import numpy as np
import torch

from . import _native
from .frustum import _ptr, _require_cuda, _stream_ptr, _workspace
from .icp import _check, pack_clouds

VOXEL_SIZE = 0.1              # kitti_pc_bin_to_npy_with_downsample_sn.py: downsample_voxel_size, sn_radius, sn_max_nn
SN_RADIUS = 0.6
SN_MAX_NN = 30
MAX_NN = 64                   # the largest max_nn the kernels hold
MAX_ATTR = 64                 # attribute channels of one voxel_downsample call


def _positive(v, name):
    v = float(v)
    if not (np.isfinite(v) and v > 0):
        raise ValueError(f"{name} must be positive (got {v})")
    return v


def _normal_params(radius, max_nn, orient):
    radius = _positive(radius, "radius")
    if int(max_nn) != max_nn or not 1 <= int(max_nn) <= MAX_NN:
        raise ValueError(f"max_nn must be an integer in [1, {MAX_NN}] (got {max_nn})")
    o = np.ascontiguousarray(orient, dtype=np.float64).reshape(-1)
    if o.shape != (3,) or not np.isfinite(o).all():
        raise ValueError("orient must be three finite numbers")
    return radius, o


def _cloud_batch(xyz, n_pts, name="xyz"):
    if not (isinstance(xyz, torch.Tensor) and xyz.is_cuda and xyz.dim() == 3 and xyz.shape[1] == 3):
        raise ValueError(f"{name} must be a [S,3,N] CUDA tensor")
    S, _, N = xyz.shape
    _check(xyz, name, xyz.dtype if xyz.dtype in (torch.float32, torch.float64) else torch.float32, (S, 3, N), None)
    if N % 16:
        raise ValueError(f"{name}'s point stride ({N}) must be a multiple of 16 (pack_clouds pads)")
    if n_pts is not None:
        _check(n_pts, "n_pts", torch.int32, (S,), xyz.device)
    if not bool(torch.isfinite(xyz).all()):
        raise ValueError(f"{name} has a non-finite coordinate")
    return S, N


def voxel_downsample(xyz, n_pts, voxel_size, attr=None, stream=None):
    """Open3D voxel_down_sample for S clouds.  xyz [S,3,N] f32, n_pts [S] int32 or None (= N), attr [S,C,N] f64 or
    None.  Returns dict(xyz [S,3,N] f64, m_pts [S] int32, attr [S,C,N] f64 when given): per cloud, the mean of each
    occupied voxel's points (and attributes) in ascending (ix, iy, iz) order; entries past m_pts are zero.  Raises
    ValueError when a cloud spans 2^21 or more voxels along an axis.  The call waits for the stream's earlier work."""
    voxel_size = _positive(voxel_size, "voxel_size")
    _require_cuda()
    lib = _native.load()
    S, N = _cloud_batch(xyz, n_pts)
    _check(xyz, "xyz", torch.float32, (S, 3, N), None)
    C = 0
    if attr is not None:
        if not (isinstance(attr, torch.Tensor) and attr.dim() == 3):
            raise ValueError("attr must be a [S,C,N] float64 CUDA tensor")
        C = attr.shape[1]
        _check(attr, "attr", torch.float64, (S, C, N), xyz.device)
        if C > MAX_ATTR:
            raise ValueError(f"at most {MAX_ATTR} attribute channels")
    dev = xyz.device
    with torch.cuda.device(dev), torch.cuda.stream(stream):
        res = dict(xyz=torch.zeros((S, 3, N), dtype=torch.float64, device=dev),
                   m_pts=torch.zeros((S,), dtype=torch.int32, device=dev))
        if C:
            res["attr"] = torch.zeros((S, C, N), dtype=torch.float64, device=dev)
        sp = _stream_ptr(stream)
        ws = _workspace(max(lib.voxel_downsample_workspace_bytes(S, N, C), 1), dev, sp)
        rc = lib.voxel_downsample_batch_f32(_ptr(xyz), _ptr(n_pts), N, S, _ptr(attr), C, voxel_size, _ptr(res["xyz"]),
                                            _ptr(res.get("attr")), _ptr(res["m_pts"]), _ptr(ws), ws.numel(), sp)
    if rc == -22:                   # the only data-dependent rejection: too many voxels along an axis
        raise ValueError(lib.dib_last_error().decode("utf-8", "replace"))
    _native.check(rc, "voxel_downsample")
    return res


def estimate_normals(xyz, m_pts, radius=SN_RADIUS, max_nn=SN_MAX_NN, orient=(0.0, 0.0, 1.0), counts=False,
                     stream=None):
    """Open3D estimate_normals(KDTreeSearchParamHybrid(radius, max_nn)) then orient_normals_to_align_with_direction
    (orient) for S clouds.  xyz [S,3,M] f32, m_pts [S] int32 or None.  Returns normals [S,3,M] f64 (entries past m_pts
    zero) and, with counts, also the neighbours used per point [S,M] int32."""
    radius, o = _normal_params(radius, max_nn, orient)
    _require_cuda()
    lib = _native.load()
    S, M = _cloud_batch(xyz, m_pts)
    _check(xyz, "xyz", torch.float32, (S, 3, M), None)
    dev = xyz.device
    with torch.cuda.device(dev), torch.cuda.stream(stream):
        nrm = torch.zeros((S, 3, M), dtype=torch.float64, device=dev)
        cnt = torch.zeros((S, M), dtype=torch.int32, device=dev) if counts else None
        sp = _stream_ptr(stream)
        ws = _workspace(max(lib.estimate_normals_workspace_bytes(S, M), 1), dev, sp)
        rc = lib.estimate_normals_batch_f32(_ptr(xyz), _ptr(m_pts), M, S, radius, int(max_nn),
                                            o.ctypes.data_as(_native._c.c_void_p), _ptr(nrm), _ptr(cnt), _ptr(ws),
                                            ws.numel(), sp)
    _native.check(rc, "estimate_normals")
    return (nrm, cnt) if counts else nrm


def nearest(q, q_pts, xyz, m_pts, stream=None):
    """Index of the nearest point of cloud s of xyz [S,3,M] f32 (m_pts [S] int32 or None) for every query of q
    [S,3,Q] f64 (q_pts [S] int32 or None); ties go to the lowest index, -1 for an empty cloud.  Returns [S,Q] int32
    (entries past q_pts are -1)."""
    _require_cuda()
    lib = _native.load()
    S, M = _cloud_batch(xyz, m_pts)
    _check(xyz, "xyz", torch.float32, (S, 3, M), None)
    if not (isinstance(q, torch.Tensor) and q.dim() == 3 and q.shape[0] == S):
        raise ValueError("q must be a [S,3,Q] float64 CUDA tensor")
    Q = q.shape[2]
    _check(q, "q", torch.float64, (S, 3, Q), xyz.device)
    if Q % 16:
        raise ValueError(f"q's point stride ({Q}) must be a multiple of 16")
    if q_pts is not None:
        _check(q_pts, "q_pts", torch.int32, (S,), xyz.device)
    if not bool(torch.isfinite(q).all()):
        raise ValueError("q has a non-finite coordinate")
    dev = xyz.device
    with torch.cuda.device(dev), torch.cuda.stream(stream):
        idx = torch.full((S, Q), -1, dtype=torch.int32, device=dev)
        sp = _stream_ptr(stream)
        ws = _workspace(max(lib.estimate_normals_workspace_bytes(S, M), 1), dev, sp)
        rc = lib.nearest_batch_f32(_ptr(q), _ptr(q_pts), Q, _ptr(xyz), _ptr(m_pts), M, S, _ptr(idx), _ptr(ws),
                                   ws.numel(), sp)
    _native.check(rc, "nearest")
    return idx


def prepare_scans(xyz, intensity, n_pts, voxel_size=VOXEL_SIZE, sn_radius=SN_RADIUS, sn_max_nn=SN_MAX_NN,
                  orient=(0.0, 0.0, 1.0), stream=None):
    """kitti_pc_bin_to_npy_with_downsample_sn.py:48-74 for S scans: voxel_down_sample(voxel_size), estimate_normals
    (sn_radius, sn_max_nn) on the centres rounded to float32, orientation toward `orient`, and the intensity of the
    nearest original point.  xyz [S,3,N] f32, intensity [S,N] f32, n_pts [S] int32 or None.  Returns (record
    [S,7,N] float32 = (x, y, z, intensity, nx, ny, nz), entries past m_pts zero; m_pts [S] int32)."""
    _positive(voxel_size, "voxel_size")
    _normal_params(sn_radius, sn_max_nn, orient)
    S, N = _cloud_batch(xyz, n_pts)
    _check(intensity, "intensity", torch.float32, (S, N), xyz.device)
    with torch.cuda.device(xyz.device), torch.cuda.stream(stream):
        down = voxel_downsample(xyz, n_pts, voxel_size, stream=stream)
        m = down["m_pts"]
        d32 = down["xyz"].to(torch.float32)
        nrm = estimate_normals(d32, m, sn_radius, sn_max_nn, orient, stream=stream)
        idx = nearest(down["xyz"], m, xyz, n_pts, stream=stream)
        valid = torch.arange(N, device=xyz.device)[None] < m[:, None]
        inten = torch.gather(intensity, 1, idx.clamp(min=0).long()).masked_fill(~valid, 0)
        rec = torch.cat([d32, inten[:, None], nrm.to(torch.float32)], 1)
    return rec, m


def _to_device_cloud(pointcloud):
    pc = np.asarray(pointcloud)
    if pc.ndim != 2 or pc.shape[0] < 3:
        raise ValueError("pointcloud must be [>=3, N]")
    if not np.isfinite(pc[:3]).all():
        raise ValueError("pointcloud has a non-finite coordinate")
    return pack_clouds(pc[:3])


def _downsample_np(pointcloud, attr_rows, voxel_grid_downsample_size):
    """Shared body of the two drop-ins: coordinates rounded to float32, attributes averaged in float64."""
    _positive(voxel_grid_downsample_size, "voxel_grid_downsample_size")
    xyz, n = _to_device_cloud(pointcloud)
    N = xyz.shape[2]
    A = np.zeros((1, len(attr_rows), N))
    for c, row in enumerate(attr_rows):
        A[0, c, :n.item()] = row
    out = voxel_downsample(xyz, n, voxel_grid_downsample_size, attr=torch.from_numpy(A).to(xyz.device))
    m = int(out["m_pts"][0])
    return out["xyz"][0, :, :m].cpu().numpy(), out["attr"][0, :, :m].cpu().numpy()


def downsample_with_intensity_sn(pointcloud, intensity, sn, voxel_grid_downsample_size):
    """Drop-in for data/kitti_pc_img_pose_loader.py:26-45.  pointcloud [3,N], intensity [1,N], sn [3,N] -> (pointcloud
    [3,M] f64, intensity [1,M] f64, sn [3,M] f64).  As the reference does, intensity / max(intensity) is formed in the
    caller's dtype, averaged in float64 and multiplied back; normals are averaged, not re-normalised."""
    intensity_max = np.max(intensity)
    scaled = np.transpose(intensity) / intensity_max                   # [N, 1] in the caller's dtype
    sn = np.asarray(sn)
    pc, A = _downsample_np(pointcloud, [scaled[:, 0].astype(np.float64)] + [sn[a].astype(np.float64) for a in range(3)],
                           voxel_grid_downsample_size)
    return pc, A[0:1] * intensity_max, A[1:4]


def downsample_with_reflectance(pointcloud, reflectance, voxel_grid_downsample_size):
    """Drop-in for data/nuscenes_pc_img_pose_loader.py:31-45 (and the Oxford loader's function of that name).
    pointcloud [3,N], reflectance [N] -> (pointcloud [3,M] f64, reflectance [M] f64)."""
    reflectance_max = np.max(reflectance)
    scaled = reflectance / reflectance_max
    pc, A = _downsample_np(pointcloud, [np.asarray(scaled).astype(np.float64)], voxel_grid_downsample_size)
    return pc, A[0] * reflectance_max


def read_velodyne_bin(path):
    """A KITTI velodyne scan: [4, N] float32 (x, y, z, reflectance) from N x 4 little-endian float32 records."""
    return np.fromfile(path, dtype="<f4").reshape(-1, 4).T.astype(np.float32)
