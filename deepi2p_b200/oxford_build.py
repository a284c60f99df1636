"""Build an Oxford RobotCar root (data/oxford/build_dataset.py) from the raw LMS-front scans and visual odometry, with
the point work on the device and without Open3D or the RobotCar SDK's Python code.

The host reads the raw text files, restates the SDK's transform and pose interpolation in numpy (marked with a warning
sign in DESIGN.md 4.24: the SDK's source is not part of this project), chains the VO rows once per traversal and plans
the clouds: the camera list, the centre walk, the windows and the velocity rule.  A ScanStore-like device store holds
the traversal's scans as fp64 planes; csrc/oxford_build.cu then walks each window (skip test, transforms), gathers
the masked points, pointprep's fp64 voxel grid averages them and the output transform packs float32 [4, M] records.
build_traversal writes the root that oxford.OxfordDataset, oxford.scan_store and oxford.oxford_batch read.
"""
import bisect
import csv
import math
import os
import shutil

import numpy as np
import torch

from . import _native, oxford, pointprep
from ._native import _ptr, _require_cuda, _stream_ptr
from .frustum import round_up

LMS_HZ = 50                                 # build_dataset.py:285, the LMS-front scan rate the velocity rule assumes
PARAMS = dict(pc_sample_distance=2.0, min_vehicle_velocity=0.2, accumulation_distance=100.0, ignore_first_n_second=20,
              voxel_grid_downsample_size=0.1, remove_ground_threshold=0.1)      # build_dataset.py:410-420
CAMERA = "stereo"                           # CameraModel(models_dir, '<t>/stereo/centre').camera
CAMERA_MODEL = "stereo_narrow_left.txt"     # the model file of the stereo centre camera


# ---------------------------------------------------------------- SDK restatements (DESIGN.md 4.24, marked there)
def euler_to_so3(rpy):
    """R = Rz(yaw) Ry(pitch) Rx(roll) for rpy [..., 3] -> [..., 3, 3]."""
    rpy = np.asarray(rpy, dtype=np.float64)
    cr, sr = np.cos(rpy[..., 0]), np.sin(rpy[..., 0])
    cp, sp = np.cos(rpy[..., 1]), np.sin(rpy[..., 1])
    cy, sy = np.cos(rpy[..., 2]), np.sin(rpy[..., 2])
    o, z = np.ones_like(cr), np.zeros_like(cr)
    Rx = np.stack([o, z, z, z, cr, -sr, z, sr, cr], -1).reshape(rpy.shape[:-1] + (3, 3))
    Ry = np.stack([cp, z, sp, z, o, z, -sp, z, cp], -1).reshape(rpy.shape[:-1] + (3, 3))
    Rz = np.stack([cy, -sy, z, sy, cy, z, z, z, o], -1).reshape(rpy.shape[:-1] + (3, 3))
    return np.matmul(np.matmul(Rz, Ry), Rx)


def se3(xyzrpy):
    """build_se3_transform for xyzrpy [..., 6] -> [..., 4, 4] (rotation euler_to_so3, translation xyz)."""
    v = np.asarray(xyzrpy, dtype=np.float64)
    out = np.zeros(v.shape[:-1] + (4, 4))
    out[..., :3, :3] = euler_to_so3(v[..., 3:6])
    out[..., :3, 3] = v[..., 0:3]
    out[..., 3, 3] = 1.0
    return out


def so3_to_quaternion(R):
    """The SDK's so3_to_quaternion for R [..., 3, 3] -> [..., 4] (w, x, y, z): w = sqrt(trace + 1) / 2 (0 when
    trace + 1 < 0), x, y, z = sqrt(max(1 +- diagonal terms, 0)) / 2, and the largest of (w, x, y, z) (the first on a
    tie) selects the branch that recomputes the other three from off-diagonal sums over 4 times it."""
    R = np.asarray(R, dtype=np.float64)
    xx, xy, xz = R[..., 0, 0], R[..., 0, 1], R[..., 0, 2]
    yx, yy, yz = R[..., 1, 0], R[..., 1, 1], R[..., 1, 2]
    zx, zy, zz = R[..., 2, 0], R[..., 2, 1], R[..., 2, 2]
    tr1 = ((xx + yy) + zz) + 1
    w = np.where(tr1 < 0, 0.0, np.sqrt(np.maximum(tr1, 0.0)) / 2)
    x = np.sqrt(np.maximum(1 + xx - yy - zz, 0.0)) / 2
    y = np.sqrt(np.maximum(1 + yy - xx - zz, 0.0)) / 2
    z = np.sqrt(np.maximum(1 + zz - yy - xx, 0.0)) / 2
    k = np.argmax(np.stack([w, x, y, z], -1), -1)
    with np.errstate(divide="ignore", invalid="ignore"):
        branches = [
            np.stack([w, (zy - yz) / (4 * w), (xz - zx) / (4 * w), (yx - xy) / (4 * w)], -1),
            np.stack([(zy - yz) / (4 * x), x, (xy + yx) / (4 * x), (zx + xz) / (4 * x)], -1),
            np.stack([(xz - zx) / (4 * y), (xy + yx) / (4 * y), y, (yz + zy) / (4 * y)], -1),
            np.stack([(yx - xy) / (4 * z), (zx + xz) / (4 * z), (yz + zy) / (4 * z), z], -1),
        ]
    out = branches[0]
    for b in (1, 2, 3):
        out = np.where((k == b)[..., None], branches[b], out)
    return out


def chain_vo(xyzrpy):
    """The VO chain over a whole traversal: abs_0 = I, abs_k = abs_{k-1} se3(row k).  Returns [n, 4, 4]."""
    rel = se3(xyzrpy)
    out = np.empty_like(rel)
    out[0] = np.identity(4)
    for k in range(1, len(rel)):
        out[k] = np.dot(out[k - 1], rel[k])
    return out


def interpolate_absolute(pose_ts, abs_poses, req_ts):
    """interpolate_poses without the origin removal: for each requested timestamp, the upper bracket bisect(pose_ts,
    t) clamped to the last pose, the lower one below it, the fraction (t - t_lo) / (t_hi - t_lo) (true division), slerp
    between the quaternions (a linear blend when d >= 1, scale1 negated when d < 0), positions blended linearly and
    the SDK's quaternion-to-matrix formula.  Returns [n, 4, 4]; no span check (plan_traversal checks spans)."""
    pose_ts = np.asarray(pose_ts, dtype=np.int64)
    req = np.asarray(req_ts, dtype=np.int64).reshape(-1)
    P = np.asarray(abs_poses, dtype=np.float64)
    q = so3_to_quaternion(P[:, :3, :3]).T                      # [4, n]
    pos = P[:, :3, 3].T                                          # [3, n]
    upper = np.searchsorted(pose_ts, req, side="right")
    lower = upper - 1
    upper = np.minimum(upper, len(pose_ts) - 1)
    with np.errstate(divide="ignore", invalid="ignore"):
        frac = (req - pose_ts[lower]) / (pose_ts[upper] - pose_ts[lower])
        ql, qu = q[:, lower], q[:, upper]
        d = (ql * qu).sum(0)
        s0 = np.zeros(d.shape)
        s1 = np.zeros(d.shape)
        lin = d >= 1
        s0[lin] = 1 - frac[lin]
        s1[lin] = frac[lin]
        sl = d < 1
        theta = np.arccos(np.abs(d[sl]))
        s0[sl] = np.sin((1 - frac[sl]) * theta) / np.sin(theta)
        s1[sl] = np.sin(frac[sl] * theta) / np.sin(theta)
    s1[d < 0] = -s1[d < 0]
    qi = np.tile(s0, (4, 1)) * ql + np.tile(s1, (4, 1)) * qu
    pi = np.multiply(np.tile(1 - frac, (3, 1)), pos[:, lower]) + np.multiply(np.tile(frac, (3, 1)), pos[:, upper])
    w, x, y, z = qi
    out = np.zeros((req.size, 4, 4))
    out[:, 0, 0] = 1 - 2 * np.square(y) - 2 * np.square(z)
    out[:, 0, 1] = 2 * np.multiply(x, y) - 2 * np.multiply(z, w)
    out[:, 0, 2] = 2 * np.multiply(x, z) + 2 * np.multiply(y, w)
    out[:, 1, 0] = 2 * np.multiply(x, y) + 2 * np.multiply(z, w)
    out[:, 1, 1] = 1 - 2 * np.square(x) - 2 * np.square(z)
    out[:, 1, 2] = 2 * np.multiply(y, z) - 2 * np.multiply(x, w)
    out[:, 2, 0] = 2 * np.multiply(x, z) - 2 * np.multiply(y, w)
    out[:, 2, 1] = 2 * np.multiply(y, z) + 2 * np.multiply(x, w)
    out[:, 2, 2] = 1 - 2 * np.square(x) - 2 * np.square(y)
    out[:, 0:3, 3] = pi.T
    out[:, 3, 3] = 1
    return out


def relative_to(origin, poses):
    """The SDK's origin removal: np.linalg.solve(origin, [P_0 P_1 ...]) on the [4, 4n] block.  Returns [n, 4, 4]."""
    poses = np.asarray(poses, dtype=np.float64)
    n = poses.shape[0]
    block = np.linalg.solve(origin, poses.transpose(1, 0, 2).reshape(4, 4 * n))
    return block.reshape(4, n, 4).transpose(1, 0, 2).copy()


def interpolate_poses(pose_ts, abs_poses, req_ts, origin_ts):
    """The SDK's interpolate_poses: the requested poses relative to the origin timestamp's.  Returns [n, 4, 4]."""
    A = interpolate_absolute(pose_ts, abs_poses, [origin_ts] + list(req_ts))
    return relative_to(A[0], A[1:])


def gj_inverse(a):
    """The device's 4x4 inverse (csrc/oxford_build.cu gj_inverse): Gauss-Jordan on [a | I] with partial pivoting
    (the first largest |pivot|), every row's eight entries updated in ascending row order.  Python floats, so the
    result is the kernel's bit for bit.  Returns [4, 4] float64."""
    aug = [[float(a[r][j]) for j in range(4)] + [1.0 if j == r else 0.0 for j in range(4)] for r in range(4)]
    for c in range(4):
        p, best = c, abs(aug[c][c])
        for r in range(c + 1, 4):
            if abs(aug[r][c]) > best:
                p, best = r, abs(aug[r][c])
        if p != c:
            aug[c], aug[p] = aug[p], aug[c]
        piv = aug[c][c]
        aug[c] = [v / piv for v in aug[c]]
        for r in range(4):
            if r != c:
                f = aug[r][c]
                aug[r] = [aug[r][j] - f * aug[c][j] for j in range(8)]
    return np.array([row[4:] for row in aug])


# ---------------------------------------------------------------- readers
def _need(path, what):
    if not os.path.isfile(path):
        raise FileNotFoundError(f"Oxford {what} not found: {path}")
    return path


def read_vo(path):
    """vo.csv: a header line, then (source ts, destination ts, x, y, z, roll, pitch, yaw) rows.  Returns (source
    timestamps int64 [n], xyzrpy [n, 6]).  Raises ValueError naming the row when a row is malformed or the source
    timestamps are not strictly ascending (the SDK's check)."""
    ts, v = [], []
    with open(_need(path, "VO file")) as f:
        next(f, None)
        for line_no, row in enumerate(csv.reader(f), start=2):
            try:
                ts.append(int(row[0]))
                v.append([float(x) for x in row[2:8]])
                if len(v[-1]) != 6:
                    raise ValueError("fewer than 8 fields")
            except (ValueError, IndexError) as e:
                raise ValueError(f"{path} line {line_no}: not a VO row ({e})") from None
            if len(ts) > 1 and ts[-1] <= ts[-2]:
                raise ValueError(f"{path} line {line_no}: VO timestamps must be strictly ascending "
                                 f"({ts[-1]} after {ts[-2]})")
    if not ts:
        raise ValueError(f"{path} has no VO row")
    return np.asarray(ts, dtype=np.int64), np.asarray(v, dtype=np.float64)


def read_timestamps(path, what="timestamps"):
    """A .timestamps file: the first space-separated field of each line, an integer."""
    out = []
    with open(_need(path, what)) as f:
        for line_no, line in enumerate(f, start=1):
            try:
                out.append(int(line.split(" ")[0]))
            except ValueError:
                raise ValueError(f"{path} line {line_no}: no integer timestamp") from None
    return out


def camera_timestamps_path(raw, t):
    """stereo.timestamps next to the stereo folder, else in the traversal folder (build_dataset.py:202-204)."""
    p = os.path.join(raw, t, "stereo", CAMERA + ".timestamps")
    return p if os.path.isfile(p) else os.path.join(raw, t, CAMERA + ".timestamps")


def read_extrinsics(path):
    """An SDK extrinsics file: one line x y z roll pitch yaw.  Returns [6] float64."""
    with open(_need(path, "extrinsics file")) as f:
        try:
            v = [float(x) for x in next(f).split(" ")]
        except (StopIteration, ValueError):
            raise ValueError(f"{path}: the first line must be x y z roll pitch yaw") from None
    if len(v) != 6:
        raise ValueError(f"{path}: the first line must hold 6 numbers (got {len(v)})")
    return np.asarray(v)


def read_camera_model(path):
    """The stereo-centre camera model file: fx fy cx cy, then the rows of G_camera_image.  fx, fy, cx and cy must be
    the loader's K_CENTRE (in float32).  Returns G_camera_image [4, 4]."""
    with open(_need(path, "camera model")) as f:
        lines = [ln for ln in f.read().splitlines() if ln.strip()]
    try:
        vals = [float(x) for x in lines[0].split()]
        G = np.asarray([[float(x) for x in ln.split()] for ln in lines[1:]], dtype=np.float64)
    except (IndexError, ValueError):
        raise ValueError(f"{path}: not a camera model (fx fy cx cy, then 4 rows of G_camera_image)") from None
    if len(vals) != 4 or G.shape != (4, 4):
        raise ValueError(f"{path}: not a camera model (fx fy cx cy, then 4 rows of G_camera_image)")
    K = oxford.K_CENTRE
    if [np.float32(v) for v in vals] != [K[0, 0], K[1, 1], K[0, 2], K[1, 2]]:
        raise ValueError(f"{path}: intrinsics {vals} are not the Oxford loader's K_CENTRE "
                         f"({K[0, 0]}, {K[1, 1]}, {K[0, 2]}, {K[1, 2]})")
    return G


def read_tags(path):
    """read_tags_csv: every field of every row."""
    with open(_need(path, "tags.csv")) as f:
        return [x for row in csv.reader(f) for x in row]


def read_scan(path):
    """An LMS scan: float64 (x, y, reflectance) triples.  Returns [3, n]."""
    a = np.fromfile(path, np.double)
    if a.size % 3:
        raise ValueError(f"{path}: {a.size} float64 values, not (x, y, reflectance) triples")
    a = a.reshape(-1, 3).T
    if not np.isfinite(a).all():
        raise ValueError(f"{path} holds a non-finite value")
    return a


# ---------------------------------------------------------------- the host plan
def _params(params):
    unknown = set(params) - set(PARAMS)
    if unknown:
        raise TypeError(f"unknown build parameters {sorted(unknown)}")
    p = dict(PARAMS, **params)
    for k in ("pc_sample_distance", "accumulation_distance", "voxel_grid_downsample_size"):
        if not (np.isfinite(p[k]) and p[k] > 0):
            raise ValueError(f"{k} must be positive (got {p[k]})")
    return p


def output_folder(remove_ground_threshold):
    """lms_front_foreground when a threshold is given (-1 included, which masks nothing), else lms_front."""
    return "lms_front_foreground" if remove_ground_threshold is not None else "lms_front"


def plan_traversal(raw, lms, out, t, sdk_dir, **params):
    """The host half of save_pc_img_for_traversal for one traversal.  Returns a dict: the parameters, lidar_dir,
    G_laser / O (the output transform inv(G_camera_image) G_camera_posesource), the trimmed camera list, the
    centres (timestamp, LMS window [lo, hi), velocity) of the clouds to build, skipped_velocity, the pc and camera
    tables, lms_ts (the traversal's LMS timestamps) and the absolute LMS poses and centre inverses for the device.

    Trimmed camera frames outside the VO span [first, last) are dropped (cameras_outside_vo counts them): a RobotCar
    download's VO rows are sourced at stereo frames, so its last frame is the last VO timestamp, where the
    interpolation has no upper bracket.  The reference gives such frames NaN poses, never keeps them as centres and
    lists them with NaN poses in the camera table.  Every window then lies between two kept frames, inside the span."""
    p = _params(params)
    G_ci = read_camera_model(os.path.join(sdk_dir, "models", CAMERA_MODEL))
    G_cam = se3(read_extrinsics(os.path.join(sdk_dir, "extrinsics", CAMERA + ".txt")))
    G_laser = se3(read_extrinsics(os.path.join(sdk_dir, "extrinsics", "lms_front.txt")))
    O = np.dot(np.linalg.inv(G_ci), G_cam)
    cams = read_timestamps(camera_timestamps_path(raw, t), "camera timestamps")
    if not cams:
        raise ValueError(f"traversal {t} has no camera timestamp")
    init = 0
    for i, c in enumerate(cams):
        if c - cams[0] > p["ignore_first_n_second"] * 1e6:
            init = i
            break
    cams = cams[init:]
    lidar_dir = os.path.join(lms, t, "lms_front")
    lms_ts = read_timestamps(os.path.join(lms, t, "lms_front.timestamps"), "LMS timestamps")
    vo_ts, vo_rows = read_vo(os.path.join(raw, t, "vo", "vo.csv"))
    vo_abs = chain_vo(vo_rows)

    in_span = [c for c in cams if vo_ts[0] <= c < vo_ts[-1]]
    outside = len(cams) - len(in_span)
    cams = in_span
    if not cams:
        raise ValueError(f"traversal {t}: no camera frame lies inside the VO span [{int(vo_ts[0])}, {int(vo_ts[-1])})")
    A_cam = interpolate_absolute(vo_ts, vo_abs, cams)
    kept = [0]                                       # the centre walk (build_dataset.py:249-263)
    idx = 1
    while idx < len(cams):
        hi = min(len(cams), idx + 4096)
        tr = relative_to(A_cam[kept[-1]], A_cam[idx:hi])[:, 0:3, 3]
        far = np.nonzero(np.linalg.norm(tr, axis=1) >= p["pc_sample_distance"])[0]
        if far.size:
            kept.append(idx + int(far[0]))
            idx = kept[-1] + 1
        else:
            idx = hi
    margin = math.ceil(0.5 * p["accumulation_distance"] / p["pc_sample_distance"])
    centres, skipped_velocity = [], []
    for i in range(margin, len(kept) - margin):
        back, centre, front = cams[kept[i - margin]], cams[kept[i]], cams[kept[i + margin]]
        lo = bisect.bisect_left(lms_ts, back)
        hi = bisect.bisect_right(lms_ts, front)
        if hi == lo:
            raise ValueError(f"traversal {t} centre {centre}: no LMS timestamp in [{back}, {front}]")
        velocity = p["accumulation_distance"] / ((hi - lo) / LMS_HZ)
        if velocity < p["min_vehicle_velocity"]:
            skipped_velocity.append(centre)
            continue
        centres.append((centre, lo, hi, velocity))
    pc_ts = [c[0] for c in centres]
    pc_poses = interpolate_poses(vo_ts, vo_abs, pc_ts, cams[0]) if pc_ts else np.zeros((0, 4, 4))
    valid = [c for c in cams if os.path.isfile(os.path.join(out, t, "stereo", "centre", "%d.jpg" % c))
             or os.path.isfile(os.path.join(raw, t, "stereo", "centre", "%d.png" % c))]
    if not valid:
        raise ValueError(f"traversal {t}: no camera frame has an image")
    cam_poses = interpolate_poses(vo_ts, vo_abs, valid, valid[0])
    lo = min((c[1] for c in centres), default=0)
    hi = max((c[2] for c in centres), default=0)
    lms_abs = interpolate_absolute(vo_ts, vo_abs, lms_ts[lo:hi]) if hi > lo else np.zeros((0, 4, 4))
    centre_abs = interpolate_absolute(vo_ts, vo_abs, pc_ts) if pc_ts else np.zeros((0, 4, 4))
    return dict(traversal=t, params=p, lidar_dir=lidar_dir, G_laser=G_laser, O=O, cameras=cams,
                cameras_outside_vo=outside, centres=centres,
                skipped_velocity=skipped_velocity, pc_timestamps=np.asarray(pc_ts, dtype=np.int64),
                pc_poses=pc_poses, camera_timestamps=np.asarray(valid, dtype=np.int64), camera_poses=cam_poses,
                lms_ts=lms_ts, lms_lo=lo, lms_hi=hi, lms_abs=lms_abs,
                centre_inv=np.stack([gj_inverse(A) for A in centre_abs]) if pc_ts else np.zeros((0, 4, 4)))


# ---------------------------------------------------------------- the device store
class RawScanStore:
    """The LMS scans of plan['lms_ts'][lms_lo:lms_hi] as fp64 (x, y, reflectance) planes on the device, read from
    disk once through a pinned staging buffer: xyr [3, total] f64, offsets [n + 1] int64 (scan i = [offsets[i],
    offsets[i+1])), present [n] uint8 (0: no file, an empty range), poses [n, 16] f64 (absolute LMS poses) and the
    host copies of present and the counts."""

    def __init__(self, plan, device="cuda"):
        _require_cuda()
        ts = plan["lms_ts"][plan["lms_lo"]:plan["lms_hi"]]
        paths = [os.path.join(plan["lidar_dir"], "%d.bin" % x) for x in ts]
        present = np.array([os.path.isfile(q) for q in paths], dtype=np.uint8)
        sizes = np.array([os.path.getsize(q) if ok else 0 for q, ok in zip(paths, present)], dtype=np.int64)
        bad = np.nonzero(sizes % 24)[0]
        if bad.size:
            raise ValueError(f"{paths[bad[0]]}: {sizes[bad[0]]} bytes, not (x, y, reflectance) float64 triples")
        counts = sizes // 24
        offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
        total = int(offsets[-1])
        stage = torch.empty((3, max(total, 1)), dtype=torch.float64, pin_memory=True)
        host = stage.numpy()
        for k in np.nonzero(present)[0]:
            host[:, offsets[k]:offsets[k + 1]] = read_scan(paths[k])
        dev = torch.device(device)
        self.device = dev
        self.xyr = stage.to(dev, non_blocking=True)
        self.offsets = torch.from_numpy(offsets).to(dev)
        self.present = torch.from_numpy(present).to(dev)
        self.poses = torch.from_numpy(np.ascontiguousarray(plan["lms_abs"].reshape(-1, 16))).to(dev)
        torch.cuda.current_stream(dev).synchronize()
        self.present_host = present
        self.counts_host = counts
        self.lo = plan["lms_lo"]
        self.n_points = total
        self.nbytes = self.xyr.numel() * 8 + self.offsets.numel() * 8 + self.present.numel() + self.poses.numel() * 8


# ---------------------------------------------------------------- the device stages
def plan_clouds(store, plan, clouds, stream=None):
    """Stage (a) for plan['centres'][c] for c in clouds: the skip walk and the transforms.  Returns a dict of device
    tensors (windows, kept_scan, kept_T, n_kept, n_skipped) and w_stride."""
    lib = _native.load()
    cen = [plan["centres"][c] for c in clouds]
    win = np.array([[lo - store.lo, hi - store.lo] for _, lo, hi, _ in cen], dtype=np.int64).reshape(-1, 2)
    for (ts, lo, hi, _), (a, b) in zip(cen, win):
        if a < 0 or b > len(store.present_host):
            raise ValueError(f"centre {ts}: its window lies outside the store")
        if not store.present_host[a:b].any():
            raise FileNotFoundError(f"no scan file of centre {ts}'s window in {plan['lidar_dir']}")
    S = len(clouds)
    W = int(max(1, (win[:, 1] - win[:, 0]).max(initial=1)))
    dev = store.device
    G = np.ascontiguousarray(plan["G_laser"], dtype=np.float64).reshape(16)
    with torch.cuda.device(dev), torch.cuda.stream(stream):
        r = dict(windows=torch.from_numpy(win).to(dev),
                 centre_inv=torch.from_numpy(np.ascontiguousarray(plan["centre_inv"][list(clouds)].reshape(S, 16))).to(dev),
                 kept_scan=torch.zeros((S, W), dtype=torch.int32, device=dev),
                 kept_T=torch.zeros((S, W, 12), dtype=torch.float64, device=dev),
                 n_kept=torch.zeros((S,), dtype=torch.int32, device=dev),
                 n_skipped=torch.zeros((S,), dtype=torch.int32, device=dev), w_stride=W)
        rc = lib.oxford_build_plan_f64(_ptr(store.poses), _ptr(store.present), len(store.present_host),
                                       _ptr(r["windows"]), _ptr(r["centre_inv"]), S,
                                       G.ctypes.data_as(_native._c.c_void_p),
                                       plan["params"]["voxel_grid_downsample_size"] / 16.0, W, _ptr(r["kept_scan"]),
                                       _ptr(r["kept_T"]), _ptr(r["n_kept"]), _ptr(r["n_skipped"]), _stream_ptr(stream))
    _native.check(rc, "oxford_build_plan")
    return r


def _mask(plan):
    thr = plan["params"]["remove_ground_threshold"]
    return (1, float(thr)) if thr is not None and thr > -1 else (0, 0.0)


def gather_clouds(store, plan, clouds, planned, stream=None):
    """Stage (b): the masked points of the kept scans, transformed, in scan then point order.  Reads the point counts
    back to size the batch.  Returns dict(xyz [S,3,N] f64, attr [S,1,N] f64 (reflectance / max), n_pts [S] int32,
    rmax [S] f64) on the device."""
    lib = _native.load()
    use_mask, thr = _mask(plan)
    S, W = len(clouds), planned["w_stride"]
    dev = store.device
    x, y, rr = store.xyr[0], store.xyr[1], store.xyr[2]
    sp = _stream_ptr(stream)
    with torch.cuda.device(dev), torch.cuda.stream(stream):
        pos = torch.zeros((S, W), dtype=torch.int32, device=dev)
        n_pts = torch.zeros((S,), dtype=torch.int32, device=dev)
        rmax = torch.zeros((S,), dtype=torch.float64, device=dev)
        ws = torch.empty((max(lib.oxford_build_count_workspace_bytes(S, W), 1),), dtype=torch.uint8, device=dev)
        rc = lib.oxford_build_count_f64(_ptr(x), _ptr(rr), _ptr(store.offsets), _ptr(planned["kept_scan"]),
                                        _ptr(planned["n_kept"]), S, W, use_mask, thr, _ptr(pos), _ptr(n_pts),
                                        _ptr(rmax), _ptr(ws), ws.numel(), sp)
        _native.check(rc, "oxford_build_count")
        n_host = n_pts.cpu().numpy()
        for c, n in zip(clouds, n_host):
            if n == 0:
                raise ValueError(f"centre {plan['centres'][c][0]}: no point of the scans in {plan['lidar_dir']} "
                                 "is left after the ground mask")
        N = round_up(int(n_host.max(initial=1)), 16)
        if S * 3 * N >= 2**31:
            raise ValueError(f"a batch of {S} clouds of up to {int(n_host.max())} points is too large; use a smaller "
                             "batch")
        xyz = torch.zeros((S, 3, N), dtype=torch.float64, device=dev)
        attr = torch.zeros((S, 1, N), dtype=torch.float64, device=dev)
        rc = lib.oxford_build_scatter_f64(_ptr(x), _ptr(y), _ptr(rr), _ptr(store.offsets), _ptr(planned["kept_scan"]),
                                          _ptr(planned["kept_T"]), _ptr(planned["n_kept"]), _ptr(pos), _ptr(rmax), S,
                                          W, use_mask, thr, N, _ptr(xyz), _ptr(attr), sp)
    _native.check(rc, "oxford_build_scatter")
    return dict(xyz=xyz, attr=attr, n_pts=n_pts, rmax=rmax, n_host=n_host)


def pack_clouds(plan, gathered, down, stream=None):
    """Stage (d): the output transform and float32 rounding.  Returns (records [S,4,M_max] f32, m_pts [S] int32)."""
    lib = _native.load()
    xyz, attr, m = down["xyz"], down["attr"], down["m_pts"]
    S, _, N = xyz.shape
    O = np.ascontiguousarray(plan["O"], dtype=np.float64).reshape(16)
    with torch.cuda.device(xyz.device), torch.cuda.stream(stream):
        M = max(int(m.max()), 1)                 # read on `stream`, after the voxel step that writes m_pts
        out = torch.empty((S, 4, M), dtype=torch.float32, device=xyz.device)
        rc = lib.oxford_build_pack_f32(_ptr(xyz), _ptr(attr), _ptr(m), _ptr(gathered["rmax"]),
                                       O.ctypes.data_as(_native._c.c_void_p), S, N, M, _ptr(out), _stream_ptr(stream))
    _native.check(rc, "oxford_build_pack")
    return out, m


def build_clouds(store, plan, clouds, stream=None):
    """my_build_pointcloud + downsample + the output transform for the clouds plan['centres'][c], c in clouds, in one
    batch.  Returns dict(records [S,4,M_max] float32 and m_pts [S] int32 on the device, written on `stream`; n_kept,
    n_skipped, n_pts [S] as numpy).  Every step, read-back and check runs on `stream` (the current stream when None),
    whichever stream is current for the caller.  Raises FileNotFoundError when a window has no scan file and ValueError
    when no point survives the mask."""
    clouds = list(clouds)
    if not clouds:
        raise ValueError("clouds is empty")
    with torch.cuda.device(store.device), torch.cuda.stream(stream):
        planned = plan_clouds(store, plan, clouds, stream)
        gathered = gather_clouds(store, plan, clouds, planned, stream)
        down = pointprep.voxel_downsample(gathered["xyz"], gathered["n_pts"],
                                          plan["params"]["voxel_grid_downsample_size"], attr=gathered["attr"],
                                          stream=stream)
        rec, m = pack_clouds(plan, gathered, down, stream)
        return dict(records=rec, m_pts=m, n_kept=planned["n_kept"].cpu().numpy(),
                    n_skipped=planned["n_skipped"].cpu().numpy(), n_pts=gathered["n_host"])


# ---------------------------------------------------------------- whole traversals
def is_night(raw, t):
    return "night" in read_tags(os.path.join(raw, t, "tags.csv"))


def build_traversal(raw, lms, out, t, sdk_dir, batch=64, device="cuda", stream=None, images=False, **params):
    """save_pc_img_for_traversal for traversal t, writing <out>/<t>/lms_front[_foreground]/<ts>.npy, pc_timestamps.npy,
    pc_poses.npy, camera_timestamps.npy, camera_poses.npy and, as the last step, a copy of tags.csv.  Every built
    cloud is listed, whether or not its record existed before.  With images=True the stereo-centre frames are
    converted too (build_dataset.py:356-377, oxford_images.convert_frames with the SDK's
    models/stereo_narrow_left_distortion_lut.bin): every frame of the camera table whose PNG exists and whose
    <out>/<t>/stereo/centre/<ts>.jpg does not yet exist, before tags.csv is written.  The device work and its
    read-backs run on `stream` (the current stream when None).  Returns a summary dict: clouds_built,
    clouds_skipped_velocity, scans_skipped (summed over the clouds), scans_missing (distinct LMS timestamps without a
    scan file in the built clouds' windows), cameras_outside_vo, camera_frames, per cloud n_kept / n_skipped / m_pts,
    and with images=True images_converted and images_skipped (frames whose JPEG already existed)."""
    if int(batch) < 1:
        raise ValueError(f"batch must be positive (got {batch})")
    plan = plan_traversal(raw, lms, out, t, sdk_dir, **params)
    folder = os.path.join(out, t, output_folder(plan["params"]["remove_ground_threshold"]))
    os.makedirs(folder, exist_ok=True)
    os.makedirs(os.path.join(out, t, "stereo", "centre"), exist_ok=True)
    n = len(plan["centres"])
    n_kept, n_skipped, m_pts = np.zeros(n, np.int64), np.zeros(n, np.int64), np.zeros(n, np.int64)
    missing = 0
    if n:
        store = RawScanStore(plan, device)
        for c0 in range(0, n, int(batch)):
            ids = list(range(c0, min(n, c0 + int(batch))))
            res = build_clouds(store, plan, ids, stream)
            with torch.cuda.device(store.device), torch.cuda.stream(stream):
                rec = res["records"].cpu().numpy()
                m = res["m_pts"].cpu().numpy()
            for k, c in enumerate(ids):
                np.save(os.path.join(folder, "%d.npy" % plan["centres"][c][0]), rec[k, :, :m[k]])
            n_kept[ids], n_skipped[ids], m_pts[ids] = res["n_kept"], res["n_skipped"], m
        covered = np.zeros(len(store.present_host), dtype=bool)      # windows overlap: count each scan once
        for _, lo, hi, _ in plan["centres"]:
            covered[lo - store.lo:hi - store.lo] = True
        missing = int((covered & (store.present_host == 0)).sum())
    d = os.path.join(out, t)
    np.save(os.path.join(d, "pc_timestamps.npy"), plan["pc_timestamps"])
    np.save(os.path.join(d, "pc_poses.npy"), np.asarray(plan["pc_poses"], dtype=np.float64))
    np.save(os.path.join(d, "camera_timestamps.npy"), plan["camera_timestamps"])
    np.save(os.path.join(d, "camera_poses.npy"), np.asarray(plan["camera_poses"], dtype=np.float64))
    summary = dict(traversal=t, clouds_built=n, clouds_skipped_velocity=len(plan["skipped_velocity"]),
                   scans_skipped=int(n_skipped.sum()), scans_missing=missing,
                   cameras_outside_vo=plan["cameras_outside_vo"], camera_frames=len(plan["camera_timestamps"]),
                   n_kept=n_kept, n_skipped=n_skipped, m_pts=m_pts)
    if images:
        summary.update(convert_images(raw, out, t, sdk_dir, plan["camera_timestamps"], batch, device, stream))
    shutil.copy(os.path.join(raw, t, "tags.csv"), os.path.join(d, "tags.csv"))
    return summary


def convert_images(raw, out, t, sdk_dir, cameras, batch=64, device="cuda", stream=None):
    """build_dataset.py:356-377 for the frames `cameras` of traversal t: each <raw>/<t>/stereo/centre/<ts>.png without
    a <out>/<t>/stereo/centre/<ts>.jpg is converted (oxford_images.convert_frames).  Returns dict(images_converted,
    images_skipped)."""
    from . import oxford_images
    from .png import parse_png
    src = os.path.join(raw, t, "stereo", "centre")
    dst = os.path.join(out, t, "stereo", "centre")
    todo = [c for c in cameras if not os.path.isfile(os.path.join(dst, "%d.jpg" % c))
            and os.path.isfile(os.path.join(src, "%d.png" % c))]
    skipped = len(cameras) - len(todo)
    if todo:
        first = os.path.join(src, "%d.png" % todo[0])
        with open(first, "rb") as f:
            try:
                hd = parse_png(f.read(), grey=True)
            except ValueError as e:
                raise ValueError(f"{first}: {e}") from None
        lut = oxford_images.read_distortion_lut(os.path.join(sdk_dir, "models", oxford_images.LUT_FILE), hd.H, hd.W)
        oxford_images.convert_frames([os.path.join(src, "%d.png" % c) for c in todo],
                                     [os.path.join(dst, "%d.jpg" % c) for c in todo], lut, batch=batch,
                                     device=device, stream=stream)
    return dict(images_converted=len(todo), images_skipped=skipped)


def select_traversals(raw, out, traversals=None):
    """main()'s selection: the raw root's traversal folders (or the given ones), sorted, without night traversals
    ('night' in tags.csv) and without those already done (<out>/<t>/tags.csv exists).  Returns (todo, night, done)."""
    names = sorted(f for f in os.listdir(raw) if os.path.isdir(os.path.join(raw, f))) if traversals is None \
        else list(traversals)
    night = [t for t in names if is_night(raw, t)]
    done = [t for t in names if t not in night and os.path.exists(os.path.join(out, t, "tags.csv"))]
    return [t for t in names if t not in night and t not in done], night, done


def write_train_split(out):
    """train_val_split.txt.py: when <out>/val.txt exists, write train.txt with every traversal folder of out (sorted)
    that is not in val.txt, has a tags.csv and has no line 'night' in it.  Returns the list, or None without val.txt."""
    val_path = os.path.join(out, "val.txt")
    if not os.path.isfile(val_path):
        return None
    with open(val_path) as f:
        val = [x.rstrip() for x in f.readlines()]
    train = []
    for t in sorted(f for f in os.listdir(out) if os.path.isdir(os.path.join(out, f))):
        tags = os.path.join(out, t, "tags.csv")
        if t in val or not os.path.isfile(tags):
            continue
        with open(tags) as f:
            if "night" in [x.rstrip() for x in f.readlines()]:
                continue
        train.append(t)
    with open(os.path.join(out, "train.txt"), "w") as f:
        f.writelines(["%s\n" % t for t in train])
    return train


def build_root(raw, lms, out, sdk_dir, traversals=None, batch=64, log=print, images=False, **params):
    """main(): every selected traversal in turn on one GPU (converting the stereo-centre frames too with
    images=True), then train.txt when val.txt exists.  Returns the traversals' summaries."""
    todo, night, done = select_traversals(raw, out, traversals)
    for t in night:
        log(f"{t} is night driving, skip.")
    for t in done:
        log(f"{t} is already done, skip.")
    out_s = []
    for t in todo:
        s = build_traversal(raw, lms, out, t, sdk_dir, batch=batch, images=images, **params)
        log(f"{t}: {s['clouds_built']} clouds, {s['clouds_skipped_velocity']} skipped for velocity, "
            f"{s['scans_skipped']} scans skipped, {s['scans_missing']} scan files missing, {s['camera_frames']} camera "
            f"frames ({s['cameras_outside_vo']} outside the VO span dropped)"
            + (f", {s['images_converted']} images converted, {s['images_skipped']} already converted or without a PNG"
               if images else ""))
        out_s.append(s)
    write_train_split(out)
    return out_s
