"""nuScenes classifier batches without the devkit: the record lookups, poses and sweep walk of
data/nuscenes_pc_img_pose_loader.py (which needs nuscenes-devkit, pyquaternion and Open3D), restated on the host, and
nuscenes_batch, which hands the sweeps to assemble.assemble_batch(**nuscenes_args) and the JPEG frames to
imageprep.assemble_images(**nuscenes_image_args()).

Tables reads the three devkit tables __getitem__ touches; rotation_matrix restates pyquaternion's; ego_pose_P /
calibration_P / pose_chain build the loader's 4 x 4s with its float32 rounding and its np.dot / np.linalg.inv calls in
its order, so they are the loader's bit for bit on the same numpy.  DESIGN.md 4.20 states the contract.
"""
import json
import os
import pickle

import numpy as np
import torch

from . import assemble, imageprep

CAMERAS = ("CAM_FRONT", "CAM_FRONT_LEFT", "CAM_FRONT_RIGHT", "CAM_BACK", "CAM_BACK_LEFT", "CAM_BACK_RIGHT")
ACCUMULATION_FRAME_NUM = 3      # nuscenes_t/options.py
ACCUMULATION_FRAME_SKIP = 4
TABLES = ("sample_data", "ego_pose", "calibrated_sensor")


class Tables:
    """<dataroot>/<version>/{sample_data, ego_pose, calibrated_sensor}.json, indexed by token.  get(table, token)
    returns the record dict as NuScenes.get does."""

    def __init__(self, dataroot, version):
        self.dataroot = dataroot
        self.version = version
        self._t = {}
        for name in TABLES:
            with open(os.path.join(dataroot, version, name + ".json")) as f:
                recs = json.load(f)
            self._t[name] = {r["token"]: r for r in recs}

    def get(self, table, token):
        if table not in self._t:
            raise ValueError(f"table must be one of {TABLES} (got {table!r})")
        try:
            return self._t[table][token]
        except KeyError:
            raise KeyError(f"no {table} record with token {token!r}") from None


def load_dataset_info(path):
    """The loader's dataset_info.list: a pickled list of (lidar_token, {camera name: [camera sample_data tokens]})."""
    with open(path, "rb") as f:
        return pickle.load(f)


def rotation_matrix(q):
    """pyquaternion's Quaternion(q).rotation_matrix for q = (w, x, y, z): q / |q| unless |1 - q.q| < 1e-14, then the
    lower-right 3 x 3 of Q(q) Qbar(q)^T (the left and right Hamilton-product matrices)."""
    q = np.array(q, dtype=np.float64).reshape(-1)
    if q.shape != (4,) or not np.isfinite(q).all():
        raise ValueError("a quaternion is four finite numbers (w, x, y, z)")
    ss = np.dot(q, q)
    if not abs(1.0 - ss) < 1e-14:
        n = np.sqrt(ss)
        if not n > 0:
            raise ValueError("the zero quaternion has no rotation")
        q = q / n
    a, b, c, d = q
    Q = np.array([[a, -b, -c, -d], [b, a, -d, c], [c, d, a, -b], [d, -c, b, a]])
    Qbar = np.array([[a, -b, -c, -d], [b, a, d, -c], [c, -d, a, b], [d, c, -b, a]])
    return np.dot(Q, Qbar.conj().transpose())[1:][:, 1:]


def P_from_record(rec):
    """get_P_from_Rt of a record's rotation and translation, each rounded to float32, in a float64 identity."""
    P = np.identity(4)
    P[0:3, 0:3] = np.asarray(rotation_matrix(rec["rotation"])).astype(np.float32)
    P[0:3, 3] = np.asarray(rec["translation"]).astype(np.float32)
    return P


def ego_pose_P(tables, sd):
    return P_from_record(tables.get("ego_pose", sd["ego_pose_token"]))


def calibration_P(tables, sd):
    return P_from_record(tables.get("calibrated_sensor", sd["calibrated_sensor_token"]))


def camera_K(tables, sd):
    return np.asarray(tables.get("calibrated_sensor", sd["calibrated_sensor_token"])["camera_intrinsic"]).astype(
        np.float32)


def sweep_walk(tables, lidar_token, frame_num=ACCUMULATION_FRAME_NUM, frame_skip=ACCUMULATION_FRAME_SKIP):
    """The loader's accumulate_lidar_points order: the anchor sweep, then up to frame_num sweeps along `next` at
    offsets frame_skip, 2 frame_skip, ..., then the same along `prev`; a direction stops at its first empty link.
    Returns [(sample_data record, offset)], offset signed (+ next, - prev), anchor 0."""
    if int(frame_num) != frame_num or frame_num < 0 or int(frame_skip) != frame_skip or frame_skip < 1:
        raise ValueError("frame_num must be >= 0 and frame_skip >= 1 (integers)")
    anchor = tables.get("sample_data", lidar_token)
    out = [(anchor, 0)]
    for direction, sign in (("next", 1), ("prev", -1)):
        lidar, counter, taken, off = anchor, 1, 0, 0
        while taken < frame_num:
            if lidar[direction] == "":
                break
            if counter % frame_skip != 0:
                counter += 1
                lidar = tables.get("sample_data", lidar[direction])
                off += 1
                continue
            out.append((tables.get("sample_data", lidar[direction]), sign * (off + 1)))
            counter += 1
            lidar = tables.get("sample_data", lidar[direction])
            off += 1
            taken += 1
    return out


def sweep_transforms(tables, walk):
    """frame_T of each sweep of a walk: the identity for the anchor, and P_ij_trans = (P_lidar_vehicle (P_io P_oj))
    P_vehicle_lidar for sweep j, with the anchor's calibration and np.dot / np.linalg.inv as the loader calls them."""
    anchor = walk[0][0]
    P_io = np.linalg.inv(ego_pose_P(tables, anchor))
    P_vehicle_lidar = calibration_P(tables, anchor)
    P_lidar_vehicle = np.linalg.inv(P_vehicle_lidar)
    Ts = [np.identity(4)]
    for sd, _ in walk[1:]:
        P_ij = np.dot(P_io, ego_pose_P(tables, sd))
        Ts.append(np.dot(np.dot(P_lidar_vehicle, P_ij), P_vehicle_lidar))
    return np.stack(Ts)


def pose_chain(tables, lidar_sd, camera_sd):
    """The loader's P_cam_pc = inv(cam_calib) (inv(cam_pose) (lidar_pose lidar_calib)) and t_ij = P_cam_pc[:3, 3]."""
    lidar_calib = calibration_P(tables, lidar_sd)
    lidar_pose = ego_pose_P(tables, lidar_sd)
    cam_calib = calibration_P(tables, camera_sd)
    cam_pose = ego_pose_P(tables, camera_sd)
    P_cam_pc = np.dot(np.linalg.inv(cam_calib), np.dot(np.linalg.inv(cam_pose), np.dot(lidar_pose, lidar_calib)))
    return P_cam_pc, P_cam_pc[0:3, 3]


def read_sweep(path):
    """LidarPointCloud.from_file's points as the loader uses them: float32 [n, 4] (x, y, z, intensity) from records of
    five float32."""
    return np.fromfile(path, dtype=np.float32).reshape(-1, 5)[:, :4]


def _rng(rng):
    return rng if isinstance(rng, np.random.Generator) else np.random.default_rng(rng)


def nuscenes_batch(tables, items, mode, seed, rng=None, input_pt_num=assemble.INPUT_PT_NUM,
                   node_a_num=assemble.NODE_NUM, node_b_num=assemble.NODE_NUM, device="cuda", stream=None):
    """nuScenesLoader.__getitem__ for S = len(items) dataset_info entries (lidar_token, {camera: [tokens]}).  The
    camera and its nearby token are drawn on the host from rng (a numpy Generator or a seed), which then draws Pr and
    the image crop and jitter; seed keys the device's Philox draws.  Returns (pc [S,3,N], intensity [S,1,N], sn
    [S,3,N] (zeros), node_a [S,3,Ma], node_b [S,3,Mb], P [S,3,4], img [S,3,160,320] float32 on the device; K [S,3,3],
    t_ij [S,3] float32 on the host)."""
    if mode not in assemble.MODES:
        raise ValueError(f"mode must be one of {assemble.MODES} (got {mode!r})")
    items = list(items)
    if not items:
        raise ValueError("items is empty")
    rng = _rng(rng)
    samples, cams = [], []
    for lidar_token, nearby in items:
        walk = sweep_walk(tables, lidar_token)
        FT = sweep_transforms(tables, walk)
        frames = []
        for sd, _ in walk:
            r = read_sweep(os.path.join(tables.dataroot, sd["filename"]))
            frames.append((r[:, :3].T, r[:, 3], None))
        samples.append((frames, FT))
        name = CAMERAS[int(rng.integers(len(CAMERAS)))]
        toks = nearby[name]
        if len(toks) == 0:
            raise ValueError(f"lidar {lidar_token}: no {name} token")
        cams.append(tables.get("sample_data", toks[int(rng.integers(len(toks)))]))
    poses = [pose_chain(tables, tables.get("sample_data", it[0]), cam) for it, cam in zip(items, cams)]
    P_cam_pc = np.stack([p[0] for p in poses])
    t_ij = np.stack([p[1] for p in poses]).astype(np.float32)
    frames = assemble.pack_frames(samples, device)
    out = assemble.assemble_batch(frames, mode, seed, input_pt_num=input_pt_num, node_a_num=node_a_num,
                                  node_b_num=node_b_num, rng=rng, stream=stream,
                                  **assemble.nuscenes_args(P_cam_pc))
    images = imageprep.read_jpeg_batch([os.path.join(tables.dataroot, c["filename"]) for c in cams], device, stream)
    K = np.stack([camera_K(tables, c) for c in cams])
    im = imageprep.assemble_images(images, K, mode, rng=rng, stream=stream, **imageprep.nuscenes_image_args())
    return (out["pc"], out["intensity"], out["sn"], out["node_a"], out["node_b"], out["P"], im["img"], im["K"],
            torch.from_numpy(t_ij))
