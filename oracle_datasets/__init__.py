"""Expected values for deepi2p_b200.kitti and deepi2p_b200.oxford: what the KITTI and Oxford loaders compute on the
host before their point and image sides, worked out here with plain numpy and no code shared with the package.

Only what decides the bits follows the loaders: the float32 roundings (calibration matrices, poses), and each
4 x 4 product or inverse as one np.dot / np.linalg.inv call on operands of the loaders' dtypes, associated as the
loaders associate them.  Draws take a numpy Generator: an integer in [a, b] is rng.integers(a, b + 1), redrawn until
it qualifies, so a caller drawing the same way consumes the same words.  Frames are returned with the 4 x 4 that moves
them into the anchor's frame (the identity for the anchor), which is what assemble.pack_frames takes.

KITTI odometry: calibration(), kitti_list(), neighbours(), frame_transform(), draw_pair(), kitti_expected().
Oxford RobotCar: conjugate(), oxford_tables(), draw_camera(), oxford_expected().
"""
import math
import os
from itertools import takewhile

import numpy as np

F32 = np.float32
KITTI_SKIP = 40                     # frames left out at each end of a sequence
KITTI_STEP, KITTI_REACH = 6, 3      # accumulation: 3 frames 6 apart on each side
PAIR_WINDOW, PAIR_LIMIT = 40, 10.0  # image pairing: |i - j| <= 40, ||t_ji|| < 10 m
OXFORD_INTERVAL = 2                 # metres between Oxford clouds
# Oxford's axis change: new = C old C^-1 with C this permutation, in float32
OXFORD_C = np.zeros((4, 4), F32)
OXFORD_C[[0, 1, 2, 3], [1, 2, 0, 3]] = 1


# ------------------------------------------------------------------------------------------------------------------
# KITTI


def _kitti_seq_dir(root, kind, seq):
    return os.path.join(root, kind, "sequences", "%02d" % seq)


def camera_translation(m):
    """The camera offset (tx, ty, tz) of a float32 3 x 4 projection m = K [I | t]: tz = m23 and (tx, ty) = (m[:2, 3] -
    (cx, cy) tz) / (fx, fy), every step in float32.  Returned as float64."""
    tz = m[2, 3]
    focal = np.array([m[0, 0], m[1, 1]], dtype=F32)
    centre = np.array([m[0, 2], m[1, 2]], dtype=F32)
    txy = (m[:2, 3] - centre * tz) / focal
    return np.array([txy[0], txy[1], tz], dtype=np.float64)


def calibration(root, seq):
    """{key: matrix} of calib/<seq>/calib.txt.  'Tr' is [m; 0 0 0 1] in float64 from the float32 3 x 4; a projection
    key P gives 'P_K' (its float32 3 x 3) and 'P' (a float64 identity carrying camera_translation)."""
    with open(os.path.join(root, "calib", "%02d" % seq, "calib.txt")) as f:
        rows = [line.split(":", 1) for line in f if line.strip()]
    out = {}
    for key, rest in rows:
        m = np.array(rest.split(), dtype=np.float64).astype(F32).reshape(3, 4)
        if key == "Tr":
            out[key] = np.vstack([m.astype(np.float64), [0.0, 0.0, 0.0, 1.0]])
            continue
        out[key + "_K"] = np.ascontiguousarray(m[:, :3])
        P = np.eye(4)
        P[:3, 3] = camera_translation(m)
        out[key] = P
    return out


def kitti_list(root, seqs):
    """The sample list: (seq, i, n, camera) for i in [40, n - 40), both cameras of a frame next to each other; n
    counts the sequence's image_2 files."""
    out = []
    for seq in seqs:
        n = len(os.listdir(os.path.join(_kitti_seq_dir(root, "data_odometry_color_npy", seq), "image_2")))
        out += [(seq, i, n, cam) for i in range(KITTI_SKIP, n - KITTI_SKIP) for cam in ("P2", "P3")]
    return out


def neighbours(i, n):
    """The accumulated frames besides the anchor: backwards first, then forwards, each side cut at the first frame
    outside [0, n)."""
    steps = [KITTI_STEP * k for k in range(1, KITTI_REACH + 1)]
    back = takewhile(lambda j: j >= 0, (i - s for s in steps))
    ahead = takewhile(lambda j: j < n, (i + s for s in steps))
    return list(back) + list(ahead)


def kitti_pose(root, seq, frame):
    with np.load(os.path.join(root, "poses", "%02d" % seq, "%06d.npz" % frame)) as z:
        return z["pose"].astype(F32)


def frame_transform(Pc, P_anchor, P_frame):
    """The 4 x 4 moving a frame's velodyne points into the anchor's: inv(Pc) ((inv(P_anchor) P_frame) Pc), with the
    poses float32 and Pc float64."""
    relative = np.dot(np.linalg.inv(P_anchor), P_frame)
    return np.dot(np.linalg.inv(Pc), np.dot(relative, Pc))


def draw_pair(rng, pose, i, n, window=PAIR_WINDOW, limit=PAIR_LIMIT):
    """The image frame j of anchor i: j drawn from [i - window, i + window] clipped to the sequence until
    rel = inv(P_j) P_i (float32) has ||rel[:3, 3]|| < limit.  limit < 0: j = i and the float64 identity, no draw.
    pose(k) gives frame k's float32 pose.  Returns (j, rel)."""
    if limit < 0:
        return i, np.eye(4)
    lo, hi = max(0, i - window), min(n - 1, i + window)
    P_i = pose(i)
    while True:
        j = int(rng.integers(lo, hi + 1))
        rel = np.dot(np.linalg.inv(pose(j)), P_i)
        if np.linalg.norm(rel[:3, 3]) < limit:
            return j, rel


def kitti_expected(root, entry, rng, limit=PAIR_LIMIT):
    """Everything a kitti_list entry's batch sample needs before the device: dict(frames [(xyz, intensity, sn)],
    frame_T [T,4,4], walk, Pc, Pji, t_ji, j, K, img), drawing j from rng."""
    seq, i, n, cam = entry
    cal = calibration(root, seq)
    Pc = np.dot(cal[cam], cal["Tr"])
    walk = [i] + neighbours(i, n)
    P_anchor = kitti_pose(root, seq, i)
    frame_T = np.stack([np.eye(4)] + [frame_transform(Pc, P_anchor, kitti_pose(root, seq, k)) for k in walk[1:]])
    rec_dir = os.path.join(_kitti_seq_dir(root, "data_odometry_velodyne_NWU", seq), "voxel0.1-SNr0.6")
    recs = [np.load(os.path.join(rec_dir, "%06d.npy" % k)).astype(F32) for k in walk]
    j, Pji = draw_pair(rng, lambda k: kitti_pose(root, seq, k), i, n, limit=limit)
    img = np.load(os.path.join(_kitti_seq_dir(root, "data_odometry_color_npy", seq), "image_" + cam[1],
                               "%06d.npy" % j))
    return dict(frames=[(r[:3], r[3], r[4:7]) for r in recs], frame_T=frame_T, walk=walk, Pc=Pc, Pji=Pji,
                t_ji=Pji[:3, 3], j=j, K=cal[cam + "_K"], img=img)


# ------------------------------------------------------------------------------------------------------------------
# Oxford


def conjugate(poses):
    """C P inv(C) for each pose of [n,4,4], everything float32."""
    C_inv = np.linalg.inv(OXFORD_C)
    return np.stack([np.dot(OXFORD_C, np.dot(P, C_inv)) for P in np.asarray(poses).astype(F32)]).reshape(-1, 4, 4)


def oxford_tables(root, mode):
    """(entries [(traversal, pc timestamp, i, n)], {traversal: dict(pc_ts, pc_P, cam_ts, cam_P)}) for the split of
    `mode` (train.txt for train, val.txt otherwise); timestamps as int64 arrays, poses conjugated."""
    split = "train.txt" if mode == "train" else "val.txt"
    with open(os.path.join(root, split)) as f:
        names = [s.strip() for s in f.read().splitlines() if s.strip()]
    tables, entries = {}, []
    for t in names:
        d = os.path.join(root, t)
        tab = dict(pc_ts=np.load(os.path.join(d, "pc_timestamps.npy")).astype(np.int64),
                   pc_P=conjugate(np.load(os.path.join(d, "pc_poses.npy"))),
                   cam_ts=np.load(os.path.join(d, "camera_timestamps.npy")).astype(np.int64),
                   cam_P=conjugate(np.load(os.path.join(d, "camera_poses.npy"))))
        tables[t] = tab
        n = len(tab["pc_ts"])
        entries += [(t, int(ts), i, n) for i, ts in enumerate(tab["pc_ts"])]
    return entries, tables


def draw_camera(rng, tab, i, limit=PAIR_LIMIT, interval=OXFORD_INTERVAL):
    """The camera frame of cloud i: clouds within ceil(limit / interval) indices either side bound a timestamp range,
    whose left insertion points into the camera timestamps give [lo, hi]; c is drawn from it until rel = inv(P_cam c)
    P_pc i (float32) has ||rel[:3, 3]|| < limit.  A c past the last camera frame does not qualify.  Returns (c, rel)."""
    k = math.ceil(limit / interval)
    last = len(tab["pc_ts"]) - 1
    lo, hi = np.searchsorted(tab["cam_ts"], tab["pc_ts"][[max(0, i - k), min(last, i + k)]], side="left")
    while True:
        c = int(rng.integers(lo, hi + 1))
        if c >= len(tab["cam_ts"]):
            continue
        rel = np.dot(np.linalg.inv(tab["cam_P"][c]), tab["pc_P"][i])
        if np.linalg.norm(rel[:3, 3]) < limit:
            return c, rel


def oxford_expected(root, tables, entry, rng, limit=PAIR_LIMIT):
    """A batch sample's host side for an oxford_tables entry: dict(frames [(xyz, intensity, None)], frame_T [1,4,4],
    P_cam_pc, t_ij, image_path, cam), drawing the camera from rng."""
    t, ts, i, _ = entry
    tab = tables[t]
    c, rel = draw_camera(rng, tab, i, limit)
    rec = np.load(os.path.join(root, t, "lms_front", "%d.npy" % ts)).astype(F32)
    return dict(frames=[(rec[:3], rec[3], None)], frame_T=np.eye(4)[None], P_cam_pc=rel, t_ij=rel[:3, 3],
                image_path=os.path.join(root, t, "stereo", "centre", "%d.jpg" % int(tab["cam_ts"][c])), cam=c)
