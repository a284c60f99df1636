"""numpy oracle of the KITTI accumulated-frame build -- TEST INFRASTRUCTURE ONLY.

Only tests/, tests/golden/ generators and the benchmark scripts may import this package; deepi2p_b200 never does.  It
restates data/kitti/frame_accumulation.py accumulate_sequence one frame at a time, in the reference's own structure
(poses and records loaded per use, the ego mask and the norm written as the reference writes them), with the project's
documented Open3D contract (DESIGN.md 4.10 / 4.29): the fixed-association fp64 transform of points and normals
(oracle_nuscenes.affine64) and the voxel grid on the fp64 cloud (oracle_nuscenes.voxel_downsample64: ascending
(ix, iy, iz), sums in ascending point index).
"""
import bisect
import os

import numpy as np

from oracle_nuscenes import affine64, voxel_downsample64


def _pose(root, seq, i):
    return np.load(os.path.join(root, "poses", "%02d" % seq, "%06d.npz" % i))["pose"]


def _record(root, seq, folder, i):
    return np.load(os.path.join(root, "data_odometry_velodyne_NWU", "sequences", "%02d" % seq, folder, "%06d.npy" % i))


def plan(root, seq, frame_stride_dist=4, accumulate_radius=50, np_folder="voxel0.1-SNr0.6"):
    """sample_num, the stride list, accumulate_frames and the per-frame windows [left, right] (inclusive positions
    into the stride list), exactly as accumulate_sequence forms them."""
    pc_nwu_folder = os.path.join(root, "data_odometry_velodyne_NWU", "sequences", "%02d" % seq, np_folder)
    sample_num = round(len(os.listdir(pc_nwu_folder)))
    accumulate_frames = int(round(accumulate_radius / frame_stride_dist))
    stride_list = [0]
    P_prev = _pose(root, seq, 0)
    for i in range(1, sample_num):
        P_i = _pose(root, seq, i)
        P_prev_i = np.dot(np.linalg.inv(P_prev), P_i)
        t_prev_i_norm = np.linalg.norm(P_prev_i[0:3, 3])
        if t_prev_i_norm > frame_stride_dist:
            stride_list.append(i)
            P_prev = P_i
    win = []
    for i in range(sample_num):
        nearest = bisect.bisect_left(stride_list, i)
        win.append((max(0, nearest - accumulate_frames), min(len(stride_list) - 1, nearest + accumulate_frames)))
    return dict(sample_num=sample_num, strides=stride_list, acc=accumulate_frames, windows=win)


def transforms(root, seq, Tr, strides, window, i):
    """[(stride frame j, P_transform)] of frame i's window."""
    Tr_inv = np.linalg.inv(Tr)
    Pi_inv = np.linalg.inv(_pose(root, seq, i))
    out = []
    for j in strides[window[0]:window[1] + 1]:
        Pij = np.dot(Pi_inv, _pose(root, seq, j))
        out.append((j, np.dot(Tr_inv, np.dot(Pij, Tr))))
    return out


def accumulate_frame(records, Ps, voxel_size, accumulate_radius):
    """The per-frame body: records [(7, n) float32] of the window in order with their P_transform [4,4].  Returns the
    [7, M] float32 record."""
    pcs, ints, sns = [], [], []
    for data_nwu, P in zip(records, Ps):
        x_inside = np.logical_and(data_nwu[0, :] < 2.7, data_nwu[0, :] > -2.7 * 0.75)
        y_inside = np.logical_and(data_nwu[1, :] < 0.8, data_nwu[1, :] > -0.8)
        data_nwu = data_nwu[:, np.logical_not(np.logical_and(x_inside, y_inside))]
        pcs.append(affine64(P, data_nwu[0:3, :]))
        ints.append(data_nwu[3:4, :])
        sns.append(affine64(P, data_nwu[4:7, :]))          # the reference moves the normals with the translation
    pc, intensity, sn = np.concatenate(pcs, 1), np.concatenate(ints, 1), np.concatenate(sns, 1)
    intensity_max = np.max(intensity)
    with np.errstate(divide="ignore", invalid="ignore"):
        colour = (np.transpose(intensity) / intensity_max)[:, 0].astype(np.float64)
    pc, A = voxel_downsample64(pc, voxel_size, np.concatenate([colour[None], sn], 0))
    intensity = A[0:1] * intensity_max
    sn = A[1:4]
    keep = np.linalg.norm(pc[0:2, :], axis=0) < accumulate_radius
    return np.concatenate((pc[:, keep], intensity[:, keep], sn[:, keep]), axis=0).astype(np.float32)


def accumulate_sequence(root, seq, Tr, frame_stride_dist=4, accumulate_radius=50, voxel_size=0.2, frames=None,
                        np_folder="voxel0.1-SNr0.6"):
    """accumulate_sequence without writing: returns plan(...) plus records {i: [7, M] float32} and the transforms
    {i: [(j, P)]} of `frames` (default all)."""
    p = plan(root, seq, frame_stride_dist, accumulate_radius, np_folder)
    p["records"], p["transforms"] = {}, {}
    for i in range(p["sample_num"]) if frames is None else frames:
        jp = transforms(root, seq, Tr, p["strides"], p["windows"][i], i)
        p["transforms"][i] = jp
        recs = [_record(root, seq, np_folder, j) for j, _ in jp]
        p["records"][i] = accumulate_frame(recs, [P for _, P in jp], voxel_size, accumulate_radius)
    return p
