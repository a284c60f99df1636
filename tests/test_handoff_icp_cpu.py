"""The ICP driver's host logic (handoff.get_p_diff, icp.calibrate_scale, register_dir.py --method icp / --monodepth):
no GPU needed."""
import os
import subprocess
import sys

import numpy as np
from scipy.spatial.transform import Rotation

from deepi2p_b200 import handoff, icp, synthetic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = os.path.join(ROOT, "scripts", "register_dir.py")


def test_calibrate_scale_matches_the_reference_rule():
    f = synthetic.make_icp_frame(3, "kitti")
    pc, P, K = f["src"].astype(np.float64), f["P_gt"], f["K"]
    homo = np.concatenate((pc, np.ones((1, pc.shape[1]))), axis=0)          # registration_icp.py:39-55, 215-216
    cam = np.dot(P, homo)[0:3, :]
    pxpy = np.dot(K, cam)[0:2, :] / np.dot(K, cam)[2:3, :]
    mask = ((pxpy[0] >= 0) & (pxpy[0] <= f["W"] - 1) & (pxpy[1] >= 0) & (pxpy[1] <= f["H"] - 1) & (cam[2] > 0.1))
    want = np.mean(cam[2, mask]) / np.mean(f["tgt"][2, :])
    got = icp.calibrate_scale(pc, P, K, f["H"], f["W"], f["tgt"])
    assert abs(got - want) <= 1e-12 * want


def _forced(P):
    P = P.copy()
    P[0, 1] = P[1, 0] = P[1, 2] = P[2, 1] = 0
    P[1, 1] = 1
    return P


def test_get_p_diff_on_forced_non_rigid_poses():
    rng = np.random.default_rng(0)
    for _ in range(20):
        R = Rotation.from_euler("xyz", rng.uniform(-0.3, 0.3, 3) + [0, rng.uniform(-3, 3), 0]).as_matrix()
        Pp = np.eye(4)
        Pp[:3, :3] = R
        Pp[:3, 3] = rng.uniform(-5, 5, 3)
        Pp = _forced(Pp)                                   # not orthonormal any more
        Pg = np.eye(4)
        Pg[:3, :3] = synthetic.ry_matrix(rng.uniform(-3, 3))
        Pg[:3, 3] = rng.uniform(-5, 5, 3)
        D = np.dot(np.linalg.inv(Pp), Pg)                  # registration_icp.py:57-65, 224-225
        r = np.sum(np.abs(Rotation.from_matrix(D[0:3, 0:3]).as_euler("xzy", degrees=True)))
        r = 360 - r if r > 180 else r
        t, rr = handoff.get_p_diff(Pp[None], Pg[None])
        assert t[0] == np.linalg.norm(D[0:3, 3]) and rr[0] == r
    # the fold: a pose 190 deg off about y reads 170
    Pg = np.eye(4)
    Pg[:3, :3] = synthetic.ry_matrix(np.radians(190.0))
    _, rr = handoff.get_p_diff(np.eye(4)[None], Pg[None])
    assert abs(rr[0] - 170.0) < 1e-9


def _run(*args):
    return subprocess.run([sys.executable, CLI, *args], capture_output=True, text=True)


def test_cli_icp_needs_monodepth_and_others_refuse_it(tmp_path):
    d = str(tmp_path / "data")
    synthetic.write_icp_handoff(d, str(tmp_path / "monodepth"), [1], "kitti")
    r = _run(d, "--H", "160", "--W", "512", "--method", "icp")
    assert r.returncode == 2 and "--monodepth" in r.stderr
    for method in ("lsq", "pnp"):
        r = _run(d, "--H", "160", "--W", "512", "--method", method, "--monodepth", str(tmp_path / "monodepth"))
        assert r.returncode == 2 and "--monodepth is only used by --method icp" in r.stderr


def test_write_icp_handoff_layout(tmp_path):
    d, md = str(tmp_path / "data"), str(tmp_path / "monodepth")
    frames = synthetic.write_icp_handoff(d, md, [4, 5], "kitti")
    assert handoff.list_records(d) == sorted(frames)
    for name, f in frames.items():
        pc, lab, K, P = handoff.load_record(d, name)
        np.testing.assert_array_equal(pc, f["src"])
        np.testing.assert_array_equal(P, f["P_gt"])
        np.testing.assert_array_equal(np.load(os.path.join(md, name + "_pc.npy")), f["tgt"])
