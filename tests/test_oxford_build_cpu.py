"""Host half of the Oxford RobotCar build (deepi2p_b200.oxford_build): the SDK restatements against scipy, the readers
and their errors, the plan against the reference's own run (tests/golden/oxford_build_small.npz), the oracle against
the fixture, the deviations' messages, train.txt and the script's arguments.  No GPU."""
import ast
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy.spatial.transform import Rotation, Slerp

import oracle_oxford_build as oo
from deepi2p_b200 import oxford_build as ob, synthetic as syn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "oxford_build_small.npz"))
RAW_ARGS = ast.literal_eval(str(GOLDEN["raw_args"]))
BUILD_ARGS = ast.literal_eval(str(GOLDEN["build_args"]))
T = str(GOLDEN["traversal"])


@pytest.fixture(scope="module")
def small(tmp_path_factory):
    d = tmp_path_factory.mktemp("oxraw")
    raw, lms, sdk, out = (str(d / x) for x in ("raw", "lms", "sdk", "out"))
    syn.write_oxford_raw(raw, lms, sdk, **RAW_ARGS)
    return raw, lms, sdk, out, ob.plan_traversal(raw, lms, out, T, sdk, **BUILD_ARGS)


def test_se3_and_quaternion_against_scipy():
    rng = np.random.default_rng(0)
    v = np.concatenate([rng.normal(0, 5, (50, 3)), rng.uniform(-3, 3, (50, 3))], 1)
    M = ob.se3(v)
    R = Rotation.from_euler("ZYX", v[:, [5, 4, 3]]).as_matrix()
    assert np.allclose(M[:, :3, :3], R, atol=1e-14) and np.array_equal(M[:, :3, 3], v[:, :3])
    q = ob.so3_to_quaternion(R)
    ref = Rotation.from_matrix(R).as_quat()[:, [3, 0, 1, 2]]
    sign = np.sign((q * ref).sum(1))[:, None]
    assert np.allclose(q, sign * ref, atol=1e-12)
    for k, Rb in enumerate([np.eye(3), np.diag([1.0, -1, -1]), np.diag([-1.0, 1, -1]), np.diag([-1.0, -1, 1])]):
        qb = ob.so3_to_quaternion(Rb)                # every branch of the largest component
        assert np.argmax(np.abs(qb)) == k and np.isclose(np.linalg.norm(qb), 1.0)


def test_interpolate_poses_brackets_hits_and_negative_d():
    ts = np.array([100, 200, 400])
    rot = Rotation.from_euler("z", [[0.0], [0.4], [1.0]])
    P = np.tile(np.eye(4), (3, 1, 1))
    P[:, :3, :3] = rot.as_matrix()
    P[:, :3, 3] = [[0, 0, 0], [1, 2, 3], [5, 0, -1]]
    A = ob.interpolate_absolute(ts, P, [100, 200, 150, 300])
    assert np.allclose(A[0], P[0], atol=1e-15) and np.allclose(A[1], P[1], atol=1e-14)
    want = Slerp(ts, rot)([150, 300]).as_matrix()
    assert np.allclose(A[2:, :3, :3], want, atol=1e-12)
    assert np.allclose(A[2, :3, 3], [0.5, 1, 1.5]) and np.allclose(A[3, :3, 3], [3, 1, 1])
    R = ob.interpolate_poses(ts, P, [150], 200)
    assert np.allclose(R[0], np.linalg.solve(P[1], A[2]), atol=1e-14)
    Pn = P.copy()                                   # d < 0: the z branch's quaternion of -3 rad has w < 0
    Pn[1, :3, :3] = Rotation.from_rotvec([0.0, 0.0, -0.4]).as_matrix()
    Pn[2, :3, :3] = Rotation.from_rotvec([0.0, 0.0, -3.0]).as_matrix()
    qa, qb = ob.so3_to_quaternion(Pn[1:, :3, :3])
    assert (qa * qb).sum() < 0
    An = ob.interpolate_absolute(ts, Pn, [300])
    assert np.allclose(An[0, :3, :3], Slerp([200, 400], Rotation.from_matrix(Pn[1:, :3, :3]))([300]).as_matrix(),
                       atol=1e-12)


def test_gj_inverse_matches_oracle_and_numpy():
    rng = np.random.default_rng(1)
    for _ in range(20):
        A = ob.se3(np.concatenate([rng.normal(0, 50, 3), rng.uniform(-3, 3, 3)]))
        inv = ob.gj_inverse(A)
        assert np.array_equal(inv, np.array(oo.gj_inverse(A)))
        assert np.allclose(inv, np.linalg.inv(A), atol=1e-12)


def test_readers_and_errors(tmp_path):
    p = tmp_path / "vo.csv"
    p.write_text("h\n10,0,1,2,3,0,0,0\n20,10,1,2,3,0,0,0.5\n")
    ts, v = ob.read_vo(str(p))
    assert ts.tolist() == [10, 20] and v.shape == (2, 6) and v[1, 5] == 0.5
    p.write_text("h\n10,0,1,2,3,0,0,0\n10,10,1,2,3,0,0,0.5\n")
    with pytest.raises(ValueError, match="line 3: VO timestamps must be strictly ascending"):
        ob.read_vo(str(p))
    p.write_text("h\n10,0,1,2\n")
    with pytest.raises(ValueError, match="line 2: not a VO row"):
        ob.read_vo(str(p))
    with pytest.raises(FileNotFoundError, match="VO file not found"):
        ob.read_vo(str(tmp_path / "none.csv"))
    e = tmp_path / "e.txt"
    e.write_text("1 2 3\n")
    with pytest.raises(ValueError, match="6 numbers"):
        ob.read_extrinsics(str(e))
    s = tmp_path / "s.bin"
    np.arange(7, dtype=np.float64).tofile(s)
    with pytest.raises(ValueError, match="triples"):
        ob.read_scan(str(s))
    t = tmp_path / "x.timestamps"
    t.write_text("5 1\n7 1\n")
    assert ob.read_timestamps(str(t)) == [5, 7]


def test_camera_model_cross_check(tmp_path):
    syn.write_oxford_sdk(str(tmp_path))
    path = tmp_path / "models" / ob.CAMERA_MODEL
    G = ob.read_camera_model(str(path))
    assert G.shape == (4, 4) and G[3, 3] == 1
    path.write_text(syn.OXFORD_CAMERA_MODEL.replace("643.788025", "640.0"))
    with pytest.raises(ValueError, match="K_CENTRE"):
        ob.read_camera_model(str(path))


def test_plan_equals_reference_fixture(small):
    *_, plan = small
    assert np.array_equal(plan["pc_timestamps"], GOLDEN["pc_timestamps"])
    assert np.array_equal(plan["camera_timestamps"], GOLDEN["camera_timestamps"])
    assert [hi - lo for _, lo, hi, _ in plan["centres"]] == GOLDEN["window_len"].tolist()
    assert len(plan["skipped_velocity"]) == 10
    # the global VO chain against the reference's window-local chains (DESIGN.md 4.24: measured 7.3e-14 for the
    # scans' relative poses and 2.0e-13 for the tables)
    assert np.abs(plan["pc_poses"] - GOLDEN["pc_poses"]).max() < 1e-11
    assert np.abs(plan["camera_poses"] - GOLDEN["camera_poses"]).max() < 1e-11
    off = 0
    for c, n in zip(GOLDEN["pose_centres"], GOLDEN["pose_lens"]):
        k = plan["pc_timestamps"].tolist().index(c)
        _, lo, hi, _ = plan["centres"][k]
        assert hi - lo == n and plan["lms_ts"][lo:hi] == GOLDEN["pose_lms_ts"][off:off + n].tolist()
        rel = np.einsum("ij,njk->nik", plan["centre_inv"][k], plan["lms_abs"][lo - plan["lms_lo"]:hi - plan["lms_lo"]])
        assert np.abs(rel - GOLDEN["pose_rel"][off:off + n]).max() < 1e-11
        off += n


def test_oracle_equals_reference_fixture(small):
    *_, plan = small
    off = np.concatenate([[0], np.cumsum(GOLDEN["m_pts"])])
    for c in range(len(plan["centres"])):
        o = oo.build_cloud(plan, c)
        ref = GOLDEN["records"][:, off[c]:off[c + 1]]
        assert o["record"].shape == ref.shape, c
        assert (o["n_kept"], o["n_skipped"]) == (GOLDEN["n_kept"][c], GOLDEN["n_skipped"][c]), c
        assert np.array_equal(o["record"][3], ref[3], equal_nan=True), c
        ulp = np.spacing(np.abs(ref[:3])).astype(np.float64)
        assert np.all(np.abs(o["record"][:3].astype(np.float64) - ref[:3]) <= ulp), c
    assert GOLDEN["n_skipped"].max() > 0 and np.isnan(GOLDEN["records"][3]).any()


def test_deviation_errors(small, tmp_path):
    raw, lms, sdk, out, _ = small
    with pytest.raises(ValueError, match=f"traversal {T}: no camera frame lies inside the VO span"):
        _truncated_vo(raw, lms, sdk, out, tmp_path / "few", keep=5)
    lms2 = str(tmp_path / "lms2")
    os.makedirs(os.path.join(lms2, T))
    with open(os.path.join(lms2, T, "lms_front.timestamps"), "w") as f:
        f.write("1 1\n")
    with pytest.raises(ValueError, match=f"traversal {T} centre .*: no LMS timestamp"):
        ob.plan_traversal(raw, lms2, out, T, sdk, **BUILD_ARGS)
    with pytest.raises(TypeError, match="unknown build parameters"):
        ob.plan_traversal(raw, lms, out, T, sdk, voxel=0.2)


def _truncated_vo(raw, lms, sdk, out, d, keep=None, drop=0):
    import shutil
    raw2 = str(d)
    shutil.copytree(os.path.join(raw, T), os.path.join(raw2, T))
    p = os.path.join(raw2, T, "vo", "vo.csv")
    lines = open(p).read().splitlines()
    with open(p, "w") as f:
        f.write("\n".join(lines[:keep] if keep else lines[:len(lines) - drop]) + "\n")
    return ob.plan_traversal(raw2, lms, out, T, sdk, **BUILD_ARGS), ob.read_vo(p)[0]


def _in_span(plan, vo_ts):
    lms = np.asarray(plan["lms_ts"])
    for c, lo, hi, _ in plan["centres"]:
        assert vo_ts[0] <= c < vo_ts[-1] and vo_ts[0] <= lms[lo] and lms[hi - 1] < vo_ts[-1]
    assert np.all((plan["camera_timestamps"] >= vo_ts[0]) & (plan["camera_timestamps"] < vo_ts[-1]))
    assert np.isfinite(plan["camera_poses"]).all() and np.isfinite(plan["pc_poses"]).all()


def test_camera_frames_past_the_vo_are_dropped(small, tmp_path):
    raw, lms, sdk, out, full = small
    plan, vo_ts = _truncated_vo(raw, lms, sdk, out, tmp_path / "short", drop=60)
    n_after = sum(c >= vo_ts[-1] for c in full["cameras"])
    assert n_after > 0 and plan["cameras_outside_vo"] == n_after
    assert plan["cameras"] == [c for c in full["cameras"] if c < vo_ts[-1]]
    assert 0 < len(plan["centres"]) < len(full["centres"])
    _in_span(plan, vo_ts)


def test_vo_sourced_at_camera_frames(tmp_path):
    """A RobotCar download's VO rows are sourced at stereo frames, so the last camera frame is the last VO timestamp:
    that frame is dropped, every other frame (each an exact VO timestamp) is planned."""
    raw, lms, sdk, out = (str(tmp_path / x) for x in ("raw", "lms", "sdk", "out"))
    syn.write_oxford_raw(raw, lms, sdk, **dict(RAW_ARGS, vo_on_cameras=True))
    vo_ts = ob.read_vo(os.path.join(raw, T, "vo", "vo.csv"))[0]
    cams = ob.read_timestamps(ob.camera_timestamps_path(raw, T))
    assert cams[-1] == vo_ts[-1] and set(cams) == set(vo_ts.tolist())
    plan = ob.plan_traversal(raw, lms, out, T, sdk, **BUILD_ARGS)
    assert plan["cameras_outside_vo"] == 1 and plan["cameras"][-1] == cams[-2]
    assert len(plan["centres"]) == len(GOLDEN["pc_timestamps"]) and len(plan["skipped_velocity"]) == 10
    _in_span(plan, vo_ts)


def test_selection_and_train_split(tmp_path):
    raw, lms, sdk, out = (str(tmp_path / x) for x in ("raw", "lms", "sdk", "out"))
    syn.write_oxford_raw(raw, lms, sdk, traversals=("a", "b"), night=("n",), seconds=3.0, n_returns=2)
    os.makedirs(os.path.join(out, "b"))
    open(os.path.join(out, "b", "tags.csv"), "w").write("sun\n")
    todo, night, done = ob.select_traversals(raw, out)
    assert (todo, night, done) == (["a"], ["n"], ["b"])
    assert ob.write_train_split(out) is None
    for t, tag in (("c", "night\n"), ("d", "sun\n"), ("v", "sun\n")):
        os.makedirs(os.path.join(out, t))
        open(os.path.join(out, t, "tags.csv"), "w").write(tag)
    os.makedirs(os.path.join(out, "incomplete"))
    open(os.path.join(out, "val.txt"), "w").write("v\n")
    assert ob.write_train_split(out) == ["b", "d"]
    assert open(os.path.join(out, "train.txt")).read() == "b\nd\n"


def test_script_arguments():
    script = os.path.join(ROOT, "scripts", "build_oxford.py")
    r = subprocess.run([sys.executable, script, "--help"], capture_output=True, text=True)
    assert r.returncode == 0 and "--sdk" in r.stdout and "--batch" in r.stdout
    r = subprocess.run([sys.executable, script, "raw", "lms"], capture_output=True, text=True)
    assert r.returncode == 2 and "OUT" in r.stderr
    r = subprocess.run([sys.executable, script, "r", "l", "o", "--sdk", "s", "--batch", "0"], capture_output=True,
                       text=True)
    assert r.returncode == 2 and "--batch" in r.stderr


def test_abi_rejects_malformed_input():
    from deepi2p_b200 import _native
    lib = _native.load()
    c = _native._c
    G = np.eye(4).reshape(16)
    Gp = G.ctypes.data_as(c.c_void_p)
    assert lib.oxford_build_plan_f64(None, None, 0, None, None, -1, Gp, 0.1, 1, None, None, None, None, None) == -22
    assert b"S must be" in lib.dib_last_error()
    bad = G.copy()
    bad[3] = np.nan
    assert lib.oxford_build_plan_f64(None, None, 0, None, None, 1, bad.ctypes.data_as(c.c_void_p), 0.1, 1, None, None,
                                     None, None, None) == -22
    assert b"G_posesource_laser" in lib.dib_last_error()
    assert lib.oxford_build_plan_f64(None, None, 0, None, None, 1, Gp, 0.1, 1, None, None, None, None, None) == -22
    assert lib.oxford_build_scatter_f64(None, None, None, None, None, None, None, None, None, 1, 1, 1, 0.1, 20, None,
                                        None, None) == -22
    assert b"multiple of 16" in lib.dib_last_error()
    assert lib.oxford_build_count_f64(None, None, None, None, None, 1, 1, 1, float("inf"), None, None, None, None, 0,
                                      None) == -22
    assert lib.oxford_build_pack_f32(None, None, None, None, Gp, 1, 16, 32, None, None) == -22
    assert lib.oxford_build_count_workspace_bytes(-1, 4) == 0
