"""Host half of the nuScenes list build (deepi2p_b200.nuscenes_build): the oracle and the host rules against the
reference's own run (tests/golden/nuscenes_build_small.npz), the devkit's reverse index, the scene filter, the lidar
counter and each camera-walk rule on hand-built tables, the stacked inverse, the deferral bound, the C ABI's
rejections and the script's refusal without a device.  No GPU."""
import ast
import json
import os
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest

import oracle_nuscenes_build as onb
from deepi2p_b200 import nuscenes, nuscenes_build as nb, synthetic as syn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_nuscenes_build_golden as mg  # noqa: E402

GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "nuscenes_build_small.npz"))
RAW_ARGS = ast.literal_eval(str(GOLDEN["raw_args"]))
V = RAW_ARGS["version"]


@pytest.fixture(scope="module")
def golden_root(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("nsraw"))
    syn.write_nuscenes_raw(d, **RAW_ARGS)
    assert mg.sample_data_digest(d) == str(GOLDEN["sample_data_sha256"])
    return d


def golden_list(k, tokens):
    return mg.decode(GOLDEN[f"lidar_{k}"], GOLDEN[f"rows_{k}"], GOLDEN[f"offsets_{k}"], tokens)


def test_oracle_and_host_rules_equal_the_reference(golden_root):
    tables = nb.RawTables(golden_root, V)
    nusc = onb.Devkit(V, golden_root)
    for k, (skip, mt) in enumerate(GOLDEN["settings"]):
        ref = golden_list(k, tables.sd_token)
        assert len(ref) > 50
        assert onb.make_dataset(nusc, int(skip), float(mt)) == ref
        p = nb.plan(tables, int(skip))
        assert nb.to_list(tables, p, nb.walks_host(tables, p, float(mt))) == ref


# ------------------------------------------------------------------ hand-built tables
def write_tables(root, scenes, sd, ego, sensors=None):
    """scenes [(token, description, first sample)], sd [dict(token, channel, sample, key, next, prev, xyz)]; sample
    tokens come from sd; one calibrated_sensor per channel whose token is not the channel's name."""
    chans = sensors or ["LIDAR_TOP", *nuscenes.CAMERAS]
    tabs = dict(sensor=[dict(token=f"s{k}", channel=c, modality="x") for k, c in enumerate(chans)],
                calibrated_sensor=[dict(token=f"c{k}", sensor_token=f"s{k}", translation=[0, 0, 0],
                                        rotation=[1, 0, 0, 0], camera_intrinsic=[]) for k in range(len(chans))],
                scene=[dict(token=t, description=d, first_sample_token=f) for t, d, f in scenes],
                sample=[dict(token=s) for s in dict.fromkeys(r["sample"] for r in sd)],
                sample_data=[dict(token=r["token"], sample_token=r["sample"], is_key_frame=r["key"],
                                  calibrated_sensor_token=f"c{chans.index(r['channel'])}", ego_pose_token=f"e{i}",
                                  next=r.get("next", ""), prev=r.get("prev", "")) for i, r in enumerate(sd)],
                ego_pose=[dict(token=f"e{i}", rotation=r.get("rot", [1.0, 0, 0, 0]), translation=r["xyz"])
                          for i, r in enumerate(sd)] + ego)
    os.makedirs(os.path.join(root, "v"), exist_ok=True)
    for name, recs in tabs.items():
        with open(os.path.join(root, "v", name + ".json"), "w") as f:
            json.dump(recs, f)
    return nb.RawTables(root, "v")


def chain(prefix, channel, xyzs, sample="S", key_at=0):
    n = len(xyzs)
    return [dict(token=f"{prefix}{i}", channel=channel, sample=sample, key=i == key_at, xyz=list(xyzs[i]),
                 next=f"{prefix}{i + 1}" if i + 1 < n else "", prev=f"{prefix}{i - 1}" if i else "")
            for i in range(n)]


def cameras(positions=None, key_at=0):
    out = []
    for k, c in enumerate(nuscenes.CAMERAS):
        out += chain(f"{c}-", c, (positions or {}).get(c, [(0.0, 0.0, 0.0)] * 3), key_at=key_at)
    return out


def test_reverse_index_channel_and_last_key_frame_wins(tmp_path):
    sd = chain("L", "LIDAR_TOP", [(0, 0, 0)] * 2) + cameras()
    sd.append(dict(token="late", channel="CAM_BACK", sample="S", key=True, xyz=[0, 0, 0]))     # competes, wins
    sd.append(dict(token="sweep", channel="CAM_FRONT", sample="S", key=False, xyz=[0, 0, 0]))  # not a key frame
    t = write_tables(str(tmp_path), [("sc", "day", "S")], sd, [])
    data = dict(zip(t.channels, t.sample_data[0]))
    assert t.sd_token[data["CAM_BACK"]] == "late" and t.sd_token[data["CAM_FRONT"]] == "CAM_FRONT-0"
    assert t.sd_token[data["LIDAR_TOP"]] == "L0"
    assert [t.channels[c] for c in t.sd_channel[:3]] == ["LIDAR_TOP"] * 2 + ["CAM_FRONT"]
    assert onb.Devkit("v", str(tmp_path)).get("sample", "S")["data"]["CAM_BACK"] == "late"


def test_scene_filter_and_order(tmp_path):
    descs = ["day", "rain at night", "Night, rain", "NIGHT drive", "day", "nightfall", "day"]
    tokens = [f"sc{i}" for i in range(len(descs))]
    tokens[4] = nb.TEST_NIGHT_SCENE_TOKENS[7]
    t = write_tables(str(tmp_path), list(zip(tokens, descs, ["S"] * len(descs))),
                     chain("L", "LIDAR_TOP", [(0, 0, 0)]) + cameras(), [])
    assert nb.daytime_scenes(t) == [0, 3, 6]
    assert len(nb.TEST_NIGHT_SCENE_TOKENS) == 18 and nb.TEST_NIGHT_SCENE_TOKENS[0] == syn.NUSCENES_NIGHT_TOKEN


def test_lidar_counter(tmp_path):
    t = write_tables(str(tmp_path), [("sc", "day", "S")], chain("L", "LIDAR_TOP", [(0, 0, 0)] * 9) + cameras(), [])
    rows = lambda s: [t.sd_token[r] for r in nb.scene_lidar_rows(t, 0, s)]
    assert rows(2) == ["L0", "L1", "L3", "L5", "L7"]
    assert rows(3) == ["L0", "L2", "L5", "L8"]
    assert rows(1) == [f"L{i}" for i in range(9)]
    assert rows(20) == ["L0"]
    nusc = onb.Devkit("v", str(tmp_path))
    for s in (1, 2, 3, 20):
        assert onb.lidar_tokens(nusc, s) == rows(s)


def walk_lists(root, positions, max_translation=10.0, key_at=0):
    t = write_tables(root, [("sc", "day", "S")], chain("L", "LIDAR_TOP", [(100.0, 200.0, 1.0)]) +
                     cameras(positions, key_at), [])
    p = nb.plan(t, 2)
    got = nb.to_list(t, p, nb.walks_host(t, p, max_translation))
    assert got == onb.make_dataset(onb.Devkit("v", root), 2, max_translation)
    return got[0][1]


def test_camera_walk_rules(tmp_path):
    far, at = (150.0, 200.0, 1.0), (101.0, 200.0, 1.0)
    pos = {
        # own never tested (50 m away), first neighbour never tested or appended (far), then append until a failure
        "CAM_FRONT": [far, far, at, at, (111.0, 200.0, 1.0), at],
        # the chain ends at the first neighbour: nothing
        "CAM_FRONT_LEFT": [at, at],
        # a NaN translation stops the walk
        "CAM_FRONT_RIGHT": [at, at, at, (float("nan"), 200.0, 1.0), at],
        # exactly 10 m is not < 10
        "CAM_BACK": [at, at, (110.0, 200.0, 1.0), at],
        "CAM_BACK_LEFT": [at],
        "CAM_BACK_RIGHT": [at, far, at],
    }
    got = walk_lists(str(tmp_path / "a"), pos)
    assert got["CAM_FRONT"] == ["CAM_FRONT-0", "CAM_FRONT-2", "CAM_FRONT-3"]
    assert got["CAM_FRONT_LEFT"] == ["CAM_FRONT_LEFT-0"]
    assert got["CAM_FRONT_RIGHT"] == ["CAM_FRONT_RIGHT-0", "CAM_FRONT_RIGHT-2"]
    assert got["CAM_BACK"] == ["CAM_BACK-0"]
    assert got["CAM_BACK_LEFT"] == ["CAM_BACK_LEFT-0"]
    assert got["CAM_BACK_RIGHT"] == ["CAM_BACK_RIGHT-0", "CAM_BACK_RIGHT-2"]
    assert list(got) == list(nuscenes.CAMERAS)
    # own in the middle: next results, then prev results; each direction skips its first neighbour
    mid = {c: [at, at, at, far, at, at, at] for c in nuscenes.CAMERAS}
    got = walk_lists(str(tmp_path / "b"), mid, key_at=3)
    assert got["CAM_FRONT"] == ["CAM_FRONT-3", "CAM_FRONT-5", "CAM_FRONT-6", "CAM_FRONT-1", "CAM_FRONT-0"]


def test_missing_camera_names_sample_and_channel(tmp_path):
    sd = chain("L", "LIDAR_TOP", [(0, 0, 0)]) + [r for r in cameras() if not r["token"].startswith("CAM_BACK-")]
    t = write_tables(str(tmp_path), [("sc", "day", "S")], sd, [])
    with pytest.raises(ValueError, match="sample S has no CAM_BACK record"):
        nb.plan(t, 2)


def test_stacked_inverse_is_the_per_matrix_inverse():
    rng = np.random.default_rng(3)
    Ps = []
    for _ in range(500):
        q = rng.normal(size=4)
        t = rng.uniform(-2000, 2000, 3) * 10.0 ** rng.uniform(-3, 0)
        Ps.append(nuscenes.P_from_record(dict(rotation=list(q / np.linalg.norm(q)), translation=list(t))))
    stack = np.linalg.inv(np.stack(Ps))
    for P, inv in zip(Ps, stack):
        assert np.array_equal(np.linalg.inv(P), inv)


def _fma(a, b, c):
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def device_norm(inv, p, fma):
    """walk_step's N and s as nvcc may compile them: plain, or with the sums contracted into FMAs."""
    t, s = [], 0.0
    for i in range(3):
        r = inv[i]
        a = [float(r[0] * p[0]), float(r[1] * p[1]), float(r[2] * p[2]), float(r[3])]
        if fma:
            t.append(_fma(r[2], p[2], _fma(r[1], p[1], a[0])) + a[3])
        else:
            t.append(((a[0] + a[1]) + a[2]) + a[3])
        s += ((abs(a[0]) + abs(a[1])) + abs(a[2])) + abs(a[3])
    sq = _fma(t[2], t[2], _fma(t[1], t[1], t[0] * t[0])) if fma else (t[0] * t[0] + t[1] * t[1]) + t[2] * t[2]
    return float(np.sqrt(sq)), s


def test_deferral_bound_covers_any_summation_order():
    rng = np.random.default_rng(11)
    worst = 0.0
    for it in range(3000):
        mag = 10.0 ** rng.uniform(-2, 3.5)
        R = nuscenes.rotation_matrix(list(rng.normal(size=4)))
        P = np.identity(4)
        P[:3, :3] = R.astype(np.float32)
        P[:3, 3] = (rng.uniform(-1, 1, 3) * mag).astype(np.float32)
        inv = np.linalg.inv(P)
        c = np.identity(4)
        c[:3, 3] = (P[:3, 3] + rng.normal(0, 10.0 ** rng.uniform(-3, 1.5), 3)).astype(np.float32)
        n_np = np.linalg.norm(np.dot(inv, c)[0:3, 3])
        rows = inv[:3].astype(np.float64)
        p = [float(v) for v in c[:3, 3]]
        # other orders numpy's BLAS might use: reversed and pairwise sums, with and without contraction
        alts = []
        for order in ((3, 2, 1, 0), (0, 2, 1, 3)):
            t = []
            for i in range(3):
                terms = [rows[i, j] * p[j] for j in range(3)] + [rows[i, 3]]
                x = terms[order[0]]
                for j in order[1:]:
                    x = x + terms[j]
                t.append(x)
            alts.append(float(np.sqrt(t[2] * t[2] + (t[1] * t[1] + t[0] * t[0]))))
        pair = [(rows[i, 0] * p[0] + rows[i, 1] * p[1]) + (rows[i, 2] * p[2] + rows[i, 3]) for i in range(3)]
        alts.append(float(np.sqrt((pair[0] * pair[0] + pair[1] * pair[1]) + pair[2] * pair[2])))
        for fma in (False, True):
            n_dev, s = device_norm(rows, p, fma)
            b = nb.deferral_bound(s, n_dev)
            assert b < 1e-14 * (s + n_dev)
            for other in [n_np] + alts:
                assert abs(other - n_dev) <= b, (it, fma, other, n_dev, b)
                worst = max(worst, abs(other - n_dev) / b)
    assert 0 < worst < 0.5          # the bound is not vacuous, and leaves a margin


def test_abi_rejects_malformed_input():
    from deepi2p_b200 import _native
    lib = _native.load()
    assert lib.nuscenes_walk_count(None, None, None, 0, None, None, -1, 10.0, None, None, None) == -22
    assert b"E must be" in lib.dib_last_error()
    assert lib.nuscenes_walk_count(None, None, None, 0, None, None, 1, float("nan"), None, None, None) == -22
    assert b"max_translation" in lib.dib_last_error()
    assert lib.nuscenes_walk_count(None, None, None, 4, None, None, 1, 10.0, None, None, None) == -22
    assert b"null" in lib.dib_last_error()
    assert lib.nuscenes_walk_fill(None, None, None, -1, None, None, 1, 10.0, None, None, None) == -22
    assert lib.nuscenes_walk_count(None, None, None, 0, None, None, 0, 10.0, None, None, None) == 0
    assert lib.nuscenes_walk_scan_workspace_bytes(-1) == 0
    assert lib.nuscenes_walk_scan_workspace_bytes(1025) == 16
    assert lib.nuscenes_walk_scan(None, -1, None, None, 0, None) == -22
    buf = np.zeros(2, dtype=np.int64)
    c = _native._c
    assert lib.nuscenes_walk_scan(buf.ctypes.data_as(c.c_void_p), 2000, buf.ctypes.data_as(c.c_void_p),
                                  buf.ctypes.data_as(c.c_void_p), 8, None) == -12


def test_script_arguments_and_no_device():
    script = os.path.join(ROOT, "scripts", "build_nuscenes.py")
    r = subprocess.run([sys.executable, script, "--help"], capture_output=True, text=True)
    assert r.returncode == 0 and "--max-translation" in r.stdout
    r = subprocess.run([sys.executable, script, "--dataroot", "r"], capture_output=True, text=True)
    assert r.returncode != 0 and "--version" in r.stderr
    r = subprocess.run([sys.executable, script, "--dataroot", "r", "--version", "v", "--frame-skip", "0"],
                       capture_output=True, text=True)
    assert r.returncode != 0 and "positive" in r.stderr
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, script, "--dataroot", "r", "--version", "v"], capture_output=True, text=True,
                       env=env)
    assert r.returncode != 0 and "needs a CUDA device" in r.stderr
    import torch
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="needs a CUDA device"):
            nb.make_dataset_info("r", "v")
