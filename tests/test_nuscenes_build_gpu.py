"""The nuScenes list build on the GPU (deepi2p_b200.nuscenes_build.make_dataset_info): the list against the reference's
own run (tests/golden/nuscenes_build_small.npz) and against oracle_nuscenes_build on a larger seeded root, the planted
ties deferred and resolved to numpy's decision, run-to-run identity, an all-night root and a built list read by
nuscenes.nuscenes_batch."""
import ast
import os
import pickle
import sys

import numpy as np
import pytest
import torch

import oracle_nuscenes_build as onb
from deepi2p_b200 import nuscenes, nuscenes_build as nb, synthetic as syn

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_nuscenes_build_golden as mg  # noqa: E402

GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "nuscenes_build_small.npz"))
RAW_ARGS = ast.literal_eval(str(GOLDEN["raw_args"]))
V = RAW_ARGS["version"]


@pytest.fixture(scope="module")
def golden_root(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("nsraw"))
    info = syn.write_nuscenes_raw(d, **RAW_ARGS)
    assert mg.sample_data_digest(d) == str(GOLDEN["sample_data_sha256"])
    return d, info


def test_list_equals_the_reference_and_the_oracle(cuda, golden_root):
    root, _ = golden_root
    tables = nb.RawTables(root, V)
    nusc = onb.Devkit(V, root)
    for k, (skip, mt) in enumerate(GOLDEN["settings"]):
        st = {}
        items = nb.make_dataset_info(root, V, int(skip), float(mt), stats=st)
        assert items == mg.decode(GOLDEN[f"lidar_{k}"], GOLDEN[f"rows_{k}"], GOLDEN[f"offsets_{k}"], tables.sd_token)
        assert items == onb.make_dataset(nusc, int(skip), float(mt))
        with open(os.path.join(root, "dataset_info.list"), "rb") as f:
            assert pickle.load(f) == items
        assert st["entries"] == len(items), st
        if mt == 10.0:                                      # the planted ties lie at 10 m
            assert st["deferred"] > 0, st


def test_larger_root_with_stationary_stretches(cuda, tmp_path):
    root = str(tmp_path)
    syn.write_nuscenes_raw(root, n_scenes=42, seed=21, seconds=(3.0, 6.0))
    st = {}
    items = nb.make_dataset_info(root, "v1.0-mini", stats=st)
    assert st["scenes"] >= 40, st
    assert items == onb.make_dataset(onb.Devkit("v1.0-mini", root), 2, 10.0)
    longest = max(len(v) for _, cams in items for v in cams.values())
    assert longest > 24, longest            # a stop keeps the cameras inside the radius for seconds


def test_planted_ties_are_deferred_and_resolved(cuda, golden_root):
    root, info = golden_root
    tables = nb.RawTables(root, V)
    p = nb.plan(tables, 2)
    walks = nb.walks_device(tables, p, 10.0)
    tie_scene = tables.scene_token.index(info["tie_scene"])
    n = 0
    for e, r in enumerate(p["lidar"]):
        if tables.sd_token[int(r)].split("-")[2] != str(tie_scene):
            continue
        for cam, pos in info["tie_lanes"]:
            k = nuscenes.CAMERAS.index(cam)
            if tables.sd_token[int(p["own"][e, k])].endswith(f"{cam}-0"):
                w = 2 * (6 * e + k)
                assert walks["status"][w] == nb.WALK_DEFERRED and walks["counts"][w] == pos - 2, (e, cam)
                n += 1
    assert n >= 8
    rows, deferred = nb.resolve(tables, p, walks, 10.0)
    assert deferred >= n
    assert rows == nb.walks_host(tables, p, 10.0)
    # numpy's decision at an exact tie: 10 is not < 10, so the walk stops there; one ulp inside is appended
    items = nb.to_list(tables, p, rows)
    first = items[[tables.sd_token[int(r)] for r in p["lidar"]].index(f"sd-{RAW_ARGS['seed']}-{tie_scene}-LIDAR_TOP-0")]
    tag = f"sd-{RAW_ARGS['seed']}-{tie_scene}-"
    assert first[1]["CAM_FRONT"] == [tag + "CAM_FRONT-0"]
    assert first[1]["CAM_FRONT_LEFT"] == [tag + "CAM_FRONT_LEFT-0", tag + "CAM_FRONT_LEFT-2"]
    assert first[1]["CAM_BACK_LEFT"] == [tag + "CAM_BACK_LEFT-0", tag + "CAM_BACK_LEFT-2"]
    assert first[1]["CAM_BACK_RIGHT"] == [tag + "CAM_BACK_RIGHT-0"]


def test_repeated_runs_are_identical(cuda, golden_root):
    root, _ = golden_root
    tables = nb.RawTables(root, V)
    p = nb.plan(tables, 2)
    a = nb.walks_device(tables, p, 10.0)
    s = torch.cuda.Stream()
    b = nb.walks_device(tables, p, 10.0, stream=s)
    for k in ("counts", "status", "offsets", "tokens"):
        assert np.array_equal(a[k], b[k]), k


def test_all_night_root_gives_an_empty_list(cuda, tmp_path):
    syn.write_nuscenes_raw(str(tmp_path), n_scenes=4, seed=2, all_night=True)
    st = {}
    assert nb.make_dataset_info(str(tmp_path), "v1.0-mini", stats=st) == []
    assert st["entries"] == 0 and st["scenes"] == 0
    with open(tmp_path / "dataset_info.list", "rb") as f:
        assert pickle.load(f) == []


def test_built_list_feeds_nuscenes_batch(cuda, tmp_path):
    g = np.load(os.path.join(ROOT, "tests", "golden", "jpeg_small.npz"))
    so = np.concatenate([[0], np.cumsum(g["stream_lens"])])
    i = int(np.nonzero((g["shapes"][:, 0] == 900) & (g["shapes"][:, 1] == 1600))[0][0])
    blob = g["streams"][so[i]:so[i + 1]].tobytes()
    syn.write_nuscenes_raw(str(tmp_path), n_scenes=2, seed=4, special=False, seconds=(2.0, 2.5), jpeg=blob)
    items = nb.make_dataset_info(str(tmp_path), "v1.0-mini")
    info = nuscenes.load_dataset_info(str(tmp_path / "dataset_info.list"))
    assert info == items and len(items) >= 4
    tab = nuscenes.Tables(str(tmp_path), "v1.0-mini")
    sel = [items[0], items[len(items) // 2], items[-1]]
    pc, inten, sn, na, nbn, P, img, K, t_ij = nuscenes.nuscenes_batch(tab, sel, "val_random_Ry", 7, rng=2)
    torch.cuda.synchronize()
    assert pc.shape == (3, 3, 20480) and img.shape == (3, 3, 160, 320) and t_ij.shape == (3, 3)
    assert torch.isfinite(pc).all() and torch.isfinite(img).all() and torch.isfinite(P).all()
