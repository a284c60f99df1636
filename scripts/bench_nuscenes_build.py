"""Benchmark of the nuScenes list build (deepi2p_b200.nuscenes_build.make_dataset_info) on a trainval-shaped synthetic
root: --scenes scenes of --seconds s (850 x 20 s by default, as v1.0-trainval), LIDAR_TOP at 20 Hz, six cameras at
12 Hz, one radar at 13 Hz, stops and reversals.  Writes BENCH_NUSCENES_BUILD.json (or --out):

  - the root's size: scenes, sample_data records, JSON bytes, entries, camera tokens;
  - the stages of one full build: JSON parse, host preparation (columns and reverse index, then the scene filter,
    lidar walk and inverses), the device passes by CUDA events (median of --reps), host resumes of the deferred walks
    and the pickle, and the total; the number of deferred walks;
  - the oracle's per-entry numpy loop (oracle_nuscenes_build, the script's own loop) on one host core over the first
    --oracle-entries entries, measured, with the device list checked equal to it there;
  - the card name and power limit, read in the same run.

The reference itself needs nuscenes-devkit, which is not installed, and is not timed.

    python scripts/bench_nuscenes_build.py [--scenes 850] [--seconds 20] [--oracle-entries 300] [--out PATH]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_oxford_build import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=850)
    ap.add_argument("--seconds", type=float, default=20.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-entries", type=int, default=300)
    ap.add_argument("--out", default=os.path.join(ROOT, "BENCH_NUSCENES_BUILD.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_nuscenes_build needs a CUDA device")
    import oracle_nuscenes_build as onb
    from deepi2p_b200 import nuscenes_build as nb, synthetic as syn
    version = "v1.0-trainval"
    res = dict(card=card(), reps=a.reps)
    with tempfile.TemporaryDirectory() as tmp:
        warm = os.path.join(tmp, "warm")
        syn.write_nuscenes_raw(warm, n_scenes=6, seed=1, version=version)
        nb.make_dataset_info(warm, version)                    # library load, CUDA context, every kernel once
        root = os.path.join(tmp, "root")
        t0 = time.perf_counter()
        syn.write_nuscenes_raw(root, n_scenes=a.scenes, seed=2, version=version, seconds=(a.seconds, a.seconds))
        res["write_root_s"] = time.perf_counter() - t0
        st = {}
        items = nb.make_dataset_info(root, version, stats=st)
        json_bytes = sum(os.path.getsize(os.path.join(root, version, n + ".json")) for n in nb.TABLES)
        res["root"] = dict(scenes=st["scenes_total"], daytime_scenes=st["scenes"], seconds_per_scene=a.seconds,
                           sample_data=st["sample_data"], json_bytes=json_bytes, entries=st["entries"],
                           walks=st["walks"], device_tokens=st["tokens"],
                           list_tokens=sum(len(v) for _, c in items for v in c.values()))
        res["stages_s"] = {k: st[k + "_seconds"] for k in ("json", "index", "plan", "walk", "assemble", "total")}
        res["stages_note"] = ("json: json.load of the six tables; index: columns and reverse index; plan: scene "
                              "filter, lidar walk, poses and the stacked inverse; walk: uploads, the three device "
                              "passes and read-backs; assemble: host resumes of deferred walks, the token lists and "
                              "the pickle")
        res["deferred_walks"] = st["deferred"]
        tables = nb.RawTables(root, version)
        p = nb.plan(tables, 2)
        dev_s = [nb.walks_device(tables, p, 10.0)["seconds"] for _ in range(a.reps)]
        res["device_passes_ms_median"] = float(np.median(dev_s)) * 1e3
        nusc = onb.Devkit(version, root)
        t0 = time.perf_counter()
        ref = onb.make_dataset(nusc, 2, 10.0, limit=a.oracle_entries)
        w = time.perf_counter() - t0
        assert ref == items[:len(ref)], "device list differs from the oracle"
        res["oracle"] = dict(entries=len(ref), seconds=w, s_per_entry=w / len(ref),
                             note="oracle_nuscenes_build's per-entry numpy loop on one host core, measured over the "
                                  "first entries only; JSON loading not included")
        res["reference_note"] = "the reference's make_datasets.py needs nuscenes-devkit, not installed; not timed"
    with open(a.out, "w") as f:
        json.dump(res, f)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
