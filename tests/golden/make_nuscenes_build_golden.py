"""Write tests/golden/nuscenes_build_small.npz: the reference's own make_nuscenes_dataset (data/nuscenes/make_datasets.py)
on a small seeded raw root (synthetic.write_nuscenes_raw with RAW_ARGS), run on the CPU.  No GPU, no network:

    python tests/golden/make_nuscenes_build_golden.py [OUT.npz] [--reference DIR]

The reference runs unedited.  Its imports are stubbed:
  - nuscenes.nuscenes.NuScenes is oracle_nuscenes_build.Devkit: the JSON tables with .scene, .get and the reverse
    index the script reads (each record's channel, sample['data'][channel]), restated from the devkit (DESIGN.md 4.28);
  - pyquaternion.Quaternion(q).rotation_matrix is deepi2p_b200.nuscenes.rotation_matrix (DESIGN.md 4.20).

Stored per setting (frame_skip, max_translation) in SETTINGS: the entries' LIDAR_TOP rows of sample_data.json and, per
entry and camera, the rows of the camera tokens in the reference's order (ragged, with offsets), plus the SHA-256 of
the root's sample_data.json so that a change to the writer is caught instead of compared.
"""
import hashlib
import importlib.util
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

VERSION = "v1.0-mini"
RAW_ARGS = dict(n_scenes=9, seed=5, version=VERSION, seconds=(2.0, 5.0))
SETTINGS = ((2, 10.0), (3, 10.0), (2, 4.0))


def import_reference(ref_dir):
    import oracle_nuscenes_build
    from deepi2p_b200 import nuscenes

    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    class Quaternion:
        def __init__(self, q):
            self.rotation_matrix = nuscenes.rotation_matrix(q)

    mod("pyquaternion", Quaternion=Quaternion)
    mod("nuscenes", __path__=[])
    mod("nuscenes.nuscenes", NuScenes=oracle_nuscenes_build.Devkit)
    spec = importlib.util.spec_from_file_location("make_datasets", os.path.join(ref_dir, "data", "nuscenes",
                                                                                "make_datasets.py"))
    md = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(md)
    return md


def encode(items, sd_index):
    """(lidar rows [E], camera rows (ragged), offsets [E * 6 + 1]) of a dataset list."""
    from deepi2p_b200.nuscenes import CAMERAS
    lidar = np.array([sd_index[t] for t, _ in items], dtype=np.int32)
    lists = [[sd_index[t] for t in cams[c]] for _, cams in items for c in CAMERAS]
    off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
    rows = np.array([r for x in lists for r in x], dtype=np.int32)
    return lidar, rows, off


def decode(lidar, rows, off, tokens):
    from deepi2p_b200.nuscenes import CAMERAS
    out = []
    for e, r in enumerate(lidar):
        cams = {c: [tokens[i] for i in rows[off[6 * e + k]:off[6 * e + k + 1]]] for k, c in enumerate(CAMERAS)}
        out.append((tokens[r], cams))
    return out


def sample_data_digest(root):
    with open(os.path.join(root, VERSION, "sample_data.json"), "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def make(out_path, ref_dir):
    import json
    from deepi2p_b200 import synthetic as syn
    md = import_reference(ref_dir)
    res = dict(raw_args=np.array(repr(RAW_ARGS)), settings=np.array(SETTINGS))
    with tempfile.TemporaryDirectory() as root:
        syn.write_nuscenes_raw(root, **RAW_ARGS)
        res["sample_data_sha256"] = np.array(sample_data_digest(root))
        with open(os.path.join(root, VERSION, "sample_data.json")) as f:
            sd_index = {r["token"]: i for i, r in enumerate(json.load(f))}
        nusc = md.NuScenes(version=VERSION, dataroot=root, verbose=True)
        for k, (skip, mt) in enumerate(SETTINGS):
            items = md.make_nuscenes_dataset(nusc, frame_skip=skip, max_translation=mt)
            res[f"lidar_{k}"], res[f"rows_{k}"], res[f"offsets_{k}"] = encode(items, sd_index)
            print(f"frame_skip {skip}, max_translation {mt}: {len(items)} entries, {len(res[f'rows_{k}'])} tokens")
    np.savez_compressed(out_path, **res)
    print(f"wrote {out_path}: {os.path.getsize(out_path)} bytes")


if __name__ == "__main__":
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    from oracle import build_ref
    ref = sys.argv[sys.argv.index("--reference") + 1] if "--reference" in sys.argv else build_ref.REF
    if "--reference" in sys.argv:
        args = [a for a in args if a != ref]
    make(args[0] if args else os.path.join(HERE, "nuscenes_build_small.npz"), ref)
