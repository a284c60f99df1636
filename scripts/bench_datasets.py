"""Throughput of the point side of KITTI and Oxford classifier batches read from a dataset root (deepi2p_b200.kitti,
deepi2p_b200.oxford), by where the scan records come from.

    python scripts/bench_datasets.py [--kitti-samples 1,12,64] [--oxford-samples 64] [--reps 5] [--out FILE.json]

Roots: synthetic.write_kitti_root (one sequence of 120 frames, records of a 64 x 1024-ray make_lidar_scan with 60-95%
of the rays kept, [7, n]) and synthetic.write_oxford_root (one traversal of 96 clouds, 32 x 1024 rays, [4, n]),
written to a temporary directory by this run, so every record read is served from the page cache ("warm").  A batch of
S samples takes S consecutive entries of the list (KITTI: interleaved P2 / P3, so neighbouring samples share their
records).  The host plan (walk, transforms, pairing draws) is made once per batch outside the timed window; the timed
window is the point side, from records to assemble_batch's outputs, in train mode with N = 20480, Ma = Mb = 128:

    device_store   store_frames on a long-lived device ScanStore, then assemble_batch
    pinned_store   the same on a pinned host ScanStore, read by the kernel through mapped memory over PCIe
    per_batch      np.load of the batch's distinct records, a per-batch pinned store, one upload, the gather
    pack_frames    np.load of every frame's record, pack_frames (padded [T,3,n] from pageable memory), assemble_batch

The readers are also timed whole (kitti_batch / oxford_batch: host plan, record reads, the point side, the image
side with its file reads and, for Oxford, the 1280 x 960 JPEG decode), with the device store and with a per-batch
store; there the host plan and the image side come on top of the point side.

Each path also reports its accumulation call alone (CUDA events around accumulate / accumulate_gather with the count
read-back) and the bytes it gathers (the frames' 28 (KITTI) or 16 (Oxford) bytes per point, plus the 12 bytes of xyz
the range mask reads again for Oxford) as a fraction of HBM3 bandwidth (3.35 TB/s, device store) or of PCIe Gen5 x16
(64 GB/s per direction, pinned store).  The GPU and its power limit are recorded beside the numbers.
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from deepi2p_b200 import assemble, kitti, oxford, synthetic  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_prep import _power_limit, _time  # noqa: E402

HBM = 3.35e12
PCIE = 64e9
N, M = 20480, 128


def _kitti_case(ds, dev, pin, S, reps):
    plan = kitti.plan_batch(ds, range(S), "train", np.random.default_rng(S))
    keys = [(p["seq"], j) for p in plan for j in p["walk"]]
    fs = np.concatenate([[s] * len(p["walk"]) for s, p in enumerate(plan)])
    FT = np.concatenate([p["frame_T"] for p in plan])
    args = assemble.kitti_args(np.stack([p["Pc"] for p in plan]), np.stack([p["Pji"] for p in plan]))
    paths = [kitti.record_path(ds.root, *k) for k in keys]
    out = _paths(keys, fs, FT, args, paths, kitti.read_record, dev, pin, reps, 28, 0, S)
    out["kitti_batch"] = _whole(lambda store: kitti.kitti_batch(ds, range(S), "train", 7, rng=S, store=store), dev,
                                reps, S)
    return out


def _whole(call, dev, reps, S):
    """The reader called end to end (host plan, records, images, point and image sides) with the device store and
    with a per-batch store."""
    out = {}
    for name, store in (("device_store", dev), ("per_batch", None)):
        t = _time(lambda: call(store), reps)
        out[name] = {"seconds": t, "samples_per_s": S / t}
    return out


def _oxford_case(ds, dev, pin, S, reps):
    plan = oxford.plan_batch(ds, range(S), "train", np.random.default_rng(S))
    keys = [(p["traversal"], p["pc_timestamp"]) for p in plan]
    fs = np.arange(S)
    FT = np.tile(np.eye(4), (S, 1, 1))
    args = assemble.oxford_args(np.stack([p["P_cam_pc"] for p in plan]))
    paths = [oxford.record_path(ds.root, *k) for k in keys]
    out = _paths(keys, fs, FT, args, paths, oxford.read_record, dev, pin, reps, 16, 12, S)
    out["oxford_batch"] = _whole(lambda store: oxford.oxford_batch(ds, range(S), "train", 7, rng=S, store=store), dev,
                                 reps, S)
    return out


def _paths(keys, fs, FT, args, paths, read, dev, pin, reps, bpp, reread, S):
    def run(frames):
        return assemble.assemble_batch(frames, "train", 7, input_pt_num=N, node_a_num=M, node_b_num=M, rng=0, **args)

    def per_batch():
        uniq, ids = assemble.unique_records(keys)
        recs = [read(paths[keys.index(k)]) for k in uniq]
        return assemble.batch_frames(recs, ids, fs, FT)

    def packed():
        samples = [([], []) for _ in range(S)]
        for k, (s, T) in enumerate(zip(fs, FT)):
            r = read(paths[k])
            samples[s][0].append((r[:3], r[3], r[4:7] if r.shape[0] == 7 else None))
            samples[s][1].append(T)
        return assemble.pack_frames(samples)

    ids_dev = [dev.index(k) for k in keys]
    fr_dev = assemble.store_frames(dev, ids_dev, fs, FT)
    fr_pin = assemble.store_frames(pin, ids_dev, fs, FT)
    npts = int(sum(dev.counts[i] for i in ids_dev))
    gathered = npts * (bpp + reread)
    rmax = args["range_max"]
    out = {"samples": S, "frames": len(keys), "distinct_records": len(set(keys)), "points_accumulated": npts,
           "gathered_bytes": gathered}
    for name, fn in (("device_store", lambda: run(fr_dev)), ("pinned_store", lambda: run(fr_pin)),
                     ("per_batch", lambda: run(per_batch())), ("pack_frames", lambda: run(packed()))):
        t = _time(fn, reps)
        out[name] = {"seconds": t, "samples_per_s": S / t}
    pk = packed()
    for name, fr, peak in (("device_store", fr_dev, HBM), ("pinned_store", fr_pin, PCIE)):
        t = _time(lambda: assemble.accumulate_gather(fr, rmax), reps)
        out[name]["accumulate_s"] = t
        out[name]["gathered_fraction_of_" + ("hbm" if peak == HBM else "pcie")] = gathered / t / peak
    t = _time(lambda: assemble.accumulate(pk["xyz"], pk["intensity"], pk["sn"], pk["n_pts"], pk["frame_sample"],
                                          pk["frame_T"], rmax), reps)
    out["pack_frames"]["accumulate_s_on_padded_device_buffers"] = t
    a = run(fr_dev)
    for fr in (fr_pin, per_batch(), packed()):
        b = run(fr)
        assert all(torch.equal(a[k], b[k]) for k in ("pc", "intensity", "sn", "node_a", "node_b")), "paths differ"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kitti-samples", default="1,12,64")
    ap.add_argument("--oxford-samples", default="64")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_datasets.py needs a CUDA device")
    result = {"gpu": torch.cuda.get_device_name(0), "power_limit": _power_limit(), "input_pt_num": N,
              "node_a_num": M, "node_b_num": M, "mode": "train",
              "file_cache": "warm: every record was written by this run and is read from the page cache",
              "hbm_bytes_per_s": HBM, "pcie_bytes_per_s": PCIE, "kitti": {}, "oxford": {}}
    with tempfile.TemporaryDirectory() as root:
        kr, orr = os.path.join(root, "kitti"), os.path.join(root, "oxford")
        synthetic.write_kitti_root(kr, seqs=(0,), n_frames=120, n_rings=64, n_azimuth=1024, n_images=1)
        synthetic.write_oxford_root(orr, train=("t0",), val=(), n_clouds=96, n_rings=32, n_azimuth=1024, n_images=1)
        ds = kitti.KittiDataset(kr, "train", seqs=(0,))
        dev = kitti.scan_store(kr, (0,), "cuda")
        pin = kitti.scan_store(kr, (0,), "pinned")
        result["kitti"]["store"] = {"records": len(dev), "bytes": dev.nbytes,
                                    "mean_points_per_record": float(dev.counts.mean())}
        for S in (int(v) for v in a.kitti_samples.split(",") if v):
            result["kitti"][str(S)] = _kitti_case(ds, dev, pin, S, a.reps)
        del dev, pin
        ods = oxford.OxfordDataset(orr, "train")
        dev = oxford.scan_store(orr, ["t0"], "cuda")
        pin = oxford.scan_store(orr, ["t0"], "pinned")
        result["oxford"]["store"] = {"records": len(dev), "bytes": dev.nbytes,
                                     "mean_points_per_record": float(dev.counts.mean())}
        for S in (int(v) for v in a.oxford_samples.split(",") if v):
            result["oxford"][str(S)] = _oxford_case(ods, dev, pin, S, a.reps)
    line = json.dumps({"datasets": result})
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
