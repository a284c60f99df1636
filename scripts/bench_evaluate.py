"""Benchmark of scripts/evaluate_dataset.py's per-batch work for each registration method, and of the accuracy entry
point (classifier.prediction_accuracy) alone.  Writes BENCH_EVALUATE.json (or --out):

  - for a synthetic KITTI and Oxford root (synthetic.write_kitti_root / write_oxford_root, 20480 points per sample)
    with the scans in a device scan store, a seeded checkpoint (torch head) and, for icp, a seeded monodepth2 model
    at the 640 x 192 feed size: the wall time per batch of --batches (16 and 64) samples, median of --reps after one
    warm-up, of (a) the whole step (batch assembly from the store, evaluate_dataset.register: classify_batch, the
    method's registration, the poses and costs read back) and (b) register alone on an assembled batch, as samples/s;
  - the accuracy entry point at S = 64, N = 20480 with fine predictions: CUDA events around --launches launches,
    with the bytes it must move (points, predictions, counts) over the data-sheet HBM3 bandwidth as a lower bound;
  - the card name and power limit, read in the same run.

    python scripts/bench_evaluate.py [--batches 16 64] [--reps 3] [--launches 200] [--out BENCH_EVALUATE.json]
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

import evaluate_dataset as ev  # noqa: E402
import oracle_monodepth as om  # noqa: E402
from bench_kitti_build import card  # noqa: E402
from deepi2p_b200 import classifier, kitti, monodepth, network, oxford, synthetic  # noqa: E402

HBM_BYTES_PER_S = 3.35e12            # H100 SXM data sheet


def loaders(dataset, root):
    """fn(items, seed, rng) -> the loader's tuple, reading the scans from a device store of the val list's scans."""
    if dataset == "kitti":
        ds = kitti.KittiDataset(root, ev.MODE)
        store = kitti.scan_store(root, sorted({e[0] for e in ds.entries}), "cuda")
        return len(ds), lambda items, seed, rng: kitti.kitti_batch(ds, items, ev.MODE, seed, rng=rng, store=store)
    ds = oxford.OxfordDataset(root, ev.MODE)
    store = oxford.scan_store(root, list(ds.traversals), "cuda")
    return len(ds), lambda items, seed, rng: oxford.oxford_batch(ds, items, ev.MODE, seed, rng=rng, store=store)


def wall(fn, reps):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t)
    return float(np.median(out))


def methods(dataset, root, batches, reps, depth_model):
    model = network.KeypointDetector(**network.SHAPES[dataset])
    network.load_checkpoint(model, synthetic.seeded_state_dict(model, 3))
    model = model.cuda()
    n, make = loaders(dataset, root)
    rows = []
    for B in batches:
        items = [k % n for k in range(B)]
        rng = np.random.default_rng(0)
        batch = make(items, 1, rng)
        for method in ("lsq", "pnp", "icp"):
            kw = dict(depth_model=depth_model) if method == "icp" else {}
            step = wall(lambda: ev.register(method, model, make(items, 1, rng), 0, 0, **kw), reps)
            reg = wall(lambda: ev.register(method, model, batch, 0, 0, **kw), reps)
            rows.append(dict(dataset=dataset, batch=B, method=method, points=int(batch[0].shape[2]),
                             step_s=step, step_samples_per_s=B / step, register_s=reg,
                             register_samples_per_s=B / reg))
            print(json.dumps(rows[-1]), flush=True)
    return rows


def accuracy_entry(launches, S=64, N=20480):
    rng = np.random.default_rng(0)
    pc = torch.from_numpy(rng.uniform(-30, 30, (S, 3, N)).astype(np.float32)).cuda()
    pc[:, 2].abs_()
    P = torch.eye(4, dtype=torch.float64).repeat(S, 1, 1).cuda()
    K = torch.tensor([[300.0, 0.0, 255.5], [0.0, 300.0, 79.5], [0.0, 0.0, 1.0]], dtype=torch.float64).repeat(S, 1, 1)
    K = K.cuda()
    cp = torch.from_numpy(rng.integers(0, 2, (S, N)).astype(np.int8)).cuda()
    fp = torch.from_numpy(rng.integers(0, 80, (S, N)).astype(np.int32)).cuda()
    for _ in range(10):
        classifier.prediction_accuracy(pc, P, K, 160, 512, cp, fp)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        classifier.prediction_accuracy(pc, P, K, 160, 512, cp, fp)
    e1.record()
    e1.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / launches
    # the same calls captured in a graph (20 per graph): the device time without the host's per-call cost
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s), torch.cuda.graph(graph, stream=s):
        for _ in range(20):
            classifier.prediction_accuracy(pc, P, K, 160, 512, cp, fp)
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    e0.record()
    for _ in range(launches // 20):
        graph.replay()
    e1.record()
    e1.synchronize()
    us_graph = e0.elapsed_time(e1) * 1e3 / (20 * (launches // 20))
    nbytes = S * N * (3 * 4 + 1 + 4) + S * 3 * 4 + S * (12 + 9) * 8
    return dict(S=S, N=N, fine=True, launches=launches, us_per_call_eager=us, us_per_call_graph=us_graph,
                bytes=nbytes, hbm_lower_bound_us=nbytes / HBM_BYTES_PER_S * 1e6,
                note="a call is the wrapper's pose slice copy and the counting kernel; eager adds the host's "
                     "per-call cost when it exceeds the device time")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[16, 64])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--out", default=os.path.join(ROOT, "BENCH_EVALUATE.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_evaluate.py needs a CUDA device")
    res = dict(card=card(), torch=torch.__version__, head="torch", inits=60)
    res["accuracy_entry"] = accuracy_entry(a.launches)
    print(json.dumps(res["accuracy_entry"]), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        kroot, oroot = os.path.join(tmp, "kitti"), os.path.join(tmp, "oxford")
        synthetic.write_kitti_root(kroot, seqs=(0, 9, 10), n_frames=90, seed=5)
        synthetic.write_oxford_root(oroot, seed=5)
        depth_model = monodepth.load_monodepth(om.write_checkpoint(os.path.join(tmp, "monodepth"), seed=7))
        res["methods"] = (methods("kitti", kroot, a.batches, a.reps, depth_model)
                          + methods("oxford", oroot, a.batches, a.reps, depth_model))
    with open(a.out, "w") as f:
        json.dump(res, f)
        f.write("\n")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
