"""List-scheduling model of the solver's persistent grid: W workers (resident warps), problems taken in queue order
(chunks of samples, rank-major inside a chunk), each problem busy for `evals` passes.  Compares scheduling orders by
the modelled makespan and the modelled tail (queue empty -> last finish), in passes.  CPU tool over the .npz written by
tests/tools/dump_solve_lengths.py, or over a directory written by bench.py --dump-outputs (init.npy, stats.npy)."""
import argparse
import heapq
import os

import numpy as np


def queue_order(rank_key, chunk):
    """rank_key [S,I]: larger = predicted longer.  Returns the list of (s, i) in queue order."""
    S, I = rank_key.shape
    perm = np.argsort(-rank_key, axis=1, kind="stable")            # perm[s][r] = init of rank r
    order = []
    nchunks = (S + chunk - 1) // chunk
    chunk = (S + nchunks - 1) // nchunks
    for s0 in range(0, S, chunk):
        gc = min(chunk, S - s0)
        for r in range(I):
            for s in range(s0, s0 + gc):
                order.append((s, perm[s, r]))
    return order


def simulate(evals, order, W):
    t_free = [0.0] * W
    heapq.heapify(t_free)
    last_start = 0.0
    end = 0.0
    for (s, i) in order:
        t = heapq.heappop(t_free)
        last_start = max(last_start, t)
        f = t + float(evals[s, i])
        end = max(end, f)
        heapq.heappush(t_free, f)
    return end, end - last_start


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("npz", help="dump_solve_lengths.py .npz or bench.py --dump-outputs directory")
    ap.add_argument("--workers", type=int, default=2640)       # H100: 132 SMs x 2 CTAs x 10 warps
    ap.add_argument("--chunk", type=int, default=86)          # the solver's chunk for 512 x 60 on an H100
    a = ap.parse_args()
    d = {k: np.load(os.path.join(a.npz, k + ".npy")) for k in ("init", "stats")} if os.path.isdir(a.npz) else np.load(a.npz)
    init, stats = d["init"], d["stats"]
    evals = stats[..., 1].astype(np.float64)
    S, I = evals.shape
    ry = init[..., 0]
    dt = init[..., 1:4] - init[..., 1:4].mean(axis=1, keepdims=True)
    keys = {
        "heading distance (shipped)": np.abs(ry - ry.mean(axis=1, keepdims=True)),
        "true length (bound)": evals,
        "random": np.random.default_rng(0).random((S, I)),
        "queue = init index": -np.arange(I)[None, :].repeat(S, 0).astype(np.float64),
        "translation offset norm": np.linalg.norm(dt, axis=2),
    }
    if "cost0" in d:                                                  # dump_solve_lengths.py only
        keys.update({"cost at init": d["cost0"], "gradient max-norm at init": d["gnorm0"]})
    ideal = evals.sum() / a.workers
    print("S %d I %d  passes mean %.1f max %d  ideal makespan %.1f passes" % (S, I, evals.mean(), evals.max(), ideal))
    from scipy.stats import spearmanr
    for name, k in keys.items():
        rho = np.mean([spearmanr(k[s], evals[s]).statistic for s in range(S)])
        for chunk in (a.chunk, S):
            end, tail = simulate(evals, queue_order(k, chunk), a.workers)
            print("%-32s chunk %4d  rank corr %+.2f  makespan %.1f (x%.3f of ideal)  tail %.1f passes" % (name, chunk, rho, end, end / ideal, tail))


if __name__ == "__main__":
    main()
