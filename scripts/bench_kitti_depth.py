"""Benchmark of the KITTI camera-frame records and LiDAR depth maps (deepi2p_b200.kitti_depth) on HDL-64-shaped
synthetic scans (synthetic.make_lidar_scan, 64 rings x 2048 azimuths = 131,072 points) and 376 x 1241 images, both
cameras.  Writes BENCH_KITTI_DEPTH.json (or --out):

  - device time per batch of --batch scans (2 x batch maps), by CUDA events around each step, median of --reps:
    the voxel grid, the normals and the nearest-point search (pointprep's existing steps), the record transform,
    the projection (kitti_depth_project_f32: both atomic passes) and the fill (kitti_depth_fill_f32: the EDT's
    column pass, then its row pass with the gather of depths and distances fused in);
  - a whole synthetic sequence of --frames scans from files to files (build_sequence: plan, scan reads, every
    batch, the .npy writes);
  - the numpy oracle's time per scan (both cameras) on one host core;
  - the card name and power limit, read in the same run.

The reference itself cannot be timed here: it needs Open3D.

    python scripts/bench_kitti_depth.py [--batch 64] [--frames 64] [--reps 5] [--out PATH]
"""
import os

os.environ.setdefault("OMP_NUM_THREADS", "1")          # the oracle runs on one host core
os.environ.setdefault("OPENBLAS_NUM_THREADS", "1")
os.environ.setdefault("MKL_NUM_THREADS", "1")

import argparse  # noqa: E402
import json  # noqa: E402
import sys  # noqa: E402
import tempfile  # noqa: E402
import time  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_kitti_build import card  # noqa: E402

H, W = 376, 1241
K = (718.856, 718.856, 607.1928, 185.2157)


def maps_ms(project, fill, reps):
    """Median (project, fill) times: each fill needs the project just before it."""
    out = []
    for _ in range(reps):
        e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        e[0].record()
        project()
        e[1].record()
        fill()
        e[2].record()
        e[2].synchronize()
        out.append((e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2])))
    return tuple(float(v) for v in np.median(np.array(out), axis=0))


def event_ms(fn, reps):
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return float(np.median(out))


def scans(n, seed0=0):
    from deepi2p_b200 import synthetic as syn
    out = []
    for s in range(n):
        sc = syn.make_lidar_scan(seed0 + s, n_rings=64, n_azimuth=2048)
        out.append(np.concatenate([sc["xyz"], sc["intensity"][None]]).astype(np.float32))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--oracle-scans", type=int, default=1)
    ap.add_argument("--out", default=os.path.join(ROOT, "BENCH_KITTI_DEPTH.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_kitti_depth needs a CUDA device")
    import oracle_kitti_depth as okd
    from deepi2p_b200 import _native, kitti_depth as kd, pointprep, synthetic as syn
    from deepi2p_b200._native import _ptr, _stream_ptr
    from deepi2p_b200.icp import pack_clouds
    lib = _native.load()
    res = dict(card=card(), batch=a.batch, reps=a.reps, image_hw=[H, W], points_per_scan=64 * 2048)
    with tempfile.TemporaryDirectory() as tmp:
        root, vel = os.path.join(tmp, "kitti"), os.path.join(tmp, "velodyne")
        t0 = time.perf_counter()
        data = scans(max(a.batch, a.frames))
        syn.write_kitti_velodyne_root(root, vel, 0, data[:a.frames], [(H, W)] * a.frames, K)
        res["write_root_s"] = time.perf_counter() - t0
        plan = kd.plan_sequence(root, vel, 0)
        S, T = a.batch, 2 * a.batch
        xyz, n = pack_clouds([d[:3] for d in data[:S]])
        inten = torch.zeros((S, xyz.shape[2]), dtype=torch.float32)
        for s in range(S):
            inten[s, :data[s].shape[1]] = torch.from_numpy(data[s][3])
        inten = inten.cuda()
        Pc = np.stack([plan["Pc"][k] for _ in range(S) for k in kd.CAMERAS])
        Kt = np.stack([plan["K"][k] for _ in range(S) for k in kd.CAMERAS])
        Pc_d, K_d = torch.from_numpy(Pc).cuda(), torch.from_numpy(Kt).cuda()
        N = xyz.shape[2]
        maps = kd.depth_maps(xyz, n, Pc, Kt, H, W)                 # warm-up, and the workspace
        recs, m = kd.camera_records(xyz, inten, n, Pc)
        down = pointprep.voxel_downsample(xyz, n, pointprep.VOXEL_SIZE)
        d32 = down["xyz"].to(torch.float32)
        dsc = pointprep.downsample_scans(xyz, inten, n)
        ws = torch.empty(lib.kitti_depth_fill_workspace_bytes(T, H, W), dtype=torch.uint8, device="cuda")
        sp = _stream_ptr()
        out = torch.empty((T, 2, H, W), dtype=torch.float32, device="cuda")
        rec_out = torch.empty((T, 7, N), dtype=torch.float32, device="cuda")

        def project():
            _native.check(lib.kitti_depth_project_f32(_ptr(xyz), N, _ptr(n), S, _ptr(Pc_d), _ptr(K_d), T, H, W,
                                                      _ptr(out), sp), "kitti_depth_project")

        def fill():
            _native.check(lib.kitti_depth_fill_f32(_ptr(xyz), N, _ptr(n), S, _ptr(Pc_d), _ptr(K_d), T, H, W, _ptr(out),
                                                   _ptr(ws), ws.numel(), sp), "kitti_depth_fill")

        def records():
            _native.check(lib.kitti_depth_records_f32(_ptr(dsc["xyz"]), _ptr(dsc["normals"]), _ptr(dsc["intensity"]),
                                                      _ptr(dsc["m_pts"]), N, S, _ptr(Pc_d), T, _ptr(rec_out), sp),
                          "kitti_depth_records")

        project()
        fill()
        torch.cuda.synchronize()
        assert torch.equal(out, maps)
        steps = dict(
            voxel_ms=event_ms(lambda: pointprep.voxel_downsample(xyz, n, pointprep.VOXEL_SIZE), a.reps),
            normals_ms=event_ms(lambda: pointprep.estimate_normals(d32, down["m_pts"]), a.reps),
            nearest_ms=event_ms(lambda: pointprep.nearest(down["xyz"], down["m_pts"], xyz, n), a.reps),
            records_ms=event_ms(records, a.reps))
        steps["project_ms"], steps["fill_ms"] = maps_ms(project, fill, a.reps)
        torch.cuda.synchronize()
        assert torch.equal(out, maps)
        steps["depth_maps_ms"] = event_ms(lambda: kd.depth_maps(xyz, n, Pc, Kt, H, W), a.reps)
        steps["camera_records_ms"] = event_ms(lambda: kd.camera_records(xyz, inten, n, Pc), a.reps)
        res["device_batch"] = dict(scans=S, maps=T, **steps,
                                   maps_per_s=T / ((steps["depth_maps_ms"] + steps["camera_records_ms"]) / 1e3),
                                   map_bytes=T * 2 * H * W * 4, voxels=int(m.sum()))
        res["device_batch"]["fill_write_GBps"] = res["device_batch"]["map_bytes"] / (steps["fill_ms"] / 1e3) / 1e9
        del out, ws, maps, recs
        t0 = time.perf_counter()
        kd.build_sequence(root, vel, 0, batch=a.batch)
        sec = time.perf_counter() - t0
        res["files_to_files"] = dict(scans=a.frames, seconds=sec, scans_per_s=a.frames / sec,
                                     bytes_written=sum(os.path.getsize(os.path.join(d, f))
                                                       for d in kd.output_dirs(root, 0) for f in os.listdir(d)))
        chk = np.load(os.path.join(kd.depth_dir(root, 0, "P2"), "000000.npy"))
        t0 = time.perf_counter()
        o_rec, o_maps = okd.process_sequence(root, vel, 0, plan["Pc"], plan["K"], plan["sizes"],
                                             frames=range(a.oracle_scans))
        res["oracle_s_per_scan"] = (time.perf_counter() - t0) / a.oracle_scans
        res["oracle_equal"] = bool(np.array_equal(o_maps[(0, "P2")], chk) and np.array_equal(
            o_rec[(0, "P3")], np.load(os.path.join(kd.record_dir(root, 0, "P3"), "000000.npy"))))
    print(json.dumps(res))
    with open(a.out, "w") as f:
        f.write(json.dumps(res) + "\n")


if __name__ == "__main__":
    main()
