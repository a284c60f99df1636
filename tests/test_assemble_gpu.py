"""Batch assembly on the GPU (deepi2p_b200.assemble) against the numpy oracle (oracle_assemble).

The oracle draws from the same Philox streams and restates the fixed-association fp64 transforms, the key order, the
repeat rule and farthest-point sampling, so indices, coordinates, attributes and node sets must be bit-identical with
the jitter off.  With the jitter on, device log / sin / cos are not correctly rounded, so coordinates agree to one
float32 ulp."""
import numpy as np
import pytest
import torch

import oracle_assemble as oa
from deepi2p_b200 import assemble, point_ops, synthetic

pytestmark = pytest.mark.gpu


def _batch(shape, seeds, **kw):
    smps = [synthetic.make_loader_sample(s, shape, **kw) for s in seeds]
    frames = assemble.pack_frames([(m["frames"], m["frame_T"]) for m in smps])
    return smps, frames


def _check_batch(smps, frames, args, mode, seed, N, Ma, Mb, stream=None):
    a = {k: v for k, v in args.items()}
    a["jitter"] = ()
    out = assemble.assemble_batch(frames, mode, seed, input_pt_num=N, node_a_num=Ma, node_b_num=Mb, rng=5,
                                  stream=stream, **a)
    torch.cuda.synchronize()
    pre = np.asarray(a["pre"])
    for s, smp in enumerate(smps):
        M = assemble.compose(out["Pr"][s], pre)
        ref = oa.assemble_sample(smp["frames"], smp["frame_T"], s, seed, M, N, Ma, Mb, a["voxel_size"],
                                 a["range_max"])
        assert int(out["n_before_resample"][s]) == ref["n_before_resample"], s
        assert np.array_equal(out["src_index"][s].cpu().numpy(), ref["src"]), s
        assert np.array_equal(out["pc"][s].cpu().numpy(), ref["pc"]), s
        assert np.array_equal(out["intensity"][s].cpu().numpy(), ref["intensity"]), s
        assert np.array_equal(out["sn"][s].cpu().numpy(), ref["sn"]), s
        for name in ("node_a", "node_b"):
            assert np.array_equal(out[name + "_idx"][s].cpu().numpy(), ref[name + "_idx"]), (s, name)
            assert np.array_equal(out[name][s].cpu().numpy(), ref[name]), (s, name)
    return out


def test_kitti_batch_voxel_path(cuda):
    smps, frames = _batch("kitti", [1, 2, 3])
    args = assemble.kitti_args(smps[0]["Pc"], smps[0]["Pji"])
    out = _check_batch(smps, frames, args, "train", 17, 20480, 128, 128)
    assert int(frames["n_pts"][:7].sum()) > 2 * 20480          # the voxel step ran
    assert out["P"].shape == (3, 3, 4) and out["P"].dtype == torch.float32
    assert out["flip"].dtype == bool


def test_oxford_batch_range_mask(cuda):
    smps, frames = _batch("oxford", [4, 5], n_azimuth=1024)
    args = assemble.oxford_args(smps[0]["P_cam_pc"])
    out = _check_batch(smps, frames, args, "train", 3, 20480, 128, 128)
    assert (out["sn"] == 0).all()


def test_ragged_batch_repeat_rule_and_full_candidates(cuda):
    smps, frames = _batch("kitti", [6, 7], n_rings=4, n_azimuth=64)
    one = ([(np.array([[1.0], [2.0], [3.0]], dtype=np.float32), np.array([0.5], dtype=np.float32),
             np.array([[0.0], [0.0], [1.0]], dtype=np.float32))], np.eye(4)[None])
    smps.append(dict(frames=one[0], frame_T=one[1]))
    frames = assemble.pack_frames([(m["frames"], m["frame_T"]) for m in smps])
    args = assemble.kitti_args(np.eye(4))
    _check_batch(smps, frames, args, "val_random_Ry", 9, 2048, 256, 32)     # 8 Ma = N


def test_fps_duplicates_and_dtypes(cuda):
    rng = np.random.default_rng(2)
    dup = np.repeat(rng.normal(0, 1, (3, 300)), 4, axis=1)
    lat = np.stack(np.meshgrid(*([np.arange(10.0)] * 3), indexing="ij")).reshape(3, -1)
    for pts in (dup, lat):
        for dt in (np.float32, np.float64):
            p = pts.astype(dt)
            x = torch.from_numpy(p[None].copy()).cuda()
            idx, nodes = assemble.farthest_point_sample(x, None, 200, start=torch.tensor([5], dtype=torch.int32,
                                                                                         device="cuda"))
            ri, rn = oa.fps(p, 200, 5)
            assert np.array_equal(idx[0].cpu().numpy(), ri) and np.array_equal(nodes[0].cpu().numpy(), rn)


@pytest.mark.parametrize("n", [8193, 20480, 65536])
def test_fps_cluster_path(cuda, n):
    rng = np.random.default_rng(n)
    S, k = 2, 96
    pts = rng.normal(0, 20, (S, 3, n)).astype(np.float32)
    n_pts = torch.tensor([n, n - 100], dtype=torch.int32, device="cuda")
    for dt in (np.float32, np.float64):
        x = torch.from_numpy(pts.astype(dt)).cuda()
        idx, nodes = assemble.farthest_point_sample(x, n_pts, k)
        for s in range(S):
            m = int(n_pts[s])
            ri, rn = oa.fps(pts[s, :, :m].astype(dt), k, 0)
            assert np.array_equal(idx[s].cpu().numpy(), ri), (dt, s)
            assert np.array_equal(nodes[s].cpu().numpy(), rn), (dt, s)


def test_second_stream(cuda):
    smps, frames = _batch("kitti", [8], n_rings=16, n_azimuth=256)
    args = assemble.kitti_args(smps[0]["Pc"])
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        _check_batch(smps, frames, args, "train", 21, 4096, 64, 64, stream=st)


def test_jitter_within_one_ulp(cuda):
    rng = np.random.default_rng(4)
    S, n, N = 3, 5000, 4096
    x = rng.normal(0, 10, (S, 3, n)).astype(np.float32)
    it = rng.random((S, n), dtype=np.float32)
    sn = rng.normal(0, 1, (S, 3, n)).astype(np.float32)
    cnt = torch.tensor([n, 3000, 1], dtype=torch.int32, device="cuda")
    out = assemble.resample(torch.from_numpy(x).cuda(), torch.from_numpy(it).cuda(), torch.from_numpy(sn).cuda(), cnt,
                            N, 77, jitter=("pc", "sn", "intensity"))
    for s in range(S):
        m = int(cnt[s])
        src = oa.resample_index(m, N, s, 77)
        assert np.array_equal(out["src"][s].cpu().numpy(), src)
        for key, base, stream in (("pc", x[s][:, src], oa.STREAM_JITTER_PC), ("sn", sn[s][:, src], oa.STREAM_JITTER_SN),
                                  ("intensity", it[s][None, src], oa.STREAM_JITTER_INTENSITY)):
            z = oa.normals3(N, s, stream, 77)[:base.shape[0]]
            want = base + oa.jitter(z)
            got = out[key][s].cpu().numpy()
            ulp = np.spacing(np.maximum(np.abs(want), np.abs(got)))
            assert (np.abs(got - want) <= ulp).all(), key
            assert np.abs(got.astype(np.float64) - base).max() <= 0.05 + np.spacing(np.float32(60.0)), key


def test_farthest_sampler_dropin(cuda):
    from test_assemble_cpu import _RefFarthestSampler
    rng = np.random.default_rng(9)
    for dim in (2, 3):
        pts = rng.normal(0, 5, (dim, 1024)).astype(np.float32)
        for seed in range(2):
            np.random.seed(seed)
            rp, ri = _RefFarthestSampler(dim).sample(pts, 128)
            after_ref = np.random.randint(1 << 30)
            np.random.seed(seed)
            gp, gi = assemble.FarthestSampler(dim).sample(pts, 128)
            assert np.random.randint(1 << 30) == after_ref          # the same draws from np.random
            assert gp.dtype == np.float64 and gi.dtype == np.int64
            assert np.array_equal(gi, ri) and np.array_equal(gp, rp)
    K = np.array([[300.0, 0, 256], [0, 300, 80], [0, 0, 1]])
    pts = np.abs(rng.normal(0, 5, (3, 800))) + np.array([[0], [0], [5.0]])
    np.random.seed(3)
    gp, gi = assemble.ProjectiveFarthestSampler().sample(pts, 64, K)
    np.random.seed(3)
    p2 = np.dot(K, pts)
    _, ri = _RefFarthestSampler(2).sample(p2[0:2] / p2[2:], 64)
    assert np.array_equal(gi, ri) and np.array_equal(gp, pts[:, ri])


def test_nodes_feed_cluster_assign(cuda):
    smps, frames = _batch("kitti", [10, 11], n_rings=16, n_azimuth=256)
    out = assemble.assemble_batch(frames, "train", 1, input_pt_num=4096, node_a_num=64, node_b_num=64, rng=0,
                                  **assemble.kitti_args(smps[0]["Pc"]))
    res = point_ops.cluster_assign_forward(out["pc"], out["node_a"], k=1)
    torch.cuda.synchronize()
    assert res["count"].sum(1).tolist() == [4096, 4096]
    # every node is one of the points, so its own cluster is never empty
    assert (res["count"] > 0).all()
