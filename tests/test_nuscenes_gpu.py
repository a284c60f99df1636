"""The nuScenes point side on the GPU (assemble_batch(**nuscenes_args): ego-box removal, fp64 sweep accumulation, the
voxel step on the fp64 cloud) against oracle_nuscenes, its poses, and one nuscenes_batch call on a mini dataroot.

With the jitter off, counts, indices, coordinates, intensities and node sets must be bit-identical; with it on, device
log / sin / cos are not correctly rounded, so values agree to one float32 ulp."""
import os

import numpy as np
import pytest
import torch

import oracle_nuscenes as onu
from deepi2p_b200 import assemble, imageprep, nuscenes, synthetic

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_small.npz")


def _frames(smps):
    return assemble.pack_frames([(m["frames"], m["frame_T"]) for m in smps])


def _run(smps, mode, seed, N, Ma, Mb, jitter=(), stream=None):
    a = assemble.nuscenes_args(np.stack([m["P_cam_pc"] for m in smps]))
    a["jitter"] = jitter
    out = assemble.assemble_batch(_frames(smps), mode, seed, input_pt_num=N, node_a_num=Ma, node_b_num=Mb, rng=5,
                                  stream=stream, **a)
    torch.cuda.synchronize()
    return out


def _check(smps, mode, seed, N=20480, Ma=128, Mb=128, stream=None):
    out = _run(smps, mode, seed, N, Ma, Mb, stream=stream)
    for s, smp in enumerate(smps):
        ref = onu.assemble_sample(smp["frames"], smp["frame_T"], s, seed, out["Pr"][s], N, Ma, Mb)
        assert int(out["n_before_resample"][s]) == ref["n_before_resample"], s
        assert np.array_equal(out["src_index"][s].cpu().numpy(), ref["src"]), s
        assert np.array_equal(out["pc"][s].cpu().numpy(), ref["pc"]), s
        assert np.array_equal(out["intensity"][s].cpu().numpy(), ref["intensity"]), s
        assert not out["sn"][s].any(), s
        for name in ("node_a", "node_b"):
            assert np.array_equal(out[name + "_idx"][s].cpu().numpy(), ref[name + "_idx"]), (s, name)
            assert np.array_equal(out[name][s].cpu().numpy(), ref[name]), (s, name)
    return out


def test_full_batch_voxel_path(cuda):
    smps = [synthetic.make_nuscenes_sample(s) for s in range(12)]
    out = _check(smps, "val_random_Ry", 11)
    assert all(sum(f[0].shape[1] for f in m["frames"]) > 2 * 20480 for m in smps)     # every sample voxelised
    assert out["pc"].shape == (12, 3, 20480) and out["P"].shape == (12, 3, 4)


def test_ragged_batch_without_voxel_step(cuda):
    smps = [synthetic.make_nuscenes_sample(20, n_sweeps=1),                   # the anchor alone, no voxel step
            synthetic.make_nuscenes_sample(21, n_sweeps=3, n_rings=4),         # 3 fp64 sweeps rounded to float32,
            synthetic.make_nuscenes_sample(22, n_sweeps=4, n_rings=8),         # fewer than N points (repeat rule)
            synthetic.make_nuscenes_sample(23, n_sweeps=3)]                   # a scene end: voxelised
    n = [sum(f[0].shape[1] for f in m["frames"]) for m in smps]
    assert n[0] < 2 * 20480 and n[1] < 20480 and 20480 < n[2] < 2 * 20480 < n[3]
    _check(smps, "test", 4)


def test_ego_box_edges(cuda):
    f32 = np.float32
    edge = np.array([-0.8, 0.8, -2.7, 2.7], dtype=f32)
    xs = np.concatenate([edge[:2], np.nextafter(edge[:2], f32(0)), np.nextafter(edge[:2], f32(10) * edge[:2]),
                         [f32(0.0)]])
    ys = np.concatenate([edge[2:], np.nextafter(edge[2:], f32(0)), np.nextafter(edge[2:], f32(10) * edge[2:]),
                         [f32(0.0)]])
    X, Y = np.meshgrid(xs, ys)
    pts = np.stack([X.ravel(), Y.ravel(), np.full(X.size, 0.25, f32)]).astype(f32)
    smp = synthetic.make_nuscenes_sample(30, n_sweeps=2, n_rings=2, n_azimuth=64)
    frames = [(np.concatenate([x, pts], 1), np.concatenate([it, np.arange(pts.shape[1], dtype=f32)]), None)
              for x, it, _ in smp["frames"]]
    smp["frames"] = frames
    keep = onu.ego_mask(frames[0][0])
    assert keep[-pts.shape[1]:].sum() == pts.shape[1] - 3 * 3     # the 3 x 3 strictly inside are dropped
    _check([smp], "test", 2, N=256, Ma=16, Mb=8)
    fr = _frames([smp])
    xyz, inten, _, _, cnt = assemble.accumulate(fr["xyz"], fr["intensity"], None, fr["n_pts"], fr["frame_sample"],
                                                fr["frame_T"], exclude_box=onu.EGO_BOX, f64=True)
    x64, it = onu.accumulate(frames, smp["frame_T"])
    assert xyz.dtype == torch.float64 and int(cnt[0]) == x64.shape[1]
    assert np.array_equal(xyz[0, :, :x64.shape[1]].cpu().numpy(), x64)
    assert np.array_equal(inten[0, :x64.shape[1]].cpu().numpy(), it)


def test_second_stream_and_repeatability(cuda):
    smps = [synthetic.make_nuscenes_sample(s, n_sweeps=5) for s in (40, 41)]
    a = _run(smps, "train", 8, 20480, 128, 128)
    st = torch.cuda.Stream()
    b = _check(smps, "test", 8, stream=st)
    c = _run(smps, "test", 8, 20480, 128, 128)
    for k in ("pc", "intensity", "node_a", "node_b", "src_index"):
        assert torch.equal(b[k], c[k]), k
    assert a["pc"].shape == c["pc"].shape


def test_jitter_within_one_ulp(cuda):
    smps = [synthetic.make_nuscenes_sample(s, n_sweeps=7) for s in (50, 51)]
    out = _run(smps, "train", 6, 20480, 128, 128, jitter=("pc", "intensity"))
    for s, smp in enumerate(smps):
        ref = onu.assemble_sample(smp["frames"], smp["frame_T"], s, 6, out["Pr"][s], 20480, 128, 128,
                                  jitter_channels=("pc", "intensity"))
        assert np.array_equal(out["src_index"][s].cpu().numpy(), ref["src"])
        g = out["intensity"][s].cpu().numpy()
        assert (np.abs(g - ref["intensity"]) <= np.spacing(np.abs(ref["intensity"]))).all(), s
        # one ulp in a jittered coordinate moves every rotated coordinate by at most one ulp of the point's largest
        g = out["pc"][s].cpu().numpy()
        assert (np.abs(g - ref["pc"]) <= 2 * np.spacing(np.abs(ref["pc"]).max(0))).all(), s


@pytest.mark.parametrize("mode", ["val_random_Ry", "train"])
def test_pose_is_a_rotation_about_z(cuda, mode):
    smps = [synthetic.make_nuscenes_sample(s, n_sweeps=1, n_rings=8) for s in (60, 61, 62, 63)]
    out = _run(smps, mode, 1, 20480, 128, 128)
    Pr = out["Pr"]
    assert np.array_equal(Pr[:, 2], np.tile([0.0, 0.0, 1.0, 0.0], (4, 1)))
    assert np.array_equal(Pr[:, :2, 2:], np.zeros((4, 2, 2)))
    assert np.allclose(np.linalg.det(Pr[:, :3, :3]), 1.0) and not np.allclose(Pr[:, :3, :3], np.eye(3))
    for s, m in enumerate(smps):
        assert np.allclose(out["P44"][s] @ Pr[s], m["P_cam_pc"], rtol=0, atol=1e-14)
    assert not out["flip"].any()


def _jpeg_1600x900():
    g = np.load(GOLDEN)
    so = np.concatenate([[0], np.cumsum(g["stream_lens"])])
    i = int(np.nonzero((g["shapes"][:, 0] == 900) & (g["shapes"][:, 1] == 1600))[0][0])
    return g["streams"][so[i]:so[i + 1]].tobytes()


def test_nuscenes_batch_on_a_mini_dataroot(cuda, tmp_path):
    blob = _jpeg_1600x900()
    items = synthetic.write_nuscenes_dataroot(str(tmp_path), [(30, 14), (6, 0), (14, 13)], seed=3, jpeg=blob)
    tab = nuscenes.Tables(str(tmp_path), "v1.0-mini")
    info = nuscenes.load_dataset_info(str(tmp_path / "dataset_info.list"))
    pc, inten, sn, na, nb, P, img, K, t_ij = nuscenes.nuscenes_batch(tab, info, "val_random_Ry", 7, rng=2)
    torch.cuda.synchronize()
    S = len(items)
    assert pc.shape == (S, 3, 20480) and inten.shape == (S, 1, 20480) and sn.shape == (S, 3, 20480)
    assert na.shape == (S, 3, 128) and nb.shape == (S, 3, 128) and not sn.any()
    assert P.shape == (S, 3, 4) and P.dtype == torch.float32
    assert img.shape == (S, 3, 160, 320) and img.dtype == torch.float32
    assert K.shape == (S, 3, 3) and t_ij.shape == (S, 3) and t_ij.dtype == torch.float32
    dec = imageprep.decode_jpeg_batch([blob] * S)
    raw_K = np.stack([nuscenes.camera_K(tab, tab.get("sample_data", it[1]["CAM_FRONT"][0])) for it in items])
    ref = imageprep.assemble_images(dec, K=raw_K, mode="val_random_Ry", **imageprep.nuscenes_image_args())
    assert torch.equal(img, ref["img"])
    # the centred crop moves the principal point by the same offsets whichever camera was drawn
    assert np.array_equal(K[:, 1].numpy(), ref["K"][:, 1].numpy()) and np.array_equal(K[:, 0, 0], ref["K"][:, 0, 0])
    for s, it in enumerate(info):
        walk = nuscenes.sweep_walk(tab, it[0])
        assert len(walk) == [7, 2, 4][s]
    assert torch.isfinite(pc).all() and torch.isfinite(P).all()
