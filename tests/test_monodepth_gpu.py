"""Monodepth depth clouds on the device (csrc/monodepth.cu, deepi2p_b200/monodepth.py): the Lanczos resize against
Pillow and torch's normalisation, the depth against torch's upsample and reciprocal, the back-projection, the device
scale, the whole pipeline against the float64 oracle, and a synthetic hand-off root end to end through
save_depth_map.py and register_dir.py."""
import os
import subprocess
import sys
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from PIL import Image

import oracle_monodepth as om
from deepi2p_b200 import handoff, icp, imageprep, monodepth, synthetic

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _frames(S, h, w, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for _ in range(S)]


@pytest.mark.parametrize("S,h,w", [(64, 384, 640), (64, 160, 512), (64, 160, 320), (5, 37, 91), (3, 1, 5),
                                   (2, 192, 640), (2, 500, 1300)])
def test_resize_is_pillow_and_torchs_normalisation(S, h, w):
    imgs = _frames(S, h, w, h * 1000 + w)
    x = monodepth.resize_normalise(imageprep.pack_images(imgs), 192, 640)
    ref = np.stack([np.asarray(Image.fromarray(a).convert("RGB").resize((640, 192), Image.LANCZOS)) for a in imgs])
    t = torch.from_numpy(ref).permute(0, 3, 1, 2).contiguous().float().div(255)     # transforms.ToTensor
    want = (t.cuda() - 0.45) / 0.225                                                    # ResnetEncoder.forward
    assert torch.equal(x, want)


def test_resize_reads_offsets_and_rejects_ragged_frames():
    imgs = _frames(3, 50, 70, 9)
    pk = imageprep.pack_images([imgs[0], np.zeros((4, 4, 3), np.uint8)] + imgs[1:])
    sub = dict(data=pk["data"], offsets=pk["offsets"][[0, 2, 3]], shapes=pk["shapes"][[0, 2, 3]])
    x = monodepth.resize_normalise(sub, 64, 96)
    y = monodepth.resize_normalise(imageprep.pack_images(imgs), 64, 96)
    assert torch.equal(x, y)
    with pytest.raises(ValueError, match="one size"):
        monodepth.resize_normalise(pk, 64, 96)


def _ulps(a, b):
    a, b = a.cpu().numpy(), b.cpu().numpy()
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    return int(np.abs(ia - ib).max()), int((ia != ib).sum())


class _Fixed(torch.nn.Module):
    """A stand-in network returning a given disparity, so kernel 2 can be checked on chosen inputs."""

    def __init__(self, disp):
        super().__init__()
        self.disp = disp
        self.feed_height, self.feed_width = disp.shape[2], disp.shape[3]

    def forward(self, x):
        return self.disp


@pytest.mark.parametrize("H,W,h,w", [(384, 640, 192, 640), (160, 512, 192, 640), (160, 320, 192, 640),
                                     (37, 91, 64, 96), (64, 96, 64, 96), (1, 5, 32, 32)])
def test_depth_cloud_and_scale(H, W, h, w):
    S = 4
    rng = np.random.default_rng(H + W)
    disp = torch.from_numpy(rng.uniform(0.005, 1.0, (S, 1, h, w)).astype(np.float32)).cuda()
    frames = [synthetic.make_icp_frame(s, "oxford") for s in range(S)]
    K = np.stack([f["K"] for f in frames]).astype(np.float32)
    K[:, 0, 2], K[:, 1, 2] = W / 2, H / 2
    P = np.stack([f["P_gt"] for f in frames])
    src, n = icp.pack_clouds([f["src"] for f in frames])
    images = imageprep.pack_images(_frames(S, H, W, 1))
    K64 = K.astype(np.float64).reshape(S, 9)
    d = monodepth.depth_clouds(_Fixed(disp).eval(), images, monodepth.k_inverse(K), src=src, n_pts=n, P_gt=P, K=K64,
                               depth=True)
    want = torch.reciprocal(F.interpolate(disp, (H, W), mode="bilinear", align_corners=False))[:, 0]
    mx, cnt = _ulps(d["depth"], want)
    assert mx == 0, f"{cnt} depths differ, by up to {mx} ulp"
    pc, depth = d["pc"].cpu().numpy(), d["depth"].cpu().numpy()
    for s in range(S):
        ref = om.convert_depth_to_pointcloud(depth[s][:, :, None], K[s])
        # any summation order of the three products: <= 2 ulp of sum |K^-1_ij v_j|
        Ki = np.linalg.inv(K[s]).astype(np.float64)
        y, x = np.divmod(np.arange(H * W), W)
        v = np.stack([depth[s].reshape(-1) * x, depth[s].reshape(-1) * y, depth[s].reshape(-1).astype(np.float64)])
        mag = np.abs(Ki) @ np.abs(v)
        assert (np.abs(pc[s] - ref) <= 2 * np.spacing(mag)).all()
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)
            want_scale = icp.calibrate_scale(frames[s]["src"], P[s], K64[s].reshape(3, 3), H, W, pc[s])
        got_scale = float(d["scale"][s])
        if np.isnan(want_scale):                    # no LiDAR point inside a tiny image: numpy's empty mean
            assert np.isnan(got_scale)
        else:
            assert abs(got_scale - want_scale) <= 1e-12 * abs(want_scale)
        np.testing.assert_array_equal(d["tgt"][s].cpu().numpy(), (pc[s] * got_scale).astype(np.float32))


def test_depth_clouds_match_the_float64_oracle():
    """TF32 off.  The input is exact (the test above), so the difference is the float32 network's: about 23
    convolutions of up to 4608 products each, whose rounding (u = 2^-24 per operation, growing like sqrt(K) u per
    layer) stays near 2^-16 of the disparity; the budget is 2^-12 relative on the depth, i.e. on every coordinate
    relative to the depth of its point."""
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        enc, dec = om.seeded_checkpoint(11, 64, 128)
        model = monodepth.DepthNet(64, 128)
        model.load_state_dict({k: v for k, v in {**enc, **dec}.items() if torch.is_tensor(v)})
        model = model.cuda().eval()
        S, H, W = 3, 90, 150
        imgs = _frames(S, H, W, 4)
        K = np.array([[120.0, 0, 75.0], [0, 120.0, 45.0], [0, 0, 1]], np.float32)
        d = monodepth.depth_clouds(model, imageprep.pack_images(imgs), monodepth.k_inverse(np.stack([K] * S)))
        for s in range(S):
            u8 = om.lanczos_resize(imgs[s], 128, 64)
            x = (torch.from_numpy(u8).permute(2, 0, 1)[None].double() / 255 - 0.45) / 0.225
            disp = om.depth_net({**enc, **dec}, x)
            depth = 1.0 / F.interpolate(disp, (H, W), mode="bilinear", align_corners=False)[0, 0]
            ref = om.convert_depth_to_pointcloud(depth.numpy()[:, :, None], K.astype(np.float64))
            err = np.abs(d["pc"][s].cpu().numpy() - ref) / ref[2]
            assert err.max() <= 2.0 ** -12, err.max()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def test_images_from_batch_rounds_like_the_script():
    img = torch.rand(2, 3, 20, 30, device="cuda") * 255
    pk = monodepth.images_from_batch(img)
    want = img.round().to(torch.uint8).permute(0, 2, 3, 1).contiguous()
    for s in range(2):
        o = int(pk["offsets"][s])
        assert torch.equal(pk["data"][o:o + 1800].view(20, 30, 3), want[s])


def _cli(script, *args):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", script), *args], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return r.stdout


def test_end_to_end_handoff_root(tmp_path):
    import cv2
    root = tmp_path / "run"
    data, vis, md = str(root / "data"), str(root / "visualization"), str(root / "monodepth")
    frames = synthetic.write_icp_handoff(data, str(tmp_path / "unused"), list(range(6)), "oxford")
    os.makedirs(vis)
    rng = np.random.default_rng(0)
    yy, xx = np.mgrid[0:384, 0:640]
    for i, name in enumerate(sorted(frames)):
        np.save(os.path.join(data, name + "_K.npy"), frames[name]["K"].astype(np.float32))   # the reference's dtype
        base = np.stack([xx * 0.3 + 40 * i, yy * 0.5, (xx + yy) * 0.2], -1) % 256
        img = np.clip(base + rng.normal(0, 12, base.shape), 0, 255).astype(np.uint8)
        cv2.imwrite(os.path.join(vis, name + "_img.png"), cv2.cvtColor(img, cv2.COLOR_RGB2BGR))
    model_dir = om.write_checkpoint(str(tmp_path / "model"), seed=7)
    # one batch everywhere: cuDNN may choose another algorithm for another batch size
    _cli("save_depth_map.py", str(root), "--depth-model", model_dir)
    out_a, out_b = str(tmp_path / "a"), str(tmp_path / "b")
    _cli("register_dir.py", data, "--H", "384", "--W", "640", "--method", "icp", "--monodepth", md, "--out", out_a)
    _cli("register_dir.py", data, "--H", "384", "--W", "640", "--method", "icp", "--depth-model", model_dir,
         "--out", out_b)

    names = sorted(frames)
    model = monodepth.load_monodepth(model_dir)
    images = imageprep.read_png_batch([os.path.join(vis, n + "_img.png") for n in names])
    recs = [handoff.load_record(data, n) for n in names]
    K_raw = np.stack([np.load(os.path.join(data, n + "_K.npy")) for n in names])
    src, n_pts = icp.pack_clouds([r[0] for r in recs])
    P = np.stack([r[3] for r in recs])
    runs = [monodepth.depth_clouds(model, images, monodepth.k_inverse(K_raw), src=src, n_pts=n_pts, P_gt=P,
                                   K=K_raw.astype(np.float64).reshape(-1, 9)) for _ in range(2)]
    for k in ("pc", "scale", "tgt"):
        assert torch.equal(runs[0][k], runs[1][k]), k
    pc = runs[0]["pc"].cpu().numpy()
    same = []
    for s, name in enumerate(names):
        on_disk = np.load(os.path.join(md, name + "_pc.npy"))
        assert on_disk.dtype == np.float64
        np.testing.assert_array_equal(on_disk, pc[s])
        host = icp.calibrate_scale(recs[s][0], P[s], recs[s][2], 384, 640, on_disk)
        dev = float(runs[0]["scale"][s])
        assert abs(dev - host) <= 1e-12 * abs(host)
        same.append(dev == host)
    Pa, Pb = np.load(os.path.join(out_a, "P_pred_all_np.npy")), np.load(os.path.join(out_b, "P_pred_all_np.npy"))
    ca, cb = np.load(os.path.join(out_a, "cost_all_np.npy")), np.load(os.path.join(out_b, "cost_all_np.npy"))
    print(f"{sum(same)} of {len(same)} frames have bit-equal host and device scales")
    for s in np.flatnonzero(same):
        np.testing.assert_array_equal(Pa[s], Pb[s])
        assert ca[s] == cb[s]
