"""Monodepth depth clouds, host side (deepi2p_b200/monodepth.py, oracle_monodepth): the numpy Lanczos against Pillow,
the kernel's coefficient tables, strict checkpoint loading, DepthNet against the independent float64 composition,
the back-projection, the ABI's argument checks and the CLIs' refusals.  No GPU needed."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from PIL import Image

import oracle_monodepth as om
from deepi2p_b200 import monodepth, synthetic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (h, w) -> the 640 x 192 feed: Oxford keeps its width (only the vertical pass), KITTI and nuScenes need both passes,
# then odd sizes, a 1-pixel side, and a downscale on both axes
SHAPES = [(384, 640), (160, 512), (160, 320), (37, 91), (1, 5), (7, 1), (500, 1300)]


@pytest.mark.parametrize("hw", SHAPES)
def test_oracle_lanczos_is_pillow(hw):
    rng = np.random.default_rng(hw[0] * 7919 + hw[1])
    for fw, fh in ((640, 192), (91, 37)):
        img = rng.integers(0, 256, hw + (3,), dtype=np.uint8)
        want = np.asarray(Image.fromarray(img).convert("RGB").resize((fw, fh), Image.LANCZOS))
        np.testing.assert_array_equal(om.lanczos_resize(img, fw, fh), want)


@pytest.mark.parametrize("n_in,n_out", [(384, 192), (512, 640), (320, 640), (160, 192), (91, 640), (37, 192),
                                        (1, 192), (1300, 640), (640, 91)])
def test_kernel_tables_are_the_oracles(n_in, n_out):
    tab = monodepth.lanczos_table(n_in, n_out)
    xmin, xsize, kk = om.lanczos_coeffs(n_in, n_out)
    np.testing.assert_array_equal(tab[:, 0], xmin)
    np.testing.assert_array_equal(tab[:, 1], xsize)
    np.testing.assert_array_equal(tab[:, 2:], kk)


def test_feed_constants_are_torchs_float32_scalars():
    # ToTensor: uint8 -> float32 / 255 (true division on the CPU); the device then multiplies by 1 / 0.225 in float32
    u = np.arange(256, dtype=np.uint8)
    np.testing.assert_array_equal(torch.from_numpy(u).float().div(255).numpy(), u.astype(np.float32) / np.float32(255))
    assert monodepth.FEED_SUB == np.float32(0.45)
    assert monodepth.FEED_MUL == np.float32(np.float32(1.0) / np.float32(0.225))


def test_checkpoint_loads_strictly_and_reads_the_feed_size(tmp_path):
    d = om.write_checkpoint(str(tmp_path / "m"), seed=3, height=128, width=416)
    model = monodepth.load_monodepth(d, device="cpu")
    assert (model.feed_height, model.feed_width) == (128, 416) and not model.training
    enc, dec = om.seeded_checkpoint(3, 128, 416)
    sd = model.state_dict()
    want = {k: v for k, v in {**enc, **dec}.items() if torch.is_tensor(v)}
    assert sorted(sd) == sorted(want)
    for k, v in want.items():
        assert torch.equal(sd[k], v), k


@pytest.mark.parametrize("edit", ["missing", "extra", "feed"])
def test_checkpoint_errors(tmp_path, edit):
    enc, dec = om.seeded_checkpoint(0)
    if edit == "missing":
        del dec["decoder.12.conv.bias"]
    elif edit == "extra":
        enc["encoder.layer5.0.conv1.weight"] = torch.zeros(1)
    else:
        enc["height"] = 200
    os.makedirs(tmp_path / "m")
    torch.save(enc, tmp_path / "m" / "encoder.pth")
    torch.save(dec, tmp_path / "m" / "depth.pth")
    with pytest.raises((RuntimeError, ValueError), match={"missing": "Missing key", "extra": "Unexpected key",
                                                          "feed": "multiple of 32"}[edit]):
        monodepth.load_monodepth(str(tmp_path / "m"), device="cpu")


def test_depthnet_float64_matches_the_oracle():
    enc, dec = om.seeded_checkpoint(5, 64, 96)
    model = monodepth.DepthNet(64, 96)
    model.load_state_dict({k: v for k, v in {**enc, **dec}.items() if torch.is_tensor(v)})
    model = model.double().eval()
    x = torch.from_numpy(np.random.default_rng(1).normal(0, 1, (2, 3, 64, 96)))
    with torch.no_grad():
        got = model(x)
    want = om.depth_net({**enc, **dec}, x)
    assert got.shape == (2, 1, 64, 96)
    err = ((got - want).abs() / want.abs()).max().item()
    assert err <= 1e-12, err


def test_oracle_back_projection_is_the_scripts_formula():
    rng = np.random.default_rng(2)
    H, W = 37, 53
    depth = rng.uniform(0.5, 80, (H, W, 1)).astype(np.float32)
    K = np.array([[482.4145, 0, 321.894], [0, 482.4145, 194.204], [0, 0, 1]], np.float32)
    pc = om.convert_depth_to_pointcloud(depth, K)
    assert pc.dtype == np.float64 and pc.shape == (3, H * W)
    Ki = np.linalg.inv(K).astype(np.float64)
    np.testing.assert_array_equal(monodepth.k_inverse(K[None]), Ki.reshape(1, 9))
    for i in rng.integers(0, H * W, 50):
        y, x = divmod(int(i), W)
        d = np.float64(depth[y, x, 0])
        np.testing.assert_array_equal(pc[:, i], Ki @ np.array([d * x, d * y, d]))


def test_abi_rejects_bad_arguments_without_a_device():
    from deepi2p_b200 import _native
    lib = _native.load()
    buf = ctypes.create_string_buffer(64)
    a = ctypes.addressof(buf)
    # a table for an axis that keeps its size
    rc = lib.monodepth_resize_f32(a, None, 1, 4, 4, 4, 8, a, 3, a, 3, 0.45, 4.4, None, 0, a, None)
    assert rc == -22 and b"exactly" in lib.dib_last_error()
    rc = lib.monodepth_resize_f32(a, None, 1, 4, 4, 8, 8, a, 3, a, 3, 0.45, 4.4, None, 0, a, None)
    assert rc == -22 and b"tmp" in lib.dib_last_error()
    rc = lib.monodepth_cloud_f32(a, 1, 4, 4, 8, 8, a, None, None, None, None, 0, None, None, None, None, None, 0, None)
    assert rc == -22 and b"no output" in lib.dib_last_error()
    rc = lib.monodepth_cloud_f32(a, 1, 4, 4, 8, 8, a, None, a, None, None, 0, None, None, None, a, None, 0, None)
    assert rc == -22 and b"needs the scale" in lib.dib_last_error()
    assert lib.monodepth_cloud_workspace_bytes(2, 384, 640) == 2 * (384 * 640 // 256) * 8


def _run(script, *args, env=None):
    return subprocess.run([sys.executable, os.path.join(ROOT, "scripts", script), *args], capture_output=True,
                          text=True, env=env)


def test_register_dir_depth_model_flags(tmp_path):
    d = str(tmp_path / "data")
    synthetic.write_icp_handoff(d, str(tmp_path / "monodepth"), [1], "kitti")
    r = _run("register_dir.py", d, "--H", "160", "--W", "512", "--method", "icp", "--monodepth", "x",
             "--depth-model", "y")
    assert r.returncode == 2 and "alternatives" in r.stderr
    for method in ("lsq", "pnp"):
        r = _run("register_dir.py", d, "--H", "160", "--W", "512", "--method", method, "--depth-model", "y")
        assert r.returncode == 2 and "--depth-model is only used by --method icp" in r.stderr


def test_save_depth_map_refuses_without_a_device(tmp_path):
    r = _run("save_depth_map.py", str(tmp_path), env={**os.environ, "CUDA_VISIBLE_DEVICES": ""})
    assert r.returncode == 2 and "--depth-model" in r.stderr
    r = _run("save_depth_map.py", str(tmp_path), "--depth-model", str(tmp_path),
             env={**os.environ, "CUDA_VISIBLE_DEVICES": ""})
    assert r.returncode != 0 and "needs a CUDA device" in r.stderr
