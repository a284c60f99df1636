"""The raw-moment Umeyama of the kernels' first ICP pass (moments about the origin) at 50 m offsets, and host-side
validation of the ICP measurement entry points.  No GPU needed."""
import ctypes
import math

import numpy as np

import oracle_icp
from deepi2p_b200 import synthetic


def _kabsch(src, dst):
    ms, md = src.mean(0), dst.mean(0)
    U, _, Vt = np.linalg.svd((dst - md).T @ (src - ms) / len(src))
    S = np.eye(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2, 2] = -1
    R = U @ S @ Vt
    return R, md - R @ ms


def test_umeyama_moments_about_the_origin_at_50m():
    """The kernels' first pass takes its moments about c = 0.  With points 50 m out and a spread of a few metres the
    raw second moments cancel about (50 / 1)^2 ~ 2.5e3 x eps in relative terms.  The largest differences to numpy
    Kabsch over these 50 sets are 4.9e-13 (rotation entries) and 3.0e-11 m (translation); the bounds leave 10x."""
    rng = np.random.default_rng(9)
    worst_r = worst_t = 0.0
    for _ in range(50):
        src = rng.normal(0, 1.0, (200, 3)) * np.array([3.0, 2.0, 1.0]) + rng.uniform(-50, 50, 3)
        R = synthetic.ry_matrix(rng.uniform(-math.pi, math.pi))
        dst = src @ R.T + rng.uniform(-3, 3, 3) + rng.normal(0, 0.01, (200, 3))
        U = oracle_icp.umeyama(src, dst, c=np.zeros(3))
        Rk, tk = _kabsch(src, dst)
        worst_r = max(worst_r, float(np.abs(U[:3, :3] - Rk).max()))
        worst_t = max(worst_t, float(np.abs(U[:3, 3] - tk).max()))
    assert worst_r < 5e-12 and worst_t < 3e-10, (worst_r, worst_t)


def test_measurement_entry_points_validate_on_the_host():
    from deepi2p_b200 import _native
    lib = _native.load()
    buf = (ctypes.c_double * 64)()
    a = ctypes.addressof(buf)
    assert lib.icp_register_batch_counted_f32(a, None, 16, a, None, 16, 1, a, 1, 1.0, 30, 1e-6, 1e-6, 1, a, a, None,
                                              None, None, None, None, None, a, 1 << 40, None) == -22
    assert b"counters" in lib.dib_last_error()
    assert lib.icp_register_batch_counted_f32(a, None, 16, a, None, 16, 1, a, 1, 0.0, 30, 1e-6, 1e-6, 1, a, a, None,
                                              None, None, None, None, a, a, 1 << 40, None) == -22
    assert b"max_corr_dist" in lib.dib_last_error()
    assert lib.icp_build_index_f32(a, None, 17, 1, a, 1 << 40, None) == -22
    assert b"multiple of 16" in lib.dib_last_error()
    assert lib.icp_build_index_f32(None, None, 16, 1, a, 1 << 40, None) == -22
    assert lib.icp_build_index_f32(a, None, 16, 1, None, 0, None) == -22
    assert b"workspace" in lib.dib_last_error()
