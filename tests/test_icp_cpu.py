"""The ICP oracle (oracle_icp) against independent numpy / scipy restatements, the contract's edge cases, the seeded
inits and synthetic frames, and the C ABI's host-side validation.  No GPU needed."""
import ctypes
import math
import os

import numpy as np
import pytest
from scipy.spatial import cKDTree

import oracle_icp
from deepi2p_b200 import icp, synthetic

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "icp_small.npz")


def _kabsch(src, dst):
    """Independent rigid Umeyama: numpy SVD with the reflection guard."""
    ms, md = src.mean(0), dst.mean(0)
    A = (dst - md).T @ (src - ms) / len(src)
    U, _, Vt = np.linalg.svd(A)
    S = np.eye(3)
    if np.linalg.det(U) * np.linalg.det(Vt) < 0:
        S[2, 2] = -1
    R = U @ S @ Vt
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = md - R @ ms
    return T


def _icp_numpy(src, tgt, T, r=1.0, max_it=30, rf=1e-6, rr=1e-6):
    """Independent restatement of one ICP problem (cKDTree neighbours, numpy Kabsch)."""
    tree = cKDTree(tgt.T.astype(np.float64))
    p = src.astype(np.float64)

    def one_pass(T):
        q = (T[:3, :3] @ p + T[:3, 3:4]).T
        d, j = tree.query(q, k=1, distance_upper_bound=r * 1.5)
        ok = np.isfinite(d)
        dd = q[ok] - tgt.T[j[ok]].astype(np.float64)
        d2 = (dd[:, 0] * dd[:, 0] + dd[:, 1] * dd[:, 1]) + dd[:, 2] * dd[:, 2]
        keep = d2 < r * r
        idx = np.flatnonzero(ok)[keep]
        nc = len(idx)
        return q[idx], tgt.T[j[idx]].astype(np.float64), nc, nc / p.shape[1], (math.sqrt(d2[keep].sum() / nc) if nc else 0.0)

    qs, ts, nc, fit, rmse = one_pass(T)
    trace = [nc]
    k = 0
    while k < max_it:
        if nc:
            T = _kabsch(qs, ts) @ T
        k += 1
        prev = (fit, rmse)
        qs, ts, nc, fit, rmse = one_pass(T)
        trace.append(nc)
        if abs(prev[0] - fit) < rf and abs(prev[1] - rmse) < rr:
            break
    return T, fit, rmse, k, trace


def _small_scene(seed, n=600, m=3000):
    """Three noisy orthogonal planes (no exact distance ties) and a source drawn from the same planes, offset."""
    rng = np.random.default_rng(seed)

    def planes(k):
        u = rng.uniform(-4, 4, (3, k))
        a = rng.integers(0, 3, k)
        u[a, np.arange(k)] = rng.normal(0, 0.02, k) + np.array([0.0, 2.0, 6.0])[a]
        return u

    tgt = planes(m).astype(np.float32)
    src = planes(n).astype(np.float32)
    return src, tgt


def _pose(ry, t):
    P = np.eye(4)
    P[:3, :3] = synthetic.ry_matrix(ry)
    P[:3, 3] = t
    return P


def test_oracle_matches_numpy_restatement():
    src, tgt = _small_scene(0)
    inits = np.stack([_pose(0.05, [0.2, 0.0, -0.3]), _pose(-0.1, [0.4, 0.1, 0.2]), _pose(0.0, [0, 0, 0])])
    r = oracle_icp.register_frame(src, tgt, inits, trace=True)
    for i, T0 in enumerate(inits):
        T, fit, rmse, k, trace = _icp_numpy(src, tgt, T0)
        assert r["stats"][i, 0] == k
        np.testing.assert_array_equal(r["trace_nc"][i, :k + 1], trace)
        np.testing.assert_allclose(r["T"][i], T, rtol=0, atol=1e-9)
        assert abs(r["fitness"][i] - fit) < 1e-15 and abs(r["rmse"][i] - rmse) < 1e-9


@pytest.mark.parametrize("offset", [0.0, 50.0])
@pytest.mark.parametrize("reflect", [False, True])
def test_umeyama_matches_numpy_kabsch(offset, reflect):
    rng = np.random.default_rng(int(offset) + 2 * reflect)
    for _ in range(20):
        src = rng.normal(0, 1.0, (40, 3)) * np.array([3.0, 2.0, 1.0]) + offset
        a = rng.normal(size=3)
        a /= np.linalg.norm(a)
        ang = rng.uniform(-math.pi, math.pi)
        Kx = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
        R = np.eye(3) + math.sin(ang) * Kx + (1 - math.cos(ang)) * Kx @ Kx
        if reflect:
            R = R @ np.diag([1.0, 1.0, -1.0])          # det < 0: the best rotation, not the reflection
        dst = src @ R.T + rng.uniform(-3, 3, 3) + rng.normal(0, 0.01, (40, 3))
        U = oracle_icp.umeyama(src, dst)
        np.testing.assert_allclose(U, _kabsch(src, dst), rtol=0, atol=1e-12 * max(1.0, offset))
        assert abs(np.linalg.det(U[:3, :3]) - 1) < 1e-12


def test_umeyama_degenerate_sets_are_finite_and_deterministic():
    one = oracle_icp.umeyama(np.array([[1.0, 2.0, 3.0]]), np.array([[1.5, 2.0, 2.0]]))
    np.testing.assert_array_equal(one[:3, :3], np.eye(3))
    np.testing.assert_allclose(one[:3, 3], [0.5, 0.0, -1.0], atol=1e-15)
    two_s = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0]])
    two_d = np.array([[0.0, 1.0, 0.0], [0.0, 2.0, 0.0]])
    a, b = oracle_icp.umeyama(two_s, two_d), oracle_icp.umeyama(two_s, two_d)
    assert np.isfinite(a).all() and np.array_equal(a, b)
    np.testing.assert_allclose(a[:3, :3] @ np.array([1.0, 0, 0]), [0, 1, 0], atol=1e-12)
    assert abs(np.linalg.det(a[:3, :3]) - 1) < 1e-12


def test_zero_correspondences_keep_the_init():
    src, tgt = _small_scene(1, 100, 500)
    far = _pose(0.3, [500.0, 0.0, 0.0])
    r = oracle_icp.register_frame(src, tgt, far[None], force_2d=False)
    np.testing.assert_array_equal(r["T"][0], far)
    assert r["fitness"][0] == 0 and r["rmse"][0] == 0 and r["stats"][0].tolist() == [1, 0]
    assert r["best"] == -1 and r["fitness_best"] == 0.001
    np.testing.assert_array_equal(r["P"], np.eye(4))


def test_one_and_two_correspondences():
    tgt = np.array([[0.0, 5.0], [0.0, 0.0], [0.0, 0.0]], dtype=np.float32)
    for src in (np.array([[0.3], [0.2], [0.1]], dtype=np.float32),
                np.array([[0.3, 5.2], [0.2, 0.1], [0.1, 0.0]], dtype=np.float32)):
        a = oracle_icp.register_frame(src, tgt, np.eye(4)[None], force_2d=False)
        b = oracle_icp.register_frame(src, tgt, np.eye(4)[None], force_2d=False)
        assert np.isfinite(a["T"]).all() and np.array_equal(a["T"], b["T"])
        assert a["stats"][0, 1] == src.shape[1]


def test_threshold_is_strict_and_ties_go_to_the_lowest_index():
    tgt = np.array([[1.0, 0.0, 0.0, 0.5], [0.0, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0, 3.0]], dtype=np.float32)
    j, d2 = oracle_icp.nearest(tgt, [[0.0, 0.0, 1.0]])          # d = 1 exactly to index 1 and 2
    assert j[0] == -1
    j, d2 = oracle_icp.nearest(tgt, [[0.0, 0.0, 0.5]])          # duplicates 1 and 2: the lower index wins
    assert j[0] == 1 and d2[0] == 0.25
    j, _ = oracle_icp.nearest(tgt, [[0.5, 0.0, 0.0]])           # tie between 0 and 1 at d2 = 0.25
    assert j[0] == 0


def test_nearest_is_exact_on_random_clouds():
    rng = np.random.default_rng(5)
    tgt = rng.uniform(-5, 5, (3, 4000)).astype(np.float32)
    q = rng.uniform(-5.5, 5.5, (2000, 3))
    j, d2 = oracle_icp.nearest(tgt, q, max_corr_dist=0.3)
    t = tgt.T.astype(np.float64)
    for i in range(0, 2000, 7):
        dd = q[i] - t
        e = (dd[:, 0] * dd[:, 0] + dd[:, 1] * dd[:, 1]) + dd[:, 2] * dd[:, 2]
        b = int(np.argmin(e))
        if e[b] < 0.09:
            assert j[i] == b and d2[i] == e[b]
        else:
            assert j[i] == -1


def test_convergence_within_max_iteration():
    src, tgt = _small_scene(3)
    r = oracle_icp.register_frame(src, tgt, _pose(0.02, [0.1, 0.0, 0.1])[None], max_iteration=30)
    assert 1 <= r["stats"][0, 0] < 30
    r5 = oracle_icp.register_frame(src, tgt, _pose(0.02, [0.1, 0.0, 0.1])[None], max_iteration=2)
    assert r5["stats"][0, 0] <= 2
    r0 = oracle_icp.register_frame(src, tgt, _pose(0.02, [0.1, 0.0, 0.1])[None], max_iteration=0)
    assert r0["stats"][0, 0] == 0
    np.testing.assert_array_equal(r0["T"][0], _pose(0.02, [0.1, 0.0, 0.1]))


def test_selection_is_strict_max_with_floor_and_2d_forcing():
    src, tgt = _small_scene(4, 300, 1500)
    good = _pose(0.02, [0.1, 0.0, 0.1])
    inits = np.stack([_pose(0.0, [900, 0, 0]), good, good, _pose(0.0, [-900, 0, 0])])
    r = oracle_icp.register_frame(src, tgt, inits, force_2d=True)
    assert r["fitness"][1] == r["fitness"][2] and r["best"] == 1       # equal fitness: the first one stays
    P = r["T"][1].copy()
    P[0, 1] = P[1, 0] = P[1, 2] = P[2, 1] = 0
    P[1, 1] = 1
    np.testing.assert_array_equal(r["P"], P)
    assert r["fitness_best"] == r["fitness"][1]
    r = oracle_icp.register_frame(src, tgt, inits[[0, 3]], force_2d=True)
    assert r["best"] == -1 and r["fitness_best"] == 0.001
    np.testing.assert_array_equal(r["P"], np.eye(4))


def test_random_inits_support_and_determinism():
    a = icp.random_inits(3, 50, seed=7)
    np.testing.assert_array_equal(a, icp.random_inits(3, 50, seed=7))
    assert not np.array_equal(a, icp.random_inits(3, 50, seed=8))
    assert a.shape == (3, 50, 4, 4)
    assert (np.abs(a[..., 0, 3]) <= 5).all() and (a[..., 1, 3] == 0).all() and (np.abs(a[..., 2, 3]) <= 10).all()
    R = a[..., :3, :3]
    np.testing.assert_allclose(R @ np.swapaxes(R, -1, -2), np.broadcast_to(np.eye(3), R.shape), atol=1e-12)
    assert (R[..., 1, 1] == 1).all() and (R[..., 0, 1] == 0).all() and (R[..., 1, 0] == 0).all()
    np.testing.assert_allclose(R[..., 0, 2], -R[..., 2, 0], atol=0)
    np.testing.assert_array_equal(a[..., 3, :], np.broadcast_to([0, 0, 0, 1.0], a[..., 3, :].shape))


def test_make_icp_frame_is_deterministic_and_registers_from_gt():
    f = synthetic.make_icp_frame(11, "kitti")
    g = synthetic.make_icp_frame(11, "kitti")
    np.testing.assert_array_equal(f["src"], g["src"])
    np.testing.assert_array_equal(f["tgt"], g["tgt"])
    assert f["src"].shape == (3, 20480) and f["src"].dtype == np.float32 and f["tgt"].shape == (3, 160 * 512)
    # save_depth_map.py order: point y * W + x is pixel (x, y) back-projected at its depth
    y, x = 100, 300
    np.testing.assert_allclose(f["tgt"][:, y * 512 + x], f["depth"][y, x] * np.linalg.inv(f["K"]) @ [x, y, 1.0],
                               rtol=1e-12)
    tgt = (f["tgt"] / f["scale"]).astype(np.float32)          # the true scale: the registration problem itself
    inits = np.concatenate([f["P_gt"][None], icp.random_inits(1, 8, seed=1)[0]])
    r = oracle_icp.register_frame(f["src"], tgt, inits, force_2d=False)
    D = np.linalg.inv(r["T"][0]) @ f["P_gt"]
    assert np.linalg.norm(D[:3, 3]) < 2.0
    assert math.degrees(math.acos(min(1.0, (np.trace(D[:3, :3]) - 1) / 2))) < 5.0
    assert r["fitness"][0] > np.median(r["fitness"][1:])


def test_abi_rejects_bad_arguments_without_gpu():
    from deepi2p_b200 import _native
    lib = _native.load()
    buf = (ctypes.c_double * 64)()
    a = ctypes.addressof(buf)

    def call(n_stride=16, m_stride=16, S=1, I=1, r=1.0, it=30, src=a, ws=a, wsb=1 << 40):
        return lib.icp_register_batch_f32(src, None, n_stride, a, None, m_stride, S, a, I, r, it, 1e-6, 1e-6, 1,
                                          a, a, None, None, None, None, None, ws, wsb, None)
    for kw, msg in ((dict(r=0.0), b"max_corr_dist"), (dict(r=-1.0), b"max_corr_dist"),
                    (dict(n_stride=17), b"multiple of 16"), (dict(m_stride=40), b"multiple of 16"),
                    (dict(src=None), b"NULL"), (dict(S=70000), b"S="), (dict(S=-1), b"S="), (dict(I=0), b"I="),
                    (dict(I=5000), b"I="), (dict(it=-1), b"max_iteration"), (dict(ws=None), b"workspace")):
        assert call(**kw) == -22, kw
        assert msg in lib.dib_last_error(), (kw, lib.dib_last_error())
    assert lib.icp_workspace_bytes(2, 60, 20480, 245760) > 2 * 245760 * 16
    assert lib.icp_workspace_bytes(2, 0, 16, 16) == 0


def test_oracle_reproduces_golden():
    g = np.load(GOLDEN)
    for f in range(int(g["n_frames"])):
        n, m = int(g["n"][f]), int(g["m"][f])
        r = oracle_icp.register_frame(g["src"][f][:, :n], g["tgt"][f][:, :m], g["init"][f],
                                      max_iteration=int(g["max_iteration"]), force_2d=True)
        np.testing.assert_array_equal(r["T"], g["T"][f])
        np.testing.assert_array_equal(r["fitness"], g["fitness"][f])
        np.testing.assert_array_equal(r["rmse"], g["rmse"][f])
        np.testing.assert_array_equal(r["stats"], g["stats"][f])
        np.testing.assert_array_equal(r["P"], g["P"][f])
        assert r["best"] == g["best"][f]
