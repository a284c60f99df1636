"""The registration metric pose_error_batch (csrc/metrics.cu), CPU half: its numpy restatement
oracle.pose_diff_restated against get_P_diff as the reference computes it (oracle.pose_diff: np.linalg.inv, then
scipy's Rotation.from_matrix(...).as_euler('xzy')), at the edges where the two could part: uniform SO(3), 180 degree
rotations, the gimbal-lock band, a P_pred that is rigid only to float32 rounding or not rigid at all, and the strict
2 m / 5 degree thresholds.  tests/test_metrics_gpu.py checks the kernel bit for bit against the restatement on the
same cases.
"""
import math
import warnings

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

import oracle

R_TOL = 1e-9        # degrees
T_TOL = 1e-12       # m
# scipy calls the middle 'xzy' angle locked when it is within 1e-7 rad of +-90 deg; cases closer than ~1e-12 to that
# threshold may legitimately go either way (rounding of the quaternion), so every offset below is at least 5e-8 clear.
LOCK_OFFSETS = (0.0, 1e-10, 1e-9, 5e-8, 1e-6)


def rigid(R, t):
    P = np.tile(np.eye(4), (len(R), 1, 1))
    P[:, :3, :3] = R
    P[:, :3, 3] = t
    return P


def scipy_pose_diff(A, B):
    """oracle.pose_diff over a batch (the same numpy / scipy calls, batched)."""
    D = np.linalg.inv(A) @ B
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")                 # scipy warns on gimbal lock
        e = Rotation.from_matrix(D[:, :3, :3]).as_euler("xzy", degrees=True)
    return np.linalg.norm(D[:, :3, 3], axis=1), np.abs(e).sum(axis=1)


def uniform_cases(S=100_000, seed=0):
    rng = np.random.default_rng(seed)
    A = rigid(Rotation.random(S, random_state=seed).as_matrix(), rng.uniform(-10, 10, (S, 3)))
    B = rigid(Rotation.random(S, random_state=seed + 1).as_matrix(), rng.uniform(-10, 10, (S, 3)))
    return A, B


def half_turn_cases(seed=1):
    """180 degree rotations about x, y, z and random axes: exact matrices against P_pred = I, and composed onto a
    random rigid P_pred."""
    rng = np.random.default_rng(seed)
    axes = np.concatenate([np.eye(3), rng.normal(size=(29, 3))])
    axes /= np.linalg.norm(axes, axis=1, keepdims=True)
    H = np.array([2.0 * np.outer(a, a) - np.eye(3) for a in axes])      # exact for the coordinate axes
    n = len(H)
    A0 = rigid(np.tile(np.eye(3), (n, 1, 1)), np.zeros((n, 3)))
    B0 = rigid(H, rng.uniform(-1, 1, (n, 3)))
    A1 = rigid(Rotation.random(n, random_state=seed).as_matrix(), rng.uniform(-10, 10, (n, 3)))
    B1 = A1.copy()
    B1[:, :3, :3] = A1[:, :3, :3] @ H
    return np.concatenate([A0, A1]), np.concatenate([B0, B1])


def lock_cases(seed=2, per=64):
    """Middle 'xzy' angle at +-(90 deg - offset), random first and third angles, P_pred = I (P_diff = P_gt exactly on
    both sides: the band's first / third angles are ill-conditioned in P_diff itself)."""
    rng = np.random.default_rng(seed)
    Bs = []
    for off in LOCK_OFFSETS:
        for sgn in (1.0, -1.0):
            e = np.stack([rng.uniform(-3, 3, per), np.full(per, sgn * (math.pi / 2 - off)), rng.uniform(-3, 3, per)], 1)
            Bs.append(rigid(Rotation.from_euler("xzy", e).as_matrix(), rng.uniform(-1, 1, (per, 3))))
    B = np.concatenate(Bs)
    return rigid(np.tile(np.eye(3), (len(B), 1, 1)), np.zeros((len(B), 3))), B


def nonrigid_cases(seed=3, S=2000):
    """P_pred rounded to float32 (fails scipy's orthogonality test: polar factor), scaled by 1 + 1e-6 (passes it:
    the quaternion of the scaled matrix), and scaled by 1 + 1e-3 with a 1e-3 shear (polar factor far from I)."""
    A, B = uniform_cases(S, seed)
    A32 = A.astype(np.float32).astype(np.float64)
    As = A.copy()
    As[:, :3, :3] *= 1.0 + 1e-6
    Ab = A.copy()
    Ab[:, :3, :3] = Ab[:, :3, :3] * (1.0 + 1e-3) + 1e-3 * np.random.default_rng(seed).normal(size=(S, 3, 3))
    return np.concatenate([A32, As, Ab]), np.concatenate([B, B, B])


def threshold_cases():
    """t exactly 2 and one ulp under (identity rotation); r exactly 5 and one ulp under in the restated arithmetic."""
    two = np.nextafter(2.0, 0.0)
    A, B = [], []
    for tx in (2.0, two):
        P = np.eye(4)
        P[0, 3] = tx
        A.append(np.eye(4)), B.append(P)
    # r = 5 exactly is out of reach: each angle is wrapped through (a + pi) % 2 pi - pi, which leaves a multiple of
    # 2^-51 rad for |a| < pi - 1, so near 5 degrees r moves on a lattice ~28 ulps wide that misses 5.0 by ~6 ulps.
    # The cases are the reachable r just under and just over 5; test_thresholds_are_strict pins the strict comparison
    # with the threshold set to a reached r itself.
    rng = np.random.default_rng(4)
    first = rng.uniform(1.0, 4.0, 4096) * math.pi / 180.0
    third = 5.0 * math.pi / 180.0 - first + rng.uniform(-1e-15, 1e-15, first.size)
    Bc = rigid(Rotation.from_euler("xzy", np.stack([first, np.zeros_like(first), third], 1)).as_matrix(),
               np.zeros((first.size, 3)))
    r = oracle.pose_diff_restated(np.tile(np.eye(4), (first.size, 1, 1)), Bc)[1]
    for pick in (np.argmax(np.where(r < 5.0, r, -np.inf)), np.argmin(np.where(r >= 5.0, r, np.inf))):
        A.append(np.eye(4)), B.append(Bc[pick])
    return np.stack(A), np.stack(B)


def all_cases():
    parts = [uniform_cases(20_000, 7), half_turn_cases(), lock_cases(), nonrigid_cases(), threshold_cases()]
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])


def old_kernel_restated(A, B):
    """The kernel before it followed scipy: rigid inverse, b = asin(R10), a = atan2(-R12, R11), c = atan2(-R20, R00)."""
    R = np.swapaxes(A[:, :3, :3], 1, 2) @ B[:, :3, :3]
    e = np.stack([np.arctan2(-R[:, 1, 2], R[:, 1, 1]), np.arcsin(np.clip(R[:, 1, 0], -1, 1)),
                  np.arctan2(-R[:, 2, 0], R[:, 0, 0])], 1)
    return np.abs(e).sum(axis=1) * (180.0 / math.pi)


def check(A, B, r_tol=R_TOL, t_tol=T_TOL):
    te, re, ok = oracle.pose_diff_restated(A, B)
    t_want, r_want = scipy_pose_diff(A, B)
    assert np.abs(te - t_want).max() <= t_tol
    assert np.abs(re - r_want).max() <= r_tol, np.abs(re - r_want).max()
    np.testing.assert_array_equal(ok, ((te < 2.0) & (re < 5.0)).astype(np.int32))
    return te, re


def test_uniform_so3():
    A, B = uniform_cases()
    check(A, B)
    for i in range(0, 100_000, 9973):                  # the batched reference is oracle.pose_diff, row by row
        t, r = oracle.pose_diff(A[i], B[i])
        te, re, _ = oracle.pose_diff_restated(A[i:i + 1], B[i:i + 1])
        assert abs(te[0] - t) <= T_TOL and abs(re[0] - r) <= R_TOL


def test_half_turns():
    _, re = check(*half_turn_cases())
    assert re.max() > 179.0


def test_gimbal_lock_band():
    A, B = lock_cases()
    check(A, B)


def test_lock_band_catches_the_old_formula():
    """The comparison above fails for the formula the kernel used before: within 1e-8 rad of lock it is off by tens
    of degrees, and away from lock it agrees."""
    A, B = lock_cases()
    _, want = scipy_pose_diff(A, B)
    assert np.abs(old_kernel_restated(A, B) - want).max() > 10.0
    A, B = uniform_cases(20_000, 5)
    _, want = scipy_pose_diff(A, B)
    assert np.abs(old_kernel_restated(A, B) - want).max() < 1e-7


def test_nonrigid_pred():
    A, B = nonrigid_cases()
    check(A, B)


def test_thresholds_are_strict():
    A, B = threshold_cases()
    te, re, ok = oracle.pose_diff_restated(A, B)
    assert te[0] == 2.0 and ok[0] == 0
    assert te[1] == np.nextafter(2.0, 0.0) and ok[1] == 1
    assert 5.0 - 1e-13 < re[2] < 5.0 and ok[2] == 1
    assert 5.0 <= re[3] < 5.0 + 1e-13 and ok[3] == 0
    # an error exactly on the threshold fails, one ulp under it succeeds
    for i in (2, 3):
        assert oracle.pose_diff_restated(A[i:i + 1], B[i:i + 1], r_thresh=re[i])[2][0] == 0
        assert oracle.pose_diff_restated(A[i:i + 1], B[i:i + 1], r_thresh=np.nextafter(re[i], 10.0))[2][0] == 1
    check(A, B)


def test_not_a_rotation():
    """A reflected or singular P_pred: scipy raises, the restatement gives r_err NaN and success 0; NaN likewise."""
    A = np.tile(np.eye(4), (3, 1, 1))
    A[0, 0, 0] = -1.0
    A[1, 2, 2] = 0.0
    A[2, 1, 3] = np.nan
    B = np.tile(np.eye(4), (3, 1, 1))
    with pytest.raises(ValueError):
        oracle.pose_diff(A[0], B[0])
    te, re, ok = oracle.pose_diff_restated(A, B)
    assert np.isnan(re).all() and (ok == 0).all()
