"""GPU tests of the evaluation-side kernels against exact references:
- pose_error_batch (csrc/metrics.cu) bit for bit against oracle.pose_diff_restated, and within the CPU bounds of
  tests/test_metrics_cpu.py of scipy + np.linalg.inv;
- inside_mask_batch against the label rule evaluated in exact rational arithmetic from the float inputs;
- frustum.residuals (the drop-in's residual vector) against oracle.residuals.
"""
from fractions import Fraction

import numpy as np
import pytest
import torch

import oracle
from deepi2p_b200 import frustum, synthetic as syn
from test_metrics_cpu import R_TOL, T_TOL, all_cases, scipy_pose_diff, threshold_cases, uniform_cases

pytestmark = pytest.mark.gpu


def run_pose_error(A, B, stream=None, **kw):
    out = frustum.pose_error_batch(torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda(), stream=stream, **kw)
    torch.cuda.synchronize()
    return out, out["t_err"].cpu().numpy(), out["r_err"].cpu().numpy(), out["success"].cpu().numpy()


def assert_bits(got, want):
    assert np.array_equal(got.view(np.int64), np.asarray(want, dtype=np.float64).view(np.int64)), \
        np.nonzero(got.view(np.int64) != np.asarray(want, dtype=np.float64).view(np.int64))[0][:10]


# ---- pose_error_batch ------------------------------------------------------------------------------------------------

def test_pose_error_all_cases_bit_exact(cuda):
    """Uniform SO(3), half turns, the gimbal-lock band, float32-rounded / scaled / sheared P_pred and the thresholds,
    in one batch."""
    A, B = all_cases()
    out, te, re, ok = run_pose_error(A, B)
    t_r, r_r, ok_r = oracle.pose_diff_restated(A, B)
    assert_bits(te, t_r)
    assert_bits(re, r_r)
    np.testing.assert_array_equal(ok, ok_r)
    t_want, r_want = scipy_pose_diff(A, B)
    assert np.abs(te - t_want).max() <= T_TOL and np.abs(re - r_want).max() <= R_TOL
    assert 0 < ok.sum() < len(ok)
    assert out["success_rate"].item() == ok.mean()


def test_pose_error_thresholds(cuda):
    A, B = threshold_cases()
    _, te, re, ok = run_pose_error(A, B)
    assert te[0] == 2.0 and te[1] == np.nextafter(2.0, 0.0)
    np.testing.assert_array_equal(ok, [0, 1, 1, 0])
    for i in (2, 3):                       # an error exactly on the threshold fails, one ulp under it succeeds
        assert run_pose_error(A[i:i + 1], B[i:i + 1], r_thresh=float(re[i]))[3][0] == 0
        assert run_pose_error(A[i:i + 1], B[i:i + 1], r_thresh=float(np.nextafter(re[i], 10.0)))[3][0] == 1


@pytest.mark.parametrize("S", [1, 100_000])
def test_pose_error_sizes(cuda, S):
    A, B = uniform_cases(S, 11)
    out, te, re, ok = run_pose_error(A, B)
    t_r, r_r, ok_r = oracle.pose_diff_restated(A, B)
    assert_bits(te, t_r)
    assert_bits(re, r_r)
    np.testing.assert_array_equal(ok, ok_r)
    assert out["success_rate"].item() == ok.mean()


def test_pose_error_second_stream_and_nan(cuda):
    A, B = uniform_cases(4096, 12)
    A[5, 1, 1] = np.nan                    # NaN in the rotation
    A[9, 2, 3] = np.nan                    # NaN in the translation
    B[7] = A[7]                            # zero error: succeeds
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        out, te, re, ok = run_pose_error(A, B, stream=s)
    t_r, r_r, ok_r = oracle.pose_diff_restated(A, B)
    assert_bits(te, t_r)
    assert_bits(re, r_r)
    assert ok[5] == 0 and ok[9] == 0 and np.isnan(re[5]) and np.isnan(te[9]) and ok[7] == 1
    np.testing.assert_array_equal(ok, ok_r)
    assert out["success_rate"].item() == ok.mean()


# ---- inside_mask_batch -----------------------------------------------------------------------------------------------

EXACT_K = np.array([[256.0, 0.0, 255.0], [0.0, 128.0, 79.0], [0.0, 0.0, 1.0]])
EXACT_H, EXACT_W = 160, 512            # W - 1 = 511 = (u - 255) / 256 at X = 1, H - 1 = 159 at Y = 0.625


def exact_mask(pts, P, K, H, W):
    """get_inside_img_mask in exact rational arithmetic from the float inputs (pts [3,n] float32, P 3x4 / 4x4)."""
    P = [[Fraction(float(v)) for v in row] for row in np.asarray(P, dtype=np.float64)[:3]]
    K = [[Fraction(float(v)) for v in row] for row in np.asarray(K, dtype=np.float64)]
    z01 = Fraction(0.1)
    out = []
    for xyz in np.asarray(pts, dtype=np.float64).T:
        if not np.isfinite(xyz).all():
            out.append(0)                  # NaN coordinates: every comparison is false
            continue
        x, y, z = (Fraction(float(v)) for v in xyz)
        c = [P[i][0] * x + P[i][1] * y + P[i][2] * z + P[i][3] for i in range(3)]
        k = [K[i][0] * c[0] + K[i][1] * c[1] + K[i][2] * c[2] for i in range(3)]
        if k[2] == 0:
            out.append(0)                  # u = +-inf or NaN
            continue
        u, v = k[0] / k[2], k[1] / k[2]
        out.append(int(0 <= u <= W - 1 and 0 <= v <= H - 1 and c[2] > z01))
    return np.array(out, dtype=np.int8)


def signed_permutation(rng):
    R = np.eye(3)[rng.permutation(3)]
    R[0] *= rng.choice([-1.0, 1.0])
    R[1] *= rng.choice([-1.0, 1.0])
    return R * np.linalg.det(R)


def exact_boundary_cases():
    """One sample per case: a signed-permutation rotation, a dyadic translation and a float32 point whose camera
    coordinates (X, Y, Z) are exact targets, so every product and sum of the rule is exact in fp64 and u, v are exact
    quotients.  Returns (xyz [S,3,n] float32, P [S,4,4], [(case, want)])."""
    d = 2.0 ** -52          # in X and Y: one ulp of u at 511 (2^-44 = 256 d) and of v at 159 (2^-45 = 128 d), Z = 1
    X = {"in": 0.25, "u0": -255 / 256, "uW": 1.0, "u0-": -255 / 256 - d, "uW+": 1.0 + d,
         "u0+": -255 / 256 + d, "uW-": 1.0 - d}
    Y = {"in": 0.125, "v0": -79 / 128, "vH": 0.625, "v0-": -79 / 128 - d, "vH+": 0.625 + d,
         "v0+": -79 / 128 + d, "vH-": 0.625 - d}
    cases = [(X["u0"], Y["in"], 1.0, 1), (X["uW"], Y["in"], 1.0, 1), (X["in"], Y["v0"], 1.0, 1),
             (X["in"], Y["vH"], 1.0, 1), (X["u0"], Y["v0"], 1.0, 1), (X["uW"], Y["vH"], 1.0, 1),
             (X["u0-"], Y["in"], 1.0, 0), (X["uW+"], Y["in"], 1.0, 0), (X["in"], Y["v0-"], 1.0, 0),
             (X["in"], Y["vH+"], 1.0, 0), (X["u0+"], Y["in"], 1.0, 1), (X["uW-"], Y["in"], 1.0, 1),
             (X["in"], Y["v0+"], 1.0, 1), (X["in"], Y["vH-"], 1.0, 1),
             (0.0, 0.0, 0.1, 0), (0.0, 0.0, np.nextafter(0.1, 1.0), 1), (0.0, 0.0, np.nextafter(0.1, 0.0), 0)]
    rng = np.random.default_rng(5)
    xyz, Ps, want = [], [], []
    for cx, cy, cz, w in cases:
        R = signed_permutation(rng)
        p = (rng.integers(-64, 64, 3) / 64.0).astype(np.float32) if cz == 1.0 else np.zeros(3, np.float32)
        target = np.array([cx, cy, cz])
        t = target - R @ p.astype(np.float64)
        P = np.eye(4)
        P[:3, :3], P[:3, 3] = R, t
        # the construction is what it claims: exact camera coordinates, exact quotients on the targets
        for i in range(3):
            assert sum(Fraction(float(R[i, j])) * Fraction(float(p[j])) for j in range(3)) + Fraction(t[i]) \
                == Fraction(target[i])
        xyz.append(p[:, None]), Ps.append(P), want.append(w)
    return np.stack(xyz), np.stack(Ps), np.array(want, dtype=np.int8)


def test_inside_mask_exact_boundaries(cuda):
    """Inclusive at u = 0, u = W - 1, v = 0, v = H - 1 and strict at Z = 0.1 (as a double); one ulp of u / v / Z
    outside each boundary is outside, one ulp inside is inside."""
    xyz, P, want = exact_boundary_cases()
    for s in range(len(want)):
        assert exact_mask(xyz[s], P[s], EXACT_K, EXACT_H, EXACT_W)[0] == want[s]
    dev, _, n_pts = frustum.pack_clouds(xyz, np.zeros((len(want), 1), np.int32))
    mask = frustum.inside_mask_batch(dev, n_pts, P, EXACT_K, EXACT_H, EXACT_W).cpu().numpy()
    np.testing.assert_array_equal(mask[:, 0], want)
    # S = 1, and P given as 3x4
    for s in (0, 7, 14, 15):
        m1 = frustum.inside_mask_batch(dev[s:s + 1], n_pts[s:s + 1], P[s:s + 1, :3], EXACT_K, EXACT_H, EXACT_W)
        assert m1[0, 0].item() == want[s] and (m1[0, 1:] == -1).all()


# A point is compared only where its exact u, v are farther than 1e-6 px from every image boundary and its exact Z
# farther than 1e-9 m from 0.1.  For |coordinates| <= 100 m, |t| <= 10 m, K entries <= 1000 and Z >= 0.1 m any fp64
# evaluation order, with or without FMA, is within ~1e-9 px and ~1e-13 m of the exact values, far inside both margins.
U_MARGIN, Z_MARGIN = 1e-6, 1e-9


def test_inside_mask_random_exact(cuda):
    for shape in ("kitti", "oxford"):
        smp = syn.make_sample(41 if shape == "kitti" else 42, 4096, shape=shape)
        pts, P, K, H, W = smp["points"], smp["P_gt"], smp["K"], smp["H"], smp["W"]
        want = exact_mask(pts, P, K, H, W)
        c = P[:3, :3] @ pts.astype(np.float64) + P[:3, 3:4]
        k = K @ c
        with np.errstate(divide="ignore", invalid="ignore"):
            u, v = k[0] / k[2], k[1] / k[2]
        near = (np.abs(c[2] - 0.1) <= Z_MARGIN) | ((c[2] > 0.1) & (
            (np.abs(u) <= U_MARGIN) | (np.abs(u - (W - 1)) <= U_MARGIN) |
            (np.abs(v) <= U_MARGIN) | (np.abs(v - (H - 1)) <= U_MARGIN)))
        print("%s: %d of %d points within the margins, left out" % (shape, near.sum(), near.size))
        assert near.sum() <= 2
        xyz, _, n_pts = frustum.pack_clouds(pts, np.zeros(pts.shape[1], np.int32))
        mask = frustum.inside_mask_batch(xyz, n_pts, P[None], K, H, W).cpu().numpy()[0, :pts.shape[1]]
        np.testing.assert_array_equal(mask[~near], want[~near])
        assert 0 < want.sum() < want.size


def test_inside_mask_contract(cuda):
    """Behind the camera with u, v in range, Z = 0, NaN coordinates, ragged n_pts with -1 padding, n_pts=None."""
    K, H, W = EXACT_K, EXACT_H, EXACT_W
    pts = np.array([[0.25, 0.25, -0.25, 0.25, 0.0, np.nan, 0.25, 1.0, 0.0],
                    [0.125, 0.125, -0.125, 0.125, 0.0, 0.0, np.nan, 0.0, 0.0],
                    [1.0, 2.0, -1.0, 0.0, 0.0, 1.0, 1.0, 0.0, 0.0]], dtype=np.float32)
    # in front; in front; behind with u, v in range after the sign flip; Z = 0 (u = inf); Z = 0 and X = 0 (u = NaN);
    # NaN x; NaN y; Z = 0 with X > 0; the origin
    want = np.array([1, 1, 0, 0, 0, 0, 0, 0, 0], dtype=np.int8)
    np.testing.assert_array_equal(exact_mask(pts, np.eye(4), K, H, W), want)
    n = pts.shape[1]
    batch = np.stack([pts, pts, pts, pts])
    n_pts = np.array([n, 5, 1, 0], dtype=np.int32)
    xyz, _, npd = frustum.pack_clouds(batch, np.zeros((4, n), np.int32), n_pts=n_pts)
    P = np.tile(np.eye(4), (4, 1, 1))
    for P_arg in (P, P[:, :3]):
        mask = frustum.inside_mask_batch(xyz, npd, P_arg, K, H, W).cpu().numpy()
        for s, m in enumerate(n_pts):
            np.testing.assert_array_equal(mask[s, :m], want[:m])
            assert (mask[s, m:] == -1).all()
    mask = frustum.inside_mask_batch(xyz, None, P, K, H, W).cpu().numpy()
    for s in range(4):
        np.testing.assert_array_equal(mask[s, :n], want)
        assert (mask[s, n:] == exact_mask(np.zeros((3, xyz.shape[2] - n), np.float32), np.eye(4), K, H, W)).all()


# ---- frustum.residuals -----------------------------------------------------------------------------------------------

RES_RTOL, RES_ATOL = 1e-12, 1e-12      # per row; rows are O(1) (the Cauchy-corrected residual is below 1 in size)


def residual_cloud(seed, n):
    """A KITTI-shaped cloud labelled at random from {0, 1, 5, -1}: label-1 points in front of the image, beside it and
    behind the camera, label-0 points inside it, and ignored labels between them."""
    smp = syn.make_sample(seed, n)
    rng = np.random.default_rng(seed)
    lab = rng.choice([0, 1, 5, -1], n, p=[0.35, 0.45, 0.1, 0.1]).astype(np.int64)
    inside = syn.inside_mask(smp["points"], smp["P_gt"], smp["K"], smp["H"], smp["W"])
    lab[inside & (rng.uniform(size=n) < 0.5)] = 0
    return smp, lab


POSES = [(True, [0.05, 0.3, 0.02, -0.5]), (False, [0.02, 0.05, -0.03, 0.3, 0.02, -0.5]),
         (False, [1e-9, -2e-9, 3e-9, 0.1, 0.0, 0.2]), (False, [1e-5, 2e-5, -1e-5, 0.1, 0.0, 0.2])]


def pose_at(smp, is_2d, dx):
    x = np.zeros(6)
    x[:len(dx)] = dx
    if is_2d:
        x[0] += smp["ry_gt"]; x[1] += smp["t_gt"][0]; x[3] += smp["t_gt"][2]
    elif abs(x[1]) > 1e-3:
        x[1] += smp["ry_gt"]; x[3] += smp["t_gt"][0]; x[5] += smp["t_gt"][2]
    return x


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("pose", range(len(POSES)))
def test_residuals_match_oracle(cuda, dtype, pose):
    is_2d, dx = POSES[pose]
    smp, lab = residual_cloud(60 + pose, 3001)
    pts = smp["points"].astype(np.float64)
    if dtype == np.float64:
        pts = pts + np.random.default_rng(pose).normal(0, 1e-9, pts.shape)    # not float32-representable
    x = pose_at(smp, is_2d, dx)
    Pn = 4 if is_2d else 6
    # the categories the rows must cover, at this pose
    from scipy.spatial.transform import Rotation
    Pose = np.eye(4)
    Pose[:3, :3] = syn.ry_matrix(x[0]) if is_2d else Rotation.from_rotvec(x[:3]).as_matrix()
    Pose[:3, 3] = x[1:4] if is_2d else x[3:6]
    cam = Pose[:3, :3] @ pts + Pose[:3, 3:4]
    fr = syn.inside_mask(pts, Pose, smp["K"], smp["H"], smp["W"])
    assert ((lab == 1) & fr).any() and ((lab == 1) & ~fr & (cam[2] > 0)).any() and ((lab == 1) & (cam[2] < 0)).any()
    assert ((lab == 0) & fr).any() and (lab == 5).any() and (lab == -1).any()
    xyz, l8, _ = frustum.pack_clouds(pts, lab, dtype=dtype)
    for n in (3001, 1777, 1, 0):
        want, cost = oracle.residuals(pts[:, :n], lab[:n], smp["K"], x[:Pn], smp["H"], smp["W"], is_2d)
        for host in (lab, None):
            got = frustum.residuals(xyz[0], l8[0], n, smp["K"], torch.from_numpy(x).cuda(), smp["H"], smp["W"],
                                    is_2d, host_labels=host).cpu().numpy()
            assert got.shape == want.shape
            np.testing.assert_allclose(got, want, rtol=RES_RTOL, atol=RES_ATOL)
        if n == 3001:
            # the rows determine the cost: 0.5 sum over points of log(1 + s), s = q / (1 - q) with q = the point's
            # sum of squared rows; the rows fix s only to ~eps / (1 - q), which bounds the comparison
            rows = np.where(lab[:n] == 1, 3, np.where(lab[:n] == 0, 1, 0))
            off = np.cumsum(rows) - rows
            q = np.array([(got[o:o + k] ** 2).sum() for o, k in zip(off, rows) if k])
            rebuilt = 0.5 * np.sum(-np.log1p(-q))
            c, _, _ = frustum.evaluate_batch(xyz, l8, torch.tensor([n], dtype=torch.int32), smp["K"], x[None],
                                             smp["H"], smp["W"], is_2d)
            slack = np.sum(2e-15 / (1.0 - q))
            assert abs(rebuilt - c.item()) <= 1e-10 * c.item() + slack
            assert abs(c.item() - cost) <= 1e-10 * max(1.0, cost)
