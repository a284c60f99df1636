"""The small dense fp64 solvers on degenerate geometry, on the CPU oracles, against exact references.

- EPnP (oracle_pnp.epnp, the restatement of warp_epnp): noise-free correspondences on exact and near planes, lines,
  4 coplanar points plus one off the plane and duplicated points.  The reference is the ground-truth pose: a set
  reported valid must reproduce it (rotation within 1e-9 rad, translation within 1e-9 of the scene size), and a set
  that cannot must be reported degenerate, the same way on every call.
- The 3x3 Jacobi eigensolver shared by EPnP and the normals (oracle_pnp.sym3_eig) against 50-digit mpmath
  eigen-decompositions: repeated and split eigenvalues, rank 1 and 2, off-diagonals at the skip threshold, rounding
  below zero, random rotations, entries from 1e-80 to 1e150.
- Normals (oracle_prep.estimate_normals, bit-identical to the kernel) on planar patches 80 m from the origin, scan
  lines, lattices, a corner and a plane whose normal is perpendicular to the orientation: neighbour sets from cKDTree
  with the (d2, index) cut, covariances and eigenvectors in mpmath.
- ICP's Umeyama step (oracle_icp.register_frame, max_iteration=1) on planar, collinear and mirrored correspondences
  against a numpy Kabsch of the first pass's pairs.

tests/test_degenerate_geometry_gpu.py runs the same cases through the kernels."""
import mpmath
import numpy as np
import pytest

import oracle_icp
import oracle_pnp
import oracle_prep

U = 2.0 ** -53                     # unit roundoff of fp64
KF = np.array([[353.5 / 32, 0.0, 250.5 / 32], [0.0, 353.5 / 32, 66.5 / 32], [0.0, 0.0, 1.0]])


# ---------------------------------------------------------------------------------------------------------------
# EPnP

def _rot(rng, amp):
    a = rng.normal(size=3) * amp
    th = np.linalg.norm(a)
    k = a / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx


def _rx(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[1.0, 0.0, 0.0], [0.0, c, -s], [0.0, s, c]])


def _project(P, rng):
    """A camera pose R, t near the identity and the exact pixels of the world points P [n,3] as given."""
    R = _rot(rng, 0.1)
    t = np.array([rng.uniform(-1, 1), rng.uniform(-0.5, 0.5), rng.uniform(-1, 1)])
    Xc = P @ R.T + t
    assert (Xc[:, 2] > 1.0).all()
    uv = Xc[:, :2] / Xc[:, 2:3] * np.array([KF[0, 0], KF[1, 1]]) + KF[:2, 2]
    return uv, R, t


def _plane_points(rng, n, tilt, thick=0.0):
    """n points of the ground plane y = 1.6 (x in [-10, 10], z in [5, 40]: a scene 35 m across), tilted about x by
    `tilt`, displaced along the plane's normal by up to thick * 35 m."""
    P = np.stack([rng.uniform(-10, 10, n), np.full(n, 1.6), rng.uniform(5, 40, n)], 1)
    P[:, 1] += thick * 35.0 * rng.uniform(-1, 1, n)
    return P @ _rx(tilt).T


def _line_points(rng, n, tilt):
    s = rng.uniform(0, 1, n)[:, None]
    return np.array([-5.0, 1.6, 6.0]) @ _rx(tilt).T + s * (np.array([10.0, 0.0, 30.0]) @ _rx(tilt).T)


EPNP_NS = (4, 5, 6, 50, 1000)


def epnp_cases():
    """(name, xyz [n,3], uv [n,2], R, t, expect): expect 'degenerate' (must be rejected), 'valid' (must be accepted
    and exact) or 'either' (if accepted, exact).  All noise-free; pixels are those of the points as given."""
    out = []

    def add(name, P, rng, expect):
        uv, R, t = _project(P, rng)
        out.append((name, P, uv, R, t, expect))

    for n in EPNP_NS:
        for seed in range(3):
            rng = np.random.default_rng([n, seed])
            for tilt in (0.0, 0.3, 1.0):
                # exact planes: the fp64 points are coplanar to rounding, so lam[2] is rounding noise
                add(f"plane tilt={tilt} n={n} f64 #{seed}", _plane_points(rng, n, tilt), rng, "degenerate")
                # float32 world points: off the tilted plane by up to half an ulp (about 1e-7 of the scene)
                P32 = _plane_points(rng, n, tilt).astype(np.float32).astype(np.float64)
                add(f"plane tilt={tilt} n={n} f32 #{seed}", P32, rng, "degenerate" if tilt == 0.0 else "either")
            for thick, expect in ((1e-9, "degenerate"), (1e-6, "valid"), (1e-3, "valid")):
                if n >= 5:          # 4 points: EPnP's linearisations are approximations (cv2's too), see DESIGN.md 4.8
                    add(f"slab {thick:g} n={n} #{seed}", _plane_points(rng, n, 0.3, thick), rng, expect)
            add(f"line n={n} f64 #{seed}", _line_points(rng, n, 0.3), rng, "degenerate")
            Pl = np.stack([rng.uniform(-5, 5, n), np.full(n, 1.5), np.full(n, 12.0)], 1)
            add(f"axis line n={n} #{seed}", Pl.astype(np.float32).astype(np.float64), rng, "degenerate")
            add(f"line n={n} f32 #{seed}", _line_points(rng, n, 0.3).astype(np.float32).astype(np.float64), rng,
                "either")
            # duplicates: three distinct points (always coplanar), and six distinct points in general position
            base3 = np.stack([rng.uniform(-4, 4, 3), rng.uniform(-2, 2, 3), rng.uniform(6, 20, 3)], 1)
            add(f"3 distinct n={n} #{seed}", base3[np.arange(n) % 3], rng, "degenerate")
            add(f"1 distinct n={n} #{seed}", np.repeat(base3[:1], n, 0), rng, "degenerate")
            if n >= 6:
                base6 = np.stack([rng.uniform(-4, 4, 6), rng.uniform(-2, 2, 6), rng.uniform(6, 20, 6)], 1)
                add(f"6 distinct n={n} #{seed}", base6[rng.permutation(np.arange(n) % 6)], rng, "valid")
    for seed in range(10):
        rng = np.random.default_rng([7, seed])
        P = _plane_points(rng, 5, 0.3)
        P[4] += 1.0 * (np.array([0.0, 1.0, 0.0]) @ _rx(0.3).T)      # 4 on the plane, one 1 m off it
        add(f"4 coplanar + 1 #{seed}", P, rng, "valid")
    return out


def pose_errors(R, t, Ro, to, P):
    """(rotation angle between R and Ro in rad, |to - t| / scene size)."""
    c = np.clip((np.trace(R.T @ Ro) - 1.0) / 2.0, -1.0, 1.0)
    ang = float(np.arccos(c)) if c < 1.0 - 1e-12 else float(np.linalg.norm(Ro - R) / np.sqrt(2.0))
    scale = float(np.max(np.ptp(P, axis=0)))
    return ang, float(np.linalg.norm(to - t)) / max(scale, 1e-300)


def check_epnp(cases, results):
    """results: (ok, R, t) per case.  Returns the (degenerate, valid) counts."""
    nd = nv = 0
    for (name, P, uv, R, t, expect), (ok, Ro, to) in zip(cases, results):
        if not ok:
            assert expect != "valid", name
            nd += 1
            continue
        assert expect != "degenerate", name
        ang, terr = pose_errors(R, t, Ro, to, P)
        assert ang <= 1e-9 and terr <= 1e-9, (name, ang, terr)
        nv += 1
    return nd, nv


def test_epnp_degenerate_sets_are_rejected_or_exact():
    cases = epnp_cases()
    res = [oracle_pnp.epnp(P, uv, KF) for _, P, uv, _, _, _ in cases]
    nd, nv = check_epnp(cases, res)
    print("%d sets: %d degenerate, %d valid and exact" % (len(cases), nd, nv))
    again = [oracle_pnp.epnp(P, uv, KF) for _, P, uv, _, _, _ in cases]
    for (a, Ra, ta), (b, Rb, tb) in zip(res, again):
        assert a == b and np.array_equal(Ra, Rb) and np.array_equal(ta, tb)


def coplanar_sweep():
    """The ground-plane sweep: y = 1.6 tilted about x by 0, 0.3 and 1.0 rad, n = 5, 6, 50, 1000, 40 seeds each."""
    out = []
    for tilt in (0.0, 0.3, 1.0):
        for n in (5, 6, 50, 1000):
            for seed in range(40):
                rng = np.random.default_rng([11, n, seed, int(tilt * 10)])
                P = _plane_points(rng, n, tilt)
                uv, R, t = _project(P, rng)
                out.append((f"sweep tilt={tilt} n={n} #{seed}", P, uv, R, t, "either"))
    return out


def sweep_counts(cases, results):
    fail = wrong = right = 0
    for (name, P, uv, R, t, _), (ok, Ro, to) in zip(cases, results):
        if not ok:
            fail += 1
            continue
        ang, terr = pose_errors(R, t, Ro, to, P)
        if ang <= 1e-9 and terr <= 1e-9:
            right += 1
        else:
            wrong += 1
    return fail, wrong, right


def test_epnp_coplanar_sweep_has_no_wrong_valid_pose():
    cases = coplanar_sweep()
    fail, wrong, right = sweep_counts(cases, [oracle_pnp.epnp(P, uv, KF) for _, P, uv, _, _, _ in cases])
    print("coplanar sweep, %d sets: %d degenerate, %d wrong but valid, %d valid and exact"
          % (len(cases), fail, wrong, right))
    assert wrong == 0


def test_epnp_degeneracy_rule_scales_with_the_set():
    """The rule is relative: the same set scaled by 2^k (exact in fp64, pixels unchanged when the translation scales
    too) gives the same verdict and the scaled pose, bit for bit."""
    for name, P, uv, R, t, expect in epnp_cases()[::5]:
        ok0, R0, t0 = oracle_pnp.epnp(P, uv, KF)
        for k in (-20, 20):
            s = 2.0 ** k
            ok, Rk, tk = oracle_pnp.epnp(P * s, uv, KF)
            assert ok == ok0, name
            if ok:
                assert np.array_equal(Rk, R0) and np.array_equal(tk, t0 * s), name


# ---------------------------------------------------------------------------------------------------------------
# sym3_eig_desc

mpmath.mp.dps = 50


def _qr_rotation(rng):
    Q, Rr = np.linalg.qr(rng.normal(size=(3, 3)))
    return Q * np.sign(np.diag(Rr))


def _sym(Q, d):
    C = Q @ np.diag(d) @ Q.T
    return (C + C.T) / 2.0


def sym3_cases():
    """(name, C [3,3] fp64 symmetric)."""
    rng = np.random.default_rng(5)
    cases = []
    spectra = {
        "triple": (2.0, 2.0, 2.0), "double hi": (3.0, 3.0, 1.0), "double lo": (3.0, 1.0, 1.0),
        "split 1e-15": (1.0 + 1e-15, 1.0, 1.0 - 1e-15), "split 2u": (1.0 + 2 * U, 1.0, 1.0 - 2 * U),
        "rank 1": (5.0, 0.0, 0.0), "rank 2": (5.0, 2.0, 0.0), "rank 2 double": (4.0, 4.0, 0.0),
        "negative rounding": (1.0, 0.5, -1e-17), "negative u": (1.0, 1e-3, -U), "generic": (7.0, 2.5, 0.3),
        "zero": (0.0, 0.0, 0.0),
    }
    for name, d in spectra.items():
        cases.append((name + " diagonal", np.diag(d).astype(np.float64)))
        for r in range(4):
            cases.append((f"{name} rotated #{r}", _sym(_qr_rotation(rng), d)))
    # off-diagonals at the Jacobi skip threshold |apq| <= 1e-17 sqrt(|app| |aqq|), just below and just above
    for a, b in ((1.0, 1.0), (1.0, 1.0 + 1e-15), (4.0, 1.0), (1e-3, 1e3)):
        thr = 1e-17 * np.sqrt(a * b)
        for f in (0.5, 1.0, np.nextafter(1.0, 2.0), 2.0, 1e3):
            for p, q in ((0, 1), (0, 2), (1, 2)):
                d = np.full(3, 0.5 * (a + b))
                d[p], d[q] = a, b
                C = np.diag(d)
                C[p, q] = C[q, p] = thr * f
                cases.append((f"skip a={a} b={b} f={f} ({p},{q})", C))
    for i in range(40):
        cases.append((f"random #{i}", _sym(_qr_rotation(rng), rng.normal(size=3) * 10.0 ** rng.uniform(-3, 3, 3))))
    return cases


def scaled_sym3_cases():
    """Every case scaled by 10^k, k = -80 ... 150 (the documented valid range)."""
    out = []
    for name, C in sym3_cases():
        for k in (-80, -40, 0, 40, 80, 120, 150):
            out.append((f"{name} x1e{k}", C * 10.0 ** k))
    return out


def mp_eig(C):
    """50-digit eigen-decomposition of the fp64 matrix C (exact input): (lam descending [3] mpf, E [3][3] mpf,
    column k the unit eigenvector of lam[k])."""
    A = mpmath.matrix([[mpmath.mpf(float(C[i, j])) for j in range(3)] for i in range(3)])
    ev, Q = mpmath.eigsy(A)
    order = sorted(range(3), key=lambda k: -ev[k])
    return [ev[k] for k in order], [[Q[r, k] for k in order] for r in range(3)]


def check_sym3(name, C, lam, E, ref=None):
    """lam [3], E [3,3] of C against the 50-digit decomposition.  Bounds are in units of u |C|_F."""
    lr, Er = ref if ref is not None else mp_eig(C)
    fro = mpmath.sqrt(mpmath.fsum(mpmath.mpf(float(x)) ** 2 for x in C.reshape(-1)))
    if fro == 0:
        assert np.array_equal(lam, np.zeros(3)) and np.array_equal(E @ E.T, np.eye(3)), name
        return
    scale = U * fro
    assert lam[0] >= lam[1] >= lam[2], (name, lam)
    for k in range(3):
        assert abs(mpmath.mpf(float(lam[k])) - lr[k]) <= 16 * scale, (name, k, lam[k], lr[k])
    assert np.abs(E.T @ E - np.eye(3)).max() <= 16 * U, name
    Em = [[mpmath.mpf(float(E[r, k])) for k in range(3)] for r in range(3)]
    Cm = [[mpmath.mpf(float(C[i, j])) for j in range(3)] for i in range(3)]
    for k in range(3):
        res = mpmath.sqrt(mpmath.fsum((mpmath.fsum(Cm[i][j] * Em[j][k] for j in range(3))
                                       - mpmath.mpf(float(lam[k])) * Em[i][k]) ** 2 for i in range(3)))
        assert res <= 16 * scale, (name, k, res / scale)
        # Davis-Kahan, component by component: the part of e_k along the exact eigenvector of a different eigenvalue
        # is at most |dC| / gap.  Repeated eigenvalues (gap ~ 0) leave only the spanned subspace constrained.
        for j in range(3):
            if j == k:
                continue
            gap = abs(lr[j] - lr[k])
            comp = abs(mpmath.fsum(Er[r][j] * Em[r][k] for r in range(3)))
            if gap > 0:
                assert comp <= 16 * scale / gap, (name, k, j, comp, gap)


def test_sym3_eig_against_50_digit_references():
    cases = scaled_sym3_cases()
    Cs = np.stack([C for _, C in cases])
    lam, E = oracle_pnp.sym3_eig(Cs)
    for (name, C), l, e in zip(cases, lam, E):
        check_sym3(name, C, l, e)


def test_sym3_eig_valid_range_ends_where_the_frobenius_sum_overflows():
    """Entries above about 1e154 overflow sum C_ij^2: the sweeps stop before the first rotation and the diagonal is
    returned.  No caller gets there: normals have |C_ij| <= radius^2 with float32 offsets (below 1e78), and EPnP
    rejects sets whose spread lam[0] reaches 1e75 before solving (DESIGN.md 4.8)."""
    C = _sym(_qr_rotation(np.random.default_rng(9)), (3.0, 2.0, 1.0))
    lam, E = oracle_pnp.sym3_eig(np.stack([C * 1e150, C * 1e155]))
    check_sym3("1e150", C * 1e150, lam[0], E[0])
    assert np.array_equal(E[1], np.eye(3)[:, np.argsort(-np.diag(C), kind="stable")])


# ---------------------------------------------------------------------------------------------------------------
# Normals

def _f32(P):
    return np.ascontiguousarray(np.asarray(P, dtype=np.float64).astype(np.float32))


def normals_clouds():
    """(name, xyz [3,m] float32, radius, max_nn, orient, kind); kind in 'plane', 'line', 'repeated', 'any'."""
    rng = np.random.default_rng(3)
    out = []
    ab = rng.uniform(-1.5, 1.5, (2, 600))
    out.append(("plane x=80", _f32([np.full(600, 80.0), 20 + ab[0], 30 + ab[1]]), 0.6, 30, (0.0, 0.0, 1.0), "plane"))
    n = np.array([1.0, 2.0, 2.0]) / 3.0
    e1 = np.array([2.0, -1.0, 0.0]) / np.sqrt(5.0)
    e2 = np.cross(n, e1)
    c = np.array([50.0, 40.0, 48.0])
    P = c[:, None] + e1[:, None] * ab[0] + e2[:, None] * ab[1]
    out.append(("tilted plane 80 m", _f32(P), 0.6, 30, (0.0, 0.0, 1.0), "plane"))
    az = np.arange(2048) * (2 * np.pi / 2048)
    out.append(("scan ring", _f32([20 * np.cos(az), 20 * np.sin(az), np.full(2048, -1.73)]), 0.6, 30,
                (0.0, 0.0, 1.0), "plane"))
    s = np.arange(200) * 0.05
    out.append(("axis line", _f32([60 + s, np.full(200, 5.0), np.full(200, -1.73)]), 0.6, 30, (0.0, 0.0, 1.0),
                "line"))
    d = np.array([0.48, 0.6, 0.64])
    out.append(("tilted line", _f32(np.array([40.0, 50.0, 45.0])[:, None] + d[:, None] * s), 0.6, 30,
                (0.0, 0.0, 1.0), "line"))
    g = np.arange(-4, 5) * 0.25
    gx, gy, gz = np.meshgrid(g, g, g, indexing="ij")
    out.append(("cubic lattice", _f32([80 + gx.ravel(), 8 + gy.ravel(), -4 + gz.ravel()]), 0.6, 64,
                (0.3, -0.2, 0.9), "repeated"))
    gx, gy = np.meshgrid(np.arange(-6, 7) * 0.25, np.arange(-6, 7) * 0.25, indexing="ij")
    out.append(("square lattice", _f32([10 + gx.ravel(), 20 + gy.ravel(), np.full(gx.size, 75.0)]), 0.6, 64,
                (0.0, 0.0, 1.0), "plane"))
    u1, u2 = rng.uniform(0, 3, (2, 400))
    wall = [np.full(400, 30.0), 10 + u1, 70 + u2]
    floor = [30 + u1[::-1], np.full(400, 10.0), 70 + u2[::-1]]
    out.append(("corner", _f32(np.concatenate([wall, floor], 1)), 0.6, 30, (1.0, 1.0, 0.0), "any"))
    out.append(("normal perpendicular to orient", _f32([20 + ab[0], 30 + ab[1], np.full(600, 80.0)]), 0.6, 30,
                (1.0, 0.0, 0.0), "plane"))
    return out


def neighbours(X, radius, max_nn):
    """Per point: indices of the min(max_nn, c) nearest points with d2 < radius^2, d2 = (dx dx + dy dy) + dz dz in
    fp64 of the float32 coordinates, ties to the lower index; candidates from cKDTree."""
    from scipy.spatial import cKDTree
    P = X.astype(np.float64).T
    tree = cKDTree(P)
    out = []
    for i, cand in enumerate(tree.query_ball_point(P, radius * (1 + 1e-6))):
        cand = np.asarray(sorted(cand), dtype=np.int64)
        d = P[cand] - P[i]
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        keep = d2 < radius * radius
        cand, d2 = cand[keep], d2[keep]
        out.append(cand[np.lexsort((cand, d2))][:max_nn])
    return out


def mp_cov_eig(X, nb):
    """Exact covariance (about the mean) of the neighbours in mpmath and its eigen-decomposition (descending)."""
    pts = [[mpmath.mpf(float(X[a, j])) for a in range(3)] for j in nb]
    k = len(pts)
    m = [mpmath.fsum(p[a] for p in pts) / k for a in range(3)]
    A = mpmath.matrix(3, 3)
    for a in range(3):
        for b in range(3):
            A[a, b] = mpmath.fsum((p[a] - m[a]) * (p[b] - m[b]) for p in pts) / k
    ev, Q = mpmath.eigsy(A)
    order = sorted(range(3), key=lambda q: -ev[q])
    return [ev[q] for q in order], [[Q[r, q] for q in order] for r in range(3)]


def check_normals(name, X, radius, max_nn, orient, kind, nrm, cnt, stride=1):
    """nrm [3,m], cnt [m] of cloud X [3,m] against the exact neighbour sets and covariances (every stride-th point
    for the mpmath part)."""
    o = np.asarray(orient, dtype=np.float64)
    nb = neighbours(X, radius, max_nn)
    assert np.array_equal(cnt, [len(x) for x in nb]), name
    assert np.isfinite(nrm).all(), name
    assert np.abs(np.sqrt((nrm * nrm).sum(0)) - 1.0).max() <= 4 * U, name
    dot = (nrm[0] * o[0] + nrm[1] * o[1]) + nrm[2] * o[2]
    assert (dot >= 0.0).all(), name                                     # n . orient < 0 is flipped
    worst = 0.0
    for i in range(0, X.shape[1], stride):
        if cnt[i] < 3:
            continue
        lr, Er = mp_cov_eig(X, nb[i])
        d = X[:, nb[i]].astype(np.float64) - X[:, i:i + 1].astype(np.float64)
        r2 = float((d * d).sum(0).max())
        eta = (3 * (cnt[i] + 8) + 60) * U * r2           # rounding of the moments and of the Jacobi eigenvalues
        n = [mpmath.mpf(float(x)) for x in nrm[:, i]]
        along = [abs(mpmath.fsum(Er[r][k] * n[r] for r in range(3))) for k in range(3)]
        if kind == "plane" or (kind == "any" and lr[1] - lr[2] > 0):
            gap = lr[1] - lr[2]
            sin = mpmath.sqrt(along[0] ** 2 + along[1] ** 2)
            assert sin <= eta / gap, (name, i, float(sin), float(eta / gap))
            worst = max(worst, float(sin * gap / eta))
        elif kind == "line":
            assert along[0] <= eta / (lr[0] - lr[1]), (name, i, float(along[0]))
    return worst


@pytest.mark.parametrize("case", range(len(normals_clouds())), ids=[c[0] for c in normals_clouds()])
def test_normals_on_degenerate_neighbourhoods(case):
    name, X, radius, max_nn, orient, kind = normals_clouds()[case]
    nrm, cnt = oracle_prep.estimate_normals(X, radius, max_nn, orient)
    worst = check_normals(name, X, radius, max_nn, orient, kind, nrm, cnt, stride=7)
    print("%s: worst angle / bound %.2e" % (name, worst))
    if name == "normal perpendicular to orient":
        assert np.array_equal(np.abs(nrm), np.tile([[0.0], [0.0], [1.0]], (1, X.shape[1])))
    if name == "axis line":
        assert (nrm[0] == 0.0).all()


# ---------------------------------------------------------------------------------------------------------------
# ICP's Umeyama step

def kabsch_ref(src, dst):
    """Rigid least-squares dst ~ R src + t (numpy fp64 SVD, proper rotation).  Returns (R, t)."""
    ms, md = src.mean(0), dst.mean(0)
    A = (dst - md).T @ (src - ms)
    Uu, S, Vt = np.linalg.svd(A)
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(Uu) * np.linalg.det(Vt))])
    R = Uu @ D @ Vt
    return R, md - R @ ms


def icp_frames():
    """(name, src [3,n] f32, tgt [3,n] f32, init [1,4,4], kind) with kind 'rank2', 'rank1' or 'reflect'.  The motion
    is small against the point spacing, so the first pass pairs every source point with its own image."""
    rng = np.random.default_rng(17)
    out = []
    g = np.arange(-5, 5) * 2.0
    gx, gy = np.meshgrid(g, g, indexing="ij")
    for tilt in (0.0, 0.4):
        P = np.stack([gx.ravel() + 0.3, gy.ravel() - 0.2, np.full(gx.size, 0.0)])
        P = _rx(tilt) @ P + np.array([[3.0], [1.0], [12.0]])
        R = _rot(rng, 0.02)
        t = np.array([0.05, -0.03, 0.04])
        out.append((f"plane tilt={tilt}", _f32(P), _f32(R @ _f32(P).astype(np.float64) + t[:, None]), np.eye(4)[None],
                    "rank2"))
    s = np.arange(30) * 1.5
    for d in (np.array([1.0, 0.0, 0.0]), np.array([0.48, 0.6, 0.64])):
        P = np.array([[2.0], [-1.0], [8.0]]) + d[:, None] * s
        R = _rot(rng, 0.004)
        out.append((f"line {d}", _f32(P), _f32(R @ _f32(P).astype(np.float64) + np.array([[0.02], [0.01], [-0.03]])),
                    np.eye(4)[None], "rank1"))
    P = np.stack([rng.uniform(-0.1, 0.1, gx.size), gx.ravel(), gy.ravel() + 10.0])
    M = np.diag([-1.0, 1.0, 1.0])                                       # a mirror: det(A) < 0
    out.append(("mirror", _f32(P), _f32(M @ _f32(P).astype(np.float64)), np.eye(4)[None], "reflect"))
    P = np.stack([gx.ravel() * 0.5, rng.uniform(-0.15, 0.15, gx.size), gy.ravel() + 10.0])
    out.append(("mirror + rotation", _f32(P), _f32(_rot(rng, 0.01) @ np.diag([1.0, -1.0, 1.0]) @ _f32(P)),
                np.eye(4)[None], "reflect"))
    return out


def check_umeyama(name, src, tgt, kind, T):
    """T [4,4] after the first update from init = I."""
    S, D = src.astype(np.float64).T, tgt.astype(np.float64).T
    R, t = T[:3, :3], T[:3, 3]
    assert np.abs(R.T @ R - np.eye(3)).max() <= 1e-14 and abs(np.linalg.det(R) - 1.0) <= 1e-14, name
    scale = float(np.max(np.abs(D)))
    if kind in ("rank2", "reflect"):
        Rr, tr = kabsch_ref(S, D)
        assert np.abs(R - Rr).max() <= 1e-12 and np.abs(t - tr).max() <= 1e-12 * scale, (name, np.abs(R - Rr).max())
    else:
        ds = S[-1] - S[0]
        dd = D[-1] - D[0]
        ds, dd = ds / np.linalg.norm(ds), dd / np.linalg.norm(dd)
        assert np.abs(R @ ds - dd).max() <= 1e-6, name              # the float32 target line is straight to ~1e-7
        assert np.abs(R @ S.mean(0) + t - D.mean(0)).max() <= 1e-12 * scale, name


@pytest.mark.parametrize("case", range(len(icp_frames())), ids=[c[0] for c in icp_frames()])
def test_umeyama_step_against_kabsch(case):
    name, src, tgt, init, kind = icp_frames()[case]
    r = oracle_icp.register_frame(src, tgt, init, max_iteration=1, force_2d=False, trace=True)
    assert r["stats"][0, 0] == 1 and (r["trace_nc"][0] == src.shape[1]).all(), name   # every point keeps its image
    j, _ = oracle_icp.nearest(tgt, src.astype(np.float64).T)
    assert np.array_equal(j, np.arange(src.shape[1])), name
    check_umeyama(name, src, tgt, kind, r["T"][0])
