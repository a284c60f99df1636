"""The solver's fp32 frustum cull at rounding-level distances from the image and depth boundaries (CPU half).

Every cost, gradient and J^T J the registration solver forms first goes through a two-level fp32 cull
(deepi2p_b200/csrc/frustum_solver.cu): box_state() tests each 32-point group's box (frustum_boxes_kernel inflates its
half extent), then maybe_active() tests each point of an undecided group against the five linear forms

    Z > 0,   fx X + cx Z > 0,   fx X + (cx - W1) Z < 0,   fy Y + cy Z > 0,   fy Y + (cy - H1) Z < 0

with a per-point margin built from gamma = 8 * 2^-24 (make_class).  A point may be skipped only when its exact
evaluation contributes zero, so the sums are those of an all-fp64 evaluation (DESIGN 4.3.1).

This module builds adversarial clouds whose points sit at controlled signed distances (1e-9 .. 1e-1 px, or m for the
Z = 0 plane) from those planes, on representable float32 / float64 coordinates, and checks them with exact rational
arithmetic: that they are where they claim to be, that each one changes the sums by far more than the tolerances
of the GPU comparison, and that an exact restatement of the fp32 cull never skips an active one while a cull without
margin would.  tests/test_frustum_cull_gpu.py runs the CUDA kernels on the same clouds against oracle.evaluate.
"""
import functools
import math
from fractions import Fraction

import numpy as np
import pytest

import oracle
from deepi2p_b200 import synthetic as syn

FLOOR = 1e-9                 # px or m: closer than this, device sincos / FMA contraction may decide differently
GAMMA = 8.0 / 16777216.0     # make_class
DBL_EPS = np.finfo(np.float64).eps
PLANES = ("u0", "uW", "v0", "vH", "z0")
EDGES = ("u0", "uW", "v0", "vH", "z0", "u0v0", "u0vH", "uWv0", "uWvH")      # single planes, then image corners
DECADES = tuple(range(-9, 0))            # target |distance| = 10^(k + 1/2)
DEPTHS = (1.2, 15.0, 78.0)               # m, for the image-edge targets
# In front of the camera a label-0 point's u, v and Jacobian carry 1 / Z: at Z = 1e-9 m the fp64 rounding of X (~1e-16
# |t|) moves them by ~1e-7 relative, and two correct fp64 evaluations no longer agree to the 1e-9 tolerance.  Label 0
# is therefore swept over Z >= 1e-5 m only; label 1 behind the camera (residual 100 |Z|, no 1 / Z) over all decades.
DECADES_DEPTH0 = tuple(k for k in DECADES if k >= -5)
COST_TOL, GRAD_TOL = 1e-10, 1e-9         # relative tolerances of test_evaluate_matches_oracle
SENSITIVITY = 100.0                      # each active boundary point moves a sum by >= this x the tolerance

# Poses (x in the solver's layout: 4-DoF (ry, tx, ty, tz), 6-DoF (ax, ay, az, tx, ty, tz)).
POSES = {
    "4dof_ry0": (True, (0.0, 0.4, 0.05, -0.7)),
    "4dof_small": (True, (1e-9, -0.3, 0.02, 1.1)),                   # ry^2 <= DBL_EPSILON: first-order rotation
    "4dof_general": (True, (0.35, 1.2, -0.06, 2.5)),
    "4dof_far": (True, (0.6, 35.0, -4.0, 60.0)),                     # |t| ~ 70 m: the constant-term margin G0 is large
    "6dof_general": (False, (0.04, -0.3, 0.025, 0.8, 0.07, -1.5)),
    "6dof_small": (False, (1e-9, -2e-9, 3e-9, 0.2, -0.05, 0.9)),     # |a|^2 <= DBL_EPSILON
    "6dof_y": (False, (0.0, 0.35, 0.0, 1.2, -0.06, 2.5)),            # a rotation a 6-DoF solve can start from
}
INTRINSICS = {"kitti": syn.KITTI, "oxford": syn.OXFORD}
DTYPES = {"f32": np.float32, "f64": np.float64}
# Each configuration is cut into three clouds ("parts"), because a point near Z = 0 has a Jacobian ~ 1/Z: in one cloud
# with the image-edge points its J^T J would set the scale of the relative tolerance and hide every other point.
#   image:  the image edges and corners, both labels, and the 32-point groups;
#   depth0: the Z = 0 plane, label 0 (active just in front of the camera: a large cost term each);
#   depth1: the Z = 0 plane, label 1 (active just behind it: a J^T J row of weight 100^2 each).
PARTS = ("image", "depth0", "depth1")
CONFIGS = [(p, k, d, q) for p in POSES for k in INTRINSICS for d in DTYPES for q in PARTS]
# Intrinsics whose fp32 coefficients overflow (fx, fy > FLT_MAX): make_class disables the cull and every labelled
# point takes the exact path.  Only the image-edge planes are targeted (their J^T J rows scale with fx^2).
OVERFLOW_K = np.array([[1e39, 0.0, 250.5], [0.0, 1e39, 66.5], [0.0, 0.0, 1.0]])
# The pose is the identity, so that X and Y of a point near the image edges (~1e-36 m) are its stored coordinates.
OVERFLOW_POSES = {"4dof_zero": (True, (0.0, 0.0, 0.0, 0.0)), "6dof_zero": (False, (0.0,) * 6)}
OVERFLOW_CONFIGS = [(p, "overflow", d, "image") for p in OVERFLOW_POSES for d in DTYPES]


def config_id(cfg):
    return "-".join(cfg)


# ------------------------------------------------------------------------------------------------------------------
# Pose and camera, as make_pose / make_cam form them in fp64.
# ------------------------------------------------------------------------------------------------------------------
def pose_rt(is_2d, x):
    x = [float(v) for v in x]
    if is_2d:
        ry = x[0]
        if ry * ry > DBL_EPS:
            c, s = math.cos(ry), math.sin(ry)
        else:
            c, s = 1.0, ry
        R = np.array([[c, 0.0, s], [0.0, 1.0, 0.0], [-s, 0.0, c]])
        return R, np.array(x[1:4])
    ax, ay, az = x[:3]
    th2 = ax * ax + ay * ay + az * az
    if th2 > DBL_EPS:
        th = math.sqrt(th2)
        s, c = math.sin(th), math.cos(th)
        wx, wy, wz = ax / th, ay / th, az / th
        omc = 1.0 - c
        R = np.array([[c + wx * wx * omc, wx * wy * omc - wz * s, wy * s + wx * wz * omc],
                      [wz * s + wx * wy * omc, c + wy * wy * omc, -wx * s + wy * wz * omc],
                      [-wy * s + wx * wz * omc, wx * s + wy * wz * omc, c + wz * wz * omc]])
    else:
        R = np.array([[1.0, -az, ay], [az, 1.0, -ax], [-ay, ax, 1.0]])
    return R, np.array(x[3:6])


def camera(K, H, W):
    K = np.asarray(K, dtype=np.float64)
    return dict(fx=float(K[0, 0]), fy=float(K[1, 1]), cx=float(K[0, 2]), cy=float(K[1, 2]), W1=float(W) - 1.0,
                H1=float(H) - 1.0)


def form_rows(cam):
    """k of the five forms k . (X, Y, Z) in make_class's order: Z, u > 0, u < W1, v > 0, v < H1."""
    return [(0.0, 0.0, 1.0), (cam["fx"], 0.0, cam["cx"]), (cam["fx"], 0.0, cam["cx"] - cam["W1"]),
            (0.0, cam["fy"], cam["cy"]), (0.0, cam["fy"], cam["cy"] - cam["H1"])]


# ------------------------------------------------------------------------------------------------------------------
# Exact evaluation: signed distances and form values as rationals from the stored coordinates and the fp64 R, t.
# ------------------------------------------------------------------------------------------------------------------
def exact_forms(points, R, t, cam):
    """Per point the exact (Z, fx X + cx Z, fx X + (cx - W1) Z, fy Y + cy Z, fy Y + (cy - H1) Z) as Fractions, with
    q = R p + t formed from the stored coordinates and the fp64 R, t (cx - W1 and cy - H1 exact, not rounded)."""
    Rf = [[Fraction(float(v)) for v in row] for row in R]
    tf = [Fraction(float(v)) for v in t]
    fx, fy, cx, cy = (Fraction(cam[k]) for k in ("fx", "fy", "cx", "cy"))
    W1, H1 = Fraction(cam["W1"]), Fraction(cam["H1"])
    cxw, cyh = cx - W1, cy - H1
    out = []
    for px, py, pz in np.asarray(points, dtype=np.float64).T.tolist():
        p = (Fraction(px), Fraction(py), Fraction(pz))
        X = Rf[0][0] * p[0] + Rf[0][1] * p[1] + Rf[0][2] * p[2] + tf[0]
        Y = Rf[1][0] * p[0] + Rf[1][1] * p[1] + Rf[1][2] * p[2] + tf[1]
        Z = Rf[2][0] * p[0] + Rf[2][1] * p[1] + Rf[2][2] * p[2] + tf[2]
        out.append((Z, fx * X + cx * Z, fx * X + cxw * Z, fy * Y + cy * Z, fy * Y + cyh * Z))
    return out


def exact_distances(forms):
    """[N, 5] signed distances, positive on the image side: u, W1 - u, v, H1 - v in px (u = (fx X + cx Z) / Z) and Z in
    m; each rounded once from its exact value, so its sign is exact.  Also the exact 'projects inside' flag."""
    d = np.empty((len(forms), 5))
    inside = np.empty(len(forms), dtype=bool)
    for i, (Z, al, ah, bl, bh) in enumerate(forms):
        if Z != 0:
            d[i, :4] = [float(al / Z), float(-ah / Z), float(bl / Z), float(-bh / Z)]
        else:
            d[i, :4] = np.nan
        d[i, 4] = float(Z)
        inside[i] = Z > 0 and al > 0 and ah < 0 and bl > 0 and bh < 0
    return d, inside


# ------------------------------------------------------------------------------------------------------------------
# Generator.
# ------------------------------------------------------------------------------------------------------------------
def _ulp_walk(v, n):
    """[..., 2n+1]: v stepped by -n .. n ulps of its own dtype (np.nextafter)."""
    inf = v.dtype.type(np.inf)
    out = np.empty(v.shape + (2 * n + 1,), dtype=v.dtype)
    out[..., n] = v
    up, dn = v.copy(), v.copy()
    for k in range(1, n + 1):
        up = np.nextafter(up, inf)
        dn = np.nextafter(dn, -inf)
        out[..., n + k] = up
        out[..., n - k] = dn
    return out


def _approx_distances(P, R, t, cam):
    """fp64 estimate of the five signed distances of points P [..., 3] (selection only; kept points are re-checked
    exactly)."""
    P = P.astype(np.float64)
    q = P @ R.T + t
    X, Y, Z = q[..., 0], q[..., 1], q[..., 2]
    with np.errstate(divide="ignore", invalid="ignore"):
        u = cam["fx"] * X / Z + cam["cx"]
        v = cam["fy"] * Y / Z + cam["cy"]
    return np.stack([u, cam["W1"] - u, v, cam["H1"] - v, Z], -1)


def _edge_planes(edge):
    if edge == "z0":
        return [4]
    idx = {"u0": 0, "uW": 1, "v0": 2, "vH": 3}
    return [idx[edge[:2]]] + ([idx[edge[2:]]] if len(edge) == 4 else [])


def _candidates(R, t, cam, dtype, edges, signs, mags, depths, rng, walk):
    """For each target (edge, signs per targeted plane, |distance|, depth): the fp64 back-projection rounded to dtype
    and its (2 walk + 1)^2 neighbours along the two coordinates that move the targeted form(s) most.  Returns the
    candidate points [T, M, 3] and their approximate distances [T, M, 5]."""
    T = len(edges)
    u = np.empty(T); v = np.empty(T); Z = np.empty(T)
    coef = np.stack([cam["fx"] * R[0] + cam["cx"] * R[2], cam["fx"] * R[0] + cam["cx"] * R[2],
                     cam["fy"] * R[1] + cam["cy"] * R[2], cam["fy"] * R[1] + cam["cy"] * R[2], R[2]])
    ax_a = np.empty(T, dtype=np.int64); ax_b = np.empty(T, dtype=np.int64)
    for i, (e, sg, m, z) in enumerate(zip(edges, signs, mags, depths)):
        u[i] = rng.uniform(0.2, 0.8) * cam["W1"]
        v[i] = rng.uniform(0.2, 0.8) * cam["H1"]
        Z[i] = z
        pl = _edge_planes(e)
        for p, s in zip(pl, sg):
            d = s * m
            if p == 0: u[i] = d
            elif p == 1: u[i] = cam["W1"] - d
            elif p == 2: v[i] = d
            elif p == 3: v[i] = cam["H1"] - d
            else: Z[i] = d
        order = np.argsort(-np.abs(coef[pl[0]]))
        ax_a[i] = order[0]
        if len(pl) == 2:
            o2 = [j for j in np.argsort(-np.abs(coef[pl[1]])) if j != order[0]]
            ax_b[i] = o2[0]
        else:
            ax_b[i] = order[1]
    X = (u - cam["cx"]) * Z / cam["fx"]
    Y = (v - cam["cy"]) * Z / cam["fy"]
    p = (np.stack([X, Y, Z], 1) - t) @ R                  # R^T (q - t)
    base = p.astype(dtype)
    n = 2 * walk + 1
    cand = np.empty((T, n, n, 3), dtype=dtype)
    for c in range(3):
        w = _ulp_walk(base[:, c], walk)
        cand[..., c] = np.where((ax_a == c)[:, None, None], w[:, :, None],
                                np.where((ax_b == c)[:, None, None], w[:, None, :], base[:, c][:, None, None]))
    cand = cand.reshape(T, n * n, 3)
    return cand, _approx_distances(cand, R, t, cam)


def _valid(dist, edge, sg, interior=1.0):
    """Candidate mask: each targeted plane on its intended side by >= 2 FLOOR, every other plane on the image side by
    a clear margin (so that the point's state is decided by the targeted planes alone)."""
    pl = _edge_planes(edge)
    ok = np.ones(dist.shape[:-1], dtype=bool)
    for p in range(5):
        if p in pl:
            ok &= sg[pl.index(p)] * dist[..., p] >= 2 * FLOOR
        elif p == 4:
            ok &= dist[..., 4] >= 0.5
        else:
            ok &= dist[..., p] >= interior
    return ok


@functools.lru_cache(maxsize=None)
def boundary_cloud(pose, intr, dt, part, seed=0):
    """Adversarial cloud for one (pose, intrinsics, record dtype) configuration.

    Groups of 32 consecutive points come first (evaluate_batch cuts unsorted input into such groups):
      * 'pure':     per image edge and label, 32 ulp-neighbours on the ACTIVE side of the edge, as close to it as
                    the coordinates allow (well inside the fp32 error: the box level must not skip them);
      * 'straddle': per image edge and label, the 16 closest representable points on each side;
      * 'mixed':    per image edge, 32 near points with alternating labels, every 8th one ignored (label 5).
    Then the decade sweep ('target'): per edge or corner, label, depth, decade k in DECADES and sign, the candidate
    on the intended side whose exact distance is closest (in log) to 10^(k + 1/2).  Where the record's coordinate
    lattice is coarser than the target, that is the representable point with the smallest distance on that side:
    the first point a margin that is too small misclassifies.

    Returns dict(points [3, N] dtype, labels [N] int32, edge [N] (index into EDGES), sign [N, 2] (intended side of
    each targeted plane, 0 = none), decade [N] (target decade, -99 for groups), kind [N] str, dist [N, 5] exact
    signed distances, inside [N] exact, forms (exact Fractions), K, H, W, x (6), is_2d, R, t).
    """
    is_2d, x = POSES[pose] if pose in POSES else OVERFLOW_POSES[pose]
    if intr == "overflow":
        K, H, W = OVERFLOW_K, syn.KITTI["H"], syn.KITTI["W"]
    else:
        K, H, W = INTRINSICS[intr]["K"], INTRINSICS[intr]["H"], INTRINSICS[intr]["W"]
    edges_sweep = ["z0"] if part != "image" else [e for e in EDGES if e != "z0"]
    # far from the origin a point at 1.2 m has a J^T J ~ (fx |t| / Z)^2 that would hide one at 78 m
    depths = DEPTHS if pose != "4dof_far" else (20.0, 60.0)
    dtype = DTYPES[dt]
    walk = 20 if dtype == np.float32 else 6
    R, t = pose_rt(is_2d, x)
    cam = camera(K, H, W)
    rng = np.random.default_rng(1000 * seed + 17 * CONFIGS_INDEX.get((pose, intr, dt, part), 99) + 5)
    pts, labs, edge_i, signs, decs, kinds = [], [], [], [], [], []

    def add(p, lab, e, sg, dec, kind):
        pts.append(np.asarray(p, dtype=dtype)); labs.append(lab); edge_i.append(EDGES.index(e))
        signs.append(tuple(sg) + (0,) * (2 - len(sg))); decs.append(dec); kinds.append(kind)

    # --- groups of 32 (image part) ----------------------------------------------------------------------------
    tiny = 10.0 ** -8.5

    def nearest(e, side, count, depth):
        cand, dist = _candidates(R, t, cam, dtype, [e], [(side,)], [tiny], [depth], rng, walk)
        p = _edge_planes(e)[0]
        idx = np.nonzero(_valid(dist[0], e, (side,)))[0]
        idx = idx[np.argsort(np.abs(dist[0][idx, p]))][:count]
        assert len(idx) == count, (e, side)
        return [(cand[0][i], side, abs(dist[0][i, p])) for i in idx]

    for e in (("u0", "uW", "v0", "vH") if part == "image" else ()):
        for lab in (0, 1):
            active_side = 1 if lab == 0 else -1            # label 0 is active inside the image, label 1 outside
            for q, side, _ in nearest(e, active_side, 32, 15.0):
                add(q, lab, e, (side,), -99, "pure")
            for q, side, _ in nearest(e, 1, 16, 15.0) + nearest(e, -1, 16, 15.0):
                add(q, lab, e, (side,), -99, "straddle")
        sel = sorted(nearest(e, 1, 16, 9.0) + nearest(e, -1, 16, 9.0), key=lambda c: c[2])
        for j, (q, side, _) in enumerate(sel):
            add(q, 5 if j % 8 == 7 else j % 2, e, (side,), -99, "mixed")

    # --- decade sweep -------------------------------------------------------------------------------------------
    T_e, T_s, T_m, T_z, T_lab, T_dec = [], [], [], [], [], []
    for e in edges_sweep:
        npl = len(_edge_planes(e))
        for lab in (0, 1) if part == "image" else (int(part[-1]),):
            for z in (depths if e != "z0" else (None,) * 4):       # Z = 0 plane: four interior (u, v) per decade
                for k in (DECADES if part != "depth0" else DECADES_DEPTH0):
                    for s in (1, -1):
                        sg = (s,) if npl == 1 else (s, s if k % 2 else -s)
                        T_e.append(e); T_s.append(sg); T_m.append(10.0 ** (k + 0.5)); T_lab.append(lab)
                        T_dec.append(k)
                        T_z.append(z if z is not None else 0.0)
    cand, dist = _candidates(R, t, cam, dtype, T_e, T_s, T_m, T_z, rng, walk)
    for i in range(len(T_e)):
        e, sg, m = T_e[i], T_s[i], T_m[i]
        ok = _valid(dist[i], e, sg)
        if not ok.any():
            continue                                     # not reachable on this record's lattice (Z = 0 plane)
        pl = _edge_planes(e)
        with np.errstate(divide="ignore"):
            score = np.max(np.abs(np.log10(np.abs(dist[i][:, pl])) - math.log10(m)), axis=1)
        score[~ok] = np.inf
        j = int(np.argmin(score))
        add(cand[i, j], T_lab[i], e, sg, T_dec[i], "target")

    points = np.stack(pts, 1)
    forms = exact_forms(points, R, t, cam)
    d, inside = exact_distances(forms)
    x6 = np.zeros(6)
    x6[:len(x)] = x
    return dict(points=points, labels=np.array(labs, dtype=np.int32), edge=np.array(edge_i),
                sign=np.array(signs, dtype=np.int64), decade=np.array(decs), kind=np.array(kinds), dist=d,
                inside=inside, forms=forms, K=np.asarray(K, dtype=np.float64), H=H, W=W, x=x6, is_2d=is_2d, R=R, t=t,
                cam=cam)


CONFIGS_INDEX = {c: i for i, c in enumerate(CONFIGS)}


def active_mask(cl):
    lab = cl["labels"]
    return ((lab == 0) & cl["inside"]) | ((lab == 1) & ~cl["inside"])


@functools.lru_cache(maxsize=None)
def _noise(cfg, is_2d, x):
    cl = boundary_cloud(*cfg)
    P = 4 if is_2d else 6
    x = np.asarray(x)
    bg, bA = np.zeros(P), np.zeros((P, P))
    d = cl["dist"]
    pts = cl["points"].astype(np.float64)
    for i in np.nonzero((cl["labels"] == 0) & cl["inside"])[0]:
        xd, yd = min(d[i, 0], d[i, 1]), min(d[i, 2], d[i, 3])
        _, gi, Ai = oracle.evaluate(pts[:, i:i + 1], cl["labels"][i:i + 1], cl["K"], x[:P], cl["H"], cl["W"], is_2d)
        f = 8 * DBL_EPS * (xd + yd) * (1 / xd + 1 / yd)
        bg += f * np.abs(gi)
        bA += f * np.abs(Ai)
    return bg, bA


def oracle_noise(cfg, x, is_2d):
    """Bound on the oracle's own rounding error in g and J^T J at x.  The reference forms a label-0 residual as
    (xd + yd) * (max(xd, 0) / xd) * (max(yd, 0) / yd); in exact arithmetic the indicator factors have zero derivative,
    but their dual-number derivative is a difference of two terms of size |d xd| / xd, so a point xd px inside an
    image edge carries an error ~ eps (xd + yd) / xd relative to its own J (the CUDA kernel differentiates the
    indicator as exactly zero; measured on an H100: 3.6e-5 in a gradient entry of 7 at xd = 3e-9 px).  Returns
    per-entry bounds (g [P], J^T J [P, P]): 8 eps (xd + yd) (1 / xd + 1 / yd) |contribution|, summed over the active
    label-0 points."""
    return _noise(tuple(cfg), bool(is_2d), tuple(float(v) for v in x))


# ------------------------------------------------------------------------------------------------------------------
# fp32 model of the cull: make_class, maybe_active and box_state restated with correctly rounded fp32 / fp64 FMAs.
# ------------------------------------------------------------------------------------------------------------------
def fma64(a, b, c):
    """Correctly rounded fp64 fma (exact rational, one rounding)."""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def fmaf(a, b, c):
    """Correctly rounded fp32 fma, vectorised: a * b is exact in fp64 (24 + 24 bits), TwoSum gives p + c = s + e
    exactly, and the fp32 rounding of s + e equals that of s unless s is a fp32 midpoint, where the sign of e
    decides (rounding s + e through fp64 would round twice)."""
    a = np.asarray(a, dtype=np.float32); b = np.asarray(b, dtype=np.float32); c = np.asarray(c, dtype=np.float32)
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        s = p + c64
        bp = s - p
        e = (p - (s - bp)) + (c64 - bp)
        r = s.astype(np.float32)
        r64 = r.astype(np.float64)
        other = np.nextafter(r, np.where(s > r64, np.float32(np.inf), np.float32(-np.inf)))
        o64 = other.astype(np.float64)
        mid = (s != r64) & ((s - r64) == (o64 - s))
        fix = mid & (e != 0) & (np.sign(e) == np.sign(o64 - r64))
    return np.where(fix, other, r)


def make_class(R, t, cam):
    """make_class (frustum_solver.cu): fp32 coefficients of the five forms [5, 4] (column 3 the constant), the margin
    scales G, G0 and the enabled flag."""
    rows = form_rows(cam)
    c = np.empty((5, 4))
    for f, (kx, ky, kz) in enumerate(rows):
        for j in range(4):
            a0, a1, a2 = (R[0, j], R[1, j], R[2, j]) if j < 3 else (t[0], t[1], t[2])
            c[f, j] = fma64(kx, a0, fma64(ky, a1, kz * a2))
    with np.errstate(over="ignore"):
        cf = c.astype(np.float32)
        amax = np.abs(c[:, :3]).max()
        cmax = np.abs(c[:, 3]).max()
        G = np.float32(GAMMA * amax * 1.0000002)
        G0 = np.float32(np.float32(GAMMA * cmax * 1.0000002) + np.float32(1e-30))
    enabled = bool(np.isfinite(cf).all() and np.isfinite(G) and np.isfinite(G0))
    return dict(c=cf, G=G, G0=G0, enabled=enabled, c64=c)


def point_forms_f32(x, y, z, cc, is_2d):
    """The five fp32 form values of maybe_active (the 4-DoF variant drops the y terms of Z, u > 0 and u < W1, whose
    coefficients are exactly zero)."""
    c = cc["c"]
    out = []
    for f in range(5):
        if is_2d and f < 3:
            out.append(fmaf(c[f, 0], x, fmaf(c[f, 2], z, c[f, 3])))
        else:
            out.append(fmaf(c[f, 0], x, fmaf(c[f, 1], y, fmaf(c[f, 2], z, c[f, 3]))))
    return out


def maybe_active(points, labels, cc, is_2d, margin=True):
    """maybe_active (frustum_solver.cu) on the record's coordinates (rounded to fp32 as the kernel does).  Returns
    (flags, the fp32 forms [5, N], the margins m)."""
    x, y, z = (np.asarray(points[k]).astype(np.float32) for k in range(3))
    lab = np.asarray(labels)
    with np.errstate(over="ignore"):
        m = fmaf(cc["G"], (np.abs(x) + np.abs(y)) + np.abs(z), cc["G0"])
    F = point_forms_f32(x, y, z, cc, is_2d)
    mm = m if margin else np.zeros_like(m)
    Z, al, ah, bl, bh = F
    lo4 = np.minimum(np.minimum(al, -ah), np.minimum(bl, -bh))
    front = Z > mm
    inside = front & (lo4 > mm)
    outside = (Z < -mm) | (front & (lo4 < -mm))
    act = np.where(lab == 1, ~inside, ~outside)
    lab_ok = (lab == 0) | (lab == 1)
    return lab_ok & (act if cc["enabled"] else True), np.stack(F), m


def box_record(gp, variant):
    """frustum_boxes_kernel's fp32 centre and half extent of one group (gp [3, n] in the record's dtype).  The half
    extent  hd * 1.000001 + (|cd| + hd) * 1.3e-7 + 1e-30  is formed in fp64; --fmad=true may contract either product
    into the first addition, so variant 0 rounds every operation and variants 1 / 2 contract one product."""
    cf = np.empty(3, dtype=np.float32); hf = np.empty(3, dtype=np.float32)
    for c in range(3):
        lo, hi = float(gp[c].astype(np.float64).min()), float(gp[c].astype(np.float64).max())
        cd = 0.5 * (lo + hi)
        cf[c] = np.float32(cd)
        hd = max(hi - float(cf[c]), float(cf[c]) - lo)
        a, b = abs(cd) + hd, hd
        if variant == 0:
            s = b * 1.000001 + a * 1.3e-7
        elif variant == 1:
            s = fma64(b, 1.000001, a * 1.3e-7)
        else:
            s = fma64(a, 1.3e-7, b * 1.000001)
        hf[c] = np.float32(s + 1e-30)
    return cf, hf


def box_state(cf, hf, flags, cc, margin=True):
    """box_state (frustum_solver.cu): 0 skip, 1 undecided, 2 surely active."""
    if flags == 0:
        return 0
    if not cc["enabled"]:
        return 1
    cx, cy, cz = (np.float32(v) for v in cf)
    hx, hy, hz = (np.float32(v) for v in hf)
    s = ((np.abs(cx) + hx) + (np.abs(cy) + hy)) + (np.abs(cz) + hz)
    m = np.float32(2.0) * fmaf(cc["G"], s, cc["G0"]) if margin else np.float32(0.0)
    lo, hi = [], []
    for k in range(5):
        c = cc["c"][k]
        mid = fmaf(c[0], cx, fmaf(c[1], cy, fmaf(c[2], cz, c[3])))
        rad = fmaf(np.abs(c[0]), hx, fmaf(np.abs(c[1]), hy, np.float32(np.abs(c[2]) * hz)))
        lo.append(np.float32(mid - rad)); hi.append(np.float32(mid + rad))
    front = lo[0] > m
    all_out = (hi[0] < -m) or (front and min(min(hi[1], -lo[2]), min(hi[3], -lo[4])) < -m)
    all_in = front and min(min(lo[1], -hi[2]), min(lo[3], -hi[4])) > m
    skip = ((not (flags & 1)) or all_out) and ((not (flags & 2)) or all_in)
    if skip:
        return 0
    return 2 if ((flags == 1 and all_in) or (flags == 2 and all_out)) else 1


def groups_of(cl):
    lab = cl["labels"]
    n = len(lab)
    for g in range(0, n, 32):
        sl = slice(g, min(g + 32, n))
        yield sl, lab[sl]


# ------------------------------------------------------------------------------------------------------------------
# Tests.
# ------------------------------------------------------------------------------------------------------------------
ALL_CONFIGS = CONFIGS + OVERFLOW_CONFIGS


@pytest.mark.parametrize("cfg", ALL_CONFIGS, ids=config_id)
def test_placement(cfg):
    """Every point's exact signed distance to each targeted plane has the intended sign, is >= FLOOR, and is no
    farther than the intended decade; float64 records (whose lattice is fine enough) hit the decade itself, float32
    ones down to 1e-4 px and below that come as close as the lattice allows; every untargeted plane is on the image
    side."""
    cl = boundary_cloud(*cfg)
    d = cl["dist"]
    assert np.isfinite(d).all()
    f64 = cfg[2] == "f64"
    hit = {}
    for i in range(len(cl["labels"])):
        e = EDGES[cl["edge"][i]]
        pl = _edge_planes(e)
        for p in range(5):
            if p in pl:
                s = cl["sign"][i, pl.index(p)]
                assert s * d[i, p] >= FLOOR, (i, e, p, d[i, p])
            elif p == 4:
                assert d[i, 4] > 0.25, (i, e)
            else:
                assert d[i, p] > 0.5, (i, e, p, d[i, p])
        k = cl["decade"][i]
        if k == -99:
            continue
        got = max(math.floor(math.log10(abs(d[i, p]))) for p in pl)
        if f64 or k >= -4:
            assert got == k, (i, e, k, d[i, pl])
        else:
            assert got <= -4, (i, e, k, d[i, pl])      # as close as the float32 lattice allows
        hit.setdefault(e, set()).add(got)
    for e, ks in hit.items():
        lowest = min(ks)
        if e == "z0":
            assert lowest <= (-8 if f64 and cfg[3] == "depth1" else -4), (e, sorted(ks))
        else:
            assert lowest <= (-9 if f64 else -6), (e, sorted(ks))
    # the Z = 0 plane is reachable on the float64 lattice at every decade
    if f64 and "z0" in hit:
        assert hit["z0"] == set(DECADES if cfg[3] == "depth1" else DECADES_DEPTH0)


@pytest.mark.parametrize("cfg", ALL_CONFIGS, ids=config_id)
def test_boundary_points_matter(cfg):
    """Each exactly-active boundary point, evaluated alone by the oracle, moves the cloud's cost by >= 100 x its
    tolerance (1e-10 relative) or some J^T J entry by >= 100 x the J^T J tolerance (1e-9 relative, as
    assert_allclose applies it, plus the oracle's own rounding bound oracle_noise): a cull that dropped any one of
    them fails the GPU comparison."""
    cl = boundary_cloud(*cfg)
    is_2d = cl["is_2d"]
    P = 4 if is_2d else 6
    pts = cl["points"].astype(np.float64)
    c_tot, _, A_tot = oracle.evaluate(pts, cl["labels"], cl["K"], cl["x"][:P], cl["H"], cl["W"], is_2d)
    ctol = COST_TOL * max(1.0, abs(c_tot))
    atol = GRAD_TOL * (np.abs(A_tot).max() + np.abs(A_tot)) + oracle_noise(cfg, cl["x"], is_2d)[1]
    act = np.nonzero(active_mask(cl))[0]
    assert len(act) > 0.3 * len(cl["labels"])
    worst = np.inf
    for i in act:
        c, _, A = oracle.evaluate(pts[:, i:i + 1], cl["labels"][i:i + 1], cl["K"], cl["x"][:P], cl["H"], cl["W"],
                                  is_2d)
        ratio = max(c / ctol, (np.abs(A) / atol).max())
        worst = min(worst, ratio)
        assert ratio >= SENSITIVITY, (i, EDGES[cl["edge"][i]], cl["labels"][i], cl["dist"][i], c, ratio)
    print("%s: %d active boundary points, weakest moves a sum by %.3g x its tolerance" % (config_id(cfg), len(act), worst))


# Non-vacuity: per (edge, label), at least this many points whose fp32 form has the wrong sign (and that a cull
# without a margin therefore drops while they are active).  Stated per record: float32 clouds on float32 coordinates,
# float64 clouds additionally through the input rounding.
MIN_WRONG_SIGN = 4
MIN_NO_MARGIN_DROPS = 40          # per image-part cloud, all edges and labels together
MIN_INPUT_FLIPS = 2
MIN_WRONG_SIGN_Z0 = 4


@pytest.mark.parametrize("cfg", ALL_CONFIGS, ids=config_id)
def test_fp32_point_cull_model(cfg):
    """Exact restatement of make_class / maybe_active on the adversarial points:
    (a) no point whose exact evaluation is active is skipped;
    (b) |fp32 form - exact form| <= m / 1.6 for every form of every point (DESIGN 4.3.1's claim);
    (c) the sets are not vacuous: per image edge and label, points whose fp32 form has the wrong sign, and active
        points that the same test with m = 0 would skip."""
    cl = boundary_cloud(*cfg)
    cc = make_class(cl["R"], cl["t"], cl["cam"])
    if cfg[1] == "overflow":
        assert not cc["enabled"]               # fx, fy > FLT_MAX: the cull is off, every labelled point is evaluated
        flags, _, _ = maybe_active(cl["points"], cl["labels"], cc, cl["is_2d"])
        assert flags[(cl["labels"] == 0) | (cl["labels"] == 1)].all()
        return
    assert cc["enabled"]
    flags, F, m = maybe_active(cl["points"], cl["labels"], cc, cl["is_2d"])
    act = active_mask(cl)
    missed = np.nonzero(act & ~flags)[0]
    assert len(missed) == 0, [(i, EDGES[cl["edge"][i]], cl["labels"][i], cl["dist"][i]) for i in missed[:5]]

    # (b) exact error of every fp32 form against its exact value at the stored (unrounded) coordinates
    worst = 0.0
    wrong = np.zeros((len(cl["labels"]), 5), dtype=bool)
    for i, fe in enumerate(cl["forms"]):
        mi = Fraction(float(m[i]))
        for f in range(5):
            err = abs(Fraction(float(F[f, i])) - fe[f])
            worst = max(worst, float(err / mi))
            wrong[i, f] = (F[f, i] > 0) != (fe[f] > 0) and fe[f] != 0
    assert worst <= 1 / 1.6, worst

    # (c) non-vacuity per edge and label
    nomargin, _, _ = maybe_active(cl["points"], cl["labels"], cc, cl["is_2d"], margin=False)
    drops = act & ~nomargin
    form_of = {"u0": 1, "uW": 2, "v0": 3, "vH": 4, "z0": 0}
    report = []
    edges = ("u0", "uW", "v0", "vH") if cfg[3] == "image" else ("z0",)
    for e in edges:
        for lab in (0, 1) if cfg[3] == "image" else (int(cfg[3][-1]),):
            sel = (cl["labels"] == lab) & np.array([EDGES[k].startswith(e) or EDGES[k].endswith(e)
                                                     for k in cl["edge"]])
            nw = int((wrong[:, form_of[e]] & sel).sum())
            nd = int((drops & sel).sum())
            report.append("%s/%d: %d wrong-sign, %d no-margin drops" % (e, lab, nw, nd))
            if e != "z0":
                assert nw >= MIN_WRONG_SIGN, (e, lab, nw)

            elif cfg[2] == "f64" and cfg[3] == "depth1":
                # float32 coordinates reach Z within the fp32 error only close to the origin: not asserted there
                assert nw >= MIN_WRONG_SIGN_Z0, (e, lab, nw)
    flips = 0
    if cfg[2] == "f64":
        # the record's coordinates rounded to fp32 land on the other side of a targeted plane: only the input-rounding
        # term of the margin keeps these points
        R, t, cam = cl["R"], cl["t"], cl["cam"]
        rounded = exact_forms(cl["points"].astype(np.float32), R, t, cam)
        for i in range(len(cl["labels"])):
            for p in _edge_planes(EDGES[cl["edge"][i]]):
                f = form_of[PLANES[p]]
                flips += int((rounded[i][f] > 0) != (cl["forms"][i][f] > 0))
        report.append("%d fp32-rounding side flips" % flips)
        if cfg[3] == "image":
            assert flips >= MIN_INPUT_FLIPS
    if cfg[3] == "image":
        assert int(drops.sum()) >= MIN_NO_MARGIN_DROPS
    print("%s: worst |fp32 - exact| / m = %.3f; %s; no-margin drops total %d"
          % (config_id(cfg), worst, "; ".join(report), int(drops.sum())))


@pytest.mark.parametrize("cfg", CONFIGS, ids=config_id)
def test_box_cull_model(cfg):
    """box_state with the box of frustum_boxes_kernel (each contraction variant of the inflation) never skips a group
    that holds an exactly-active point; reports how many label-pure groups the same test without its margin skips
    wrongly."""
    cl = boundary_cloud(*cfg)
    cc = make_class(cl["R"], cl["t"], cl["cam"])
    act = active_mask(cl)
    pts = cl["points"]
    wrong_nomargin = {0: 0, 1: 0, 2: 0}
    pure = 0
    for sl, lab in groups_of(cl):
        flags = (1 if (lab == 0).any() else 0) | (2 if (lab == 1).any() else 0)
        keep = (lab == 0) | (lab == 1)
        if not keep.any():
            continue
        gp = pts[:, sl][:, keep]
        has_active = bool(act[sl][keep].any())
        pure += int(flags in (1, 2))
        for variant in (0, 1, 2):
            cf, hf = box_record(gp, variant)
            # the fp32 box contains every point of the group
            for c in range(3):
                lo = Fraction(float(cf[c])) - Fraction(float(hf[c]))
                hi = Fraction(float(cf[c])) + Fraction(float(hf[c]))
                assert all(lo <= Fraction(float(v)) <= hi for v in gp[c])
            st = box_state(cf, hf, flags, cc)
            assert not (has_active and st == 0), (sl, variant)
            if flags in (1, 2) and has_active and box_state(cf, hf, flags, cc, margin=False) == 0:
                wrong_nomargin[variant] += 1
    print("%s: label-pure groups %d; wrongly skipped by box_state without margin: %s (inflation rounded / "
          "contracted variants)" % (config_id(cfg), pure, wrong_nomargin))
