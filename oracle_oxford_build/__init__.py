"""numpy oracle of the Oxford cloud build's device part -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and the benchmark scripts may import this package; deepi2p_b200 never does.  It
restates DESIGN.md 4.24 one cloud at a time from the host plan of deepi2p_b200.oxford_build.plan_traversal: the skip
walk in Python floats (rel = M_c P_i and the Gauss-Jordan inverse in the kernel's order), the fp64 transform of each
kept scan's masked points in numpy in the kernel's association, oracle_nuscenes' voxel grid and the output transform.
"""
import os

import numpy as np

import oracle_nuscenes


def _dot4(A, r, B, c):
    return ((A[r][0] * B[0][c] + A[r][1] * B[1][c]) + A[r][2] * B[2][c]) + A[r][3] * B[3][c]


def _matmul(A, B):
    return [[_dot4(A, r, B, c) for c in range(4)] for r in range(4)]


def gj_inverse(a):
    """csrc/oxford_build.cu's Gauss-Jordan inverse, restated on its own in Python floats."""
    aug = [[float(a[r][j]) for j in range(4)] + [1.0 if j == r else 0.0 for j in range(4)] for r in range(4)]
    for c in range(4):
        p, best = c, abs(aug[c][c])
        for r in range(c + 1, 4):
            if abs(aug[r][c]) > best:
                p, best = r, abs(aug[r][c])
        aug[c], aug[p] = aug[p], aug[c]
        piv = aug[c][c]
        aug[c] = [v / piv for v in aug[c]]
        for r in range(4):
            if r != c:
                f = aug[r][c]
                aug[r] = [aug[r][j] - f * aug[c][j] for j in range(8)]
    return [row[4:] for row in aug]


def walk(poses, present, lo, hi, M_c, G, skip_threshold):
    """The plan kernel for one window [lo, hi) of absolute poses [n, 4, 4].  Returns (kept indices, their T [k, 3, 4],
    skipped count)."""
    M = [[float(v) for v in row] for row in M_c]
    Gl = [[float(v) for v in row] for row in G]
    kept, Ts, skipped, inv = [], [], 0, None
    for i in range(lo, hi):
        if not present[i]:
            continue
        P = [[float(v) for v in row] for row in poses[i]]
        rel = _matmul(M, P)
        if inv is not None:
            d = [((inv[r][0] * rel[0][3] + inv[r][1] * rel[1][3]) + inv[r][2] * rel[2][3]) + inv[r][3] * rel[3][3]
                 for r in range(3)]
            if float(np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])) < skip_threshold:
                skipped += 1
                continue
        kept.append(i)
        Ts.append(np.array(_matmul(rel, Gl))[:3])
        inv = gj_inverse(rel)
    return kept, np.array(Ts).reshape(-1, 3, 4), skipped


def cloud(scans, kept, Ts, use_mask, threshold, voxel, O):
    """Gather, voxel grid and pack for one cloud.  scans[i] = [3, n] (x, y, reflectance) f64 of LMS index i.
    Returns (record [4, m] float32, n_pts)."""
    xs, rs = [], []
    for i, T in zip(kept, Ts):
        x, y, r = scans[i]
        keep = x < threshold if use_mask else np.ones(x.shape, bool)
        x, y, r = x[keep], y[keep], r[keep]
        z = np.zeros_like(x)
        xs.append(np.stack([((T[a, 0] * x + T[a, 1] * y) + T[a, 2] * z) + T[a, 3] for a in range(3)]))
        rs.append(r)
    p = np.concatenate(xs, 1)
    r = np.concatenate(rs)
    rmax = np.max(r)
    with np.errstate(invalid="ignore", divide="ignore"):
        px, A = oracle_nuscenes.voxel_downsample64(p, voxel, (r / rmax)[None])
    rec = np.stack([((O[a, 0] * px[0] + O[a, 1] * px[1]) + O[a, 2] * px[2]) + O[a, 3] for a in range(3)]
                   + [A[0] * rmax]).astype(np.float32)
    return rec, p.shape[1]


def read_scans(plan, indices):
    """{LMS index: [3, n] f64} for the given indices of plan['lms_ts'] (None for a missing file)."""
    out = {}
    for i in indices:
        path = os.path.join(plan["lidar_dir"], "%d.bin" % plan["lms_ts"][i])
        out[i] = np.fromfile(path, np.double).reshape(-1, 3).T if os.path.isfile(path) else None
    return out


def build_cloud(plan, c, scans=None):
    """Cloud plan['centres'][c] from the host plan.  Returns dict(record [4, m] f32, n_kept, n_skipped, n_pts)."""
    ts, lo, hi, _ = plan["centres"][c]
    p = plan["params"]
    scans = scans if scans is not None else read_scans(plan, range(lo, hi))
    base = plan["lms_lo"]
    present = {i: scans[i] is not None for i in range(lo, hi)}
    poses = {i: plan["lms_abs"][i - base] for i in range(lo, hi)}
    kept, Ts, skipped = walk(poses, present, lo, hi, plan["centre_inv"][c], plan["G_laser"],
                             p["voxel_grid_downsample_size"] / 16.0)
    thr = p["remove_ground_threshold"]
    use_mask = thr is not None and thr > -1
    rec, n = cloud(scans, kept, Ts, use_mask, thr if use_mask else 0.0, p["voxel_grid_downsample_size"], plan["O"])
    return dict(record=rec, n_kept=len(kept), n_skipped=skipped, n_pts=n)
