"""CPU statistics for a form-selective point classification (DESIGN 8, item 3: tried, slower on the H100): which of the
five activity forms (Z > 0, u > 0, u < W1, v > 0, v < H1) the undecided 32-point groups still straddle after the box
test, and how many forms a per-point fp32 classification would evaluate per point: five today, and with the form
subsets below.

Same clouds, orders and poses as cull_model.py (the shipped (x, z) Morton order; the inits of each sample and its
ground-truth pose, around which most passes of a solve are spent).  The box test is box_state in float64 without the
fp32 margins; a form is dropped when the box bound puts every point of the group on its inside side, and when an image
form lies wholly on its outside side only that one of the four image forms is kept (--inside-only: the first rule alone).  Groups
are dealt to rounds and paired into classification steps (DIB_GPS = 2, surely-active groups first) as in the kernel.

    python tests/tools/formmask_stats.py --samples 8 --inits 60
"""
import argparse
import collections
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import cull_model as cm  # noqa: E402
import oracle  # noqa: E402
from deepi2p_b200 import synthetic as syn  # noqa: E402

FORM_NAMES = ("Z", "u0", "uW", "v0", "vH")
GPS = 2


def mask_name(m):
    return "+".join(FORM_NAMES[k] for k in range(5) if m >> k & 1) or "-"


def step_class(m):
    """Forms evaluated per point for a step whose OR-ed mask is m, in the scheme that was measured: all five when the
    step needs both u forms or both v forms, else one u form, one v form and Z if the mask holds it."""
    if (m & 0b00110) == 0b00110 or (m & 0b11000) == 0b11000:
        return 5
    return 2 + (m & 1)


def pass_masks(p, lab, order, K, H, W, xpose, inside_only=False):
    p = p[:, order]; lab = lab[order]
    n = p.shape[1]; G = (n + 31) // 32
    pad = G * 32 - n
    pp = np.concatenate([p, np.full((3, pad), np.nan)], 1).reshape(3, G, 32)
    ll = np.concatenate([lab, np.full(pad, -1)]).reshape(G, 32)
    lo = np.nanmin(pp, 2); hi = np.nanmax(pp, 2)
    ctr = 0.5 * (lo + hi); half = 0.5 * (hi - lo)
    flo, fhi = [], []
    for a, c0 in cm.forms(K, H, W, xpose):
        mid = a @ ctr + c0; rad = np.abs(a) @ half
        flo.append(mid - rad); fhi.append(mid + rad)
    has0 = (ll == 0).any(1); has1 = (ll == 1).any(1)
    front = flo[0] > 0
    all_out = (fhi[0] < 0) | (front & (np.minimum(np.minimum(fhi[1], -flo[2]), np.minimum(fhi[3], -flo[4])) < 0))
    all_in = front & (np.minimum(np.minimum(flo[1], -fhi[2]), np.minimum(flo[3], -fhi[4])) > 0)
    skip = (~has0 | all_out) & (~has1 | all_in)
    sure = ~skip & ((has0 & ~has1 & all_in) | (has1 & ~has0 & all_out))
    und = ~skip & ~sure
    proven = [flo[0] > 0, flo[1] > 0, fhi[2] < 0, flo[3] > 0, fhi[4] < 0]    # inside side of each form
    out = [None, fhi[1] < 0, flo[2] > 0, fhi[3] < 0, flo[4] > 0]              # outside side of an image form
    mask = sum(((~proven[k]).astype(np.int64) << k) for k in range(5))
    if not inside_only:
        # an image form on its outside side for every point decides the image test alone: keep it, drop the others
        img = np.zeros_like(mask)
        for k in (4, 3, 2, 1):
            img = np.where(out[k], 1 << k, img)
        mask = np.where(img != 0, (mask & 1) | img, mask)
    mask = np.where(has0 & has1, 0b11111, mask)                               # mixed-label groups: all five forms
    return G, und, sure, mask


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=8)
    ap.add_argument("--inits", type=int, default=60)
    ap.add_argument("--inside-only", action="store_true")
    a = ap.parse_args()
    per_group = collections.Counter()     # straddled-form mask of undecided groups
    per_step = collections.Counter()      # OR-ed mask of classification steps
    npts_before = npts_after = 0
    npass = 0
    for s in range(a.samples):
        smp = syn.make_sample(100 + s)
        iy, pf, lf, _ = oracle.initial_guess(smp["points"], smp["pred"])
        pf = np.asarray(pf, dtype=np.float64); lf = np.asarray(lf)
        ry, t = syn.make_inits(100 + s, iy, a.inits)
        K = np.asarray(smp["K"], dtype=np.float64).reshape(3, 3)
        poses = [np.array([ry[i], t[i][0], t[i][1], t[i][2]]) for i in range(a.inits)]
        poses.append(np.array([smp["ry_gt"], *smp["t_gt"]]))
        order = cm.keys(pf, lf, "xz6")
        for xp in poses:
            G, und, sure, mask = pass_masks(pf, lf, order, K, smp["H"], smp["W"], xp, a.inside_only)
            npass += 1
            for g in np.nonzero(und)[0]:
                per_group[int(mask[g])] += 1
            R = (G + 31) // 32
            for r in range(R):                      # round r holds groups q * R + r, q = 0..31 (frustum_boxes_kernel)
                ids = [q * R + r for q in range(32) if q * R + r < G]
                seq = [("s", g) for g in ids if sure[g]] + [("u", g) for g in ids if und[g]]
                for i in range(0, len(seq), GPS):
                    step = seq[i:i + GPS]
                    if all(k == "s" for k, _ in step):
                        continue                    # a step of surely-active groups only is not classified
                    m = 0
                    for _, g in step:
                        m |= int(mask[g])
                    per_step[m] += 1
                    npts_before += 32 * len(step) * 5
                    npts_after += 32 * len(step) * step_class(m)
    tot_g = sum(per_group.values())
    tot_s = sum(per_step.values())
    print("passes %d, undecided groups per pass %.1f, classification steps per pass %.1f" % (npass, tot_g / npass, tot_s / npass))
    print("\nstraddled-form mask of undecided groups (share of groups)")
    for m, c in per_group.most_common():
        print("  %-16s %6.2f %%" % (mask_name(m), 100.0 * c / tot_g))
    print("\nOR-ed mask of a classification step of %d groups (share of steps) -> forms evaluated per point" % GPS)
    for m, c in per_step.most_common():
        print("  %-16s %6.2f %%  -> %d" % (mask_name(m), 100.0 * c / tot_s, step_class(m)))
    print("\nforms evaluated per classified point: before 5.00, after %.2f" % (5.0 * npts_after / npts_before))


if __name__ == "__main__":
    main()
