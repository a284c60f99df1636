"""The small dense fp64 solvers on degenerate geometry, on the GPU: EPnP (pnp.epnp_batch), the shared 3x3 Jacobi
eigensolver (pointprep.sym3_eig_batch), the normals (pointprep.estimate_normals) and ICP's Umeyama step
(icp.icp_register_batch).  Each kernel meets the same exact references as the CPU oracles in
tests/test_degenerate_geometry_cpu.py, is bit-identical to its oracle on every case, and gives the same bits on a
second run and on another stream."""
import numpy as np
import pytest
import torch

import oracle_icp
import oracle_pnp
import oracle_prep
from deepi2p_b200 import icp, pnp, pointprep
from deepi2p_b200.icp import pack_clouds
from test_degenerate_geometry_cpu import (KF, check_epnp, check_normals, check_sym3, check_umeyama, coplanar_sweep,
                                          epnp_cases, icp_frames, normals_clouds, scaled_sym3_cases, sweep_counts)

pytestmark = pytest.mark.gpu


def test_epnp_degenerate_sets_match_the_oracle_and_the_true_pose():
    cases = epnp_cases() + coplanar_sweep()
    sets = [(P, uv) for _, P, uv, _, _, _ in cases]
    pose, ok = pnp.epnp_batch(sets, KF)
    res = [(bool(o), p[:9].reshape(3, 3), p[9:]) for o, p in zip(ok, pose)]
    nd, nv = check_epnp(cases, res)
    fail, wrong, right = sweep_counts(cases, res)
    print("%d sets: %d degenerate, %d valid and exact" % (len(cases), nd, nv))
    assert wrong == 0 and fail == nd
    for (name, P, uv, _, _, _), o, p in zip(cases, ok, pose):
        rok, R, t = oracle_pnp.epnp(P, uv, KF)
        assert bool(o) == rok, name
        assert np.array_equal(p, np.concatenate([R.reshape(9), t]) if rok else np.zeros(12)), name
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        pose2, ok2 = pnp.epnp_batch(sets, KF)
    assert np.array_equal(ok2, ok) and np.array_equal(pose2, pose)


def test_sym3_eig_hook_against_50_digit_references_and_the_oracle():
    cases = scaled_sym3_cases()
    Cs = np.stack([C for _, C in cases])
    lam, E = pointprep.sym3_eig_batch(Cs)
    rl, rE = oracle_pnp.sym3_eig(Cs)
    assert np.array_equal(lam, rl) and np.array_equal(E, rE)
    for (name, C), l, e in zip(cases, lam, E):
        check_sym3(name, C, l, e)


@pytest.mark.parametrize("case", range(len(normals_clouds())), ids=[c[0] for c in normals_clouds()])
def test_normals_on_degenerate_neighbourhoods(case):
    name, X, radius, max_nn, orient, kind = normals_clouds()[case]
    xyz, m = pack_clouds([X])
    nrm, cnt = pointprep.estimate_normals(xyz, m, radius, max_nn, orient, counts=True)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        nrm2, cnt2 = pointprep.estimate_normals(xyz, m, radius, max_nn, orient, counts=True, stream=side)
    side.synchronize()
    k = X.shape[1]
    g, gc = nrm[0, :, :k].cpu().numpy(), cnt[0, :k].cpu().numpy()
    assert torch.equal(nrm, nrm2) and torch.equal(cnt, cnt2)
    rn, rc = oracle_prep.estimate_normals(X, radius, max_nn, orient)
    assert np.array_equal(gc, rc) and np.array_equal(g, rn), name
    check_normals(name, X, radius, max_nn, orient, kind, g, gc, stride=7)


def test_umeyama_step_against_kabsch_and_the_oracle():
    frames = icp_frames()
    src, n = icp.pack_clouds([f[1] for f in frames])
    tgt, m = icp.pack_clouds([f[2] for f in frames])
    init = torch.from_numpy(np.stack([f[3] for f in frames])).cuda()
    kw = dict(max_iteration=1, return_all=True, force_2d=False)
    o = icp.icp_register_batch(src, n, tgt, m, init, **kw)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        o2 = icp.icp_register_batch(src, n, tgt, m, init, stream=side, **kw)
    side.synchronize()
    g = {k: v.cpu().numpy() for k, v in o.items()}
    for k in g:
        np.testing.assert_array_equal(o2[k].cpu().numpy(), g[k], err_msg=k)
    for s, (name, S, D, ini, kind) in enumerate(frames):
        r = oracle_icp.register_frame(S, D, ini, max_iteration=1, force_2d=False)
        for k, rk in (("T", "T"), ("fitness_all", "fitness"), ("rmse_all", "rmse"), ("stats", "stats")):
            np.testing.assert_array_equal(g[k][s], r[rk], err_msg=f"{name} {k}")
        assert g["stats"][s, 0, 0] == 1 and g["stats"][s, 0, 1] == S.shape[1], name
        check_umeyama(name, S, D, kind, g["T"][s, 0])
