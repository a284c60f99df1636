"""CPU oracle of the PnP-RANSAC path -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py may import this package; deepi2p_b200.pnp never does.
pnp_oracle.cpp restates the contract of evaluation/registration_pnp.py:95-148 serially (DESIGN.md "PnP-RANSAC").
It is a package of its own next to oracle/ (the frustum and point-op oracles), built into oracle_pnp/_build/.

    python -m oracle_pnp            # g++ only, a few seconds
"""
import ctypes
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_build")
LIB = os.path.join(OUT, "libpnp_oracle.so")
SRC = os.path.join(HERE, "pnp_oracle.cpp")
FLAGS = ["-std=c++17", "-O2", "-ffp-contract=off"]
_lib = None


def build(force=False, verbose=False):
    if force or not os.path.exists(LIB) or os.path.getmtime(SRC) > os.path.getmtime(LIB):
        os.makedirs(OUT, exist_ok=True)
        cmd = ["g++", "-shared", "-fPIC", *FLAGS, "-o", LIB + ".tmp", SRC, "-lm"]
        if verbose:
            print(" ".join(cmd))
        subprocess.check_call(cmd)
        os.replace(LIB + ".tmp", LIB)
    return LIB


def _load():
    global _lib
    if _lib is None:
        lib = ctypes.CDLL(build())
        vp, i32, f64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_double
        lib.pnp_oracle_sample.restype = None
        lib.pnp_oracle_sample.argtypes = [i32, i32, i32, ctypes.c_uint64, vp]
        lib.pnp_oracle_update_niters.restype = i32
        lib.pnp_oracle_update_niters.argtypes = [i32, i32, i32, f64]
        lib.pnp_oracle_epnp.restype = i32
        lib.pnp_oracle_epnp.argtypes = [vp, vp, i32, vp, vp]
        lib.pnp_oracle_frame.restype = i32
        lib.pnp_oracle_frame.argtypes = [vp, vp, vp, i32, i32, vp, f64, f64, f64, i32, f64, f64, ctypes.c_uint64,
                                         vp, vp, vp, vp, vp, vp, vp, vp, vp]
        _lib = lib
    return _lib


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def sample(h, s, n, seed):
    """The 5 distinct point indices hypothesis h of frame s draws (n >= 5)."""
    out = np.zeros(5, dtype=np.int32)
    _load().pnp_oracle_sample(h, s, n, seed, _ptr(out))
    return out


def update_niters(niters, cnt, n, confidence=0.99):
    return int(_load().pnp_oracle_update_niters(niters, cnt, n, confidence))


def epnp(xyz, uv, K):
    """EPnP on n correspondences: xyz [n,3], uv [n,2] pixels, K 3x3.  Returns (ok, R 3x3, t 3)."""
    xyz = np.ascontiguousarray(xyz, dtype=np.float64)
    uv = np.ascontiguousarray(uv, dtype=np.float64)
    K9 = np.ascontiguousarray(np.asarray(K, dtype=np.float64).reshape(9))
    out = np.zeros(12)
    ok = _load().pnp_oracle_epnp(_ptr(xyz), _ptr(uv), xyz.shape[0], _ptr(K9), _ptr(out))
    return bool(ok), out[:9].reshape(3, 3), out[9:].copy()


def ransac_frame(xyz, coarse, fine, K, H, W, s=0, scale=1 / 32.0, iterations=500, reproj_err=0.6, confidence=0.99,
                 seed=0):
    """The whole contract for frame s.  xyz [3,n] (float32-representable), coarse [n], fine [n].  Returns a dict with
    P, outlier_ratio, inliers, n_sel, hyp_used, winner, mask [n], hyp_pose [hyp_used,12], hyp_inliers [hyp_used]."""
    xyz = np.ascontiguousarray(np.asarray(xyz, dtype=np.float32))
    n = xyz.shape[1]
    coarse = np.ascontiguousarray(np.asarray(coarse).astype(np.int8))
    fine = np.ascontiguousarray(np.asarray(fine).astype(np.int32))
    K9 = np.ascontiguousarray(np.asarray(K, dtype=np.float64).reshape(9))
    P16 = np.zeros(16)
    ratio = np.zeros(1)
    ints = np.zeros(4, dtype=np.int32)
    mask = np.zeros(max(n, 1), dtype=np.uint8)
    hp = np.zeros((max(iterations, 1), 12))
    hi = np.zeros(max(iterations, 1), dtype=np.int32)
    _load().pnp_oracle_frame(_ptr(xyz), _ptr(coarse), _ptr(fine), n, s, _ptr(K9), H, W, scale, iterations, reproj_err,
                             confidence, seed, _ptr(P16), _ptr(ratio), _ptr(ints[0:]), _ptr(ints[1:]), _ptr(ints[2:]),
                             _ptr(ints[3:]), _ptr(mask), _ptr(hp), _ptr(hi))
    used = int(ints[2])
    return dict(P=P16.reshape(4, 4), outlier_ratio=float(ratio[0]), inliers=int(ints[0]), n_sel=int(ints[1]),
                hyp_used=used, winner=int(ints[3]), mask=mask[:n].copy(), hyp_pose=hp[:used].copy(),
                hyp_inliers=hi[:used].copy())
