"""CPU oracle of the batched ICP path -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and the benchmark scripts may import this package; deepi2p_b200.icp never does.
icp_oracle.cpp restates the contract of evaluation/icp/registration_icp.py:115-162 (DESIGN.md "ICP") with its own
exact nearest-neighbour search and the kernels' summation order.  It is built into oracle_icp/_build/.

    python -m oracle_icp            # g++ only, a few seconds
"""
import ctypes
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_build")
LIB = os.path.join(OUT, "libicp_oracle.so")
SRC = os.path.join(HERE, "icp_oracle.cpp")
FLAGS = ["-std=c++17", "-O2", "-ffp-contract=off", "-fopenmp"]
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
        lib.icp_oracle_frame.restype = None
        lib.icp_oracle_frame.argtypes = [vp, i32, i32, vp, i32, i32, vp, i32, f64, i32, f64, f64, i32,
                                         vp, vp, vp, vp, vp, vp, vp, vp]
        lib.icp_oracle_umeyama.restype = None
        lib.icp_oracle_umeyama.argtypes = [vp, vp, i32, vp, vp]
        lib.icp_oracle_nearest.restype = None
        lib.icp_oracle_nearest.argtypes = [vp, i32, i32, vp, i32, f64, vp, vp]
        _lib = lib
    return _lib


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _cloud(pc):
    pc = np.asarray(pc)
    if pc.ndim != 2 or pc.shape[0] != 3:
        raise ValueError("clouds are [3, N]")
    p32 = np.ascontiguousarray(pc.astype(np.float32))
    if pc.dtype != np.float32 and not np.array_equal(p32.astype(pc.dtype), pc):
        raise ValueError("coordinates are not float32-representable")
    return p32


def register_frame(src, tgt, init, max_corr_dist=1.0, max_iteration=30, relative_fitness=1e-6, relative_rmse=1e-6,
                   force_2d=True, trace=False):
    """The whole contract for one frame.  src [3,n], tgt [3,m] (float32-representable), init [I,4,4].  Returns dict(
    T [I,4,4], fitness [I], rmse [I], stats [I,2] (update steps, n_corr), P [4,4], fitness_best, best) and, with
    trace, trace_nc [I, max_iteration + 1] (n_corr of every pass, -1 after the last)."""
    s32, t32 = _cloud(src), _cloud(tgt)
    init = np.ascontiguousarray(np.asarray(init, dtype=np.float64).reshape(-1, 16))
    I = init.shape[0]
    T = np.zeros((I, 16))
    fit = np.zeros(I)
    rmse = np.zeros(I)
    stats = np.zeros((I, 2), dtype=np.int32)
    tr = np.zeros((I, max_iteration + 1), dtype=np.int32) if trace else None
    P = np.zeros(16)
    fb = np.zeros(1)
    best = np.zeros(1, dtype=np.int32)
    _load().icp_oracle_frame(_ptr(s32), s32.shape[1], s32.shape[1], _ptr(t32), t32.shape[1], t32.shape[1], _ptr(init),
                             I, float(max_corr_dist), int(max_iteration), float(relative_fitness), float(relative_rmse),
                             int(bool(force_2d)), _ptr(T), _ptr(fit), _ptr(rmse), _ptr(stats),
                             _ptr(tr) if trace else None, _ptr(P), _ptr(fb), _ptr(best))
    out = dict(T=T.reshape(I, 4, 4), fitness=fit, rmse=rmse, stats=stats, P=P.reshape(4, 4), fitness_best=float(fb[0]),
               best=int(best[0]))
    if trace:
        out["trace_nc"] = tr
    return out


def umeyama(src, dst, c=None):
    """Rigid Umeyama of pairs src [n,3] -> dst [n,3] with the moments taken about c (default dst[0]).  Returns 4x4."""
    src = np.ascontiguousarray(src, dtype=np.float64)
    dst = np.ascontiguousarray(dst, dtype=np.float64)
    c = np.ascontiguousarray(dst[0] if c is None else c, dtype=np.float64)
    U = np.zeros(12)
    _load().icp_oracle_umeyama(_ptr(src), _ptr(dst), src.shape[0], _ptr(c), _ptr(U))
    return np.vstack([U.reshape(3, 4), [0.0, 0.0, 0.0, 1.0]])


def nearest(tgt, q, max_corr_dist=1.0):
    """Nearest target index (ties -> lowest) and d2 of each query q [k,3] f64 when d2 < r^2, else (-1, inf)."""
    t32 = _cloud(tgt)
    q = np.ascontiguousarray(q, dtype=np.float64).reshape(-1, 3)
    j = np.zeros(q.shape[0], dtype=np.int32)
    d2 = np.zeros(q.shape[0])
    _load().icp_oracle_nearest(_ptr(t32), t32.shape[1], t32.shape[1], _ptr(q), q.shape[0], float(max_corr_dist),
                               _ptr(j), _ptr(d2))
    return j, d2
