"""CPU oracle of the scan-preparation path -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and the benchmark scripts may import this package; deepi2p_b200.pointprep never
does.  prep_oracle.cpp restates the contract (DESIGN.md "Scan preparation") with its own radius search (a uniform
grid) and the kernels' summation order; the 1-nearest-neighbour query is oracle_icp's k-d tree.  It is built into
oracle_prep/_build/.

    python -m oracle_prep           # g++ only, a few seconds
"""
import ctypes
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_build")
LIB = os.path.join(OUT, "libprep_oracle.so")
SRC = os.path.join(HERE, "prep_oracle.cpp")
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
        lib.prep_oracle_voxel.restype = i32
        lib.prep_oracle_voxel.argtypes = [vp, i32, i32, vp, i32, f64, vp, vp, vp]
        lib.prep_oracle_normals.restype = None
        lib.prep_oracle_normals.argtypes = [vp, i32, i32, f64, i32, vp, vp, vp, vp]
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


def voxel_downsample(xyz, voxel_size, attr=None):
    """One cloud xyz [3,n] (float32-representable), attr [C,n] f64 or None.  Returns (xyz [3,m] f64, attr [C,m] f64
    or None) in ascending (ix, iy, iz) order; ValueError when the cloud spans 2^21 or more voxels along an axis."""
    p = _cloud(xyz)
    n = p.shape[1]
    A = np.zeros((0, n)) if attr is None else np.ascontiguousarray(attr, dtype=np.float64).reshape(-1, n)
    C = A.shape[0]
    xo = np.zeros((3, n))
    ao = np.zeros((C, n))
    m = np.zeros(1, dtype=np.int32)
    rc = _load().prep_oracle_voxel(_ptr(p), n, n, _ptr(A), C, float(voxel_size), _ptr(xo), _ptr(ao), _ptr(m))
    if rc != 0:
        raise ValueError("the cloud spans 2^21 or more voxels along an axis")
    m = int(m[0])
    return xo[:, :m].copy(), (None if attr is None else ao[:, :m].copy())


def estimate_normals(xyz, radius, max_nn, orient=(0.0, 0.0, 1.0), neighbours=False):
    """One cloud xyz [3,m] (float32-representable).  Returns (normals [3,m] f64, count [m] i32) and, with neighbours,
    nbr [m,max_nn] i32: each point's neighbours in ascending (d2, index) order, -1 padded."""
    p = _cloud(xyz)
    m = p.shape[1]
    o = np.ascontiguousarray(orient, dtype=np.float64)
    nrm = np.zeros((3, m))
    cnt = np.zeros(m, dtype=np.int32)
    nbr = np.full((m, int(max_nn)), -1, dtype=np.int32) if neighbours else None
    _load().prep_oracle_normals(_ptr(p), m, m, float(radius), int(max_nn), _ptr(o), _ptr(nrm), _ptr(cnt),
                                _ptr(nbr) if neighbours else None)
    return (nrm, cnt, nbr) if neighbours else (nrm, cnt)


def nearest(xyz, q):
    """Index of the nearest point of xyz [3,m] (float32-representable) for each query q [3,k] f64, ties -> lowest."""
    import oracle_icp
    q = np.asarray(q, dtype=np.float64)
    j, _ = oracle_icp.nearest(xyz, q.T, max_corr_dist=1e300)
    return j


def prepare_scan(xyz, intensity, voxel_size=0.1, sn_radius=0.6, sn_max_nn=30, orient=(0.0, 0.0, 1.0)):
    """kitti_pc_bin_to_npy_with_downsample_sn.py:48-74 for one scan under the contract: returns the [7,M] float32
    record (xyz, intensity of the nearest original point, surface normal); normals from the float32-rounded centres."""
    p = _cloud(xyz)
    down, _ = voxel_downsample(p, voxel_size)
    d32 = down.astype(np.float32)
    nrm, _ = estimate_normals(d32, sn_radius, sn_max_nn, orient)
    idx = nearest(p, down)
    inten = np.asarray(intensity, dtype=np.float32).reshape(-1)[idx]
    return np.concatenate([down, inten[None].astype(np.float64), nrm], 0).astype(np.float32)
