"""The C-ABI library builds, loads without a GPU and exports every symbol include/*.h declares;
the host-side argument validation of the Python mirror behaves like the reference's binding."""
import ctypes
import glob
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    names = set()
    for h in glob.glob(os.path.join(ROOT, "include", "*.h")):
        src = open(h).read()
        src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
        for m in re.finditer(r"^\s*(?:const\s+)?[A-Za-z_][A-Za-z0-9_]*\s*\*?\s+\*?([a-z_0-9]+)\s*\(", src, flags=re.M):
            names.add(m.group(1))
    return names


def test_library_exports_every_header_prototype():
    from deepi2p_b200 import build, _native
    lib = build.build()
    handle = ctypes.CDLL(lib)
    decl = declared_symbols()
    assert {"frustum_solve_batch_f32", "frustum_solve_batch_f64", "index_max_forward", "ball_query_forward",
            "frustum_prepare_batch_f32", "frustum_evaluate_f32", "frustum_residuals_f32"} <= decl
    for name in decl:
        assert hasattr(handle, name), name
    assert set(_native.parse_header(open(build.HEADER).read())) == decl
    handle.dib_abi_version.restype = ctypes.c_int
    assert handle.dib_abi_version() == 4
    handle.frustum_solve_workspace_bytes.restype = ctypes.c_size_t
    handle.frustum_solve_workspace_bytes.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int]
    assert handle.frustum_solve_workspace_bytes(4096, 60, 20480) >= 4096 * 60 * (6 * 8 + 8 + 16)


def test_every_prototype_is_bound_with_the_header_types():
    """load() binds each prototype of the header with the types parse_header reads from it (compared by identity: an
    int64_t or uint64_t argument bound as c_int would be truncated without an error)."""
    from deepi2p_b200 import build, _native
    c = ctypes
    sigs = _native.parse_header(open(build.HEADER).read())
    lib = _native.load()
    assert len(sigs) >= 121
    for name, (restype, argtypes) in sigs.items():
        fn = getattr(lib, name)
        assert fn.restype is restype, name
        assert len(fn.argtypes) == len(argtypes) and all(a is b for a, b in zip(fn.argtypes, argtypes)), name
    assert len(sigs["frustum_solve_batch_f32"][1]) == 23
    loss = sigs["classifier_loss_forward_f32"][1]
    assert loss[1] is c.c_int64 and loss[3] is c.c_int64
    assert sigs["assemble_resample_f32"][1][7] is c.c_uint64
    assert sigs["ball_query_xyz_forward"][1][2] is c.c_float
    assert sigs["dib_last_error"] == (c.c_char_p, [])
    assert sigs["dib_profile_solve_events"] == (None, [c.c_void_p, c.c_void_p])
    sizes = [n for n in sigs if n.endswith("_workspace_bytes")]
    assert sizes and all(sigs[n][0] is c.c_size_t for n in sizes)


def test_header_parser_rejects_unknown_types():
    from deepi2p_b200 import _native
    c = ctypes
    assert _native.parse_header("/* x; */\n#define A 1\ntypedef void* dib_stream_t;\n"
                                "int f(const int64_t* p,\n      uint64_t seed, dib_stream_t s);") == \
        {"f": (c.c_int, [c.c_void_p, c.c_uint64, c.c_void_p])}
    for bad in ("unsigned int f(int a);", "int f(long n);", "long f(void);"):
        with pytest.raises(_native.NativeError, match="f"):
            _native.parse_header(bad)


def test_argument_validation_without_gpu():
    """Pure host-side checks: bad arguments are rejected before any device work."""
    from deepi2p_b200 import _native
    lib = _native.load()
    lb = (ctypes.c_double * 3)(-1, -1, -1)
    buf = ctypes.create_string_buffer(64)
    # n_stride not a multiple of 16
    rc = lib.frustum_solve_batch_f32(ctypes.addressof(buf), ctypes.addressof(buf), None, 17, ctypes.addressof(buf),
                                     ctypes.addressof(buf), ctypes.addressof(lb), ctypes.addressof(lb), 160.0, 512.0,
                                     500, 1, 1, 1, ctypes.addressof(buf), ctypes.addressof(buf), None, None, None,
                                     None, ctypes.addressof(buf), 64, None)
    assert rc == -22 and b"multiple of 16" in lib.dib_last_error()
    rc = lib.index_max_forward(None, None, None, 1, 1, 1, 1, None)
    assert rc == -22
    rc = lib.ball_query_forward(ctypes.addressof(buf), 1.0, ctypes.addressof(buf), 1, 1, 4, 0, None)
    assert rc == -22


def test_dropin_modules_import_and_fail_loudly_without_gpu():
    import torch
    import deepi2p_b200
    deepi2p_b200.install_dropins()
    import FrustumRegistration
    import ball_query
    import index_max
    assert FrustumRegistration.solve is FrustumRegistration.solvePGivenK
    assert callable(index_max.forward_cuda_shared_mem) and callable(ball_query.forward_cuda_shared_mem)
    with pytest.raises(RuntimeError):          # CHECK_CUDA of the reference (index_max.cpp:119-121)
        index_max.forward_cuda_shared_mem(torch.zeros(1, 1, 4), torch.zeros(1, 4, dtype=torch.int32), 2)
    with pytest.raises(RuntimeError):
        ball_query.forward_cuda_shared_mem(torch.zeros(1, 1, 4), 1.0, 2)
    if not torch.cuda.is_available():
        from deepi2p_b200 import _native
        with pytest.raises(_native.NativeError):      # no CPU fallback
            FrustumRegistration.solvePGivenK(np.zeros((3, 8)), np.zeros(8, dtype=np.int64), np.eye(3), 0.0,
                                             np.zeros(3), 160, 512, [-1, -1, -1], [1, 1, 1], 10, False, True)


def test_pack_clouds_layout_and_precision_choice():
    from deepi2p_b200 import frustum
    pts = np.arange(3 * 21, dtype=np.float64).reshape(3, 21) / 4
    lab = np.array([0, 1, 2] * 7)
    xyz, l8, n = frustum.pack_clouds(pts, lab, device="cpu")
    assert xyz.dtype.is_floating_point and str(xyz.dtype) == "torch.float32" and tuple(xyz.shape) == (1, 3, 32)
    assert l8[0, :21].tolist() == [0, 1, -1] * 7 and (l8[0, 21:] == -1).all() and n.tolist() == [21]
    pts2 = pts + 1e-9
    xyz2, _, _ = frustum.pack_clouds(pts2, lab, device="cpu")
    assert str(xyz2.dtype) == "torch.float64"


def test_header_is_plain_c_and_cluster_assign_validates_on_host(tmp_path):
    """The boundary must be bindable from C / cgo / JNI: the header has to compile as C11 without CUDA headers."""
    import subprocess
    src = tmp_path / "use_header.c"
    src.write_text('#include "deepi2p_b200.h"\n'
                   'int probe(void) { return dib_abi_version() + (int)frustum_solve_workspace_bytes(1, 1, 16); }\n')
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"),
                           str(src)])
    from deepi2p_b200 import _native
    lib = _native.load()
    buf = ctypes.create_string_buffer(256)
    a = ctypes.addressof(buf)
    assert lib.cluster_assign_forward(a, a, 1, 4, 2, 3, a, a, a, a, None, None, a, 256, None) == -22     # k > M
    assert b"k" in lib.dib_last_error()
    assert lib.cluster_assign_forward(a, a, 1, 4, 4000, 1, a, a, a, a, None, None, a, 256, None) == -22  # M > 2048
    assert lib.cluster_assign_workspace_bytes(8, 128) == 8 * 3 * 128 * 8
