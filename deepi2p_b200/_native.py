"""ctypes binding of the C ABI declared in include/deepi2p_b200.h, and the host helpers every wrapper around it shares.

The signatures are read from the header itself when the library is loaded, so the header is the only place an entry
point is declared.  There is no CPU fallback: if the library is missing or a call fails, this raises.
"""
import ctypes
import os
import re

import torch

from . import build as _build

_c = ctypes
_lib = None

EXPECTED_ABI = 4        # dib_abi_version() of the library include/deepi2p_b200.h declares

_SCALARS = {"int": _c.c_int, "int32_t": _c.c_int, "int64_t": _c.c_int64, "uint64_t": _c.c_uint64,
            "size_t": _c.c_size_t, "float": _c.c_float, "double": _c.c_double, "dib_stream_t": _c.c_void_p}


class NativeError(RuntimeError):
    pass


def parse_header(text):
    """{name: (restype, argtypes)} of every prototype in the C header `text`: plain C with block comments, #-lines,
    typedefs and extern "C" guards.  Pointers bind as c_void_p, a `const char*` return as c_char_p and a `void` return
    as None; any type outside those and _SCALARS raises NativeError, so no argument is bound with a guessed width."""
    text = re.sub(r"/\*.*?\*/|^\s*#[^\n]*|extern\s*\"C\"\s*\{|\}", " ", text, flags=re.S | re.M)
    sigs = {}
    for decl in text.split(";"):
        decl = " ".join(re.sub(r"\s*\*", "* ", decl).split())
        if not decl or decl.startswith("typedef "):
            continue
        m = re.fullmatch(r"(.+) (\w+) ?\((.*)\)", decl)
        if m is None:
            raise NativeError(f"cannot read the declaration {decl!r}")
        ret, name, args = m.groups()

        def ctype(spec):
            if spec.endswith("*"):
                return _c.c_void_p
            t = _SCALARS.get(spec.removeprefix("const "))
            if t is None:
                raise NativeError(f"{name}: no ctypes binding for the type {spec!r} in {decl!r}")
            return t
        restype = None if ret == "void" else _c.c_char_p if ret == "const char*" else ctype(ret)
        argtypes = [] if args in ("", "void") else [ctype(a.strip().rpartition(" ")[0]) for a in args.split(",")]
        sigs[name] = (restype, argtypes)
    return sigs


def _require_cuda():
    if not torch.cuda.is_available():
        raise NativeError("deepi2p_b200 needs a CUDA device (sm_90a); there is no CPU fallback")


def _stream_ptr(stream=None):
    s = stream if stream is not None else torch.cuda.current_stream()
    return s.cuda_stream


def _ptr(t):
    return 0 if t is None else t.data_ptr()


def _workspace(cache, need, device, stream=None, floor=1 << 20):
    """Scratch buffer of at least max(need, floor) bytes for launches on `stream` (None: the current stream), cached in
    the caller's pool `cache` per (device index, stream pointer): launches on one stream run in order, so they can
    share it; launches on different streams may overlap.  It is allocated while `stream` is current, so the allocator
    ties it to the stream that uses it.  While that stream is being captured into a CUDA graph the buffer is a new
    allocation from the graph's private pool and is not cached: a graph-pool buffer is never handed to a later eager
    call, and a cached eager buffer is never resized under a graph that captured its address."""
    with torch.cuda.stream(stream):
        if torch.cuda.is_current_stream_capturing():
            return torch.empty(max(need, floor), dtype=torch.uint8, device=device)
        key = (device.index if device.index is not None else torch.cuda.current_device(), _stream_ptr(stream))
        ws = cache.get(key)
        if ws is None or ws.numel() < need:
            ws = torch.empty(max(need, floor), dtype=torch.uint8, device=device)
            cache[key] = ws
    return ws


# dtypes of the feature operands of the ops that run under bfloat16 autocast (DESIGN.md 4.37), with the suffix of their
# entry points
FEATURE_DTYPES = {torch.float32: "f32", torch.bfloat16: "bf16"}


def feature_dtype(named):
    """The one dtype of an op's feature operands [(tensor or None, name)], float32 or bfloat16; returns (dtype, entry
    point suffix).  Any other dtype raises RuntimeError "<name> must have dtype ...", operands of both dtypes raise
    RuntimeError naming both."""
    first = None
    for t, name in named:
        if t is None:
            continue
        if t.dtype not in FEATURE_DTYPES:
            raise RuntimeError(f"{name} must have dtype {torch.float32} or {torch.bfloat16}")
        if first is None:
            first = (t.dtype, name)
        elif t.dtype != first[0]:
            raise RuntimeError(f"{first[1]} and {name} must have the same dtype, got {first[0]} and {t.dtype}")
    return first[0], FEATURE_DTYPES[first[0]]


def lib_path():
    return _build.LIB


def load():
    """Load (building first if nvcc is available and the .so is stale/missing)."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB
    override = os.environ.get("DIB_LIB_OVERRIDE")       # tuning aid: a prebuilt variant of the same library
    if override:
        if not os.path.exists(override):
            raise NativeError(f"DIB_LIB_OVERRIDE={override} does not exist")
        path = override
    elif not os.path.exists(path) or _build.is_stale():
        try:
            _build.build()
        except Exception as e:  # noqa: BLE001 - turn any build problem into a loud, specific error
            if not os.path.exists(path):
                raise NativeError(
                    f"deepi2p_b200 CUDA library is missing ({path}) and could not be built: {e}. "
                    "There is no CPU fallback; run `python -m deepi2p_b200.build`.") from e
            import warnings
            warnings.warn(f"deepi2p_b200: {path} is older than its sources and the rebuild failed ({e}); "
                          "loading the stale library (its ABI version is checked)")
    lib = ctypes.CDLL(path)
    sigs = parse_header(open(_build.HEADER).read())
    lib.dib_abi_version.restype, lib.dib_abi_version.argtypes = sigs["dib_abi_version"]
    abi = lib.dib_abi_version()
    if abi != EXPECTED_ABI:
        raise NativeError(f"{path} has ABI version {abi}, this binding was written for {EXPECTED_ABI}: "
                          "rebuild with `python -m deepi2p_b200.build --force`")
    for name, (restype, argtypes) in sigs.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    _lib = lib
    return lib


def check(rc, what):
    if rc != 0:
        msg = load().dib_last_error().decode("utf-8", "replace")
        raise NativeError(f"{what} failed (code {rc}): {msg}")
