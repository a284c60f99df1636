"""Compile the REFERENCE's own index_max / ball_query extensions, unmodified, from the sources where
they lie under /root/reference, into oracle/_ref/ (TEST INFRASTRUCTURE ONLY; git-ignored, but it
travels to the GPU box with the working tree).

    python oracle/build_ref.py

Used (a) here, on CPU: index_max.forward_cpu is the true reference that pins the index_max oracle and
writes tests/golden/index_max_*.npz (tests/golden/make_golden.py); (b) on the GPU box: the reference's
CUDA kernels forward_cuda_shared_mem are the bit-exact checkers and the on-box GPU baselines in
bench.py --ops.  No reference source is copied into this repository.

The registration solver itself cannot be built: it needs Ceres + Eigen (find_package(Ceres REQUIRED),
evaluation/frustum_reg/CMakeLists.txt:9), neither of which exists offline.
"""
import glob
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
REF = "/root/reference"
EXTS = {
    "index_max": ["models/index_max_ext/index_max.cpp", "models/index_max_ext/index_max_cuda.cu"],
    "ball_query": ["models/ball_query_ext/ball_query.cpp", "models/ball_query_ext/ball_query_cuda.cu"],
}


def available():
    return os.path.isdir(REF) and all(os.path.exists(os.path.join(REF, s)) for v in EXTS.values() for s in v)


def built(name):
    return sorted(glob.glob(os.path.join(OUT, name + "*.so")))


def build(verbose=False):
    if not available():
        return None
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.environ.setdefault("MAX_JOBS", "4")
    from torch.utils import cpp_extension
    os.makedirs(OUT, exist_ok=True)
    for name, srcs in EXTS.items():
        if built(name):
            continue
        bdir = os.path.join(OUT, "build_" + name)
        os.makedirs(bdir, exist_ok=True)
        cpp_extension.load(name=name, sources=[os.path.join(REF, s) for s in srcs], build_directory=bdir,
                           extra_cflags=["-O2", "-w"], extra_cuda_cflags=["-O2", "-w", "-lineinfo"],
                           verbose=verbose, is_python_module=False)
        so = glob.glob(os.path.join(bdir, name + "*.so"))
        if not so:
            raise RuntimeError("reference extension %s did not produce a .so" % name)
        shutil.copy2(so[0], os.path.join(OUT, name + ".so"))
        shutil.rmtree(bdir, ignore_errors=True)
    return OUT


def load(name):
    """Import a built reference extension (torch must be imported first)."""
    import importlib.util
    import torch  # noqa: F401
    so = built(name)
    if not so:
        raise FileNotFoundError("oracle/_ref/%s.so not built" % name)
    spec = importlib.util.spec_from_file_location(name, so[0])
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    r = build(verbose="-v" in sys.argv)
    print("reference extensions:", r, [os.path.basename(p) for n in EXTS for p in built(n)])
