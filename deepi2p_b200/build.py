"""Build the sm_90a (H100) CUDA library in-tree: deepi2p_b200/lib/libdeepi2p_b200.so.

    python -m deepi2p_b200.build [--force] [--verbose]

nvcc cross-compiles without a GPU.  The .so is git-ignored but travels with the working tree.
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libdeepi2p_b200.so")
SOURCES = ["frustum_solver.cu", "prepare.cu", "point_ops.cu", "metrics.cu", "ball_query_xyz.cu", "cluster_assign.cu",
           "pnp_ransac.cu", "icp.cu", "pointprep.cu", "assemble.cu", "interp.cu", "imageprep.cu", "classifier_loss.cu",
           "encoder_ops.cu", "fusion.cu", "jpeg.cu", "png.cu", "pointwise_mlp.cu", "oxford_build.cu", "oxford_images.cu",
           "jpeg_encode.cu", "knn_fusion.cu", "node_mlp.cu"]
# Compiled on their own without FMA contraction: oracle_pnp/pnp_oracle.cpp, oracle_icp/icp_oracle.cpp and
# oracle_prep/prep_oracle.cpp, oracle_assemble/, oracle_interp/, oracle_image/ and oracle.pose_diff_restated (metrics.cu)
# restate their arithmetic bit for bit (oracle_oxford_build/ and oracle_oxford_images/ too); metrics.cu and
# classifier_loss.cu share the label rule of project.cuh.
NOFMA_SOURCES = ["pnp_ransac.cu", "icp.cu", "pointprep.cu", "assemble.cu", "interp.cu", "imageprep.cu", "metrics.cu",
                 "classifier_loss.cu", "oxford_build.cu", "oxford_images.cu"]
HEADERS = ["common.cuh", "morton_index.cuh", "sym3_eig.cuh", "project.cuh", "nearest_k.cuh", "tf32_mma.cuh", os.path.join("..", "..", "include", "deepi2p_b200.h")]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
    "--fmad=true",
    "--threads", "4",             # the translation units compile in parallel
]


def nvcc_path():
    p = shutil.which("nvcc")
    if p:
        return p
    p = "/usr/local/cuda/bin/nvcc"
    if os.path.exists(p):
        return p
    raise RuntimeError("nvcc not found; the CUDA library cannot be built")


def is_stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def _nofma_objects(objdir, extra, verbose):
    """Compile NOFMA_SOURCES to objects in objdir with --fmad=false; returns their paths."""
    flags = [f for f in NVCC_FLAGS if f not in ("-shared", "--fmad=true")]
    objs = []
    for s in NOFMA_SOURCES:
        obj = os.path.join(objdir, os.path.splitext(s)[0] + ".nofma.o")
        cmd = [nvcc_path(), *flags, "--fmad=false", *extra, *os.environ.get("DIB_NVCC_EXTRA", "").split(), "-c",
               "-o", obj, os.path.join(CSRC, s)]
        if verbose:
            print(" ".join(cmd), flush=True)
        subprocess.check_call(cmd)
        objs.append(obj)
    return objs


def build(force=False, verbose=False, extra=(), out=None):
    """Compile the library in-tree.  `out` names a variant file (lib/variants/<out>.so) instead of the default
    library; variants are a tuning aid (scripts/ab_prebuilt.sh) selected at run time with DIB_LIB_OVERRIDE."""
    if out is not None:
        vdir = os.path.join(LIBDIR, "variants")
        os.makedirs(vdir, exist_ok=True)
        target = os.path.join(vdir, out + ".so")
        srcs = [os.path.join(CSRC, s) for s in SOURCES if s not in NOFMA_SOURCES] + _nofma_objects(vdir, extra, verbose)
        cmd = [nvcc_path(), *NVCC_FLAGS, *extra, *os.environ.get("DIB_NVCC_EXTRA", "").split(), "-o", target, *srcs]
        if verbose:
            print(" ".join(cmd), flush=True)
        subprocess.check_call(cmd)
        return target
    if not force and not is_stale():
        return LIB
    os.makedirs(LIBDIR, exist_ok=True)
    srcs = [os.path.join(CSRC, s) for s in SOURCES if s not in NOFMA_SOURCES and os.path.exists(os.path.join(CSRC, s))]
    srcs += _nofma_objects(LIBDIR, extra, verbose)
    env_extra = os.environ.get("DIB_NVCC_EXTRA", "").split()
    cmd = [nvcc_path(), *NVCC_FLAGS, *extra, *env_extra, "-o", LIB + ".tmp", *srcs]
    if verbose:
        print(" ".join(cmd), flush=True)
    subprocess.check_call(cmd)
    os.replace(LIB + ".tmp", LIB)
    return LIB


if __name__ == "__main__":
    extra = ["-Xptxas", "-v"] if "--ptxas" in sys.argv else []
    out = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else None
    print(build(force="--force" in sys.argv or bool(extra), verbose=True, extra=extra, out=out))
