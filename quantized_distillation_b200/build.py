"""Builds libqd_b200.so (sm_90a, H100) in-tree with nvcc.  Used by
__graft_entry__.build(); the built .so is a build product and stays out of git."""
from __future__ import annotations

import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SOURCES = [os.path.join(HERE, "csrc", f) for f in ("qd_launch.cu", "qd_quant.cu", "qd_codec.cu", "qd_recurrent.cu", "qd_nmt_loss.cu", "qd_beam.cu", "qd_plans.cu", "qd_stats.cu",
                                                   "qd_host.cu")]
HEADERS = [os.path.join(HERE, "csrc", f) for f in ("qd_launch.h", "qd_common.cuh", "qd_rowops.cuh", "qd_warp_path.cuh", "qd_block_path.cuh",
                                                   "qd_staged_path.cuh", "qd_abs_path.cuh", "qd_select.cuh", "qd_grid_path.cuh", "qd_points_grad.cuh", "qd_plan.cuh", "qd_huffman.cuh",
                                                   "qd_packed_walk.cuh", "qd_lse.cuh")]
HEADERS.append(os.path.join(ROOT, "include", "qd_b200.h"))
OUT = os.path.join(HERE, "libqd_b200.so")

# -fmad=false + explicit _rn intrinsics: one IEEE rounding per reference torch op (DESIGN.md)
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-fmad=false", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared", "-I", os.path.join(ROOT, "include")]


def nvcc() -> str:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found; the sm_90a extension cannot be built")
    return exe


def is_stale() -> bool:
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    return any(os.path.getmtime(f) > t for f in SOURCES + HEADERS)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not is_stale():
        return OUT
    cmd = [nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", OUT] + SOURCES
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    if verbose:
        print(res.stderr)
    return OUT


# ---- optional compiled front door of the per-tensor API (csrc/qd_torch_fast.cpp) ---------------------------------
FAST_SRC = os.path.join(HERE, "csrc", "qd_torch_fast.cpp")
FAST_DIR = os.path.join(HERE, "_fastcall")
FAST_OUT = os.path.join(FAST_DIR, "_qd_fast.so")


def fast_is_stale() -> bool:
    if not os.path.exists(FAST_OUT):
        return True
    t = os.path.getmtime(FAST_OUT)
    return os.path.getmtime(FAST_SRC) > t or os.path.getmtime(os.path.join(ROOT, "include", "qd_b200.h")) > t


def build_fast(force: bool = False, verbose: bool = False) -> str:
    """Compiles the pybind11 / ATen front door against the torch of this interpreter and links it to the in-tree
    libqd_b200.so.  Host C++ only: no device code, nothing arch specific."""
    if not force and not fast_is_stale():
        return FAST_OUT
    build()                                        # the library it links against
    from torch.utils import cpp_extension as ce
    os.makedirs(FAST_DIR, exist_ok=True)
    ce.load(name="_qd_fast", sources=[FAST_SRC], extra_include_paths=[os.path.join(ROOT, "include")],
            extra_cflags=["-O2", "-std=c++17"], with_cuda=True,
            extra_ldflags=[f"-L{HERE}", "-lqd_b200", "-Wl,-rpath," + HERE],      # the loader also pre-loads libqd_b200.so by path
            build_directory=FAST_DIR, verbose=verbose, is_python_module=False)
    if not os.path.exists(FAST_OUT):
        raise RuntimeError("the fast-call module was not produced")
    return FAST_OUT


if __name__ == "__main__":
    import sys
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
