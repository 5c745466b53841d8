"""Builds the reference's own SRU kernels into oracle/_ref/ -- TEST AND BENCHMARK INFRASTRUCTURE ONLY.

SRU_CODE (onmt/modules/SRU.py:71-346) is read from the reference with `ast`: nothing of the reference is imported or
executed.  It is written unchanged to oracle/_ref/sru_ref_kernels.cu and compiled for sm_90a with the launcher
oracle/sru_ref_launch.cu twice:
  libsru_ref_nofma.so  -fmad=false, as libqd_b200.so: the tests compare bit for bit against it;
  libsru_ref.so        the default contraction, what NVRTC gave the reference.
oracle/_ref/ is not in git.  Without a reference checkout (QD_REFERENCE_ROOT, default /root/reference) the existing
artefacts are kept and nothing fails; the tests that need them skip when they are absent.

    python oracle/sru_ref_build.py
"""
from __future__ import annotations

import ast
import os
import shutil
import subprocess
import warnings

HERE = os.path.dirname(os.path.abspath(__file__))
OUT_DIR = os.path.join(HERE, "_ref")
LAUNCHER = os.path.join(HERE, "sru_ref_launch.cu")
KERNELS = os.path.join(OUT_DIR, "sru_ref_kernels.cu")
LIBS = {"nofma": os.path.join(OUT_DIR, "libsru_ref_nofma.so"), "fma": os.path.join(OUT_DIR, "libsru_ref.so")}
FLAGS = {"nofma": ["-fmad=false"], "fma": []}


def reference_source(ref_root: str) -> str | None:
    """SRU_CODE of the reference's onmt/modules/SRU.py, or None when the file is absent or unreadable."""
    path = os.path.join(ref_root, "onmt", "modules", "SRU.py")
    if not os.access(path, os.R_OK):
        return None
    with open(path) as f, warnings.catch_warnings():
        warnings.simplefilter("ignore", SyntaxWarning)          # the reference's grep pattern 'cupy\|pynvrtc'
        tree = ast.parse(f.read(), path)
    for node in tree.body:
        if isinstance(node, ast.Assign) and any(isinstance(t, ast.Name) and t.id == "SRU_CODE" for t in node.targets):
            return ast.literal_eval(node.value)
    raise RuntimeError(f"{path} has no SRU_CODE assignment")


def build(ref_root: str | None = None) -> dict:
    """Writes and compiles the reference kernels when a reference checkout is present and the libraries are stale;
    returns {variant: path} of the libraries that exist afterwards."""
    ref_root = ref_root or os.environ.get("QD_REFERENCE_ROOT", "/root/reference")
    src = reference_source(ref_root)
    if src is not None:
        os.makedirs(OUT_DIR, exist_ok=True)
        old = open(KERNELS).read() if os.path.exists(KERNELS) else None
        if old != src:
            with open(KERNELS, "w") as f:
                f.write(src)
        nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
        newest = max(os.path.getmtime(KERNELS), os.path.getmtime(LAUNCHER))
        for variant, lib in LIBS.items():
            if os.path.exists(lib) and os.path.getmtime(lib) >= newest:
                continue
            cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", *FLAGS[variant],
                   "-Xcompiler", "-fPIC", "-shared", "-I", OUT_DIR, "-o", lib, LAUNCHER]
            res = subprocess.run(cmd, capture_output=True, text=True)
            if res.returncode != 0:
                raise RuntimeError("nvcc failed on the reference SRU kernels:\n" + res.stdout + res.stderr)
    return {v: p for v, p in LIBS.items() if os.path.exists(p)}


if __name__ == "__main__":
    print(build())
