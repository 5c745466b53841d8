"""Generates tests/golden/reference_sru.npz: the reference's own SRU kernels (SRU_CODE of onmt/modules/SRU.py:71-346,
read with `ast`, nothing imported or executed) compiled unchanged for the CPU with g++ -ffp-contract=off, under a
small shim for the CUDA keywords and a host loop that runs each column as the thread the reference launches for it.

Per case: the inputs (float32), and the float32 outputs of the kernel pair: h, c, grad_u, grad_x (k = 3), the
per-(batch, column) grad_bias partials [2, batch, dir*d] and grad_init.  The cases cover both directions, k = 3 and
4, the three activations, with and without mask_h, len 1 and len > 1, and zero and non-zero init and grad_last.  The
file is written with fixed zip timestamps, so a rerun gives the same bytes.

Run in the build container only:  python tests/golden/make_golden_sru.py
"""
import ctypes as C
import io
import os
import subprocess
import sys
import tempfile
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
OUT = os.path.join(HERE, "reference_sru.npz")

from oracle.sru_ref_build import reference_source  # noqa: E402

SHIM = r"""
#include <cmath>
#include <math.h>
#include <cassert>
#include <cstddef>
#define __global__
#define __device__
#define __forceinline__ inline
struct qd_dim3 { int x; };
static qd_dim3 blockIdx, blockDim, threadIdx;
"""

HOST = r"""
extern "C" void host_fwd(int bi, const float* u, const float* x, const float* bias, const float* init,
                         const float* mask_h, int len, int batch, int d, int k, float* h, float* c, int act) {
    const int ncols = batch * d * (bi ? 2 : 1);
    blockDim.x = 1; threadIdx.x = 0;
    for (int col = 0; col < ncols; ++col) {
        blockIdx.x = col;
        if (bi) sru_bi_fwd(u, x, bias, init, mask_h, len, batch, d, k, h, c, act);
        else sru_fwd(u, x, bias, init, mask_h, len, batch, d, k, h, c, act);
    }
}
extern "C" void host_bwd(int bi, const float* u, const float* x, const float* bias, const float* init,
                         const float* mask_h, const float* c, const float* gh, const float* gl, int len, int batch,
                         int d, int k, float* gu, float* gx, float* gb, float* gi, int act) {
    const int ncols = batch * d * (bi ? 2 : 1);
    blockDim.x = 1; threadIdx.x = 0;
    for (int col = 0; col < ncols; ++col) {
        blockIdx.x = col;
        if (bi) sru_bi_bwd(u, x, bias, init, mask_h, c, gh, gl, len, batch, d, k, gu, gx, gb, gi, act);
        else sru_bwd(u, x, bias, init, mask_h, c, gh, gl, len, batch, d, k, gu, gx, gb, gi, act);
    }
}
"""

# (bidirectional, k, activation, mask_h, len, batch, d, init, grad_last)
CASES = [
    (0, 4, 1, 0, 5, 3, 4, 1, 1), (0, 3, 1, 1, 5, 3, 4, 1, 0), (1, 4, 1, 1, 6, 2, 3, 1, 1), (1, 3, 1, 0, 6, 2, 3, 0, 1),
    (0, 4, 0, 1, 4, 2, 5, 0, 0), (1, 4, 0, 0, 4, 3, 2, 1, 1), (0, 3, 2, 1, 7, 2, 3, 1, 1), (1, 3, 2, 1, 7, 2, 3, 1, 0),
    (0, 4, 2, 0, 1, 4, 3, 1, 1), (1, 3, 1, 1, 1, 3, 2, 1, 1), (0, 3, 0, 0, 1, 2, 2, 0, 0), (1, 4, 1, 0, 9, 1, 1, 1, 1),
    (1, 4, 2, 1, 3, 2, 6, 0, 1), (0, 4, 1, 1, 12, 3, 7, 1, 1),
]


def _lib(tmp):
    src = os.path.join(tmp, "sru_host.cpp")
    with open(src, "w") as f:
        f.write(SHIM + reference_source(os.environ.get("QD_REFERENCE_ROOT", "/root/reference")) + HOST)
    so = os.path.join(tmp, "libsru_host.so")
    subprocess.run(["g++", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-o", so, src], check=True)
    lib = C.CDLL(so)
    lib.host_fwd.argtypes = [C.c_int] + [C.c_void_p] * 5 + [C.c_int] * 4 + [C.c_void_p] * 2 + [C.c_int]
    lib.host_bwd.argtypes = [C.c_int] + [C.c_void_p] * 8 + [C.c_int] * 4 + [C.c_void_p] * 4 + [C.c_int]
    return lib


def _p(a):
    return None if a is None else a.ctypes.data


def run_case(lib, i, bi, k, act, with_mask, L, B, d, with_init, with_gl):
    rng = np.random.default_rng(1000 + i)
    D = d * (2 if bi else 1)
    f = lambda *s: rng.standard_normal(s).astype(np.float32)  # noqa: E731
    u = f(L, B, D, k)
    x = f(L, B, D) if k == 3 else None
    bias = (0.5 * f(2 * D)).astype(np.float32)
    init = f(B, D) if with_init else np.zeros((B, D), np.float32)
    mask = (rng.random((B, D)) < 0.7).astype(np.float32) / np.float32(0.7) if with_mask else None
    gh = f(L, B, D)
    gl = f(B, D) if with_gl else np.zeros((B, D), np.float32)
    h, c = np.zeros((L, B, D), np.float32), np.zeros((L, B, D), np.float32)
    lib.host_fwd(bi, _p(u), _p(x), _p(bias), _p(init), _p(mask), L, B, d, k, _p(h), _p(c), act)
    gu = np.zeros_like(u)
    gx = np.zeros((L, B, D), np.float32) if k == 3 else None
    gb, gi = np.zeros((2, B, D), np.float32), np.zeros((B, D), np.float32)
    lib.host_bwd(bi, _p(u), _p(x), _p(bias), _p(init), _p(mask), _p(c), _p(gh), _p(gl), L, B, d, k, _p(gu), _p(gx),
                 _p(gb), _p(gi), act)
    out = {"u": u, "bias": bias, "init": init, "grad_h": gh, "grad_last": gl, "h": h, "c": c, "grad_u": gu,
           "grad_bias_partial": gb, "grad_init": gi}
    if x is not None:
        out.update(x=x, grad_x=gx)
    if mask is not None:
        out["mask_h"] = mask
    return {f"c{i}_{k_}": v for k_, v in out.items()}


def _write_npz(path, arrays):
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asarray(arrays[k]), allow_pickle=False)
            z.writestr(zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0)), buf.getvalue(), zipfile.ZIP_DEFLATED)


def main():
    with tempfile.TemporaryDirectory() as tmp:
        lib = _lib(tmp)
        out = {"cases": np.array(CASES, np.int64)}
        for i, c in enumerate(CASES):
            out.update(run_case(lib, i, *c))
    _write_npz(OUT, out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
