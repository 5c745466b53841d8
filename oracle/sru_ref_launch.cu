// sru_ref_launch.cu -- host launchers of the reference's own SRU kernels (onmt/modules/SRU.py:71-347), for tests and
// tools/sru_bench.py only.  The kernels are not in this repository: oracle/sru_ref_build.py extracts SRU_CODE from
// the reference into oracle/_ref/sru_ref_kernels.cu and compiles it with this file, once with -fmad=false and once
// with the default contraction (what NVRTC gave the reference).  Launch shape and argument order are the
// reference's SRU_Compute (SRU.py:379-474): min(512, ncols) threads per block, one thread per column, and
// grad_bias as the per-(batch, column) partials [2, batch, dir*d] that the reference sums with torch.
#include <cassert>
#include <cstddef>

#include <cuda_runtime.h>

#include "sru_ref_kernels.cu"

namespace {
dim3 blocks(int ncols) { return dim3((unsigned)((ncols - 1) / (ncols < 512 ? ncols : 512) + 1)); }
dim3 threads(int ncols) { return dim3((unsigned)(ncols < 512 ? ncols : 512)); }
}  // namespace

extern "C" int sru_ref_fwd(int bidirectional, const float* u, const float* x, const float* bias, const float* init,
                           const float* mask_h, int len, int batch, int d, int k, float* h, float* c, int activation,
                           void* stream) {
    const int ncols = batch * d * (bidirectional ? 2 : 1);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (bidirectional)
        sru_bi_fwd<<<blocks(ncols), threads(ncols), 0, st>>>(u, x, bias, init, mask_h, len, batch, d, k, h, c, activation);
    else
        sru_fwd<<<blocks(ncols), threads(ncols), 0, st>>>(u, x, bias, init, mask_h, len, batch, d, k, h, c, activation);
    return (int)cudaGetLastError();
}

extern "C" int sru_ref_bwd(int bidirectional, const float* u, const float* x, const float* bias, const float* init,
                           const float* mask_h, const float* c, const float* grad_h, const float* grad_last, int len,
                           int batch, int d, int k, float* grad_u, float* grad_x, float* grad_bias, float* grad_init,
                           int activation, void* stream) {
    const int ncols = batch * d * (bidirectional ? 2 : 1);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (bidirectional)
        sru_bi_bwd<<<blocks(ncols), threads(ncols), 0, st>>>(u, x, bias, init, mask_h, c, grad_h, grad_last, len, batch,
                                                             d, k, grad_u, grad_x, grad_bias, grad_init, activation);
    else
        sru_bwd<<<blocks(ncols), threads(ncols), 0, st>>>(u, x, bias, init, mask_h, c, grad_h, grad_last, len, batch, d,
                                                          k, grad_u, grad_x, grad_bias, grad_init, activation);
    return (int)cudaGetLastError();
}
