// qd_launch.h -- host layer shared by every translation unit of libqd_b200.so (state in qd_launch.cu): the
// per-thread error message, device properties and grid sizing.  Host code only.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>
#include <type_traits>

#include "qd_b200.h"

namespace qd {

// Sets the calling thread's qd_last_error() message and returns `code`.
int fail(int code, const char* fmt, ...) __attribute__((format(printf, 2, 3)));

#define QD_CUDA(call)                                                                                  \
    do {                                                                                               \
        cudaError_t e_ = (call);                                                                       \
        if (e_ != cudaSuccess) return ::qd::fail(QD_ERR_CUDA, "%s: %s", #call, cudaGetErrorString(e_)); \
    } while (0)

struct DevInfo {
    int device = 0, sms = 0, major = 0, minor = 0;
    size_t smem_optin = 0;
    // grid of `need` CTAs, at most `per_sm` CTAs per SM
    int grid(int64_t need, int64_t per_sm) const { return (int)(need < sms * per_sm ? need : sms * per_sm); }
};
// properties of the calling thread's current device (queried once per device)
int dev_info(DevInfo** out);
// CTAs of (kernel, threads, dynamic smem) resident per SM of `device`, cached; 1 when the query fails
int resident_ctas(const void* kernel, int device, int threads, size_t smem);

// Grid of `need` CTAs, at most `per_sm` CTAs per SM of the current device.
int capped_grid(int64_t need, int64_t per_sm, int* grid);
// Grid of `need` CTAs, at most as many as are resident at once for (kernel, threads, dynamic smem).
int resident_grid(const void* kernel, int threads, size_t smem, int64_t need, int* grid);
// Opts `kernel` into `smem` bytes of dynamic shared memory; `opted` is the kernel's own per-device table (64 slots).
int opt_in_smem(const void* kernel, size_t smem, size_t* opted);

inline cudaStream_t as_stream(qd_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Calls f(std::integral_constant<int, R>{}) with the registers per lane of the warp-row kernels for rows of
// `row_len` floats: R = 2 up to 256, 4 up to 512, 8 above.  MAX_R = 4 leaves R = 8 uninstantiated.
template <int MAX_R = 8, class F>
int with_row_regs(int64_t row_len, F&& f) {
    static_assert(MAX_R == 4 || MAX_R == 8, "warp-row kernels exist for R = 2, 4, 8");
    if (row_len <= 256) return f(std::integral_constant<int, 2>{});
    if constexpr (MAX_R == 8)
        if (row_len > 512) return f(std::integral_constant<int, 8>{});
    return f(std::integral_constant<int, 4>{});
}

// code widths of the fixed-width packed codec
inline bool bits_ok(int bits) { return bits == 1 || bits == 2 || bits == 4 || bits == 8; }
// smallest code width that holds `symbols` distinct codes (symbols in [1, 256])
inline int bits_for(int symbols) { return symbols <= 2 ? 1 : symbols <= 4 ? 2 : symbols <= 16 ? 4 : 8; }

// Calls f(std::integral_constant<int, BITS>{}) for a code width `bits` already checked to be 1, 2, 4 or 8.
template <class F>
decltype(auto) with_bits(int bits, F&& f) {
    if (bits == 8) return f(std::integral_constant<int, 8>{});
    if (bits == 4) return f(std::integral_constant<int, 4>{});
    if (bits == 2) return f(std::integral_constant<int, 2>{});
    return f(std::integral_constant<int, 1>{});
}

}  // namespace qd
