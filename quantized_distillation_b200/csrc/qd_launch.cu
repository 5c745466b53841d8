// qd_launch.cu -- state of the shared host layer (qd_launch.h) and the entry points that read it: last error,
// version, device info.
#include "qd_launch.h"

#include <cstdarg>
#include <cstdio>
#include <mutex>
#include <unordered_map>

namespace qd {

// ------------------------------------------------------------------ errors
static thread_local char g_err[512] = "";

int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

// ------------------------------------------------------------------ device info
static DevInfo g_dev[64];
static std::mutex g_mu;

int dev_info(DevInfo** out) {
    int d = 0;
    QD_CUDA(cudaGetDevice(&d));
    if (d < 0 || d >= 64) return fail(QD_ERR_CUDA, "device ordinal %d out of range", d);
    std::lock_guard<std::mutex> lk(g_mu);
    if (g_dev[d].sms == 0) {
        int v = 0;
        g_dev[d].device = d;
        QD_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, d)); g_dev[d].sms = v;
        QD_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMajor, d)); g_dev[d].major = v;
        QD_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMinor, d)); g_dev[d].minor = v;
        QD_CUDA(cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, d)); g_dev[d].smem_optin = (size_t)v;
    }
    *out = &g_dev[d];
    return QD_OK;
}

// ------------------------------------------------------------------ grid sizing
struct OccKey {
    const void* kernel;
    int device, threads;
    size_t smem;
    bool operator==(const OccKey& o) const {
        return kernel == o.kernel && device == o.device && threads == o.threads && smem == o.smem;
    }
};
struct OccKeyHash {
    size_t operator()(const OccKey& k) const {
        return std::hash<const void*>()(k.kernel) ^ (k.smem << 16) ^ ((size_t)k.threads << 6) ^ (size_t)k.device;
    }
};
static std::unordered_map<OccKey, int, OccKeyHash> g_occ;

int resident_ctas(const void* kernel, int device, int threads, size_t smem) {
    const OccKey key{kernel, device, threads, smem};
    {
        std::lock_guard<std::mutex> lk(g_mu);
        auto it = g_occ.find(key);
        if (it != g_occ.end()) return it->second;
    }
    int n = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, threads, smem) != cudaSuccess || n < 1) n = 1;
    std::lock_guard<std::mutex> lk(g_mu);
    g_occ[key] = n;
    return n;
}

int capped_grid(int64_t need, int64_t per_sm, int* grid) {
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    *grid = di->grid(need, per_sm);
    return QD_OK;
}

int resident_grid(const void* kernel, int threads, size_t smem, int64_t need, int* grid) {
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    *grid = di->grid(need, resident_ctas(kernel, di->device, threads, smem));
    return QD_OK;
}

// The attribute only ever grows (per kernel and device) and changes under the library mutex, so two host threads
// launching the same kernel with different row lengths can never lower it between the other thread's opt-in and
// its launch.
int opt_in_smem(const void* kernel, size_t smem, size_t* opted) {
    int d = 0;
    QD_CUDA(cudaGetDevice(&d));
    std::lock_guard<std::mutex> lk(g_mu);
    if (smem > opted[d & 63]) {
        QD_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        opted[d & 63] = smem;
    }
    return QD_OK;
}

}  // namespace qd

using namespace qd;

extern "C" int qd_version(void) { return 106; }
extern "C" const char* qd_last_error(void) { return g_err; }

extern "C" int qd_device_info(int* sm_count, int* cc_major, int* cc_minor) {
    DevInfo* di;
    int rc = dev_info(&di);
    if (rc) return rc;
    if (sm_count) *sm_count = di->sms;
    if (cc_major) *cc_major = di->major;
    if (cc_minor) *cc_minor = di->minor;
    return QD_OK;
}
