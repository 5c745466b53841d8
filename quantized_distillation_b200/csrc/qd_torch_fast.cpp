// qd_torch_fast.cpp -- optional compiled front door of the reference-shaped per-tensor API.
//
// The ctypes shim costs tens of microseconds of host time per call (torch.empty x3, views, ctypes argument marshalling); the
// training loops avoid it with the multi-tensor plans, but code that keeps the reference's per-tensor loop
// (INTEGRATION.md, level 1) pays it once per tensor per step.  This module does the same work from C++: output
// allocation through ATen's caching allocator, torch's current stream, ONE call into the C ABI of libqd_b200.so.
// Nothing is computed here -- it is plumbing around qd_uniform_fwd / qd_uniform_bwd, and the Python layer falls
// back to ctypes when the module has not been built.
#include <torch/extension.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>

#include <tuple>

#include "qd_b200.h"

namespace {

void check_input(const at::Tensor& t, const char* name) {
    TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kFloat && t.is_contiguous(), name,
                " must be a contiguous float32 CUDA tensor");
    TORCH_CHECK(t.numel() > 0, name, " is empty");
}

void raise_status(int rc) {
    if (rc == QD_OK) return;
    const std::string msg = qd_last_error();
    if (rc == QD_ERR_INVALID_ARG) throw py::value_error(msg);
    if (rc == QD_ERR_UNSUPPORTED) {
        PyErr_SetString(PyExc_NotImplementedError, msg.c_str());
        throw py::error_already_set();
    }
    TORCH_CHECK(false, "libqd_b200 error ", rc, ": ", msg);
}

// uniformQuantization (deterministic, linear scaling, no pre-ops): (q, alpha, beta, argmin, argmax)
std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor> uniform_fwd(const at::Tensor& x, int64_t levels, int64_t bucket,
                                                                                   bool in_place) {
    check_input(x, "tensor");
    const c10::cuda::CUDAGuard guard(x.device());
    const int64_t n = x.numel();
    int64_t rows = 1, row_len = n, padded = n;
    raise_status(qd_bucket_geometry(n, bucket, &rows, &row_len, &padded));
    at::Tensor q = in_place ? x : at::empty_like(x);
    const auto fopt = x.options();
    at::Tensor ab = bucket > 0 ? at::empty({2, rows, 1}, fopt) : at::empty({2, 1}, fopt);
    at::Tensor mm = bucket > 0 ? at::empty({2, rows, 1}, fopt.dtype(at::kLong)) : at::empty({2, 1}, fopt.dtype(at::kLong));
    at::Tensor ws;
    void* ws_ptr = nullptr;
    size_t ws_bytes = 0;
    if ((bucket == 0 || bucket > QD_MAX_STAGED_BUCKET) && n > QD_MAX_STAGED_BUCKET) {   // grid path only
        ws_bytes = qd_workspace_bytes(n, bucket);
        ws = at::empty({(int64_t)ws_bytes}, fopt.dtype(at::kByte));
        ws_ptr = ws.data_ptr();
    }
    float* a = ab.data_ptr<float>();
    int64_t* m = mm.data_ptr<int64_t>();
    raise_status(qd_uniform_fwd(x.data_ptr<float>(), q.data_ptr<float>(), nullptr, a, a + rows, m, m + rows, n, bucket, (int)levels,
                                nullptr, 0.f, 0, 0, 0, ws_ptr, ws_bytes, c10::cuda::getCurrentCUDAStream().stream()));
    return {q, ab.select(0, 0), ab.select(0, 1), mm.select(0, 0), mm.select(0, 1)};
}

// uniformQuantization_variable.backward ('complicated' min/max gradient) and the truncated mask
at::Tensor uniform_bwd(const at::Tensor& x, const at::Tensor& g, int64_t levels, int64_t bucket, int64_t mode) {
    check_input(x, "saved input");
    check_input(g, "grad_output");
    TORCH_CHECK(x.numel() == g.numel(), "grad_output does not match the saved input");
    const c10::cuda::CUDAGuard guard(x.device());
    at::Tensor out = at::empty_like(g);
    const int64_t n = x.numel();
    at::Tensor ws;
    void* ws_ptr = nullptr;
    size_t ws_bytes = 0;
    if ((bucket == 0 || bucket > QD_MAX_STAGED_BUCKET) && n > QD_MAX_STAGED_BUCKET) {   // grid path only
        ws_bytes = qd_workspace_bytes(n, bucket);
        ws = at::empty({(int64_t)ws_bytes}, x.options().dtype(at::kByte));
        ws_ptr = ws.data_ptr();
    }
    raise_status(qd_uniform_bwd(x.data_ptr<float>(), g.data_ptr<float>(), out.data_ptr<float>(), n, bucket, (int)levels, (int)mode,
                                ws_ptr, ws_bytes, c10::cuda::getCurrentCUDAStream().stream()));
    return out;
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
    m.doc() = "compiled front door of quantized_distillation_b200's per-tensor ops (plumbing around libqd_b200.so)";
    m.def("uniform_fwd", &uniform_fwd, "x -> (q, alpha, beta, argmin, argmax)");
    m.def("uniform_bwd", &uniform_bwd, "(x, g) -> gout");
}
