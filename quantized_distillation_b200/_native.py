"""ctypes binding of libqd_b200.so (C ABI declared in include/qd_b200.h).

There is no CPU implementation behind this module: if the shared library is
missing, or no CUDA device is present when an op is called, the call raises.
"""
from __future__ import annotations

import ctypes as C
import os
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libqd_b200.so")

QD_OK, QD_ERR_INVALID_ARG, QD_ERR_UNSUPPORTED, QD_ERR_CUDA, QD_ERR_WORKSPACE = range(5)
BWD_STE, BWD_TRUNCATED, BWD_MINMAX = 0, 1, 2
RULE_NEAREST, RULE_MIDPOINT = 0, 1
SCALE_ABSMAX, SCALE_ABSNORM = 1, 2
MAX_STAGED_BUCKET = 49152
PACKED_LINEAR_MAX_ROWS = 64     # QD_PACKED_LINEAR_MAX_ROWS
PACKED_LSTM_MAX_ROWS = 64       # QD_PACKED_LSTM_MAX_ROWS
PACKED_GRU_MAX_ROWS = 64        # QD_PACKED_GRU_MAX_ROWS
BEAM_MAX = 16                   # QD_BEAM_MAX

_p, _i64, _i32, _u64, _f32, _sz = C.c_void_p, C.c_int64, C.c_int, C.c_uint64, C.c_float, C.c_size_t

# name -> (restype, argtypes); mirrors include/qd_b200.h one to one
SIGNATURES = {
    "qd_version": (C.c_int, []),
    "qd_last_error": (C.c_char_p, []),
    "qd_device_info": (C.c_int, [C.POINTER(C.c_int)] * 3),
    "qd_bucket_geometry": (C.c_int, [_i64, _i64, C.POINTER(_i64), C.POINTER(_i64), C.POINTER(_i64)]),
    "qd_workspace_bytes": (_sz, [_i64, _i64]),
    "qd_scale_down": (C.c_int, [_p, _p, _p, _p, _p, _p, _i64, _i64, _p, _f32, _p, _sz, _p]),
    "qd_inv_scale_down": (C.c_int, [_p, _p, _p, _p, _p, _i64, _i64, _p]),
    "qd_scale_down_abs": (C.c_int, [_p, _p, _p, _p, _i64, _i64, _i32, _p, _f32, _p]),
    "qd_inv_scale_down_abs": (C.c_int, [_p, _p, _p, _p, _p, _i64, _i64, _p]),
    "qd_uniform_fwd_abs": (C.c_int, [_p, _p, _p, _p, _i64, _i64, _i32, _i32, _p, _f32, _p]),
    "qd_uniform_fwd": (C.c_int, [_p, _p, _p, _p, _p, _p, _p, _i64, _i64, _i32, _p, _f32, _i32, _u64, _u64, _p, _sz, _p]),
    "qd_uniform_bwd": (C.c_int, [_p, _p, _p, _i64, _i64, _i32, _i32, _p, _sz, _p]),
    "qd_uniform_fwd_bwd": (C.c_int, [_p, _p, _p, _p, _i64, _i64, _i32, _i32, _p, _sz, _p]),
    "qd_nonuniform_fwd": (C.c_int, [_p, _p, _i32, _i32, _p, _p, _p, _p, _p, _i64, _i64, _p, _f32, _p, _sz, _p]),
    "qd_nonuniform_bwd": (C.c_int, [_p, _p, _p, _p, _i32, _p, _i64, _i64, _p, _sz, _p]),
    "qd_centroid_index": (C.c_int, [_p, _p, _i32, _i32, _p, _p, _p, _i64, _p]),
    "qd_index_histogram": (C.c_int, [_p, _i64, _i32, _p, _p]),
    "qd_pack_indices": (C.c_int, [_p, _p, _i64, _i32, _p]),
    "qd_unpack_indices": (C.c_int, [_p, _i32, _p, _i64, _p]),
    "qd_unpack_dequant_uniform": (C.c_int, [_p, _i32, _p, _p, _p, _i64, _i64, _i32, _p]),
    "qd_unpack_dequant_nonuniform": (C.c_int, [_p, _i32, _p, _i32, _p, _p, _p, _i64, _i64, _p]),
    "qd_packed_workspace_bytes": (_sz, [_i64, _i64]),
    "qd_uniform_fwd_packed": (C.c_int, [_p, _p, _i32, _p, _p, _i64, _i64, _i32, _p, _sz, _p]),
    "qd_nonuniform_fwd_packed": (C.c_int, [_p, _p, _i32, _i32, _p, _i32, _p, _p, _i64, _i64, _p, _sz, _p]),
    "qd_unpack_model_workspace_bytes": (_sz, [_i32]),
    "qd_unpack_dequant_model": (C.c_int, [_p, _i32, _i64, _i32, _p, _sz, _p]),
    "qd_packed_linear": (C.c_int, [_p, _i64, _i64, _i64, _p, _i32, _p, _p, _p, _i32, _i32, _i64, _p, _p, _p]),
    "qd_packed_conv2d": (C.c_int, [_p, _i64, _i64, _i64, _i64, _i64, _i32, _i32, _i32, _i32, _i32, _i32, _p, _i32, _p, _p, _p, _i32,
                                   _i32, _i64, _p, _p, _p]),
    "qd_packed_embedding": (C.c_int, [_p, _i32, _i64, _i64, _i64, _p, _i32, _p, _p, _p, _i32, _i32, _i64, _p, _p, _p]),
    "qd_packed_lstm_cell": (C.c_int, [_p, _i64, _p, _i64, _p, _i64, _i64, _i64, _p, _p, _i32, _i64, _p, _p, _p, _i64, _p, _p]),
    "qd_packed_lstm_layer": (C.c_int, [_p, _i64, _p, _i64, _i32, _i64, _i64, _p, _p, _i32, _i64, _p, _p, _p, _p, _p, _i64, _p, _p, _p]),
    "qd_packed_gru_cell": (C.c_int, [_p, _i64, _p, _i64, _i64, _i64, _i64, _p, _p, _i32, _i64, _p, _p, _p, _i64, _p]),
    "qd_packed_gru_layer": (C.c_int, [_p, _i64, _p, _i64, _i32, _i64, _i64, _p, _p, _i32, _i64, _p, _p, _p, _p, _i64, _p, _p]),
    "qd_nmt_loss_workspace_bytes": (_sz, [_i64]),
    "qd_nmt_loss_fwd": (C.c_int, [_p, _p, _p, _i64, _i64, _i64, _f32, _p, _p, _p, _p, _sz, _p]),
    "qd_nmt_loss_bwd": (C.c_int, [_p, _p, _p, _p, _p, _i64, _i64, _i64, _f32, _p, _p]),
    "qd_beam_workspace_bytes": (_sz, [_i64, _i32]),
    "qd_beam_step": (C.c_int, [_p, _i32, _i64, _i32, _i64, _i64, _i32, _p, _p, _p, _p, _p, _p, _p, _p, _sz, _p]),
    "qd_huffman_encode":(C.c_int, [_p, _i64, _p, _p, _i64, _p, _p, _p]),
    "qd_huffman_decode_dequant_uniform": (C.c_int, [_p, _i64, _p, _p, _p, _p, _p, _i64, _i64, _i32, _p]),
    "qd_huffman_decode_dequant_nonuniform": (C.c_int, [_p, _i64, _p, _p, _p, _i32, _p, _p, _p, _i64, _i64, _p]),
    "qd_huffman_model_workspace_bytes": (_sz, [_i32]),
    "qd_huffman_decode_dequant_model": (C.c_int, [_p, _i32, _p, _i64, _i32, _p, _sz, _p]),
    "qd_huffman_repack_model_workspace_bytes": (_sz, [_i32]),
    "qd_huffman_decode_packed_model": (C.c_int, [_p, _i32, _p, _p, _p, _sz, _p]),
    "qd_plan_create": (C.c_int, [C.POINTER(_p), _i32, _p, _p, _p, _p, _i64]),
    "qd_plan_destroy": (C.c_int, [_p]),
    "qd_plan_set_shadow": (C.c_int, [_p, _p]),
    "qd_plan_uniform_fwd": (C.c_int, [_p, _p]),
    "qd_plan_uniform_fwd_save": (C.c_int, [_p, _p]),
    "qd_plan_uniform_bwd": (C.c_int, [_p, _p, _i32, _p]),
    "qd_plan_set_momentum": (C.c_int, [_p, _p]),
    "qd_plan_sgd_step": (C.c_int, [_p, _p, _i32, C.c_double, C.c_double, C.c_double, _i32, _p]),
    "qd_plan_nonuniform_create": (C.c_int, [C.POINTER(_p), _i32, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i64]),
    "qd_plan_nonuniform_destroy": (C.c_int, [_p]),
    "qd_plan_nonuniform_fwd": (C.c_int, [_p, _p]),
    "qd_plan_nonuniform_bwd": (C.c_int, [_p, _p, _p]),
    "qd_plan_nonuniform_bwd_partial": (C.c_int, [_p, _p, _p, _p]),
    "qd_plan_nonuniform_bwd_finish": (C.c_int, [_p, _p, C.c_double, _p]),
    "qd_order_statistics_workspace_bytes": (_sz, [_i64]),
    "qd_order_statistics": (C.c_int, [_p, _i64, _p, _i32, _p, _p, _sz, _p]),
    "qd_multi_l2norm": (C.c_int, [_p, _p, _i32, _p, _p]),
    "qd_uniform_fwd_host": (C.c_int, [_p, _p, _i64, _i64, _i32, _i32]),
    "qd_uniform_fwd_bwd_host": (C.c_int, [_p, _p, _p, _p, _i64, _i64, _i32, _i32, _i32]),
    "qd_selftest_division": (C.c_int, [_i64, _u64, C.POINTER(_i64), _p]),
}

_lib = None
_lock = threading.Lock()


def lib() -> C.CDLL:
    """Loads libqd_b200.so once; raises (never falls back) when it is absent."""
    global _lib
    if _lib is None:
        with _lock:
            if _lib is None:
                if not os.path.exists(LIB_PATH):
                    raise ImportError(
                        f"{LIB_PATH} not found: build the sm_90a extension first "
                        "(python -c 'import __graft_entry__ as g; g.build()'). There is no CPU fallback.")
                handle = C.CDLL(LIB_PATH)
                for name, (res, args) in SIGNATURES.items():
                    fn = getattr(handle, name)      # AttributeError if the ABI and the header drift apart
                    fn.restype, fn.argtypes = res, args
                _lib = handle
    return _lib


_fast = None
_fast_tried = False


def fast():
    """The optional compiled front door of the per-tensor ops (csrc/qd_torch_fast.cpp, built by
    build.build_fast() / __graft_entry__.build()): ATen allocation + one C-ABI call from C++ instead of
    ctypes marshalling.  None when it has not been built -- callers then use the ctypes path; either way the
    arithmetic happens in libqd_b200.so."""
    global _fast, _fast_tried
    if not _fast_tried:
        _fast_tried = True
        path = os.path.join(_HERE, "_fastcall", "_qd_fast.so")
        if os.path.exists(path):
            try:
                import importlib.util
                lib()                                            # libqd_b200.so first: the module links against it
                spec = importlib.util.spec_from_file_location("_qd_fast", path)
                mod = importlib.util.module_from_spec(spec)
                spec.loader.exec_module(mod)
                _fast = mod
            except Exception:                                    # stale build, other torch: ctypes still works
                _fast = None
    return _fast


def check(rc: int) -> None:
    """Maps qd_status to the exception type the reference raises for the same
    condition (ValueError / NotImplementedError, quant_functions.py:22-33,
    138-139, 230-236, 326-337)."""
    if rc == QD_OK:
        return
    msg = lib().qd_last_error().decode("utf-8", "replace")
    if rc == QD_ERR_INVALID_ARG:
        raise ValueError(msg)
    if rc == QD_ERR_UNSUPPORTED:
        raise NotImplementedError(msg)
    raise RuntimeError(f"libqd_b200 error {rc}: {msg}")


def require_cuda() -> None:
    if not torch.cuda.is_available():
        raise RuntimeError("quantized_distillation_b200 needs a CUDA device (H100, sm_90a); "
                           "there is no CPU implementation of the quantization ops in this package")


def ptr(t):
    # a plain int is accepted for a c_void_p argument: no ctypes object per pointer on the per-call path
    return None if t is None else t.data_ptr()


def stream_ptr(device=None):
    return torch.cuda.current_stream(device).cuda_stream


def needs_workspace(n: int, bucket: int) -> bool:
    """Only rows beyond the staging limit (grid path: bucket None / huge buckets on big tensors) use the
    caller's scratch in the forward ops; everything else runs on chip."""
    return (bucket == 0 or bucket > MAX_STAGED_BUCKET) and n > MAX_STAGED_BUCKET


_ws = {}
_WS_MAX_STREAMS = 16
_WS_FLOOR = 1 << 22          # covers every op whose rows are staged on chip (qd_workspace_bytes <= ~2.5 MB)


def workspace(n: int, bucket: int, device) -> torch.Tensor:
    """Per (device, stream) scratch buffer, grown on demand."""
    # only rows longer than the staging limit (grid path) can need more than the floor
    need = _WS_FLOOR
    if (bucket == 0 or bucket > MAX_STAGED_BUCKET) and n > MAX_STAGED_BUCKET:
        need = max(need, int(lib().qd_workspace_bytes(n, bucket)))
    key = (device.index if device.index is not None else torch.cuda.current_device(),
           torch.cuda.current_stream(device).cuda_stream)
    buf = _ws.pop(key, None)
    if buf is None or buf.numel() < need:
        buf = torch.empty(need, dtype=torch.uint8, device=device)
    _ws[key] = buf                       # re-inserted last: the dict doubles as an LRU list
    while len(_ws) > _WS_MAX_STREAMS:    # streams come and go (graph capture, user side streams): bound the cache
        _ws.pop(next(iter(_ws)))
    return buf


def geometry(n: int, bucket: int):
    """(rows, row_len, padded_len) of create_bucket_tensor (help_functions.py:67-94); same
    arithmetic as qd_bucket_geometry, kept in Python to save an FFI round trip per call
    (tests/test_cpu_boundary.py checks the two against each other and against the oracle)."""
    if n <= 0 or bucket < 0:
        raise ValueError(f"n must be > 0 and bucket >= 0 (n={n} bucket={bucket})")
    if bucket == 0 or n < bucket:
        return 1, n, n
    rows = -(-n // bucket)
    return rows, bucket, rows * bucket


def geometry_native(n: int, bucket: int):
    rows, row_len, padded = _i64(), _i64(), _i64()
    check(lib().qd_bucket_geometry(n, bucket, C.byref(rows), C.byref(row_len), C.byref(padded)))
    return rows.value, row_len.value, padded.value
