"""CPU-side checks (no GPU): the C-ABI library loads and exports every symbol the
header declares, host-side logic matches the reference, argument validation raises
the reference's exception types, and the product never silently falls back to CPU."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "qd_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(qd_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from quantized_distillation_b200 import _native as N
    assert os.path.exists(N.LIB_PATH), "build the extension first: python -c 'import __graft_entry__ as g; g.build()'"
    handle = ctypes.CDLL(N.LIB_PATH)
    syms = header_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(handle, s), f"{s} declared in include/qd_b200.h but not exported"
    assert set(N.SIGNATURES) == set(syms), set(N.SIGNATURES) ^ set(syms)
    assert N.lib().qd_version() >= 100


def test_geometry_matches_oracle_without_gpu():
    from oracle import quant_oracle as O
    from quantized_distillation_b200 import _native as N
    for n in (1, 10, 255, 256, 257, 1000, 4099, 1 << 26):
        for b in (None, 1, 7, 256, 1024, 100000):
            assert N.geometry(n, 0 if b is None else b) == O.bucket_geometry(n, b)
            assert N.geometry_native(n, 0 if b is None else b) == O.bucket_geometry(n, b)   # C ABI agrees too
    with pytest.raises(ValueError):
        N.geometry(0, 256)
    with pytest.raises(ValueError):
        N.geometry_native(0, 256)
    assert N.lib().qd_workspace_bytes(1 << 34, 0) >= N.lib().qd_workspace_bytes(1 << 20, 256) > 0


def test_no_cpu_fallback():
    """Without a CUDA device every op raises instead of computing on the host."""
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import quantized_distillation_b200.quantization as Q
    x = torch.randn(1000)
    with pytest.raises(RuntimeError):
        Q.uniformQuantization(x, 16, bucket_size=256)
    with pytest.raises(RuntimeError):
        Q.nonUniformQuantization(x, [0.0, 0.5, 1.0], bucket_size=256)
    with pytest.raises(RuntimeError):
        Q.ScalingFunction("linear", False, False, 256).scale_down(x)


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "quantized_distillation_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", text, flags=re.M), f"{f} imports the oracle"
                assert "/root/reference" not in text, f"{f} reads the reference at run time"


def test_argument_validation_matches_reference_exceptions():
    import quantized_distillation_b200.quantization as Q
    with pytest.raises(ValueError):
        Q.ScalingFunction("cubic", False, False, None)
    with pytest.raises(ValueError):
        Q.ScalingFunction("linear", False, False, 0)
    with pytest.raises(ValueError):
        Q.ScalingFunction("linear", False, False, 2.5)
    with pytest.raises(ValueError):
        Q.ScalingFunction("linear", True, False, None)
    with pytest.raises(NotImplementedError):
        Q.ScalingFunction("absmax", False, False, None)
    with pytest.raises(ValueError):
        Q.nonUniformQuantization(torch.randn(4), [0.0, 1.0], scaling_function=object())
    with pytest.raises(ValueError):
        Q.nonUniformQuantization_variable(pre_process_tensors=True, tensor=None)
    with pytest.raises(TypeError):
        Q.uniformQuantization(torch.randn(4).double(), 16)
    f = Q.uniformQuantization_variable(16, bucket_size=256)
    with pytest.raises(ValueError):
        f.backward(torch.randn(4))
    assert Q.__all__ == ("uniformQuantization", "ScalingFunction", "nonUniformQuantization",
                         "uniformQuantization_variable", "nonUniformQuantization_variable")


def test_install_as_quantization_aliases_the_reference_name():
    import sys
    import quantized_distillation_b200 as pkg
    saved = {k: sys.modules.get(k) for k in ("quantization", "quantization.quant_functions", "quantization.help_functions")}
    try:
        pkg.install_as_quantization()
        import quantization
        import quantization.help_functions as qhf
        assert quantization.uniformQuantization is pkg.quantization.uniformQuantization
        assert qhf.create_bucket_tensor is pkg.quantization.help_functions.create_bucket_tensor
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def test_create_bucket_tensor_semantics():
    from oracle import quant_oracle as O
    from quantized_distillation_b200.quantization.help_functions import create_bucket_tensor
    for n in (1, 5, 256, 257, 1000):
        for b in (None, 2, 256):
            t = torch.arange(n, dtype=torch.float32)
            got = create_bucket_tensor(t, b)
            if b is None:
                assert got is t
            else:
                assert np.array_equal(got.numpy(), O.bucketed(t.numpy(), b))
    nanfill = create_bucket_tensor(torch.arange(5.0), 2, fill_values="nan")
    assert torch.isnan(nanfill[-1, -1]) and nanfill.shape == (3, 2)


def test_assign_bits_and_huffman_host_logic(golden):
    from oracle import quant_oracle as O
    from quantized_distillation_b200.quantization import help_functions as H
    # assign_bits_automatically: budget is preserved, more gradient -> not fewer points
    alloc = H.assign_bits_automatically([1.0, 2.0, 4.0, 1.0], 4, input_is_point=True)
    assert sum(alloc) == 16 and alloc[2] == max(alloc)
    alloc = H.assign_bits_automatically([1.0, 1.0], [4, 8])
    assert sum(alloc) == 12
    with pytest.raises(ValueError):
        H.assign_bits_automatically([1.0], [4, 4])
    code = dict((sym, bits) for sym, bits in H.huffman_encode({0: 0.5, 1: 0.25, 2: 0.125, 3: 0.125}))
    assert [len(code[k]) for k in range(4)] == [1, 2, 3, 3]
    counts = [50, 25, 13, 12]
    freq = {i: c / 100 for i, c in enumerate(counts)}
    mean = sum(freq[s] * len(b) for s, b in H.huffman_encode(freq))
    assert abs(mean - O.huffman_mean_bit_length(counts)) < 1e-12


def test_percentile_plan_is_numpy_percentile():
    from quantized_distillation_b200.quantization import help_functions as H
    rng = np.random.default_rng(0)
    # restated index / interpolation arithmetic (no numpy private imports) == np.percentile, bit for bit
    for n in (1, 2, 3, 10, 255, 256, 257, 1000, 4099, 100003):
        for K in (1, 2, 3, 4, 16, 17, 40, 256):
            v = rng.random(n).astype(np.float32)
            o = np.sort(v)
            p, nx, g = H.percentile_plan(n, K)
            ours = np.asarray(H.percentile_combine(o[p], o[nx], g), dtype=np.float64)
            ref = np.asarray(np.percentile(v, np.linspace(0, 100, num=K)), dtype=np.float64)
            assert np.array_equal(ours.view(np.uint64), ref.view(np.uint64)), (n, K)


def test_compiled_front_door_builds_and_refuses_cpu_tensors():
    """csrc/qd_torch_fast.cpp: host-only C++ (pybind11 + ATen) around the C ABI.  It must build against this
    interpreter's torch, load next to libqd_b200.so, and -- like everything else here -- never compute on the CPU."""
    import torch
    from quantized_distillation_b200 import _native as N
    from quantized_distillation_b200 import build as B
    try:
        B.build_fast()
    except Exception as e:                       # no ninja / C++ toolchain on this host: the ctypes path is the product
        pytest.skip(f"fast-call module cannot be built here: {e}")
    N._fast_tried = False
    mod = N.fast()
    assert mod is not None and hasattr(mod, "uniform_fwd") and hasattr(mod, "uniform_bwd")
    with pytest.raises(RuntimeError):
        mod.uniform_fwd(torch.zeros(16), 16, 0, False)


def test_host_helpers_match_reference_executed_fixtures():
    """The host-side helpers around the hot path against outputs of the reference's own functions
    (tests/golden/make_golden_host.py -> reference_host_logic.json): bit allocation, Huffman code, bucket view,
    learning-rate schedules, size accounting, state-dict prefixes."""
    import json
    import math
    from collections import OrderedDict
    from quantized_distillation_b200 import codec, distributed as D
    from quantized_distillation_b200.cnn_models import help_fun as hf
    from quantized_distillation_b200.quantization import help_functions as H
    with open(os.path.join(ROOT, "tests", "golden", "reference_host_logic.json")) as f:
        ref = json.load(f)

    for c in ref["assign_bits_automatically"]:
        init = c["initial"] if isinstance(c["initial"], int) else list(c["initial"])
        assert H.assign_bits_automatically(list(c["norms"]), init, input_is_point=c["input_is_point"]) == c["result"]

    for c in ref["huffman_encode"]:
        freq = {int(s): f for s, f in c["freq"]}
        assert [[s, bits] for s, bits in H.huffman_encode(freq)] == [[int(s), bits] for s, bits in c["code"]]

    for c in ref["create_bucket_tensor"]:
        t = torch.arange(c["n"], dtype=torch.float32) * 0.5 - 3
        r = H.create_bucket_tensor(t.clone(), c["bucket"], fill_values=c["fill"])
        assert list(r.shape) == c["shape"], c
        tail = [None if v != v else v for v in r.reshape(-1)[-8:].tolist()]
        assert tail == c["tail"], c

    for c in ref["learning_rate_scheduler"]:
        sch = hf.LearningRateScheduler(c["initial"], c["style"])
        for epoch, err, lr, stop in c["trace"]:
            got_lr, got_stop = sch.update_learning_rate(epoch, err)
            assert got_lr == lr and bool(got_stop) == stop, (c["style"], epoch, got_lr, lr, got_stop, stop)

    for c in ref["get_size_reduction"]:
        assert math.isclose(codec.get_size_reduction(c["bits"], bucket_size=c["bucket"], full_precision_bits=c["full"]), c["result"],
                            rel_tol=0, abs_tol=0), c

    p = ref["state_dict_prefix"]
    sd = OrderedDict((k, 0) for k in p["keys"])
    wrapped = D.convert_state_dict_to_data_parallel(sd)
    assert list(wrapped) == p["to"] and list(D.convert_state_dict_from_data_parallel(wrapped)) == p["from_of_to"]
    assert p["from_with_unprefixed_key"] == "ValueError"
    with pytest.raises(ValueError):
        D.convert_state_dict_from_data_parallel(sd)


def test_built_library_is_sm_90a_code_with_tma_and_mbarrier():
    """Static proof that the product is hand-written sm_90a code (runs without a GPU): the library embeds only
    sm_90a cubins, and their SASS holds the instructions the design rests on -- UBLKCP + SYNCS (TMA bulk copies
    completing on mbarriers: the staged chunk ring), NaN-propagating float min/max (FMNMX) for the row statistics,
    no tensor-core instruction (the path is elementwise + reductions)."""
    import shutil
    import subprocess
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    from quantized_distillation_b200 import _native as N
    elfs = subprocess.run([cuobjdump, "-lelf", N.LIB_PATH], capture_output=True, text=True, check=True).stdout.split("\n")
    elfs = [line for line in elfs if line.startswith("ELF file")]
    assert elfs and all(".sm_90a." in line for line in elfs), elfs
    sass = subprocess.run([cuobjdump, "-sass", N.LIB_PATH], capture_output=True, text=True, check=True).stdout
    count = lambda mnemonic: len(re.findall(r"\b" + mnemonic, sass))
    assert count(r"FMNMX\.NAN") > 500
    assert count("UBLKCP") > 20 and count("SYNCS") > 50
    assert count("HMMA") == 0 and count("HGMMA") == 0
    for kernel in ("warp_rows_kernel", "staged_rows_kernel", "points_grad_partial", "plan_sgd_step", "grid_apply"):
        assert kernel in sass, kernel
