"""H100 counterpart of the reference's ``quantization/help_functions.py``:
bucketing view, centroid initialisation, bit allocation and Huffman statistics.
Only what the quantized-distillation / differentiable-quantization loops and the
size accounting call is provided (the hyperspherical helpers, :8-65, are unused
by the reference itself)."""
from __future__ import annotations

import heapq
from collections import defaultdict

import numpy as np
import torch

from .. import _native as N

__all__ = ("create_bucket_tensor", "assign_bits_automatically", "initialize_quantization_points", "huffman_encode",
           "get_huffman_encoding_mean_bit_length", "huffman_code_of_histogram", "index_histogram", "order_statistics",
           "gradient_norms")


def create_bucket_tensor(tensor, bucket_size, fill_values="last"):
    """Row view of a tensor: ``(ceil(n/b), b)`` with the tail padded with the
    last element (or NaN), ``(1, n)`` when n < b (reference: help_functions.py:67-94).
    The kernels never materialise this view -- they do the index arithmetic --
    so this is only for callers that want the padded tensor itself."""
    if bucket_size is None:
        return tensor
    tensor = tensor.view(-1)
    n = tensor.numel()
    multiple, rest = divmod(n, bucket_size)
    if multiple != 0 and rest != 0:
        fill = float("nan") if fill_values == "nan" else tensor[-1]
        pad = torch.ones(bucket_size - rest, dtype=tensor.dtype, device=tensor.device) * fill
        tensor = torch.cat([tensor, pad])
    return tensor.view(1, n) if multiple == 0 else tensor.view(-1, bucket_size)


def assign_bits_automatically(gradient_norms, inital_bits_to_assign, input_is_point=False):
    """Redistribute a bit (or point) budget across tensors in proportion to
    their gradient norms (reference: help_functions.py:97-138)."""
    norms = [float(g) for g in gradient_norms]
    if isinstance(inital_bits_to_assign, int):
        inital_bits_to_assign = [inital_bits_to_assign] * len(norms)
    if len(inital_bits_to_assign) != len(norms):
        raise ValueError("There should be as many gradients as there are initial points.")
    budget = sum(inital_bits_to_assign)
    floor_alloc = [x // 2 for x in inital_bits_to_assign] if input_is_point else [x - 1 for x in inital_bits_to_assign]
    spare = budget - sum(floor_alloc)
    total_norm = sum(norms)
    alloc = [base + round(g / total_norm * spare) for g, base in zip(norms, floor_alloc)]
    excess = sum(alloc) - budget
    if excess > 0:
        alloc[alloc.index(max(alloc))] -= excess
    elif excess < 0:
        alloc[alloc.index(min(alloc))] += -excess
    return alloc


def percentile_plan(n: int, num_points: int, dtype=np.float32):
    """Which order statistics ``np.percentile(v, linspace(0,100,K))`` reads and with which
    weights, for ``len(v) == n`` and the default ``method='linear'``: virtual index
    ``(n-1)*q`` in float64 with ``q = linspace(0,100,K) / float32(100)`` (the division numpy
    makes for a float32 array), previous = floor, next = previous+1, both set to the last
    element once the virtual index reaches ``n-1``; gamma = virtual - previous.  Restated
    from the documented algorithm; pinned against ``np.percentile`` itself in
    tests/test_cpu_boundary.py.  Returns (prev_idx, next_idx, gamma)."""
    q = np.true_divide(np.linspace(0, 100, num=num_points), dtype(100))
    virt = (n - 1) * q
    prev = np.floor(virt).astype(np.intp)
    nxt = prev + 1
    above = virt >= n - 1
    prev[above] = n - 1
    nxt[above] = n - 1
    below = virt < 0
    prev[below] = 0
    nxt[below] = 0
    gamma = np.asarray(virt - prev, dtype=virt.dtype)
    return prev, nxt, gamma


def percentile_combine(prev_vals: np.ndarray, next_vals: np.ndarray, gamma: np.ndarray) -> np.ndarray:
    """numpy's linear interpolation of the two neighbours: ``a + (b-a)*t``, and
    ``b - (b-a)*(1-t)`` where ``t >= 0.5`` (float32 difference, float64 product and sum)."""
    a, b = np.asarray(prev_vals), np.asarray(next_vals)
    diff = np.subtract(b, a)
    out = np.asarray(np.add(a, diff * gamma))
    hi = gamma >= 0.5
    out[hi] = np.subtract(b, diff * (1 - gamma))[hi]
    return out


def initialize_quantization_points(tensor, scaling_function, num_points):
    """Percentile initialisation of the centroids on the scaled tensor
    (reference: help_functions.py:140-154).  The scaling runs on the GPU and the 2K order
    statistics numpy's percentile would read are SELECTED there (qd_order_statistics: value
    histogram + compaction + radix select, no sort); only those 2K floats come to the host,
    where they are combined with numpy's interpolation formula, so the result is bit-identical
    to ``np.percentile`` over the whole array."""
    scaled = scaling_function.scale_down(tensor).view(-1)[0:scaling_function.original_tensor_length]
    n = scaled.numel()
    if not scaled.is_cuda:
        N.require_cuda()
        scaled = scaled.cuda()
    prev, nxt, gamma = percentile_plan(n, num_points)
    picks = order_statistics(scaled, np.concatenate([prev, nxt])).cpu().numpy()
    initial_points = percentile_combine(picks[:num_points], picks[num_points:], gamma)
    initial_points = torch.from_numpy(np.asarray(initial_points)).type_as(tensor)
    return initial_points.to(tensor.device)


def order_statistics(values: torch.Tensor, ranks) -> torch.Tensor:
    """The ``ranks``-th smallest elements (0-based) of a float32 CUDA tensor, exactly, without
    sorting it (qd_order_statistics).  At most 512 ranks per call."""
    N.require_cuda()
    values = values.contiguous().view(-1)
    ranks_t = torch.as_tensor(np.asarray(ranks, dtype=np.int64)).to(values.device)
    out = torch.empty(ranks_t.numel(), dtype=torch.float32, device=values.device)
    ws_bytes = int(N.lib().qd_order_statistics_workspace_bytes(values.numel()))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=values.device)
    N.check(N.lib().qd_order_statistics(N.ptr(values), values.numel(), N.ptr(ranks_t), ranks_t.numel(), N.ptr(out),
                                        N.ptr(ws), ws_bytes, N.stream_ptr(values.device)))
    return out


def gradient_norms(tensors):
    """L2 norm of every tensor of a list in two launches (qd_multi_l2norm), as a float32 CUDA tensor."""
    import ctypes as C
    N.require_cuda()
    tensors = [t.contiguous() for t in tensors]
    dev = tensors[0].device
    out = torch.empty(len(tensors), dtype=torch.float32, device=dev)
    ptrs = (C.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])
    ns = (C.c_int64 * len(tensors))(*[t.numel() for t in tensors])
    with torch.cuda.device(dev):
        N.check(N.lib().qd_multi_l2norm(ptrs, ns, len(tensors), N.ptr(out), N.stream_ptr(dev)))
    return out


def huffman_encode(symb2freq):
    """Huffman code of a {symbol: weight} dict as a list of [symbol, code]
    (reference: help_functions.py:157-172)."""
    heap = [[wt, [sym, ""]] for sym, wt in symb2freq.items()]
    heapq.heapify(heap)
    while len(heap) > 1:
        lo, hi = heapq.heappop(heap), heapq.heappop(heap)
        for pair in lo[1:]:
            pair[1] = "0" + pair[1]
        for pair in hi[1:]:
            pair[1] = "1" + pair[1]
        heapq.heappush(heap, [lo[0] + hi[0]] + lo[1:] + hi[1:])
    return sorted(heapq.heappop(heap)[1:], key=lambda p: (len(p[-1]), p))


def index_histogram(idx_u8: torch.Tensor, num_bins: int, counts: torch.Tensor = None) -> torch.Tensor:
    """counts[b] += #{idx == b} on the GPU (qd_index_histogram)."""
    N.require_cuda()
    idx_u8 = idx_u8.contiguous().view(-1)
    if counts is None:
        counts = torch.zeros(num_bins, dtype=torch.int64, device=idx_u8.device)
    N.check(N.lib().qd_index_histogram(N.ptr(idx_u8), idx_u8.numel(), num_bins, N.ptr(counts), N.stream_ptr(idx_u8.device)))
    return counts


def _add_counts(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    if a.numel() < b.numel():
        a, b = b, a
    a = a.clone()
    a[: b.numel()] += b
    return a


def get_huffman_encoding_mean_bit_length(model_param_iter, quantization_functions, type_quantization="uniform", s=None):
    """Mean Huffman code length over the quantization indices of a whole model
    (reference: help_functions.py:175-232).

    ``quantization_functions`` are callables with the reference's contracts:
    uniform -> ``(q, ScalingFunction)``, nonUniform -> ``(q, indices, sf)``.  For
    the uniform case the reference recovers the integer level from the
    quantized tensor with ``np.digitize`` on the re-scaled values (:213-218);
    here the same re-scaling runs on the GPU and the level is
    ``floor(x_hat*(s-1) + 1e-5*(s-1))``-equivalent digitisation done on device,
    followed by a device histogram -- no per-tensor numpy round trip."""
    type_quantization = type_quantization.lower()
    if type_quantization not in ("uniform", "nonuniform"):
        raise ValueError("type_quantization not recognized")
    if s is None and type_quantization == "uniform":
        raise ValueError("If type of quantization is uniform, you must provide s")
    if not isinstance(quantization_functions, list):
        quantization_functions = [quantization_functions]
    single = len(quantization_functions) == 1
    total_length = 0
    counts = None
    tol = 1e-5
    for idx, param in enumerate(model_param_iter):
        param = param.data if hasattr(param, "data") else param
        param = param.clone()
        total_length += param.numel()
        quant_fun = quantization_functions[0] if single else quantization_functions[idx]
        if type_quantization == "uniform":
            q_tensor, scal = quant_fun(param)
            scaled = scal.scale_down(q_tensor).view(-1)[0:scal.original_tensor_length]
            edges = torch.tensor([x / (s - 1) - tol for x in range(s)], dtype=torch.float64, device=scaled.device)
            # np.digitize(v, edges) - 1 == (number of edges <= v) - 1, compared in float64 like numpy does
            bins = (torch.searchsorted(edges, scaled.to(torch.float64), right=True) - 1).clamp_(min=0)
            nbins = s
        else:
            _, bins, _ = quant_fun(param)
            bins = bins.view(-1)
            nbins = 256
        if not bins.is_cuda:
            N.require_cuda()
            bins = bins.cuda()
        if nbins > 256:
            # more than 8 bits per weight (the reference accepts any s): uint8 codes do not exist,
            # count the int64 levels with torch instead of the uint8 histogram kernel
            wide = torch.bincount(bins.view(-1).to(torch.int64), minlength=nbins)
            counts = wide if counts is None else _add_counts(counts, wide)
            continue
        bins_u8 = bins.to(torch.uint8)
        if counts is None:
            counts = torch.zeros(256, dtype=torch.int64, device=bins_u8.device)
        elif counts.numel() < 256:
            counts = _add_counts(counts, torch.zeros(256, dtype=torch.int64, device=counts.device))
        index_histogram(bins_u8, max(nbins, 1), counts[:256])
    counts = counts.cpu().numpy()
    assert total_length == int(counts.sum())                                              # :227
    frequency, code = huffman_code_of_histogram(counts)
    return sum(frequency[sym] * len(bits) for sym, bits in code)


def huffman_code_of_histogram(counts):
    """(frequency, code) of a level histogram the way the reference builds them (help_functions.py:226-231):
    ``frequency[level] = count / total`` over the non-zero bins, then ``huffman_encode`` on that dict.  The
    size accounting above and the Huffman codec (codec.py) both take their code from here, so float ties
    break identically and the stored stream has exactly the accounted length."""
    counts = np.asarray(counts)
    total_length = int(counts.sum())
    frequency = defaultdict(int)
    for val in np.nonzero(counts)[0]:
        frequency[int(val)] = counts[val] / total_length
    return frequency, huffman_encode(frequency)
