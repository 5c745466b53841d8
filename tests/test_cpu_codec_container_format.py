"""Both stored-model file formats, pinned byte for byte (no GPU): the models of tests/golden/make_golden_containers.py
must save to exactly the bytes in tests/golden/containers.npz, and every stored file must load back to the sections,
points and buffers of the model it was written from.  The cases cover Huffman version 1 and version 2 (float32, int64,
scalar and empty buffers), a non-uniform Huffman model with per-tensor points, no buckets and a single-symbol code,
and fixed-width models with mixed code widths and buffers, with per-tensor points, and without a buffers key."""
import importlib.util
import os

import numpy as np
import pytest
import torch

from quantized_distillation_b200 import codec

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location("make_golden_containers", os.path.join(HERE, "golden", "make_golden_containers.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)

GOLDEN = np.load(os.path.join(HERE, "golden", "containers.npz"))
MODELS = G.models()


def test_the_fixtures_cover_every_case():
    assert sorted(GOLDEN.files) == sorted(MODELS)


@pytest.mark.parametrize("case", sorted(MODELS))
def test_writer_reproduces_the_stored_bytes(case):
    model, fmt = MODELS[case]
    assert G.file_bytes(model, fmt) == GOLDEN[case].tobytes()


def _same(a, b, what):
    assert (a is None) == (b is None), what
    if a is not None:
        assert not b.is_cuda and a.dtype == b.dtype and tuple(a.shape) == tuple(b.shape) and torch.equal(a, b), what


@pytest.mark.parametrize("case", sorted(MODELS))
def test_stored_file_loads_to_the_model_it_was_written_from(case, tmp_path):
    model, fmt = MODELS[case]
    path = tmp_path / "m"
    path.write_bytes(GOLDEN[case].tobytes())
    back = codec.load_compressed(path) if fmt == "huffman" else codec.load_packed(path)
    assert type(back) is type(model)
    assert (back.kind, back.levels, back.bucket_size) == (model.kind, model.levels, model.bucket_size)
    fields = ["words", "chunk_offsets", "alpha", "beta", "raw"] if fmt == "huffman" else ["packed", "alpha", "beta", "raw"]
    if fmt == "huffman":
        assert back.code_lengths == model.code_lengths and back.chunk == model.chunk
    assert len(back.tensors) == len(model.tensors)
    for a, b in zip(model.tensors, back.tensors):
        assert (a.name, tuple(a.shape), a.quantized) == (b.name, tuple(b.shape), b.quantized)
        assert (a.code_bits if fmt == "huffman" else a.bits) == (b.code_bits if fmt == "huffman" else b.bits)
        for f in fields:
            x = getattr(a, f)
            _same(None if x is None else x.reshape(-1), getattr(b, f), f"{a.name}.{f}")
        _same(a.points, b.points, f"{a.name}.points")
    assert (back.buffers is None) == (model.buffers is None)
    assert [n for n, _ in back.buffers or []] == [n for n, _ in model.buffers or []]
    for (name, a), (_, b) in zip(model.buffers or [], back.buffers or []):
        _same(a, b, name)
    assert back.size_breakdown() == model.size_breakdown()
