"""Generates tests/golden/containers.npz: the exact bytes save_compressed and save_packed write for a few small models
built on the host, so that tests/test_cpu_codec_container_format.py pins both file formats byte for byte.  The models
come from seeded NumPy draws: Huffman streams encoded by oracle/huffman_oracle.py, fixed-width codes packed in NumPy.
No GPU is needed:

    python tests/golden/make_golden_containers.py
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "containers.npz")


def _f32(rng, *shape):
    import torch
    return torch.from_numpy(rng.standard_normal(shape).astype(np.float32))


def _buffers(rng):
    """float32 and int64 buffers, a scalar of each and an empty one."""
    import torch
    return [("bn.running_mean", _f32(rng, 7)), ("bn.running_var", torch.from_numpy(rng.random((3, 2)).astype(np.float32))),
            ("bn.num_batches_tracked", torch.tensor(5, dtype=torch.int64)), ("scale", torch.tensor(1.5)),
            ("steps", torch.arange(-3, 6, dtype=torch.int64).view(3, 3)), ("empty", torch.zeros(0))]


def _huffman(kind, levels, bucket, shapes, symbols, points=None, buffers=None, seed=0):
    """A CompressedModel: float32 first and last tensors around quantized ones whose level indices are ``symbols``."""
    import torch
    from oracle import huffman_oracle as HO
    from quantized_distillation_b200 import codec
    rng = np.random.default_rng(seed)
    counts = np.bincount(np.concatenate(symbols), minlength=256)
    lengths = {0: 0} if np.count_nonzero(counts) == 1 else codec.huffman_code_lengths(counts)
    tensors = [codec.HuffmanTensor("first", (3, 5), raw=_f32(rng, 15))]
    for k, (shape, s) in enumerate(zip(shapes, symbols)):
        words, offs = HO.encode(s, lengths)
        rows = codec._rows(s.size, bucket)
        tensors.append(codec.HuffmanTensor(f"layer{k}.weight", shape, words=torch.from_numpy(words.view(np.int32)),
                                           chunk_offsets=torch.from_numpy(offs.view(np.int32)),
                                           alpha=torch.from_numpy(rng.random(rows).astype(np.float32)), beta=_f32(rng, rows),
                                           points=None if points is None else torch.tensor(points[k], dtype=torch.float32),
                                           code_bits=int(sum(lengths[v] for v in s.tolist()))))
    tensors.append(codec.HuffmanTensor("last", (4,), raw=_f32(rng, 4)))
    return codec.CompressedModel(kind, levels, bucket, lengths, tensors, buffers=buffers)


def _pack(codes, bits):
    """The qd_pack_indices layout: code of element e in byte e*bits/8 at bit (e*bits)%8, little endian."""
    out = np.zeros((codes.size * bits + 7) // 8, np.uint8)
    for e, c in enumerate(codes.tolist()):
        out[e * bits // 8] |= (c << (e * bits % 8)) & 0xFF
    return out


def _packed(kind, levels, bucket, shapes, bits, points=None, buffers=None, seed=0):
    """A PackedModel: a float32 first tensor, then quantized tensors of the given code widths, then a float32 one."""
    import torch
    from quantized_distillation_b200 import codec
    rng = np.random.default_rng(seed)
    tensors = [codec.PackedEntry("first", (2, 3), raw=_f32(rng, 6))]
    for k, (shape, b) in enumerate(zip(shapes, bits)):
        n = int(np.prod(shape))
        count = levels if kind == "uniform" else len(points[k])
        rows = codec._rows(n, bucket)
        tensors.append(codec.PackedEntry(f"layer{k}.weight", shape, bits=b, packed=torch.from_numpy(_pack(rng.integers(0, count, n), b)),
                                         alpha=torch.from_numpy(rng.random(rows).astype(np.float32)), beta=_f32(rng, rows),
                                         points=None if points is None else torch.tensor(points[k], dtype=torch.float32)))
    tensors.append(codec.PackedEntry("last", (5,), raw=_f32(rng, 5)))
    return codec.PackedModel(kind, levels, bucket, tensors, buffers=buffers)


def models():
    """{case: (model, "huffman" | "packed")}, the same objects on every call."""
    rng = np.random.default_rng(7)
    sym = [rng.integers(0, 16, n).astype(np.uint8) for n in (2000, 7 * 300)]
    sym4 = [rng.integers(0, 4, n).astype(np.uint8) for n in (1500, 64)]
    zeros = [np.zeros(n, np.uint8) for n in (1000, 37)]
    return {
        "huffman_v1_uniform_bucket256": (_huffman("uniform", 16, 256, [(2000,), (7, 300)], sym, seed=1), "huffman"),
        "huffman_v2_buffers": (_huffman("uniform", 4, 64, [(1500,), (8, 8)], sym4, buffers=_buffers(np.random.default_rng(2)),
                                        seed=3), "huffman"),
        "huffman_nonuniform_single_symbol": (_huffman("nonuniform", None, None, [(10, 100), (37,)], zeros,
                                                      points=[[-0.5, 0.0, 0.25], [-1.0, -0.1, 0.2, 0.6, 1.5]], seed=4), "huffman"),
        "packed_mixed_widths_buffers": (_packed("uniform", 4, 256, [(2048,), (30, 50), (513,)], (2, 4, 8),
                                                buffers=_buffers(np.random.default_rng(5)), seed=6), "packed"),
        "packed_nonuniform_points": (_packed("nonuniform", None, 100, [(999,), (4, 250)], (2, 4),
                                             points=[[-0.5, 0.0, 0.25], [-1.0, -0.1, 0.2, 0.6, 0.7, 0.8, 1.5, 2.0, 2.5]], seed=8),
                                     "packed"),
        "packed_no_buffers": (_packed("uniform", 2, None, [(100,), (3, 17)], (1, 1), seed=9), "packed"),
    }


def file_bytes(model, fmt):
    from quantized_distillation_b200 import codec
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "m")
        (codec.save_compressed if fmt == "huffman" else codec.save_packed)(model, path)
        with open(path, "rb") as f:
            return f.read()


def main():
    sys.path.insert(0, ROOT)
    out = {case: np.frombuffer(file_bytes(m, fmt), np.uint8) for case, (m, fmt) in models().items()}
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, len(out), "files")


if __name__ == "__main__":
    main()
