"""NumPy restatement of the Huffman-coded model format (checker only; the product never imports it).

Canonical code: codewords assigned in (length, symbol) order, each the previous one plus one, shifted left to
its length.  Stream: symbols cut into chunks of CHUNK; a chunk's codes are concatenated MSB-first into uint32
words starting on a fresh word; offsets[c] = first word of chunk c."""
import numpy as np

CHUNK = 1024


def canonical_codes(lengths):
    out, code, prev = {}, 0, None
    for sym in sorted(lengths, key=lambda s: (lengths[s], s)):
        l = lengths[sym]
        code = 0 if prev is None else (code + 1) << (l - prev)
        out[sym] = code
        prev = l
    return out


def encode(symbols, lengths):
    """(words uint32, offsets uint32) of a uint8 symbol array."""
    sym = np.asarray(symbols, dtype=np.int64).reshape(-1)
    n = sym.size
    codes = canonical_codes(lengths)
    len_tab = np.zeros(256, np.int64)
    code_tab = np.zeros(256, np.uint64)
    for s, l in lengths.items():
        len_tab[s], code_tab[s] = l, codes[s]
    L, C = len_tab[sym], code_tab[sym]
    chunks = -(-n // CHUNK)
    chunk_of = np.arange(n) // CHUNK
    csum = np.cumsum(L)
    chunk_end = csum[np.minimum(np.arange(1, chunks + 1) * CHUNK, n) - 1]
    chunk_bits = np.diff(np.concatenate([[0], chunk_end]))
    chunk_words = (chunk_bits + 31) // 32
    offsets = np.concatenate([[0], np.cumsum(chunk_words)[:-1]]).astype(np.int64)
    pos_in_chunk = csum - L - np.concatenate([[0], chunk_end])[chunk_of]
    total = int(chunk_words.sum())
    words = np.zeros(total + 2, np.uint64)      # 2 words of slack for the placement below, dropped at the end
    keep = L > 0
    g = offsets[chunk_of[keep]] * 32 + pos_in_chunk[keep]
    Lk, Ck = L[keep].astype(np.uint64), C[keep]
    w = g // 32
    t = (g % 32).astype(np.uint64) + Lk            # end bit of the code counted from the start of word w, <= 88
    # 96-bit big-endian window starting at word w: code occupies bits [t - L, t)
    lo = t <= 64
    v = np.where(lo, Ck << (np.uint64(64) - np.minimum(t, np.uint64(64))), Ck >> (np.maximum(t, np.uint64(64)) - np.uint64(64)))
    np.bitwise_or.at(words, w, v >> np.uint64(32))
    np.bitwise_or.at(words, w + 1, v & np.uint64(0xFFFFFFFF))
    hi = ~lo
    third = (Ck[hi] << (np.uint64(96) - t[hi])) & np.uint64(0xFFFFFFFF)
    np.bitwise_or.at(words, w[hi] + 2, third)
    return words[:total].astype(np.uint32), offsets.astype(np.uint32)


def decode(words, offsets, lengths, n):
    """Symbols back from (words, offsets): bit-serial canonical decoding (small inputs only)."""
    words = np.asarray(words, dtype=np.uint32)
    out = np.zeros(n, np.uint8)
    if len(lengths) == 1:
        out[:] = next(iter(lengths))
        return out
    codes = canonical_codes(lengths)
    by_code = {(lengths[s], c): s for s, c in codes.items()}
    for c, off in enumerate(np.asarray(offsets, dtype=np.int64)):
        bitpos = int(off) * 32
        for e in range(c * CHUNK, min(n, (c + 1) * CHUNK)):
            code, l = 0, 0
            while True:
                bit = (int(words[bitpos // 32]) >> (31 - bitpos % 32)) & 1
                bitpos += 1
                code, l = (code << 1) | bit, l + 1
                if (l, code) in by_code:
                    out[e] = by_code[(l, code)]
                    break
                if l > 64:
                    raise ValueError("not a codeword")
    return out
