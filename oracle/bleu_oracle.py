"""Plain-Python restatement of perl_scripts/multi-bleu.perl (the moses script the reference's get_bleu_moses runs with
-lc), on bytes: how perl reads, chops, lowercases and splits lines, the per-sentence statistics with hash-free
n-gram counts, the printed line, and the byte streams get_bleu_moses builds (list mode) or finds (file mode).

Test infrastructure only: tests/test_cpu_bleu_oracle.py pins it on the script's own output (tests/golden/
reference_bleu.json), and the GPU tests pin the kernels on it.
"""
from __future__ import annotations

import gzip
import math
import os
import re

_LOWER = bytes.maketrans(b"ABCDEFGHIJKLMNOPQRSTUVWXYZ", b"abcdefghijklmnopqrstuvwxyz")


def perl_lines(data: bytes) -> list:
    """`while (<FH>) { chop; ... }`: lines end at \\n (the last one may not), and chop drops each line's last byte."""
    parts = data.split(b"\n")
    lines = parts[:-1]                             # each ended on \n, which chop removed
    if parts[-1]:
        lines.append(parts[-1][:-1])               # an unterminated last line: chop eats its own last byte
    return lines


def perl_words(line: bytes, lowercase: bool) -> list:
    """`$_ = lc if $lowercase; split`: lc on a byte string maps A-Z only; split ' ' cuts on space, \\t, \\n, \\r, \\v
    and \\f and drops empty fields (bytes.split() uses exactly those six)."""
    return (line.translate(_LOWER) if lowercase else line).split()


def _ngrams(words, n):
    counts = {}
    for i in range(len(words) - n + 1):
        g = tuple(words[i:i + n])
        counts[g] = counts.get(g, 0) + 1
    return counts


def sentence_stats(hyp, refs) -> list:
    """[hyp_len, closest ref_len, correct1..4, total1..4] of one hypothesis (a word list) against its references."""
    L = len(hyp)
    closest_diff, closest_len = 9999, 9999
    ref_max = {}
    for ref in refs:
        diff = abs(L - len(ref))
        if diff < closest_diff:
            closest_diff, closest_len = diff, len(ref)
        elif diff == closest_diff and len(ref) < closest_len:
            closest_len = len(ref)
        for n in range(1, 5):
            for g, c in _ngrams(ref, n).items():
                ref_max[g] = max(ref_max.get(g, 0), c)
    correct, total = [0] * 4, [0] * 4
    for n in range(1, 5):
        for g, c in _ngrams(hyp, n).items():
            total[n - 1] += c
            correct[n - 1] += min(c, ref_max.get(g, 0))
    return [L, closest_len] + correct + total


def corpus_stats(hyps, refs_per_sentence) -> list:
    """Per-sentence rows; sentence s has the references refs_per_sentence[s] (none past its end)."""
    return [sentence_stats(h, refs_per_sentence[s] if s < len(refs_per_sentence) else []) for s, h in enumerate(hyps)]


def fold(rows) -> list:
    return [sum(r[c] for r in rows) for c in range(10)] if rows else [0] * 10


def _my_log(x):
    return -9999999999 if not x else math.log(x)


def format_line(totals):
    """(stdout bytes, exit status) of multi-bleu.perl's end for the 10 corpus totals, float64 as perl computes it.
    Status 255 with no output is perl's death on a zero hypothesis length against a positive reference length."""
    hyp_len, ref_len = totals[0], totals[1]
    correct, total = totals[2:6], totals[6:10]
    prec = [(correct[n] / total[n]) if total[n] else 0 for n in range(4)]
    if ref_len == 0:
        return b"BLEU = 0, 0/0/0/0 (BP=0, ratio=0, hyp_len=0, ref_len=0)\n", 1
    bp = 1
    if hyp_len < ref_len:
        if hyp_len == 0:
            return b"", 255                        # Illegal division by zero
        bp = math.exp(1 - ref_len / hyp_len)
    s = _my_log(prec[0]) + _my_log(prec[1])
    s = s + _my_log(prec[2])
    s = s + _my_log(prec[3])
    bleu = bp * math.exp(s / 4)
    line = "BLEU = %.2f, %.1f/%.1f/%.1f/%.1f (BP=%.3f, ratio=%.3f, hyp_len=%d, ref_len=%d)\n" % (
        100 * bleu, 100 * prec[0], 100 * prec[1], 100 * prec[2], 100 * prec[3], bp, hyp_len / ref_len, hyp_len, ref_len)
    return line.encode(), 0


def multi_bleu(stdin: bytes, ref_files, lowercase: bool):
    """(stdout, status) of `perl multi-bleu.perl [-lc] stem < stdin`, ref_files the contents of the files it reads,
    in its order.  No reference line at all: perl dies before reading stdin (status nonzero, no output)."""
    refs = []
    for data in ref_files:
        for s, line in enumerate(perl_lines(data)):
            if s == len(refs):
                refs.append([])
            refs[s].append(perl_words(line, lowercase))
    if not refs:
        return b"", 255                            # die "could not find reference file"
    hyps = [perl_words(line, lowercase) for line in perl_lines(stdin)]
    return format_line(fold(corpus_stats(hyps, refs)))


def find_reference_files(stem: str) -> list:
    """The files multi-bleu.perl reads for `stem`: stem0, stem1, ... then stem itself (stem.ref0, ... when neither
    stem nor stem0 exists), each decompressed when its name ends like .gz."""
    if not os.path.exists(stem) and not os.path.exists(stem + "0") and os.path.exists(stem + ".ref0"):
        stem += ".ref"
    names = []
    i = 0
    while os.path.exists(f"{stem}{i}"):
        names.append(f"{stem}{i}")
        i += 1
    if os.path.exists(stem):
        names.append(stem)
    out = []
    for name in names:
        with open(name, "rb") as f:
            data = f.read()
        out.append(gzip.decompress(data) if re.search(r".gz\n?\Z", name) else data)
    return out


def list_mode_streams(hypotheses, reference):
    """The bytes get_bleu_moses feeds perl in list mode: the hypotheses joined by \\n with no trailing newline on
    stdin, and one reference file of `ref + '\\n'` lines."""
    return "\n".join(hypotheses).encode(), "".join(r + "\n" for r in reference).encode()


def get_bleu_moses(hypotheses, reference, file_input=False):
    """The bytes the reference's get_bleu_moses returns (always -lc)."""
    if file_input:
        with open(hypotheses, "rb") as f:
            stdin = f.read()
        refs = find_reference_files(reference)
    else:
        stdin, ref = list_mode_streams(hypotheses, reference)
        refs = [ref]
    return multi_bleu(stdin, refs, True)[0]
