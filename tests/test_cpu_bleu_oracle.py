"""The BLEU oracle (oracle/bleu_oracle.py) against the reference's own multi-bleu.perl, run by
tests/golden/make_golden_bleu.py into tests/golden/reference_bleu.json: every case's stdout byte for byte, with and
without -lc, in list mode (the drop-in's joined strings) and in file mode (perl's reference-file search); and the host
half of quantized_distillation_b200.bleu (line reading, lowercasing, splitting, word table, format_line, reference-file
search) against the oracle."""
import base64
import json
import os
import random

import pytest

from oracle import bleu_oracle as O
from quantized_distillation_b200 import bleu

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = json.load(open(os.path.join(HERE, "golden", "reference_bleu.json")))["cases"]


def _d(s):
    return base64.b64decode(s)


def _write_files(c, d):
    stem = os.path.join(d, "ref")
    for suffix, data in c["files"]:
        with open(stem + suffix, "wb") as f:
            f.write(_d(data))
    return stem


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_oracle_reproduces_perl(c, tmp_path):
    out = _d(c["stdout"])
    got, status = O.multi_bleu(_d(c["stdin"]), [_d(b) for _, b in c["files"]], c["lowercase"])
    assert got == out
    assert (status == 0) == (c["status"] == 0)
    if c["mode"] == "list":
        assert O.list_mode_streams(c["hypotheses"], c["reference"]) == (_d(c["stdin"]), _d(c["files"][0][1]))
        if c["lowercase"]:
            assert O.get_bleu_moses(c["hypotheses"], c["reference"]) == out
    stem = _write_files(c, str(tmp_path))
    if c["mode"] == "list":
        assert O.find_reference_files(stem) == [_d(c["files"][0][1])]
    if c["mode"] == "file" and c["lowercase"]:
        hyp = os.path.join(str(tmp_path), "hyp.txt")
        with open(hyp, "wb") as f:
            f.write(_d(c["stdin"]))
        assert O.get_bleu_moses(hyp, stem, file_input=True) == out


def test_file_mode_finds_references_as_perl(tmp_path):
    for c in CASES:
        if c["mode"] != "file":
            continue
        d = tmp_path / c["name"]
        d.mkdir()
        stem = _write_files(c, str(d))
        got = bleu.reference_files(stem)
        assert got == O.find_reference_files(stem)
        # perl's order: stem0, stem1, ..., then stem itself
        order = sorted((s for s, _ in c["files"]), key=lambda s: (s == "", s))
        assert got == [_d(dict(c["files"])[s]) for s in order]


def test_host_tokeniser_matches_oracle():
    blobs = [_d(c["stdin"]) for c in CASES] + [_d(b) for c in CASES for _, b in c["files"]]
    g = random.Random(1)
    alphabet = b"aAbBzZ \t\n\r\x0b\x0c\xa0\x85\xc3\x84\xe4."
    blobs += [bytes(g.choice(alphabet) for _ in range(g.randint(0, 60))) for _ in range(300)]
    for data in blobs:
        assert bleu.perl_lines(data) == O.perl_lines(data)
        for line in O.perl_lines(data):
            for lc in (True, False):
                assert bleu.perl_words(line, lc) == O.perl_words(line, lc)
    assert bleu.perl_words(b"A\xa0B\x85C \xc3\x84\tD", True) == [b"a\xa0b\x85c", b"\xc3\x84", b"d"]
    assert bleu.perl_lines(b"ab\ncd") == [b"ab", b"c"] and bleu.perl_lines(b"") == [] and bleu.perl_lines(b"\n") == [b""]


def test_word_table_interns_by_equality():
    t = bleu.WordTable()
    words = [b"a", b"b", b"a", b"\xc3\x84", b"A", b"b"]
    ids = t.intern(words)
    assert ids == [0, 1, 0, 2, 3, 1] and len(t) == 4
    assert t.intern([b"A", b"new"]) == [3, 4]


def test_format_line_matches_oracle():
    totals = []
    for c in CASES:
        refs = []
        for _, b in c["files"]:
            for s, line in enumerate(O.perl_lines(_d(b))):
                if s == len(refs):
                    refs.append([])
                refs[s].append(O.perl_words(line, c["lowercase"]))
        hyps = [O.perl_words(line, c["lowercase"]) for line in O.perl_lines(_d(c["stdin"]))]
        totals.append(O.fold(O.corpus_stats(hyps, refs)))
    g = random.Random(2)
    for _ in range(2000):
        total = [g.choice([0, g.randint(1, 50), g.randint(1, 10 ** 6)]) for _ in range(4)]
        correct = [g.randint(0, t) for t in total]
        totals.append([g.choice([0, g.randint(1, 10 ** 6)]), g.choice([0, g.randint(1, 10 ** 6)])] + correct + total)
    for t in totals:
        assert bleu.format_line(t) == O.format_line(t)[0], t
        line = bleu.format_line(t)
        if line and t[1]:
            assert line.startswith(b"BLEU = %.2f," % bleu.bleu_value(t))
