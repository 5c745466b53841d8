"""Generates tests/golden/reference_bleu.json: the reference's own perl_scripts/multi-bleu.perl, run by path with perl
as the reference's get_bleu_moses runs it (translation_models/help_fun.py:313-352), with and without -lc:

- list mode: the hypotheses joined by '\\n' with no trailing newline on stdin, and one reference file holding
  `ref + '\\n'` per reference (the strings are kept, so the drop-in can be called on them);
- file mode: a hypothesis file on stdin and the reference files perl finds for a stem (stem0, stem1, ..., stem itself,
  or stem.ref0, ...), stored as (suffix, bytes) pairs.

Each case stores its inputs, perl's stdout bytes and its exit status; bytes are base64.  The corpora cover small
vocabularies (clipping), 0, 1 and 3 references and more hypotheses than references, empty lines, runs of every ASCII
whitespace byte and unterminated last lines, ASCII capitals next to UTF-8, Latin-1 and NBSP bytes, a 2,000-token line,
a line of one repeated token, a corpus without 4-grams, ref_len == 0 and hyp_len == 0.

Run in the build container only (it needs perl and the reference):  python tests/golden/make_golden_bleu.py
"""
import base64
import json
import os
import random
import subprocess
import tempfile

SCRIPT = "/root/reference/perl_scripts/multi-bleu.perl"
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "reference_bleu.json")
WS = [" ", "\t", "\n", "\r", "\x0b", "\x0c"]


def b64(b):
    return base64.b64encode(b).decode()


def run(stdin, files, lowercase):
    """perl multi-bleu.perl [-lc] <dir>/ref < stdin, with files [(suffix, bytes)] written as <dir>/ref<suffix>."""
    with tempfile.TemporaryDirectory() as d:
        stem = os.path.join(d, "ref")
        for suffix, data in files:
            with open(stem + suffix, "wb") as f:
                f.write(data)
        cmd = ["perl", SCRIPT] + (["-lc"] if lowercase else []) + [stem]
        p = subprocess.run(cmd, input=stdin, capture_output=True)
    return p.stdout, p.returncode


def sentence(rng, vocab, lo, hi):
    return " ".join(rng.choice(vocab) for _ in range(rng.randint(lo, hi)))


def list_case(name, hyps, refs, lowercase=True):
    stdin = "\n".join(hyps).encode()
    ref = "".join(r + "\n" for r in refs).encode()
    out, status = run(stdin, [("", ref)], lowercase)
    return {"name": name, "mode": "list", "lowercase": lowercase, "hypotheses": hyps, "reference": refs,
            "stdin": b64(stdin), "files": [["", b64(ref)]], "stdout": b64(out), "status": status}


def file_case(name, stdin, files, lowercase=True):
    out, status = run(stdin, files, lowercase)
    return {"name": name, "mode": "file", "lowercase": lowercase, "stdin": b64(stdin),
            "files": [[s, b64(d)] for s, d in files], "stdout": b64(out), "status": status}


def lines(strs, terminated=True):
    return ("\n".join(strs) + ("\n" if terminated else "")).encode()


def main():
    rng = random.Random(0)
    small = ["a", "b", "c", "A", "the"]
    cases = []
    # small vocabularies: repeated n-grams, so clipping decides the counts
    hyps = [sentence(rng, small, 1, 12) for _ in range(40)]
    refs = [sentence(rng, small, 1, 12) for _ in range(40)]
    for lc in (True, False):
        cases.append(list_case(f"small_vocab_list_lc{int(lc)}", hyps, refs, lc))
    # three references per sentence (stem0..2), of different line counts; more hypotheses than references
    h = [sentence(rng, small, 0, 10) for _ in range(25)]
    r3 = [[sentence(rng, small, 0, 10) for _ in range(n)] for n in (25, 20, 12)]
    for lc in (True, False):
        cases.append(file_case(f"three_refs_lc{int(lc)}", lines(h), [(str(i), lines(r)) for i, r in enumerate(r3)], lc))
    cases.append(file_case("stem_and_numbered", lines(h), [("0", lines(r3[0])), ("1", lines(r3[1])), ("", lines(r3[2]))]))
    cases.append(file_case("dot_ref_names", lines(h), [(".ref0", lines(r3[0])), (".ref1", lines(r3[2]))]))
    cases.append(list_case("more_hyps_than_refs", h, r3[1][:7]))
    # one reference: a larger random corpus with mixed case
    vocab = [w + s for w in ("x", "Y", "zz", "Quo", "w") for s in ("", "1", "2", "E")]
    hyps = [sentence(rng, vocab, 0, 30) for _ in range(200)]
    refs = [sentence(rng, vocab, 0, 30) for _ in range(200)]
    for lc in (True, False):
        cases.append(list_case(f"random_mixed_case_lc{int(lc)}", hyps, refs, lc))
    # empty lines and runs of every ASCII whitespace byte; an unterminated last line loses its last byte to chop
    def ws_sentence():
        words = [rng.choice(small) for _ in range(rng.randint(0, 8))]
        return "".join(rng.choice(["", " "]) + w + "".join(rng.choice(WS[:2] + WS[3:]) for _ in range(rng.randint(1, 3)))
                       for w in words)
    hyps = [ws_sentence() for _ in range(20)] + ["", "   ", "a\tb\x0bc\x0cd\re"]
    refs = [ws_sentence() for _ in range(20)] + ["", "a", "a b c d e"]
    cases.append(list_case("whitespace_runs_list", hyps, refs))
    cases.append(list_case("hyp_with_newline_inside", ["a b\nc d", "c d e", "a"], ["a b", "c d", "c d e"]))
    hb = lines(["a b c", "", "b\t\tc  a", "a b\r", "c a b cc"], terminated=False)
    rb = lines(["a b c", "b c", "b c a", "a b", "c a b c"], terminated=False)
    for lc in (True, False):
        cases.append(file_case(f"unterminated_last_lines_lc{int(lc)}", hb, [("", rb)], lc))
    cases.append(file_case("crlf_lines", b"A B C\r\nd e\r\nF\r\n", [("", b"a b c\r\nD E\r\nf g\r\n")]))
    # ASCII capitals next to UTF-8 umlauts, Latin-1 bytes, NBSP and NEL, which neither lc nor split touch
    hyps = ["Über ÄPFEL und Äpfel", "DAS Haus IST grün", "Straße STRASSE straße", "nbsp word nbsp word", "ÀB àb AB ab"]
    refs = ["über äpfel und äpfel", "das haus ist grün", "straße strasse straße", "nbsp word nbsp word", "àb àb ab ab"]
    for lc in (True, False):
        cases.append(list_case(f"utf8_capitals_lc{int(lc)}", hyps, refs, lc))
    hb = b"\xc4PFEL \xe4pfel APFEL\nNBSP\xa0JOIN nbsp join\nNEL\x85JOIN nel\x85join X\nMIX\xc3\x84 mix\xc3\xa4\n"
    rb = b"\xe4pfel \xe4pfel apfel\nnbsp\xa0join nbsp join\nnel\x85join nel\x85join x\nmix\xc3\x84 mix\xc3\xa4\n"
    for lc in (True, False):
        cases.append(file_case(f"latin1_nbsp_nel_lc{int(lc)}", hb, [("", rb)], lc))
    # long lines: 2,000 tokens, one token repeated, and a corpus without 4-grams
    long_h = sentence(rng, ["p", "q", "r", "s", "t", "u"], 2000, 2000)
    long_r = sentence(rng, ["p", "q", "r", "s", "t", "u"], 1990, 1990)
    cases.append(list_case("long_line_2000", [long_h, "p q", "the the the"], [long_r, "p q r", " ".join(["the"] * 300)]))
    cases.append(list_case("one_token_repeated", [" ".join(["the"] * 500), " ".join(["a"] * 7)],
                           [" ".join(["the"] * 120), " ".join(["a"] * 9)]))
    cases.append(list_case("no_four_grams", ["a b", "c", "a b c", ""], ["a b c d", "c", "a b", "x y"]))
    # degenerate totals: every reference empty (ref_len 0), every hypothesis empty (hyp_len 0), no reference line
    cases.append(list_case("ref_len_zero", ["a b", "c"], ["", ""]))
    cases.append(list_case("ref_len_zero_no_hyps", [], ["", ""]))
    cases.append(list_case("hyp_len_zero", ["", "  ", ""], ["a b", "c", ""]))
    cases.append(list_case("hyp_len_zero_no_refs_left", ["", ""], ["a"]))
    cases.append(list_case("no_reference_lines", ["a b"], []))
    cases.append(list_case("perfect", ["the cat sat on the mat", "a b c d e"], ["the cat sat on the mat", "a b c d e"]))
    cases.append(list_case("nothing_matches", ["a b c d"], ["e f g h"]))
    with open(OUT, "w") as f:
        json.dump({"script": "perl_scripts/multi-bleu.perl", "cases": cases}, f, indent=0, ensure_ascii=True)
    print(f"wrote {len(cases)} cases to {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main()
