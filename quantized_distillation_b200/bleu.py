"""Corpus BLEU on the GPU, identical to the moses multi-bleu.perl the reference runs (perl_scripts/multi-bleu.perl,
translation_models/help_fun.py:313-381), with no file and no perl.

Words are interned to int32 ids on the host, following perl on bytes: lines end at \\n and `chop` drops each line's last
byte whatever it is; -lc lowercases ASCII A-Z only; split cuts on space, \\t, \\n, \\r, \\v and \\f only (not on NBSP or
NEL).  qd_bleu_stats computes each sentence's 10 integers on the device and qd_bleu_fold sums them; format_line prints
multi-bleu's line from the 10 corpus totals in float64 on the host.

    References(refs, lowercase=True, device=None)       a test set's references, uploaded once
    BleuStats(references)                               per-sentence statistics, filled batch by batch
    format_line(totals) -> bytes                        multi-bleu's stdout for the 10 totals
    corpus_bleu(hypotheses, references, lowercase=True) -> float
    get_bleu_moses(hypotheses, reference, file_input=False, path_to_multi_bleu_moses=None) -> bytes   (drop-in)
    bleu_model(model, batches, references, *, src_vocab, tgt_vocab, ...) -> bytes                      (drop-in)

There is no CPU implementation: without a CUDA device the statistics raise RuntimeError.
"""
from __future__ import annotations

import gzip
import math
import os
import re

import torch

from . import _native as N

_LOWER = bytes.maketrans(b"ABCDEFGHIJKLMNOPQRSTUVWXYZ", b"abcdefghijklmnopqrstuvwxyz")
ZERO_LINE = b"BLEU = 0, 0/0/0/0 (BP=0, ratio=0, hyp_len=0, ref_len=0)\n"


def perl_lines(data: bytes) -> list:
    """`while (<FH>) { chop; ... }` on bytes: one line per \\n, plus an unterminated last line; chop drops each line's
    last byte (the \\n, or the last byte of an unterminated line)."""
    parts = data.split(b"\n")
    lines = parts[:-1]
    if parts[-1]:
        lines.append(parts[-1][:-1])
    return lines


def perl_words(line: bytes, lowercase: bool = True) -> list:
    """`lc` (ASCII A-Z only on a byte string) and `split` (ASCII whitespace only: bytes.split() cuts on the same six
    bytes as perl's split ' ')."""
    return (line.translate(_LOWER) if lowercase else line).split()


def _as_bytes(s) -> bytes:
    return s if isinstance(s, bytes) else s.encode()


class WordTable:
    """Interns words (bytes) to int32 ids, in first-seen order."""

    def __init__(self):
        self.ids = {}

    def __len__(self):
        return len(self.ids)

    def intern(self, words) -> list:
        ids = self.ids
        return [ids.setdefault(w, len(ids)) for w in words]


def _device(device):
    N.require_cuda()
    dev = torch.device(device if device is not None else "cuda")
    if dev.type != "cuda":
        raise ValueError("the BLEU statistics live on a CUDA device")
    return torch.device("cuda", torch.cuda.current_device()) if dev.index is None else dev


class References:
    """A test set's references as word ids on the device: words [n_words] int32, offsets [n_refs+1] int64 and, per
    sentence, its first reference (first [n]) and count (count [n]).  refs[s] is one reference line (str or bytes) or
    a sequence of them (0 or more).  Each line is split as perl splits a line it has read (no chop: the line has no
    \\n), lowercased when `lowercase`."""

    def __init__(self, refs, lowercase=True, device=None, table: WordTable | None = None):
        self.device = _device(device)
        self.lowercase = bool(lowercase)
        self.table = table if table is not None else WordTable()
        per_sentence = [[r] if isinstance(r, (str, bytes)) else list(r) for r in refs]
        self._upload([[perl_words(_as_bytes(r), self.lowercase) for r in rs] for rs in per_sentence])

    @classmethod
    def from_words(cls, word_lists, lowercase, device, table):
        """References already split into words: word_lists[s] is a list of word lists (bytes words)."""
        self = cls.__new__(cls)
        self.device, self.lowercase, self.table = _device(device), lowercase, table
        self._upload(word_lists)
        return self

    def _upload(self, word_lists):
        words, offsets, first, count = [], [0], [], []
        for rs in word_lists:
            first.append(len(offsets) - 1)
            count.append(len(rs))
            for r in rs:
                words.extend(self.table.intern(r))
                offsets.append(len(words))
        dev = self.device
        self.n = len(word_lists)
        self.words = torch.tensor(words, dtype=torch.int32).to(dev)
        self.offsets = torch.tensor(offsets, dtype=torch.int64).to(dev)
        self.first = torch.tensor(first, dtype=torch.int64).to(dev)
        self.count = torch.tensor(count, dtype=torch.int64).to(dev)
        self._vocab_tables = {}

    def __len__(self):
        return self.n

    def vocab_tables(self, src_itos, tgt_itos, eos, unk):
        """(src word ids, tgt word ids, tgt is-EOS, tgt is-UNK) on the device for a vocabulary pair, built once per
        pair and kept with these references (their word table interns the words).  buildTargetTokens compares words,
        so every index whose entry is the EOS (UNK) entry's string counts as EOS (UNK)."""
        key = (tuple(src_itos), tuple(tgt_itos), eos, unk)
        t = self._vocab_tables.get(key)
        if t is None:
            dev = self.device
            eos_word, unk_word = tgt_itos[eos], tgt_itos[unk]
            t = (_vocab_table(src_itos, self.table, self.lowercase, dev), _vocab_table(tgt_itos, self.table, self.lowercase, dev),
                 torch.tensor([w == eos_word for w in tgt_itos], dtype=torch.bool).to(dev),
                 torch.tensor([w == unk_word for w in tgt_itos], dtype=torch.bool).to(dev))
            self._vocab_tables[key] = t
        return t


class BleuStats:
    """Per-sentence multi-bleu statistics [n, 10] int64 on the device, against `references`.  add() writes the rows of
    a batch of hypotheses at their sentence indices; a sentence never added counts nothing, as a line perl never
    read.  totals() folds the rows into the 10 corpus integers (one device-to-host read)."""

    def __init__(self, references: References):
        self.references = references
        self.stats = torch.zeros(len(references), N.BLEU_STATS, dtype=torch.int64, device=references.device)

    def add_words(self, words: torch.Tensor, offsets: torch.Tensor, indices: torch.Tensor) -> torch.Tensor:
        """Hypotheses as device word ids in CSR form (words int32, offsets int64 [b+1]) for the sentences `indices`
        (int64 [b], distinct, in range).  Returns their rows [b, 10]; no host synchronisation."""
        R, dev = self.references, self.references.device
        b = int(indices.numel())
        if words.dtype != torch.int32 or offsets.dtype != torch.int64 or offsets.numel() != b + 1:
            raise ValueError("words must be int32 and offsets int64 [len(indices) + 1]")
        if words.device != dev or offsets.device != dev or indices.device != dev:
            raise ValueError(f"words, offsets and indices must be on {dev}")
        words, offsets = words.contiguous(), offsets.contiguous()
        first, count = R.first.index_select(0, indices), R.count.index_select(0, indices)
        rows = torch.empty(b, N.BLEU_STATS, dtype=torch.int64, device=dev)
        with torch.cuda.device(dev):
            N.check(N.lib().qd_bleu_stats(N.ptr(words), words.numel(), N.ptr(offsets), b, N.ptr(R.words), R.words.numel(),
                                          N.ptr(R.offsets), R.offsets.numel() - 1, N.ptr(first), N.ptr(count), N.ptr(rows),
                                          N.stream_ptr(dev)))
        self.stats.index_copy_(0, indices, rows)
        return rows

    def add(self, hypotheses, indices=None) -> torch.Tensor:
        """Hypothesis lines (str or bytes, split as perl splits a line it has read) for the sentences `indices`
        (default 0 .. len-1)."""
        R = self.references
        words, offsets = [], [0]
        for h in hypotheses:
            words.extend(R.table.intern(perl_words(_as_bytes(h), R.lowercase)))
            offsets.append(len(words))
        if indices is None:
            indices = range(len(offsets) - 1)
        dev = R.device
        return self.add_words(torch.tensor(words, dtype=torch.int32).to(dev), torch.tensor(offsets, dtype=torch.int64).to(dev),
                              torch.as_tensor(list(indices), dtype=torch.int64).to(dev))

    def totals_device(self) -> torch.Tensor:
        out = torch.empty(N.BLEU_STATS, dtype=torch.int64, device=self.stats.device)
        with torch.cuda.device(self.stats.device):
            N.check(N.lib().qd_bleu_fold(N.ptr(self.stats), self.stats.shape[0], N.ptr(out), N.stream_ptr(self.stats.device)))
        return out

    def totals(self) -> list:
        """[hyp_len, ref_len, correct1..4, total1..4] of the corpus."""
        return self.totals_device().tolist()

    def score(self) -> float:
        """The BLEU value multi-bleu prints (in percent, before rounding); 0.0 where it prints no score."""
        return bleu_value(self.totals())


def _my_log(x):
    return -9999999999 if not x else math.log(x)


def _terms(totals):
    """(bleu, precisions, brevity penalty) in float64, as multi-bleu.perl:125-153 computes them; None when perl dies
    (hyp_len 0 against ref_len > 0: division by zero)."""
    hyp_len, ref_len = int(totals[0]), int(totals[1])
    prec = [totals[2 + n] / totals[6 + n] if totals[6 + n] else 0 for n in range(4)]
    bp = 1
    if hyp_len < ref_len:
        if hyp_len == 0:
            return None
        bp = math.exp(1 - ref_len / hyp_len)
    logs = _my_log(prec[0]) + _my_log(prec[1])
    logs = logs + _my_log(prec[2])
    logs = logs + _my_log(prec[3])
    return bp * math.exp(logs / 4), prec, bp


def format_line(totals) -> bytes:
    """multi-bleu.perl's stdout for the 10 corpus totals: its `BLEU = ...` line, its zero line when ref_len is 0, and
    b"" where perl dies (hyp_len 0 against ref_len > 0)."""
    hyp_len, ref_len = int(totals[0]), int(totals[1])
    if ref_len == 0:
        return ZERO_LINE
    t = _terms(totals)
    if t is None:
        return b""
    bleu, prec, bp = t
    return ("BLEU = %.2f, %.1f/%.1f/%.1f/%.1f (BP=%.3f, ratio=%.3f, hyp_len=%d, ref_len=%d)\n" % (
        100 * bleu, 100 * prec[0], 100 * prec[1], 100 * prec[2], 100 * prec[3], bp, hyp_len / ref_len, hyp_len,
        ref_len)).encode()


def bleu_value(totals) -> float:
    if int(totals[1]) == 0:
        return 0.0
    t = _terms(totals)
    return 0.0 if t is None else 100 * t[0]


def corpus_bleu(hypotheses, references, lowercase=True, device=None) -> float:
    """BLEU of hypothesis lines against references (as References takes them), one per sentence."""
    if len(hypotheses) != len(references):
        raise ValueError(f"{len(hypotheses)} hypotheses for {len(references)} sentences of references")
    stats = BleuStats(References(references, lowercase, device))
    stats.add(hypotheses)
    return stats.score()


def multi_bleu(stdin: bytes, ref_files, lowercase=True, device=None) -> bytes:
    """The stdout of `perl multi-bleu.perl [-lc] stem < stdin`, where ref_files are the contents (bytes) of the files
    perl reads for the stem, in its order.  With no reference line at all perl dies: b""."""
    table = WordTable()
    refs = []
    for data in ref_files:
        for s, line in enumerate(perl_lines(data)):
            if s == len(refs):
                refs.append([])
            refs[s].append(perl_words(line, lowercase))
    if not refs:
        return b""
    hyps = [perl_words(line, lowercase) for line in perl_lines(stdin)]
    refs += [[] for _ in range(len(hyps) - len(refs))]          # lines past the references: no reference
    R = References.from_words(refs, lowercase, device, table)
    stats = BleuStats(R)
    words, offsets = [], [0]
    for h in hyps:
        words.extend(table.intern(h))
        offsets.append(len(words))
    dev = R.device
    stats.add_words(torch.tensor(words, dtype=torch.int32).to(dev), torch.tensor(offsets, dtype=torch.int64).to(dev),
                    torch.arange(len(hyps), dtype=torch.int64).to(dev))
    return format_line(stats.totals())


def reference_files(stem: str) -> list:
    """The contents of the files multi-bleu.perl reads for `stem` (multi-bleu.perl:23-33): stem0, stem1, ... then
    stem itself, or stem.ref0, ... when neither stem nor stem0 exists; a name ending like .gz is decompressed."""
    if not os.path.exists(stem) and not os.path.exists(stem + "0") and os.path.exists(stem + ".ref0"):
        stem += ".ref"
    names, i = [], 0
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


def get_bleu_moses(hypotheses, reference, file_input=False, path_to_multi_bleu_moses=None) -> bytes:
    """Drop-in for the reference's get_bleu_moses (help_fun.py:313-352): the bytes perl would print with -lc.  List
    mode: hypotheses and reference are lists of str; the hypotheses are joined by \\n with no trailing newline (so the
    last one loses its last character to chop) and each reference line ends on \\n.  File mode: hypotheses is a file
    path and reference a stem, found as perl finds it.  path_to_multi_bleu_moses is accepted and not used."""
    if file_input:
        with open(hypotheses, "rb") as f:
            stdin = f.read()
        refs = reference_files(reference)
    else:
        stdin = "\n".join(hypotheses).encode()
        refs = ["".join(r + "\n" for r in reference).encode()]
    return multi_bleu(stdin, refs, True)


# ---- translation ---------------------------------------------------------------------------------------------------

def _itos(vocab):
    return vocab.itos if hasattr(vocab, "itos") else vocab


def _vocab_table(itos, table: WordTable, lowercase: bool, device) -> torch.Tensor:
    """Word id of every vocabulary entry, as perl reads the entry in a translation line: it must be one word."""
    ids = []
    for w in itos:
        words = perl_words(_as_bytes(w), lowercase)
        if len(words) != 1:
            raise ValueError(f"vocabulary entry {w!r} is not one word once written and split; it cannot be scored "
                             "word by word")
        ids.extend(table.intern(words))
    return torch.tensor(ids, dtype=torch.int32).to(device)


@torch.no_grad()
def bleu_model(model, batches, references, *, src_vocab, tgt_vocab, replace_unk=True, beam_size=5, max_sent_length=100,
               bos, eos, pad, unk) -> bytes:
    """Analogue of the reference's get_bleu_model (help_fun.py:366-381): translate every batch with the batched beam
    search (n_best 1, the drivers' setting), build each sentence's words as Translator.buildTargetTokens does
    (Translator.py:43-60: tgt_itos[token], cut at the first EOS, and with replace_unk an UNK word becomes
    src_itos[src[argmax of its attention row]]), and score them against `references` with -lc.  Returns multi-bleu's
    stdout bytes.

    batches yields (src [S, B], src_lengths) or (src, src_lengths, indices): the test-set index of each column
    (default: consecutive from 0).  references: a References (lowercase) or what References takes.  src_vocab,
    tgt_vocab: itos lists or vocabularies with .itos.  Everything from the search to the statistics stays on the
    device; the 10 totals are read once, after the last batch.  Pass a References to reuse its upload and the
    vocabulary tables it keeps across calls."""
    from .beam import beam_search_on_device
    if not isinstance(references, References):
        references = References(references, True)
    if not references.lowercase:
        raise ValueError("get_bleu_model scores with -lc: the references must be lowercased")
    dev = references.device
    src_itos, tgt_itos = _itos(src_vocab), _itos(tgt_vocab)
    src_ids, tgt_ids, is_eos, is_unk = references.vocab_tables(src_itos, tgt_itos, eos, unk)
    V = getattr(model.generator[0], "out_features", None)
    if V is not None and V > len(tgt_itos):
        raise ValueError(f"the generator has {V} outputs and the target vocabulary {len(tgt_itos)} entries")
    stats = BleuStats(references)
    start = 0
    for batch in batches:
        src, lengths = batch[0], batch[1]
        B = int(src.shape[1])
        idx = (torch.as_tensor(batch[2], dtype=torch.int64) if len(batch) > 2 else torch.arange(start, start + B)).to(dev)
        start += B
        hyp = beam_search_on_device(model, src, lengths, beam_size, 1, max_sent_length, bos=bos, eos=eos, pad=pad)
        T = hyp.tokens.shape[2]
        tok = hyp.tokens[:, 0].clamp(min=0)                                         # [B, T]; -1 past the length
        pos = torch.arange(T, device=dev)
        valid = pos < hyp.lengths[:, 0:1]
        stop = valid & is_eos[tok]
        cut = torch.where(stop.any(1), stop.int().argmax(1), hyp.lengths[:, 0])     # tokens before the first EOS
        keep = pos < cut[:, None]
        words = tgt_ids[tok]
        if replace_unk and T:
            s_tok = src if src.dim() == 2 else src[:, :, 0]                           # the word feature
            arg = hyp.attn_argmax[:, 0].clamp(min=0)
            from_src = src_ids[s_tok.to(dev).t().gather(1, arg)]
            words = torch.where(is_unk[tok], from_src, words)
        lens = keep.sum(1)
        offsets = torch.zeros(B + 1, dtype=torch.int64, device=dev)
        torch.cumsum(lens, 0, out=offsets[1:])
        # compact the kept words without a host read: every dropped position goes to one spare slot past the end
        dest = torch.where(keep, offsets[:-1, None] + pos, B * T)
        flat = torch.empty(B * T + 1, dtype=torch.int32, device=dev)
        flat.scatter_(0, dest.reshape(-1), words.reshape(-1))
        stats.add_words(flat, offsets, idx)
    return format_line(stats.totals())
