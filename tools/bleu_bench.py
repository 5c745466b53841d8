"""Times the GPU BLEU path against the host path it replaces.

(a) qd_bleu_stats + qd_bleu_fold at N = 3,000 and 100,000 sentences of about 25 words (one reference each), against
    the plain-Python oracle (oracle/bleu_oracle.py) on the host;
(b) per translated batch, B in {1, 30, 64}, K = 5, on the NMT-shaped model of tools/beam_bench.py (V = 50,004):
    BatchBeam.finish() against BatchBeam.finish_on_device() on the same finished search;
(c) sentences/s of bleu_model against beam_search + finish() + buildTargetTokens strings + the oracle's multi-bleu.

The card name, power limit and SM clock are read in the same run.  Without a CUDA device it refuses, except
`--perl SCRIPT`, which only times `perl SCRIPT -lc` on the (a) corpora on the host (perl is not on the GPU machines).

    python tools/bleu_bench.py [--out profiles/bleu_bench.json] [--quick]
    python tools/bleu_bench.py --perl path/to/multi-bleu.perl
"""
import argparse
import importlib.util
import json
import os
import random
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import bleu_oracle as O  # noqa: E402

VOCAB_WORDS = 5_000


def _beam_bench():
    spec = importlib.util.spec_from_file_location("beam_bench", os.path.join(ROOT, "tools", "beam_bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def corpus(n, seed=0):
    """n hypothesis and reference lines of 15-35 words over a Zipf-like vocabulary."""
    g = random.Random(seed)
    words = [f"w{i}" for i in range(VOCAB_WORDS)]
    weights = [1.0 / (i + 1) for i in range(VOCAB_WORDS)]

    def line():
        return " ".join(g.choices(words, weights, k=g.randint(15, 35)))
    return [line() for _ in range(n)], [line() for _ in range(n)]


def bench_stats(n, iters):
    import torch
    from quantized_distillation_b200 import bleu
    from quantized_distillation_b200 import _native as N
    hyps, refs = corpus(n)
    R = bleu.References(refs)
    st = bleu.BleuStats(R)
    st.add(hyps)
    words, offsets = [], [0]
    for h in hyps:
        words += R.table.intern(bleu.perl_words(h.encode()))
        offsets.append(len(words))
    hw = torch.tensor(words, dtype=torch.int32, device="cuda")
    ho = torch.tensor(offsets, dtype=torch.int64, device="cuda")
    rows = torch.empty(n, 10, dtype=torch.int64, device="cuda")
    tot = torch.empty(10, dtype=torch.int64, device="cuda")

    def run():
        N.check(N.lib().qd_bleu_stats(N.ptr(hw), hw.numel(), N.ptr(ho), n, N.ptr(R.words), R.words.numel(), N.ptr(R.offsets),
                                      R.offsets.numel() - 1, N.ptr(R.first), N.ptr(R.count), N.ptr(rows), N.stream_ptr()))
        N.check(N.lib().qd_bleu_fold(N.ptr(rows), n, N.ptr(tot), N.stream_ptr()))
    for _ in range(3):
        run()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        run()
    e1.record()
    torch.cuda.synchronize()
    gpu_ms = e0.elapsed_time(e1) / iters
    t0 = time.perf_counter()
    want = O.multi_bleu("".join(h + "\n" for h in hyps).encode(), ["".join(r + "\n" for r in refs).encode()], True)[0]
    host_ms = (time.perf_counter() - t0) * 1e3
    assert bleu.format_line(tot.tolist()) == want, "GPU totals differ from the oracle"
    words_total = len(words) + R.words.numel()
    return {"sentences": n, "words": words_total, "gpu_stats_fold_ms": gpu_ms, "oracle_host_ms": host_ms,
            "line": want.decode().strip()}


def bench_finish(model, B, K, iters, bb_mod, max_len=100):
    import torch
    from quantized_distillation_b200.beam import _search
    g = torch.Generator().manual_seed(B)
    src = torch.randint(4, model.generator[0].out_features, (bb_mod.SRC_LEN, B), generator=g).cuda()
    lengths = torch.full((B,), bb_mod.SRC_LEN)
    with torch.no_grad():
        beam = _search(model, src, lengths, K, 1, max_len, bb_mod.BOS, bb_mod.EOS, bb_mod.PAD, None)
    res = {"B": B, "K": K, "steps": beam.steps}
    for name, fn in (("finish_host", beam.finish), ("finish_on_device", beam.finish_on_device)):
        fn()
        torch.cuda.synchronize()
        times = []
        for _ in range(iters):
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times.append((time.perf_counter() - t0) * 1e3)
        times.sort()
        res[name + "_ms_median"] = times[len(times) // 2]
    return res


def bench_end_to_end(model, V, sentences, batch, bb_mod, max_len=100):
    import torch
    from quantized_distillation_b200 import bleu
    from quantized_distillation_b200.beam import beam_search
    specials = ["<unk>", "<blank>", "<s>", "</s>"]
    itos = specials + [f"w{i}" for i in range(4, V)]
    g = torch.Generator().manual_seed(7)
    src_all = torch.randint(4, V, (bb_mod.SRC_LEN, sentences), generator=g).cuda()
    lengths = torch.full((sentences,), bb_mod.SRC_LEN)
    rg = random.Random(5)
    refs = [" ".join(rg.choice(itos[4:200]) for _ in range(rg.randint(3, 12))) for _ in range(sentences)]
    batches = [(src_all[:, a:a + batch], lengths[a:a + batch]) for a in range(0, sentences, batch)]
    kw = dict(bos=bb_mod.BOS, eos=bb_mod.EOS, pad=bb_mod.PAD)

    R = bleu.References(refs)                        # uploaded once, as a test set's references are

    def device_path():
        return bleu.bleu_model(model, batches, R, src_vocab=itos, tgt_vocab=itos, replace_unk=True, beam_size=5,
                               max_sent_length=max_len, unk=0, **kw)

    def host_path():
        lines = []
        for src, ln in batches:
            hyps, _, attn = beam_search(model, src, ln, 5, 1, max_len, **kw)
            for b in range(src.shape[1]):
                toks = []
                for t in hyps[b][0]:
                    toks.append(itos[t])
                    if toks[-1] == "</s>":
                        toks = toks[:-1]
                        break
                for i in range(len(toks)):
                    if toks[i] == "<unk>":
                        toks[i] = itos[int(src[int(attn[b][0][i].max(0)[1]), b])]
                lines.append(" ".join(toks))
        return O.multi_bleu("".join(s + "\n" for s in lines).encode(), ["".join(r + "\n" for r in refs).encode()], True)[0]

    res = {"sentences": sentences, "batch": batch}
    outs = {}
    for name, fn in (("bleu_model", device_path), ("beam_search_finish_strings_oracle", host_path)):
        fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        outs[name] = fn()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        res[name] = {"seconds": dt, "sentences_per_s": sentences / dt}
    res["same_line"] = outs["bleu_model"] == outs["beam_search_finish_strings_oracle"]
    res["line"] = outs["bleu_model"].decode().strip()
    return res


def bench_perl(script, sizes):
    res = []
    for n in sizes:
        hyps, refs = corpus(n)
        with tempfile.TemporaryDirectory() as d:
            ref = os.path.join(d, "ref")
            with open(ref, "w") as f:
                f.write("".join(r + "\n" for r in refs))
            stdin = "\n".join(hyps).encode()
            t0 = time.perf_counter()
            out = subprocess.run(["perl", script, "-lc", ref], input=stdin, capture_output=True).stdout
            dt = time.perf_counter() - t0
        t0 = time.perf_counter()
        want = O.multi_bleu(stdin, ["".join(r + "\n" for r in refs).encode()], True)[0]
        res.append({"sentences": n, "perl_ms": dt * 1e3, "oracle_ms": (time.perf_counter() - t0) * 1e3,
                    "same_line": out == want})
        print(json.dumps(res[-1]), flush=True)
    return res


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "bleu_bench.json"))
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--quick", action="store_true", help="small shapes, for a rehearsal")
    ap.add_argument("--perl", metavar="SCRIPT", help="only time perl SCRIPT -lc on the (a) corpora (host, no GPU)")
    args = ap.parse_args(argv)
    sizes = [300, 1_000] if args.quick else [3_000, 100_000]
    if args.perl:
        bench_perl(args.perl, sizes)
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bleu_bench needs a CUDA device: there is nothing to time without one")
    bb = _beam_bench()
    card = bb._card()
    print(json.dumps(card), flush=True)
    out = {"card": card, "stats": [], "finish": [], "end_to_end": {}}
    print("(a) statistics: N, words, GPU stats+fold ms, oracle host ms")
    for n in sizes:
        r = bench_stats(n, args.iters)
        out["stats"].append(r)
        print(f"  {r['sentences']:7d} {r['words']:9d}  {r['gpu_stats_fold_ms']:9.3f}  {r['oracle_host_ms']:10.1f}", flush=True)
    V = 1_004 if args.quick else 50_004
    with torch.no_grad():
        model = bb._model(V, 0)
    print("(b) finish per batch: B, K, steps, finish() ms, finish_on_device() ms")
    for B in ([1, 4] if args.quick else [1, 30, 64]):
        r = bench_finish(model, B, 5, args.iters, bb)
        out["finish"].append(r)
        print(f"  {B:3d} {r['K']:2d} {r['steps']:4d}  {r['finish_host_ms_median']:9.3f}  {r['finish_on_device_ms_median']:9.3f}",
              flush=True)
    print("(c) end to end, sentences/s")
    for packed in (False, True):
        m = model
        if packed:
            from quantized_distillation_b200 import codec
            pm = codec.pack_model(model, 4, 256, quantize_first_and_last_layer=True)
            m = bb._model(V, 1)
            codec.attach_packed_(pm, m, embeddings=True, recurrent=True)
            m.eval()
        r = bench_end_to_end(m, V, 8 if args.quick else 60, 4 if args.quick else 30, bb)
        out["end_to_end"]["packed" if packed else "float32"] = r
        print(f"  {'packed ' if packed else 'float32'} bleu_model {r['bleu_model']['sentences_per_s']:.2f}, host path "
              f"{r['beam_search_finish_strings_oracle']['sentences_per_s']:.2f} (same line: {r['same_line']})", flush=True)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(out, f, indent=1)
    print(f"wrote {args.out}")


if __name__ == "__main__":
    main()
