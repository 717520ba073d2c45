"""stb_embed_text against host tokenisation + stb_embed: python scripts/embed_text_probe.py [lines] [reps]

Workload: `lines` (default 1M) printable-ASCII lines from a seeded word model (Zipf over 20k random words,
lognormal words per line) and a tokenizer.json of the reference model's shape -- a 30k-piece Unigram trained by
sentencepiece on text from the same word model, the nmt_nfkc charsmap, Replace(" {2,}"), Metaspace.
Paths, each timed with a host clock around calls that end in a synchronise, after a warm-up call, all appending
the rows to a corpus in HBM (as ingestion does):
  gpu_text  stb_embed_text (the rule, the GPU tokenizer, K3)
  hf        HF tokenizers encode_batch (all cores) + stb_embed
  cpp       the C++ host tokenizer (HfTokenizer::encode on all cores) + K3, the C++ host's path before
            stb_embed_text: stb_embed_text with the same tokenizer plus a string Replace that never matches, a shape
            the GPU does not take, so every line goes through the library's host half (the same HfTokenizer threads,
            one more normaliser pass per line)
  cpp_bench the C++ CLI's own tokenisation benchmark (semtools_b200_search --tokenize-bench) with the same
            tokenizer on its synthetic lines, when the CLI is built: the tokenizer alone, for scale
Also: per-kernel times of one gpu_text call from torch.profiler, the card's name and power limit.  Rows of the
three paths must be bit-identical.  Writes its JSON lines to stdout only.
"""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from semtools_b200 import capi  # noqa: E402


def word_model(rng, n_words=20000):
    letters = np.array(list("abcdefghijklmnopqrstuvwxyz"))
    lens = np.clip(rng.poisson(5, n_words), 1, 14)
    words = ["".join(rng.choice(letters, l)) for l in lens]
    p = 1.0 / np.arange(1, n_words + 1) ** 1.05
    return words, p / p.sum()


def make_lines(rng, words, p, n):
    k = np.clip(np.round(rng.lognormal(2.53, 0.6, n)), 1, 200).astype(np.int64)
    w = rng.choice(len(words), int(k.sum()), p=p)
    out, at = [], 0
    for c in k:
        line = " ".join(words[j] for j in w[at:at + c])
        out.append(line.capitalize() if c % 3 == 0 else line + ".")
        at += c
    return out


def build_tokenizer(d, rng, words, p):
    import sentencepiece as spm
    from sentencepiece import sentencepiece_model_pb2 as pb
    from tokenizers import Regex, Tokenizer
    from tokenizers.models import Unigram
    from tokenizers.normalizers import Precompiled, Replace, Sequence
    from tokenizers.pre_tokenizers import Metaspace
    with open(os.path.join(d, "corpus.txt"), "w") as f:
        f.write("\n".join(make_lines(rng, words, p, 300000)) + "\n")
    spm.SentencePieceTrainer.train(input=os.path.join(d, "corpus.txt"), model_prefix=os.path.join(d, "m"), vocab_size=30000,
                                   model_type="unigram", normalization_rule_name="nmt_nfkc", character_coverage=1.0,
                                   hard_vocab_limit=False, minloglevel=2, num_threads=os.cpu_count())
    mp = pb.ModelProto()
    mp.ParseFromString(open(os.path.join(d, "m.model"), "rb").read())
    tk = Tokenizer(Unigram([(x.piece, x.score) for x in mp.pieces], unk_id=next(i for i, x in enumerate(mp.pieces) if x.type == 2),
                           byte_fallback=False))
    tk.normalizer = Sequence([Precompiled(mp.normalizer_spec.precompiled_charsmap), Replace(Regex(" {2,}"), " ")])
    tk.pre_tokenizer = Metaspace(replacement="▁", prepend_scheme="always")
    gpu_json = tk.to_str().encode()
    tk.normalizer = Sequence([Precompiled(mp.normalizer_spec.precompiled_charsmap), Replace(Regex(" {2,}"), " "),
                              Replace("\x01\x02", "")])
    host_json = tk.to_str().encode()
    tk.normalizer = Sequence([Precompiled(mp.normalizer_spec.precompiled_charsmap), Replace(Regex(" {2,}"), " ")])
    return tk, gpu_json, host_json


def timed(fn, reps):
    fn()                                                       # warm-up: modules, scratch growth
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = fn()
        ts.append(time.perf_counter() - t0)
    return min(ts), float(np.median(ts)), r


def main():
    n_lines = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    import torch
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    rng = np.random.default_rng(2024)
    words, p = word_model(rng)
    cpp_bench = None
    with tempfile.TemporaryDirectory() as d:
        t0 = time.perf_counter()
        tk, gpu_json, host_json = build_tokenizer(d, rng, words, p)
        train_s = time.perf_counter() - t0
        cli = os.path.join(os.path.dirname(capi.LIB_PATH), "semtools_b200_search")
        if os.path.exists(cli):
            with open(os.path.join(d, "tok.json"), "wb") as f:
                f.write(gpu_json)
            r = subprocess.run([cli, "--tokenize-bench", "1000000", str(os.cpu_count()), os.path.join(d, "tok.json")],
                               capture_output=True, text=True)
            cpp_bench = [json.loads(x) for x in r.stdout.split("\n") if x.startswith("{")]
    lines = make_lines(rng, words, p, n_lines)
    dev = torch.device("cuda:0")
    s = torch.cuda.Stream(dev)
    torch.cuda.set_stream(s)
    ctx = capi.Context(0, s.cuda_stream)
    V = tk.get_vocab_size()
    table = capi.Table(ctx, (rng.standard_normal((V, 256), dtype=np.float32) * np.float32(0.1)))
    gtok, htok = capi.Tokenizer(ctx, gpu_json), capi.Tokenizer(ctx, host_json)
    taken = gtok.gpu_lines(lines)
    assert taken.all() and not htok.gpu_lines(lines[:100]).any()

    def hf_path():
        encs = tk.encode_batch(lines, add_special_tokens=False)
        ids = [e.ids[:2048] for e in encs]
        off = np.zeros(len(ids) + 1, dtype=np.uint64)
        off[1:] = np.cumsum([len(x) for x in ids])
        corpus.clear()
        capi.embed(ctx, table, off, np.fromiter((i for x in ids for i in x), dtype=np.uint32, count=int(off[-1])), out=False,
                   append_to=corpus)
        return int(off[-1])

    text, offsets = capi.pack_lines(lines)                    # packed once: the calls below time the library

    corpus = capi.Corpus(ctx, n_lines)

    def text_path(tok):                                       # rows into the corpus in HBM, as ingestion does
        corpus.clear()
        capi._check(capi.lib().stb_embed_text(ctx._h, tok._h, table._h, capi._np_ptr(text), capi._np_ptr(offsets), n_lines,
                                              2048, None, corpus._h))
        return corpus

    tg = timed(lambda: text_path(gtok), reps)
    rows_g = corpus.read()
    tc = timed(lambda: text_path(htok), reps)
    rows_c = corpus.read()
    th = timed(hf_path, max(1, reps // 3))
    tokens = th[2]
    rows_h = corpus.read()
    same = bool(np.array_equal(rows_g.view(np.uint32), rows_h.view(np.uint32)) and
                np.array_equal(rows_c.view(np.uint32), rows_h.view(np.uint32)))
    # the GPU span of one call (CUDA events on the library's stream) and its kernels (torch.profiler)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(s)
    text_path(gtok)
    e1.record(s)
    torch.cuda.synchronize()
    span_ms = e0.elapsed_time(e1)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        text_path(gtok)
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.events():
        if ev.device_type.name == "CUDA" and ("stb_" in ev.name or "Memcpy" in ev.name):
            name = ev.name.split("(")[0].replace("void ", "")
            kern[name] = kern.get(name, 0.0) + ev.device_time_total / 1e3
    rate = lambda t: {"s": round(t[0], 4), "median_s": round(t[1], 4), "lines_per_s": round(n_lines / t[0]),
                      "tokens_per_s": round(tokens / t[0])}
    print(json.dumps({"card": card, "lines": n_lines, "tokens": tokens, "tokens_per_line": round(tokens / n_lines, 2),
                      "vocab": V, "taken": int(taken.sum()), "cores": os.cpu_count(), "train_s": round(train_s, 1),
                      "gpu_text": rate(tg), "cpp_host_tokenizer": rate(tc), "hf_encode_batch": rate(th),
                      "gpu_text_event_span_ms": round(span_ms, 3), "kernel_ms": {k: round(v, 3) for k, v in sorted(kern.items())},
                      "cpp_tokenize_bench": cpp_bench, "rows_bit_identical": same}))
    assert same


if __name__ == "__main__":
    main()
