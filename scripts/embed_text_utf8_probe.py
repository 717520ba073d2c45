"""stb_embed_text through a STB_TOKENIZER_UTF8 handle: python scripts/embed_text_utf8_probe.py [lines] [reps]

Workload: `lines` (default 1M) seeded multilingual lines -- Latin with diacritics, Cyrillic, Greek, CJK, Hangul,
Devanagari, Arabic, Thai and compatibility characters (ligatures, full- and half-width forms, circled digits,
curly quotes, dashes, ellipses), a line in one script with English words mixed in -- and a tokenizer.json of the
reference model's shape: a 30k-piece Unigram trained by sentencepiece on text from the same model, the nmt_nfkc
charsmap, Replace(" {2,}"), Metaspace.
Paths, each timed with a host clock around calls that end in a synchronise, after a warm-up call, all appending
the rows to a corpus in HBM:
  utf8   stb_embed_text, UTF-8 handle (every valid line is a GPU candidate; the give-back goes to host threads)
  ascii  stb_embed_text, flags-0 handle (printable-ASCII lines on the GPU, the rest on host threads)
  hf     HF tokenizers encode_batch (all cores) + stb_embed
ASCII control: embed_text_probe.py's ASCII workload (its word model and line lengths) through the UTF-8 and
flags-0 handles of the same tokenizer, alternated in the same process.
Also: the candidate and give-back fractions (and how many given-back lines have a Metaspace piece past
STB_TOKENIZER_PIECE_CAP; the others outgrew their region or lost the "first" offset), per-kernel times of one
UTF-8 call from torch.profiler in a separate run, the card's name and power limit.  Rows of every path must be
bit-identical.  Writes its JSON line to stdout only.
"""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from semtools_b200 import capi  # noqa: E402
import embed_text_probe as ascii_probe  # noqa: E402


def _span(a, b):
    return [chr(c) for c in range(a, b + 1)]


SCRIPTS = {   # name: (weight, characters, words per line (lognormal mean), joiner)
    "latin": (0.25, list("abcdefghijklmnopqrstuvwxyz") * 3 + list("éèêëàâäôöüûçñßøåæœíóúÉÀÇ"), 2.3, " "),
    "cyrillic": (0.15, _span(0x430, 0x44F) + ["ё", "Д", "П", "М"], 2.3, " "),
    "greek": (0.08, _span(0x3B1, 0x3C9) + list("άέήίόύώΑΣΩ"), 2.2, " "),
    "cjk": (0.14, _span(0x4E00, 0x4E00 + 2500) + list("、。「」"), 1.2, ""),
    "hangul": (0.10, [chr(0xAC00 + i * 37) for i in range(300)], 2.0, " "),
    "devanagari": (0.08, _span(0x915, 0x939) + _span(0x93E, 0x94C) + ["्"], 2.0, " "),
    "arabic": (0.08, _span(0x627, 0x64A), 2.1, " "),
    "thai": (0.06, _span(0xE01, 0xE2E) + _span(0xE31, 0xE3A) + _span(0xE40, 0xE44), 1.2, ""),
    "compat": (0.06, list("ﬁﬂ①②③™ＡＢＣ１２３ｶﾞｷﾞ㎏㎝½“”‘’—–…") + list("abcdefghij"), 2.0, " "),
}
ENGLISH = ["the", "data", "model", "search", "file", "line", "GPU", "token", "index", "query"]


def word_pools(rng, n_words=4000):
    """Per script: n_words random words (1-8 characters; 1-3 for the scripts written without spaces) and Zipf
    weights, with the English words added at 8 % of the mass."""
    pools = {}
    zipf = 1.0 / np.arange(1, n_words + 1) ** 1.05
    for name, (_, chars, _, joiner) in SCRIPTS.items():
        lens = rng.integers(1, 4 if joiner == "" else 9, n_words)
        idx = rng.integers(0, len(chars), int(lens.sum()))
        ends = np.cumsum(lens)
        words = ["".join(chars[j] for j in idx[e - l:e]) for e, l in zip(ends, lens)]
        p = np.concatenate([zipf / zipf.sum() * 0.92, np.full(len(ENGLISH), 0.08 / len(ENGLISH))])
        pools[name] = (words + ENGLISH, p)
    return pools


def make_lines(rng, pools, n):
    names = list(SCRIPTS)
    w = np.array([SCRIPTS[k][0] for k in names])
    pick = rng.choice(len(names), n, p=w / w.sum())
    out = [""] * n
    for si, name in enumerate(names):
        _, _, mu, joiner = SCRIPTS[name]
        rows = np.nonzero(pick == si)[0]
        k = np.clip(np.round(rng.lognormal(mu, 0.5, len(rows))), 1, 60).astype(np.int64)
        words, p = pools[name]
        wi = rng.choice(len(words), int(k.sum()), p=p)
        gap = rng.random(int(k.sum())) < 0.15            # scripts without spaces: an occasional one
        ends = np.cumsum(k)
        for r, e, c in zip(rows, ends, k):
            if joiner:
                out[r] = " ".join(words[j] for j in wi[e - c:e])
            else:
                out[r] = "".join(words[j] + (" " if g else "") for j, g in zip(wi[e - c:e], gap[e - c:e])).strip() or "x"
    return out


def build_tokenizer(d, rng, pools):
    import sentencepiece as spm
    from sentencepiece import sentencepiece_model_pb2 as pb
    from tokenizers import Regex, Tokenizer
    from tokenizers.models import Unigram
    from tokenizers.normalizers import Precompiled, Replace, Sequence
    from tokenizers.pre_tokenizers import Metaspace
    with open(os.path.join(d, "corpus.txt"), "w", encoding="utf-8") as f:
        f.write("\n".join(make_lines(rng, pools, 100000)) + "\n")
    spm.SentencePieceTrainer.train(input=os.path.join(d, "corpus.txt"), model_prefix=os.path.join(d, "m"), vocab_size=30000,
                                   model_type="unigram", normalization_rule_name="nmt_nfkc", character_coverage=1.0,
                                   hard_vocab_limit=False, minloglevel=2, num_threads=os.cpu_count())
    mp = pb.ModelProto()
    mp.ParseFromString(open(os.path.join(d, "m.model"), "rb").read())
    tk = Tokenizer(Unigram([(x.piece, x.score) for x in mp.pieces], unk_id=next(i for i, x in enumerate(mp.pieces) if x.type == 2),
                           byte_fallback=False))
    tk.normalizer = Sequence([Precompiled(mp.normalizer_spec.precompiled_charsmap), Replace(Regex(" {2,}"), " ")])
    tk.pre_tokenizer = Metaspace(replacement="▁", prepend_scheme="always")
    return tk, tk.to_str().encode()


def main():
    n_lines = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    import torch
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    rng = np.random.default_rng(2025)
    t_start = time.perf_counter()
    log = lambda what: print(f"[{time.perf_counter() - t_start:7.1f}s] {what}", file=sys.stderr, flush=True)
    pools = word_pools(rng)
    with tempfile.TemporaryDirectory() as d:
        t0 = time.perf_counter()
        tk, tok_json = build_tokenizer(d, rng, pools)
        train_s = time.perf_counter() - t0
    log("tokenizer trained")
    lines = make_lines(rng, pools, n_lines)
    a_words, a_p = ascii_probe.word_model(rng)
    a_lines = ascii_probe.make_lines(rng, a_words, a_p, n_lines)
    log("lines made")
    dev = torch.device("cuda:0")
    s = torch.cuda.Stream(dev)
    torch.cuda.set_stream(s)
    ctx = capi.Context(0, s.cuda_stream)
    V = tk.get_vocab_size()
    table = capi.Table(ctx, (rng.standard_normal((V, 256), dtype=np.float32) * np.float32(0.1)))
    utok, atok = capi.Tokenizer(ctx, tok_json, utf8=True), capi.Tokenizer(ctx, tok_json)
    corpus = capi.Corpus(ctx, n_lines)
    packed = capi.pack_lines(lines)
    a_packed = capi.pack_lines(a_lines)

    def text_path(tok, tab, pk):                              # rows into the corpus in HBM, as ingestion does
        text, offsets = pk
        corpus.clear()
        capi._check(capi.lib().stb_embed_text(ctx._h, tok._h, tab._h, capi._np_ptr(text), capi._np_ptr(offsets),
                                              len(offsets) - 1, 2048, None, corpus._h))

    def hf_path():
        encs = tk.encode_batch(lines, add_special_tokens=False)
        ids = [e.ids[:2048] for e in encs]
        off = np.zeros(len(ids) + 1, dtype=np.uint64)
        off[1:] = np.cumsum([len(x) for x in ids])
        corpus.clear()
        capi.embed(ctx, table, off, np.fromiter((i for x in ids for i in x), dtype=np.uint32, count=int(off[-1])), out=False,
                   append_to=corpus)
        return int(off[-1])

    # the rule and the give-back
    cand = utok.gpu_lines(lines)
    ascii_taken = atok.gpu_lines(lines)
    _, _, on_gpu = utok.debug_tokenize(lines, 2048)
    back = [l for l, c, g in zip(lines, cand, on_gpu) if c and not g]
    cap = capi.STB_TOKENIZER_PIECE_CAP
    long_piece = sum(1 for l in back if any(len(("▁" + p).encode()) > cap for p in tk.normalizer.normalize_str(l).split(" ")))
    log("rule and give-back counted")

    tu = ascii_probe.timed(lambda: text_path(utok, table, packed), reps)
    rows_u = corpus.read()
    ta = ascii_probe.timed(lambda: text_path(atok, table, packed), reps)
    rows_a = corpus.read()
    log("utf8 and flags-0 handles timed")
    th = ascii_probe.timed(hf_path, max(1, reps // 3))
    log("hf timed")
    tokens = th[2]
    rows_h = corpus.read()
    same = bool(np.array_equal(rows_u.view(np.uint32), rows_h.view(np.uint32)) and
                np.array_equal(rows_a.view(np.uint32), rows_h.view(np.uint32)))
    # ASCII control, alternated: UTF-8 handle, flags-0 handle, ... (after one warm-up call of each)
    text_path(atok, table, a_packed)
    rows_aa = corpus.read()
    text_path(utok, table, a_packed)
    same = same and bool(np.array_equal(corpus.read().view(np.uint32), rows_aa.view(np.uint32)))
    t_au, t_aa = [], []
    for _ in range(reps):
        for tok, acc in ((utok, t_au), (atok, t_aa)):
            t0 = time.perf_counter()
            text_path(tok, table, a_packed)
            acc.append(time.perf_counter() - t0)
    a_off, _, a_on_gpu = utok.debug_tokenize(a_lines, 2048)
    a_tokens = int(a_off[-1])
    log("ascii control timed")
    # per-kernel times of one UTF-8 call (a separate run)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        text_path(utok, table, packed)
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.events():
        if ev.device_type.name == "CUDA" and ("stb_" in ev.name or "Memcpy" in ev.name):
            name = ev.name.split("(")[0].replace("void ", "")
            kern[name] = kern.get(name, 0.0) + ev.device_time_total / 1e3
    rate = lambda t, n, k: {"s": round(t[0], 4), "median_s": round(t[1], 4), "lines_per_s": round(n / t[0]),
                            "tokens_per_s": round(k / t[0])}
    print(json.dumps({
        "card": card, "lines": n_lines, "tokens": tokens, "tokens_per_line": round(tokens / n_lines, 2), "vocab": V,
        "cores": os.cpu_count(), "train_s": round(train_s, 1),
        "candidate_fraction": round(float(cand.mean()), 5), "ascii_rule_fraction": round(float(ascii_taken.mean()), 5),
        "give_back_fraction": round(len(back) / n_lines, 5), "give_back_piece_cap": long_piece,
        "give_back_other": len(back) - long_piece,
        "utf8": rate(tu, n_lines, tokens), "ascii_handle": rate(ta, n_lines, tokens), "hf_encode_batch": rate(th, n_lines, tokens),
        "ascii_control": {"lines": n_lines, "tokens": a_tokens, "gpu_fraction": round(float(a_on_gpu.mean()), 5),
                          "utf8": rate((min(t_au), float(np.median(t_au))), n_lines, a_tokens),
                          "ascii_handle": rate((min(t_aa), float(np.median(t_aa))), n_lines, a_tokens)},
        "utf8_kernel_ms": {k: round(v, 3) for k, v in sorted(kern.items())},
        "rows_bit_identical": same}))
    assert same


if __name__ == "__main__":
    main()
