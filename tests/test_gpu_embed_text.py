"""K3 from text (stb_embed_text): the Unigram tokenizer on the GPU for the lines the rule takes, the host
tokenizer for the rest, one CSR pooled by the K3 kernel.  Ids are checked id for id against HF `tokenizers`
(encode_batch(add_special_tokens=False), then encode_with_args' unk drop and truncation), rows bit for bit
against stb_embed on those ids."""
import json
import os
import random
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_host_cpp import _synthetic_unigram, _u, nmt_nfkc_tokenizer  # noqa: E402,F401

from semtools_b200 import capi  # noqa: E402

pytestmark = pytest.mark.gpu
SP = _u("\\u2581")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAP = capi.STB_TOKENIZER_PIECE_CAP


def hf_csr(tk, lines, max_length, unk_token_id=None):
    encs = tk.encode_batch(lines, add_special_tokens=False)
    rows = []
    for e in encs:
        ids = [i for i in e.ids if unk_token_id is None or i != unk_token_id]
        rows.append(ids[:max_length])
    off = np.zeros(len(rows) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(r) for r in rows]) if rows else []
    return off, np.array([i for r in rows for i in r], dtype=np.uint32)


def edge_lines(words):
    rnd = random.Random(17)
    many = " ".join(rnd.choice(words) for _ in range(3000))
    return ["", " ", "   ", "hello world", " leading", "trailing ", "a  b   c  ", "  two  leading", "XYZ qqq ZZZ",
            "<s>", "<unk>", "<mask>", "a <s> b </s>", SP, "x" + SP + "y", "tab\there", "ctl\x01x", "del\x7fx",
            "a" * (CAP - 3), "b " + "a" * (CAP - 3) + " c", "a" * (CAP - 2), "b " + "a" * (CAP - 2),
            many, " ".join(many.split()[:600]), many[:1200], "!!! ??? ~~~ @@@ ### $$$ %%% ^^^ &&& *** ((( ))) {{{ }}} [[[ ]]] ||| \\\\ ```",
            "0123456789 " * 20, "MiXeD CaSe WoRdS"] + \
           [" ".join(rnd.choice(words) for _ in range(rnd.randint(0, 12))) for _ in range(300)]


def check_ids(ctx, tk, path, lines, unk_token_id=None, taken_only=False):
    """Ids of every line (taken_only: of the lines the GPU takes) equal HF's."""
    tok = capi.Tokenizer(ctx, open(path, "rb").read())
    taken = None
    for max_length in (2048, 512, 7):
        off, ids, taken = tok.debug_tokenize(lines, max_length)
        w_off, w_ids = hf_csr(tk, lines, max_length, unk_token_id)
        for i, line in enumerate(lines):
            if taken_only and not taken[i]:
                continue
            got = ids[off[i]:off[i + 1]].tolist()
            want = w_ids[w_off[i]:w_off[i + 1]].tolist()
            assert got == want, (max_length, bool(taken[i]), repr(line)[:120])
        assert np.array_equal(taken, tok.gpu_lines(lines))
    return tok, taken


def test_nmt_nfkc_ids_match_hf(ctx, nmt_nfkc_tokenizer):
    tk, path, corpus_lines = nmt_nfkc_tokenizer
    words = sorted({w for l in corpus_lines[:200] for w in l.split() if w.isascii()}) + ["the", "quick", "Brown", "fox"]
    lines = edge_lines(words) + corpus_lines[:100]
    tok, taken = check_ids(ctx, tk, path, lines)
    by = dict(zip(lines, taken))
    # both sides of the rule
    for l in ["", " ", "hello world", "a" * (CAP - 3), "b " + "a" * (CAP - 3) + " c", "<s>"]:
        assert by[l], l
    for l in [SP, "tab\there", "ctl\x01x", "del\x7fx", "a" * (CAP - 2), "b " + "a" * (CAP - 2)]:
        assert not by[l], l
    assert sum(taken) > 250 and sum(not t for t in taken) >= 6
    n_ids = [len(e.ids) for e, t in zip(tk.encode_batch(lines, add_special_tokens=False), taken) if t]
    assert max(n_ids) > 2048 and sum(512 < k <= 2048 for k in n_ids) >= 1        # both truncations bite on the GPU
    tok.close()


@pytest.mark.parametrize("scheme", ["always", "first", "never"])
@pytest.mark.parametrize("norm", ["none", "lower+multispace", "strip_prepend"])
def test_synthetic_unigram_ids_match_hf(ctx, tmp_path, scheme, norm):
    from tokenizers import Regex, normalizers
    n = {"none": None,
         "lower+multispace": normalizers.Sequence([normalizers.Lowercase(), normalizers.Replace(Regex(" {2,}"), " ")]),
         "strip_prepend": normalizers.Sequence([normalizers.Strip(), normalizers.Prepend("ab"), normalizers.Lowercase()])}[norm]
    tk, path, alphabet = _synthetic_unigram(tmp_path, seed=5 + len(norm), normalizer=n, prepend_scheme=scheme)
    words = ["the", "thing", "abab", "ababab", "ing", "X", "Q", "THE", "ab", "zzz", "a.b,c-d"] + \
            ["".join(random.Random(i).choice("abcdefghijklmnopqrstuvwxyz0123456789.,-XQ!") for _ in range(1 + i % 9)) for i in range(80)]
    lines = edge_lines(words)
    # a left Strip under "first": HF prepends by the split's ORIGINAL offset, which a stripped leading space moves
    # off 0; the rule declines lines that start with a space there (the host tokenizer, which tokenises declined
    # lines in the library, prepends by the normalised text, so only the taken lines are compared with HF)
    strip_first = (norm, scheme) == ("strip_prepend", "first")
    tok, taken = check_ids(ctx, tk, path, lines, taken_only=strip_first)
    assert sum(taken) > 250
    if strip_first:
        assert not any(t for l, t in zip(lines, taken) if l.startswith(" "))
    tok.close()


def test_added_tokens_are_declined_and_exact(ctx, tmp_path):
    from tokenizers import AddedToken, Regex, normalizers
    tk, path, _ = _synthetic_unigram(tmp_path, seed=9, normalizer=normalizers.Sequence(
        [normalizers.Lowercase(), normalizers.Replace(Regex(" {2,}"), " ")]))
    tk.add_special_tokens(["<s>", "</s>", AddedToken("<mask>", lstrip=True, special=True)])
    tk.add_tokens([AddedToken("Foo Bar", normalized=True)])
    tk.save(str(path))
    lines = ["<s>hello</s>", "a <mask> b", "foo bar", "FOO  BAR x", "foo barx", "plain line", "fo obar", "<S>"]
    tok, taken = check_ids(ctx, tk, path, lines)
    # "<S>" lowercases to "<s>": declined, although HF matches "<s>" (normalized = false) on the raw text only
    assert taken.tolist() == [False, False, False, False, False, True, True, False]


def random_table(rng, V):
    return (rng.standard_normal((V, 256)) * 0.1).astype(np.float32)


def test_rows_match_stb_embed_bit_for_bit(ctx, nmt_nfkc_tokenizer):
    tk, path, corpus_lines = nmt_nfkc_tokenizer
    rng = np.random.default_rng(3)
    V = tk.get_vocab_size()
    table = capi.Table(ctx, random_table(rng, V), weights=rng.uniform(0.5, 2, V).astype(np.float32))
    tok = capi.Tokenizer(ctx, open(path, "rb").read())
    words = sorted({w for l in corpus_lines[:200] for w in l.split()})
    rnd = random.Random(4)
    # more than one chunk (65536 lines), taken and declined lines interleaved
    lines = [" ".join(rnd.choice(words) for _ in range(rnd.randint(0, 9))) for _ in range(70000)]
    for j, l in enumerate(edge_lines(["the", "quick", "brown"])):
        lines[j * 200] = l
    for k in range(0, len(lines), 97):
        lines[k] = "tab\tline " + lines[k]
    taken = tok.gpu_lines(lines)
    assert 0 < taken.sum() < len(lines)
    off, ids = hf_csr(tk, lines, 2048)
    want = capi.embed(ctx, table, off, ids)
    got = capi.embed_text(ctx, tok, table, lines, 2048)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    for make in (lambda: capi.Corpus(ctx, 16), lambda: capi.Corpus.in_host_memory(ctx, 16)):
        c = make()
        c.append(want[:3])
        rows = capi.embed_text(ctx, tok, table, lines, 2048, out=True, append_to=c)
        assert np.array_equal(rows.view(np.uint32), want.view(np.uint32))
        assert len(c) == 3 + len(lines)
        assert np.array_equal(c.read(3).view(np.uint32), want.view(np.uint32))
        c.close()
    # the query form: 512 ids
    q = [lines[1] * 60]
    off, ids = hf_csr(tk, q, 512)
    assert np.array_equal(capi.embed_text(ctx, tok, table, q, 512).view(np.uint32),
                          capi.embed(ctx, table, off, ids).view(np.uint32))


def test_out_of_range_token_appends_nothing(ctx, nmt_nfkc_tokenizer):
    tk, path, corpus_lines = nmt_nfkc_tokenizer
    rng = np.random.default_rng(8)
    table = capi.Table(ctx, random_table(rng, 8))             # far fewer rows than the vocabulary
    tok = capi.Tokenizer(ctx, open(path, "rb").read())
    for make in (lambda: capi.Corpus(ctx, 16), lambda: capi.Corpus.in_host_memory(ctx, 16)):
        c = make()
        base = random_table(rng, 5)
        c.append(base)
        before = c.read()
        with pytest.raises(capi.StbError) as e:
            capi.embed_text(ctx, tok, table, ["the quick brown fox", "tab\tx"], 2048, out=False, append_to=c)
        assert e.value.status == capi.STB_ERR_RANGE
        assert len(c) == 5 and np.array_equal(c.read().view(np.uint32), before.view(np.uint32))
        c.close()


def test_other_shapes_take_no_line_and_stay_exact(ctx, tmp_path):
    from tokenizers import Tokenizer, models, pre_tokenizers
    tk, path, _ = _synthetic_unigram(tmp_path, seed=21, normalizer=None)
    lines = ["the thing", "abab ab", " x  y ", "", "ing ing"]
    for pre in (pre_tokenizers.WhitespaceSplit(),
                pre_tokenizers.Sequence([pre_tokenizers.WhitespaceSplit(), pre_tokenizers.Metaspace(replacement=SP)])):
        tk.pre_tokenizer = pre
        p = tmp_path / "other.json"
        tk.save(str(p))
        tok, taken = check_ids(ctx, tk, p, lines)
        assert not taken.any()
        rng = np.random.default_rng(1)
        table = capi.Table(ctx, random_table(rng, tk.get_vocab_size()))
        off, ids = hf_csr(tk, lines, 2048)
        assert np.array_equal(capi.embed_text(ctx, tok, table, lines, 2048).view(np.uint32),
                              capi.embed(ctx, table, off, ids).view(np.uint32))
    wl = Tokenizer(models.WordLevel({"[UNK]": 0, "a": 1}, unk_token="[UNK]"))
    wl.pre_tokenizer = pre_tokenizers.WhitespaceSplit()
    with pytest.raises(capi.StbError) as e:
        capi.Tokenizer(ctx, wl.to_str().encode())
    assert e.value.status == capi.STB_ERR_ARG and "Unigram only" in str(e.value)


def test_refused_line_fails_the_call_and_writes_nothing(ctx, tmp_path):
    from tokenizers import normalizers
    tk, path, _ = _synthetic_unigram(tmp_path, seed=4, normalizer=normalizers.Sequence([normalizers.NFKC()]))
    tok = capi.Tokenizer(ctx, open(path, "rb").read())
    rng = np.random.default_rng(2)
    table = capi.Table(ctx, random_table(rng, tk.get_vocab_size()))
    c = capi.Corpus(ctx, 4)
    with pytest.raises(capi.StbError) as e:
        capi.embed_text(ctx, tok, table, ["plain", "café"], 2048, out=False, append_to=c)
    assert e.value.status == capi.STB_ERR_ARG and len(c) == 0
    assert not tok.gpu_lines(["plain"]).any()                   # a Unicode form: the tokenizer takes no line
    j = json.loads(open(path).read())
    j["model"]["byte_fallback"] = True
    with pytest.raises(capi.StbError) as e:
        capi.Tokenizer(ctx, json.dumps(j).encode())
    assert e.value.status == capi.STB_ERR_ARG


def test_python_host_output_is_unchanged(ctx, tmp_path, nmt_nfkc_tokenizer, monkeypatch):
    """search_files / the stdin document / workspace indexing of the Python host through stb_embed_text
    print the same bytes as through HF tokenizers + stb_embed."""
    import io
    import shutil
    from safetensors.numpy import save_file
    from semtools_b200 import cmds
    from semtools_b200.model import StaticModel
    monkeypatch.setenv("HOME", str(tmp_path))
    monkeypatch.delenv("SEMTOOLS_WORKSPACE", raising=False)
    tk, path, corpus_lines = nmt_nfkc_tokenizer
    d = tmp_path / "model"
    d.mkdir()
    shutil.copy(path, d / "tokenizer.json")
    rng = np.random.default_rng(6)
    save_file({"embeddings": random_table(rng, tk.get_vocab_size())}, str(d / "model.safetensors"))
    (d / "config.json").write_text(json.dumps({"normalize": True}))
    ascii_lines = [l for l in corpus_lines if l.isascii()][:40] + ["the quick brown fox", "hello  world", ""]
    (tmp_path / "a.txt").write_text("\n".join(ascii_lines) + "\n")
    (tmp_path / "b.txt").write_text("\n".join(corpus_lines[:30]) + "\n")      # non-ASCII: the HF path
    files = [str(tmp_path / "a.txt"), str(tmp_path / "b.txt")]

    def run(text_path):
        monkeypatch.setenv("HOME", str(tmp_path / f"home_{text_path}"))
        monkeypatch.delenv("SEMTOOLS_WORKSPACE", raising=False)
        model = StaticModel.from_pretrained(str(d), ctx=ctx)
        if not text_path:
            model._tokenizer_json = None
        outs = []
        for kw in [dict(n_lines=1, top_k=5, max_distance=None, ignore_case=False, json=False),
                   dict(n_lines=0, top_k=3, max_distance=None, ignore_case=True, json=True)]:
            out = io.StringIO()
            cmds.search_cmd("quick fox", files, kw["n_lines"], kw["top_k"], kw["max_distance"], kw["ignore_case"],
                            kw["json"], None, model, out=out)
            outs.append(out.getvalue())
        out = io.StringIO()
        cmds.search_cmd("fox", [], 1, 2, None, False, True, None, model, stdin_lines=ascii_lines, stdin_is_tty=False, out=out)
        outs.append(out.getvalue())
        monkeypatch.setenv("SEMTOOLS_WORKSPACE", "ws")                 # workspace indexing: encode_with_args batches
        for _ in range(2):                                                # index, then answer from the store
            out, err = io.StringIO(), io.StringIO()
            cmds.search_cmd("quick fox", files, 1, 4, None, False, False, None, model, out=out, err=err)
            outs += [out.getvalue(), err.getvalue()]
        assert (model.text_tokenizer() is not None) == text_path
        return outs, model

    want, _ = run(False)
    got, model = run(True)
    assert got == want
    assert model._prepare(ascii_lines, 2048)[0] == "text" and model._prepare(corpus_lines[:30], 2048)[0] == "ids"
    rows = model.encode_with_args(ascii_lines * 30, 2048, 256)
    ref = StaticModel.from_pretrained(str(d), ctx=ctx)
    ref._tokenizer_json = None
    assert np.array_equal(rows.view(np.uint32), ref.encode_with_args(ascii_lines * 30, 2048, 256).view(np.uint32))


def test_cpp_cli_output_is_unchanged(ctx, tmp_path, nmt_nfkc_tokenizer):
    """The C++ CLI on a model directory loads its tokenizer.json into the library and embeds every document
    (and, in a workspace, every new line) through stb_embed_text; it prints the bytes the Python host prints
    through HF tokenizers + stb_embed, with and without a workspace."""
    import io
    import shutil
    import subprocess
    from safetensors.numpy import save_file
    from semtools_b200 import cmds
    from semtools_b200.model import StaticModel
    subprocess.run(["bash", os.path.join(ROOT, "scripts", "build_host.sh")], check=True, cwd=ROOT)
    tk, path, corpus_lines = nmt_nfkc_tokenizer
    d = tmp_path / "model"
    d.mkdir()
    shutil.copy(path, d / "tokenizer.json")
    rng = np.random.default_rng(11)
    save_file({"embeddings": random_table(rng, tk.get_vocab_size())}, str(d / "model.safetensors"))
    (d / "config.json").write_text(json.dumps({"normalize": True}))
    ascii_lines = [l for l in corpus_lines if l.isascii()][:40] + ["the quick brown fox", "hello  world", "", "tab\tline"]
    (tmp_path / "a.txt").write_text("\n".join(ascii_lines) + "\n")
    (tmp_path / "b.txt").write_text("\n".join(corpus_lines[:30]) + "\n")
    files = [str(tmp_path / "a.txt"), str(tmp_path / "b.txt")]
    model = StaticModel.from_pretrained(str(d), ctx=ctx)
    model._tokenizer_json = None                                  # the Python host on HF tokenizers + stb_embed
    binary = os.path.join(ROOT, "semtools_b200", "lib", "semtools_b200_search")
    for ws in (None, "ws"):
        home_py, home_cpp = tmp_path / f"py_{ws}", tmp_path / f"cpp_{ws}"
        home_py.mkdir(); home_cpp.mkdir()
        env = dict(os.environ, HOME=str(home_cpp))
        env.pop("SEMTOOLS_WORKSPACE", None)
        if ws:
            env["SEMTOOLS_WORKSPACE"] = ws
        for extra, kw in [([], dict(n_lines=3, top_k=3, ignore_case=False, json=False)),
                          (["-n", "1", "--top-k", "5", "-j", "-i"], dict(n_lines=1, top_k=5, ignore_case=True, json=True))]:
            out, err = io.StringIO(), io.StringIO()
            old = dict(os.environ)
            os.environ["HOME"] = str(home_py)
            os.environ.pop("SEMTOOLS_WORKSPACE", None)
            if ws:
                os.environ["SEMTOOLS_WORKSPACE"] = ws
            try:
                cmds.search_cmd("quick fox", files, kw["n_lines"], kw["top_k"], None, kw["ignore_case"], kw["json"], None, model,
                                out=out, err=err)
            finally:
                os.environ.clear()
                os.environ.update(old)
            r = subprocess.run([binary, "--model", str(d), "quick fox"] + files + extra, capture_output=True, text=True,
                               stdin=subprocess.DEVNULL, env=env)
            assert r.returncode == 0, r.stderr
            assert r.stdout == out.getvalue(), (ws, extra)
            assert r.stderr == err.getvalue(), (ws, extra)
