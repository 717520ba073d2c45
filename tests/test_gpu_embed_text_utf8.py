"""K3 from text with a STB_TOKENIZER_UTF8 handle: the GPU normalises (Precompiled charsmap cluster by cluster,
Lowercase per character, Strip on Unicode White_Space, ...) and tokenises every valid UTF-8 line, and gives the
lines it cannot finish exactly back to the host tokenizer inside the same call.  Every line's ids equal a flags-0
handle's; the ids of the lines the GPU finished are checked id for id against HF `tokenizers`
(encode_batch(add_special_tokens=False), then encode_with_args' unk drop and truncation), rows bit for bit
against stb_embed on HF's ids."""
import json
import os
import random
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_host_cpp import _synthetic_unigram, _u, nmt_nfkc_tokenizer  # noqa: E402,F401
from test_gpu_embed_text import edge_lines, hf_csr, random_table  # noqa: E402

from semtools_b200 import capi  # noqa: E402

pytestmark = pytest.mark.gpu
SP = _u("\\u2581")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CJK = _u("\\u4e2d")

# the edge set: one entry per kind of text the normaliser and the splitter have to get right
EDGE = [_u(x) for x in (
    "caf\\u00e9 cafe\\u0301", "e\\u0301\\u0301\\u0301", "\\u00e9\\u0301\\u0301 x", "a\\u0300\\u0301\\u0302\\u0303b",
    "\\uff21\\uff22\\uff23 \\uff11\\uff12\\uff13", "\\uff76\\uff9e\\uff77\\uff9e \\uff8a\\uff9f", "\\uff21\\u0301",
    "\\ufb01ne \\ufb02ow \\ufb05", "\\u2460\\u2461 \\u00b2\\u00b3 \\u2122 \\u338f \\u3300",
    "\\ufdfa", "x \\ufdfa\\ufdfa\\ufdfa", "\\ufdfa \\ufdf2 ok",
    "\\u2028ls\\u2029", "\\u0085nel", "\\u3000ideographic\\u3000space", "a\\u00a0b\\u2009c",
    "a\\u200bb\\u200cc\\u200dd", "\\ufeffbom", "soft\\u00adhyphen", "ctl\\x01\\x02x", "tab\\there", "del\\x7fx", "a\\rb",
    "\\x00nul", "a\\x00b", "\\x00",
    "\\U0001f468\\u200d\\U0001f469\\u200d\\U0001f467\\u200d\\U0001f466 family", "\\U0001f1fa\\U0001f1f8\\U0001f1e6 flags",
    "\\u2764\\ufe0f \\U0001f44d\\U0001f3fd", "\\U0001d400\\U0001d401 \\U0001d7d8",
    "\\u0915\\u094d\\u0937 \\u0924\\u094d\\u0930 \\u091c\\u094d\\u091e", "\\u0915\\u094d\\u200d\\u0937",
    "\\u1100\\u1161\\u11a8 \\uac01 \\u1100 \\u1161", "\\u0e2a\\u0e27\\u0e31\\u0e2a\\u0e14\\u0e35 \\u0e33",
    "\\u0645\\u0631\\u062d\\u0628\\u0627 \\u0634\\u0643\\u0631\\u0627",
    "\\u2581start", "x\\u2581y", "\\u2581", "\\u2581\\u2581", "a \\u2581 b", "\\u2581 \\u2581x",
    "\\u200b", "\\u200b\\u200c", "\\u00ad", "\\ufeff", "\\x01\\x02", "\\x01",
    "  multiple   spaces  ", "", " ", "\\u2026  \\u2025 \\u2024",
)] + [CJK * 84, CJK * 85, "x " + CJK * 84 + " y", "x " + CJK * 85 + " y", "ab" + CJK * 84]
DELETED = [_u(x) for x in ("\\u200b", "\\u200b\\u200c", "\\u00ad", "\\ufeff", "\\x01\\x02", "\\x01")]
# lines that every host splits the same way (no line or paragraph separators, no NUL)
FILE_EDGE = [l for l in EDGE if not any(c in l for c in _u("\\n\\r\\x00\\x0b\\x0c\\x1c\\x1d\\x1e\\x85\\u2028\\u2029"))]


def handles(ctx, path):
    data = open(path, "rb").read()
    return capi.Tokenizer(ctx, data, utf8=True), capi.Tokenizer(ctx, data)


def check_lines(ctx, tk, path, lines, unk_token_id=None):
    """The UTF-8 handle's CSR equals the flags-0 handle's on every line, and HF's on every line it finished on
    the GPU; taken is a subset of the rule's lines.  Returns (rule, taken) at max_length 2048."""
    utf8, plain = handles(ctx, path)
    rule = utf8.gpu_lines(lines)
    first = None
    for max_length in (2048, 512, 7):
        off, ids, taken = utf8.debug_tokenize(lines, max_length)
        p_off, p_ids, _ = plain.debug_tokenize(lines, max_length)
        assert np.array_equal(off, p_off) and np.array_equal(ids[:off[-1]], p_ids[:p_off[-1]]), max_length
        assert not (taken & ~rule).any()
        w_off, w_ids = hf_csr(tk, lines, max_length, unk_token_id)
        for i, line in enumerate(lines):
            if taken[i]:
                got = ids[off[i]:off[i + 1]].tolist()
                assert got == w_ids[w_off[i]:w_off[i + 1]].tolist(), (max_length, [hex(ord(c)) for c in line[:40]])
        first = taken if first is None else first
    utf8.close()
    plain.close()
    return rule, first


def test_multilingual_and_edge_ids_match_hf(ctx, nmt_nfkc_tokenizer):
    tk, path, corpus_lines = nmt_nfkc_tokenizer
    lines = corpus_lines[:400] + EDGE + edge_lines(["the", "quick", "Brown", "fox"])
    rule, taken = check_lines(ctx, tk, path, lines)
    by = {l: (bool(r), bool(t)) for l, r, t in zip(lines, rule, taken)}
    assert all(rule)                                                     # every line is valid UTF-8 with no added token
    assert taken[:400].mean() > 0.9                                      # most multilingual lines run on the GPU
    back = [l for l, (r, t) in by.items() if r and not t]
    assert _u("\\ufdfa") in back and CJK * 85 in back and "x " + CJK * 85 + " y" in back   # region overflow, piece cap
    assert by[CJK * 84][1] and by["x " + CJK * 84 + " y"][1]
    for l in ["tab\there", SP, "x" + SP + "y", "\x00nul", _u("\\u3000ideographic\\u3000space")]:
        assert by[l][1], repr(l)
    # a line whose characters the charsmap deletes: zero ids, on the GPU
    zero = [l for l in DELETED if not tk.encode(l, add_special_tokens=False).ids]
    assert zero and all(by[l][1] for l in zero)
    # truncation bites on GPU lines
    n_ids = [len(e.ids) for e, t in zip(tk.encode_batch(lines, add_special_tokens=False), taken) if t]
    assert max(n_ids) > 2048 and sum(512 < k <= 2048 for k in n_ids) >= 1


@pytest.mark.parametrize("scheme", ["always", "first", "never"])
@pytest.mark.parametrize("norm", ["none", "lower+multispace", "strip_prepend"])
def test_synthetic_unigram_non_ascii(ctx, tmp_path, scheme, norm):
    from tokenizers import Regex, normalizers
    n = {"none": None,
         "lower+multispace": normalizers.Sequence([normalizers.Lowercase(), normalizers.Replace(Regex(" {2,}"), " ")]),
         "strip_prepend": normalizers.Sequence([normalizers.Strip(), normalizers.Prepend("ab"), normalizers.Lowercase()])}[norm]
    tk, path, alphabet = _synthetic_unigram(tmp_path, seed=7 + len(norm), normalizer=n, prepend_scheme=scheme)
    rnd = random.Random(len(norm) + len(scheme))
    pool = alphabet + [_u(x) for x in ("\\u0130", "\\u03a3", "\\u0391\\u03a3", "\\u00c9", "\\u0412", "\\u1e9e", "\\u2126")] + ["X", "THE", "ab"]
    lines = [_u(x) for x in ("\\u0130stanbul \\u0130", "\\u03a3 \\u03c2 \\u0391\\u03a3 \\u03a3\\u0391\\u03a3 \\u03c3\\u03b1\\u03c2",
                             "\\u3000lead", "\\u3000\\u3000x y", "\\u3000", " \\u3000 z", "x\\u3000", "\\u00a0nb\\u00a0",
                             "\\u2581lead", "a\\u2581b \\u2581", "\\u2028x\\u2029")] + [" leading", "", " ", "a  b"]
    for _ in range(300):
        words = ["".join(rnd.choice(pool) for _ in range(rnd.randint(1, 8))) for _ in range(rnd.randint(0, 10))]
        lines.append((" " * rnd.randint(1, 3)).join(words) if rnd.random() < 0.3 else " ".join(words))
    rule, taken = check_lines(ctx, tk, path, lines)
    assert rule.all() and taken.sum() > 250
    if (norm, scheme) == ("strip_prepend", "first"):
        # a left Strip moved the split off original offset 0: given back (HF does not prepend there)
        led = [t for l, t in zip(lines, taken) if l[:1] in (" ", _u("\\u3000")) and l.strip()]
        assert led and not any(led)


def test_rows_match_stb_embed_bit_for_bit(ctx, nmt_nfkc_tokenizer):
    tk, path, corpus_lines = nmt_nfkc_tokenizer
    rng = np.random.default_rng(13)
    V = tk.get_vocab_size()
    table = capi.Table(ctx, random_table(rng, V), weights=rng.uniform(0.5, 2, V).astype(np.float32))
    tok = capi.Tokenizer(ctx, open(path, "rb").read(), utf8=True)
    rnd = random.Random(6)
    # more than one chunk (65536 lines), given-back lines interleaved
    lines = [rnd.choice(corpus_lines) for _ in range(70000)]
    for j, l in enumerate(EDGE):
        lines[j * 300] = l
    for k in range(0, len(lines), 89):
        lines[k] = _u("\\ufdfa") + " " + lines[k]
    off, ids, taken = tok.debug_tokenize(lines, 2048)
    assert 0 < (~taken).sum() and taken.sum() > len(lines) * 0.9
    w_off, w_ids = hf_csr(tk, lines, 2048)
    want = capi.embed(ctx, table, w_off, w_ids)
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
    q = [corpus_lines[1] * 40, CJK * 85 + " " + corpus_lines[2]]
    off, ids = hf_csr(tk, q, 512)
    assert np.array_equal(capi.embed_text(ctx, tok, table, q, 512).view(np.uint32),
                          capi.embed(ctx, table, off, ids).view(np.uint32))


def test_out_of_range_token_appends_nothing(ctx, nmt_nfkc_tokenizer):
    tk, path, corpus_lines = nmt_nfkc_tokenizer
    rng = np.random.default_rng(9)
    table = capi.Table(ctx, random_table(rng, 8))             # far fewer rows than the vocabulary
    tok = capi.Tokenizer(ctx, open(path, "rb").read(), utf8=True)
    for make in (lambda: capi.Corpus(ctx, 16), lambda: capi.Corpus.in_host_memory(ctx, 16)):
        c = make()
        c.append(random_table(rng, 5))
        before = c.read()
        with pytest.raises(capi.StbError) as e:
            capi.embed_text(ctx, tok, table, [corpus_lines[0], _u("\\ufdfa")], 2048, out=False, append_to=c)
        assert e.value.status == capi.STB_ERR_RANGE
        assert len(c) == 5 and np.array_equal(c.read().view(np.uint32), before.view(np.uint32))
        c.close()


def test_rule_on_bytes_and_added_tokens(ctx, tmp_path, nmt_nfkc_tokenizer):
    from tokenizers import AddedToken, Regex, normalizers
    tk, path, corpus_lines = nmt_nfkc_tokenizer
    utf8, plain = handles(ctx, path)
    bad = [b"ok \x80 cont", b"over \xc0\xaf long", b"\xe0\x80\xaf", b"sur \xed\xa0\x80 gate", b"\xf4\x90\x80\x80 big",
           b"cut \xe4\xb8", b"\xff"]
    good = ["ok", corpus_lines[0], "tab\tx"]
    lines = bad + [g.encode() for g in good]
    rule = utf8.gpu_lines(lines)
    assert rule.tolist() == [False] * len(bad) + [True] * len(good)
    for max_length in (2048, 7):
        off, ids, taken = utf8.debug_tokenize(lines, max_length)
        p_off, p_ids, _ = plain.debug_tokenize(lines, max_length)
        assert np.array_equal(off, p_off) and np.array_equal(ids[:off[-1]], p_ids[:p_off[-1]])
        assert not (taken & ~rule).any() and taken[len(bad):].all()
    # added tokens: raw content declined, normalised content declined
    tk2, path2, _ = _synthetic_unigram(tmp_path, seed=19, normalizer=normalizers.Sequence(
        [normalizers.Lowercase(), normalizers.Replace(Regex(" {2,}"), " ")]))
    tk2.add_special_tokens(["<s>", "</s>", AddedToken("<mask>", lstrip=True, special=True)])
    tk2.add_tokens([AddedToken(_u("F\\u00f6\\u00f6 Bar"), normalized=True)])
    tk2.save(str(path2))
    lines = ["<s>héllo</s>", "a <mask> ß", "föö bar", "FÖÖ  BAR x", "plain λ line", "<S>"]
    rule, taken = check_lines(ctx, tk2, path2, lines)
    assert rule.tolist() == [False, False, False, False, True, False] and taken.tolist() == rule.tolist()


def test_other_shapes_take_no_line(ctx, tmp_path):
    from tokenizers import normalizers, pre_tokenizers
    tk, path, _ = _synthetic_unigram(tmp_path, seed=23, normalizer=normalizers.Sequence([normalizers.NFKC()]))
    utf8 = capi.Tokenizer(ctx, open(path, "rb").read(), utf8=True)
    assert not utf8.gpu_lines(["plain", "café"]).any()
    tk, path, _ = _synthetic_unigram(tmp_path, seed=24, normalizer=None)
    tk.pre_tokenizer = pre_tokenizers.WhitespaceSplit()
    tk.save(str(path))
    rule, taken = check_lines(ctx, tk, path, ["the thing", "é 中", ""])
    assert not rule.any() and not taken.any()
    h = capi.vp()                                                # an unknown flag is refused
    buf = np.frombuffer(open(path, "rb").read(), dtype=np.uint8)
    assert capi.lib().stb_tokenizer_load_ex(ctx._h, capi._np_ptr(buf), buf.size, 2, capi.C.byref(h)) == capi.STB_ERR_ARG


def _model_dir(tmp_path, tk, path, seed):
    import shutil
    from safetensors.numpy import save_file
    d = tmp_path / "model"
    d.mkdir()
    shutil.copy(path, d / "tokenizer.json")
    save_file({"embeddings": random_table(np.random.default_rng(seed), tk.get_vocab_size())}, str(d / "model.safetensors"))
    (d / "config.json").write_text(json.dumps({"normalize": True}))
    return d


def test_python_host_output_is_unchanged(ctx, tmp_path, nmt_nfkc_tokenizer, monkeypatch):
    """With gpu_tokenizer="utf8" multilingual batches go to stb_embed_text; search_files, the stdin document and
    workspace indexing print the same bytes as through HF tokenizers + stb_embed."""
    import io
    from semtools_b200 import cmds
    from semtools_b200.model import StaticModel
    tk, path, corpus_lines = nmt_nfkc_tokenizer
    d = _model_dir(tmp_path, tk, path, 16)
    multi = corpus_lines[:60] + FILE_EDGE
    (tmp_path / "a.txt").write_text("\n".join(multi[:50]) + "\n")
    (tmp_path / "b.txt").write_text("\n".join(multi[50:]) + "\n")
    files = [str(tmp_path / "a.txt"), str(tmp_path / "b.txt")]
    query = corpus_lines[3].split()[0] + " " + corpus_lines[7].split()[-1]

    def run(gpu):
        monkeypatch.setenv("HOME", str(tmp_path / f"home_{gpu}"))
        monkeypatch.delenv("SEMTOOLS_WORKSPACE", raising=False)
        model = StaticModel.from_pretrained(str(d), ctx=ctx, gpu_tokenizer="utf8")
        if not gpu:
            model._tokenizer_json = None
        outs = []
        for kw in [dict(n_lines=1, top_k=5, ignore_case=False, json=False), dict(n_lines=0, top_k=3, ignore_case=True, json=True)]:
            out = io.StringIO()
            cmds.search_cmd(query, files, kw["n_lines"], kw["top_k"], None, kw["ignore_case"], kw["json"], None, model, out=out)
            outs.append(out.getvalue())
        out = io.StringIO()
        cmds.search_cmd(query, [], 1, 2, None, False, True, None, model, stdin_lines=multi, stdin_is_tty=False, out=out)
        outs.append(out.getvalue())
        monkeypatch.setenv("SEMTOOLS_WORKSPACE", "ws")
        for _ in range(2):                                                # index, then answer from the store
            out, err = io.StringIO(), io.StringIO()
            cmds.search_cmd(query, files, 1, 4, None, False, False, None, model, out=out, err=err)
            outs += [out.getvalue(), err.getvalue()]
        return outs, model

    want, _ = run(False)
    got, model = run(True)
    assert got == want
    assert model._prepare(corpus_lines[:30], 2048)[0] == "text" and model._prepare(multi, 2048)[0] == "text"
    ascii_model = StaticModel.from_pretrained(str(d), ctx=ctx)
    assert ascii_model._prepare(corpus_lines[:30], 2048)[0] == "ids"          # the default stays the ASCII rule
    with pytest.raises(ValueError):
        StaticModel.from_pretrained(str(d), ctx=ctx, gpu_tokenizer="nfkc")


def test_cpp_cli_gpu_tokenizer_utf8(ctx, tmp_path, nmt_nfkc_tokenizer):
    """--gpu-tokenizer utf8 on multilingual files prints the bytes the Python host prints through HF tokenizers
    + stb_embed, with and without a workspace."""
    import io
    import subprocess
    from semtools_b200 import cmds
    from semtools_b200.model import StaticModel
    subprocess.run(["bash", os.path.join(ROOT, "scripts", "build_host.sh")], check=True, cwd=ROOT)
    tk, path, corpus_lines = nmt_nfkc_tokenizer
    d = _model_dir(tmp_path, tk, path, 17)
    multi = corpus_lines[:60] + FILE_EDGE
    (tmp_path / "a.txt").write_text("\n".join(multi[:50]) + "\n")
    (tmp_path / "b.txt").write_text("\n".join(multi[50:]) + "\n")
    files = [str(tmp_path / "a.txt"), str(tmp_path / "b.txt")]
    query = corpus_lines[5].split()[0]
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
                cmds.search_cmd(query, files, kw["n_lines"], kw["top_k"], None, kw["ignore_case"], kw["json"], None, model,
                                out=out, err=err)
            finally:
                os.environ.clear()
                os.environ.update(old)
            r = subprocess.run([binary, "--model", str(d), "--gpu-tokenizer", "utf8", query] + files + extra, capture_output=True,
                               text=True, stdin=subprocess.DEVNULL, env=env)
            assert r.returncode == 0, r.stderr
            assert r.stdout == out.getvalue(), (ws, extra)
            assert r.stderr == err.getvalue(), (ws, extra)
    r = subprocess.run([binary, "--model", str(d), "--gpu-tokenizer", "nfkc", "x", files[0]], capture_output=True, text=True)
    assert r.returncode == 2 and "--gpu-tokenizer" in r.stderr
