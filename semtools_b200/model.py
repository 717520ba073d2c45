"""Host side of the static-embedding model: the reference's
`StaticModel::from_pretrained` / `encode_with_args` / `encode_single`
(model2vec-rs 0.1.3; call sites src/cmds/search.rs:123-128,136,154 and
src/search/mod.rs:69,138,153) with tokenisation on the host CPU (HF `tokenizers`, the same
library the reference links) and gather + pool + normalise on the GPU (K3, stb_embed).

Only LOCAL model directories are supported (tokenizer.json, model.safetensors,
config.json): this environment has no network, the hub download path of the reference
(hf-hub) is out of scope.  There is no CPU pooling path: without an H100, encode* raises.
"""
from __future__ import annotations

import json
import os

import numpy as np

from . import capi

MODEL_NAME = "minishlab/potion-multilingual-128M"      # src/search/mod.rs:16


class StaticModel:
    def __init__(self, tokenizer, embeddings, weights, mapping, normalize, median_token_length, unk_token_id,
                 ctx: capi.Context | None = None):
        self.tokenizer = tokenizer
        self.embeddings = embeddings
        self.weights, self.mapping = weights, mapping
        self.normalize = normalize
        self.median_token_length = median_token_length
        self.unk_token_id = unk_token_id
        self.ctx = ctx
        self._table = None
        self._tokenizer_json = None                              # tokenizer.json bytes (from_pretrained)
        self._text_tok = None
        self.gpu_tokenizer = "ascii"                             # the GPU rule of text_tokenizer(): "ascii" | "utf8"

    # -- StaticModel::from_pretrained(path, token, normalize, subfolder) -----------------------
    @classmethod
    def from_pretrained(cls, repo_or_path: str, token=None, normalize=None, subfolder=None,
                        ctx: capi.Context | None = None, gpu_tokenizer: str = "ascii") -> "StaticModel":
        """gpu_tokenizer: which lines the library's tokenizer takes on the GPU -- "ascii" (printable ASCII lines)
        or "utf8" (every valid UTF-8 line; lines the kernels cannot finish exactly go back to the host inside
        the call).  Both give the same ids."""
        if gpu_tokenizer not in ("ascii", "utf8"):
            raise ValueError(f"gpu_tokenizer must be 'ascii' or 'utf8', got {gpu_tokenizer!r}")
        from safetensors import safe_open
        from tokenizers import Tokenizer
        base = os.path.join(repo_or_path, subfolder) if subfolder else repo_or_path
        if not os.path.isdir(base):
            raise FileNotFoundError(
                f"{repo_or_path!r} is not a local model directory; hub download ({MODEL_NAME}) is not available offline")
        tok_path = os.path.join(base, "tokenizer.json")
        tokenizer = Tokenizer.from_file(tok_path)
        with open(os.path.join(base, "config.json")) as f:
            cfg = json.load(f)
        cfg_norm = bool(cfg.get("normalize", True))
        normalize = cfg_norm if normalize is None else bool(normalize)
        # median token length over the vocabulary (byte lengths, as `tk.len()` upstream)
        lens = sorted(len(t.encode("utf-8")) for t in tokenizer.get_vocab(False).keys())
        median = lens[len(lens) // 2] if lens else 1
        with open(tok_path) as f:
            spec = json.load(f)
        unk = (spec.get("model") or {}).get("unk_token")
        unk_id = tokenizer.token_to_id(unk) if isinstance(unk, str) else None
        weights = mapping = None
        with safe_open(os.path.join(base, "model.safetensors"), framework="np") as st:
            emb = st.get_tensor("embeddings")
            if emb.dtype == np.int8 or emb.dtype == np.float16:
                emb = emb.astype(np.float32)                    # F16 / I8 are upcast upstream
            emb = np.ascontiguousarray(emb, dtype=np.float32)
            keys = set(st.keys())
            if "weights" in keys:
                weights = np.ascontiguousarray(st.get_tensor("weights"), dtype=np.float32).reshape(-1)
            if "mapping" in keys:
                mapping = np.ascontiguousarray(st.get_tensor("mapping")).astype(np.uint32).reshape(-1)
        if emb.ndim != 2 or emb.shape[1] != capi.STB_DIM:
            raise ValueError(f"embedding table must be V x {capi.STB_DIM}, got {emb.shape}")
        m = cls(tokenizer, emb, weights, mapping, normalize, median, unk_id, ctx)
        m.gpu_tokenizer = gpu_tokenizer
        with open(tok_path, "rb") as f:
            m._tokenizer_json = f.read()
        m._tokenizer_file_hash = capi.fnv1a64(m._tokenizer_json)     # the C++ host hashes the same bytes (load_model_dir)
        return m

    def fingerprint(self) -> str:
        """Identity of the embedder (tokenizer spec + table + pooling flags), recorded in the
        workspace store so vectors of different models / tokenizers never mix silently."""
        ht = getattr(self, "_tokenizer_file_hash", None)
        if ht is None:                                           # built in memory (tests): hash the serialised spec
            tok = self.tokenizer.to_str().encode("utf-8") if hasattr(self.tokenizer, "to_str") else repr(self.tokenizer).encode()
            ht = capi.fnv1a64(tok)
        e = np.ascontiguousarray(self.embeddings, dtype=np.float32)
        head = e.reshape(-1)[: 262144].tobytes()
        h = ht ^ (capi.fnv1a64(head) * 0x9E3779B97F4A7C15 & 0xFFFFFFFFFFFFFFFF)
        return f"model2vec:{e.shape[0]}x{e.shape[1]}:n{int(self.normalize)}:{h:016x}"

    # -- tokenisation (host) --------------------------------------------------------------------
    @staticmethod
    def truncate_str(text: str, max_tokens: int, median_token_length: int) -> str:
        """Keep the first max_tokens * median_token_length chars (char boundary safe)."""
        return text[: max_tokens * median_token_length]

    def truncated(self, sentences, max_length):
        return [self.truncate_str(s, max_length, self.median_token_length) if max_length is not None else s
                for s in sentences]

    def tokenize(self, sentences, max_length):
        """-> (offsets u64[n+1], ids u32[...]) exactly as encode_with_args prepares them:
        char-truncate, encode_batch_fast(add_special_tokens=false), drop unk, truncate."""
        texts = self.truncated(sentences, max_length)
        encs = self.tokenizer.encode_batch(texts, add_special_tokens=False) if texts else []
        rows = []
        for e in encs:
            ids = e.ids
            if self.unk_token_id is not None:
                ids = [i for i in ids if i != self.unk_token_id]
            if max_length is not None:
                ids = ids[:max_length]
            rows.append(ids)
        offsets = np.zeros(len(rows) + 1, dtype=np.uint64)
        if rows:
            offsets[1:] = np.cumsum([len(r) for r in rows])
        ids = np.fromiter((i for r in rows for i in r), dtype=np.uint32, count=int(offsets[-1]))
        return offsets, ids

    # -- GPU residency ------------------------------------------------------------------------------
    def table(self) -> capi.Table:
        if self.ctx is None:
            self.ctx = capi.Context(0)
        if self._table is None:
            self._table = capi.Table(self.ctx, self.embeddings, self.weights, self.mapping, self.normalize)
        return self._table

    def text_tokenizer(self) -> capi.Tokenizer | None:
        """The model's tokenizer.json loaded into the library (stb_embed_text tokenises on the GPU), or None:
        a model built in memory, or a tokenizer shape the library's tokenizer does not read."""
        if self._text_tok is None and self._tokenizer_json is not None:
            self.table()
            try:
                self._text_tok = capi.Tokenizer(self.ctx, self._tokenizer_json, utf8=self.gpu_tokenizer == "utf8")
            except capi.StbError as e:
                if e.status != capi.STB_ERR_ARG:
                    raise
                self._text_tok = False
        return self._text_tok or None

    def _prepare(self, sentences, max_length):
        """One batch, ready for the GPU: ("text", truncated lines) when the library's tokenizer takes every line
        (stb_tokenizer_gpu_lines), else ("ids", CSR) from HF `tokenizers` -- the same ids either way."""
        tok = self.text_tokenizer() if max_length is not None else None
        if tok is not None:
            texts = self.truncated(sentences, max_length)
            if len(texts) and tok.gpu_lines(texts).all():
                return "text", texts
        return "ids", self.tokenize(sentences, max_length)

    def _embed_prepared(self, item, max_length, append_to):
        kind, data = item
        table = self.table()
        if kind == "text":
            return capi.embed_text(self.ctx, self.text_tokenizer(), table, data, max_length, out=append_to is None,
                                   append_to=append_to)
        offsets, ids = data
        return capi.embed(self.ctx, table, offsets, ids, out=append_to is None, append_to=append_to)

    def embed_batch(self, sentences, max_length, append_to: capi.Corpus | None = None):
        """encode_with_args for one batch, without the producer thread: rows, or None with append_to."""
        return self._embed_prepared(self._prepare(sentences, max_length), max_length, append_to)

    # -- encode_with_args(&sentences, max_length, batch_size) -> Vec<Vec<f32>> -------------------------
    def encode_with_args(self, sentences, max_length=512, batch_size=1024, append_to: capi.Corpus | None = None):
        """Batches are prepared on a producer thread while the previous batch is pooled on the GPU.  A batch
        whose every line the library's tokenizer takes is tokenised on the GPU (stb_embed_text); any other is
        tokenised by HF tokenizers (which releases the GIL and is itself multi-threaded), overlapping K3."""
        import queue
        import threading
        out = [] if append_to is None else None
        self.table()
        starts = list(range(0, len(sentences), batch_size))
        if not starts:
            return None if append_to is not None else np.zeros((0, capi.STB_DIM), dtype=np.float32)
        q: "queue.Queue" = queue.Queue(maxsize=2)

        def producer():
            try:
                for b in starts:
                    q.put(self._prepare(sentences[b:b + batch_size], max_length))
            except BaseException as e:          # surface tokenizer failures on the consumer side
                q.put(e)

        t = threading.Thread(target=producer, daemon=True)
        t.start()
        for _ in starts:
            item = q.get()
            if isinstance(item, BaseException):
                raise item
            res = self._embed_prepared(item, max_length, append_to)
            if out is not None:
                out.append(res)
        t.join()
        if append_to is not None:
            return None
        return np.concatenate(out) if out else np.zeros((0, capi.STB_DIM), dtype=np.float32)

    def encode(self, sentences):
        return self.encode_with_args(sentences, 512, 1024)            # model2vec-rs defaults

    def encode_single(self, sentence: str) -> np.ndarray:
        return self.encode([sentence])[0]
