"""Host-side mirror of the reference's search interface on top of the C ABI.

Names and argument meaning follow reference src/search/mod.rs:
  Document        :18-22   (embeddings live in HBM, not in a Vec<Vec<f32>>)
  SearchConfig    :32-38
  SearchResult    :40-47
  search_documents:77-120  -> Searcher.search_documents
and src/workspace/store.rs:
  RankedLine      :91-96
  Store::search_line_embeddings :481-546 -> Searcher.search_line_embeddings

Everything numeric happens in libsemtools_b200.so; this file only keeps the
row <-> (document, line) bookkeeping and builds the context windows.
"""
from __future__ import annotations

from bisect import bisect_right
from dataclasses import dataclass, field

import numpy as np

from . import capi


@dataclass
class SearchConfig:
    """reference src/search/mod.rs:32-38; CLI defaults 3/3/None/false
    (src/bin/semtools.rs:61-74)."""
    n_lines: int = 3
    top_k: int = 3
    max_distance: float | None = None
    ignore_case: bool = False


@dataclass
class Document:
    """reference src/search/mod.rs:18-22.  `row_start` is the document's first
    row in the corpus matrix; its embeddings are rows [row_start, row_start+len(lines))."""
    filename: str
    lines: list
    row_start: int = 0


@dataclass
class SearchResult:
    """reference src/search/mod.rs:40-47."""
    filename: str
    lines: list
    start: int
    end: int
    match_line: int
    distance: float


@dataclass
class RankedLine:
    """reference src/workspace/store.rs:91-96 (distance is f32 there)."""
    path: str
    line_number: int
    distance: float


@dataclass
class Searcher:
    """Owns one context + corpus; documents are appended in order, so global row
    order equals the reference's (document, line) iteration order."""
    ctx: capi.Context
    corpus: capi.Corpus
    documents: list = field(default_factory=list)
    _starts: list = field(default_factory=list)

    @classmethod
    def create(cls, device: int = 0, capacity_rows: int = 1024, stream: int | None = None):
        ctx = capi.Context(device, stream)
        return cls(ctx, capi.Corpus(ctx, capacity_rows))

    # -- create_document_from_content (src/search/mod.rs:49-75) minus tokenisation
    def add_document_embeddings(self, filename: str, lines: list, embeddings: np.ndarray):
        """Append a document whose line embeddings were computed elsewhere."""
        if len(lines) == 0:
            return None                      # :57-59 empty content -> None
        emb = np.ascontiguousarray(embeddings, dtype=np.float32)
        assert emb.shape == (len(lines), capi.STB_DIM)
        doc = Document(filename, list(lines), len(self.corpus))
        self.corpus.append(emb)
        self.documents.append(doc)
        self._starts.append(doc.row_start)
        return doc

    def add_document_lines(self, filename: str, lines: list, model, emb_lines: list):
        """Same, with the model embedding emb_lines straight into HBM (encode_with_args(lines, Some(2048), 16384)
        at :69; StaticModel.embed_batch picks the GPU tokenizer or HF tokenizers)."""
        if len(lines) == 0:
            return None
        doc = Document(filename, list(lines), len(self.corpus))
        model.embed_batch(emb_lines, 2048, append_to=self.corpus)
        self.documents.append(doc)
        self._starts.append(doc.row_start)
        return doc

    def _locate(self, row: int):
        d = bisect_right(self._starts, row) - 1
        doc = self.documents[d]
        return doc, row - doc.row_start

    # -- search_documents (src/search/mod.rs:77-120)
    def search_documents(self, query_embedding, config: SearchConfig):
        hits = self.corpus.search(query_embedding, config.top_k, config.max_distance,
                                  capi.STB_MODE_SEARCH_DOCUMENTS)
        return self._results(hits, config)

    def _results(self, hits, config: SearchConfig):
        """SearchResults with their context windows (:88-119) for hits ordered by (distance, row)."""
        out = []
        for h in hits:
            doc, idx = self._locate(int(h["row"]))
            start = max(0, idx - config.n_lines)                      # :90
            end = min(len(doc.lines), idx + config.n_lines + 1)       # :91
            out.append(SearchResult(doc.filename, doc.lines[start:end], start, end, idx,
                                    float(h["distance"])))
        return out

    # -- search_documents for a batch of queries: element i equals search_documents(query_embeddings[i], config)
    def search_documents_batch(self, query_embeddings, config: SearchConfig):
        q = np.ascontiguousarray(query_embeddings, dtype=np.float32).reshape(-1, capi.STB_DIM)
        if config.max_distance is None:
            hits = self.corpus.search_batch(q, config.top_k)
        else:
            hits = self.corpus.search_batch_threshold(q, config.max_distance)
        return [self._results(h, config) for h in hits]

    # -- Store::search_line_embeddings (src/workspace/store.rs:481-546)
    def search_line_embeddings(self, query_vec, subset_paths, top_k: int, max_distance=None):
        if len(subset_paths) == 0 or top_k == 0:                      # :489-491
            return []
        wanted = set(subset_paths)
        ranges = [(d.row_start, d.row_start + len(d.lines)) for d in self.documents
                  if d.filename in wanted]
        if not ranges:
            return []
        hits = self.corpus.search(query_vec, top_k, max_distance, capi.STB_MODE_STORE_QUERY,
                                  row_ranges=np.array(ranges, dtype=np.uint64))
        out = []
        for h in hits:
            doc, idx = self._locate(int(h["row"]))
            out.append(RankedLine(doc.filename, idx, float(np.float32(h["distance"]))))   # :531 f32
        return out
