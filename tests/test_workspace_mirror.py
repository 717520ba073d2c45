"""CPU suite: an open workspace Store keeps its GPU mirror current with in-place calls.  capi.Corpus is
replaced by a recording stub (a numpy matrix), so this checks what the store sends, not the GPU."""
import numpy as np
import pytest

from conftest import unit_rows
from semtools_b200 import capi
from semtools_b200 import workspace as ws


class RecordingCorpus:
    """Stands in for capi.Corpus: a numpy matrix plus the list of calls it received."""

    def __init__(self, ctx, capacity_rows=1024, row_base=0):
        self.rows = np.zeros((0, 256), dtype=np.float32)
        self.calls = []
        self.fail = None

    def __len__(self):
        return len(self.rows)

    def append(self, rows):
        self.calls.append(("append", len(rows)))
        self.rows = np.concatenate([self.rows, np.asarray(rows, dtype=np.float32)])

    def update(self, idx, rows):
        self.calls.append(("update", np.array(idx), np.array(rows)))
        if self.fail == "update":
            raise capi.StbError(capi.STB_ERR_STATE, "injected")
        self.rows[np.asarray(idx, dtype=np.int64)] = rows

    def remove(self, ranges):
        self.calls.append(("remove", np.array(ranges)))
        keep = np.ones(len(self.rows), dtype=bool)
        for b, e in np.asarray(ranges, dtype=np.int64):
            keep[b:e] = False
        self.rows = self.rows[keep]

    def search(self, q, top_k=3, max_distance=None, mode=0, row_ranges=None, cap=None):
        return np.zeros(0, dtype=capi.HIT_DTYPE)


@pytest.fixture
def store(tmp_path, monkeypatch):
    monkeypatch.setattr(ws.capi, "Corpus", RecordingCorpus)
    return ws.Store.open(str(tmp_path), ctx=object())


def lines(path, vecs, first=0):
    return [ws.LineEmbedding(path, first + i, v) for i, v in enumerate(vecs)]


def mirror_calls(store):
    return [c for c in store._corpus.calls if c[0] != "append"]


def test_patches_reach_update_with_the_last_value_of_the_batch(store):
    rng = np.random.default_rng(0)
    a, b = unit_rows(rng, 5), unit_rows(rng, 4)
    store.upsert_line_embeddings(lines("a", a) + lines("b", b))
    store.search_line_embeddings(a[0], ["a", "b"], 3)                 # uploads rows 0..8
    mirror = store._corpus
    v1, v2, v3, c_new = unit_rows(rng, 4)
    # a:1 twice (the last value wins), b:2, and a new document that is not uploaded
    store.upsert_line_embeddings(lines("a", [v1], 1) + lines("b", [v3], 2) + lines("a", [v2], 1) + lines("c", [c_new]))
    assert store._corpus is mirror
    (kind, idx, rows), = mirror_calls(store)
    assert kind == "update" and idx.tolist() == [1, 7]
    assert np.array_equal(rows, np.stack([v2, v3]))
    assert np.array_equal(mirror.rows, np.asarray(store._emb)[:9])
    # a patch of a row that was never uploaded is never sent; the lazy append takes it
    store.upsert_line_embeddings(lines("c", [v1]))
    assert len(mirror_calls(store)) == 1
    store.search_line_embeddings(a[0], ["a"], 3)
    assert mirror.calls[-1] == ("append", 1)
    assert np.array_equal(mirror.rows, np.asarray(store._emb))


def test_deletions_reach_remove_as_ranges_of_the_uploaded_prefix(store):
    rng = np.random.default_rng(1)
    docs = {p: unit_rows(rng, n) for p, n in (("a", 3), ("b", 4), ("c", 2), ("d", 5))}
    store.upsert_line_embeddings([le for p, v in docs.items() for le in lines(p, v)])
    store.search_line_embeddings(docs["a"][0], ["a"], 3)              # rows 0..13 uploaded
    mirror = store._corpus
    store.upsert_line_embeddings(lines("e", unit_rows(rng, 3)) + lines("b", unit_rows(rng, 2), 10))   # rows 14..18, not uploaded
    store.delete_documents(["b", "d", "e"])
    assert store._corpus is mirror
    (kind, ranges), = mirror_calls(store)
    assert kind == "remove" and ranges.tolist() == [[3, 7], [9, 14]]
    assert store._corpus_n == 5 and np.array_equal(mirror.rows, np.asarray(store._emb)[:5])
    store.search_line_embeddings(docs["a"][0], ["a", "c"], 3)
    assert np.array_equal(mirror.rows, np.asarray(store._emb))
    # only rows that were never uploaded: no call
    store.upsert_line_embeddings(lines("f", unit_rows(rng, 2)))
    store.delete_documents(["f"])
    assert len(mirror_calls(store)) == 1 and store._corpus is mirror


def test_a_failed_call_drops_the_mirror(store):
    rng = np.random.default_rng(2)
    store.upsert_line_embeddings(lines("a", unit_rows(rng, 4)))
    store.search_line_embeddings(unit_rows(rng, 1)[0], ["a"], 3)
    store._corpus.fail = "update"
    store.upsert_line_embeddings(lines("a", unit_rows(rng, 1)))
    assert store._corpus is None
    store.search_line_embeddings(unit_rows(rng, 1)[0], ["a"], 3)      # uploads everything again
    assert np.array_equal(store._corpus.rows, np.asarray(store._emb))
