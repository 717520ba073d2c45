"""The state of the candidate copies (the 16-bit shadow and the q8 copy) across one scripted sequence of calls, on
a device corpus and on a host-rows corpus.  After every step the test records the call's status, the kernels it
launched, the corpus's rows, tier_stats (tries, proven, built rows per tier) and the rows each copy covers
(stb_debug_corpus_copy), and compares the record with the pinned one below.  Every copy that is usable must
also be byte-equal, over the rows it covers, to a fresh build of those rows on a device corpus.

The sequence: append, prepare the q8 copy, append behind its prefix, two searches (the first one extends the
prefix), prepare the shadow, an update with a row that cannot be normalised (both copies marked bad), a search
(f32 rows), a K2 batch (its bad shadow sends it to K1), a removal (the bad copies are dropped; on a host-rows
corpus the q8 copy is built again at once), a K2 batch on the q8 route (the device corpus's q8 copy built again),
an append, the shadow prepared again, a removal that recounts both prefixes and pads the shadow's last tile, a
search (the q8 prefix extended) and a clear."""
import numpy as np
import pytest

import oracle
from conftest import unit_rows
from semtools_b200 import capi

pytestmark = pytest.mark.gpu

Q8_COPIES = (capi.STB_COPY_Q8_CODES, capi.STB_COPY_Q8_SCALES, capi.STB_COPY_Q8_PLANE, capi.STB_COPY_Q8_SR)
BAD_ROW = 100


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def fresh_copies_match(ctx, c, model, cov_q8, cov_h16, st):
    """each usable copy (built rows == covered rows) equals a fresh build of the rows it covers"""
    for cov, usable, whats in ((cov_q8, st["q8"]["built_rows"] == cov_q8, Q8_COPIES),
                               (cov_h16, st["h16"]["built_rows"] == cov_h16, (capi.STB_COPY_H16_TILES,))):
        if not cov or not usable:
            continue
        f = capi.Corpus(ctx, cov)
        f.append(model[:cov])
        f.prepare(3)
        for w in whats:
            n = (cov + 255) // 256 if w == capi.STB_COPY_H16_TILES else cov
            assert np.array_equal(bits(c.debug_copy(w, 0, n)[0]), bits(f.debug_copy(w, 0, n)[0])), w
        f.close()


def run_sequence(ctx, host):
    """Runs the sequence on a fresh corpus; returns one record per step:
    [step, status, kernels launched, rows, tries[f32, h16, q8], proven[...], built rows[h16, q8], covered[q8, h16]]
    (the status's message follows it when it is not STB_OK; the K2 route ends the q8-route batch's record)."""
    rng = np.random.default_rng(2024)
    rows = unit_rows(rng, 36_000)
    qs = np.ascontiguousarray(np.concatenate([unit_rows(rng, 4), rows[[7, 20_000, 33_500]] + np.float32(1e-3) * unit_rows(rng, 3)]))
    bad = (rows[BAD_ROW] * np.float32(1e-25))[None]                    # its fp32 squared norm underflows
    model = np.zeros((0, 256), np.float32)
    c = capi.Corpus.in_host_memory(ctx, 1024) if host else capi.Corpus(ctx, 1024)
    records = []

    def search(q):
        r, d = oracle.search_rows(model, q, top_k=10)
        hits = c.search(q, top_k=10)
        assert hits["row"].tolist() == [int(x) for x in r]
        assert np.array_equal(hits["distance"], np.asarray(d, dtype=np.float64))

    def batch():
        for q, hits in zip(qs, c.search_batch(qs, top_k=10)):
            r, d = oracle.search_rows(model, q, top_k=10)
            assert hits["row"].tolist() == [int(x) for x in r]
            assert np.array_equal(hits["distance"], np.asarray(d, dtype=np.float64))

    def step(name, fn):
        nonlocal model
        before = ctx.counters()["kernel_launches"]
        rec = [name]
        try:
            out = fn()
            if isinstance(out, np.ndarray):
                model = out
                out = None
            rec += [capi.STB_OK]
        except capi.StbError as e:
            out = None
            rec += [e.status, str(e)]
        rec += [ctx.counters()["kernel_launches"] - before, len(c)]
        assert len(c) == len(model)
        st = c.tier_stats()
        cov_q8 = c.debug_copy(capi.STB_COPY_Q8_SCALES, 0, 0)[1]
        cov_h16 = c.debug_copy(capi.STB_COPY_H16_TILES, 0, 0)[1]
        rec += [[st[t]["tries"] for t in ("f32", "h16", "q8")], [st[t]["proven"] for t in ("f32", "h16", "q8")],
                [st["h16"]["built_rows"], st["q8"]["built_rows"]], [cov_q8, cov_h16]]
        if out is not None:
            rec.append(out)
        records.append(rec)
        fresh_copies_match(ctx, c, model, cov_q8, cov_h16, st)

    def append(a, b):
        c.append(rows[a:b])
        return np.concatenate([model, rows[a:b]])

    def update_bad():
        c.update(np.array([BAD_ROW], dtype=np.uint64), bad)
        m = model.copy()
        m[BAD_ROW] = bad[0]
        return m

    def remove(ranges):
        c.remove(np.asarray(ranges, dtype=np.uint64))
        keep = np.ones(len(model), dtype=bool)
        for b, e in ranges:
            keep[b:e] = False
        return np.ascontiguousarray(model[keep])

    def no_shadow_batch():
        with ctx.batch_no_shadow():
            batch()
        return ctx.batch_last()["route"]

    step("append", lambda: append(0, 33_000))
    step("prepare_q8", lambda: c.prepare(1))
    step("append_behind_prefix", lambda: append(33_000, 34_234))
    step("search_extends", lambda: search(qs[0]))
    step("search_again", lambda: search(qs[4]))
    step("prepare_h16", lambda: c.prepare(2))
    step("update_bad_row", update_bad)
    step("search_f32", lambda: search(qs[5]))
    step("batch_bad_shadow", batch)
    step("remove_drops_bad", lambda: remove([(50, 150), (20_000, 20_100)]))
    step("batch_q8_route", no_shadow_batch)
    step("append_more", lambda: append(34_234, 35_000))
    step("prepare_h16_again", lambda: c.prepare(2))
    step("remove_recounts", lambda: remove([(1_000, 1_100), (len(model) - 300, len(model) - 250)]))
    step("search_after_remove", lambda: search(qs[6]))
    step("clear", lambda: (c.clear(), np.zeros((0, 256), np.float32))[1])
    c.close()
    return records


# recorded on an H100 80GB HBM3; the library before the copies had one owner records the same
EXPECTED = {
    "device": [
        ["append", 0, 0, 33000, [0, 0, 0], [0, 0, 0], [0, 0], [0, 0]],
        ["prepare_q8", 0, 1, 33000, [0, 0, 0], [0, 0, 0], [0, 33000], [33000, 0]],
        ["append_behind_prefix", 0, 0, 34234, [0, 0, 0], [0, 0, 0], [0, 33000], [33000, 0]],
        ["search_extends", 0, 2, 34234, [0, 0, 1], [0, 0, 1], [0, 34234], [34234, 0]],
        ["search_again", 0, 1, 34234, [0, 0, 2], [0, 0, 2], [0, 34234], [34234, 0]],
        ["prepare_h16", 0, 1, 34234, [0, 0, 2], [0, 0, 2], [34234, 34234], [34234, 34234]],
        ["update_bad_row", 0, 1, 34234, [0, 0, 0], [0, 0, 0], [0, 0], [34234, 34234]],
        ["search_f32", 0, 1, 34234, [1, 0, 0], [1, 0, 0], [0, 0], [34234, 34234]],
        ["batch_bad_shadow", 0, 7, 34234, [8, 0, 0], [8, 0, 0], [0, 0], [34234, 34234]],
        ["remove_drops_bad", 0, 2, 34034, [0, 0, 0], [0, 0, 0], [0, 0], [0, 0]],
        ["batch_q8_route", 0, 6, 34034, [0, 0, 0], [0, 0, 0], [0, 34034], [34034, 0], 7],
        ["append_more", 0, 0, 34800, [0, 0, 0], [0, 0, 0], [0, 34034], [34034, 0]],
        ["prepare_h16_again", 0, 1, 34800, [0, 0, 0], [0, 0, 0], [34800, 34034], [34034, 34800]],
        ["remove_recounts", 0, 3, 34650, [0, 0, 0], [0, 0, 0], [34650, 33934], [33934, 34650]],
        ["search_after_remove", 0, 2, 34650, [0, 0, 1], [0, 0, 1], [34650, 34650], [34650, 34650]],
        ["clear", 0, 0, 0, [0, 0, 0], [0, 0, 0], [0, 0], [0, 0]],
    ],
    "host": [
        ["append", 0, 1, 33000, [0, 0, 0], [0, 0, 0], [0, 33000], [33000, 0]],
        ["prepare_q8", 0, 0, 33000, [0, 0, 0], [0, 0, 0], [0, 33000], [33000, 0]],
        ["append_behind_prefix", 0, 1, 34234, [0, 0, 0], [0, 0, 0], [0, 34234], [34234, 0]],
        ["search_extends", 0, 1, 34234, [0, 0, 1], [0, 0, 1], [0, 34234], [34234, 0]],
        ["search_again", 0, 1, 34234, [0, 0, 2], [0, 0, 2], [0, 34234], [34234, 0]],
        ["prepare_h16", 0, 1, 34234, [0, 0, 2], [0, 0, 2], [34234, 34234], [34234, 34234]],
        ["update_bad_row", 0, 1, 34234, [0, 0, 0], [0, 0, 0], [0, 0], [34234, 34234]],
        ["search_f32", 0, 4, 34234, [0, 0, 0], [0, 0, 0], [0, 0], [34234, 34234]],
        ["batch_bad_shadow", 0, 28, 34234, [0, 0, 0], [0, 0, 0], [0, 0], [34234, 34234]],
        ["remove_drops_bad", 0, 3, 34034, [0, 0, 0], [0, 0, 0], [0, 34034], [34034, 0]],
        ["batch_q8_route", 0, 5, 34034, [0, 0, 0], [0, 0, 0], [0, 34034], [34034, 0], 7],
        ["append_more", 0, 1, 34800, [0, 0, 0], [0, 0, 0], [0, 34800], [34800, 0]],
        ["prepare_h16_again", 0, 1, 34800, [0, 0, 0], [0, 0, 0], [34800, 34800], [34800, 34800]],
        ["remove_recounts", 0, 3, 34650, [0, 0, 0], [0, 0, 0], [34650, 34650], [34650, 34650]],
        ["search_after_remove", 0, 1, 34650, [0, 0, 1], [0, 0, 1], [34650, 34650], [34650, 34650]],
        ["clear", 0, 0, 0, [0, 0, 0], [0, 0, 0], [0, 0], [0, 0]],
    ],
}


@pytest.mark.parametrize("kind", ["device", "host"])
def test_copy_state_across_a_sequence(ctx, kind):
    got = run_sequence(ctx, kind == "host")
    exp = EXPECTED[kind]
    assert [r[0] for r in got] == [r[0] for r in exp]
    for g, e in zip(got, exp):
        assert g == e, (g, e)
