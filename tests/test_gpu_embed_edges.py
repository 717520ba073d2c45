"""GPU: K3 embed (csrc/embed_pool.cu) at its edges, against the oracle's restatement of pool_ids.

The reference is oracle.embed_csr / oracle.pool_ids: C built with -ffp-contract=off, f32 operations in
the kernel's order.  Outputs are compared as u32 bit patterns.  The one exception is NaN: a NaN component
must be NaN exactly where the oracle's is, but its payload is not compared (the GPU writes the canonical
quiet NaN, x86 propagates the payload of a NaN input).

Covered here: every table option (weights and mapping shorter than the vocabulary, many-to-one mapping,
mapping rows outside the table) through all four ways of calling the kernel; line lengths around the
4-token gather depth, the 32-lane warp and far past the resident warps; subnormal, overflowing,
underflowing, cancelling, NaN and infinite values; a table larger than 2 GiB; appends into corpora that
grow, have their reduced-width copies built or carry a live IVF-PQ index; and the isolation of
stb_embed_dev's sticky range flag from every other call on the context.
"""
import ctypes as C

import numpy as np
import pytest

import oracle
from conftest import unit_rows
from semtools_b200 import capi

pytestmark = pytest.mark.gpu

D = 256
LAZY_ROWS = 32768              # rows from which the second search builds the q8 copy by itself
COPIES = (capi.STB_COPY_Q8_CODES, capi.STB_COPY_Q8_SCALES, capi.STB_COPY_Q8_PLANE, capi.STB_COPY_Q8_SR,
          capi.STB_COPY_H16_TILES)


@pytest.fixture(scope="module")
def torch():
    return pytest.importorskip("torch")


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def assert_pool_equal(got, want, what=""):
    """Bit-identical, except that NaN payloads are not compared (NaN positions are)."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape, what
    gn, wn = np.isnan(got), np.isnan(want)
    assert np.array_equal(gn, wn), f"{what}: NaN at {np.argwhere(gn != wn)[:5].tolist()}"
    g, w = bits(got), bits(want)
    bad = (g != w) & ~wn
    assert not bad.any(), f"{what}: {int(bad.sum())} components differ, first at {np.argwhere(bad)[:5].tolist()}"


def csr(lines):
    lens = [len(x) for x in lines]
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    ids = np.concatenate([np.asarray(x, np.uint32) for x in lines]) if sum(lens) else np.zeros(0, np.uint32)
    return offsets, ids.astype(np.uint32)


def embed_dev_out(torch, ctx, t, offsets, ids):
    """stb_embed_dev on device copies of the CSR; returns (rows, status error or None)."""
    dev = torch.device("cuda:0")
    n = offsets.size - 1
    off_d = torch.from_numpy(offsets.astype(np.uint64).view(np.int64)).to(dev)
    ids_d = torch.from_numpy((ids if ids.size else np.zeros(1, np.uint32)).astype(np.uint32).view(np.int32)).to(dev)
    out_d = torch.full((max(n, 1), D), float("nan"), dtype=torch.float32, device=dev)
    torch.cuda.synchronize()
    capi.embed_dev(ctx, t, off_d.data_ptr(), ids_d.data_ptr(), n, out_d.data_ptr())
    err = None
    try:
        capi.embed_status(ctx)
    except capi.StbError as e:
        err = e.status
    return out_d[:n].cpu().numpy(), err


def all_forms(torch, ctx, t, offsets, ids):
    """The four ways to run K3 -- stb_embed into `out`, into a corpus, into both, stb_embed_dev -- must give
    the same bits (the kernel and its launch are the same); returns that output."""
    n = offsets.size - 1
    a = capi.embed(ctx, t, offsets, ids)
    c1 = capi.Corpus(ctx, max(n, 1))
    assert capi.embed(ctx, t, offsets, ids, out=False, append_to=c1) is None
    c2 = capi.Corpus(ctx, max(n, 1))
    b = capi.embed(ctx, t, offsets, ids, out=True, append_to=c2)
    d, err = embed_dev_out(torch, ctx, t, offsets, ids)
    assert err is None
    assert len(c1) == n and len(c2) == n
    for name, x in (("append_to", c1.read()), ("out+append_to", b), ("append_to of both", c2.read()), ("dev", d)):
        assert np.array_equal(bits(x), bits(a)), name
    c1.close(); c2.close()
    return a


def check(torch, ctx, E, offsets, ids, weights=None, mapping=None, normalize=True, what=""):
    t = capi.Table(ctx, E, weights, mapping, normalize=normalize)
    try:
        got = all_forms(torch, ctx, t, offsets, ids)
    finally:
        t.close()
    want = oracle.embed_csr(E, offsets, ids, weights, mapping, normalize)
    assert_pool_equal(got, want, what)
    return got, want


def random_lines(rng, n_lines, V, max_len=40, min_len=0):
    """min_len=1 for corpus rows: an empty line pools to a zero row, which the reduced-width copies refuse."""
    lens = rng.integers(max(min_len, 1), max_len, n_lines)
    if min_len == 0:
        lens[rng.random(n_lines) < 0.05] = 0
    return csr([rng.integers(0, V, l) for l in lens])


# ----------------------------------------------------------------------------------- table options ---
def table_options(rng, V):
    """Weights 0.6 V long with 0, -0.0, negative, subnormal and 1e30 entries; a many-to-one mapping
    0.5 V long into the first 600 rows."""
    w = rng.uniform(0.2, 2.0, int(0.6 * V)).astype(np.float32)
    special = rng.choice(w.size, 60, replace=False)
    w[special[0:12]] = 0.0
    w[special[12:24]] = -0.0
    w[special[24:36]] = -rng.uniform(0.1, 3.0, 12)
    w[special[36:48]] = np.float32(3e-39)                      # subnormal weight
    w[special[48:60]] = np.float32(1e30)
    m = rng.integers(0, 600, V // 2).astype(np.uint32)
    return w, m


@pytest.mark.parametrize("normalize", [True, False], ids=["norm", "nonorm"])
@pytest.mark.parametrize("option", ["plain", "short_weights", "short_mapping", "both"])
def test_table_options_match_the_oracle_through_every_entry_point(ctx, torch, option, normalize):
    rng = np.random.default_rng(0xE3 + len(option) + normalize)
    V = 5000
    E = (rng.standard_normal((V, D)) * 0.1).astype(np.float32)
    w, m = table_options(rng, V)
    w = w if option in ("short_weights", "both") else None
    m = m if option in ("short_mapping", "both") else None
    offsets, ids = random_lines(rng, 3000, V)
    # every special weight and both sides of the short arrays' ends are used
    extra = [[int(x)] for x in range(2400, 2600)] + [[int(x)] for x in range(2950, 3050)] + [[V - 1, 0]]
    if w is not None:
        extra += [[int(x), int(x) + 1] for x in np.flatnonzero((w == 0) | (w < 0) | (w < 1e-30) | (w > 1e29))]
    o2, i2 = csr(extra)
    offsets = np.concatenate([offsets, offsets[-1] + o2[1:]]).astype(np.uint64)
    ids = np.concatenate([ids, i2]).astype(np.uint32)
    check(torch, ctx, E, offsets, ids, w, m, normalize, f"{option}/{normalize}")


@pytest.mark.parametrize("normalize", [True, False], ids=["norm", "nonorm"])
def test_mapping_outside_the_table_is_a_range_error(ctx, torch, normalize):
    rng = np.random.default_rng(41)
    V = 300
    E = (rng.standard_normal((V, D)) * 0.1).astype(np.float32)
    m = rng.integers(0, V, 100).astype(np.uint32)
    m[37] = V                                                   # first row past the end
    m[38] = 0xFFFFFFFF
    t = capi.Table(ctx, E, mapping=m, normalize=normalize)
    good_off, good_ids = csr([[1, 2, 3], [150, 299]])
    for bad in (37, 38):
        off, ids = csr([[1, 2], [5, bad, 7], [9]])
        with pytest.raises(IndexError):
            oracle.embed_csr(E, off, ids, mapping=m)
        c = capi.Corpus(ctx, 4)
        capi.embed(ctx, t, good_off, good_ids, out=False, append_to=c)
        before = c.read()
        for kw in (dict(), dict(out=False, append_to=c), dict(append_to=c)):
            with pytest.raises(capi.StbError) as e:
                capi.embed(ctx, t, off, ids, **kw)
            assert e.value.status == capi.STB_ERR_RANGE
        assert len(c) == 2 and np.array_equal(bits(c.read()), bits(before))  # nothing appended
        _, err = embed_dev_out(torch, ctx, t, off, ids)
        assert err == capi.STB_ERR_RANGE                       # the device form raises the flag
        capi.embed_status(ctx)                                  # ... which the status call cleared
        c.close()
    # a token id >= V that the mapping does not cover passes through unchanged, and is out of range too
    off, ids = csr([[V + 3]])
    with pytest.raises(capi.StbError) as e:
        capi.embed(ctx, t, off, ids)
    assert e.value.status == capi.STB_ERR_RANGE
    t.close()


# ------------------------------------------------------------------------------------- line shapes ---
SHAPE_LENGTHS = [0, 1, 2, 3, 4, 5, 7, 8, 9, 31, 32, 33, 63, 64, 65, 2047, 2048, 2049, 70000]


@pytest.mark.parametrize("normalize", [True, False], ids=["norm", "nonorm"])
def test_line_lengths_around_the_gather_depth_and_the_warp(ctx, torch, normalize):
    rng = np.random.default_rng(0x51 + normalize)
    V = 20000
    E = (rng.standard_normal((V, D)) * 0.1).astype(np.float32)
    w = rng.uniform(0.1, 2.0, V).astype(np.float32)
    lens = list(SHAPE_LENGTHS)
    rng.shuffle(lens)
    lens = [0] + lens + [0]                                     # empty lines at both ends
    offsets, ids = csr([rng.integers(0, V, l) for l in lens])
    got, _ = check(torch, ctx, E, offsets, ids, w, None, normalize, "shapes")
    assert not bits(got[0]).any() and not bits(got[-1]).any()  # empty line: +0 everywhere


def test_single_line_batches(ctx, torch):
    rng = np.random.default_rng(52)
    V = 1000
    E = (rng.standard_normal((V, D)) * 0.1).astype(np.float32)
    for l in (0, 1, 4, 33, 2049):
        offsets, ids = csr([rng.integers(0, V, l)])
        got, _ = check(torch, ctx, E, offsets, ids, what=f"n_lines=1 len={l}")
        assert np.array_equal(bits(got[0]), bits(oracle.pool_ids(E, ids)))


def test_many_more_lines_than_resident_warps(ctx, torch):
    """200k short lines: the grid (sm_count x occupancy x 8 warps, ~3k on an H100) strides many times."""
    rng = np.random.default_rng(53)
    V = 4000
    E = (rng.standard_normal((V, D)) * 0.1).astype(np.float32)
    n = 200_000
    lens = rng.integers(0, 7, n)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    ids = rng.integers(0, V, int(offsets[-1])).astype(np.uint32)
    check(torch, ctx, E, offsets, ids, what="200k lines")


def test_batch_of_only_empty_lines(ctx, torch):
    E = np.ones((10, D), np.float32)
    offsets = np.zeros(1001, np.uint64)
    for normalize in (True, False):
        got, _ = check(torch, ctx, E, offsets, np.zeros(0, np.uint32), normalize=normalize, what="empty")
        assert not bits(got).any()


# ------------------------------------------------------------------------------------- value edges ---
def edge_table(rng):
    """Rows by kind; returns (E, weights, kinds) where kinds maps a name to its row ids."""
    rows, kinds = [], {}

    def add(name, block):
        kinds[name] = list(range(len(rows), len(rows) + len(block)))
        rows.extend(np.asarray(block, np.float32))

    tiny = np.float32(1.4e-45)
    add("normal", rng.standard_normal((40, D)) * 0.1)
    add("subnormal", rng.integers(-2000, 2000, (6, D)) * tiny)          # every value subnormal (or 0)
    add("small", rng.standard_normal((6, D)) * 1e-20)                   # x weight 1e-20 -> subnormal products
    add("underflow", rng.standard_normal((6, D)) * 1e-25)               # squares of the mean underflow to 0
    add("big", rng.standard_normal((6, D)) * 1e20)                      # squares overflow, the sum does not
    huge = rng.standard_normal((6, D)) * 1e37
    huge[:, :8] = 3.0e38                                                # two of these overflow the sum
    add("huge", huge)
    half_zero = rng.standard_normal((2, D)) * 0.1
    half_zero[:, ::2] = 0.0                                             # x an infinite weight -> NaN
    add("half_zero", half_zero)
    r = rng.standard_normal((4, D)) * 0.1
    add("pos", r)
    add("neg", -r)                                                      # row i + its negation = 0 exactly
    special = (rng.standard_normal((8, D)) * 0.1).astype(np.float32)     # f32: the NaN payloads stay as set
    nan_bits = np.array([0x7FC00000, 0xFFC00000, 0x7FC01234, 0x7F800001], np.uint32).view(np.float32)
    for i in range(8):
        cols = rng.choice(D, 5, replace=False)
        if i < 4:
            special[i, cols] = nan_bits[i]
        else:
            special[i, cols] = np.inf if i % 2 else -np.inf
    add("special", special)
    E = np.ascontiguousarray(np.stack(rows), np.float32)
    V = E.shape[0]
    w = np.ones(V + 20, np.float32)
    w[kinds["small"]] = 1e-20
    w[kinds["normal"][:4]] = nan_bits[:4]
    w[kinds["normal"][4:6]] = [np.inf, -np.inf]
    w[kinds["normal"][6:8]] = np.float32(1e-44)                         # subnormal weight
    w[kinds["half_zero"]] = [np.inf, -np.inf]
    return E, w, kinds


def subnormal(x):
    return (np.abs(x) > 0) & (np.abs(x) < np.finfo(np.float32).tiny)


@pytest.mark.parametrize("normalize", [True, False], ids=["norm", "nonorm"])
def test_value_edges(ctx, torch, normalize):
    rng = np.random.default_rng(0x7A + normalize)
    E, w, kinds = edge_table(rng)
    V = E.shape[0]
    K = kinds
    designed = {
        "subnormal": [K["subnormal"][0]],
        "subnormal_mix": K["subnormal"][:4] + K["normal"][10:12],
        "small_products": K["small"][:3],
        "underflow": K["underflow"][:2],
        "big": K["big"][:3],
        "huge_sum": [K["huge"][0], K["huge"][1]],
        "huge_one": [K["huge"][2]],
        "cancel": [K["pos"][0], K["neg"][0]],
        "cancel_mean": [K["pos"][1], K["neg"][1], K["pos"][1], K["neg"][1]],
        "nan_row": [K["special"][2], K["normal"][20]],
        "inf_row": [K["special"][4]],
        "inf_minus_inf": [K["special"][5], K["special"][4]],
        "nan_weight": [K["normal"][2], K["normal"][21]],
        "inf_weight": [K["normal"][4]],
        "inf_weight_zero_entry": [K["half_zero"][0], K["neg"][2]],
        "subnormal_weight": [K["normal"][6]],
    }
    names = list(designed)
    lines = [designed[k] for k in names]
    # plus random mixtures of every kind
    for _ in range(3000):
        lines.append(rng.integers(0, V, rng.integers(1, 7)).tolist())
    offsets, ids = csr(lines)
    for weights in (None, w):
        got, want = check(torch, ctx, E, offsets, ids, weights, None, normalize, f"edges w={weights is not None}")
        row = {k: got[i] for i, k in enumerate(names)}
        assert not bits(row["cancel"]).any() and not bits(row["cancel_mean"]).any()   # +0, never -0
        if not normalize:
            assert subnormal(row["subnormal"]).any()           # a flush-to-zero build would fail here
            if weights is not None:
                assert subnormal(row["small_products"]).any()
            assert np.isinf(row["huge_sum"]).any()
        else:
            assert np.isnan(row["huge_sum"]).any()             # inf / inf
            assert (row["big"] == 0).all()                     # finite / inf norm = +-0
            # the squares underflow to 0, so the norm is the 1e-12 clamp: components ~1e-13, not ~0.1
            assert np.isfinite(row["underflow"]).all() and 0 < np.abs(row["underflow"]).max() < 1e-10
            assert np.isnan(row["inf_row"]).any()
        assert np.isnan(row["nan_row"]).any()
        if weights is not None:
            assert np.isnan(row["nan_weight"]).all() and np.isnan(row["inf_weight_zero_entry"]).any()
        assert np.isnan(want).any() and np.isnan(got).any()


# --------------------------------------------------------------------------------------- big table ---
def test_table_over_2_gib(ctx, torch):
    """V = 2^21 + 1000 rows (2 GiB + 1000 KiB): rows at and past 2^21 sit beyond a 32-bit byte offset."""
    rng = np.random.default_rng(0xB16)
    V = (1 << 21) + 1000
    near_top = np.arange(V - 40, V)
    near_2g = np.arange((1 << 21) - 20, (1 << 21) + 20)
    low = np.arange(0, 20)
    used = np.concatenate([low, near_2g, near_top])
    E = np.zeros((V, D), np.float32)
    E[used] = rng.standard_normal((used.size, D)).astype(np.float32)
    lines = [rng.choice(used, rng.integers(1, 9)).tolist() for _ in range(400)]
    lines += [[V - 1], [1 << 21], [(1 << 21) - 1], [V - 1, 0, 1 << 21]]
    offsets, ids = csr(lines)
    want = oracle.embed_csr(E, offsets, ids)
    t = capi.Table(ctx, E)
    del E
    try:
        got = capi.embed(ctx, t, offsets, ids)
        assert_pool_equal(got, want, "big table")
        dev, err = embed_dev_out(torch, ctx, t, offsets, ids)
        assert err is None and np.array_equal(bits(dev), bits(got))
        with pytest.raises(capi.StbError) as e:
            capi.embed(ctx, t, *csr([[V]]))
        assert e.value.status == capi.STB_ERR_RANGE
    finally:
        t.close()


# ------------------------------------------------------------------------------- corpus interplay ---
def snapshot(c):
    return [bits(c.read())] + [np.ascontiguousarray(c.debug_copy(w)[0]).view(np.uint8) for w in COPIES]


def coverage(c):
    return c.debug_copy(capi.STB_COPY_Q8_SCALES, 0, 0)[1], c.debug_copy(capi.STB_COPY_H16_TILES, 0, 0)[1]


def assert_copies_match_fresh(ctx, c, rows):
    """Every copy of c equals the one a fresh corpus of the same rows builds."""
    fresh = capi.Corpus(ctx, len(rows))
    fresh.append(rows)
    fresh.prepare(3)
    assert coverage(c) == coverage(fresh) == (len(rows), len(rows))
    for w in COPIES:
        assert np.array_equal(np.ascontiguousarray(c.debug_copy(w)[0]).view(np.uint8),
                              np.ascontiguousarray(fresh.debug_copy(w)[0]).view(np.uint8)), w
    fresh.close()


def test_append_past_capacity_keeps_the_earlier_rows(ctx):
    rng = np.random.default_rng(61)
    V = 2000
    E = (rng.standard_normal((V, D)) * 0.1).astype(np.float32)
    t = capi.Table(ctx, E)
    head = unit_rows(rng, 10)
    c = capi.Corpus(ctx, 16)
    c.append(head)
    expect = [head]
    for n_lines in (5, 100, 3000):                              # the second and third batch grow the corpus
        offsets, ids = random_lines(rng, n_lines, V, min_len=1)
        capi.embed(ctx, t, offsets, ids, out=False, append_to=c)
        expect.append(oracle.embed_csr(E, offsets, ids))
        assert np.array_equal(bits(c.read()), bits(np.concatenate(expect)))
    c.close(); t.close()


def test_append_into_a_prepared_corpus_extends_its_copies(ctx):
    rng = np.random.default_rng(62)
    V = 3000
    E = (rng.standard_normal((V, D)) * 0.1).astype(np.float32)
    t = capi.Table(ctx, E)
    n0 = 3000
    head = unit_rows(rng, n0)
    c = capi.Corpus(ctx, n0 + 100)
    c.append(head)
    c.prepare(3)
    snap = snapshot(c)
    offsets, ids = random_lines(rng, 700, V, min_len=1)
    capi.embed(ctx, t, offsets, ids, out=False, append_to=c)
    rows = np.concatenate([head, oracle.embed_csr(E, offsets, ids)])
    assert np.array_equal(bits(c.read()), bits(rows))
    assert coverage(c) == (n0, n0)                              # the copies still cover the old prefix ...
    after = snapshot(c)
    for a, b in zip(snap[1:], after[1:]):
        assert np.array_equal(a, b)                             # ... unchanged
    for q in (rows[n0 + 5], rows[17], unit_rows(rng, 1)[0]):
        want_r, want_d = oracle.search_rows(rows, q, top_k=10)
        hits = c.search(q, top_k=10)                            # extends the q8 copy over the new rows
        assert hits["row"].tolist() == [int(x) for x in want_r]
        assert np.array_equal(hits["distance"].view(np.uint64), np.asarray(want_d, np.float64).view(np.uint64))
    assert c.tier_stats()["q8"]["built_rows"] == len(rows)
    c.prepare(3)
    assert_copies_match_fresh(ctx, c, rows)
    c.close(); t.close()


def test_append_under_a_live_ivfpq_index_then_extend(ctx):
    rng = np.random.default_rng(63)
    V = 3000
    E = (rng.standard_normal((V, D)) * 0.1).astype(np.float32)
    t = capi.Table(ctx, E)
    n0 = 1500
    head = unit_rows(rng, n0)
    c = capi.Corpus(ctx, n0)
    c.append(head)
    nlist = 4
    idx = capi.IvfPq(c, nlist=nlist, train_rows=n0, iters=4)
    offsets, ids = random_lines(rng, 600, V, min_len=1)
    capi.embed(ctx, t, offsets, ids, out=False, append_to=c)
    assert idx.extend() == 600
    rows = np.concatenate([head, oracle.embed_csr(E, offsets, ids)])
    n = len(rows)
    for q in (rows[n0 + 3], rows[42], unit_rows(rng, 1)[0]):
        got, _ = idx.search(q, nprobe=nlist, top_k=10, rerank=n)
        want = c.search(q, top_k=10)
        assert np.array_equal(got, want)
        want_r, _ = oracle.search_rows(rows, q, top_k=10)
        assert got["row"].tolist() == [int(x) for x in want_r]
    idx.close(); c.close(); t.close()


def test_failed_append_leaves_the_corpus_and_its_copies_unchanged(ctx):
    rng = np.random.default_rng(64)
    V = 1000
    E = (rng.standard_normal((V, D)) * 0.1).astype(np.float32)
    t = capi.Table(ctx, E)
    c = capi.Corpus(ctx, 600)
    c.append(unit_rows(rng, 520))
    c.prepare(3)
    before = snapshot(c)
    cov = coverage(c)
    offsets, ids = random_lines(rng, 400, V, min_len=1)         # grows the corpus past its capacity
    ids[len(ids) // 2] = V
    with pytest.raises(capi.StbError) as e:
        capi.embed(ctx, t, offsets, ids, out=False, append_to=c)
    assert e.value.status == capi.STB_ERR_RANGE
    assert len(c) == 520 and coverage(c) == cov
    for a, b in zip(before, snapshot(c)):
        assert np.array_equal(a, b)
    c.close(); t.close()


# ---------------------------------------------------------------------------- range flag isolation ---
@pytest.fixture
def fresh():
    """A context of its own, so no call from another test can set or clear its flags in between."""
    c = capi.Context(0)
    c.owned = []
    yield c
    for h in reversed(c.owned):                                 # handles go before their context
        h.close()
    c.close()


def flag_setup(torch, ctx, n_rows=4096):
    rng = np.random.default_rng(71)
    V = 500
    E = (rng.standard_normal((V, D)) * 0.1).astype(np.float32)
    t = capi.Table(ctx, E)
    c = capi.Corpus(ctx, n_rows)
    c.append(unit_rows(rng, n_rows))
    ctx.owned += [t, c]
    offsets, ids = random_lines(rng, 50, V, min_len=1)
    good = (offsets, ids)
    bad_ids = ids.copy()
    bad_ids[3] = V + 1
    return rng, E, t, c, good, (offsets, bad_ids)


def dev_csr(torch, offsets, ids):
    dev = torch.device("cuda:0")
    off_d = torch.from_numpy(offsets.view(np.int64)).to(dev)
    ids_d = torch.from_numpy(ids.view(np.int32)).to(dev)
    out_d = torch.zeros((offsets.size - 1, D), dtype=torch.float32, device=dev)
    torch.cuda.synchronize()
    return off_d, ids_d, out_d


def bad_embed_dev(torch, ctx, t, bad):
    off_d, ids_d, out_d = dev_csr(torch, *bad)
    capi.embed_dev(ctx, t, off_d.data_ptr(), ids_d.data_ptr(), bad[0].size - 1, out_d.data_ptr())
    ctx.sync()
    return off_d, ids_d, out_d


def expect_range_once(ctx):
    with pytest.raises(capi.StbError) as e:
        capi.embed_status(ctx)
    assert e.value.status == capi.STB_ERR_RANGE
    capi.embed_status(ctx)                                      # reported once, then clear


def search_batch_dev(torch, c, queries, k=10):
    dev = torch.device("cuda:0")
    q = torch.from_numpy(np.ascontiguousarray(queries, np.float32)).to(dev)
    hits = torch.zeros((len(queries), k, 2), dtype=torch.float64, device=dev)
    status = torch.zeros((len(queries), 2), dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    c.search_batch_dev(q.data_ptr(), len(queries), k, hits.data_ptr(), status.data_ptr())
    c.ctx.sync()
    return status.cpu().numpy()


def test_range_flag_survives_an_explicit_copy_build(fresh, torch):
    _, _, t, c, _, bad = flag_setup(torch, fresh)
    assert coverage(c) == (0, 0)
    bad_embed_dev(torch, fresh, t, bad)
    c.prepare(3)
    assert coverage(c) == (len(c), len(c))
    expect_range_once(fresh)


def test_range_flag_survives_a_lazy_q8_build(fresh, torch):
    rng, _, t, c, _, bad = flag_setup(torch, fresh, n_rows=LAZY_ROWS)
    q = unit_rows(rng, 1)[0]
    c.search(q, top_k=10)
    assert c.tier_stats()["q8"]["built_rows"] == 0
    bad_embed_dev(torch, fresh, t, bad)
    c.search(q, top_k=10)                                       # second search: builds the q8 copy
    assert c.tier_stats()["q8"]["built_rows"] == LAZY_ROWS
    expect_range_once(fresh)


def test_range_flag_survives_a_batched_device_search(fresh, torch):
    rng, _, t, c, _, bad = flag_setup(torch, fresh)
    bad_embed_dev(torch, fresh, t, bad)
    search_batch_dev(torch, c, unit_rows(rng, 8))
    expect_range_once(fresh)


def test_range_flag_survives_a_valid_host_embed(fresh, torch):
    _, _, t, c, good, bad = flag_setup(torch, fresh)
    bad_embed_dev(torch, fresh, t, bad)
    capi.embed(fresh, t, *good)
    capi.embed(fresh, t, *good, out=False, append_to=c)
    expect_range_once(fresh)


def test_a_nan_query_in_a_batched_device_search_is_not_an_embed_error(fresh, torch):
    rng, E, t, c, good, _ = flag_setup(torch, fresh)
    queries = unit_rows(rng, 4)
    queries[1, 7] = np.nan
    status = search_batch_dev(torch, c, queries)
    assert status[1, 1] == 0                                    # the NaN query comes back unproven
    capi.embed_status(fresh)
    search_batch_dev(torch, c, queries)
    off_d, ids_d, out_d = dev_csr(torch, *good)
    capi.embed_dev(fresh, t, off_d.data_ptr(), ids_d.data_ptr(), good[0].size - 1, out_d.data_ptr())
    capi.embed_status(fresh)
    assert np.array_equal(bits(out_d.cpu().numpy()), bits(oracle.embed_csr(E, *good)))


def test_a_failed_host_embed_reports_through_its_return_value_only(fresh, torch):
    _, _, t, c, good, bad = flag_setup(torch, fresh)
    with pytest.raises(capi.StbError) as e:
        capi.embed(fresh, t, *bad, out=False, append_to=c)
    assert e.value.status == capi.STB_ERR_RANGE
    capi.embed_status(fresh)
    with pytest.raises(capi.StbError):
        capi.embed(fresh, t, *bad)
    capi.embed(fresh, t, *good)
    capi.embed_status(fresh)


# --------------------------------------------------------------------------------------- arguments ---
def test_arguments(ctx, fresh):
    L = capi.lib()
    vp = C.c_void_p
    E = np.ones((10, D), np.float32)
    t = capi.Table(ctx, E)
    c = capi.Corpus(ctx, 4)
    # n_lines = 0 with null pointers: a no-op
    assert L.stb_embed(ctx._h, t._h, None, None, 0, None, None) == capi.STB_OK
    assert L.stb_embed(ctx._h, t._h, None, None, 0, None, c._h) == capi.STB_OK
    assert L.stb_embed_dev(ctx._h, t._h, None, None, 0, None) == capi.STB_OK
    assert len(c) == 0
    capi.embed_status(ctx)

    def rc(offsets, ids):
        offsets = np.asarray(offsets, np.uint64)
        out = np.zeros((max(offsets.size - 1, 1), D), np.float32)
        return L.stb_embed(ctx._h, t._h, offsets.ctypes.data_as(vp),
                           None if ids is None else np.asarray(ids, np.uint32).ctypes.data_as(vp),
                           offsets.size - 1, out.ctypes.data_as(vp), c._h)

    assert rc([1, 2], [0, 1]) == capi.STB_ERR_ARG               # offsets[0] != 0
    assert rc([0, 3, 2, 4], [0, 1, 2, 3]) == capi.STB_ERR_ARG   # not monotone
    assert rc([0, 2], None) == capi.STB_ERR_ARG                 # tokens but no ids
    assert rc([0, 0, 0], None) == capi.STB_OK                   # no tokens, no ids: fine
    assert len(c) == 2
    # handles of another context
    t2 = capi.Table(fresh, E)
    c2 = capi.Corpus(fresh, 4)
    fresh.owned += [t2, c2]
    with pytest.raises(capi.StbError) as e:
        capi.embed(ctx, t2, [0, 1], [1])
    assert e.value.status == capi.STB_ERR_ARG
    with pytest.raises(capi.StbError) as e:
        capi.embed(ctx, t, [0, 1], [1], append_to=c2)
    assert e.value.status == capi.STB_ERR_ARG
    assert len(c2) == 0
    assert L.stb_embed_dev(ctx._h, t2._h, None, None, 0, None) == capi.STB_ERR_ARG
    c.close(); t.close()
