"""K1's per-row score contracts, checked row by row on the GPU against an f64 reference (DESIGN.md section 5).

The scan hooks (stb_debug_scan_scores, stb_debug_q4_scan) run the production passes with a sink that records every
score, so each pass is held to its own contract on every row, not only through the final hits:
  f32   |s - c| <= STB_SCORE_EPS; +inf for rows whose fp32 ||x||^2 is outside [1e-30, 1e30]; zero rows 0 (1 under
        a zero query)
  h16   |s - c| <= STB_SHADOW_SCAN_EPS
  q8    u8 >= c - 1e-5; +inf for an unusable query
  q4    u4 >= c - 1e-5, l8 <= c - 1e-5, T <= c_k - 1e-5 at every skip decision (a skipped row has c < c_k)
  hist  bin = clamp(floor((1 - s) * 2048)) over the finite scores
where c = x.q / (||x|| ||q||) in f64 from the f32 inputs (0 for zero rows) and c_k the k-th best c.  The large-k
routes are then run at the bin edges those histograms expose.  The adversarial rows and queries come from the numpy
models of the bounds (test_q8_bound_model, test_q4_bound_model)."""
import numpy as np
import pytest

import oracle
from semtools_b200 import capi
from test_q4_bound_model import nibble_edge_rows, pack_plane
from test_q8_bound_model import build_q8, exact_cos, q8_scores, unit

pytestmark = pytest.mark.gpu

F = np.float32
SCORE_EPS = 1e-5             # STB_SCORE_EPS
BOUND_EPS = 1e-5             # u8, u4 >= c - 1e-5; l8 <= c - 1e-5
SKIP_EPS = F(2e-5)           # STB_Q4_SKIP_EPS
Q8_ROUTE_MARGIN = 0.04       # the q8 large-k route's floor below the k-th bound's bin
COUNTS = (1, 31, 32, 33, 255, 257)
BIG = 300_007

# worst observed margins: name -> (value, row kind); printed by the last test
MARGINS = {}


def note(name, values, kinds, worst=np.argmin):
    """Keep the worst value of a margin seen so far, over all rows and over the non-zero rows."""
    kinds = np.asarray(kinds)
    for label, m in ((name, np.ones(len(values), bool)), (name + ", non-zero rows", kinds != "zero")):
        if not m.any():
            continue
        i = int(worst(values[m]))
        v = float(values[m][i])
        old = MARGINS.get(label)
        if old is None or (v < old[0] if worst is np.argmin else v > old[0]):
            MARGINS[label] = (v, str(kinds[m][i]))


# ---- rows ---------------------------------------------------------------------------------------------------
def adversarial_rows(rng):
    """(rows, kind) with every row's fp32 ||x||^2 a normal number inside [1e-30, 1e30]: the q8 copy accepts them."""
    parts = []
    parts.append(("unit", unit(rng, 300)))
    dom = unit(rng, 200)
    dom[:, 0] += F(3.0)
    parts.append(("dominant", dom))
    base = unit(rng, 200)                                     # codes parked on nibble and rounding boundaries
    grid = np.abs(base).max(axis=1, keepdims=True) / 127.0
    cells = np.clip(np.rint(base / grid / 16.0), -7, 7) * 16.0
    parked = ((cells + rng.choice([-0.5001, -0.4999, 0.4999, 15.4999], base.shape)) * grid).astype(F)
    parked[:, 0] = (127.0 * grid[:, 0]).astype(F)
    parts.append(("parked", parked))
    parts.append(("nibble_edge", np.concatenate([nibble_edge_rows(rng, 40, o) for o in (0, 7, 15)])))
    parts.append(("scaled", (unit(rng, 200) * F(10.0) ** rng.uniform(-12, 12, (200, 1))).astype(F)))
    sparse = np.zeros((100, 256), dtype=F)
    sparse[np.arange(100), rng.integers(0, 256, 100)] = 1.0
    sparse[np.arange(100), rng.integers(0, 256, 100)] += F(0.5)
    parts.append(("sparse", sparse))
    parts.append(("sign", np.sign(unit(rng, 50)).astype(F)))
    parts.append(("constant", np.concatenate([np.ones((1, 256), F), np.full((1, 256), -0.5, F)])))
    parts.append(("zero", np.zeros((10, 256), dtype=F)))
    rows = np.concatenate([p for _, p in parts]).astype(F)
    kind = np.concatenate([[k] * len(p) for k, p in parts])
    dup = rng.choice(len(rows), 30, replace=False)
    rows = np.concatenate([rows, rows[dup]])
    kind = np.concatenate([kind, ["duplicate"] * 30])
    return rows, kind


def special_rows(rng):
    """Rows the f32 pass must force (+inf) or score, at the edges of the fp32 norm range; the q8 copy refuses them."""
    u = unit(rng, 12).astype(np.float64)
    rows = np.stack([u[0] * np.sqrt(1.02e-30), u[1] * np.sqrt(0.98e-30),     # ||x||^2 just inside / outside 1e-30
                     u[2] * np.sqrt(0.98e30), u[3] * np.sqrt(1.02e30),       # just inside / outside 1e30
                     u[4] * 1e-25, u[5] * 1e-22]).astype(F)                  # fp32 ||x||^2 underflows to 0 / denormal
    kind = ["norm_lo_in", "norm_lo_out", "norm_hi_in", "norm_hi_out", "underflow", "denormal"]
    bad = unit(rng, 4)
    bad[0, 17] = np.nan
    bad[1, 200] = np.inf
    bad[2, 3] = -np.inf
    bad[3, :] = np.inf
    return np.concatenate([rows, bad]).astype(F), np.array(kind + ["nan", "inf", "-inf", "all_inf"])


def f32_expected_class(rows):
    """'forced' | 'zero' | 'scored' from the f64 squared norm (the specials sit >= 2 % away from the edges)."""
    r = rows.astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        n2 = (r * r).sum(axis=1)
    nz = np.any(rows != 0, axis=1)
    return np.where(~nz, "zero", np.where(np.isfinite(n2) & (n2 >= 1e-30) & (n2 <= 1e30), "scored", "forced"))


_MIXED = {}


def mixed(n, seed):
    """n rows: a sample of the adversarial rows, or all of them spread over unit rows; cached per (n, seed)."""
    if (n, seed) not in _MIXED:
        rng = np.random.default_rng(seed)
        adv, kind = adversarial_rows(rng)
        if n <= len(adv):
            pick = rng.permutation(len(adv))[:n]
            rows, kinds = np.ascontiguousarray(adv[pick]), kind[pick]
        else:
            rows = unit(rng, n)
            kinds = np.array(["unit"] * n, dtype=object)
            at = rng.choice(n, len(adv), replace=False)
            rows[at] = adv
            kinds[at] = kind
        _MIXED[(n, seed)] = (rows, kinds)
    return _MIXED[(n, seed)]


_F64 = {}


def cos_ref(rows, q):
    """exact_cos of test_q8_bound_model, with the f64 rows and their norms kept per matrix."""
    if id(rows) not in _F64:
        r = rows.astype(np.float64)
        with np.errstate(over="ignore", invalid="ignore"):
            _F64[id(rows)] = (rows, r, np.sqrt((r * r).sum(axis=1)))
    _, r, rn = _F64[id(rows)]
    qq = q.astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        n = rn * np.sqrt((qq * qq).sum())
        return np.divide(r @ qq, n, out=np.zeros(len(r)), where=n > 0)


def queries(rng, rows, kind):
    qs = []
    for _ in range(2):
        q = unit(rng, 1)[0]
        qs += [("random", q), ("-random", -q)]
    for k in ("dominant", "parked", "nibble_edge", "scaled", "sparse"):
        idx = np.flatnonzero(kind == k)
        if len(idx):
            r = rows[idx[0]].copy()
            qs += [(f"row:{k}", r), (f"-row:{k}", -r)]
    spike = unit(rng, 1)[0]
    spike[7] = 40.0
    onehot = np.zeros(256, F)
    onehot[3] = 1.0
    qs += [("spike", spike), ("sign", np.sign(unit(rng, 1)[0])), ("ones", np.ones(256, F)), ("onehot", onehot)]
    q = unit(rng, 1)[0]
    qs += [("x1e-4", q * F(1e-4)), ("x1e4", q * F(1e4))]
    return [(name, np.ascontiguousarray(v, dtype=F)) for name, v in qs]


def bad_queries(rng):
    q = unit(rng, 1)[0]
    nanq, infq = q.copy(), q.copy()
    nanq[5] = np.nan
    infq[9] = np.inf
    return [("nan", nanq), ("inf", infq), ("underflow", (q * F(1e-16)).astype(F)), ("overflow", (q * F(1e16)).astype(F))]


# ---- corpora ------------------------------------------------------------------------------------------------
_CORPORA = {}


def corpus(ctx, key, rows, host=False, prepare=0):
    k = (key, host, prepare)
    if k not in _CORPORA:
        c = capi.Corpus.in_host_memory(ctx, max(len(rows), 1)) if host else capi.Corpus(ctx, max(len(rows), 1))
        c.append(rows)
        if prepare:
            c.prepare(prepare)
        _CORPORA[k] = c
    return _CORPORA[k]


@pytest.fixture(scope="module", autouse=True)
def _release_corpora():
    yield
    for c in _CORPORA.values():
        c.close()
    _CORPORA.clear()
    _MIXED.clear()
    _F64.clear()


def h16_eps():
    f16, _ = capi.batch_params()
    return 0.00052 if f16 else 0.0040     # STB_SHADOW_SCAN_EPS


def in_scope(n, ranges):
    m = np.zeros(n, dtype=bool)
    if ranges is None:
        m[:] = True
    else:
        for b, e in ranges:
            m[b:min(e, n)] = True
    return m


def check_coverage(seen, scope):
    assert np.all(seen[scope] == 1), ("rows scored != once", np.flatnonzero(seen[scope] != 1)[:10], seen[scope].max())
    assert np.all(seen[~scope] == 0), ("rows outside the ranges scored", np.flatnonzero(seen[~scope])[:10])


# ---- per-pass contracts ---------------------------------------------------------------------------------------
def check_f32(c, rows, kind, q, ranges=None, cls=None):
    s, seen, _ = c.debug_scan_scores(q, "f32", row_ranges=ranges)
    scope = in_scope(len(rows), ranges)
    check_coverage(seen, scope)
    cls = f32_expected_class(rows) if cls is None else cls
    cc = cos_ref(rows, q)
    scored = scope & (cls == "scored")
    err = np.abs(s[scored].astype(np.float64) - cc[scored])
    assert np.all(err <= SCORE_EPS), (float(err.max()), kind[scored][int(err.argmax())])
    note("f32 |s - c| (max)", err, kind[scored], worst=np.argmax)
    assert np.all(s[scope & (cls == "forced")] == np.inf)
    assert np.all(s[scope & (cls == "zero")] == 0.0)
    return s


@pytest.mark.parametrize("n", COUNTS + (BIG,))
def test_f32_h16_q8_scores_meet_their_contracts(ctx, n):
    rows, kind = mixed(n, 100 + n)
    rng = np.random.default_rng(200 + n)
    c = corpus(ctx, ("mixed", n), rows, prepare=3)                 # q8 copy + 16-bit shadow
    eps16 = h16_eps()
    ranges_list = [None]
    if n >= 33:
        ranges_list.append([[1, n - 1]])
    if n == BIG:
        ranges_list += [[[5, BIG - 3]],
                        [[37 + 300 * i, 37 + 300 * i + 1 + i % 9] for i in range(900)],
                        [[0, 1], [33, 97], [1000, 1031], [150_001, 150_300], [BIG - 1, BIG]]]
    for qi, (qname, q) in enumerate(queries(rng, rows, kind)):
        cc = cos_ref(rows, q)
        for ranges in (ranges_list if qi < 2 else ranges_list[:1]):
            scope = in_scope(n, ranges)
            check_f32(c, rows, kind, q, ranges, cls=np.where(np.any(rows != 0, axis=1), "scored", "zero"))
            s16, seen, _ = c.debug_scan_scores(q, "h16", row_ranges=ranges)
            check_coverage(seen, scope)
            err = np.abs(s16[scope].astype(np.float64) - cc[scope])
            assert np.all(err <= eps16), (qname, float(err.max()), kind[scope][int(err.argmax())])
            note("h16 |s - c| (max)", err, kind[scope], worst=np.argmax)
            u8, seen, _ = c.debug_scan_scores(q, "q8", row_ranges=ranges)
            check_coverage(seen, scope)
            slack = u8[scope].astype(np.float64) - cc[scope]
            assert np.all(slack >= -BOUND_EPS), (qname, float(slack.min()), kind[scope][int(slack.argmin())])
            note("u8 - c (min)", slack, kind[scope])


def test_f32_pass_forces_rows_outside_the_norm_range_and_scores_the_rest(ctx):
    rng = np.random.default_rng(7)
    adv, kind = adversarial_rows(rng)
    sp, sk = special_rows(rng)
    rows = np.concatenate([adv[:150], sp, adv[150:400], sp[:6], adv[400:]]).astype(F)
    kind = np.concatenate([kind[:150], sk, kind[150:400], sk[:6], kind[400:]])
    cls = f32_expected_class(rows)
    assert set(cls[np.isin(kind, ["norm_lo_out", "norm_hi_out", "underflow", "denormal", "nan", "inf", "-inf", "all_inf"])]) == {"forced"}
    assert set(cls[np.isin(kind, ["norm_lo_in", "norm_hi_in"])]) == {"scored"}
    c = corpus(ctx, "special", rows, prepare=3)                # both reduced copies refuse such rows ...
    assert c.tier_stats()["q8"]["built_rows"] == 0 and c.tier_stats()["h16"]["built_rows"] == 0
    for tier in ("q8", "h16"):                                 # ... and so does the hook
        with pytest.raises(capi.StbError) as e:
            c.debug_scan_scores(np.ones(256, F), tier)
        assert e.value.status == capi.STB_ERR_STATE
    for _, q in queries(rng, rows, kind):
        check_f32(c, rows, kind, q, cls=cls)
        check_f32(c, rows, kind, q, ranges=[[3, 160], [401, 402], [700, len(rows)]], cls=cls)
    # a zero query: every scored row 0, zero rows 1, forced rows +inf
    s, seen, _ = c.debug_scan_scores(np.zeros(256, F), "f32")
    assert np.all(seen == 1)
    assert np.all(s[cls == "scored"] == 0.0) and np.all(s[cls == "zero"] == 1.0) and np.all(s[cls == "forced"] == np.inf)
    # a query that cannot be normalised: every row +inf except the zero rows (0)
    for name, q in bad_queries(rng):
        s, seen, _ = c.debug_scan_scores(q, "f32")
        assert np.all(seen == 1)
        assert np.all(s[cls == "zero"] == 0.0) and np.all(s[cls != "zero"] == np.inf), name


def test_unusable_queries_make_every_reduced_score_inf(ctx):
    rng = np.random.default_rng(8)
    rows, kind = mixed(257, 8)
    c = corpus(ctx, ("mixed", 257), rows, prepare=3)
    for name, q in bad_queries(rng) + [("zero", np.zeros(256, F))]:
        u8, seen, _ = c.debug_scan_scores(q, "q8")
        assert np.all(seen == 1) and np.all(u8 == np.inf), name
        d = c.debug_q4_scan(q, 10, pin=False)
        assert np.all(d["refined"] == 1) and np.all(d["u8"] == np.inf), name   # nothing skipped, nothing published
        assert np.all(d["words"] == 0), name
        if name != "zero":
            s16, _, _ = c.debug_scan_scores(q, "h16")
            assert np.all(s16 == np.inf), name


# ---- the 4-bit prefilter -----------------------------------------------------------------------------------
def f2ord(x):
    b = np.asarray(x, dtype=F).view(np.uint32).astype(np.uint64)
    return np.where(b & 0x80000000, (~b) & 0xFFFFFFFF, b | 0x80000000).astype(np.uint64)


def check_words(d, k, scope):
    ref = d["refined"] > 0
    words = d["words"]
    assert np.all((words >> np.uint64(32) == 1) | (words == 0)), [hex(int(w)) for w in words]   # this launch's tag
    rows = np.flatnonzero(ref & scope)
    for w in range(k):
        mine = rows[rows % k == w]
        want = int(f2ord(d["l8"][mine].max())) if len(mine) else None
        got = int(words[w]) & 0xFFFFFFFF
        assert (want is None and int(words[w]) == 0) or got == want, (k, w, hex(got), want)


def check_q4_pinned(c, rows, kind, q, k, ranges=None):
    d = c.debug_q4_scan(q, k, row_ranges=ranges, pin=True)
    scope = in_scope(len(rows), ranges)
    check_coverage(d["refined"], scope)
    assert np.all(d["t"][scope] == -np.inf)
    cc = cos_ref(rows, q)
    slack4 = d["u4"][scope].astype(np.float64) - cc[scope]
    assert np.all(slack4 >= -BOUND_EPS), (float(slack4.min()), kind[scope][int(slack4.argmin())])
    note("u4 - c (min)", slack4, kind[scope])
    low = cc[scope] - d["l8"][scope].astype(np.float64)
    assert np.all(low >= BOUND_EPS), (float(low.min()), kind[scope][int(low.argmin())])
    note("c - l8 (min)", low, kind[scope])
    u8, _, _ = c.debug_scan_scores(q, "q8", row_ranges=ranges)
    assert np.array_equal(d["u8"][scope].view(np.uint32), u8[scope].view(np.uint32))
    check_words(d, k, scope)


@pytest.mark.parametrize("n", COUNTS + (BIG,))
def test_q4_bounds_hold_for_every_row_when_everything_is_refined(ctx, n):
    rows, kind = mixed(n, 100 + n)
    rng = np.random.default_rng(300 + n)
    c = corpus(ctx, ("mixed", n), rows, prepare=3)
    qs = queries(rng, rows, kind)
    for qi, (_, q) in enumerate(qs):
        check_q4_pinned(c, rows, kind, q, (1, 10, 16)[qi % 3])
    if n >= 33:
        check_q4_pinned(c, rows, kind, qs[0][1], 10, ranges=[[1, n - 1]])
    if n == BIG:
        check_q4_pinned(c, rows, kind, qs[1][1], 16, ranges=[[37 + 300 * i, 37 + 300 * i + 1 + i % 9] for i in range(900)])


def check_q4_live(c, rows, kind, q, k, ranges=None):
    d = c.debug_q4_scan(q, k, row_ranges=ranges, pin=False)
    scope = in_scope(len(rows), ranges)
    cc = cos_ref(rows, q)
    ck = np.sort(cc[scope])[::-1][k - 1]
    assert np.all(d["refined"][~scope] == 0) and np.all(d["refined"][scope] <= 1)
    assert np.all(d["t"][scope] <= ck - BOUND_EPS), (k, float(d["t"][scope].max()), ck)
    skipped = scope & (d["refined"] == 0)
    assert skipped.sum() > 0, "no row was skipped: the live threshold was never tested"
    assert np.all(d["u4"][skipped] + SKIP_EPS < d["t"][skipped])
    assert np.all(cc[skipped] < ck)
    refined = scope & (d["refined"] == 1)
    slack4 = d["u4"][scope].astype(np.float64) - cc[scope]
    assert np.all(slack4 >= -BOUND_EPS)
    assert np.all(cc[refined] - d["l8"][refined].astype(np.float64) >= BOUND_EPS)
    check_words(d, k, scope)
    return d, ck, skipped.sum()


def test_q4_live_threshold_only_skips_rows_below_the_kth_best(ctx):
    rows, kind = mixed(BIG, 100 + BIG)
    rng = np.random.default_rng(400)
    c = corpus(ctx, ("mixed", BIG), rows, prepare=3)
    q = unit(rng, 1)[0]
    for k in (1, 10, 16):
        check_q4_live(c, rows, kind, q, k)
        check_q4_live(c, rows, kind, rows[np.flatnonzero(kind == "dominant")[0]], k)
    check_q4_live(c, rows, kind, q, 10, ranges=[[5, BIG - 3]])
    check_q4_live(c, rows, kind, q, 16, ranges=[[0, 1], [33, 97], [1000, 1031], [150_001, 290_300], [BIG - 1, BIG]])


def test_q4_live_threshold_with_negative_bounds(ctx):
    """A clustered corpus queried against its cluster direction: every cosine, every l8 and T are negative, so the
    threshold words order negative floats (stb_f2ord)."""
    rng = np.random.default_rng(401)
    n = 200_000
    d = unit(rng, 1)[0].astype(np.float64)
    spread = rng.uniform(0.1, 3.0, (n, 1))
    rows = (d[None, :] + spread * rng.standard_normal((n, 256)) / 16.0).astype(F)
    kind = np.array(["clustered"] * n)
    c = corpus(ctx, "clustered", rows, prepare=1)
    q = (-d).astype(F)
    for k in (1, 10, 16):
        dd, ck, _ = check_q4_live(c, rows, kind, q, k)
        assert ck < 0 and np.nanmax(dd["l8"]) < 0 and dd["t"].max() < 0
        assert np.all(dd["words"] & np.uint64(0x80000000) == 0)     # ordered negative floats


# ---- histogram, parity with host rows, the copies -------------------------------------------------------------
def np_hist(s):
    s = s[np.isfinite(s)].astype(F)
    b = np.floor((F(1.0) - s) * F(2048.0))
    return np.bincount(np.clip(b, 0, 4095).astype(np.int64), minlength=4096).astype(np.uint32)


def test_histogram_bins_exactly_the_finite_scores(ctx):
    rng = np.random.default_rng(9)
    rows, kind = mixed(BIG, 100 + BIG)
    c = corpus(ctx, ("mixed", BIG), rows, prepare=3)
    sp, _ = special_rows(rng)
    rows2 = np.concatenate([rows[:20_000], sp, sp]).astype(F)
    c2 = corpus(ctx, "hist_special", rows2)
    for name, q in queries(rng, rows, kind)[:6]:
        for tier in ("f32", "q8"):
            for ranges in (None, [[3, 77_777], [100_003, 100_005], [200_000, BIG - 1]]):
                s, _, h = c.debug_scan_scores(q, tier, row_ranges=ranges, hist=True)
                scope = in_scope(len(rows), ranges)
                assert np.array_equal(h, np_hist(s[scope])), (name, tier)
        s, _, h = c2.debug_scan_scores(q, "f32", hist=True)
        assert np.isinf(s).sum() == 2 * 8
        assert np.array_equal(h, np_hist(s)), name                 # forced rows (+inf) are not counted
    with pytest.raises(capi.StbError) as e:
        c.debug_scan_scores(rows[0], "h16", hist=True)
    assert e.value.status == capi.STB_ERR_ARG


def test_host_rows_corpus_gives_the_same_scores(ctx):
    rng = np.random.default_rng(10)
    rows, kind = mixed(20_011, 10)
    sp, _ = special_rows(rng)
    dev = corpus(ctx, "parity", rows, prepare=1)
    host = corpus(ctx, "parity", rows, host=True)
    both = np.concatenate([rows, sp]).astype(F)
    dev2, host2 = corpus(ctx, "parity2", both), corpus(ctx, "parity2", both, host=True)
    for _, q in queries(rng, rows, kind)[:8]:
        for tier in ("f32", "q8"):
            a, sa, ha = dev.debug_scan_scores(q, tier, hist=True)
            b, sb, hb = host.debug_scan_scores(q, tier, hist=True)
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)) and np.array_equal(sa, sb) and np.array_equal(ha, hb)
        a, _, _ = dev2.debug_scan_scores(q, "f32", row_ranges=[[7, 15_000], [20_000, len(both)]])
        b, _, _ = host2.debug_scan_scores(q, "f32", row_ranges=[[7, 15_000], [20_000, len(both)]])
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
        da, db = dev.debug_q4_scan(q, 10, pin=True), host.debug_q4_scan(q, 10, pin=True)
        for key in ("u4", "u8", "l8", "refined", "words"):
            assert np.array_equal(da[key].view(np.uint32) if da[key].dtype == F else da[key],
                                  db[key].view(np.uint32) if db[key].dtype == F else db[key]), key


def test_q8_copy_matches_its_f64_definitions(ctx):
    rows, kind = mixed(BIG, 100 + BIG)
    c = corpus(ctx, ("mixed", BIG), rows, prepare=3)
    codes, cov = c.debug_copy(capi.STB_COPY_Q8_CODES)
    assert cov == len(rows)
    s = c.debug_copy(capi.STB_COPY_Q8_SCALES)[0].astype(np.float64)
    plane = c.debug_copy(capi.STB_COPY_Q8_PLANE)[0]
    rho = c.debug_copy(capi.STB_COPY_Q8_SR)[0].astype(np.float64)
    assert np.array_equal(rho[:, 0], s)
    rho = rho[:, 1]
    codes = codes.astype(np.int64)
    r = rows.astype(np.float64)
    norm = np.sqrt((r * r).sum(axis=1))
    zero = norm == 0
    assert np.all(s[zero] == 0) and np.all(codes[zero] == 0) and np.all(rho[zero] == np.float64(F(1e-6)))
    xh = r[~zero] / norm[~zero, None]
    sz, cz, rz = s[~zero], codes[~zero], rho[~zero]
    err = np.abs(xh / sz[:, None] - cz).max(axis=1)
    assert np.all(err <= 0.5 + 1e-4), (float(err.max()), kind[~zero][int(err.argmax())])
    want_s = np.abs(xh).max(axis=1) / 127.0
    assert np.all(np.abs(sz - want_s) <= 1e-6 * want_s)
    assert np.array_equal(plane, pack_plane((codes + 128) >> 4))
    resid = np.sqrt(((xh - sz[:, None] * (16.0 * (cz >> 4) + 7.5)) ** 2).sum(axis=1))
    assert np.all(rz >= resid), float((resid - rz).max())
    assert np.all(rz <= 1.0001 * 128.0 * sz + 1e-6)


# ---- large-k routes at bin edges ------------------------------------------------------------------------------
def bin_of(s):
    return np.clip(np.floor((F(1.0) - s.astype(F)) * F(2048.0)), 0, 4095).astype(np.int64)


def edge_ks(scores, n_forced, lo=97, hi=5000, want=50):
    """k in (96, 5000] where the k-th scored row opens a bin, or the k-th and (k - F)-th lie in different bins."""
    b = bin_of(np.sort(scores[np.isfinite(scores)])[::-1])
    ks = [k for k in range(lo, min(hi, len(b)) + 1)
          if b[k - 1] != b[k - 2] or (n_forced and k - n_forced >= 1 and b[k - 1] != b[k - 1 - n_forced])]
    if len(ks) > want:
        ks = [ks[i] for i in np.linspace(0, len(ks) - 1, want).round().astype(int)]
    return ks


def check_hits(hits, r, d):
    assert hits["row"].tolist() == [int(x) for x in r]
    assert np.array_equal(hits["distance"], np.asarray(d, dtype=np.float64))


def test_large_k_f32_route_at_bin_edges_with_forced_rows(ctx):
    rng = np.random.default_rng(11)
    n = 30_000
    rows = unit(rng, n)
    q = unit(rng, 1)[0]
    forced = rng.choice(n, 37, replace=False)
    big = (q[None, :] + F(0.3) * unit(rng, 37)) * F(1e16)              # ||x||^2 > 1e30: forced, some near the top
    rows[forced[:20]] = big[:20].astype(F)
    rows[forced[20:]] = (unit(rng, 17) * F(1e-25)).astype(F)            # fp32 ||x||^2 underflows: forced
    c = corpus(ctx, "large_k_f32", rows)
    s, _, _ = c.debug_scan_scores(q, "f32")
    assert np.isinf(s).sum() == 37
    ks = edge_ks(s, 37)
    assert len(ks) >= 20
    fb = ctx.counters()["fallback_searches"]
    for k in ks:
        r, d = oracle.search_rows(rows, q, top_k=k)
        check_hits(c.search(q, top_k=k), r, d)
    assert ctx.counters()["fallback_searches"] == fb


def test_large_k_q8_route_at_bin_edges(ctx):
    rng = np.random.default_rng(12)
    n = 40_000
    rows = unit(rng, n)
    c = corpus(ctx, "large_k_q8", rows, prepare=1)
    for q in (unit(rng, 1)[0], rows[17].copy()):
        u8, _, _ = c.debug_scan_scores(q, "q8")
        ks = edge_ks(u8, 0)
        assert len(ks) >= 20
        fb = ctx.counters()["fallback_searches"]
        for k in ks:
            r, d = oracle.search_rows(rows, q, top_k=k)
            check_hits(c.search(q, top_k=k), r, d)
        assert ctx.counters()["fallback_searches"] == fb


def proof_failure_data():
    """Dominant-component rows under a sign query: every row's u8 sits ~0.06 above its c, beyond the route's 0.04
    margin, so the floor below the k-th bound's bin lies above the k-th best cosine.  Designed with the numpy model
    of the q8 pass (checked in the test), then confirmed with the hook."""
    rng = np.random.default_rng(13)
    q = np.sign(unit(rng, 1)[0]).astype(F)
    rows = unit(rng, 20_000)
    rows[:, 0] = F(3.0) * q[0]
    return rows, q


def test_q8_route_proof_failure_falls_back_exactly(ctx):
    rows, q = proof_failure_data()
    k = 500
    codes, s = build_q8(rows)
    u_model, _, _ = q8_scores(codes, s, q)
    cc = exact_cos(rows, q)
    top = np.argsort(-u_model, kind="stable")[:k]
    assert (u_model[top].astype(np.float64) - cc[top]).min() > Q8_ROUTE_MARGIN
    dev = corpus(ctx, "q8_fail", rows, prepare=1)
    host = corpus(ctx, "q8_fail", rows, host=True)
    u8, _, _ = dev.debug_scan_scores(q, "q8")
    assert (u8[top].astype(np.float64) - cc[top]).min() > Q8_ROUTE_MARGIN     # the hook confirms the design
    r, d = oracle.search_rows(rows, q, top_k=k)
    for c in (dev, host):
        fb = ctx.counters()["fallback_searches"]
        check_hits(c.search(q, top_k=k), r, d)
        assert ctx.counters()["fallback_searches"] == fb + 1


# ---- argument checks -----------------------------------------------------------------------------------------
def test_hooks_check_their_arguments(ctx):
    rows, _ = mixed(33, 14)
    c = corpus(ctx, ("mixed", 33), rows, prepare=3)
    q = rows[0].copy()
    buf = np.zeros(64, np.float32)
    cnt = np.zeros(64, np.uint32)
    L = capi.lib()
    P = capi._np_ptr
    assert L.stb_debug_scan_scores(ctx._h, c._h, 0, P(q), None, 0, 32, P(buf), P(cnt), None) == capi.STB_ERR_ARG   # cap < n
    assert L.stb_debug_scan_scores(ctx._h, c._h, 0, P(q), None, 0, 33, None, P(cnt), None) == capi.STB_ERR_ARG
    assert L.stb_debug_scan_scores(ctx._h, c._h, 3, P(q), None, 0, 33, P(buf), P(cnt), None) == capi.STB_ERR_ARG
    w = np.zeros(16, np.uint64)
    args = [P(buf), P(buf), P(cnt), P(buf), P(buf), P(w)]
    assert L.stb_debug_q4_scan(ctx._h, c._h, P(q), 10, None, 0, 1, 32, *args) == capi.STB_ERR_ARG
    assert L.stb_debug_q4_scan(ctx._h, c._h, P(q), 17, None, 0, 1, 33, *args) == capi.STB_ERR_ARG
    assert L.stb_debug_q4_scan(ctx._h, c._h, P(q), 10, None, 0, 1, 33, *(args[:5] + [None])) == capi.STB_ERR_ARG
    plain = corpus(ctx, ("plain", 33), rows)                                  # no q8 copy, no shadow
    for tier in ("h16", "q8"):
        with pytest.raises(capi.StbError) as e:
            plain.debug_scan_scores(q, tier)
        assert e.value.status == capi.STB_ERR_STATE
    with pytest.raises(capi.StbError) as e:
        plain.debug_q4_scan(q, 10)
    assert e.value.status == capi.STB_ERR_STATE


def test_report_worst_margins():
    """The smallest observed u4 - c, u8 - c, c - l8 and the largest |s - c| of the f32 and h16 passes, with the row
    kind each came from (run with -s to see them)."""
    for name in sorted(MARGINS):
        v, kind = MARGINS[name]
        print(f"worst {name}: {v:.3e} ({kind})")
