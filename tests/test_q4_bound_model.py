"""CPU model of the q8 tier's 4-bit prefilter (csrc/scan_topk.cu: stb_q8_build_kernel, stb_scan_q4).
A row is skipped when its 4-bit score u4 is below a threshold T by more than STB_Q4_SKIP_EPS, which is
only sound if u4 is an UPPER bound of the exact cosine (u4 >= c - 1e-5) and T a LOWER bound of the k-th
best exact cosine (built from l8 <= c + 1e-5 of k distinct rows).  The kernels' arithmetic is restated in
numpy float32 / int64 and checked against the f64 cosine on random and adversarial rows and queries,
together with the nibble plane's byte layout.  No GPU: this pins the BOUNDS, the GPU tests pin the kernels."""
import numpy as np

from test_q8_bound_model import build_q8, exact_cos, q8_scores, unit

F = np.float32
SKIP_EPS = 2.0e-5        # STB_Q4_SKIP_EPS
Q8_EPS = 2.0e-5          # STB_Q8_SCAN_EPS, subtracted from l8


def build_q4(codes, s, rows):
    """The plane half of stb_q8_build_kernel: nibbles h + 8 = (code + 128) >> 4 and the stored rho, evaluated in
    the kernel's order in f32.  Checked here against rho's definition, ||x^ - s (16 (code >> 4) + 7.5)||_2 in f64
    (x^ as the kernel normalises it): the stored value must not be smaller, and must stay <= 128 s + margin."""
    rows = rows.astype(F)
    ss = (rows * rows).sum(axis=1, dtype=F)
    with np.errstate(divide="ignore"):
        inv = np.where(ss > 0, F(1) / np.sqrt(ss, dtype=F), F(0)).astype(F)
    xh = (rows * inv[:, None]).astype(F)
    nib = (codes + 128) >> 4
    assert nib.min() >= 0 and nib.max() <= 15
    sc = s[:, None]
    centre = (F(0.5) * (32 * nib - 241).astype(F)).astype(F)          # 16 h + 7.5 with h = nib - 8, exact
    d = (xh - (sc * centre).astype(F)).astype(F)
    rho = (np.sqrt((d * d).sum(axis=1, dtype=F)) * F(1.0001) + F(1e-6)).astype(F)
    # the definition, in f64 and written independently of the kernel's expression
    h = (codes >> 4).astype(np.float64)
    ref = np.sqrt(((xh.astype(np.float64) - s.astype(np.float64)[:, None] * (16.0 * h + 7.5)) ** 2).sum(axis=1))
    assert np.all(rho.astype(np.float64) >= ref), float((ref - rho).max())
    assert np.all(ref <= 128.0 * s.astype(np.float64) * (1 + 1e-6) + 1e-7)
    return nib, rho


def pack_plane(nib):
    """Byte 16m + r holds component 32m + r (low nibble) and 32m + 16 + r (high nibble)."""
    n = len(nib)
    v = nib.reshape(n, 8, 2, 16).astype(np.uint8)
    return (v[:, :, 0, :] | (v[:, :, 1, :] << 4)).reshape(n, 128)


def unpack_plane(plane):
    """What lane j sees: word k of its 16-byte chunk, masked with 0x0F0F0F0F and (>> 4) & 0x0F0F0F0F."""
    w = plane.reshape(len(plane), 8, 4, 4).copy().view(np.uint32)[..., 0]        # [n][lane j][word k]
    out = np.zeros((len(plane), 256), dtype=np.int64)
    for j in range(8):
        for k in range(4):
            lo, hi = w[:, j, k] & 0x0F0F0F0F, (w[:, j, k] >> 4) & 0x0F0F0F0F
            for b in range(4):
                out[:, 32 * j + 4 * k + b] = (lo >> (8 * b)) & 0xFF
                out[:, 32 * j + 16 + 4 * k + b] = (hi >> (8 * b)) & 0xFF
    return out


def q4_scores(nib, s, rho, q16, S):
    """stb_scan_q4: D = q16 . (nib - 8) in int32, u4 = s * (D * 16/S + 7.5 sum q16 / S) + (rho + 19.4 / S)."""
    inv_S = F(1.0) / F(S)
    sumq = int(q16.sum())
    A = F(F(16.0) * inv_S)
    B = F(F(7.5) * F(sumq) * inv_S)
    e_q4 = F(F(19.4) * inv_S)
    raw = nib.astype(np.int64) @ q16
    assert np.abs(raw).max() < 2 ** 31
    D = raw - 8 * sumq
    inner = (D.astype(F) * A + B).astype(F)
    return (s * inner + (rho + e_q4).astype(F)).astype(F)


def l8_scores(codes, s, q16, S):
    """The lower bound a refined row publishes: s * (dot / S - h_l1) - e_q - 2e-5."""
    inv_S = F(1.0) / F(S)
    h_l1 = F(F(0.50025) * F(int(np.abs(q16).sum())) * inv_S)
    e_q = F(F(9.7) * inv_S)
    dot = codes.astype(np.int64) @ q16
    return ((s * (dot.astype(F) * inv_S - h_l1).astype(F)).astype(F) - e_q - F(Q8_EPS)).astype(F)


def check(rows, q):
    codes, s = build_q8(rows)
    nib, rho = build_q4(codes, s, rows)
    _, q16, S = q8_scores(codes, s, q)
    c = exact_cos(rows, q)
    u4 = q4_scores(nib, s, rho, q16, S).astype(np.float64)
    l8 = l8_scores(codes, s, q16, S).astype(np.float64)
    assert (u4 - c).min() >= -1e-5, ((u4 - c).min(), int((u4 - c).argmin()))
    assert (c - l8).min() >= 1e-5 - 1e-7, ((c - l8).min(), int((c - l8).argmin()))
    return u4 - c, c, l8, u4


def test_u4_bound_holds_on_random_unit_rows_and_is_useful():
    rng = np.random.default_rng(11)
    rows = unit(rng, 20000)
    for _ in range(6):
        slack, _, _, _ = check(rows, unit(rng, 1)[0])
        # ~0.11 on isotropic rows: a bound, but tight enough to skip most rows against a 10M-row c_k
        assert 0.05 < np.median(slack) < 0.2 and slack.max() < 0.35


def test_u4_bound_holds_on_scaled_rows_and_scaled_queries():
    rng = np.random.default_rng(12)
    rows = (unit(rng, 5000) * rng.uniform(1e-3, 1e3, (5000, 1))).astype(F)
    for scale in (1e-4, 1.0, 37.5, 1e4):
        check(rows, (unit(rng, 1)[0] * F(scale)).astype(F))


def test_u4_bound_holds_on_adversarial_rows_and_queries():
    rng = np.random.default_rng(13)
    n = 5000
    rows = unit(rng, n)
    rows[:500, 0] += F(3.0)                                   # one dominant component
    base = unit(rng, 500)                                     # codes parked on nibble boundaries (16 m - 1/2 .. 16 m + 1/2)
    grid = np.abs(base).max(axis=1, keepdims=True) / 127.0
    cells = np.clip(np.rint(base / grid / 16.0), -7, 7) * 16.0
    rows[500:1000] = ((cells + rng.choice([-0.5001, -0.4999, 0.4999, 15.4999], base.shape)) * grid).astype(F)
    rows[500:1000, 0] = (127.0 * grid[:, 0]).astype(F)       # keep the row's own grid
    rows[1000:1100] = 0.0                                     # zero rows
    rows[1100:1200] *= F(1e-12)                               # tiny rows
    sparse = np.zeros((300, 256), dtype=F)                    # one-hot and two-hot rows
    sparse[np.arange(300), rng.integers(0, 256, 300)] = 1.0
    sparse[np.arange(300), rng.integers(0, 256, 300)] += F(0.5)
    rows[1200:1500] = sparse
    rows[1500:1600] = np.sign(unit(rng, 100)).astype(F)      # all components +-1: every code +-127
    rows[1600:1700] = -np.abs(unit(rng, 100)).astype(F) - F(1.0)   # all components near -max: nibble -8
    queries = [unit(rng, 1)[0] for _ in range(3)]
    spike = unit(rng, 1)[0]; spike[7] = 40.0
    queries.append(spike.astype(F))
    queries.append(np.sign(unit(rng, 1)[0]).astype(F))
    queries.append(np.ones(256, dtype=F))
    onehot = np.zeros(256, dtype=F); onehot[3] = 1.0
    queries.append(onehot)
    for r in (0, 600, 1250, 1550, 1650):
        queries.append(rows[r].copy())
        queries.append((-rows[r]).astype(F))
    for q in queries:
        check(rows, q)


def nibble_edge_rows(rng, n, offset):
    """Rows whose codes all sit at one offset inside their nibble (code = 16 m + offset), plus one component at
    the largest code so the row keeps its own grid: the residual around the nibble midpoints is one-sided."""
    m = rng.integers(-8, 7, (n, 256))
    codes = 16 * m + offset
    codes = np.clip(codes, -127, 127)
    codes[:, 0] = 127
    return (codes / 127.0).astype(F)


def test_u4_bound_holds_when_codes_sit_at_one_end_of_their_nibbles():
    """A constant row (every code 127 = 16*7 + 15), rows with every code at the top (offset 15) or the bottom
    (offset 0) of its nibble, each queried with itself and its negation: the residual is far from zero-mean and
    the query is aligned with it, so a wrong nibble centre or rho fails here."""
    rng = np.random.default_rng(16)
    rows = np.concatenate([np.ones((1, 256), dtype=F), np.full((1, 256), -0.5, dtype=F),
                           nibble_edge_rows(rng, 40, 15), nibble_edge_rows(rng, 40, 0), nibble_edge_rows(rng, 40, 7)])
    for r in list(range(0, len(rows), 9)) + [0, 1]:
        check(rows, rows[r].copy())
        check(rows, (-rows[r]).astype(F))


def test_an_exact_match_behind_near_copies_is_never_skipped():
    """k near-copies of the query fill every threshold word before the exact match (c = 1) arrives: the match's
    u4 must still clear T, or the scan would drop the true best row."""
    rng = np.random.default_rng(17)
    for q in (np.ones(256, dtype=F), nibble_edge_rows(rng, 1, 15)[0], unit(rng, 1)[0]):
        for k in (1, 10, 16):
            near = (q[None, :] + F(1e-3) * unit(rng, k)).astype(F)
            rows = np.concatenate([near, unit(rng, 500), q[None, :]]).astype(F)
            codes, s = build_q8(rows)
            nib, rho = build_q4(codes, s, rows)
            _, q16, S = q8_scores(codes, s, q)
            c = exact_cos(rows, q)
            l8 = l8_scores(codes, s, q16, S).astype(np.float64)
            u4 = q4_scores(nib, s, rho, q16, S).astype(np.float64)
            words = np.full(k, -np.inf)
            np.maximum.at(words, np.arange(len(rows) - 1) % k, l8[:-1])   # everything before the match
            assert not (u4[-1] + SKIP_EPS < words.min()), (k, u4[-1], words.min(), c[-1])
            assert u4[-1] >= c[-1] - 1e-5


def test_nibble_plane_round_trip_is_exact():
    rng = np.random.default_rng(14)
    codes = rng.integers(-127, 128, (300, 256))
    codes[0] = -127; codes[1] = 127; codes[2] = 0
    nib = (codes + 128) >> 4
    plane = pack_plane(nib)
    assert plane.shape == (300, 128) and plane.dtype == np.uint8
    assert np.array_equal(unpack_plane(plane), nib)
    # h = code >> 4 (floor), the 16 codes a nibble stands for straddle the midpoint 16 h + 7.5
    h = nib - 8
    assert np.array_equal(h, codes >> 4) and np.all(codes - 16 * h >= 0) and np.all(codes - 16 * h <= 15)


def test_bucketed_threshold_never_exceeds_the_kth_cosine():
    """T = min over k words of max l8 of the rows with row % k == word: k distinct rows have c >= T, so a row
    with u4 + eps < T has c < c_k.  Checked on whole corpora and on prefixes (what a partial scan has seen),
    including heavy duplication of the best row and a corpus where every row is the query."""
    rng = np.random.default_rng(15)
    rows = unit(rng, 30000)
    dup = unit(rng, 30000)
    q0 = unit(rng, 1)[0]
    dup[rng.choice(30000, 400, replace=False)] = (q0 + F(0.01) * unit(rng, 1)[0]).astype(F)
    same = np.tile(q0, (200, 1)).astype(F)
    for data, q in ((rows, unit(rng, 1)[0]), (dup, q0), (same, q0)):
        codes, s = build_q8(data)
        nib, rho = build_q4(codes, s, data)
        _, q16, S = q8_scores(codes, s, q)
        c = exact_cos(data, q)
        l8 = l8_scores(codes, s, q16, S).astype(np.float64)
        u4 = q4_scores(nib, s, rho, q16, S).astype(np.float64)
        for k in (1, 3, 10, 16):
            ck = np.sort(c)[::-1][k - 1]
            for seen in (len(data), len(data) // 3, 5 * k):
                words = np.full(k, -np.inf)
                np.maximum.at(words, np.arange(seen) % k, l8[:seen])
                T = words.min()
                assert T <= ck - 1e-5, (k, seen, T, ck)
                skipped = u4 + SKIP_EPS < T
                assert np.all(c[skipped] < ck)
    # on isotropic rows the final T leaves only a small share of rows to refine
    codes, s = build_q8(rows)
    nib, rho = build_q4(codes, s, rows)
    q = unit(rng, 1)[0]
    _, q16, S = q8_scores(codes, s, q)
    l8 = l8_scores(codes, s, q16, S).astype(np.float64)
    u4 = q4_scores(nib, s, rho, q16, S).astype(np.float64)
    words = np.full(10, -np.inf)
    np.maximum.at(words, np.arange(len(rows)) % 10, l8)
    assert np.mean(u4 + SKIP_EPS >= words.min()) < 0.25
