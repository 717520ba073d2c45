"""CPU model of the K2 pipeline-v2 selection rule (semtools_b200/csrc/batch_scan.cu, "Pipeline
v2"): with a = 16-bit (fp16 by default, or bf16) approximate score and c = exact cosine, |a - c| <= EPS, the rows with
a >= S_k - 2 EPS (S_k = k-th largest sampled COMPLETE-tile maximum) contain the oracle's top-k,
and so do the rows with a >= A_k - 2 EPS (A_k = k-th largest approximate score).  This checks
the arithmetic claim on data with ties, duplicates, exact hits (c >= 1 clamps), zero rows and a
ragged last tile; the kernels themselves are checked on the GPU (tests/test_gpu_batch.py and
tests/test_gpu_batch_contract.py)."""
import numpy as np
import pytest

import oracle
from conftest import unit_rows

TILE = 256


def to16(x, dtype="bfloat16"):
    torch = pytest.importorskip("torch")
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(getattr(torch, dtype)).to(torch.float32).numpy()


def bf16(x):
    return to16(x, "bfloat16")


def approx_scores(rows, queries, dtype="bfloat16"):
    norm = np.linalg.norm(rows.astype(np.float64), axis=1, keepdims=True)
    rn = to16(np.divide(rows, norm, out=np.zeros_like(rows), where=norm > 0).astype(np.float32), dtype)
    qn = to16((queries / np.linalg.norm(queries.astype(np.float64), axis=1, keepdims=True)).astype(np.float32), dtype)
    return qn @ rn.T                                            # f32 accumulation, like the wgmma accumulators


# STB_BATCH_EPS of the two shadow types: fp16 (the default build) and bf16 (-DSTB_SHADOW_F16=0)
@pytest.mark.parametrize("dtype,EPS", [("bfloat16", 0.0080), ("float16", 0.0012)])
@pytest.mark.parametrize("n,k,n_sample", [(20_000, 10, 37), (20_000, 1, 78), (20_001, 64, 78), (5_000, 3, 5), (300, 5, 1)])
def test_threshold_rule_keeps_the_exact_topk(n, k, n_sample, dtype, EPS):
    rng = np.random.default_rng(n + k)
    rows = (unit_rows(rng, n) * rng.uniform(0.25, 4.0, (n, 1))).astype(np.float32)
    queries = unit_rows(rng, 12)
    rows[rng.integers(0, n, 30)] = rows[rng.integers(0, n, 30)]                 # duplicates
    rows[[1, n // 2]] = 0.0                                                      # zero rows
    queries[0] = rows[7] / np.linalg.norm(rows[7])                               # exact hit: c ~ 1
    dense = rng.choice(n, 200, replace=False)
    rows[dense] = (queries[1] + 0.01 * unit_rows(rng, 200)).astype(np.float32)   # 200 near-ties at the top
    a = approx_scores(rows, queries, dtype)
    n_full = n // TILE
    stride = max(n_full // n_sample, 1)
    for qi, q in enumerate(queries):
        d = oracle.distances(rows, q)
        c = 1.0 - d
        live = d != 1.0                                                          # not the ab == 0 -> 1 special case (zero rows)
        assert np.max(np.abs(a[qi][live] - c[live])) <= EPS                       # the bound the proof rests on
        r_top, _ = oracle.search_rows(rows, q, top_k=k)
        tile_max = a[qi][: n_full * TILE].reshape(n_full, TILE).max(axis=1)
        sample = tile_max[::stride][:n_sample]
        if len(sample) >= k:
            s_k = np.sort(sample)[-k]
            emitted = a[qi] >= np.float32(s_k) - np.float32(2 * EPS)
        else:
            emitted = np.ones(n, bool)                                           # thr = -inf
        assert emitted[r_top].all(), (qi, "emission threshold lost a top-k row")
        a_k = np.sort(a[qi][emitted])[-min(k, int(emitted.sum()))]
        narrowed = emitted & (a[qi] >= np.float32(a_k) - np.float32(2 * EPS))
        assert narrowed[r_top].all(), (qi, "narrowing lost a top-k row")
        # and the exact order restricted to the narrowed set is the oracle's answer
        idx = np.flatnonzero(narrowed)
        order = idx[np.lexsort((idx, d[idx]))][:k]
        assert order.tolist() == [int(x) for x in r_top]


def test_fp16_shadow_bound():
    """-DSTB_SHADOW_F16=1: |fp16 approximate - exact cosine| <= 0.0012 on unit rows, including rows with
    many tiny (fp16-subnormal) components."""
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(11)
    rows = unit_rows(rng, 4000)
    spiky = rng.standard_normal((200, 256)).astype(np.float32) * np.float32(1e-6)      # components far below 2^-14 ...
    spiky[np.arange(200), rng.integers(0, 256, 200)] = 1.0                              # ... next to one dominant one
    rows[:200] = spiky / np.linalg.norm(spiky, axis=1, keepdims=True)
    queries = unit_rows(rng, 6)
    queries[0] = rows[3]
    h = lambda x: torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(torch.float16).to(torch.float32).numpy()
    a = h(queries) @ h(rows).T
    for qi, q in enumerate(queries):
        c = 1.0 - oracle.distances(rows, q)
        assert np.max(np.abs(a[qi] - c)) <= 0.0012


@pytest.mark.parametrize("dtype,eps", [("bfloat16", 0.0040), ("float16", 0.00052)])
def test_shadow_scan_margin_with_f32_query(dtype, eps):
    """K1's half-width scan (tier h16) rounds only the ROW; the query stays f32:
    |q^ . round(x^) - exact cosine| <= STB_SHADOW_SCAN_EPS."""
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(21)
    rows = (unit_rows(rng, 6000) * rng.uniform(0.1, 10.0, (6000, 1))).astype(np.float32)
    spiky = rng.standard_normal((300, 256)).astype(np.float32) * np.float32(1e-6)
    spiky[np.arange(300), rng.integers(0, 256, 300)] = 1.0
    rows[:300] = spiky
    rows[300] = 0.0
    queries = unit_rows(rng, 8) * np.float32(3.0)
    queries[0] = rows[5]
    norm = np.linalg.norm(rows.astype(np.float64), axis=1, keepdims=True)
    xn = np.divide(rows, norm, out=np.zeros_like(rows), where=norm > 0).astype(np.float32)
    xs = torch.from_numpy(xn).to(getattr(torch, dtype)).to(torch.float32).numpy()
    for q in queries:
        qn = (q / np.float32(np.linalg.norm(q.astype(np.float64)))).astype(np.float32)
        a = xs @ qn
        c = 1.0 - oracle.distances(rows, q)
        assert np.max(np.abs(a - c)) <= eps, np.max(np.abs(a - c))


def test_bf16_margins_hold_for_the_adversarial_row():
    """bf16 keeps 8 significand bits: unit roundoff 2^-8, not 2^-9.  A unit row whose components sit
    just below a rounding midpoint loses ~2^-8 relatively in EVERY component, so the both-rounded
    score is off by ~2u and the row-only score by ~u.  The margins in the kernels (0.0080 / 0.0040)
    cover it; the values they replaced (0.0045 / 0.0020) did not."""
    v = np.float32(2.0 ** -4 * (1 + 0.498 * 2.0 ** -7))                 # rounds down by ~half a bf16 ulp
    m = 250
    w = np.sqrt((1.0 - m * float(v) ** 2) / (256 - m))
    x = np.array([v] * m + [w] * (256 - m), dtype=np.float64)
    xn = (x / np.linalg.norm(x)).astype(np.float32)
    xb = bf16(xn).astype(np.float64)
    both = abs(float(xb @ xb) - 1.0)                                    # query = the row itself, exact cosine 1
    row_only = abs(float(xb @ xn.astype(np.float64)) - 1.0)
    assert 0.0045 < both <= 0.0080
    assert 0.0020 < row_only <= 0.0040
