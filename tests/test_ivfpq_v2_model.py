"""CPU model of the fused IVF-PQ search's candidate funnel (semtools_b200/csrc/ivfpq.cu,
ivf_adc_finish_kernel): 32-code chunks dealt round-robin over CTAs first, then warps; per-warp
top-64 -> per-CTA top-ADC2_KEEP -> global top-`rerank`.  Checks the index arithmetic (every code is
scanned exactly once) and that the funnel is lossless for the best `rerank` codes even when
they are CONTIGUOUS in code order (a tight cluster inside one inverted list), which is what the
CTA-first dealing is for.  The launch shape and the per-CTA keep are read from the kernel source,
so the model cannot drift from it."""
import os
import re

import numpy as np
import pytest

_SRC = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                         "semtools_b200", "csrc", "ivfpq.cu")).read()


def _define(name):
    return int(re.search(rf"^#define {name} (\d+)", _SRC, flags=re.M).group(1))


N_CTAS, KEEP_CTA = _define("ADC2_MAX_CTAS"), _define("ADC2_KEEP")
WARPS, KEEP_WARP = _define("ADC2_THREADS") // 32, 64          # AdcTop: 2 entries per lane


def deal(total):
    """(cta, warp) -> code positions v, exactly as the kernel's loop."""
    owner = {}
    n_chunks = (total + 31) // 32
    for b in range(N_CTAS):
        for w in range(WARPS):
            g = b + N_CTAS * w
            vs = []
            while g * 32 < total:
                vs.extend(range(g * 32, min(g * 32 + 32, total)))
                g += N_CTAS * WARPS
            owner[(b, w)] = np.asarray(vs, dtype=np.int64)
    return owner, n_chunks


def funnel(scores, rerank):
    owner, _ = deal(len(scores))
    survivors = []
    for b in range(N_CTAS):
        cta = []
        for w in range(WARPS):
            v = owner[(b, w)]
            if len(v):
                o = v[np.lexsort((v, -scores[v]))][:KEEP_WARP]        # score desc, position asc
                cta.append(o)
        if cta:
            v = np.concatenate(cta)
            survivors.append(v[np.lexsort((v, -scores[v]))][:KEEP_CTA])
    v = np.concatenate(survivors)
    return v[np.lexsort((v, -scores[v]))][:rerank]


@pytest.mark.parametrize("total", [0, 1, 31, 32, 33, 16_384, 16_385, 62_395, 200_003])
def test_every_code_is_scanned_exactly_once(total):
    owner, _ = deal(total)
    allv = np.concatenate([v for v in owner.values()]) if total else np.zeros(0, np.int64)
    assert len(allv) == total and np.array_equal(np.sort(allv), np.arange(total))


def test_model_matches_the_kernel_shape():
    assert "struct AdcTop {          // 2 entries per lane = 64 per warp" in _SRC     # KEEP_WARP
    assert WARPS * KEEP_WARP * 8 <= 32768                   # the CTA reduction keys fit dyn[32 KiB, 64 KiB)


def scores(case, total=62_395):
    rng = np.random.default_rng(3)
    s = rng.standard_normal(total).astype(np.float32)
    if case == "contiguous_cluster":
        s[20_000:20_700] += 10.0                                       # the best 700 codes are contiguous
    elif case == "two_lists":
        s[1_000:1_300] += 10.0; s[40_000:40_400] += 10.0
    elif case == "ties":
        s[5_000:9_000] = 7.0                                           # 4000 equal scores: position order decides
    return s


@pytest.mark.parametrize("case", ["uniform", "contiguous_cluster", "two_lists", "ties"])
def test_funnel_is_lossless_for_the_best_rerank(case):
    s = scores(case)
    total, rerank = len(s), 512
    want = np.arange(total)[np.lexsort((np.arange(total), -s))][:rerank]
    got = funnel(s, rerank)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("case", ["uniform", "contiguous_cluster", "two_lists", "ties"])
def test_funnel_at_rerank_1024_is_lossless_exactly_when_no_warp_or_cta_holds_more_than_64(case):
    """The precondition the header states: the funnel returns the `rerank` best codes iff no warp holds
    more than 64 and no CTA more than ADC2_KEEP of them.  two_lists puts 64 of the best 1024 plus a few
    ordinary winners into seven CTAs (chunks 31..40 and 1250..1262 share CTAs 2..8), so it must lose some."""
    s = scores(case)
    total, rerank = len(s), 1024
    want = np.arange(total)[np.lexsort((np.arange(total), -s))][:rerank]
    best = np.zeros(total, bool)
    best[want] = True
    owner, _ = deal(total)
    per_warp = max(int(best[v].sum()) for v in owner.values())
    per_cta = max(sum(int(best[owner[(b, w)]].sum()) for w in range(WARPS)) for b in range(N_CTAS))
    holds = per_warp <= KEEP_WARP and per_cta <= KEEP_CTA
    assert holds == (case != "two_lists"), (per_warp, per_cta)
    assert np.array_equal(funnel(s, rerank), want) == holds
