"""K2 route 7's plan (api.cu: batch_q8_plan), checked on the host: which batches run on the q8 copy and the int8
tensor cores at the corpus sizes where the 16-bit shadow stops fitting on an 80 GB card (~41M rows on the device,
~88M with host rows, up to the ~190M rows a host-rows corpus holds), and the invariants the kernels rely on."""
import pytest

from semtools_b200 import capi

SM = 132            # H100 SXM
MAX_SAMPLE = 49152  # the threshold kernel's 192 KiB of sampled maxima


def tiles(n):
    return (n + 255) // 256


@pytest.mark.parametrize("n_rows,k_max", [(41_000_000, 64), (45_000_000, 64), (50_000_000, 64),
                                          (88_000_000, 36), (100_000_000, 32), (190_000_000, 16)])
def test_envelope(n_rows, k_max):
    """every top_k up to k_max runs on the route, k_max + 1 does not"""
    for k in range(1, k_max + 1):
        assert capi.batch_q8_plan(SM, n_rows, k)[2], (n_rows, k)
    assert not capi.batch_q8_plan(SM, n_rows, k_max + 1)[2]


def test_envelope_formula():
    """a batch fits exactly while ceil(tiles / 49152) <= floor(256 / top_k), top_k <= 64"""
    for n_rows in (1_000_000, 10_000_000, 33_500_000, 41_000_000, 64_000_000, 100_000_000, 150_000_000, 190_000_000):
        for k in range(1, 70):
            fits = capi.batch_q8_plan(SM, n_rows, k)[2]
            assert fits == (k <= 64 and -(-tiles(n_rows) // MAX_SAMPLE) <= 256 // k), (n_rows, k)


def test_baseline_config_4():
    """100M rows, top_k = 10 (a host-rows corpus past its shadow's limit) runs on the route"""
    n_sample, stride, fits = capi.batch_q8_plan(SM, 100_000_000, 10)
    assert fits and n_sample % SM == 0 and n_sample * stride <= tiles(100_000_000)


@pytest.mark.parametrize("sm", [78, 114, 132])
def test_invariants(sm):
    for n_rows in (1, 255, 256, 5000, 300_000, 4_000_000, 45_000_000, 120_000_000, 400_000_000):
        for k in (1, 2, 10, 16, 33, 64, 65, 100):
            n_sample, stride, fits = capi.batch_q8_plan(sm, n_rows, k)
            t = tiles(n_rows)
            assert n_sample <= min(t, MAX_SAMPLE)
            if fits:
                # at least k sampled tiles, each with a real row; the sampled tiles lie inside the corpus; the
                # expected emission (8 top_k per sampled tile's share) stays within half of the 4096 keys
                assert k <= 64 and n_sample >= k and stride >= 1 and (n_sample - 1) * stride < t
                assert 8 * k * -(-t // n_sample) <= 2048
            else:
                assert stride == 0
    assert capi.batch_q8_plan(132, 45_000_000, 10) == (7128, 24, True)   # the size scripts/batch_q8_probe.py runs
