"""GPU: K4 hits merge (csrc/hits_merge.cu) at its edges, against a plain f64 sort written here.

Reference: drop every entry whose row is UINT64_MAX (padding) or whose distance is NaN, then sort by
(distance, row) with Python floats and ints.  -0.0 and +0.0 compare equal there, so they tie and are
ordered by row; the merged entries must keep their own bits.  Inputs are unsorted lists with many ties,
padding in the middle, NaN distances, +inf on real rows and rows at and above 2^32 and 2^63; rows are
unique within a merge, so the expected order is fully determined.

The three entry points are checked against the reference and against each other:
  - stb_hits_merge (host buffers): totals around the power-of-two sort sizes up to the 4096-hit capacity;
  - stb_hits_merge_dev: exactly top_k entries written, with a (+inf, UINT64_MAX) tail;
  - stb_hits_merge_batch_dev: the [n_lists][nq][per_list] layout, up to 2048 hits per query.
"""
import ctypes as C

import numpy as np
import pytest

from semtools_b200 import capi

pytestmark = pytest.mark.gpu

NO_ROW = np.uint64(0xFFFFFFFFFFFFFFFF)
MERGE_CAP = 4096          # hits one stb_hits_merge(_dev) call merges
BATCH_CAP = 2048          # hits per query of stb_hits_merge_batch_dev
SENTINEL = 0xAB           # byte pattern of output memory the merge must not touch


@pytest.fixture(scope="module")
def torch():
    return pytest.importorskip("torch")


def ref_merge(flat):
    """The merged order of a 1-D HIT_DTYPE array: valid entries sorted by (f64 distance, row)."""
    flat = np.ascontiguousarray(flat).reshape(-1)
    keep = (flat["row"] != NO_ROW) & ~np.isnan(flat["distance"])
    v = flat[keep]
    order = sorted(range(len(v)), key=lambda i: (float(v["distance"][i]), int(v["row"][i])))
    return v[np.asarray(order, dtype=np.int64)]


def padded(hits, k):
    """hits[:k] followed by (+inf, UINT64_MAX) up to k entries."""
    out = np.zeros(k, dtype=capi.HIT_DTYPE)
    out["distance"] = np.inf
    out["row"] = NO_ROW
    n = min(k, len(hits))
    out[:n] = hits[:n]
    return out


def raw(h):
    """Hits as raw bytes: distances compared bit for bit (-0.0 != +0.0 here)."""
    return np.ascontiguousarray(h, dtype=capi.HIT_DTYPE).view(np.uint8)


def edge_hits(rng, shape):
    """Unsorted hits with many ties, -0.0 / +0.0, +inf on real rows, NaN distances (several payloads),
    padding anywhere, and unique rows below 2^32, at 2^32 and above 2^63."""
    n = int(np.prod(shape))
    h = np.zeros(n, dtype=capi.HIT_DTYPE)
    ties = np.array([0.0, -0.0, 0.125, 0.25, 0.5, 1.0, 1.5, 2.0, np.inf])
    d = rng.choice(ties, n)
    fresh = rng.random(n) < 0.3
    d[fresh] = rng.uniform(-0.5, 2.0, int(fresh.sum()))
    nan = rng.random(n) < 0.05
    nans = np.array([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0x7FF80000DEADBEEF],
                    dtype=np.uint64).view(np.float64)
    d[nan] = rng.choice(nans, int(nan.sum()))
    h["distance"] = d
    bases = np.array([0, 1 << 32, 1 << 63, (1 << 64) - (1 << 20)], dtype=np.uint64)
    h["row"] = rng.permutation(n).astype(np.uint64) + rng.choice(bases, n)
    pad = rng.random(n) < 0.1
    h["row"][pad] = NO_ROW                         # padding carries any distance, finite ones included
    return h.reshape(shape)


def n_valid(h):
    h = h.reshape(-1)
    return int(((h["row"] != NO_ROW) & ~np.isnan(h["distance"])).sum())


# ------------------------------------------------------------------------------ reference self-check ---
def test_reference_orders_signed_zeros_and_inf_as_documented():
    h = np.zeros(7, dtype=capi.HIT_DTYPE)
    h["distance"] = [np.inf, 0.0, -0.0, np.nan, 0.0, -1.0, 0.5]
    h["row"] = [1, 9, 3, 0, 2 ** 63, 7, NO_ROW]
    got = ref_merge(h)
    assert got["row"].tolist() == [7, 3, 9, 2 ** 63, 1]
    assert np.signbit(got["distance"]).tolist() == [True, True, False, False, False]


# -------------------------------------------------------------------------------------- host form ---
SHAPES = {1: (1, 1), 2: (2, 1), 3: (1, 3), 255: (15, 17), 256: (16, 16), 257: (1, 257), 1000: (8, 125),
          2047: (23, 89), 2048: (64, 32), 2049: (3, 683), 4095: (4095, 1), 4096: (2, 2048)}


@pytest.mark.parametrize("total", sorted(SHAPES))
def test_host_merge_matches_the_f64_sort(ctx, total):
    n_lists, per_list = SHAPES[total]
    rng = np.random.default_rng(0x4E + total)
    lists = edge_hits(rng, (n_lists, per_list))
    if total > 1:
        lists["row"][0, 0] = 5                    # at least one valid hit in every shape
        lists["distance"][0, 0] = 0.5
    want = ref_merge(lists)
    assert len(want) == n_valid(lists)
    for k in sorted({1, total - 1, total, total + 5} - {0}):
        got = ctx.hits_merge(lists, k)
        assert len(got) == min(k, len(want)), (total, k)
        assert np.array_equal(raw(got), raw(want[:k])), (total, k)


def test_host_merge_single_entry_edges(ctx):
    for d, r, keep in [(np.inf, 0, True), (-0.0, (1 << 64) - 2, True), (np.nan, 4, False), (0.0, NO_ROW, False)]:
        h = np.zeros((1, 1), dtype=capi.HIT_DTYPE)
        h["distance"], h["row"] = d, r
        got = ctx.hits_merge(h, 3)
        assert np.array_equal(raw(got), raw(h.reshape(-1)[:1] if keep else h.reshape(-1)[:0])), (d, r)


def test_host_merge_over_capacity_is_an_argument_error_and_writes_nothing(ctx):
    lists = edge_hits(np.random.default_rng(7), (1, MERGE_CAP + 1))
    out = np.zeros(8, dtype=capi.HIT_DTYPE)
    out.view(np.uint8)[:] = SENTINEL
    before = out.copy()
    n = C.c_uint32(0)
    rc = capi.lib().stb_hits_merge(ctx._h, lists.ctypes.data_as(C.c_void_p), 1, MERGE_CAP + 1, 8,
                                   out.ctypes.data_as(C.c_void_p), C.byref(n))
    assert rc == capi.STB_ERR_ARG
    assert np.array_equal(raw(out), raw(before))
    assert n.value == 0
    assert len(ctx.hits_merge(lists[:, :MERGE_CAP], 8)) == 8          # the context still merges


# --------------------------------------------------------------------------------------- dev form ---
def to_dev(torch, h):
    return torch.from_numpy(np.ascontiguousarray(h).view(np.uint8).reshape(-1).copy()).to("cuda:0")


def from_dev(buf):
    return buf.cpu().numpy().view(capi.HIT_DTYPE)


def sentinel_out(torch, n_hits):
    return torch.full((n_hits * 16,), SENTINEL, dtype=torch.uint8, device="cuda:0")


@pytest.mark.parametrize("n_lists,per_list", [(1, 1), (1, 3), (16, 16), (3, 683), (4095, 1), (2, 2048)])
def test_dev_merge_writes_exactly_top_k_and_equals_the_host_form(ctx, torch, n_lists, per_list):
    total = n_lists * per_list
    rng = np.random.default_rng(0xDE + total)
    lists = edge_hits(rng, (n_lists, per_list))
    want = ref_merge(lists)
    guard = 4
    lists_d = to_dev(torch, lists)
    for k in sorted({1, max(total - 1, 1), total, total + 5}):
        out_d = sentinel_out(torch, k + guard)
        torch.cuda.synchronize()
        ctx.hits_merge_dev(lists_d.data_ptr(), n_lists, per_list, k, out_d.data_ptr())
        ctx.sync()
        got = from_dev(out_d)
        assert np.array_equal(raw(got[:k]), raw(padded(want, k))), (n_lists, per_list, k)
        assert (out_d[k * 16:].cpu().numpy() == SENTINEL).all()            # nothing past top_k
        host = ctx.hits_merge(lists, k)
        assert np.array_equal(raw(got[:len(host)]), raw(host))
        assert (got["row"][len(host):k] == NO_ROW).all()


def test_dev_merge_arguments(ctx, torch):
    lists_d = to_dev(torch, edge_hits(np.random.default_rng(9), (1, MERGE_CAP + 1)))
    out_d = sentinel_out(torch, 8)
    torch.cuda.synchronize()
    for n_lists, per_list, k in [(1, MERGE_CAP + 1, 8), (0, 4, 8), (1, 0, 8), (1, 4, 0)]:
        with pytest.raises(capi.StbError) as e:
            ctx.hits_merge_dev(lists_d.data_ptr(), n_lists, per_list, k, out_d.data_ptr())
        assert e.value.status == capi.STB_ERR_ARG
    ctx.sync()
    assert (out_d.cpu().numpy() == SENTINEL).all()


# ------------------------------------------------------------------------------------- batch form ---
@pytest.mark.parametrize("n_lists,nq,per_list,top_k",
                         [(1, 1, 1, 1), (2, 5, 10, 10), (8, 3, 256, 256), (3, 4096, 7, 5), (16, 17, 128, 200),
                          (5, 9, 409, 100)])
def test_batch_merge_layout_matches_the_f64_sort_per_query(ctx, torch, n_lists, nq, per_list, top_k):
    rng = np.random.default_rng(n_lists * 1000 + nq * 10 + per_list)
    lists = edge_hits(rng, (n_lists, nq, per_list))            # every query different content
    lists_d = to_dev(torch, lists)
    guard = 4
    out_d = sentinel_out(torch, nq * top_k + guard)
    torch.cuda.synchronize()
    ctx.hits_merge_batch_dev(lists_d.data_ptr(), n_lists, nq, per_list, top_k, out_d.data_ptr())
    ctx.sync()
    got = from_dev(out_d)
    assert (out_d[nq * top_k * 16:].cpu().numpy() == SENTINEL).all()
    got = got[:nq * top_k].reshape(nq, top_k)
    for q in range(nq):
        want = padded(ref_merge(lists[:, q, :]), top_k)
        assert np.array_equal(raw(got[q]), raw(want)), q
    # each query's row == stb_hits_merge_dev on that query's lists alone
    qs = range(nq) if nq <= 32 else sorted({0, nq - 1, *rng.choice(nq, 14, replace=False).tolist()})
    for q in qs:
        one_d = to_dev(torch, lists[:, q, :])
        single = sentinel_out(torch, top_k)
        torch.cuda.synchronize()
        ctx.hits_merge_dev(one_d.data_ptr(), n_lists, per_list, top_k, single.data_ptr())
        ctx.sync()
        assert np.array_equal(raw(from_dev(single)), raw(got[q])), q


def test_batch_merge_capacity_and_empty_batch(ctx, torch):
    lists_d = to_dev(torch, edge_hits(np.random.default_rng(11), (3, 2, 683)))       # 2049 hits per query
    out_d = sentinel_out(torch, 2 * 10)
    torch.cuda.synchronize()
    with pytest.raises(capi.StbError) as e:
        ctx.hits_merge_batch_dev(lists_d.data_ptr(), 3, 2, 683, 10, out_d.data_ptr())
    assert e.value.status == capi.STB_ERR_ARG
    ctx.hits_merge_batch_dev(lists_d.data_ptr(), 3, 0, 683, 10, out_d.data_ptr())     # nq = 0: no-op
    ctx.sync()
    assert (out_d.cpu().numpy() == SENTINEL).all()
    # 2048 hits per query is the edge that still merges
    ctx.hits_merge_batch_dev(lists_d.data_ptr(), 2, 2, 1024, 10, out_d.data_ptr())
    ctx.sync()
    flat = from_dev(lists_d)[:2 * 2 * 1024].reshape(2, 2, 1024)
    got = from_dev(out_d).reshape(2, 10)
    for q in range(2):
        assert np.array_equal(raw(got[q]), raw(padded(ref_merge(flat[:, q, :]), 10)))
