"""Host-rows corpora (stb_corpus_create_host): the f32 rows in page-locked host memory, only the q8 copy in HBM.
Every search must return, bit for bit, the hits and counts of a device corpus holding the same rows (the "twin"),
and on a subset the oracle's; the q8 copy must always cover every row and be byte-equal to what
stb_corpus_prepare(STB_PREPARE_Q8) writes on the twin; the refusals must change nothing.

The parity corpus has 300k rows (above the twin's 32768-row lazy-build threshold) plus adversarial rows:
duplicates and ties, zero rows, rows scaled by 1e-12 and 1e12 (still normalisable in fp32, so the q8 copy stays
usable) and near-copies of the queries.  A row scaled by 1e-20 (squared norm below fp32's normal range) makes the
q8 copy unusable; that case has a test of its own."""
import numpy as np
import pytest

import oracle
from conftest import unit_rows
from semtools_b200 import capi

pytestmark = pytest.mark.gpu

N = 300_000
CHUNK = 262144          # staging rows per chunk (STB_MUT_CHUNK_ROWS)
COPIES = (capi.STB_COPY_Q8_CODES, capi.STB_COPY_Q8_SCALES, capi.STB_COPY_Q8_PLANE, capi.STB_COPY_Q8_SR)
TOPKS = (1, 10, 16, 17, 50, 100, 1000)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def same_hits(a, b):
    assert len(a) == len(b)
    assert np.array_equal(bits(a), bits(b))


def adversarial_rows(rng, n):
    rows = unit_rows(rng, n)
    rows[100:110] = rows[5]                                 # exact duplicates: ties at every distance
    rows[200:204] = 0.0                                     # zero rows
    rows[300:310] *= np.float32(1e-12)
    rows[400:410] *= np.float32(1e12)
    rows[500:510] = -rows[500:510]
    return np.ascontiguousarray(rows)


def queries_for(rng, rows, nq=6):
    q = unit_rows(rng, nq)
    near = rows[[5, 1234, 77_777]] + np.float32(1e-3) * unit_rows(rng, 3)
    return np.ascontiguousarray(np.concatenate([q, near]).astype(np.float32))


def host_corpus(ctx, rows, chunks=1, capacity=1024):
    c = capi.Corpus.in_host_memory(ctx, capacity)
    for part in np.array_split(rows, chunks):
        c.append(part)
    return c


@pytest.fixture(scope="module")
def data():
    rng = np.random.default_rng(20261017)
    rows = adversarial_rows(rng, N)
    return rows, queries_for(rng, rows)


@pytest.fixture(scope="module")
def pair(ctx, data):
    rows, _ = data
    dev = capi.Corpus(ctx, N)
    dev.append(rows)
    host = host_corpus(ctx, rows, chunks=3)
    yield dev, host
    dev.close()
    host.close()


def q8_bytes(c):
    return [bits(c.debug_copy(w)[0]) for w in COPIES]


def check_q8_matches_twin(ctx, host, model):
    """the host corpus's q8 copy covers every row and equals a prepared device corpus of the same rows"""
    twin = capi.Corpus(ctx, max(len(model), 1))
    if len(model):
        twin.append(model)
    twin.prepare(1)
    got, want = q8_bytes(host), q8_bytes(twin)
    assert host.debug_copy(capi.STB_COPY_Q8_SCALES, 0, 0)[1] == len(model)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)
    assert host.tier_stats()["q8"]["built_rows"] == twin.tier_stats()["q8"]["built_rows"]
    twin.close()


def search_matrix(dev, host, queries, n):
    ranges = np.array([[10, 5000], [n // 2, n // 2 + 500], [n - 3000, n]], dtype=np.uint64)
    for mode in (capi.STB_MODE_SEARCH_DOCUMENTS, capi.STB_MODE_STORE_QUERY):
        for k in TOPKS:
            for md in (None, 0.9):
                for rr in (None, ranges, np.zeros((0, 2), dtype=np.uint64)):
                    for q in queries[[0, 6]]:
                        a = dev.search(q, k, md, mode, row_ranges=rr)
                        b = host.search(q, k, md, mode, row_ranges=rr)
                        same_hits(a, b)
    for q in queries[:3]:                                   # threshold mode (search_documents with a cap)
        same_hits(dev.search(q, 0, 0.75), host.search(q, 0, 0.75))


def batch_matrix(dev, host, queries, n):
    for k in (1, 10, 16, 100):
        for a, b in zip(dev.search_batch(queries, k), host.search_batch(queries, k)):
            same_hits(a, b)
    rr = np.array([[0, n // 3], [n // 2, n]], dtype=np.uint64)
    for k, md in ((10, None), (50, 0.9)):
        for a, b in zip(dev.search_batch_filtered(queries, rr, k, md), host.search_batch_filtered(queries, rr, k, md)):
            same_hits(a, b)
    for a, b in zip(dev.search_batch_threshold(queries, 0.8), host.search_batch_threshold(queries, 0.8)):
        same_hits(a, b)


def test_parity_matrix(ctx, data, pair):
    rows, queries = data
    dev, host = pair
    check_q8_matches_twin(ctx, host, rows)
    search_matrix(dev, host, queries, N)
    for k in (1, 10, 16):
        for a, b in zip(dev.search_many(queries, k), host.search_many(queries, k)):
            same_hits(a, b)
    import torch
    q_dev = torch.from_numpy(queries[0]).cuda()
    torch.cuda.synchronize()
    for k in (1, 10, 16):
        outs = []
        for c in (dev, host):
            hits = torch.zeros(k * 2, dtype=torch.float64, device="cuda")
            st = torch.zeros(8, dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            c.search_topk_dev(q_dev.data_ptr(), k, hits.data_ptr(), st.data_ptr())
            ctx.sync()
            outs.append((hits.cpu().numpy().view(np.uint8).copy(), st.cpu().numpy()[:2].copy()))
        if outs[0][1][1] and outs[1][1][1]:                  # both proven: the same hits
            assert np.array_equal(outs[0][0], outs[1][0]) and outs[0][1][0] == outs[1][1][0]
    batch_matrix(dev, host, queries, N)
    # a subset against the oracle
    for q in queries[[0, 7]]:
        r, d = oracle.search_rows(rows, q, top_k=10)
        h = host.search(q, 10)
        assert np.array_equal(h["row"], np.asarray(r, dtype=np.uint64)) and np.array_equal(h["distance"], d)


def test_unusable_q8_copy_takes_the_f32_route(ctx, data):
    rows, queries = data
    bad = rows[:120_000].copy()
    bad[321] = unit_rows(np.random.default_rng(3), 1)[0] * np.float32(1e-20)
    dev = capi.Corpus(ctx, len(bad)); dev.append(bad)
    host = host_corpus(ctx, bad)
    assert host.tier_stats()["q8"]["built_rows"] == 0
    check_q8_matches_twin(ctx, host, bad)
    search_matrix(dev, host, queries, len(bad))
    batch_matrix(dev, host, queries, len(bad))
    with pytest.raises(capi.StbError) as e:                  # no HBM copy serves it: refused, not streamed
        host.search_many(queries, 10)
    assert e.value.status == capi.STB_ERR_STATE
    dev.close(); host.close()


def test_mutations_keep_rows_copies_and_hits(ctx, table_small):
    rng = np.random.default_rng(7)
    E, tab = table_small
    model = unit_rows(rng, 5000)
    host = capi.Corpus.in_host_memory(ctx, 16)               # grows several times
    for part in np.array_split(model, 4):
        host.append(part)
    import torch
    extra = unit_rows(rng, 3000)
    extra_dev = torch.from_numpy(extra).cuda()
    torch.cuda.synchronize()                                 # the context's stream does not wait for torch's
    host.append_dev(extra_dev.data_ptr(), len(extra))
    model = np.concatenate([model, extra])
    qs = unit_rows(rng, 3)

    def step():
        assert len(host) == len(model)
        assert np.array_equal(bits(host.read()), bits(model))
        check_q8_matches_twin(ctx, host, model)
        twin = capi.Corpus(ctx, max(len(model), 1)); twin.append(model)
        for q in qs:
            for k in (10, 50):
                same_hits(twin.search(q, k), host.search(q, k))
        twin.close()

    step()
    # K3 into the corpus with more lines than one staging chunk
    n_lines = CHUNK + 1000
    lens = rng.integers(1, 4, n_lines)
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    ids = rng.integers(0, E.shape[0], int(offsets[-1])).astype(np.uint32)
    out = capi.embed(ctx, tab, offsets, ids, out=True, append_to=host)
    model = np.concatenate([model, out])
    step()
    # a refused K3 call (token outside the table) appends nothing
    before = [bits(host.read())] + q8_bytes(host)
    bad_ids = ids[:10].copy(); bad_ids[3] = E.shape[0] + 5
    with pytest.raises(capi.StbError):
        capi.embed(ctx, tab, np.arange(11, dtype=np.uint64), bad_ids, out=False, append_to=host)
    for x, y in zip([bits(host.read())] + q8_bytes(host), before):
        assert np.array_equal(x, y)
    idx = np.sort(rng.choice(len(model), 700, replace=False)).astype(np.uint64)
    new = unit_rows(rng, 700)
    host.update(idx, new)
    model[idx.astype(np.int64)] = new
    step()
    ranges = np.array([[3, 50], [4000, 4100], [len(model) - 10, len(model)]], dtype=np.uint64)
    host.remove(ranges)
    keep = np.ones(len(model), bool)
    for b, e in ranges.astype(np.int64):
        keep[b:e] = False
    model = np.ascontiguousarray(model[keep])
    step()
    # refused calls: bad ranges, unsorted ids -> rows and copies byte for byte unchanged
    before = [bits(host.read())] + q8_bytes(host)
    with pytest.raises(capi.StbError) as e1:
        host.remove(np.array([[10, 5], [20, 30]], dtype=np.uint64))
    with pytest.raises(capi.StbError) as e2:
        host.update(np.array([9, 3], dtype=np.uint64), unit_rows(rng, 2))
    assert e1.value.status == capi.STB_ERR_RANGE and e2.value.status == capi.STB_ERR_RANGE
    for x, y in zip([bits(host.read())] + q8_bytes(host), before):
        assert np.array_equal(x, y)
    # an update that writes an unnormalisable row, then one that replaces it again
    host.update(np.array([17], dtype=np.uint64), model[17:18] * np.float32(1e-20))
    model[17] *= np.float32(1e-20)
    step()
    assert host.tier_stats()["q8"]["built_rows"] == 0
    fix = unit_rows(rng, 1)
    host.update(np.array([17], dtype=np.uint64), fix)
    model[17] = fix[0]
    step()
    assert host.tier_stats()["q8"]["built_rows"] == len(model)
    host.clear()
    model = unit_rows(rng, 2000)
    host.append(model)
    step()
    host.close()


@pytest.fixture(scope="module")
def table_small(ctx):
    E = unit_rows(np.random.default_rng(11), 500)
    t = capi.Table(ctx, E)
    yield E, t
    t.close()


def test_routes_read_no_f32_rows(ctx, data, pair):
    rows, _ = data
    dev, _ = pair
    host = host_corpus(ctx, rows)
    rng = np.random.default_rng(99)
    qs = unit_rows(rng, 12)
    fb0 = ctx.counters()["fallback_searches"]
    f32_0 = host.tier_stats()["f32"]["tries"]
    for q in qs:
        host.search(q, 10)
    st = host.tier_stats()
    assert st["f32"]["tries"] == f32_0 and st["q8"]["proven"] >= len(qs)
    assert ctx.counters()["fallback_searches"] == fb0
    assert st["h16"]["built_rows"] == 0                     # never built lazily on host rows
    for q in qs[:4]:                                         # k = 50, no shadow: the q8 histogram / collect route
        same_hits(dev.search(q, 50), host.search(q, 50))
    assert host.tier_stats()["f32"]["tries"] == f32_0
    assert ctx.counters()["fallback_searches"] == fb0
    host.close()


def test_refusals_change_nothing(ctx, data):
    rows, _ = data
    host = host_corpus(ctx, rows[:50_000])
    before = [bits(host.read())] + q8_bytes(host)
    launches = ctx.counters()["kernel_launches"]
    import torch
    q_dev = torch.from_numpy(rows[0]).cuda()
    hits = torch.zeros(64 * 2, dtype=torch.float64, device="cuda")
    st = torch.zeros(8, dtype=torch.int32, device="cuda")
    calls = [
        lambda: host.data_dev,
        lambda: capi.IvfPq(host, nlist=16, train_rows=4096),
        lambda: host.search_topk_dev(q_dev.data_ptr(), 17, hits.data_ptr(), st.data_ptr()),
        lambda: host.search_many(rows[:2], 17),
    ]
    x = capi.Exchange(ctx, 1, 0, 16, max_nq=4)
    calls += [
        lambda: x.search(host, rows[0], 10),
        lambda: x.search_topk(host, q_dev.data_ptr(), 10, hits.data_ptr(), st.data_ptr()),
        lambda: x.search_batch_dev(host, q_dev.data_ptr(), 1, 10, hits.data_ptr(), st.data_ptr()),
        lambda: host.search_many(rows[:2], 10, xchg=x),
    ]
    for call in calls:
        with pytest.raises(capi.StbError) as e:
            call()
        assert e.value.status == capi.STB_ERR_STATE
    assert ctx.counters()["kernel_launches"] == launches
    for a, b in zip([bits(host.read())] + q8_bytes(host), before):
        assert np.array_equal(a, b)
    x.close(); host.close()


def test_python_store_builds_a_host_mirror_when_hbm_is_full(ctx, tmp_path, monkeypatch):
    from semtools_b200.workspace import LineEmbedding, Store
    rng = np.random.default_rng(5)

    def lines(path, n, scale=1.0):
        return [LineEmbedding(path, i, unit_rows(rng, 1)[0] * np.float32(scale)) for i in range(n)]

    docs = lines("a.txt", 400) + lines("b.txt", 300) + lines("c.txt", 200)
    sd, sh = Store.open(str(tmp_path / "d"), ctx), Store.open(str(tmp_path / "h"), ctx)
    for s in (sd, sh):
        s.upsert_line_embeddings(docs)
    real_init = capi.Corpus.__init__

    def nomem(self, *a, **k):
        raise capi.StbError(capi.STB_ERR_NOMEM, "device mirror does not fit")

    qs = unit_rows(rng, 4)

    def compare():
        for subset in (["a.txt", "c.txt"], ["b.txt"]):
            for q in qs:
                assert sd.search_line_embeddings(q, subset, 7) == sh.search_line_embeddings(q, subset, 7)
            assert sd.search_line_embeddings_batch(qs, subset, 5, 0.99) == sh.search_line_embeddings_batch(qs, subset, 5, 0.99)

    monkeypatch.setattr(capi.Corpus, "__init__", nomem)
    sh._gpu_corpus()
    monkeypatch.setattr(capi.Corpus, "__init__", real_init)
    assert sh._corpus.host_rows and not sd._gpu_corpus().host_rows
    compare()
    upd = lines("a.txt", 10, 2.0) + lines("d.txt", 50)
    for s in (sd, sh):
        s.upsert_line_embeddings(upd)
    compare()
    for s in (sd, sh):
        s.delete_documents(["b.txt"])
    compare()
    assert sh._corpus.host_rows


def test_lifetime_corpus_after_context(data):
    rows, _ = data
    c2 = capi.Context(0)
    host = host_corpus(c2, rows[:40_000])
    host.search(rows[1], 10)
    c2.close()                                               # the corpus outlives its context
    host.close()
    c3 = capi.Context(0)
    h = host_corpus(c3, rows[:40_000], chunks=2)
    h.update(np.array([5], dtype=np.uint64), rows[6:7])
    h.close()                                                # destroyed in the middle of a workflow
    c3.sync()
    c3.close()


CPP_DRIVER = r"""
#include <cstdio>
#include <cstring>
#include <vector>
#include "semtools_store.hpp"
static int nomem(stb_ctx *, uint32_t, uint64_t, uint64_t, stb_corpus **) { return STB_ERR_NOMEM; }
int main(int argc, char **argv) {
  if (argc != 3) return 2;
  auto load = [](const char *p) { std::vector<float> v; FILE *f = fopen(p, "rb"); float x;
                                   while (fread(&x, 4, 1, f) == 1) v.push_back(x); fclose(f); return v; };
  std::vector<float> rows = load(argv[1]), qs = load(argv[2]);
  const uint64_t n = rows.size() / 256, nq = qs.size() / 256;
  stb_ctx *ctx = nullptr; stb_corpus *dev = nullptr, *host = nullptr;
  if (stb_ctx_create(0, nullptr, &ctx)) return 3;
  if (semtools::upload_mirror(ctx, rows.data(), n, &dev) || semtools::upload_mirror(ctx, rows.data(), n, &host, nomem)) return 4;
  float *p = nullptr;
  if (stb_corpus_data_dev(dev, &p) != STB_OK || stb_corpus_data_dev(host, &p) != STB_ERR_STATE) return 5;
  const uint64_t ranges[4] = {0, n / 3, n / 2, n};
  for (uint64_t i = 0; i < nq; ++i) {
    stb_hit a[20], b[20]; uint64_t na = 0, nb = 0;
    memset(a, 0, sizeof(a)); memset(b, 0, sizeof(b));
    if (stb_search(ctx, dev, &qs[i * 256], 20, 1, 0.95, STB_MODE_STORE_QUERY, ranges, 2, a, 20, &na) ||
        stb_search(ctx, host, &qs[i * 256], 20, 1, 0.95, STB_MODE_STORE_QUERY, ranges, 2, b, 20, &nb)) return 6;
    if (na != nb || memcmp(a, b, sizeof(a)) != 0) { printf("differ at query %llu\n", (unsigned long long)i); return 7; }
  }
  stb_corpus_destroy(dev); stb_corpus_destroy(host); stb_ctx_destroy(ctx);
  printf("mirror rule ok\n");
  return 0;
}
"""


def test_cpp_store_builds_a_host_mirror_when_hbm_is_full(tmp_path):
    """semtools::upload_mirror with a device attempt that fails with STB_ERR_NOMEM: the mirror keeps its rows in
    host memory and the store query returns the device mirror's hits"""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = os.path.join(root, "semtools_b200", "lib")
    (tmp_path / "drv.cpp").write_text(CPP_DRIVER)
    host = os.path.join(root, "semtools_b200", "host")
    subprocess.run(["/usr/bin/g++", "-std=c++17", "-O2", "-I", host, "-I", os.path.join(root, "include"),
                    "-o", str(tmp_path / "drv"), str(tmp_path / "drv.cpp"), os.path.join(host, "semtools_store.cpp"),
                    os.path.join(host, "semtools_host.cpp"), "-L", lib, "-lsemtools_b200", f"-Wl,-rpath,{lib}"], check=True)
    rng = np.random.default_rng(21)
    unit_rows(rng, 70_000).tofile(tmp_path / "rows.f32")
    unit_rows(rng, 8).tofile(tmp_path / "q.f32")
    r = subprocess.run([str(tmp_path / "drv"), str(tmp_path / "rows.f32"), str(tmp_path / "q.f32")],
                       capture_output=True, text=True)
    assert r.returncode == 0 and "mirror rule ok" in r.stdout, (r.returncode, r.stdout, r.stderr)
