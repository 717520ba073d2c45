"""GPU: K5 IVF-PQ saved to a file and loaded onto its corpus (stb_ivfpq_save / stb_ivfpq_load, csrc/ivfpq.cu).

The file format and the digest are restated here from include/semtools_b200.h: `digest` is a numpy restatement
of the header's definition, `read_file` / `write_file` take a file apart and put one together with every
checksum recomputed, so a crafted file passes the checksums and reaches the GPU checks it is aimed at.  A loaded
index is held to the index it was saved from: the same export and statistics, the same hits on every search
mode, and the same results of extend, update and remove afterwards.
"""

import os
import struct
import sys

import numpy as np
import pytest

import oracle
from semtools_b200 import capi

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_corpus_update import bits  # noqa: E402
from test_gpu_ivfpq_batch import clustered, edge_queries, make_centers  # noqa: E402

pytestmark = pytest.mark.gpu

# ------------------------------------------------------------------------- the header's definitions ---
HEADER = struct.Struct("<8s6I4Q18QQ")            # magic, version, d, pq_m, pq_ksub, pq_dsub, nlist, n, n_listed,
assert HEADER.size == 216                        # n_forced, rows_digest, 6 x {offset, bytes, checksum}, header_checksum
SECTIONS = ("centroids", "codebooks", "list_off", "order", "codes", "forced")
K1, K2, K3 = np.uint64(0x9E3779B97F4A7C15), np.uint64(0xC2B2AE3D27D4EB4F), np.uint64(0x165667B19E3779F9)


def mix(z):
    z = np.asarray(z, np.uint64)
    with np.errstate(over="ignore"):
        z = z ^ (z >> np.uint64(30)); z = z * np.uint64(0xBF58476D1CE4E5B9)
        z = z ^ (z >> np.uint64(27)); z = z * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def digest(data: bytes) -> int:
    L = len(data)
    padded = bytes(data) + bytes(-L % 1024)
    w = np.frombuffer(padded, dtype="<u8").reshape(-1, 128)
    with np.errstate(over="ignore"):
        h = mix(w ^ (np.arange(1, 129, dtype=np.uint64) * K1)).sum(axis=1, dtype=np.uint64)
        d = mix(h ^ (np.arange(1, len(w) + 1, dtype=np.uint64) * K2)).sum(dtype=np.uint64)
        return int((d + mix(np.uint64(L) ^ K3)) & np.uint64(0xFFFFFFFFFFFFFFFF))


def read_file(path):
    raw = open(path, "rb").read()
    f = HEADER.unpack(raw[:216])
    hdr = dict(magic=f[0], version=f[1], d=f[2], pq_m=f[3], pq_ksub=f[4], pq_dsub=f[5], nlist=f[6], n=f[7], n_listed=f[8],
               n_forced=f[9], rows_digest=f[10], header_checksum=f[29])
    secs = [(f[11 + 3 * k], f[12 + 3 * k], f[13 + 3 * k]) for k in range(6)]
    return hdr, {name: raw[o:o + b] for name, (o, b, _) in zip(SECTIONS, secs)}, secs


def write_file(path, hdr, sec):
    """a file of these header fields and sections, laid out and checksummed as the header defines"""
    off, table, body = 216, [], b""
    for name in SECTIONS:
        b = bytes(sec[name])
        table += [off, len(b), digest(b)]
        off += len(b)
        body += b
    head = HEADER.pack(hdr["magic"], hdr["version"], hdr["d"], hdr["pq_m"], hdr["pq_ksub"], hdr["pq_dsub"], hdr["nlist"], hdr["n"],
                       hdr["n_listed"], hdr["n_forced"], hdr["rows_digest"], *table, 0)
    head = head[:208] + struct.pack("<Q", digest(head[:208]))
    with open(path, "wb") as fh:
        fh.write(head + body)


# ------------------------------------------------------------------------------------------ helpers ---
def same_export(a, b):
    return all(np.array_equal(bits(a[k]), bits(b[k])) for k in SECTIONS)


def clone(ctx, c, row_base=None, extra=0):
    """a second corpus holding c's rows"""
    rows = c.read()
    d = capi.Corpus(ctx, len(rows) + extra, row_base=c.row_base if row_base is None else row_base)
    d.append(rows)
    return d


def history(rng, centers, idx, c, base):
    """extend, update (listed <-> forced moves) and remove on idx; the same calls on two indexes give the same index"""
    n = len(c)
    c.append(clustered(rng, centers, 1500))
    idx.extend()
    forced = idx.export()["forced"]
    loc = np.unique(np.concatenate([forced[:2].astype(np.int64), rng.choice(n, 400, replace=False)]))
    vals = clustered(rng, centers, len(loc))
    vals[5] = 0.0; vals[9, 4] = np.nan                                    # listed -> forced
    idx.update(loc + base, vals)                                          # forced[:2] -> listed
    idx.remove(np.array([[base + 10, base + 60], [base + 3000, base + 3001]], np.uint64))


def all_searches(idx, c, Q):
    """every search mode's answer to Q, as plain arrays"""
    torch = pytest.importorskip("torch")
    base, n = c.row_base, idx.stats()["rows"]
    out = []
    for rerank in (256, 2048):                                            # fused v2, then v1
        for q in Q:
            out.append(idx.search(q, nprobe=8, top_k=10, rerank=rerank)[0])
    dev = torch.device("cuda:0")
    q_dev = torch.from_numpy(np.ascontiguousarray(Q)).to(dev)
    hits = torch.zeros((10, 2), dtype=torch.float64, device=dev)
    st = torch.zeros(2, dtype=torch.int32, device=dev)
    for i in range(len(Q)):
        idx.search_dev(q_dev[i].data_ptr(), 8, 10, 256, hits.data_ptr(), st.data_ptr())
        c.ctx.sync()
        out += [hits.cpu().numpy().copy(), st.cpu().numpy().copy()]
    out += list(idx.search_batch(Q, nprobe=8, top_k=10, rerank=512))
    ranges = np.array([[base + 5, base + 900], [base + 2000, base + n // 2]], np.uint64)
    for dist in (None, 0.8):
        out += list(idx.search_filtered(Q, ranges, max_distance=dist, nprobe=8, top_k=10, rerank=256))
    subsets = [ranges, np.array([[base + n // 3, base + n]], np.uint64), np.zeros((0, 2), np.uint64)]
    out += list(idx.search_subsets(Q, subsets, np.arange(len(Q)) % 3, nprobe=8, top_k=10, rerank=256))
    thr, scanned, reranked = idx.search_threshold(Q, nprobe=8, max_distance=0.35)
    out += thr + [scanned, reranked]
    return out


def assert_same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert np.array_equal(bits(np.asarray(x)), bits(np.asarray(y)))


def edge_rows(rng, centers, n):
    rows = clustered(rng, centers, n)
    rows[11, 7] = np.nan; rows[n // 3] = 0.0; rows[n // 2 + 1] *= np.float32(1e-20)    # forced rows
    return rows


def make_saved(ctx, path, rows=20_000, nlist=48):
    """an index built, then extended, updated and removed from, then saved to path; its corpus and queries"""
    rng = np.random.default_rng(8101)
    centers = make_centers(rng, nlist)
    base = 7 << 32
    c = capi.Corpus(ctx, 2 * rows, row_base=base)
    c.append(edge_rows(rng, centers, rows))
    idx = capi.IvfPq(c, nlist=nlist, train_rows=rows, iters=4)
    history(rng, centers, idx, c, base)
    E = idx.export()
    assert len(E["forced"]) >= 2
    idx.save(path)
    R = c.read()
    Q = np.concatenate([clustered(rng, centers, 12), np.stack(edge_queries(rng, R, rng.permutation(len(R))[:16]))])
    return c, idx, Q, centers, base


@pytest.fixture(scope="module")
def saved(ctx, tmp_path_factory):
    path = str(tmp_path_factory.mktemp("ivf") / "index.stbivf")
    c, idx, Q, centers, base = make_saved(ctx, path)
    yield c, idx, path, Q, centers, base
    idx.close(); c.close()


# --------------------------------------------------------------------------------------- round trip ---
def test_round_trip_after_history_is_the_same_index(ctx, saved):
    c, idx, path, Q, _, _ = saved
    E, S = idx.export(), idx.stats()
    d = clone(ctx, c)
    loaded = capi.IvfPq.load(d, path)
    try:
        assert same_export(loaded.export(), E) and loaded.stats() == S
        assert_same(all_searches(loaded, d, Q), all_searches(idx, c, Q))
        assert loaded.load_ms()[0] > 0 and idx.load_ms() == (0.0, 0.0)
        on_c = capi.IvfPq.load(c, path)                                   # a second index on the same corpus
        assert_same(all_searches(on_c, c, Q), all_searches(idx, c, Q))
        on_c.close()
    finally:
        loaded.close(); d.close()


def test_exhaustive_probe_of_a_loaded_index_equals_stb_search(ctx, tmp_path):
    """the index saved after extend, update and remove, small enough (listed rows <= 4096) that rerank 4096
    re-ranks every listed row"""
    c, idx, Q, _, _ = make_saved(ctx, tmp_path / "small", rows=2000, nlist=8)
    idx.close()
    loaded = capi.IvfPq.load(c, tmp_path / "small")
    try:
        assert len(loaded.export()["order"]) <= 4096
        for q in Q:
            for top_k in (1, 10, 100):
                got, scanned = loaded.search(q, nprobe=8, top_k=top_k, rerank=4096)
                assert scanned == len(loaded.export()["order"])
                assert np.array_equal(bits(got), bits(c.search(q, top_k=top_k)))
    finally:
        loaded.close(); c.close()


def test_after_the_load_calls_behave_as_on_the_original(ctx, tmp_path):
    """rows appended since the save, then extend, update and remove on the original index and on the loaded
    one (on a copy of the original's corpus): the same exports and hits on both sides"""
    path = tmp_path / "index"
    a, ia, Q, centers, base = make_saved(ctx, path)                        # the original, with its history
    b = clone(ctx, a, extra=4000)
    ib = capi.IvfPq.load(b, path)
    n0 = ia.stats()["rows"]
    try:
        assert same_export(ia.export(), ib.export())
        new = clustered(np.random.default_rng(5), centers, 2000)
        new[3] = 0.0
        for x, cx in ((ia, a), (ib, b)):
            cx.append(new)
            assert x.stats()["rows"] == n0                                   # appended rows stay outside until extend
            assert x.extend() == 2000
            history(np.random.default_rng(6), centers, x, cx, base)
        assert same_export(ia.export(), ib.export()) and ia.stats() == ib.stats()
        assert np.array_equal(bits(a.read()), bits(b.read()))
        assert_same(all_searches(ia, a, Q), all_searches(ib, b, Q))
        # and a save of the edited loaded index loads again to the same index
        ib.save(tmp_path / "again")
        ic = capi.IvfPq.load(a, tmp_path / "again")
        assert same_export(ic.export(), ia.export())
        ic.close()
    finally:
        ia.close(); ib.close(); a.close(); b.close()


def test_a_corpus_with_another_row_base_shifts_the_hits(ctx, saved):
    c, idx, path, Q, _, base = saved
    d = clone(ctx, c, row_base=base + 12345)
    loaded = capi.IvfPq.load(d, path)
    try:
        want, wn, _ = idx.search_batch(Q, nprobe=8, top_k=10, rerank=256)
        got, gn, _ = loaded.search_batch(Q, nprobe=8, top_k=10, rerank=256)
        assert np.array_equal(gn, wn)
        for i in range(len(Q)):
            k = int(wn[i])
            assert np.array_equal(got[i][:k]["row"], want[i][:k]["row"] + np.uint64(12345))
            assert np.array_equal(bits(got[i][:k]["distance"]), bits(want[i][:k]["distance"]))
    finally:
        loaded.close(); d.close()


# ------------------------------------------------------------------------------------------- save ---
def test_save_is_deterministic_changes_nothing_and_matches_the_restated_format(ctx, saved, tmp_path):
    c, idx, path, _, _, _ = saved
    E0 = idx.export()
    idx.save(tmp_path / "one")
    idx.save(tmp_path / "two")
    one = open(tmp_path / "one", "rb").read()
    assert one == open(tmp_path / "two", "rb").read() == open(path, "rb").read()
    assert same_export(idx.export(), E0)
    hdr, sec, table = read_file(tmp_path / "one")
    assert hdr["magic"] == b"STBIVFPQ" and hdr["version"] == 1 and (hdr["d"], hdr["pq_m"], hdr["pq_ksub"], hdr["pq_dsub"]) == (256, 32, 256, 8)
    n = idx.stats()["rows"]
    assert hdr["n"] == n and hdr["n_listed"] == len(E0["order"]) and hdr["n_forced"] == len(E0["forced"])
    assert hdr["rows_digest"] == digest(c.read(0, n).tobytes())
    assert hdr["header_checksum"] == digest(one[:208])
    for name, (_, nbytes, chk) in zip(SECTIONS, table):
        assert nbytes == len(sec[name]) and chk == digest(sec[name])
        assert sec[name] == np.ascontiguousarray(E0[name]).tobytes(), name
    assert len(one) == 216 + sum(len(s) for s in sec.values())
    assert sorted(os.listdir(tmp_path)) == ["one", "two"]                  # no temporary file stays behind


def test_save_refusals(ctx, tmp_path):
    rng = np.random.default_rng(8103)
    c = capi.Corpus(ctx, 4000)
    c.append(clustered(rng, make_centers(rng, 8), 4000))
    idx = capi.IvfPq(c, nlist=8, train_rows=4000, iters=2)
    L = capi.lib()
    try:
        assert L.stb_ivfpq_save(None, b"x") == capi.STB_ERR_ARG and L.stb_ivfpq_save(idx._h, None) == capi.STB_ERR_ARG
        # no such directory; a directory as the target: the temporary file is written beside it, in tmp_path, and
        # removed when the rename over the directory fails
        (tmp_path / "adir").mkdir()
        for bad in (tmp_path / "missing" / "f", tmp_path / "adir"):
            with pytest.raises(capi.StbError) as e:
                idx.save(bad)
            assert e.value.status == capi.STB_ERR_ARG
        assert sorted(os.listdir(tmp_path)) == ["adir"] and os.listdir(tmp_path / "adir") == []
        locked = tmp_path / "locked"
        locked.mkdir()
        locked.chmod(0o555)
        if not os.access(locked, os.W_OK):                                  # (a superuser writes anyway)
            with pytest.raises(capi.StbError) as e:
                idx.save(locked / "f")
            assert e.value.status == capi.STB_ERR_ARG
        assert os.listdir(locked) == [] and sorted(os.listdir(tmp_path)) == ["adir", "locked"]
        locked.chmod(0o755)
        # temporary names already taken (files a crashed process with this pid left behind): the save moves on
        stale = [tmp_path / f"taken.tmp.{os.getpid()}.{k}" for k in range(300)]
        for f in stale:
            f.write_bytes(b"stale")
        idx.save(tmp_path / "taken")
        assert capi.IvfPq.load(c, tmp_path / "taken").export()["list_off"][-1] == idx.export()["list_off"][-1]
        assert all(f.read_bytes() == b"stale" for f in stale)
        assert len(os.listdir(tmp_path)) == 2 + len(stale) + 1
        (tmp_path / "keep").write_bytes(b"old")
        c.clear()                                                            # the index no longer has its rows
        with pytest.raises(capi.StbError) as e:
            idx.save(tmp_path / "keep")
        assert e.value.status == capi.STB_ERR_STATE and (tmp_path / "keep").read_bytes() == b"old"
    finally:
        idx.close(); c.close()


# ---------------------------------------------------------------------------------------- refusals ---
@pytest.fixture(scope="module")
def refusal_setup(ctx, tmp_path_factory):
    """a corpus with forced rows and no live index, and the file of an index on it"""
    rng = np.random.default_rng(8104)
    centers = make_centers(rng, 16)
    rows = edge_rows(rng, centers, 8000)
    c = capi.Corpus(ctx, 8000)
    c.append(rows)
    idx = capi.IvfPq(c, nlist=16, train_rows=8000, iters=3)
    d = tmp_path_factory.mktemp("refuse")
    idx.save(d / "good")
    E = idx.export()
    idx.close()
    q = clustered(rng, centers, 1)[0]
    yield c, rows, d, E, q
    c.close()


def load_status(ctx, c, path, why=None):
    """stb_ivfpq_load's status; a refusal's message must contain `why` (the check that refused)"""
    h = capi.vp()
    rc = capi.lib().stb_ivfpq_load(ctx._h, c._h, os.fsencode(str(path)), capi.C.byref(h))
    assert (rc == 0) == bool(h.value)
    if rc == 0:
        capi.lib().stb_ivfpq_destroy(h)
    elif why is not None:
        msg = capi.lib().stb_last_error().decode()
        assert why in msg, (why, msg)
    return rc


# the lists pass's messages: exactly one of them names each crafted defect below
LIST_CHECKS = {"off": "list_off does not run", "row": "an order entry is >= n", "order": "a list is not strictly ascending",
               "forced": "forced is not strictly ascending", "dup": "a row appears twice"}


def lists_refusal(ctx, c, path, check):
    """refused by the lists pass for `check` alone"""
    assert load_status(ctx, c, path, LIST_CHECKS[check]) == capi.STB_ERR_ARG
    msg = capi.lib().stb_last_error().decode()
    assert [k for k, m in LIST_CHECKS.items() if m in msg] == [check], msg


def still_usable(ctx, c, rows, q):
    """no index counted on the corpus (an update works), and a search answers right"""
    c.update(np.array([77], np.uint64), rows[77:78])                       # the same value: the rows stay
    want, _ = oracle.search_rows(rows, q, 5)
    assert c.search(q, top_k=5)["row"].tolist() == [int(r) for r in want]


def test_refusals_of_damaged_files(ctx, refusal_setup):
    c, rows, d, E, q = refusal_setup
    good = open(d / "good", "rb").read()
    hdr, sec, table = read_file(d / "good")
    A = capi.STB_ERR_ARG
    cases = {"missing": (None, "cannot open"), "empty": (b"", "shorter than the 216-byte header")}
    ends = sorted({o for o, _, _ in table} | {o + b for o, b, _ in table})
    for cut in [8, 100, 215]:
        cases[f"truncated at {cut}"] = (good[:cut], "shorter than the 216-byte header")
    for cut in [e for e in ends if e < len(good)] + [o + b // 2 for o, b, _ in table if b > 1]:
        cases[f"truncated at {cut}"] = (good[:cut], f"file is {cut} bytes")
    cases["magic"] = (b"STBIVFPX" + good[8:], "magic")
    cases["version"] = (good[:8] + struct.pack("<I", 2) + good[12:], "version 2")
    cases["trailing byte"] = (good + b"\0", f"file is {len(good) + 1} bytes")
    cases["header byte 0"] = (bytes([good[0] ^ 0x10]) + good[1:], "magic")
    for at in (9, 29, 40, 57, 70, 150, 210):                                # one flipped byte in the header
        why = "version" if at == 9 else "header_checksum"
        cases[f"header byte {at}"] = (good[:at] + bytes([good[at] ^ 0x10]) + good[at + 1:], why)
    for name, (o, b, _) in zip(SECTIONS, table):                           # one flipped byte in each section
        at = o + b // 3
        cases[f"{name} byte"] = (good[:at] + bytes([good[at] ^ 0x01]) + good[at + 1:], f"section {name} does not match")
    for what, (data, why) in cases.items():
        p = d / "case"
        if data is None:
            p = d / "does-not-exist"
        else:
            p.write_bytes(data)
        assert load_status(ctx, c, p, why) == A, what
    still_usable(ctx, c, rows, q)
    assert load_status(ctx, c, d / "good") == 0


def crafted(hdr, sec, **change):
    """header fields and sections with the given arrays / fields replaced (counts follow the arrays)"""
    h, s = dict(hdr), dict(sec)
    for k, v in change.items():
        if k in SECTIONS:
            s[k] = np.ascontiguousarray(v).tobytes()
        else:
            h[k] = v
    return h, s


def test_refusals_of_crafted_files(ctx, refusal_setup):
    """Files whose checksums are right: each is refused by the one check its defect is aimed at."""
    c, rows, d, E, q = refusal_setup
    hdr, sec, _ = read_file(d / "good")
    n, off, order, forced, codes = hdr["n"], E["list_off"], E["order"], E["forced"], E["codes"]
    sizes = np.diff(off.astype(np.int64))
    big = int(np.argmax(sizes))                                             # a list of several rows
    b0, e0 = int(off[big]), int(off[big + 1])
    assert e0 - b0 >= 3 and len(forced) == 3
    others = np.concatenate([order[:b0], order[e0:]])                      # rows of the other lists
    lists = {}
    o = order.copy(); o[e0 - 1] = n                                         # still ascending: only the bound
    lists["order entry = n"] = (dict(order=o), "row")
    dup = int(others[others > order[e0 - 2]].min())                         # a row of another list, above its
    o = order.copy(); o[e0 - 1] = dup                                       # predecessor: only the bitmap
    lists["row in two lists"] = (dict(order=o), "dup")
    listed = int(others[(others > forced[0]) & (others < forced[2])][0])    # a listed row put into forced, in order
    f = forced.copy(); f[1] = listed
    lists["forced row also listed"] = (dict(forced=f), "dup")
    o = order.copy(); o[b0], o[b0 + 1] = o[b0 + 1], o[b0]
    lists["descending list"] = (dict(order=o), "order")
    lo = off.copy(); lo[-2] = lo[-1] + 1                                    # decreasing, and past n_listed
    lists["list_off decreases at its end"] = (dict(list_off=lo), "off")
    lo = off.copy(); lo[-1] -= 1
    lists["list_off ends short"] = (dict(list_off=lo), "off")
    lo = off.copy(); lo[0] = 1
    lists["list_off starts at 1"] = (dict(list_off=lo), "off")
    f = forced.copy(); f[[0, 1]] = f[[1, 0]]
    lists["forced not ascending"] = (dict(forced=f), "forced")
    f = forced.copy(); f[2] = n
    lists["forced entry = n"] = (dict(forced=f), "forced")
    for what, (change, check) in lists.items():
        write_file(d / "crafted", *crafted(hdr, sec, **change))
        lists_refusal(ctx, c, d / "crafted", check)
    # decreasing inside the lists: the lists around it then overlap, so other checks may fire as well
    lo = off.copy(); lo[big], lo[big + 1] = off[big + 1], off[big]
    write_file(d / "crafted", *crafted(hdr, sec, list_off=lo))
    assert load_status(ctx, c, d / "crafted", LIST_CHECKS["off"]) == capi.STB_ERR_ARG
    A, S = capi.STB_ERR_ARG, capi.STB_ERR_STATE
    cases = {}
    # a listed row moved to forced: the lists stay a partition, forced gains a normal row
    r = int(order[b0])
    lo = off.copy(); lo[big + 1:] -= 1
    cases["normal row as forced"] = (crafted(hdr, sec, order=np.delete(order, b0), codes=np.delete(codes, b0, axis=0), list_off=lo,
                                             forced=np.sort(np.append(forced, r)).astype(np.uint32), n_listed=hdr["n_listed"] - 1,
                                             n_forced=hdr["n_forced"] + 1), A, "cannot be normalised")
    # a forced row moved into the first list: forced misses a row that cannot be normalised
    r = int(forced[0])
    at = int(np.searchsorted(order[:off[1]], r))
    lo = off.copy(); lo[1:] += 1
    cases["forced row listed"] = (crafted(hdr, sec, order=np.insert(order, at, r), codes=np.insert(codes, at, codes[0], axis=0),
                                          list_off=lo, forced=forced[1:], n_listed=hdr["n_listed"] + 1, n_forced=hdr["n_forced"] - 1),
                                  A, "cannot be normalised")
    cases["n_forced 1025"] = (crafted(hdr, sec, n_forced=1025, n=hdr["n_listed"] + 1025), A, "n_forced 1025")
    for nl in (0, 8193):
        cases[f"nlist {nl}"] = (crafted(hdr, sec, nlist=nl), A, f"nlist {nl}")
    cases["n_listed + n_forced != n"] = (crafted(hdr, sec, n=n - 1), A, "n_listed")
    cases["n above the corpus"] = (crafted(hdr, sec, n=n + 1, n_forced=hdr["n_forced"] + 1,
                                           forced=np.append(forced, n).astype(np.uint32)), S, "the corpus holds")
    for what, ((h, s), want, why) in cases.items():
        write_file(d / "crafted", h, s)
        assert load_status(ctx, c, d / "crafted", why) == want, what
    # the restatement itself: an unchanged rewrite loads
    write_file(d / "crafted", hdr, sec)
    assert open(d / "crafted", "rb").read() == open(d / "good", "rb").read()
    assert load_status(ctx, c, d / "crafted") == 0
    still_usable(ctx, c, rows, q)


def test_refusals_of_the_corpus(ctx, refusal_setup):
    c, rows, d, E, q = refusal_setup
    A, S = capi.STB_ERR_ARG, capi.STB_ERR_STATE
    one = rows.copy()
    one[1234, 17] = np.nextafter(one[1234, 17], np.float32(2))             # one component of one row
    short = capi.Corpus(ctx, 8000); short.append(rows[:7999])
    changed = capi.Corpus(ctx, 8000); changed.append(one)
    host = capi.Corpus.in_host_memory(ctx, 8000); host.append(rows)
    other = capi.Context(0)
    theirs = capi.Corpus(other, 8000); theirs.append(rows)
    try:
        assert load_status(ctx, changed, d / "good", "rows_digest") == S
        assert load_status(ctx, short, d / "good", "the corpus holds 7999") == S
        assert load_status(ctx, host, d / "good", "host memory") == S
        assert load_status(ctx, theirs, d / "good", "another context") == A
        L = capi.lib()
        h = capi.vp()
        assert L.stb_ivfpq_load(None, c._h, b"x", capi.C.byref(h)) == A and L.stb_ivfpq_load(ctx._h, c._h, None, capi.C.byref(h)) == A
        for x in (changed, short):
            x.update(np.array([5], np.uint64), x.read(5, 1))                 # no index counted on them
        still_usable(ctx, c, rows, q)
        loaded = capi.IvfPq.load(theirs, d / "good")                         # on its own context it loads
        assert same_export(loaded.export(), E)
        loaded.close()
    finally:
        theirs.close(); other.close(); host.close(); changed.close(); short.close()
