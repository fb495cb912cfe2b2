"""GPU tests of a corpus's life: appends, removals and clears, and a pending search_device across every other call.

The reference of every mutation test is the *fresh* corpus: one built in a single append from the surviving rows and rowids.
Every engine reads the same per-row arrays (rows, rowids, the cached inv_norm), so a corpus after any sequence of mutations
must answer every call bit for bit as the fresh corpus does.  Two read-backs check those arrays directly: search_all_matching
returns the rowid and exact score of every row, and debug_stage1_scores returns stage-1 scores by row position, which a
misplaced inv_norm or an unstable compaction changes.  Flags are compared only while nothing has been removed since the last
clear: removals keep the norm statistics as upper bounds, so eps, and with it a fallback, may differ.  Each group of cases is
also anchored to the CPU oracle, so that a fault both corpora share cannot pass.

remove compacts each per-row array in batches of max(1, 256 MiB / row bytes) rows (knn.cu compact_array); the shapes below
are chosen so that every unit width of that copy (16, 4 and 2 bytes) crosses at least two batches."""
import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_knn_exact import near_tie_corpus

pytestmark = pytest.mark.gpu

BATCH_BYTES = 256 << 20


@pytest.fixture(scope="module")
def Y():
    import yams_b200
    assert yams_b200.device_count() > 0
    assert yams_b200.plugin_init() == 0, yams_b200.health()
    return yams_b200


def rows_per_batch(row_bytes):
    """the batch of remove's compaction (knn.cu compact_array)"""
    return max(1, BATCH_BYTES // row_bytes)


def stored_rows(O, dtype_name, rows32):
    """the rows as the corpus holds them: fp16 bits (the truncating conversion) or fp32"""
    return O.f16_from_float(rows32).reshape(rows32.shape) if dtype_name == "f16" else rows32


def make_corpus(Y, d, dtype_name, metric, rows, rowids):
    c = Y.Corpus(d, Y.F16 if dtype_name == "f16" else Y.F32, metric)
    if len(rows):
        c.append(rows, rowids=rowids)
    return c


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def assert_same(got, fresh, queries, k, engines, flags, spans=None, allowed=(None,)):
    """got answers search, debug_stage1_scores (every engine, over spans = [(row_start, nrows)], default all rows) and
    search_all_matching (the first query, over each allowed list) bit for bit as fresh does; flags and eps as well when
    `flags`.  -> fresh's search result"""
    n = len(fresh)
    assert len(got) == n
    a, b = got.search(queries, k), fresh.search(queries, k)
    for x, y in zip(a[:3], b[:3]):
        assert x.tobytes() == y.tobytes()
    if flags:
        assert np.array_equal(a[3], b[3])
        assert bits(got.debug_last_eps(len(queries))).tobytes() == bits(fresh.debug_last_eps(len(queries))).tobytes()
    if n == 0:
        assert not a[2].any()
        return b
    for e in engines:
        for s, m in spans or [(0, n)]:
            sa = got.debug_stage1_scores(queries, e, row_start=s, nrows=m)
            sb = fresh.debug_stage1_scores(queries, e, row_start=s, nrows=m)
            assert np.array_equal(bits(sa), bits(sb)), (e, s, m)
    if got.metric == 0:   # COSINE
        for al in allowed:
            ra, rb = got.search_all_matching(queries[0], allowed=al), fresh.search_all_matching(queries[0], allowed=al)
            assert ra[0].tobytes() == rb[0].tobytes() and ra[1].tobytes() == rb[1].tobytes()
    return b


def removal_patterns(n, B, rng):
    """-> {name: positions removed}: the first row, the last, exactly one whole batch, a run straddling every batch boundary,
    1 in 7 at random, all but the last row, all rows (B = rows per batch)"""
    r = min(B // 4, 2000)
    straddle = np.unique(np.concatenate([np.arange(b - r, min(b + r, n)) for b in range(B, n, B)]))
    return {"first": np.array([0]), "last": np.array([n - 1]), "one_batch": np.arange(B, min(2 * B, n)), "straddle": straddle,
            "one_in_7": np.flatnonzero(rng.random(n) < 1 / 7), "all_but_last": np.arange(n - 1), "all": np.arange(n)}


def unknown_rowids(rowids):
    """rowids the corpus does not hold: between two held ones (odd rowids), past the last, negative"""
    return np.array([rowids[0] + 1, rowids[len(rowids) // 2] + 1, rowids[-1] + 1, rowids[-1] + 10**9, -5], dtype=np.int64)


# ---- a. compaction across batches, every unit width ----

# (dtype, d, n, engines of debug_stage1_scores): the search's engine is wgmma at d = 768, CUDA-core at d = 33 and d = 385
SHAPES = [("f16", 768, 600_000, (0, 1)), ("f32", 768, 300_000, (0, 1)), ("f32", 33, 4_500_000, (0,)), ("f16", 385, 1_000_000, (0,))]


def planted_corpus(O, dtype_name, d, n, queries, rng):
    """random rows + 4 perturbed, scaled copies of every query direction just past each batch boundary and in the last
    batch, so that each query's top-k lies in rows that a removal before them moves across a boundary"""
    B = rows_per_batch(d * (2 if dtype_name == "f16" else 4))
    rows32 = O.gen_rows_f32(42, 0, n, d)
    bounds = list(range(B, n, B))
    spots = bounds + [(bounds[-1] + n) // 2]
    planted = []
    for b in spots:
        for j, q in enumerate(queries):
            qn = q / np.linalg.norm(q)
            for t in range(4):
                p = b + 1 + 4 * j + t
                noise = rng.normal(size=d).astype(np.float32) * np.float32(0.05 / np.sqrt(d))
                rows32[p] = (qn + noise) * np.float32(rng.uniform(0.5, 4.0))
                planted.append(p)
    return stored_rows(O, dtype_name, rows32), np.array(planted), B


@pytest.mark.parametrize("dtype_name,d,n,engines", SHAPES)
def test_remove_compacts_across_batches(Y, oracle, dtype_name, d, n, engines):
    """Every removal pattern on its own copy of a corpus whose row array spans >= 3 compaction batches: the corpus then equals
    the fresh corpus bit for bit, and on the 1-in-7 pattern the CPU oracle's answer."""
    O = oracle
    rng = np.random.default_rng(d + n)
    k, nq = 10, 6
    queries = O.gen_rows_f32(43, 0, nq, d)
    rows, planted, B = planted_corpus(O, dtype_name, d, n, queries, rng)
    assert (n + B - 1) // B >= 3
    rowids = np.arange(n, dtype=np.int64) * 2 + 1
    # before any removal, the top-k of every query is planted rows past the boundaries
    c = make_corpus(Y, d, dtype_name, Y.COSINE, rows, rowids)
    rid, _, cnt, _ = c.search(queries, k)
    assert np.all(cnt == k) and np.isin(rid, rowids[planted]).all()
    assert c.remove(unknown_rowids(rowids)) == 0                      # the early return: nothing moves
    fresh = make_corpus(Y, d, dtype_name, Y.COSINE, rows, rowids)
    assert_same(c, fresh, queries, k, engines, True)
    fresh.close()
    c.close()
    for name, gone in removal_patterns(n, B, rng).items():
        c = make_corpus(Y, d, dtype_name, Y.COSINE, rows, rowids)
        assert c.remove(rowids[gone]) == len(gone), name
        keep = np.ones(n, dtype=bool)
        keep[gone] = False
        fresh = make_corpus(Y, d, dtype_name, Y.COSINE, rows[keep], rowids[keep])
        want = assert_same(c, fresh, queries, k, engines, False)
        if name == "one_in_7":
            rc, wr, ws, wc = O.exact_scan_cosine_batch(rows[keep], queries[:3], k)
            assert rc == 0
            assert np.array_equal(want[0][:3], np.where(wr >= 0, rowids[keep][wr], -1)) and np.array_equal(want[1][:3], ws)
            assert np.array_equal(want[2][:3], wc)
        c.close()
        fresh.close()


def synth_windows(bounds, n_old, kept_ranges, r=256):
    """new row positions [(start, nrows)] around where each old position in `bounds` lands, and at both ends"""
    lo_hi = [(a, b) for a, b in kept_ranges]
    n_new = sum(b - a for a, b in lo_hi)
    out = [(0, min(r, n_new))]
    for p in bounds:
        at = sum(min(max(p - a, 0), b - a) for a, b in lo_hi)      # kept rows before old position p
        s = max(0, min(at - r, n_new - 2 * r))
        out.append((s, min(2 * r, n_new - s)))
    out.append((max(0, n_new - r), min(r, n_new)))
    return [(s, m) for s, m in out if m > 0]


def test_remove_compacts_70m_rows_rowids_and_norms_in_batches(Y, oracle):
    """fp16, d = 8 (16-byte rows): 70 M rows take 5 row batches, 3 rowid batches and 2 inv_norm batches.  Both the corpus
    and its fresh copy are built by append_synthetic (the fresh one once per kept range), so no rows go through the host;
    the run-shaped removal patterns, queries that are synthetic rows just past every boundary, stage 1 and all_matching on
    windows around the boundaries.  The windows are anchored to the CPU oracle."""
    O = oracle
    d, n, seed, first = 8, 70_000_000, 5, 1000
    B = rows_per_batch(16)
    assert ((n + B - 1) // B, (n + rows_per_batch(8) - 1) // rows_per_batch(8), (n + rows_per_batch(4) - 1) // rows_per_batch(4)) == (5, 3, 2)
    bounds = sorted(set(range(B, n, B)) | set(range(rows_per_batch(8), n, rows_per_batch(8))) | {rows_per_batch(4)})
    qpos = [b + 7 for b in bounds] + [n - 3]
    queries = np.concatenate([O.gen_rows_f32(seed, first + p, 1, d) for p in qpos])
    r = 2000
    patterns = {"unknown": [], "first": [(0, 1)], "last": [(n - 1, n)], "one_batch": [(B, 2 * B)],
                "straddle": [(b - r, b + r) for b in bounds], "all_but_last": [(0, n - 1)], "all": [(0, n)]}
    for name, runs in patterns.items():
        c = Y.Corpus(d, Y.F16, Y.COSINE)
        c.append_synthetic(seed, first, n)
        gone = np.concatenate([np.arange(first + a, first + b, dtype=np.int64) for a, b in runs]) if runs else \
            np.array([first - 1, first + n, -3], dtype=np.int64)
        assert c.remove(gone) == (len(gone) if runs else 0), name
        del gone
        kept, at = [], 0
        for a, b in runs:
            if a > at:
                kept.append((at, a))
            at = b
        if at < n:
            kept.append((at, n))
        fresh = Y.Corpus(d, Y.F16, Y.COSINE)
        for a, b in kept:
            fresh.append_synthetic(seed, first + a, b - a)
        n_new = len(fresh)
        if n_new == 0:
            assert_same(c, fresh, queries, 10, (0,), False)
            c.close(); fresh.close()
            continue
        spans = synth_windows(bounds, n, kept)
        # the rowids of each window on the fresh corpus: kept ranges laid end to end
        starts = np.cumsum([0] + [b - a for a, b in kept])
        def rowid_at(pos):
            i = np.searchsorted(starts, pos, side="right") - 1
            return first + kept[i][0] + (pos - starts[i])
        allowed = [np.array([rowid_at(p) for p in range(s, s + m)], dtype=np.int64) for s, m in spans]
        assert_same(c, fresh, queries, 10, (0,), not runs, spans=spans, allowed=allowed)
        for al in allowed[:4]:
            win = O.f16_from_float(np.concatenate([O.gen_rows_f32(seed, int(x), 1, d) for x in al])).reshape(len(al), d)
            rc, wr, ws = O.exact_scan_cosine(win, queries[0], len(al), rowids=al, all_matching=True)
            assert rc == 0
            gr, gs = c.search_all_matching(queries[0], allowed=al)
            assert np.array_equal(gr, wr) and np.array_equal(gs, ws), name
        c.close()
        fresh.close()


def test_remove_on_an_l2_corpus(Y, oracle):
    """L2 (inv_norm holds |r|^2), fp32, d = 64 over 3 compaction batches: every removal pattern equals the fresh corpus bit
    for bit (search and both stage-1 engines), and the oracle's vec0 answer on the 1-in-7 pattern."""
    O = oracle
    d, n, k = 64, 2_500_000, 10
    B = rows_per_batch(d * 4)
    rng = np.random.default_rng(64)
    rows = O.gen_rows_f32(42, 0, n, d) * rng.uniform(0.5, 3.0, size=(n, 1)).astype(np.float32)
    rowids = np.arange(n, dtype=np.int64) * 3 + 2
    queries = O.gen_rows_f32(43, 0, 4, d) * np.float32(2.0)
    queries[1] = rows[B + 5]                                         # distance 0 to a row past the first boundary
    c = make_corpus(Y, d, "f32", Y.L2, rows, rowids)
    assert c.remove(unknown_rowids(rowids)) == 0
    fresh = make_corpus(Y, d, "f32", Y.L2, rows, rowids)
    assert_same(c, fresh, queries, k, (0, 1), True)
    c.close(); fresh.close()
    for name, gone in removal_patterns(n, B, rng).items():
        c = make_corpus(Y, d, "f32", Y.L2, rows, rowids)
        assert c.remove(rowids[gone]) == len(gone), name
        keep = np.ones(n, dtype=bool)
        keep[gone] = False
        fresh = make_corpus(Y, d, "f32", Y.L2, rows[keep], rowids[keep])
        rid, dist, cnt, _ = assert_same(c, fresh, queries, k, (0, 1), False)
        if name == "one_in_7":
            for qi in range(len(queries)):
                wr, wd = O.vec0_exact(rows[keep], queries[qi], k=k + 5, rowids=rowids[keep])
                assert cnt[qi] == k and np.allclose(dist[qi], wd[:k], rtol=1e-5, atol=1e-6), qi
                assert set(rid[qi]) <= set(wr), qi                  # float summation order may swap near-equal neighbours
        c.close(); fresh.close()


# ---- b. consumers after a removal ----

def consumer_case(O, n=100_000, d=64):
    rows = stored_rows(O, "f16", O.gen_rows_f32(21, 0, n, d))
    rowids = np.arange(n, dtype=np.int64) * 3 + 5                    # not dense
    queries = O.gen_rows_f32(22, 0, 6, d)
    return rows, rowids, queries


def test_consumers_after_a_removal(Y, oracle):
    """~100 k fp16 rows with non-dense rowids; the removal takes each query's 3 best rows and 1 in 5 of the rest.  Candidate
    sets (direct lists holding removed rowids, a masked list), the semantic graph, k-means, exact document search and the PQ
    index then answer as on the fresh corpus, and as the oracle where it has an answer."""
    O = oracle
    n, d, k = 100_000, 64, 10
    rows, rowids, queries = consumer_case(O, n, d)
    rng = np.random.default_rng(9)
    c = make_corpus(Y, d, "f16", Y.COSINE, rows, rowids)
    m, kc = 8, 16
    codebooks = (rng.normal(size=(m, kc, d // m)) / np.sqrt(d)).astype(np.float32).reshape(-1)
    stale = Y.PqIndex(c, m, kc, codebooks)
    top, _, _, _ = c.search(queries, k)
    gone = np.union1d(top[:, :3].reshape(-1), rowids[rng.random(n) < 0.2])
    assert c.remove(gone) == len(gone)
    keep = ~np.isin(rowids, gone)
    krows, kids = rows[keep], rowids[keep]
    fresh = make_corpus(Y, d, "f16", Y.COSINE, krows, kids)
    assert_same(c, fresh, queries, k, (0, 1), False)
    # candidate sets: ascending lists (direct path) holding removed rowids, then the same lists descending (masked path)
    lists = [np.sort(np.union1d(rng.choice(rowids, 1500, replace=False), top[q, :5])) for q in range(len(queries))]
    for al in (lists, [a[::-1] for a in lists]):
        ga, fa = c.search(queries, k, allowed=al), fresh.search(queries, k, allowed=al)
        for x, y in zip(ga[:3], fa[:3]):
            assert x.tobytes() == y.tobytes()
        for q in range(len(queries)):
            rc, wr, ws = O.exact_scan_cosine(krows, queries[q], k, rowids=kids, allowed=lists[q])
            assert rc == 0 and ga[2][q] == len(wr)
            assert np.array_equal(ga[0][q, :len(wr)], wr) and np.array_equal(ga[1][q, :len(wr)], ws), q
    # the semantic graph, every source, and sources that include removed rowids
    ga, fa = c.semantic_neighbors(k), fresh.semantic_neighbors(k)
    for x, y in zip(ga, fa):
        assert x.tobytes() == y.tobytes()
    src = np.sort(np.concatenate([gone[:20], kids[::997]]))
    ga, fa = c.semantic_neighbors(k, sources=src), fresh.semantic_neighbors(k, sources=src)
    for x, y in zip(ga, fa):
        assert x.tobytes() == y.tobytes()
    removed = np.isin(src, gone)
    assert not ga[2][removed].any() and np.all(ga[3][removed] == Y.FLAG_NOT_A_SOURCE)
    assert np.all(ga[2][~removed] == k)
    # k-means: the result depends on row order
    ga, fa = c.topology_kmeans(40, 4), fresh.topology_kmeans(40, 4)
    assert np.array_equal(ga[0], fa[0]) and np.array_equal(bits(ga[1]), bits(fa[1])) and ga[2:] == fa[2:]
    # exact document search over documents that hold removed rows
    docs = [[rowids[i:i + 40] for i in range(q * 2000, q * 2000 + 2000, 40)] for q in range(len(queries))]
    ga, fa = c.search_documents(queries, k, docs), fresh.search_documents(queries, k, docs)
    for x, y in zip(ga, fa):
        assert x.tobytes() == y.tobytes()
    # PQ: an index built before the removal is stale; a rebuilt one equals one built on the fresh corpus
    for call in (lambda: stale.search(queries, k), lambda: c.search_documents(queries, k, docs, pq=stale)):
        with pytest.raises(Y.YamsB200Error) as e:
            call()
        assert e.value.status == 1
    stale.close()
    pa, pb = Y.PqIndex(c, m, kc, codebooks), Y.PqIndex(fresh, m, kc, codebooks)
    ca, cb = pa.codes(), pb.codes()
    assert np.array_equal(ca[0], cb[0]) and np.array_equal(ca[1], cb[1])
    for x, y in zip(pa.search(queries, k), pb.search(queries, k)):
        assert x.tobytes() == y.tobytes()
    for x, y in zip(c.search_documents(queries, k, docs, pq=pa), fresh.search_documents(queries, k, docs, pq=pb)):
        assert x.tobytes() == y.tobytes()
    for h in (pa, pb, c, fresh):
        h.close()


def test_removal_and_append_across_the_dense_limit(Y, oracle):
    """70 000 rows (the sampled threshold path) -> remove 10 000 -> 60 000 (dense path) -> append 20 000 -> 80 000 (sampled
    again): equal to the fresh corpus at every step, and to the oracle at the end."""
    O = oracle
    d, k = 64, 10
    rows, rowids, queries = consumer_case(O, 90_000, d)
    rng = np.random.default_rng(12)
    c = make_corpus(Y, d, "f16", Y.COSINE, rows[:70_000], rowids[:70_000])
    gone = np.sort(rng.choice(rowids[:70_000], 10_000, replace=False))
    assert c.remove(gone) == 10_000
    keep = ~np.isin(rowids, gone)
    keep[70_000:] = False
    fresh = make_corpus(Y, d, "f16", Y.COSINE, rows[keep], rowids[keep])
    assert len(c) == 60_000
    assert_same(c, fresh, queries, k, (0, 1), False)
    fresh.close()
    c.append(rows[70_000:], rowids=rowids[70_000:])
    keep[70_000:] = True
    fresh = make_corpus(Y, d, "f16", Y.COSINE, rows[keep], rowids[keep])
    assert len(c) == 80_000
    rid, sc, cnt, _ = assert_same(c, fresh, queries, k, (0, 1), False)
    rc, wr, ws, wc = O.exact_scan_cosine_batch(rows[keep], queries, k)
    assert rc == 0 and np.array_equal(rid, rowids[keep][wr]) and np.array_equal(sc, ws)
    c.close(); fresh.close()


# ---- c. append sequences ----

def test_append_sequence_with_removals_and_a_clear(Y, oracle):
    """~300 appends of 0..5000 rows by append, append_f32_as_f16 and append_synthetic (the buffers grow many times), with
    removals and one clear in between: equal to the fresh corpus every 20 steps (flags too while nothing has been removed
    since the clear), and to the oracle at the end."""
    O = oracle
    d, k, seed = 32, 10, 77
    rng = np.random.default_rng(30)
    queries = O.gen_rows_f32(31, 0, 5, d)
    c = Y.Corpus(d, Y.F16, Y.COSINE)
    rows = np.zeros((0, d), dtype=np.uint16)
    ids = np.zeros(0, dtype=np.int64)
    nxt, removed = 0, False
    for step in range(300):
        kind = step % 3
        m = int(rng.integers(0, 5001))
        nxt += int(rng.integers(0, 3))                              # gaps between rowids now and then
        new_ids = np.arange(nxt, nxt + m, dtype=np.int64)
        if kind == 2:
            c.append_synthetic(seed, nxt, m)
            r32 = O.gen_rows_f32(seed, nxt, m, d) if m else np.zeros((0, d), np.float32)
        else:
            r32 = O.gen_rows_f32(1000 + step, 0, m, d) * np.float32(rng.uniform(0.01, 50.0)) if m else np.zeros((0, d), np.float32)
            c.append(r32 if kind == 1 else stored_rows(O, "f16", r32), rowids=new_ids if m else None)
        rows = np.concatenate([rows, stored_rows(O, "f16", r32).reshape(m, d)])
        ids = np.concatenate([ids, new_ids])
        nxt += m
        if step % 23 == 11 and len(ids):
            gone = ids[rng.random(len(ids)) < 0.1]
            assert c.remove(gone) == len(gone)
            keep = ~np.isin(ids, gone)
            rows, ids, removed = rows[keep], ids[keep], removed or len(gone) > 0
        if step == 150:
            c.clear()
            rows, ids, removed = rows[:0], ids[:0], False
            nxt = 0
        if step % 20 == 19 or step == 299:
            assert len(c) == len(ids)
            fresh = make_corpus(Y, d, "f16", Y.COSINE, rows, ids)
            want = assert_same(c, fresh, queries, k, (0, 1), not removed)
            fresh.close()
    rc, wr, ws, wc = O.exact_scan_cosine_batch(rows, queries, k)
    assert rc == 0 and np.array_equal(want[0], ids[wr]) and np.array_equal(want[1], ws)
    c.close()


def test_rejected_appends_leave_the_corpus_unchanged(Y, oracle):
    """A rejected batch leaves the length, the results and the norm statistics (debug_last_eps after the same search)
    unchanged; each rejected batch carries a row of extreme norm, so that a leak into the statistics would widen eps."""
    O = oracle
    d, k, n = 64, 10, 50_000
    queries = O.gen_rows_f32(3, 0, 4, d)
    for dtype_name in ("f16", "f32"):
        rows = stored_rows(O, dtype_name, O.gen_rows_f32(2, 0, n, d))
        rowids = np.arange(n, dtype=np.int64) * 2 + 10
        c = make_corpus(Y, d, dtype_name, Y.COSINE, rows, rowids)
        before = c.search(queries, k)
        eps = c.debug_last_eps(len(queries))
        bad32 = O.gen_rows_f32(4, 0, 8, d)
        bad32[3] *= np.float32(1000.0)                               # huge norm
        bad32[5] *= np.float32(1e-3)                                 # tiny norm
        bad = stored_rows(O, dtype_name, bad32)
        last = int(rowids[-1])
        attempts = [
            lambda: c.append(bad, rowids=np.array([last + 1, last + 2, last + 3, last + 2, last + 9, last + 10, last + 11, last + 12])),
            lambda: c.append(bad, rowids=np.array([-1] + list(range(last + 1, last + 8)))),
            lambda: c.append_synthetic(9, last, 8),
            lambda: c.append_synthetic(9, 0, 8),
        ]
        if dtype_name == "f32":
            attempts.append(lambda: Y._lib._check(Y.lib().yams_b200_corpus_append_f32_as_f16(
                c.handle, bad32.ctypes.data_as(C.POINTER(C.c_float)), 8, None), "corpus_append_f32_as_f16"))
        for i, attempt in enumerate(attempts):
            with pytest.raises(Y.YamsB200Error) as e:
                attempt()
            assert e.value.status == 1, i
            assert len(c) == n, i
            after = c.search(queries, k)
            for x, y in zip(before, after):
                assert x.tobytes() == y.tobytes(), i
            assert bits(c.debug_last_eps(len(queries))).tobytes() == bits(eps).tobytes(), i
        rc, wr, ws, wc = O.exact_scan_cosine_batch(rows, queries, k)
        assert rc == 0 and np.array_equal(before[0], rowids[wr]) and np.array_equal(before[1], ws)
        c.close()


def test_append_f32_as_f16_at_the_conversion_edges(Y, oracle):
    """append_f32_as_f16 against a corpus built from the oracle's truncating conversion (f16_from_float) of the same
    values: the largest finite half and values just above it, values that truncate to it or overflow, subnormals, values
    that flush to zero, +-inf, NaN and -0."""
    O = oracle
    d = 16
    edges = np.array([65504.0, 65505.0, 65519.0, 65519.99, 65520.0, 65536.0, 1e6, -65504.0, -65520.0, 6.1035156e-05, 6.0e-05,
                      5.9604645e-08, 5.0e-08, 2.9802322e-08, 1.0e-08, 1e-30, -5.9604645e-08, 1.4e-45, np.inf, -np.inf, np.nan,
                      -0.0, 0.0, 1.0009766, 1.0004883, 0.33333334, -2.7182817], dtype=np.float32)
    base = O.gen_rows_f32(50, 0, 256, d)
    rows32 = base.copy()
    for i, v in enumerate(edges):                                   # one edge per row, each in a row of its own and in a mixed one
        rows32[i, i % d] = v
        rows32[64 + i, :] = v
        rows32[128 + i, (i + 3) % d] = v * np.float32(1e-3) if np.isfinite(v) else v
    rows32[200:210] *= np.float32(1e-4)                             # ordinary rows whose elements become subnormal
    rowids = np.arange(256, dtype=np.int64) * 5
    got = Y.Corpus(d, Y.F16, Y.COSINE)
    got.append(rows32, rowids=rowids)                               # append_f32_as_f16
    want_rows = O.f16_from_float(rows32).reshape(256, d)
    want = make_corpus(Y, d, "f16", Y.COSINE, want_rows, rowids)
    queries = np.concatenate([O.gen_rows_f32(51, 0, 3, d), np.ones((1, d), np.float32)])
    assert_same(got, want, queries, 10, (0,), True)
    for q in queries:
        ra, sa = got.search_all_matching(q)
        rc, wr, ws = O.exact_scan_cosine(want_rows, q, 256, rowids=rowids, all_matching=True)
        assert rc == 0 and np.array_equal(ra, wr) and np.array_equal(sa, ws)
    got.close(); want.close()


# ---- d. norm statistics through clear and remove ----

def test_norm_statistics_through_clear_and_remove(Y, oracle):
    """A corpus with a tiny-norm row (scale 1e-20) and a huge one: after a clear and ordinary appends its eps equals the fresh
    corpus's bit for bit; after removing only the outliers eps is at least the fresh corpus's and the results stay exact."""
    O = oracle
    d, n, k = 64, 40_000, 10
    rows = O.gen_rows_f32(60, 0, n, d)
    rowids = np.arange(n, dtype=np.int64)
    queries = O.gen_rows_f32(61, 0, 6, d)
    odd = rows.copy()
    odd[100] *= np.float32(1e-20)
    odd[n - 100] *= np.float32(1e15)
    c = make_corpus(Y, d, "f32", Y.COSINE, odd, rowids)
    c.search(queries, k)
    c.clear()
    assert len(c) == 0
    c.append(rows, rowids=rowids)
    fresh = make_corpus(Y, d, "f32", Y.COSINE, rows, rowids)
    for e in (0, 1):                                                # eps of both engines, from stage 1 and from a search
        c.debug_stage1_scores(queries, e)
        fresh.debug_stage1_scores(queries, e)
        assert bits(c.debug_last_eps(len(queries))).tobytes() == bits(fresh.debug_last_eps(len(queries))).tobytes()
    assert_same(c, fresh, queries, k, (0, 1), True)
    c.close()
    c = make_corpus(Y, d, "f32", Y.COSINE, odd, rowids)
    assert c.remove([100, n - 100]) == 2
    keep = np.ones(n, dtype=bool)
    keep[[100, n - 100]] = False
    fresh.close()
    fresh = make_corpus(Y, d, "f32", Y.COSINE, rows[keep], rowids[keep])
    rid, sc, cnt, _ = assert_same(c, fresh, queries, k, (0, 1), False)
    c.search(queries, k)
    fresh.search(queries, k)
    assert np.all(c.debug_last_eps(len(queries)) >= fresh.debug_last_eps(len(queries)))
    rc, wr, ws, wc = O.exact_scan_cosine_batch(rows[keep], queries, k)
    assert rc == 0 and np.array_equal(rid, rowids[keep][wr]) and np.array_equal(sc, ws)
    c.close(); fresh.close()


# ---- e. a pending search_device across every other call ----

PEND_N, PEND_D, PEND_K = 100_000, 128, 10


@pytest.fixture(scope="module")
def pending_case(oracle):
    """the near-tie batch of test_gpu_knn_host_paths: 7 ordinary queries and one the certificate rejects; the oracle's
    answer on the table as it is at enqueue"""
    O = oracle
    rng = np.random.default_rng(11)
    q_adv = O.gen_rows_f32(77, 0, 1, PEND_D)[0]
    rows32, _ = near_tie_corpus(O, PEND_N, PEND_D, q_adv, 300, 1e-4, 42, rng)
    rows = O.f16_from_float(rows32).reshape(PEND_N, PEND_D)
    queries = np.concatenate([O.gen_rows_f32(43, 0, 7, PEND_D), q_adv[None, :]])
    rc, wr, ws, wc = O.exact_scan_cosine_batch(rows, queries, PEND_K)
    assert rc == 0
    return rows, queries, wr, ws


def intervening_calls(Y, O, rows, queries, wr):
    """name -> call(corpus) -> a value to compare with the same call on a corpus without a pending search"""
    n, d = rows.shape
    q_adv = queries[-1]
    along = (np.linspace(0.5, 2.0, 5)[:, None] * (q_adv / np.linalg.norm(q_adv))[None, :]).astype(np.float32)
    docs = [[np.arange(i, i + 50) for i in range(0, 5000, 50)] for _ in range(2)]
    return {
        "remove": lambda c: c.remove(np.concatenate([wr[0, :3], wr[-1, :3]])),
        "append": lambda c: c.append(O.f16_from_float(along).reshape(5, d), rowids=np.arange(n, n + 5)),
        "append_synthetic": lambda c: c.append_synthetic(5, n + 10, 1000),
        "append_f32_as_f16": lambda c: c.append(O.gen_rows_f32(6, 0, 100, d), rowids=np.arange(n, n + 100)),
        "clear": lambda c: c.clear(),
        "search": lambda c: c.search(queries[::-1], PEND_K),
        "search_exhaustive": lambda c: c.search_exhaustive(queries[:2], PEND_K),
        "search_all_matching": lambda c: c.search_all_matching(queries[1], allowed=np.arange(0, n, 7)),
        "semantic_neighbors": lambda c: c.semantic_neighbors(PEND_K, sources=np.arange(0, n, 997)),
        "topology_kmeans": lambda c: c.topology_kmeans(8, 2),
        "search_documents": lambda c: c.search_documents(queries[:2], 5, docs),
    }


def same_value(a, b):
    if isinstance(a, tuple):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            same_value(x, y)
    elif isinstance(a, np.ndarray):
        assert a.tobytes() == b.tobytes()
    else:
        assert a == b


@pytest.mark.parametrize("zero_query", [False, True])
@pytest.mark.parametrize("call", ["remove", "append", "append_synthetic", "append_f32_as_f16", "clear", "search", "search_exhaustive",
                                  "search_all_matching", "semantic_neighbors", "topology_kmeans", "search_documents"])
def test_pending_search_device_is_finished_on_the_corpus_it_was_enqueued_on(Y, oracle, pending_case, call, zero_query):
    """search_device, one other call on the corpus, search_device_finish: the whole batch equals the oracle on the table as
    it was at enqueue and finish reports the near-tie query resolved (or, with a zero query in the batch, finish raises
    the invalid argument), while the intervening call answers as it does without a pending search and leaves the same
    corpus behind."""
    import torch
    O = oracle
    rows, queries, wr, ws = pending_case
    nq, k = len(queries), PEND_K
    op = intervening_calls(Y, O, rows, queries, wr)[call]
    batch = queries.copy()
    if zero_query:
        batch[2] = 0
    c = make_corpus(Y, PEND_D, "f16", Y.COSINE, rows, None)
    ref = make_corpus(Y, PEND_D, "f16", Y.COSINE, rows, None)
    dq = torch.from_numpy(batch).cuda()
    out_r = torch.full((nq, k), -7, dtype=torch.int64, device="cuda")
    out_s = torch.zeros((nq, k), dtype=torch.float32, device="cuda")
    c.search_device(dq.data_ptr(), nq, k, -1.0, out_r.data_ptr(), out_s.data_ptr())
    got = op(c)
    if zero_query:
        with pytest.raises(Y.YamsB200Error) as e:
            c.search_device_finish()
        assert e.value.status == 1
    else:
        assert c.search_device_finish() >= 1                          # the near-tie query went through the exhaustive level
        assert np.array_equal(out_r.cpu().numpy(), wr) and np.array_equal(out_s.cpu().numpy(), ws)
    assert c.search_device_finish() == 0                              # nothing is pending any more
    same_value(got, op(ref))
    assert len(c) == len(ref)
    if len(ref):
        assert_same(c, ref, queries, k, (0, 1), False)
    c.close(); ref.close()


def test_a_second_search_device_supersedes_the_first(Y, oracle, pending_case):
    """The documented exception: a later search_device supersedes a pending one, and finish finishes the later one."""
    import torch
    rows, queries, wr, ws = pending_case
    nq, k = len(queries), PEND_K
    c = make_corpus(Y, PEND_D, "f16", Y.COSINE, rows, None)
    dq = torch.from_numpy(queries).cuda()
    outs = [(torch.empty((nq, k), dtype=torch.int64, device="cuda"), torch.empty((nq, k), dtype=torch.float32, device="cuda"))
            for _ in range(2)]
    for r, s in outs:
        c.search_device(dq.data_ptr(), nq, k, -1.0, r.data_ptr(), s.data_ptr())
    assert c.search_device_finish() >= 1
    r, s = outs[1]
    assert np.array_equal(r.cpu().numpy(), wr) and np.array_equal(s.cpu().numpy(), ws)
    c.close()
