"""Candidate-set PQ search (PqIndex.search(allowed=...)) and document-level top-k (Corpus.search_documents).

* PQ candidates against the reference: simeon's own ADC scores (oracle.pq_scores_ref) around a restatement of
  simeonPqSearchUnlocked's candidate branch (sqlite_vec_backend.cpp:3910-4051), stored in tests/golden/ref_pq_candidates.json
  by tests/golden/make_ref_pq_candidates.py (ordinary data, and rows whose approximate scores differ only by the order of the
  float sum); and bit-identity with the full scan when every list holds every row.
* DocumentTopK (retainBestRecordPerDocument, sqlite_vec_backend.cpp:86-125) in both arithmetic modes against the C oracle:
  the exact fallback against exact_scan_cosine(all_matching=True), the PQ branch against yo_cosine_similarity_f64 over the
  rows the index holds, each grouped in Python.
* The C++ adapter's searchDocumentCandidates (tests/host_cpp/test_document_search.cpp)."""
import functools
import json
import os
import subprocess

import numpy as np
import pytest

from tests import ref_checks

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def Y():
    import yams_b200
    assert yams_b200.device_count() > 0
    assert yams_b200.plugin_init() == 0, yams_b200.health()
    return yams_b200


# ---- PQ candidate sets ------------------------------------------------------------------------------------------------

PQC_SEARCHES = ((10, 3, -1.0), (4, 1, 0.05))   # (k, rerank_factor, threshold): approxK 30 and 4
PQC_GOLDEN = os.path.join(ref_checks.GOLDEN, "ref_pq_candidates.json")


@functools.lru_cache(maxsize=None)
def pq_golden() -> dict:
    with open(PQC_GOLDEN) as f:
        return json.load(f)


def pq_candidates_case(O, dtype: str):
    """The corpus, index and candidate lists of the "pq_candidates" check.  -> dict(rows to append, held float32 values, rowids,
    tie keys, codebooks, m, kc, queries[600], lists[600])"""
    n, d, m, kc = 6000, 128, 16, 64
    rng = np.random.default_rng(21)
    rows = O.gen_rows_f32(42, 0, n, d) * rng.uniform(0.5, 2.0, size=(n, 1)).astype(np.float32)
    rows[100:140] = rows[99]                        # identical rows: identical codes, equal ADC scores -> tie keys decide
    zero = [7, 3001, 5999]
    rows[zero] = 0                                  # left out of the index
    rowids = np.arange(n, dtype=np.int64) * 3 + 1   # rowids % 3 != 1 are unknown to the corpus
    tie_keys = rng.integers(0, 1 << 62, size=n).astype(np.uint64)
    codebooks = (rng.normal(size=(m, kc, d // m)) / np.sqrt(d)).astype(np.float32).reshape(-1)
    queries = O.gen_rows_f32(43, 0, 600, d) * np.float32(1.5)
    queries[3::50] = rows[99] * np.float32(0.5)      # hit the run of identical rows
    queries[11] = 0                                 # cannot be normalised: no results
    lists = []
    for i in range(600):
        kind = i % 6
        if kind == 0:
            idx = np.zeros(0, dtype=np.int64)                                              # empty list
        elif kind == 1:
            idx = rng.choice(n, size=5, replace=False)                                     # fewer than approxK
        elif kind == 2:
            idx = np.concatenate([rng.choice(n, size=800, replace=False), np.arange(99, 140)])   # approxK .. 4096, with the ties
        elif kind == 3:
            idx = rng.choice(n, size=5000, replace=False)                                  # more than 4096
        elif kind == 4:
            base = rng.choice(n, size=300, replace=False)                                  # repeats, unindexed and unknown rowids
            idx = np.concatenate([base, base[:50], np.array(zero), np.arange(99, 140), np.arange(99, 110)])
        else:
            idx = np.arange(n)                                                              # every row
        ids = rowids[np.asarray(idx, dtype=np.int64)]
        if kind == 4:
            ids = np.concatenate([ids, np.array([0, 2, 3 * n + 7, -5], dtype=np.int64)])
        lists.append(rng.permutation(ids))
    if dtype == "f16":
        bits = O.f16_from_float(rows).reshape(n, d)
        held = O.f16_to_float(bits).reshape(n, d)
        append = bits.view(np.float16)
    else:
        held = append = rows
    return dict(append=append, held=held, rowids=rowids, tie_keys=tie_keys, codebooks=codebooks, m=m, kc=kc, queries=queries, lists=lists)


@pytest.mark.parametrize("dtype", ["f32", "f16"])
def test_pq_candidates_match_the_reference_engine(Y, oracle, dtype):
    want = pq_golden()[dtype]
    cs = pq_candidates_case(oracle, dtype)
    d = cs["held"].shape[1]
    assert ref_checks.digest(cs["held"], cs["queries"], *cs["lists"]) == want["inputs"]
    c = Y.Corpus(d, Y.F16 if dtype == "f16" else Y.F32, Y.COSINE)
    c.append(cs["append"], rowids=cs["rowids"])
    pq = Y.PqIndex(c, cs["m"], cs["kc"], cs["codebooks"], tie_break_keys=cs["tie_keys"])
    for (k, rf, thr), results in zip(PQC_SEARCHES, want["searches"]):
        for nq in (1, 7, 600):                      # 600 crosses the 512-query slice
            rid, sc, cnt, flags = pq.search(cs["queries"][:nq], k, rerank_factor=rf, threshold=thr, allowed=cs["lists"][:nq])
            for qi in range(nq):
                n, dg = results[qi]
                assert cnt[qi] == n, (qi, k, nq)
                assert ref_checks.digest(rid[qi, :n].astype(np.int64), sc[qi, :n].astype(np.float32)) == dg, (qi, k, nq)
                assert np.all(rid[qi, n:] == -1)
    pq.close()
    c.close()


def pq_order_case(O):
    """Approximate scores that differ only by the ORDER of the float sum: every subspace has the same 16 centroids (all of norm
    1/4, so a row made of them is unit length and encodes to exactly the centroids it was built from), every query repeats one
    sub-vector (so the lookup table is the same in every subspace), and each query's candidates are 12 rows whose codes are
    permutations of one multiset of code bytes.  Their ADC sums are equal in exact arithmetic; which one the selection keeps
    (k = 1, rerank_factor = 1: approxK = 1) depends on the float order of inner_product_from_lut.
    -> dict(rows, rowids, codes, codebooks, m, kc, queries[256], lists[256])"""
    m, kc, dsub = 16, 16, 4
    d = m * dsub
    rng = np.random.default_rng(33)
    cents = rng.normal(size=(kc, dsub))
    cents = (cents / np.linalg.norm(cents, axis=1, keepdims=True) * 0.25).astype(np.float32)
    codebooks = np.ascontiguousarray(np.broadcast_to(cents, (m, kc, dsub))).reshape(-1)
    nq, per = 256, 12
    codes = np.empty((nq * per, m), dtype=np.uint8)
    for g in range(nq):
        base = rng.integers(0, kc, size=m)
        for j in range(per):
            codes[g * per + j] = rng.permutation(base)
    rows = cents[codes.astype(np.int64)].reshape(len(codes), d)
    rowids = np.arange(len(codes), dtype=np.int64) * 2 + 1
    queries = np.tile(rng.normal(size=(nq, dsub)).astype(np.float32), (1, m))
    lists = [rng.permutation(rowids[g * per:(g + 1) * per]) for g in range(nq)]
    return dict(rows=rows, rowids=rowids, codes=codes, codebooks=codebooks, m=m, kc=kc, queries=queries, lists=lists)


def test_pq_candidates_adc_summation_order(Y, oracle):
    """The candidate gather must sum the lookup table in the reference's order: with approxK = 1 the row kept among rows of
    equal exact ADC sum is decided by float rounding alone (answers from simeon's own ADC scores)."""
    want = pq_golden()["order"]
    cs = pq_order_case(oracle)
    n, d = cs["rows"].shape
    assert ref_checks.digest(cs["rows"], cs["queries"], *cs["lists"]) == want["inputs"]
    c = Y.Corpus(d, Y.F32, Y.COSINE)
    c.append(cs["rows"], rowids=cs["rowids"])
    pq = Y.PqIndex(c, cs["m"], cs["kc"], cs["codebooks"], tie_break_keys=np.arange(n, dtype=np.uint64))
    codes, _ = pq.codes()
    assert np.array_equal(codes, cs["codes"])                  # the rows encode to the codes they were built from
    rid, sc, cnt, _ = pq.search(cs["queries"], 1, rerank_factor=1, threshold=-1.0, allowed=cs["lists"])
    for qi, (nres, dg) in enumerate(want["searches"][0]):
        assert cnt[qi] == nres, qi
        assert ref_checks.digest(rid[qi, :nres].astype(np.int64), sc[qi, :nres].astype(np.float32)) == dg, qi
    pq.close()
    c.close()


def test_pq_candidates_with_every_row_equal_the_full_scan(Y, oracle):
    """Every list = every indexed row: results AND flags bit-identical to pq_search (the filtered-scan shape of
    test_pq_filtered_scan_large_index, where tie keys decide among equal approximate scores)."""
    O = oracle
    n, d, m, kc = 300_000, 64, 8, 16
    rng = np.random.default_rng(11)
    rows = O.gen_rows_f32(42, 0, n, d)
    rows[1000:1064] = rows[2000]
    rows[5] = 0                                      # not in the index: its rowid is ignored
    rowids = np.arange(n, dtype=np.int64) + 3
    tie_keys = rng.permutation(n).astype(np.uint64)
    codebooks = (rng.normal(size=(m, kc, d // m)) / np.sqrt(d)).astype(np.float32).reshape(-1)
    c = Y.Corpus(d, Y.F32, Y.COSINE)
    c.append(rows, rowids=rowids)
    pq = Y.PqIndex(c, m, kc, codebooks, tie_break_keys=tie_keys)
    queries = O.gen_rows_f32(43, 0, 5, d)
    queries[1] = rows[2000]
    every = [rng.permutation(rowids) for _ in range(5)]
    for k, rf, thr in ((10, 2, -1.0), (40, 3, 0.0), (1, 1, -1.0)):
        full = pq.search(queries, k, rerank_factor=rf, threshold=thr)
        cand = pq.search(queries, k, rerank_factor=rf, threshold=thr, allowed=every)
        for a, b in zip(full, cand):
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), (k, rf)
    pq.close()
    c.close()


def test_pq_candidates_limits(Y, oracle):
    O = oracle
    n, d, m, kc = 3000, 32, 4, 16
    rng = np.random.default_rng(5)
    rows = O.gen_rows_f32(42, 0, n, d)
    c = Y.Corpus(d, Y.F32, Y.COSINE)
    c.append(rows)
    pq = Y.PqIndex(c, m, kc, (rng.normal(size=(m, kc, d // m)) / np.sqrt(d)).astype(np.float32).reshape(-1))
    q = O.gen_rows_f32(43, 0, 2, d)
    # k * rerank_factor > 1024 is fine while a query has at most 1024 distinct indexed candidates (approxK = candidateCount)
    short = [np.arange(1000), np.concatenate([np.arange(900), np.arange(900), [n + 5]])]
    rid, sc, cnt, _ = pq.search(q, 600, rerank_factor=4, threshold=-1.0, allowed=short)
    assert list(cnt) == [600, 600]
    with pytest.raises(Y.YamsB200Error) as e:
        pq.search(q, 600, rerank_factor=4, threshold=-1.0, allowed=[np.arange(1025), np.arange(3)])
    assert e.value.status == 1 and "1024" in str(e.value)
    # k == 0 and empty lists give nothing
    assert list(pq.search(q, 0, allowed=short)[2]) == [0, 0]
    assert list(pq.search(q, 5, allowed=[[], []])[2]) == [0, 0]
    c.append(rows[:1], rowids=[n])
    with pytest.raises(Y.YamsB200Error):
        pq.search(q, 5, allowed=short)
    pq.close()
    c.close()


# ---- document top-k ------------------------------------------------------------------------------------------------------

N_DOC, D_DOC = 8000, 64
ZERO, INF, NAN, TINY = 5, 6, 7, 8


def doc_corpus(O):
    rows = O.gen_rows_f32(42, 0, N_DOC, D_DOC) * np.float32(1.3)
    rows[21] = rows[20]
    rows[22] = rows[20]
    rows[30] = rows[31]
    rows[ZERO] = 0
    rows[INF, 3] = np.inf
    rows[NAN, 9] = np.nan
    rows[TINY] = O.gen_rows_f32(9, 0, 1, D_DOC)[0] * np.float32(3e-8)   # |r|^2 ~ 1e-15: in the index, skipped by the exact scan
    rowids = np.arange(N_DOC, dtype=np.int64) * 2 + 10                  # odd rowids are unknown
    return rows, rowids


def expected_sims(O, rows, rowids, query, rids, threshold, pq_mode):
    """rowid -> similarity of every row of `rids` that is a result (the oracle's arithmetic of each mode)"""
    want = np.unique(np.asarray(rids, dtype=np.int64))
    if not pq_mode:
        rc, r, s = O.exact_scan_cosine(rows, query, 0, threshold=threshold, rowids=rowids, allowed=want, all_matching=True)
        assert rc == 0
        return dict(zip(r.tolist(), s.tolist()))
    _, ok = O.normalize_like_reference(query[None, :])
    if not ok[0]:
        return {}
    _, in_index = O.normalize_like_reference(rows)
    pos = {int(r): i for i, r in enumerate(rowids)}
    q = np.ascontiguousarray(query, dtype=np.float32)
    out = {}
    for r in want.tolist():
        i = pos.get(r)
        if i is None or not in_index[i]:
            continue
        row = np.ascontiguousarray(rows[i], dtype=np.float32)
        s = np.float32(O.lib().yo_cosine_similarity_f64(q.ctypes.data_as(O.f32p), row.ctypes.data_as(O.f32p), D_DOC))
        if s == s and not s < np.float32(threshold):
            out[r] = float(s)
    return out


def group(docs, sims, k):
    """retainBestRecordPerDocument: best row by (sim desc, position asc); documents by (sim desc, index asc); first k"""
    best = []
    for di, rs in enumerate(docs):
        b = None
        for r in rs:
            s = sims.get(int(r))
            if s is not None and (b is None or s > b[0]):
                b = (s, int(r))
        if b is not None:
            best.append((b[0], di, b[1]))
    best.sort(key=lambda t: (-t[0], t[1]))
    return best[:k]


def check_documents(Y, O, c, pq, rows, rowids, queries, docs, k, threshold):
    got_d, got_r, got_s, got_c = c.search_documents(queries, k, docs, threshold=threshold, pq=pq)
    for qi in range(len(queries)):
        flat = [r for ds in docs[qi] for r in ds]
        exp = group(docs[qi], expected_sims(O, rows, rowids, queries[qi], flat, threshold, pq is not None), k)
        n = len(exp)
        assert got_c[qi] == n, (qi, k, pq is not None)
        assert list(got_d[qi, :n]) == [e[1] for e in exp], qi
        assert list(got_r[qi, :n]) == [e[2] for e in exp], qi
        assert np.array_equal(got_s[qi, :n], np.array([e[0] for e in exp], dtype=np.float32)), qi
        assert np.all(got_d[qi, n:] == -1) and np.all(got_r[qi, n:] == -1) and np.all(got_s[qi, n:] == 0)
    return got_d, got_r, got_s, got_c


@pytest.fixture(scope="module")
def doc_setup(Y, oracle):
    O = oracle
    rows, rowids = doc_corpus(O)
    c = Y.Corpus(D_DOC, Y.F32, Y.COSINE)
    c.append(rows, rowids=rowids)
    rng = np.random.default_rng(8)
    m, kc = 8, 16
    pq = Y.PqIndex(c, m, kc, (rng.normal(size=(m, kc, D_DOC // m)) / np.sqrt(D_DOC)).astype(np.float32).reshape(-1))
    rid = lambda i: int(rowids[i])   # noqa: E731
    queries = O.gen_rows_f32(43, 0, 3, D_DOC)
    queries[0] = rows[20] * np.float32(0.7)
    q0 = [
        [rid(22), rid(20)],                              # identical rows, chunk order the reverse of rowid order: position decides
        [rid(21)],                                       # ties document 0: the lower document index first
        [],                                              # empty
        [rid(TINY)],                                     # PQ mode only
        [rid(ZERO), rid(INF), rid(NAN), 11],             # never a result (11 is an unknown rowid)
        [rid(i) for i in range(200, 233)],               # 33 rows
        [rid(i) for i in range(3000, 6000)][::-1],       # 3000 rows
        [rid(40)],
        [rid(31), rid(30)],
    ]
    q1 = [[rid(i)] for i in range(1000, 6000)]           # 5000 documents of one row
    q2 = [[rid(i) for i in range(s, s + 7)] for s in range(100, 900, 7)] + [[rid(20)], [rid(21), rid(TINY)]]
    docs = [q0, q1, q2]
    yield O, c, pq, rows, rowids, queries, docs
    pq.close()
    c.close()


@pytest.mark.parametrize("mode", ["exact", "pq"])
def test_documents_match_the_oracle(Y, doc_setup, mode):
    O, c, pq, rows, rowids, queries, docs = doc_setup
    p = pq if mode == "pq" else None
    for k in (1, 10, 4096):                              # 4096 > the valid documents of queries 0 and 2
        check_documents(Y, O, c, p, rows, rowids, queries, docs, k, -1.0)
    got_d, got_r, _, _ = check_documents(Y, O, c, p, rows, rowids, queries, docs, 3, -1.0)
    assert list(got_d[0, :2]) == [0, 1] and got_r[0, 0] == rowids[22]   # the in-document and the between-document ties
    # a threshold equal to a document's best score keeps that document
    _, _, s, cnt = c.search_documents(queries, 50, docs, threshold=-1.0, pq=p)
    thr = float(s[2, 5])
    _, _, s2, cnt2 = check_documents(Y, O, c, p, rows, rowids, queries, docs, 50, thr)
    assert s2[2, cnt2[2] - 1] == np.float32(thr)
    # k == 0
    assert list(c.search_documents(queries, 0, docs, pq=p)[3]) == [0, 0, 0]


def test_documents_modes_differ_on_tiny_rows(Y, doc_setup):
    """Rows with 1e-20 < |r|^2 <= 1e-12 are in the PQ index (scored) but skipped by the exact scan."""
    O, c, pq, rows, rowids, queries, docs = doc_setup
    tiny_only = [[[int(rowids[TINY])]]]
    assert c.search_documents(queries[:1], 5, tiny_only)[3][0] == 0
    d, r, s, cnt = c.search_documents(queries[:1], 5, tiny_only, pq=pq)
    assert cnt[0] == 1 and r[0, 0] == rowids[TINY] and d[0, 0] == 0
    # zero / unknown / non-finite rows are nothing in either mode
    never = [[[int(rowids[ZERO]), int(rowids[NAN]), int(rowids[INF]), 13]]]
    assert c.search_documents(queries[:1], 5, never)[3][0] == 0
    assert c.search_documents(queries[:1], 5, never, pq=pq)[3][0] == 0


def test_documents_many_queries_cross_slices(Y, doc_setup):
    O, c, pq, rows, rowids, queries, docs = doc_setup
    rng = np.random.default_rng(4)
    nq = 520
    qs = O.gen_rows_f32(44, 0, nq, D_DOC)
    many = []
    for i in range(nq):
        pick = rowids[rng.choice(N_DOC, size=7, replace=False)]
        many.append([list(pick[:3]), list(pick[3:4]), [], list(pick[4:])])
    for p in (None, pq):
        check_documents(Y, O, c, p, rows, rowids, qs, many, 3, -1.0)


def test_documents_errors(Y, doc_setup, oracle):
    O, c, pq, rows, rowids, queries, docs = doc_setup
    zero_q = np.zeros((1, D_DOC), dtype=np.float32)
    one = [[[int(rowids[20]), int(rowids[40])]]]
    with pytest.raises(Y.YamsB200Error) as e:            # exact mode: a zero query is an error
        c.search_documents(zero_q, 5, one)
    assert e.value.status == 1
    assert c.search_documents(zero_q, 5, one, pq=pq)[3][0] == 0   # PQ mode: no results
    bad = queries[:1].copy()
    bad[0, 2] = np.inf
    with pytest.raises(Y.YamsB200Error):
        c.search_documents(bad, 5, one)
    # a rowid in two documents of one query; the same rowid in two QUERIES is fine
    with pytest.raises(Y.YamsB200Error) as e:
        c.search_documents(queries[:1], 5, [[[int(rowids[20])], [int(rowids[40]), int(rowids[20])]]])
    assert e.value.status == 1
    assert list(c.search_documents(queries[:2], 5, [one[0], one[0]])[3]) == [1, 1]
    # an index of another corpus, a stale index
    c2 = Y.Corpus(D_DOC, Y.F32, Y.COSINE)
    c2.append(rows[:100])
    with pytest.raises(Y.YamsB200Error):
        c2.search_documents(queries[:1], 5, [[[0, 1]]], pq=pq)
    rng = np.random.default_rng(1)
    pq2 = Y.PqIndex(c2, 8, 16, (rng.normal(size=(8, 16, D_DOC // 8))).astype(np.float32).reshape(-1))
    c2.append(rows[100:101], rowids=[100])
    with pytest.raises(Y.YamsB200Error):
        c2.search_documents(queries[:1], 5, [[[0, 1]]], pq=pq2)
    assert c2.search_documents(queries[:1], 5, [[[0], [1]]])[3][0] == 2   # the exact mode does not need the index
    pq2.close()
    c2.close()


def test_cpp_document_search(Y, tmp_path):
    """B200VectorStore::searchDocumentCandidates (IDocumentCandidateVectorStore) over the C ABI."""
    exe = str(tmp_path / "test_document_search")
    subprocess.check_call(["/usr/bin/g++", "-std=c++20", "-O1", os.path.join(ROOT, "tests", "host_cpp", "test_document_search.cpp"),
                           "-o", exe, "-L" + os.path.join(ROOT, "yams_b200"), "-lyams_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "yams_b200")])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "ALL OK" in out.stdout, out.stdout + out.stderr
