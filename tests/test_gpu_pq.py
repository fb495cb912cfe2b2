"""GPU parity of the SimeonPqAdc engine (SURVEY.md §8f N3): index build (normalise + encode) and search (lookup table, ADC scan,
best approxK, exact rerank) against simeon's own ProductQuantizer / PQInnerProductQuery and a restatement of
simeonPqSearchUnlocked (src/vector/sqlite_vec_backend.cpp:3868-4056) around them.  The reference's codes and answers are stored
in tests/golden/ref_checks.json."""
import os

import numpy as np
import pytest

from tests import ref_checks

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def Y():
    import yams_b200
    assert yams_b200.device_count() > 0
    assert yams_b200.plugin_init() == 0, yams_b200.health()
    return yams_b200


# simeon's own Lloyd training over the first 4096 normalised rows of the (20000, 128, 8, 64) case, stored as int8 x 2^-10
TRAINED_CODEBOOKS = os.path.join(ref_checks.GOLDEN, "pq_codebooks_20000x128.npy")


def check_searches(pq, queries, k, rerank, thr, want):
    """want[qi] = [count, digest of (rowids, scores)] of the reference engine's answer"""
    rid, sc, cnt, flags = pq.search(queries, k, rerank_factor=rerank, threshold=thr)
    for qi in range(len(queries)):
        n, dg = want[qi]
        assert cnt[qi] == n, (qi, k)
        assert ref_checks.digest(rid[qi, :n].astype(np.int64), sc[qi, :n].astype(np.float32)) == dg, (qi, k)
    return rid, sc, cnt, flags


PQ_CFGS = [(12_000, 768, 32, 256), (9_000, 384, 32, 256), (20_000, 128, 8, 64), (5_000, 96, 4, 16)]
PQ_SEARCHES = ((10, 2, 0.0), (5, 4, -1.0), (25, 1, 0.1))      # (k, rerank_factor, threshold) of the "pq" answers


def pq_case(O, cfg):
    """The corpus, index and queries of the "pq" check (fp32 rows).  -> dict(rows, rowids, tie_keys, codebooks, m, kc, queries)"""
    n, d, m, kc = cfg
    rng = np.random.default_rng(n)
    rows = O.gen_rows_f32(42, 0, n, d) * rng.uniform(0.5, 3.0, size=(n, 1)).astype(np.float32)   # not unit length: the index normalises
    rows[17] = 0                                                                    # cannot be normalised: left out of the index
    rows[n // 3] = rows[n // 3 + 1]                                                 # identical codes -> equal ADC scores -> tie keys decide
    rowids = (np.arange(n, dtype=np.int64) * 2 + 5)
    tie_keys = rng.integers(0, 1 << 62, size=n).astype(np.uint64)
    if (n, d) == (20_000, 128):
        codebooks = np.load(TRAINED_CODEBOOKS).astype(np.float32) * np.float32(2.0 ** -10)   # the reference's own Lloyd training
    else:
        codebooks = (rng.normal(size=(m, kc, d // m)) / np.sqrt(d)).astype(np.float32).reshape(-1)
    queries = O.gen_rows_f32(43, 0, 6, d) * np.float32(2.0)
    queries[2] = rows[n // 3] * np.float32(0.5)                                     # hits the duplicated row pair
    return dict(rows=rows, rowids=rowids, tie_keys=tie_keys, codebooks=codebooks, m=m, kc=kc, queries=queries)


@pytest.mark.parametrize("cfg", PQ_CFGS)
def test_pq_index_and_search_match_the_reference_engine(Y, oracle, cfg):
    O = oracle
    want = ref_checks.load()["pq"][ref_checks.key(cfg)]
    n, d, m, kc = cfg
    cs = pq_case(O, cfg)
    rows, rowids, queries = cs["rows"], cs["rowids"], cs["queries"]
    normed, ok = O.normalize_like_reference(rows)
    c = Y.Corpus(d, Y.F32, Y.COSINE)
    c.append(rows, rowids=rowids)
    pq = Y.PqIndex(c, m, kc, cs["codebooks"], tie_break_keys=cs["tie_keys"])
    codes, code_rowids = pq.codes()
    assert np.array_equal(code_rowids, rowids[ok]) and len(codes) == n - 1
    assert ref_checks.digest(codes) == want["codes"]                                # every code byte equals simeon's encode
    for (k, rerank, thr), results in zip(PQ_SEARCHES, want["searches"]):
        check_searches(pq, queries, k, rerank, thr, results)
    # a query that cannot be normalised returns nothing (:3896-3898); k == 0 returns nothing
    rid, sc, cnt, flags = pq.search(np.zeros((1, d), dtype=np.float32), 5)
    assert cnt[0] == 0
    assert pq.search(queries[:1], 0)[2][0] == 0
    # a mutated corpus invalidates the index (the reference marks it dirty and rebuilds)
    c.append(rows[:1], rowids=[int(rowids[-1]) + 1])
    with pytest.raises(Y.YamsB200Error):
        pq.search(queries[:1], 5)
    pq.close()
    c.close()


PQ_FP16_SEARCH = (10, 2, -1.0)


def pq_fp16_case(O):
    """The fp16 corpus of the "pq_fp16" check, no tie keys.  -> dict(bits u16[n, d], held f32 values, codebooks, m, kc, queries)"""
    n, d, m, kc = 12_000, 256, 16, 256
    rng = np.random.default_rng(3)
    rows16 = O.f16_from_float(O.gen_rows_f32(42, 0, n, d)).reshape(n, d)
    rows = O.f16_to_float(rows16).reshape(n, d)
    rows[100] = rows[50]
    rows16[100] = rows16[50]
    codebooks = (rng.normal(size=(m, kc, d // m)) / np.sqrt(d)).astype(np.float32).reshape(-1)
    queries = O.gen_rows_f32(43, 0, 4, d)
    queries[1] = rows[50]
    return dict(bits=rows16, held=rows, codebooks=codebooks, m=m, kc=kc, queries=queries)


def test_pq_over_an_fp16_corpus_and_row_order_ties(Y, oracle):
    """fp16 corpus (the C2 layout): the index is built from the stored (fp16) values; without tie keys equal approximate
    scores are ordered by row."""
    cs = pq_fp16_case(oracle)
    d = cs["held"].shape[1]
    c = Y.Corpus(d, Y.F16, Y.COSINE)
    c.append(cs["bits"].view(np.float16))
    pq = Y.PqIndex(c, cs["m"], cs["kc"], cs["codebooks"])
    rid, sc, cnt, flags = check_searches(pq, cs["queries"], *PQ_FP16_SEARCH, ref_checks.load()["pq_fp16"])
    assert list(rid[1, :2]) == [50, 100] and flags[1] & Y.FLAG_TIE_AT_K == 0
    pq.close()
    c.close()


PQ_LARGE_SEARCHES = ((10, 2, -1.0), (40, 3, 0.0))


def pq_large_case(O):
    """The 300k-row corpus of the "pq_large" check.  -> dict(rows, rowids, tie_keys, codebooks, m, kc, queries[5])"""
    n, d, m, kc = 300_000, 64, 8, 16
    rng = np.random.default_rng(11)
    rows = O.gen_rows_f32(42, 0, n, d)
    rows[1000:1064] = rows[2000]                                                    # a run of identical rows across the list boundary
    rowids = np.arange(n, dtype=np.int64) + 3
    tie_keys = rng.permutation(n).astype(np.uint64)
    codebooks = (rng.normal(size=(m, kc, d // m)) / np.sqrt(d)).astype(np.float32).reshape(-1)
    queries = O.gen_rows_f32(43, 0, 5, d)
    queries[1] = rows[2000]
    return dict(rows=rows, rowids=rowids, tie_keys=tie_keys, codebooks=codebooks, m=m, kc=kc, queries=queries)


def test_pq_filtered_scan_large_index(Y, oracle):
    """>= 64 tiles: the sampled-threshold (filtered) ADC pass replaces the per-tile sorting network; 1, 2 and 5 queries walk the
    1-, 2- and 4-table CTA variants.  Small k (16 centroids) makes equal approximate scores common: tie keys decide."""
    cs = pq_large_case(oracle)
    d = cs["rows"].shape[1]
    c = Y.Corpus(d, Y.F32, Y.COSINE)
    c.append(cs["rows"], rowids=cs["rowids"])
    pq = Y.PqIndex(c, cs["m"], cs["kc"], cs["codebooks"], tie_break_keys=cs["tie_keys"])
    for nq in (1, 2, 5):
        for (k, rerank, thr), results in zip(PQ_LARGE_SEARCHES, ref_checks.load()["pq_large"]):
            check_searches(pq, cs["queries"][:nq], k, rerank, thr, results[:nq])
    pq.close()
    c.close()


PQ_OVERFLOW_SEARCH = (10, 2, -1.0)


def pq_overflow_case(O):
    """The sampled tiles (every 4th of 74) hold only rows pointing away from the query, every other tile rows pointing at it.
    -> dict(rows, rowids, tie_keys, codebooks, m, kc, query[1, d])"""
    n, d, m, kc = 300_000, 64, 8, 16
    rng = np.random.default_rng(12)
    query = O.gen_rows_f32(43, 0, 1, d)
    noise = O.gen_rows_f32(42, 0, n, d)
    tile = np.arange(n) // 4096
    sign = np.where((tile % 4 == 0) & (tile < 64), -1.0, 1.0).astype(np.float32)[:, None]
    rows = (noise * np.float32(0.7) + sign * query).astype(np.float32)
    rowids = np.arange(n, dtype=np.int64)
    tie_keys = np.arange(n, dtype=np.uint64)
    codebooks = (rng.normal(size=(m, kc, d // m)) / np.sqrt(d)).astype(np.float32).reshape(-1)
    return dict(rows=rows, rowids=rowids, tie_keys=tie_keys, codebooks=codebooks, m=m, kc=kc, query=query)


def test_pq_filtered_scan_overflow_falls_back(Y, oracle):
    """The sample's threshold admits ~237 k rows into a 32 k list; the engine must notice and redo the selection unfiltered."""
    cs = pq_overflow_case(oracle)
    d = cs["rows"].shape[1]
    c = Y.Corpus(d, Y.F32, Y.COSINE)
    c.append(cs["rows"], rowids=cs["rowids"])
    pq = Y.PqIndex(c, cs["m"], cs["kc"], cs["codebooks"], tie_break_keys=cs["tie_keys"])
    check_searches(pq, cs["query"], *PQ_OVERFLOW_SEARCH, ref_checks.load()["pq_overflow"])
    assert pq.last_path() == {"filtered": True, "qg": 1, "sample_tiles": 16, "rerun": True}
    pq.close()
    c.close()
