"""GPU tests of the exact scan's two host routes: the blocking search and search_device + search_device_finish enqueue and
finish the same plan, so they must return the same bytes and report the same resolution counts on every path of the scan
(dense, sampled threshold, exhaustive level 1, full exact pass).  A pending search_device is finished against the corpus
it was enqueued on before any other call on that corpus runs, so it also survives a remove that changes nothing
(test_gpu_corpus_lifecycle.py puts every other call between a search_device and its finish)."""
import numpy as np
import pytest

from tests.test_gpu_knn_exact import near_tie_corpus

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def Y():
    import yams_b200
    assert yams_b200.device_count() > 0
    assert yams_b200.plugin_init() == 0, yams_b200.health()
    return yams_b200


def case_rows(O, case):
    """-> (fp16 rows as uint16 [n, d], queries f32 [nq, d], queries sent to level 1, queries sent to the full pass)"""
    if case == "dense":
        n, d = 50_000, 64
        rows32 = O.gen_rows_f32(42, 0, n, d)
        return O.f16_from_float(rows32).reshape(n, d), O.gen_rows_f32(43, 0, 32, d), 0, 0
    if case == "sampled":
        n, d = 200_000, 64
        rows32 = O.gen_rows_f32(42, 0, n, d)
        return O.f16_from_float(rows32).reshape(n, d), O.gen_rows_f32(43, 0, 32, d), 0, 0
    if case == "level1":   # the near-tie corpus of test_gpu_knn_exact: its last query leaves the fast path
        n, d = 100_000, 128
        rng = np.random.default_rng(11)
        q_adv = O.gen_rows_f32(77, 0, 1, d)[0]
        rows32, _ = near_tie_corpus(O, n, d, q_adv, 300, 1e-4, 42, rng)
        queries = np.concatenate([O.gen_rows_f32(43, 0, 7, d), q_adv[None, :]])
        return O.f16_from_float(rows32).reshape(n, d), queries, 1, 0
    assert case == "level2"   # more identical rows than level 1 re-scores: only the full exact pass answers query 0
    n, d = 20_000, 64
    rows32 = O.gen_rows_f32(42, 0, n, d)
    rows32[3000:9000] = rows32[17]
    queries = np.stack([rows32[17], O.gen_rows_f32(43, 0, 1, d)[0]])
    return O.f16_from_float(rows32).reshape(n, d), queries, 1, 1


def device_route(Y, c, queries, k):
    import torch
    nq = len(queries)
    dq = torch.from_numpy(np.ascontiguousarray(queries, dtype=np.float32)).cuda()
    out_r = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    out_s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    c.search_device(dq.data_ptr(), nq, k, -1.0, out_r.data_ptr(), out_s.data_ptr())
    resolved = c.search_device_finish()
    return out_r.cpu().numpy(), out_s.cpu().numpy(), resolved


@pytest.mark.parametrize("case", ["dense", "sampled", "level1", "level2"])
def test_search_and_search_device_agree(Y, oracle, case):
    """Same corpus, same queries: byte-identical rowids and scores, equal counts, and the same number of queries resolved
    exhaustively and by the full pass -- which last_timings reports after either route (device route first, on a fresh
    corpus, so that nothing an earlier blocking search left in the slots can stand in for it)."""
    O = oracle
    k = 10
    rows, queries, want_resolved, want_full = case_rows(O, case)
    c = Y.Corpus(rows.shape[1], Y.F16, Y.COSINE)
    c.append(rows.view(np.float16))
    dr, ds, resolved = device_route(Y, c, queries, k)
    t = c.last_timings()
    assert resolved == want_resolved
    assert t["resolved_exhaustively"] == resolved and t["resolved_full_pass"] == want_full, t
    rid, sc, cnt, flags = c.search(queries, k, threshold=-1.0)
    t = c.last_timings()
    assert int(np.count_nonzero(flags & Y.FLAG_FALLBACK_PATH)) == resolved
    assert t["resolved_exhaustively"] == resolved and t["resolved_full_pass"] == want_full, t
    assert rid.tobytes() == dr.tobytes() and sc.tobytes() == ds.tobytes()
    assert np.array_equal(cnt, (dr >= 0).sum(axis=1).astype(np.uint32))
    c.close()


def test_search_device_finish_after_noop_remove(Y, oracle):
    """search_device, then a corpus_remove of a rowid the corpus does not hold (its prefix scan still runs, on the
    corpus's scratch buffer), then search_device_finish: the near-tie query is re-scored by the exhaustive level with its
    own query norm, so every result equals the reference's, bit for bit."""
    import torch
    O = oracle
    n, d, nq, k = 150_000, 64, 16, 10
    rng = np.random.default_rng(3)
    q_adv = O.gen_rows_f32(78, 0, 1, d)[0]
    rows32, _ = near_tie_corpus(O, n, d, q_adv, 250, 1e-4, 42, rng)
    rows = O.f16_from_float(rows32).reshape(n, d)
    queries = O.gen_rows_f32(43, 0, nq, d)
    queries[4] = q_adv
    c = Y.Corpus(d, Y.F16, Y.COSINE)
    c.append(rows.view(np.float16))
    dq = torch.from_numpy(queries).cuda()
    out_r = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    out_s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    c.search_device(dq.data_ptr(), nq, k, -1.0, out_r.data_ptr(), out_s.data_ptr())
    assert c.remove([n + 5]) == 0
    assert c.search_device_finish() >= 1                             # the near-tie query went through the exhaustive level
    rc, wr, ws, wc = O.exact_scan_cosine_batch(rows, queries, k)
    assert rc == 0
    assert np.array_equal(out_r.cpu().numpy(), wr) and np.array_equal(out_s.cpu().numpy(), ws)
    c.close()
