"""The lead-text field (yams_b200_bm25_build_lead) and the strategy router (yams_b200_bm25_score_strategy: its three pools and the
entropy route) on the device, bit for bit: against the stored answers of simeon's own build (tests/golden/ref_strategy.json) and the restatement
(tests/strategy_restated.py), for both variants, with and without concepts; lead cuts at every whitespace byte, documents
shorter and longer than 64 tokens, corpora whose lead texts are all empty, a query longer than 64 tokens, n_docs across the
score tile; the aux accessors against the reference's postings, the Atire view's aux word field, an index built without the
lead field; both sides of the keyphrase gate, stopword-only queries, the route's replay taken and not taken; 4 101 queries
across a memory-budget split, 200 000 documents against the reference, two threads scoring concurrently, the argument errors."""
import json
import os
import threading

import numpy as np
import pytest

import yams_b200 as Y
from tests import bm25_restated as B
from tests import concepts_restated as R
from tests import strategy_restated as S
from tests.golden import make_strategy_golden as G

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STORED = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_strategy.json")))
CCFG = R.CCfg(**STORED["concept_config"])
POOLS = (Y.BM25_STRATEGY_BM25, Y.BM25_STRATEGY_KEYPHRASE, Y.BM25_STRATEGY_LEAD_FIELD, Y.BM25_STRATEGY_ROUTED)


def _index(variant, docs, lead):
    return Y.Bm25Index(docs, lead_tokens=lead, variant=variant)


def _pool(X, pool, q):
    return S.route(X.score(q)) if pool == Y.BM25_STRATEGY_ROUTED else pool


def _check(got, i, want, k, pool):
    assert got["scores"][i].tobytes() == want.tobytes(), i
    wd, ws = B.topk(want, k)
    c = int(got["counts"][i])
    assert c == len(wd) and np.array_equal(got["docs"][i, :c], wd) and got["topk_scores"][i, :c].tobytes() == ws.tobytes(), i
    assert np.all(got["docs"][i, c:] == 0xFFFFFFFF) and np.all(got["topk_scores"][i, c:] == 0)
    assert got["chosen"][i] == pool


def _check_all(D, X, queries, docs, k=10, K=None, C=None):
    for pool in POOLS:
        for blend in (False, True):
            got = D.score_strategy(queries, pool, k=k, concepts=C if blend else None, weight=0.5)
            for i, q in enumerate(queries):
                _check(got, i, S.score(X, pool, q, K if blend else None, 0.5), k, _pool(X, pool, q))


@pytest.mark.parametrize("case", STORED["cases"], ids=[c["name"] for c in STORED["cases"]])
def test_stored_answers(case):
    docs, queries = G.case_inputs(case)
    D = _index(G.VARIANTS[case["variant"]], docs, case["lead"])
    C = D.mine_concepts(docs, **CCFG.kw())
    a = D.aux_stats()
    for f, want in zip((0, 1), case["aux"]):
        assert a["terms"][f] == want["terms"] and a["postings"][f] == want["postings"]
    assert a["n_docs"] == case["aux"][0]["docs"] and a["total_tokens"] == case["aux"][0]["sum"] and float(a["avg_dl"]) == case["aux"][0]["avg"]
    assert float(a["ngram_avg_dl"]) == case["aux"][1]["avg"]
    for pool in POOLS:
        for w in (None, 0.5):
            got = D.score_strategy(queries, pool, k=10, concepts=C if w is not None else None, weight=w or 0.0)
            assert [G.digest(r) for r in got["scores"]] == case["scores"][f"{pool}/{w}"], (pool, w)
            assert got["chosen"].tolist() == (case["routed"] if pool == Y.BM25_STRATEGY_ROUTED else [pool] * len(queries))


GRID = [(v, n, L) for v in (B.SAB, B.ATIRE) for n, L in ((1, 64), (2, 64), (9, 1), (10, 64), (11, 2), (4096, 64), (4097, 64), (4097, 5))]


@pytest.mark.parametrize("variant,n,L", GRID)
def test_grid(variant, n, L):
    docs, voc = S.gen_lead_corpus(500 + n + L, n)
    queries = S.gen_lead_queries(600 + n, voc, 16)
    X = S.Index(B.Config(variant=variant), docs, L)
    K = R.Concepts(docs, docs, CCFG)
    D = _index(variant, docs, L)
    _check_all(D, X, queries, docs, k=7, K=K, C=D.mine_concepts(docs, **CCFG.kw()))
    for f in range(4):
        assert np.array_equal(D.doc_lengths(f), X.doc_lengths(f)), f
    a = D.aux_stats()
    assert a["n_docs"] == (n if X.aux_active else 0) and a["avg_dl"] == X.aux_words.avg and a["ngram_avg_dl"] == X.aux_ngrams.avg
    assert a["terms"] == (len(X.aux_words.postings), len(X.aux_ngrams.postings)) and a["pruned"] == X.aux_ngrams.pruned


def test_every_space_byte_and_long_query():
    """lead cuts at each isspace byte; a query of 80 tokens, where pool 0's aux query (its first 64) differs from pool 2's"""
    docs = []
    for sp in S.SPACE:
        c = bytes([sp])
        docs += [c.join(b"w%d" % i for i in range(70)), c + c.join(b"x%d" % (i % 9) for i in range(66)) + c, b"a" + c * 3 + b"b"]
    long_q = b" ".join(b"w%d" % (i % 70) for i in range(80)) + b" x3"
    queries = [long_q, b"w1 w65", b"w63 w64", b"x8", b"a b", b""]
    for variant in (B.SAB, B.ATIRE):
        X = S.Index(B.Config(variant=variant), docs, 64)
        D = _index(variant, docs, 64)
        _check_all(D, X, queries, docs, K=R.Concepts(docs, docs, CCFG), C=D.mine_concepts(docs, **CCFG.kw()))
        assert not np.array_equal(S.score(X, 0, long_q), S.score(X, 2, long_q))


def test_keyphrase_gate_and_route_replay(monkeypatch):
    """queries on both sides of the 0.30 gate and stopword-only ones; the route certified, then replayed on demand"""
    docs, voc = S.gen_lead_corpus(81, 3000)
    queries = S.gen_lead_queries(82, voc, 60) + [b"the and of", b"THE a an", b"it is", b"zz", b"a1 b2"]
    X = S.Index(B.Config(), docs, 64)
    gated = [S.keyphrase_entropy(X.score(q)) >= np.float32(0.30) and bool(S.keyphrases(q)) for q in queries]
    assert any(gated) and not all(gated)
    D = _index(B.SAB, docs, 64)
    _check_all(D, X, queries, docs)
    got = D.score_strategy(queries, Y.BM25_STRATEGY_KEYPHRASE)
    st = D.strategy_stats()
    assert st["replayed"] == 0 and st["queries"] == (0, len(queries), 0) and st["keyphrase_boosted"] == sum(gated)
    base = D.score_strategy(queries, Y.BM25_STRATEGY_ROUTED, k=10)
    assert D.strategy_stats()["replayed"] == 0
    monkeypatch.setenv("YAMS_B200_BM25_ROUTE_MARGIN", "1")
    wide = D.score_strategy(queries, Y.BM25_STRATEGY_ROUTED, k=10)
    positive = sum(bool((X.score(q) > 0).any()) for q in queries)
    assert positive > 0 and D.strategy_stats()["replayed"] == positive
    for key in ("scores", "docs", "topk_scores", "counts", "chosen"):
        assert wide[key].tobytes() == base[key].tobytes(), key
    monkeypatch.delenv("YAMS_B200_BM25_ROUTE_MARGIN")
    D.score_strategy(queries, Y.BM25_STRATEGY_ROUTED)
    assert D.strategy_stats()["replayed"] == 0
    assert got["scores"].tobytes() != D.score(queries)["scores"].tobytes()


def test_budget_split():
    """4 101 routed queries over 33 000 documents: the score and match rows (8 bytes a document) split them at 4 067"""
    docs, voc = B.gen_corpus(83, 33_000, mean_words=8)
    X = S.Index(B.Config(), docs, 64)
    D = _index(B.SAB, docs, 64)
    queries = B.gen_queries(84, voc, 4101)
    C = D.mine_concepts(docs, **CCFG.kw())
    K = R.Concepts(docs, docs, CCFG)
    got = D.score_strategy(queries, Y.BM25_STRATEGY_ROUTED, k=5, concepts=C)
    for i in list(range(0, 4101, 199)) + [4066, 4067, 4100]:
        _check(got, i, S.score(X, 3, queries[i], K, 0.5), 5, S.route(X.score(queries[i])))


@pytest.mark.skipif(not S.have_ref(), reason="oracle/_ref/libref_strategy.so not built")
def test_200k_documents_against_reference():
    docs, voc = B.gen_corpus(85, 200_000, mean_words=6)
    queries = B.gen_queries(86, voc, 12) + [b"the", docs[5][:400]]
    ref = S.RefStrategy(B.Config(), docs, 64, CCFG)
    D = _index(B.SAB, docs, 64)
    C = D.mine_concepts(docs, **CCFG.kw())
    for pool in POOLS:
        got = D.score_strategy(queries, pool, k=10, concepts=C)
        for i, q in enumerate(queries):
            want, chosen = ref.score(pool, q, 0.5, chosen=True)
            assert got["scores"][i].tobytes() == want.tobytes() and got["chosen"][i] == chosen, (pool, i)


def test_all_leads_empty_and_no_lead_field():
    docs, voc = S.gen_lead_corpus(77, 300)
    queries = S.gen_lead_queries(78, voc, 12)
    empty = [b"", b" ", b"\t\n", b"\v\f\r "] * 5
    for variant in (B.SAB, B.ATIRE):
        D = _index(variant, empty, 64)
        assert D.aux_stats()["n_docs"] == 0 and not D.doc_lengths(2).any()
        _check_all(D, S.Index(B.Config(variant=variant), empty, 64), [b"a", b""], empty)
        # without the lead field: BM25F is wb * body, and plain scores are unchanged
        P = _index(variant, docs, 0)
        X0 = S.Index(B.Config(variant=variant), docs, 0)
        _check_all(P, X0, queries, docs)
        L = _index(variant, docs, 64)
        assert L.score(queries)["scores"].tobytes() == P.score(queries)["scores"].tobytes()
        assert L.stats() == P.stats()


@pytest.mark.skipif(not S.have_ref(), reason="oracle/_ref/libref_strategy.so not built")
def test_accessors_against_reference():
    docs, voc = S.gen_lead_corpus(91, 900)
    queries = S.gen_lead_queries(92, voc, 8)
    for variant in (B.SAB, B.ATIRE):
        cfg = B.Config(variant=variant)
        ref = S.RefStrategy(cfg, docs, 64, CCFG)
        D = _index(variant, docs, 64)
        X = S.Index(cfg, docs, 64)
        for f in range(4):
            assert np.array_equal(D.doc_lengths(f), ref.doc_lengths(f)), f
            for h in list(X.field(f).postings)[:40] + [12345]:
                a, b = D.postings(f, h), ref.postings(f, h)
                assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2] == b[2] and a[3] == b[3], (f, h)
        got = D.score_strategy(queries, 2)
        for i, q in enumerate(queries):
            assert got["scores"][i].tobytes() == ref.score(2, q).tobytes()


def test_atire_view_aux_field():
    docs, voc = S.gen_lead_corpus(93, 1500)
    queries = S.gen_lead_queries(94, voc, 12)
    P = _index(B.SAB, docs, 64)
    V = P.atire_view()
    A = _index(B.ATIRE, docs, 64)
    XA = S.Index(B.Config(variant=B.ATIRE), docs, 64)
    assert V.aux_stats() == A.aux_stats()
    for f in (2, 3):
        assert np.array_equal(V.doc_lengths(f), A.doc_lengths(f))
    for h in list(XA.aux_words.postings)[:40]:
        a, b = V.postings(2, h), A.postings(2, h)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2] == b[2] and a[3] == b[3]
    _check_all(V, XA, queries, docs)
    del P   # the view keeps the shared fields alive
    _check_all(V, XA, queries[:3], docs)


def test_many_queries_and_threads():
    docs, voc = S.gen_lead_corpus(95, 2000)
    X = S.Index(B.Config(), docs, 64)
    D = _index(B.SAB, docs, 64)
    queries = S.gen_lead_queries(96, voc, 4101)
    got = D.score_strategy(queries, Y.BM25_STRATEGY_BM25, k=5)
    for i in range(0, 4101, 97):
        _check(got, i, S.score(X, 0, queries[i]), 5, 0)
    assert got["scores"][4100].tobytes() == S.score(X, 0, queries[4100]).tobytes()
    got = D.score_strategy(queries, Y.BM25_STRATEGY_KEYPHRASE, k=5)
    for i in range(0, 4101, 131):
        _check(got, i, S.score(X, 1, queries[i]), 5, 1)
    want = {p: D.score_strategy(queries[:200], p, k=5) for p in POOLS}
    errs = []

    def run(p):
        try:
            for _ in range(3):
                g = D.score_strategy(queries[:200], p, k=5)
                assert g["scores"].tobytes() == want[p]["scores"].tobytes() and g["docs"].tobytes() == want[p]["docs"].tobytes()
        except Exception as e:   # reported below
            errs.append(e)

    ts = [threading.Thread(target=run, args=(p,)) for p in POOLS]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs


def test_argument_errors():
    D = _index(B.SAB, [b"a b c", b"b c d"], 64)
    for bad in (4, 99):
        with pytest.raises(Y.YamsB200Error):
            D.score_strategy([b"a"], bad)
    with pytest.raises(Y.YamsB200Error):
        D.score_strategy([b"a"], 0, k=4097)
    with pytest.raises(Y.YamsB200Error):
        D.postings(4, 1)
    with pytest.raises(Y.YamsB200Error):
        D.doc_lengths(4)
    assert D.score_strategy([], 0)["scores"].shape == (0, 2)
    E = _index(B.SAB, [], 64)
    for pool in POOLS:
        assert E.score_strategy([b"a"], pool, k=3)["counts"].tolist() == [0]


def test_cpp_host_adapter(tmp_path):
    """B200Bm25Index with the lead field and score_strategy (the stand-ins for the backend's primary and its strategies)"""
    import subprocess
    exe = str(tmp_path / "test_bm25_strategy")
    subprocess.check_call(["/usr/bin/g++", "-std=c++20", "-O1", os.path.join(ROOT, "tests", "host_cpp", "test_bm25_strategy.cpp"),
                           "-o", exe, "-L" + os.path.join(ROOT, "yams_b200"), "-lyams_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "yams_b200")])
    docs, voc = S.gen_lead_corpus(97, 400)
    queries = S.gen_lead_queries(98, voc, 10)

    def texts(ts):
        return np.array([len(ts)], np.uint64).tobytes() + b"".join(np.array([len(t)], np.uint64).tobytes() + t for t in ts)

    path = tmp_path / "in.bin"
    path.write_bytes(texts(docs) + texts(queries))
    out = subprocess.run([exe, str(path)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.endswith("ALL OK\n"), out.stdout[-500:] + out.stderr
    lines = out.stdout.split("\n")
    assert int(lines[0]) == len(docs)
    X = S.Index(B.Config(), docs, 64)
    K = R.Concepts(docs, docs, R.CCfg(min_ttf=2))

    def row(i):
        return [int(v) for v in lines[i].split()]

    for i, q in enumerate(queries):
        assert row(1 + 5 * i) == S.score(X, 0, q).view(np.uint32).tolist(), q
        assert row(2 + 5 * i) == S.score(X, 2, q).view(np.uint32).tolist(), q
        assert row(3 + 5 * i) == S.score(X, 2, q, K, 0.5).view(np.uint32).tolist(), q
        assert row(4 + 5 * i) == S.score(X, 1, q).view(np.uint32).tolist(), q
        assert row(5 + 5 * i) == [S.route(X.score(q))] + S.score(X, 3, q, K, 0.5).view(np.uint32).tolist(), q
