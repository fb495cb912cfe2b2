"""Reciprocal-rank fusion of BM25 variants on the device (yams_b200_bm25_score_rrf) and the Atire view of an index
(yams_b200_bm25_atire_view), bit for bit: against the stored answers of simeon's own score_bm25_variants_rrf
(tests/golden/ref_rrf.json) and the restatement (tests/rrf_restated.py), with separately built Atire indexes and with views;
the view against a separately built Atire index across configurations, prune ratios and hostile texts (scores, blended scores,
top-k, stats, postings, document lengths, concepts mined against it), its lifetime and concurrency with its parent; batches
across the query cap and the memory budget, score-tile edges, the 4096-wide top-k with fused ties, 200 000 documents, two
threads fusing the same indexes in opposite orders, the argument errors, and the C++ adapter."""
import hashlib
import json
import os
import threading

import numpy as np
import pytest

import yams_b200 as Y
from tests import bm25_restated as B
from tests import concepts_restated as R
from tests import rrf_restated as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STORED = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_rrf.json")))
GOLDEN = STORED["cases"]
CCFG = R.CCfg(**STORED["concept_config"])


def _digest(a):
    a = np.ascontiguousarray(a)
    return a.tobytes().hex() if a.size <= 64 and a.dtype == np.float32 else "sha256:" + hashlib.sha256(a.tobytes()).hexdigest()


def _bits(x):
    return int(np.array([x], np.float32).view(np.uint32)[0])


def _index(cfg: B.Config, docs):
    return Y.Bm25Index(docs, k1=cfg.k1, b=cfg.b, delta=cfg.delta, subword_gamma=cfg.gamma, variant=cfg.variant, ngram_min=cfg.ngram_min,
                       ngram_max=cfg.ngram_max, ngram_df_prune_ratio=cfg.prune_ratio, hash_seed=cfg.hash_seed)


def _devices(cfgs, docs, views=False):
    """device indexes of the configs; with views, an Atire config after a SubwordAwareBackoff one of the same k1, b and seed is
    that index's Atire view (the backend's pair), not a second build"""
    out = []
    for c in cfgs:
        sab = next((d for d, dc in zip(out, cfgs) if dc.variant == B.SAB and (dc.k1, dc.b, dc.hash_seed) == (c.k1, c.b, c.hash_seed)), None)
        out.append(sab.atire_view() if views and c.variant == B.ATIRE and sab is not None else _index(c, docs))
    return out


def _check_rows(got, i, want, k):
    assert got["scores"][i].tobytes() == want.tobytes(), i
    wd, ws = B.topk(want, k)
    c = int(got["counts"][i])
    assert c == len(wd) and np.array_equal(got["docs"][i, :c], wd) and got["topk_scores"][i, :c].tobytes() == ws.tobytes(), i
    assert np.all(got["docs"][i, c:] == 0xFFFFFFFF) and np.all(got["topk_scores"][i, c:] == 0)


def _check_rrf(D, X, queries, k_rrf=60.0, C=None, K=None, weight=0.5, k=10):
    got = Y.bm25_score_rrf(D, queries, k=k, k_rrf=k_rrf, concepts=C, weight=weight)
    for i, q in enumerate(queries):
        _check_rows(got, i, F.score(X, q, k_rrf, K, weight), k)
    return got


@pytest.mark.parametrize("views", [False, True])
@pytest.mark.parametrize("case", GOLDEN, ids=[c["name"] for c in GOLDEN])
def test_stored_answers(case, views):
    docs, queries, cfgs = F.case_inputs(case)
    D = _devices(cfgs, docs, views)
    C = (D[0] if D else _index(F.SAB, docs)).mine_concepts(docs, **CCFG.kw())
    for s in case["scores"]:
        w = s["weight"]
        got = Y.bm25_score_rrf(D, queries, k=10, k_rrf=s["k_rrf"], concepts=C if w is not None else None, weight=w or 0.0)
        if not D:   # no variant: no document count, nothing ranked
            assert got["scores"].shape == (len(queries), 0) and not got["counts"].any() and np.all(got["docs"] == 0xFFFFFFFF)
            continue
        for i, d in enumerate(s["digests"]):
            assert _digest(got["scores"][i]) == d, (s["k_rrf"], w, i)
            wd, ws = B.topk(got["scores"][i], 10)
            assert int(got["counts"][i]) == len(wd) and np.array_equal(got["docs"][i, :len(wd)], wd)


@pytest.mark.parametrize("n,variants,k_rrf,weight", F.GRID)
def test_grid(n, variants, k_rrf, weight):
    docs, queries, cfgs = F.grid_case(n, variants)
    X = [B.Index(c, docs) for c in cfgs]
    K = R.Concepts(docs, docs, CCFG) if weight is not None else None
    for views in (False, True):
        D = _devices(cfgs, docs, views)
        C = D[0].mine_concepts(docs, **CCFG.kw()) if weight is not None else None
        _check_rrf(D, X, queries, k_rrf, C, K, weight or 0.0, k=7)


# ---- the Atire view against a separately built Atire index ----
def _check_view(pcfg: B.Config, docs, queries, words=(), k=7):
    P = _index(pcfg, docs)
    V = P.atire_view()
    acfg = B.Config(variant=B.ATIRE, k1=pcfg.k1, b=pcfg.b, hash_seed=pcfg.hash_seed)
    A = _index(acfg, docs)
    XA = B.Index(acfg, docs)
    gv, ga = V.score(queries, k=k), A.score(queries, k=k)
    for i, q in enumerate(queries):
        _check_rows(gv, i, XA.score(q), k)
        _check_rows(ga, i, XA.score(q), k)
    sv, sa = V.stats(), A.stats()
    assert {**sv, "avg_dl": _bits(sv["avg_dl"]), "ngram_avg_dl": _bits(sv["ngram_avg_dl"])} == \
        {**sa, "avg_dl": _bits(sa["avg_dl"]), "ngram_avg_dl": _bits(sa["ngram_avg_dl"])}
    assert sv["ngram_avg_dl"] == 0 and sv["terms"][1] == sv["postings"][1] == sv["pruned"] == 0
    for fld in (0, 1):
        assert np.array_equal(V.doc_lengths(fld), A.doc_lengths(fld))
    assert not V.doc_lengths(1).any()
    for w in words:
        h = XA.h(w.lower())
        a, b = V.postings(0, h), A.postings(0, h)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and _bits(a[2]) == _bits(b[2]) and a[3] == b[3], w
        for g in XA.gram_hashes(w.lower())[:3] + [h]:
            d, t, idf, ttf = V.postings(1, g)
            assert len(d) == len(t) == 0 and idf == 0 and ttf == 0
    if len(docs) >= 2:
        CV, CA = V.mine_concepts(docs, min_ttf=2), A.mine_concepts(docs, min_ttf=2)
        assert np.array_equal(CV.hashes(), CA.hashes()) and CV.stats() == CA.stats()
        bv, ba = V.score(queries, k=k, concepts=CV), A.score(queries, k=k, concepts=CA)
        assert bv["scores"].tobytes() == ba["scores"].tobytes() and bv["docs"].tobytes() == ba["docs"].tobytes()
        assert bv["counts"].tobytes() == ba["counts"].tobytes()
    return P, V, A


VIEW_GRID = [(v, n, g, ngr, r) for v in (B.SAB, B.ATIRE) for n in (0, 1, 3, 1000)
             for g, ngr, r in [(5.0, (3, 4), 0.5), (0.0, (1, 1), 0.5), (1e-3, (2, 8), 0.0), (1e6, (3, 4), 1e-4)]]


@pytest.mark.parametrize("variant,n,gamma,ngr,ratio", VIEW_GRID)
def test_view_equals_an_atire_build(variant, n, gamma, ngr, ratio):
    docs, voc = B.gen_corpus(900 + n, n, 30, 1500)
    queries = B.gen_queries(n + 1, voc, 48) + [b"", b"!!", voc[0] + b" " + voc[0] + b" " + voc[0].upper()]
    cfg = B.Config(variant=variant, ngram_min=ngr[0], ngram_max=ngr[1], gamma=gamma, prune_ratio=ratio, k1=1.2 + 0.1 * (n % 3),
                   b=0.75 - 0.05 * (n % 2))
    _check_view(cfg, docs, queries, words=voc[:6])


def test_view_hostile_texts():
    rng = np.random.default_rng(5)
    docs, voc = B.gen_corpus(77, 2000, 20, 800)
    big_word = bytes(rng.integers(97, 123, 100_000).astype(np.uint8))
    docs += [b"", b"\x80\x81\xfe\xff", b"...,,, --", b"A a B b Ab aB x", big_word, b"the " * 3000 + b"The THE", b"\x00\x00word\x00"]
    queries = B.gen_queries(3, voc, 300) + [b"", b"\xff\xfe", b"the the THE", b"zqxjvwkp", big_word[:5000], b"word"]
    _check_view(B.Config(), docs, queries, words=[b"the", b"a", big_word[:10], b"word"])


def test_view_lifetimes_and_nesting():
    docs, voc = B.gen_corpus(12, 800, 20, 600)
    queries = B.gen_queries(13, voc, 32)
    X = B.Index(F.ATIRE, docs)
    want = [X.score(q) for q in queries]
    P = _index(F.SAB, docs)
    V1, V2 = P.atire_view(), P.atire_view()
    V1.close()                                  # a view before its parent
    assert P.score(queries[:1])["scores"][0].tobytes() == B.Index(F.SAB, docs).score(queries[0]).tobytes()
    P.close()                                   # the parent before a view
    VV = V2.atire_view()                        # a view of a view (of an Atire index) is the index
    for D in (V2, VV):
        got = D.score(queries)["scores"]
        assert all(got[i].tobytes() == w.tobytes() for i, w in enumerate(want))
    V2.close()
    assert VV.score(queries)["scores"].tobytes() == np.stack(want).tobytes()
    A = _index(F.ATIRE, docs)
    assert A.atire_view().score(queries)["scores"].tobytes() == A.score(queries)["scores"].tobytes()


def test_view_scored_concurrently_with_parent():
    docs, voc = B.gen_corpus(14, 5000, 20, 1500)
    queries = B.gen_queries(15, voc, 200)
    P = _index(F.SAB, docs)
    V = P.atire_view()
    want = {id(P): P.score(queries, k=10), id(V): V.score(queries, k=10)}
    errors = []

    def run(D):
        try:
            for _ in range(8):
                got = D.score(queries, k=10)
                assert all(got[key].tobytes() == want[id(D)][key].tobytes() for key in got)
        except Exception as e:   # surfaced below
            errors.append(e)

    ts = [threading.Thread(target=run, args=(D,)) for D in (P, V, P, V)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors


# ---- batching ----
def _rrf_per_batch(n, nv, nq):
    return max(1, min((1 << 30) // (n * (20 * nv + 4)), nq, 4096))


def test_batches_across_the_query_cap():
    """4 101 queries in one call: batches of 4 096 + 5"""
    docs, voc, ph = R.gen_concept_corpus(51, 3000, 20, 1000, 30, 4)
    queries = R.gen_concept_queries(52, voc, ph, 4101)
    assert _rrf_per_batch(len(docs), 2, len(queries)) == 4096
    X = [B.Index(F.SAB, docs), B.Index(F.ATIRE, docs)]
    D = _devices([F.SAB, F.ATIRE], docs, views=True)
    C, K = D[0].mine_concepts(docs, **CCFG.kw()), R.Concepts(docs, docs, CCFG)
    _check_rrf(D, X, queries, C=C, K=K, k=5)
    topk_only = Y.bm25_score_rrf(D, queries, k=5, full=False, concepts=C)
    full = Y.bm25_score_rrf(D, queries, concepts=C)
    want = Y.bm25_score_rrf(D, queries, k=5, concepts=C)
    assert all(topk_only[key].tobytes() == want[key].tobytes() for key in ("docs", "topk_scores", "counts"))
    assert full["scores"].tobytes() == want["scores"].tobytes()


def test_batches_split_by_the_memory_budget():
    """1 000 queries over 270 000 documents and two variants: 1 GiB holds the rows, keys and sort buffers of 90 queries, so the
    call runs 12 batches; every row and top-k equals the same query fused alone"""
    docs, voc = B.gen_corpus(2025, 270_000, 8, 20_000)
    queries = B.gen_queries(2026, voc, 1000)
    per = _rrf_per_batch(len(docs), 2, len(queries))
    assert per < len(queries) and len(queries) % per
    D = _devices([F.SAB, F.ATIRE], docs, views=True)
    got = Y.bm25_score_rrf(D, queries, k=10)
    for i, q in enumerate(queries):
        one = Y.bm25_score_rrf(D, [q], k=10)
        assert got["scores"][i].tobytes() == one["scores"][0].tobytes(), i
        assert got["docs"][i].tobytes() == one["docs"][0].tobytes() and got["counts"][i] == one["counts"][0], i
    assert any(int(c) > 0 for c in got["counts"])


@pytest.mark.parametrize("n", [4095, 4096, 4097])
def test_score_tile_edges(n):
    docs, voc, ph = R.gen_concept_corpus(60 + n, n, 15, 800, 30, 4)
    queries = R.gen_concept_queries(61, voc, ph, 40) + F.ngram_queries(voc, 8, n)
    cfgs = [F.SAB, F.ATIRE, F.OTHER]
    X = [B.Index(c, docs) for c in cfgs]
    D = _devices(cfgs, docs, views=True)
    _check_rrf(D, X, queries, C=D[0].mine_concepts(docs, **CCFG.kw()), K=R.Concepts(docs, docs, CCFG), k=9)


def test_topk_4096_with_fused_ties():
    """10 000 documents, many identical.  SubwordAwareBackoff and an Atire index with b = 0 order the document kinds differently,
    and at k_rrf = 1e6 two documents of equal rank sums fuse to the same float: a fused tie crosses rank 4 096"""
    docs = [b"red fox jumps", b"red fox", b"blue whale", b"red fox red fox", b"fox red", b"", b"red fox jumps high"] * 1430
    docs = docs[:10_000]
    queries = [b"red fox", b"red fox jumps", b"blue whale red fox", b"fox", b"foxes"]
    X = [B.Index(F.SAB, docs), B.Index(F.ATIRE, docs)]
    D = _devices([F.SAB, F.ATIRE], docs, views=True)
    _check_rrf(D, X, queries, k=4096)
    _check_rrf(D, X, queries, k=4096, C=D[0].mine_concepts(docs, min_ttf=1, pmi_floor=-1e30),
               K=R.Concepts(docs, docs, R.CCfg(min_ttf=1, pmi_floor=-1e30)), weight=1.0)
    flat = B.Config(variant=B.ATIRE, b=0.0)
    got = _check_rrf([D[0], _index(flat, docs)], [X[0], B.Index(flat, docs)], queries, k_rrf=1e6, k=4096)
    s, cut = got["scores"][0], got["topk_scores"][0, 4095]
    assert got["counts"][0] == 4096 and np.count_nonzero(s == cut) > np.count_nonzero(got["topk_scores"][0] == cut)


def test_200k_documents():
    docs, voc, ph = R.gen_concept_corpus(2024, 200_000, 8, 20_000, 400, 20)
    queries = R.gen_concept_queries(8, voc, ph, 24)
    X = [B.Index(F.SAB, docs), B.Index(F.ATIRE, docs)]
    D = _devices([F.SAB, F.ATIRE], docs, views=True)
    _check_rrf(D, X, queries, C=D[0].mine_concepts(docs), K=R.Concepts(docs, docs), k=100)


# ---- concurrency and arguments ----
def test_two_threads_in_opposite_orders():
    """RRF over {A, B} and {B, A} on two threads at once, with plain scores in between: no deadlock, the serial answers"""
    docs, voc = B.gen_corpus(16, 20_000, 15, 3000)
    queries = B.gen_queries(17, voc, 64)
    A = _index(F.SAB, docs)
    Bv = A.atire_view()
    Bb = _index(F.OTHER, docs)
    pairs = [[A, Bb], [Bb, A], [A, Bv], [Bv, A]]
    want = [Y.bm25_score_rrf(p, queries, k=10) for p in pairs]
    plain = {id(D): D.score(queries, k=10) for D in (A, Bv, Bb)}
    errors = []

    def run(j):
        try:
            for it in range(6):
                got = Y.bm25_score_rrf(pairs[j], queries, k=10)
                assert all(got[key].tobytes() == want[j][key].tobytes() for key in got)
                D = pairs[j][it % 2]
                got = D.score(queries, k=10)
                assert all(got[key].tobytes() == plain[id(D)][key].tobytes() for key in got)
        except Exception as e:   # surfaced below
            errors.append(e)

    ts = [threading.Thread(target=run, args=(j,)) for j in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=300)
    assert not any(t.is_alive() for t in ts), "deadlock"
    assert not errors, errors


def test_arguments():
    docs = [b"a b", b"a b c", b"c d"]
    A, Bx = _index(F.SAB, docs), _index(F.ATIRE, docs)
    other = _index(F.SAB, docs + [b"e"])

    def status(fn):
        with pytest.raises(Y.YamsB200Error) as e:
            fn()
        return e.value.status

    assert status(lambda: Y.bm25_score_rrf([A, other], [b"a"])) == 1
    for bad in (float("nan"), float("inf"), -1.0):
        assert status(lambda: Y.bm25_score_rrf([A, Bx], [b"a"], k_rrf=bad)) == 1
    assert status(lambda: Y.bm25_score_rrf([A, Bx], [b"a"], k=4097)) == 1
    hs = (Y._lib.C.c_void_p * 2)(A._h, None)
    assert Y.lib().yams_b200_bm25_score_rrf(hs, 2, 60.0, None, 0.5, None, None, 0, None, 0, None, None, None) == 1
    assert Y.lib().yams_b200_bm25_atire_view(None, Y._lib.C.byref(Y._lib.C.c_void_p())) == 1
    # concepts of another document count: no blend, as score_blended
    C = other.mine_concepts(docs + [b"e"], min_ttf=1, pmi_floor=-1e30)
    assert C.stats()["size"] > 0
    assert Y.bm25_score_rrf([A, Bx], [b"a b"], concepts=C)["scores"].tobytes() == Y.bm25_score_rrf([A, Bx], [b"a b"])["scores"].tobytes()
    # the same index twice: each rank counts twice
    got = Y.bm25_score_rrf([A, A], [b"a b"])["scores"][0]
    assert got.tobytes() == F.score([B.Index(F.SAB, docs)] * 2, b"a b").tobytes() and got.max() > 0
    assert Y.bm25_score_rrf([A, Bx], [])["scores"].shape == (0, 3)


def test_different_devices():
    """indexes on different devices are refused with YAMS_ERR_UNSUPPORTED; one plugin context serves one device, so the case
    cannot be built here with fewer than two GPUs"""
    if Y.device_count() < 2:
        pytest.skip("one GPU: indexes on different devices need two")
    pytest.skip("the plugin binds one device per process: a second device needs a second plugin context")


def test_cpp_host_adapter(tmp_path):
    """B200Bm25Index::atire_view and score_bm25_variants_rrf (the stand-ins for the backend's Atire index and simeon's fusion)"""
    import subprocess
    exe = str(tmp_path / "test_bm25_rrf")
    subprocess.check_call(["/usr/bin/g++", "-std=c++20", "-O1", os.path.join(ROOT, "tests", "host_cpp", "test_bm25_rrf.cpp"),
                           "-o", exe, "-L" + os.path.join(ROOT, "yams_b200"), "-lyams_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "yams_b200")])
    docs, voc, ph = R.gen_concept_corpus(71, 300, 20, 400, 20, 3)
    queries = R.gen_concept_queries(72, voc, ph, 12) + F.ngram_queries(voc, 4, 73) + [b""]

    def texts(ts):
        return np.array([len(ts)], np.uint64).tobytes() + b"".join(np.array([len(t)], np.uint64).tobytes() + t for t in ts)

    path = tmp_path / "in.bin"
    path.write_bytes(texts(docs) + texts(queries))
    out = subprocess.run([exe, str(path)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.endswith("ALL OK\n"), out.stdout[-500:] + out.stderr
    lines = out.stdout.split("\n")
    X = [B.Index(F.SAB, docs), B.Index(F.ATIRE, docs)]
    assert lines[0].split() == [str(len(docs)), str(_bits(X[1].words.avg))]
    K = R.Concepts(docs, docs, R.CCfg(min_ttf=2))

    def row(i):
        return [int(v) for v in lines[i].split()]

    for i, q in enumerate(queries):
        assert row(1 + 3 * i) == X[1].score(q).view(np.uint32).tolist(), q
        assert row(2 + 3 * i) == F.score(X, q).view(np.uint32).tolist(), q
        assert row(3 + 3 * i) == F.score(X, q, concepts=K, weight=0.5).view(np.uint32).tolist(), q
    assert row(1 + 3 * len(queries)) == X[1].score(queries[0]).view(np.uint32).tolist()
