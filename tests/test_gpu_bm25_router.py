"""The query router on the device (yams_b200_bm25_score_routed), bit for bit: against the stored answers of simeon's own
QueryRouter and the backend's routed dispatch (tests/golden/ref_router.json) and the restatement (tests/router_restated.py) --
every feature, the recipe, full rows, the top-k and the projected candidate pools -- for both primaries, with and without
concepts, under default and forcing router configs; pools with unindexed ids, empty pools and pools longer than n; n from 1 to
200 000; 4 101 queries split by the memory budget with mixed recipes in one batch; two threads; the argument errors; the C++
adapter."""
import ctypes as C
import hashlib
import json
import os
import subprocess
import threading

import numpy as np
import pytest

import yams_b200 as Y
from tests import bm25_restated as B
from tests import concepts_restated as R
from tests import router_restated as T

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STORED = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_router.json")))
CCFG = R.CCfg(**STORED["concept_config"])
CASES = {c[0]: c for c in T.CASES}


def _digest(a):
    a = np.ascontiguousarray(a)
    return a.tobytes().hex() if a.size <= 64 and a.dtype == np.float32 else "sha256:" + hashlib.sha256(a.tobytes()).hexdigest()


def _feature_bits(row):
    return [int(row[k]) if k == "n_terms" else int(np.float32(row[k]).view(np.uint32)) for k in T.FEATURES]


def _restated_bits(f):
    return [int(f[k]) if k == "n_terms" else int(np.float32(f[k]).view(np.uint32)) for k in T.FEATURES]


def _router(rcfg: T.RCfg):
    return Y.RouterConfig.default(**rcfg.kw())


def _check(got, i, r, f, row, k, cands=None):
    assert int(got["recipe"][i]) == r, i
    assert _feature_bits(got["features"][i]) == _restated_bits(f), i
    if "scores" in got:
        assert got["scores"][i].tobytes() == row.tobytes(), i
    if k:
        wd, ws = B.topk(row, k)
        c = int(got["counts"][i])
        assert c == len(wd) and np.array_equal(got["docs"][i, :c], wd) and got["topk_scores"][i, :c].tobytes() == ws.tobytes(), i
        assert np.all(got["docs"][i, c:] == 0xFFFFFFFF) and np.all(got["topk_scores"][i, c:] == 0)
    if cands is not None:
        assert got["candidates"][i].tobytes() == T.project(row, cands).tobytes(), i


def _check_all(D, X, A, queries, rcfg=T.RCfg(), C=None, K=None, weight=0.5, k=7, pool_seed=1):
    n = X.n
    pools = [T.pool(pool_seed, n, i) for i in range(len(queries))]
    got = D.score_routed(queries, k=k, concepts=C, weight=weight, router=_router(rcfg), candidates=pools)
    only = D.score_routed(queries, full=False, concepts=C, weight=weight, router=_router(rcfg), candidates=pools)
    for i, q in enumerate(queries):
        r, f, row = T.score(X, A, q, rcfg, K, weight)
        _check(got, i, r, f, row, k, pools[i])
        _check(only, i, r, f, row, 0, pools[i])
    return got


@pytest.mark.parametrize("stored", STORED["cases"], ids=[c["name"] for c in STORED["cases"]])
def test_stored_answers(stored):
    docs, queries, cfg, rcfg = T.case_inputs(*CASES[stored["name"]])
    D = Y.Bm25Index(docs, variant=cfg.variant)
    C = D.mine_concepts(docs, **CCFG.kw())
    pools = [T.pool(stored["seed"], stored["n"], i) for i in range(len(queries))]
    for w, answers in stored["answers"].items():
        got = D.score_routed(queries, k=10, concepts=C if w != "None" else None, weight=0.5, router=_router(rcfg), candidates=pools)
        for i, a in enumerate(answers):
            assert int(got["recipe"][i]) == a["recipe"] and _feature_bits(got["features"][i]) == a["features"], (w, i)
            assert _digest(got["scores"][i]) == a["scores"] and _digest(got["candidates"][i]) == a["pool"], (w, i)
            wd, _ = B.topk(got["scores"][i], 10)
            assert int(got["counts"][i]) == len(wd) and np.array_equal(got["docs"][i, :len(wd)], wd)


RCFGS = [T.RCfg(), T.RCfg(high_idf_threshold=-1.0, atire_max_clarity=float("inf")),
         T.RCfg(high_idf_threshold=1e30, cascade_min_terms=0, cascade_max_idf=1e30),
         T.RCfg(oov_threshold=0.5, atire_min_terms=2, atire_min_idf_floor=1.5, atire_min_scq=10.0, atire_max_pool_jaccard=0.5)]
GRID = [(v, n, j) for v in (B.SAB, B.ATIRE) for n, j in ((1, 0), (2, 1), (37, 2), (600, 0), (4096, 3), (4097, 1))]


@pytest.mark.parametrize("variant,n,j", GRID)
def test_grid(variant, n, j):
    docs, voc, ph, burst = T.gen_router_corpus(60 + n, n)
    queries = T.gen_router_queries(61 + n, voc, ph, burst, 40) + T.edge_queries(voc, burst)
    cfg = B.Config(variant=variant)
    X = B.Index(cfg, docs)
    A = B.Index(T.atire_of(cfg), docs) if T.atire_of(cfg) else None
    D = Y.Bm25Index(docs, variant=variant)
    K = R.Concepts(docs, docs, CCFG)
    C = D.mine_concepts(docs, **CCFG.kw())
    _check_all(D, X, A, queries, RCFGS[j], pool_seed=n)
    _check_all(D, X, A, queries, RCFGS[j], C, K, 0.5, pool_seed=n + 1)


def test_atire_rows_equal_the_view():
    """a row routed to Bm25Atire is the Atire view's row; SubwordAwareBackoff and Cascade rows are the primary's"""
    docs, voc, ph, burst = T.gen_router_corpus(70, 800)
    queries = T.gen_router_queries(71, voc, ph, burst, 200)
    D = Y.Bm25Index(docs)
    V = D.atire_view()
    got = D.score_routed(queries, router=Y.RouterConfig.default(atire_max_clarity=float("inf")))
    plain, atire = D.score(queries)["scores"], V.score(queries)["scores"]
    assert set(got["recipe"].tolist()) == {0, 1, 2}
    for i, r in enumerate(got["recipe"]):
        assert got["scores"][i].tobytes() == (atire if r == Y.BM25_RECIPE_ATIRE else plain)[i].tobytes(), i


def test_empty_index_and_pools():
    E = Y.Bm25Index([])
    got = E.score_routed([b"a b", b""], k=3, candidates=[[Y.BM25_NOT_INDEXED] * 5, []])
    assert got["scores"].shape == (2, 0) and got["counts"].tolist() == [0, 0]
    assert got["candidates"][0].tolist() == [0.0] * 5 and len(got["candidates"][1]) == 0
    assert got["features"]["oov_rate"][0] == 1.0 and got["recipe"].tolist() == [1, 1]
    D = Y.Bm25Index([b"alpha beta", b"beta gamma"])
    got = D.score_routed([b"beta"] * 3, full=False, candidates=[[], [1, 0, 1, Y.BM25_NOT_INDEXED, 1], []])
    s = D.score([b"beta"])["scores"][0]
    assert got["candidates"][1].tolist() == [s[1], s[0], s[1], 0.0, s[1]] and len(got["candidates"][0]) == 0


@pytest.mark.skipif(not T.have_ref(), reason="oracle/_ref/libref_router.so not built")
def test_200k_documents_against_reference():
    docs, voc, ph, burst = T.gen_router_corpus(80, 200_000)
    queries = T.gen_router_queries(81, voc, ph, burst, 24) + T.edge_queries(voc, burst)
    cfg = B.Config()
    RX, RA = T.RefIndex(cfg, docs), T.RefIndex(T.atire_of(cfg), docs)
    RK = T.RefConcepts(RX, docs, CCFG)
    D = Y.Bm25Index(docs)
    C = D.mine_concepts(docs, **CCFG.kw())
    pools = [T.pool(82, 200_000, i) for i in range(len(queries))]
    got = D.score_routed(queries, k=10, concepts=C, candidates=pools)
    recipes = set()
    for i, q in enumerate(queries):
        r, f, row, proj = T.ref_score(RX, RA, q, T.RCfg(), RK, 0.5, pools[i])
        recipes.add(r)
        assert int(got["recipe"][i]) == r and _feature_bits(got["features"][i]) == _restated_bits(f), i
        assert got["scores"][i].tobytes() == row.tobytes() and got["candidates"][i].tobytes() == proj.tobytes(), i
    assert len(recipes) >= 2


def test_budget_split_with_mixed_recipes():
    """4 101 queries over 70 000 documents: the score rows (4 bytes a document) split them at 3 834, each batch mixing recipes"""
    docs, voc, ph, burst = T.gen_router_corpus(90, 70_000)
    docs = [d[:200] for d in docs]
    queries = T.gen_router_queries(91, voc, ph, burst, 4101)
    cfg = B.Config()
    X, A = B.Index(cfg, docs), B.Index(T.atire_of(cfg), docs)
    D = Y.Bm25Index(docs)
    pools = [T.pool(92, 70_000, i)[:300] for i in range(4101)]
    rcfg = T.RCfg(atire_max_clarity=float("inf"))   # the 200-byte documents keep no bursty word: lift the clarity gate
    got = D.score_routed(queries, k=5, full=False, router=_router(rcfg), candidates=pools)
    assert len(set(got["recipe"][:3834].tolist())) == 3 and len(set(got["recipe"][3834:].tolist())) == 3
    for i in list(range(0, 4101, 173)) + [3833, 3834, 4100]:
        r, f, row = T.score(X, A, queries[i], rcfg)
        _check(got, i, r, f, row, 5, pools[i])


def test_threads():
    docs, voc, ph, burst = T.gen_router_corpus(95, 3000)
    queries = T.gen_router_queries(96, voc, ph, burst, 300)
    D = Y.Bm25Index(docs)
    C = D.mine_concepts(docs, **CCFG.kw())
    pools = [T.pool(97, 3000, i) for i in range(300)]
    cfgs = [RCFGS[0], RCFGS[1]]
    want = [D.score_routed(queries, k=5, concepts=C, router=_router(c), candidates=pools) for c in cfgs]
    errs = []

    def run(j):
        try:
            for _ in range(3):
                g = D.score_routed(queries, k=5, concepts=C, router=_router(cfgs[j]), candidates=pools)
                assert g["scores"].tobytes() == want[j]["scores"].tobytes() and g["docs"].tobytes() == want[j]["docs"].tobytes()
                assert g["recipe"].tobytes() == want[j]["recipe"].tobytes()
                assert all(a.tobytes() == b.tobytes() for a, b in zip(g["candidates"], want[j]["candidates"]))
        except Exception as e:   # reported below
            errs.append(e)

    ts = [threading.Thread(target=run, args=(j,)) for j in (0, 1)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs
    assert want[0]["recipe"].tobytes() != want[1]["recipe"].tobytes()


def test_argument_errors():
    D = Y.Bm25Index([b"a b c", b"b c d"])
    with pytest.raises(Y.YamsB200Error):
        D.score_routed([b"a"], k=4097)
    with pytest.raises(Y.YamsB200Error):
        D.score_routed([b"a"], candidates=[[0, 2]])   # 2 >= n_docs and not 0xFFFFFFFF
    L = Y.lib()
    q = (C.c_char_p * 2)(b"a", b"b")
    ln = (C.c_size_t * 2)(1, 1)
    docs = (C.c_uint32 * 2)(0, 1)
    out = (C.c_float * 2)()
    for off in ((1, 1, 2), (0, 2, 1)):   # offsets not from 0, decreasing
        o = (C.c_uint64 * 3)(*off)
        assert L.yams_b200_bm25_score_routed(D._h, None, None, 0.5, q, ln, 2, None, 0, None, None, None, o, docs, out, None, None) != 0
    o = (C.c_uint64 * 3)(0, 1, 2)
    assert L.yams_b200_bm25_score_routed(D._h, None, None, 0.5, q, ln, 2, None, 0, None, None, None, o, None, out, None, None) != 0
    assert L.yams_b200_bm25_score_routed(None, None, None, 0.5, q, ln, 2, None, 0, None, None, None, None, None, None, None, None) != 0
    assert L.yams_b200_bm25_score_routed(D._h, None, None, 0.5, q, ln, 2, None, 0, None, None, None, o, docs, out, None, None) == 0
    assert D.score_routed([])["scores"].shape == (0, 2)


def test_cpp_host_adapter(tmp_path):
    """B200Bm25Index::score_routed (full rows and the backend's RescoreDecision pool) and router_features"""
    exe = str(tmp_path / "test_bm25_router")
    subprocess.check_call(["/usr/bin/g++", "-std=c++20", "-O1", os.path.join(ROOT, "tests", "host_cpp", "test_bm25_router.cpp"),
                           "-o", exe, "-L" + os.path.join(ROOT, "yams_b200"), "-lyams_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "yams_b200")])
    docs, voc, ph, burst = T.gen_router_corpus(98, 500)
    queries = T.gen_router_queries(99, voc, ph, burst, 12) + T.edge_queries(voc, burst)[:4]

    def texts(ts):
        return np.array([len(ts)], np.uint64).tobytes() + b"".join(np.array([len(t)], np.uint64).tobytes() + t for t in ts)

    path = tmp_path / "in.bin"
    path.write_bytes(texts(docs) + texts(queries))
    out = subprocess.run([exe, str(path)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.endswith("ALL OK\n"), out.stdout[-500:] + out.stderr
    lines = out.stdout.split("\n")
    assert int(lines[0]) == len(docs)
    cfg = B.Config()
    X, A = B.Index(cfg, docs), B.Index(T.atire_of(cfg), docs)
    K = R.Concepts(docs, docs, R.CCfg(min_ttf=2))
    cands = np.array([(7 * j) % len(docs) for j in range(40)] + [T.NOT_INDEXED, 3, 3], np.uint32)

    def row(i):
        return [int(v) for v in lines[i].split()]

    for i, q in enumerate(queries):
        r, f, full = T.score(X, A, q, T.RCfg(), K, 0.5)
        assert row(1 + 3 * i) == [r] + full.view(np.uint32).tolist(), q
        assert row(2 + 3 * i) == [r] + T.project(full, cands).view(np.uint32).tolist(), q
        assert row(3 + 3 * i) == _restated_bits(f), q
