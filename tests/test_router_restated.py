"""The restated query router and routed dispatch (tests/router_restated.py) against the stored answers of simeon's own
QueryRouter and the backend's dispatch (tests/golden/ref_router.json) and, where oracle/_ref/libref_router.so exists, against
that build on a grid of document counts, primaries, router configs and blend weights.  The stored cases reach every recipe and
both sides of each threshold; the teeth checks show that lowercasing the router's words, or counting a repeated word once in
n_terms, changes stored answers."""
import hashlib
import json
import os

import numpy as np
import pytest

from tests import bm25_restated as B
from tests import concepts_restated as R
from tests import router_restated as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STORED = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_router.json")))
CCFG = R.CCfg(**STORED["concept_config"])
CASES = {c[0]: c for c in T.CASES}


def _digest(a):
    a = np.ascontiguousarray(a)
    return a.tobytes().hex() if a.size <= 64 and a.dtype == np.float32 else "sha256:" + hashlib.sha256(a.tobytes()).hexdigest()


def _bits(f):
    return [int(f[k]) if k == "n_terms" else int(np.float32(f[k]).view(np.uint32)) for k in T.FEATURES]


def restated(stored):
    docs, queries, cfg, rcfg = T.case_inputs(*CASES[stored["name"]])
    X = B.Index(cfg, docs)
    A = B.Index(T.atire_of(cfg), docs) if T.atire_of(cfg) else None
    return docs, queries, rcfg, X, A, R.Concepts(docs, docs, CCFG)


@pytest.mark.parametrize("stored", STORED["cases"], ids=[c["name"] for c in STORED["cases"]])
def test_stored_answers(stored):
    docs, queries, rcfg, X, A, K = restated(stored)
    for w, answers in stored["answers"].items():
        assert len(answers) == len(queries)
        for i, (q, a) in enumerate(zip(queries, answers)):
            r, f, row = T.score(X, A, q, rcfg, K if w != "None" else None, 0.5)
            assert (r, _bits(f)) == (a["recipe"], a["features"]), (w, q)
            assert _digest(row) == a["scores"], (w, q)
            assert _digest(T.project(row, T.pool(stored["seed"], stored["n"], i))) == a["pool"], (w, q)


def test_stored_cases_reach_their_edges():
    """every recipe, both sides of avg_idf 3 and clarity 3 (avg_idf > 3), n_terms 3 and 4 around avg_idf 5, an uppercase word the
    index holds lowercased, duplicates, blends that change rows, pools with unindexed ids and empty pools"""
    by = {c["name"]: c for c in STORED["cases"]}
    feats = [(a["recipe"], dict(zip(T.FEATURES, a["features"]))) for a in by["sab_default"]["answers"]["None"]]

    def val(f, k):
        return f[k] if k == "n_terms" else float(np.uint32(f[k]).view(np.float32))

    assert {r for r, _ in feats} == {T.ATIRE, T.SAB_SMOOTH, T.CASCADE}
    clean = [f for _, f in feats if f["n_terms"] and f["oov_rate"] == 0]
    assert any(2.5 <= val(f, "avg_idf") <= 3 for f in clean) and any(3 < val(f, "avg_idf") <= 3.5 for f in clean)
    hi = [f for f in clean if val(f, "avg_idf") > 3]
    assert any(2.5 <= val(f, "simplified_clarity") <= 3 for f in hi) and any(3 < val(f, "simplified_clarity") <= 3.5 for f in hi)
    for nt in (3, 4):
        assert any(f["n_terms"] == nt and 4 < val(f, "avg_idf") <= 5 for f in clean)
    assert any(f["n_terms"] == 4 and val(f, "avg_idf") > 5 for f in clean)
    for name in ("sab_forced_atire", "sab_forced_cascade", "sab_strict_gates"):
        assert len({a["recipe"] for a in by[name]["answers"]["None"]}) == 2, name
    docs, queries, rcfg, X, A, K = restated(by["sab_default"])
    up = [q for q in queries if any(w != w.lower() for w in T.router_words(q))]
    assert any(T.features(A, q)["oov_rate"] > 0 and T.features(A, q, fold=True)["oov_rate"] == 0 for q in up)
    assert any(len(set(T.router_words(q))) < len(T.router_words(q)) for q in queries)
    plain, blended = by["sab_default"]["answers"]["None"], by["sab_default"]["answers"]["0.5"]
    assert any(p["scores"] != b["scores"] for p, b in zip(plain, blended))
    pools = [T.pool(7, 600, i) for i in range(len(queries))]
    assert any(len(p) == 0 for p in pools) and any(len(p) > 600 for p in pools)
    assert all(np.any(p == T.NOT_INDEXED) for p in pools if len(p) > 50)


def test_teeth():
    """lowercasing the router's words, or counting a repeated word once in n_terms, changes stored answers"""
    by = {c["name"]: c for c in STORED["cases"]}
    docs, queries, rcfg, X, A, K = restated(by["sab_default"])
    answers = by["sab_default"]["answers"]["None"]
    for kw in ({"fold": True}, {"distinct_terms": True}):
        changed = 0
        for q, a in zip(queries, answers):
            r, f, row = T.score(X, A, q, rcfg, **kw)
            changed += (r, _bits(f)) != (a["recipe"], a["features"])
        assert changed > 0, kw


needs_ref = pytest.mark.skipif(not T.have_ref(), reason="oracle/_ref/libref_router.so not built (no reference tree)")

GRID = [(n, v, rc, w) for n in (0, 1, 2, 37, 600) for v in (B.SAB, B.ATIRE)
        for rc, w in (({}, None), ({}, 0.5), ({"high_idf_threshold": 0.5, "atire_max_clarity": 100.0}, 0.5),
                      ({"cascade_min_terms": 2, "cascade_max_idf": 4.0, "oov_threshold": 0.3}, None))]


@needs_ref
@pytest.mark.parametrize("n,variant,overrides,weight", GRID)
def test_against_reference(n, variant, overrides, weight):
    docs, voc, ph, burst = T.gen_router_corpus(40 + n, n)
    queries = T.gen_router_queries(41 + n, voc, ph, burst, 40) + T.edge_queries(voc, burst)
    cfg, rcfg = B.Config(variant=variant), T.RCfg(**overrides)
    X, RX = B.Index(cfg, docs), T.RefIndex(cfg, docs)
    A = B.Index(T.atire_of(cfg), docs) if T.atire_of(cfg) else None
    RA = T.RefIndex(T.atire_of(cfg), docs) if T.atire_of(cfg) else None
    K = R.Concepts(docs, docs, CCFG) if weight is not None else None
    RK = T.RefConcepts(RX, docs, CCFG) if weight is not None else None
    for i, q in enumerate(queries):
        cands = T.pool(n, n, i)
        r, f, row = T.score(X, A, q, rcfg, K, weight or 0.0)
        wr, wf, wrow, wproj = T.ref_score(RX, RA, q, rcfg, RK, weight or 0.0, cands)
        assert (r, _bits(f)) == (wr, _bits(wf)), q
        assert row.tobytes() == wrow.tobytes() and T.project(row, cands).tobytes() == wproj.tobytes(), q
