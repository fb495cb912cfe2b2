"""The restated reciprocal-rank fusion of BM25 variants (tests/rrf_restated.py) against the stored answers of simeon's own
score_bm25_variants_rrf (tests/golden/ref_rrf.json) and, where oracle/_ref/libref_rrf.so exists, against that build on a grid of
document counts, variant lists (orders, repeats, one config), k_rrf values and blend weights.  The teeth checks show that the
two order-dependent steps matter: the document order of tied scores within a ranking, and the variant order of the
accumulation."""
import hashlib
import json
import os

import numpy as np
import pytest

from tests import bm25_restated as B
from tests import concepts_restated as R
from tests import rrf_restated as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STORED = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_rrf.json")))
GOLDEN = STORED["cases"]
CCFG = R.CCfg(**STORED["concept_config"])


def _digest(a):
    a = np.ascontiguousarray(a)
    return a.tobytes().hex() if a.size <= 64 and a.dtype == np.float32 else "sha256:" + hashlib.sha256(a.tobytes()).hexdigest()


def restated(case):
    """(docs, queries, restated indexes, restated concepts) of a stored case"""
    docs, queries, cfgs = F.case_inputs(case)
    return docs, queries, [B.Index(c, docs) for c in cfgs], R.Concepts(docs, docs, CCFG)


@pytest.mark.parametrize("case", GOLDEN, ids=[c["name"] for c in GOLDEN])
def test_stored_answers(case):
    docs, queries, X, K = restated(case)
    ranked = 0
    for s in case["scores"]:
        w = s["weight"]
        for q, d in zip(queries, s["digests"]):
            got = F.score(X, q, s["k_rrf"], K if w is not None else None, w or 0.0, n=len(docs))
            assert _digest(got) == d, (s["k_rrf"], w, q[:80])
            ranked += int(np.count_nonzero(got))
    assert (ranked > 0) == (case["name"] not in ("zero_variants", "matches_nothing"))


def test_stored_cases_reach_their_edges():
    """the stored corpora really have tied rankings, documents only the n-gram field ranks, and fused values that the blend
    changes"""
    by = {c["name"]: c for c in GOLDEN}
    docs, queries, X, _ = restated(by["score_ties"])
    assert any(len(np.unique(X[0].score(q)[F.ranking(X[0].score(q))])) < len(F.ranking(X[0].score(q))) for q in queries)
    docs, queries, X, _ = restated(by["ngram_only"])
    assert any(len(F.ranking(X[0].score(q))) > len(F.ranking(X[1].score(q))) > 0 for q in queries)
    s = by["sab_atire"]["scores"]
    assert s[0]["digests"] != s[1]["digests"]   # plain and blended differ


needs_ref = pytest.mark.skipif(not F.have_ref(), reason="oracle/_ref/libref_rrf.so not built (no reference tree)")


@needs_ref
@pytest.mark.parametrize("n,variants,k_rrf,weight", F.GRID)
def test_against_reference(n, variants, k_rrf, weight):
    docs, queries, cfgs = F.grid_case(n, variants)
    X = [B.Index(c, docs) for c in cfgs]
    RI = [F.RefIndex(c, docs) for c in cfgs]
    K = R.Concepts(docs, docs, CCFG) if weight is not None else None
    RK = F.RefConcepts(RI[0], docs, CCFG) if weight is not None else None
    for q in queries:
        want = F.ref_score(RI, q, k_rrf, RK, weight or 0.0)
        assert F.score(X, q, k_rrf, K, weight or 0.0).tobytes() == want.tobytes(), q


@needs_ref
def test_zero_variants_and_catch2_case():
    docs = [b"alpha beta", b"gamma delta"]
    RI = [F.RefIndex(F.SAB, docs), F.RefIndex(F.ATIRE, docs)]
    assert F.ref_score(RI, b"absent").tolist() == [0.0, 0.0]            # no prior for documents nothing ranks
    assert F.ref_score([], b"alpha", n=3).tolist() == [0.0, 0.0, 0.0]
    X = [B.Index(F.SAB, docs), B.Index(F.ATIRE, docs)]
    assert F.ref_score(RI, b"alpha").tobytes() == F.score(X, b"alpha").tobytes()


@needs_ref
def test_teeth():
    """reversing the tie order within a ranking, or the order the variants accumulate in, changes the reference's answer"""
    by = {c["name"]: c for c in GOLDEN}
    docs, queries, X, _ = restated(by["score_ties"])
    RI = [F.RefIndex(c, docs) for c in F.case_inputs(by["score_ties"])[2]]
    assert any(F.score(X, q, ties_descending=True).tobytes() != F.ref_score(RI, q).tobytes() for q in queries)
    docs, queries, X, _ = restated(by["three_configs"])
    RI = [F.RefIndex(c, docs) for c in F.case_inputs(by["three_configs"])[2]]
    assert all(F.score(X, q).tobytes() == F.ref_score(RI, q).tobytes() for q in queries)
    assert any(F.score(X[::-1], q).tobytes() != F.ref_score(RI, q).tobytes() for q in queries)
