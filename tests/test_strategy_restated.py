"""The restatement of the lead-text field and the strategy router's BM25F strategies (tests/strategy_restated.py), pinned to the
stored answers of simeon's own build (tests/golden/ref_strategy.json) and, where oracle/_ref exists, to that build itself on a
grid.  The pin has teeth: scaling the body after the aux legs instead of before, or dropping the zero scores simeon::top_k keeps
from the keyphrase gate's top-10, changes stored answers.  The z-score's sums in double of float32 scores are exact on the stored
corpora, so no order of them can change a stored answer; their order is pinned on a row where it shows."""
import hashlib
import json
import os

import numpy as np
import pytest

from tests import bm25_restated as B
from tests import concepts_restated as R
from tests import strategy_restated as S
from tests.golden import make_strategy_golden as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STORED = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_strategy.json")))
CCFG = R.CCfg(**STORED["concept_config"])
needs_ref = pytest.mark.skipif(not S.have_ref(), reason="oracle/_ref/libref_strategy.so not built (no reference tree)")


def test_lead_texts():
    texts, _ = S.gen_lead_corpus(STORED["lead_corpus_seed"], STORED["lead_corpus_n"])
    for rec in STORED["leads"]:
        leads = [S.lead(t, rec["L"]) for t in texts]
        assert [len(x) for x in leads] == rec["cuts"]
        assert hashlib.sha256(b"\0".join(leads)).hexdigest() == rec["digest"]


def test_lead_edges():
    for sp in S.SPACE:
        c = bytes([sp])
        assert S.lead(b"a" + c + b"b" + c + b"c", 2) == b"a b"
        assert S.lead(c + b"a" + c * 2 + b"b", 1) == b" a"
        assert S.lead(c * 3, 64) == b""
    assert S.lead(b"a\x00b c\x85d e", 2) == b"a\x00b c\x85d"   # NUL and bytes >= 0x80 are token bytes
    assert S.lead(b"one two", 5) == b"one two"


def _case(c):
    docs, queries = G.case_inputs(c)
    X = S.Index(B.Config(variant=G.VARIANTS[c["variant"]]), docs, c["lead"])
    K = R.Concepts(docs, docs, CCFG)
    return docs, queries, X, K


@pytest.mark.parametrize("case", STORED["cases"], ids=[c["name"] for c in STORED["cases"]])
def test_stored_answers(case):
    docs, queries, X, K = _case(case)
    for f, want in zip((2, 3), case["aux"]):
        F = X.field(f)
        assert len(F.lengths) == want["docs"] and int(F.lengths.astype(np.uint64).sum()) == want["sum"]
        assert float(F.avg) == want["avg"] and len(F.postings) == want["terms"]
        assert sum(len(v[0]) for v in F.postings.values()) == want["postings"]
    for pool in (0, 1, 2, 3):
        for w in (None, 0.5):
            got = [G.digest(S.score(X, pool, q, K if w is not None else None, w or 0.0)) for q in queries]
            assert got == case["scores"][f"{pool}/{w}"], (pool, w)
    assert [S.route(X.score(q)) for q in queries] == case["routed"]


def test_teeth_body_scale_order():
    """scaling the body after the aux legs changes some stored answer of each lead case"""
    for case in STORED["cases"]:
        if case["lead"] == 0 or case["name"] in ("all_leads_empty",):
            continue
        docs, queries, X, K = _case(case)
        moved = [G.digest(S.score(X, 2, q, scale_after_aux=True)) for q in queries]
        assert moved != case["scores"]["2/None"], case["name"]


def _changed(mistake):
    n = 0
    for case in STORED["cases"]:
        docs, queries, X, K = _case(case)
        n += [G.digest(X.keyphrase(q, **mistake)) for q in queries] != case["scores"]["1/None"]
    return n


def test_teeth_pairwise_zscore():
    """on 200 000 scores spanning 12 decades the sequential sums (the reference's order) differ from pairwise ones"""
    rng = np.random.default_rng(1)
    x = (10.0 ** rng.uniform(-8, 4, 200_000)).astype(np.float32)
    x[::7] = 0
    seq, pw = S.zscore_sums(x), S.zscore_sums(x, pairwise=True)
    assert seq[0] != pw[0] and seq[1] != pw[1]
    xd = x.astype(np.float64)
    acc = 0.0
    for v in xd.tolist():   # a plain loop: Python's sum() of floats is compensated
        acc += v
    assert seq[0] == acc / len(x)


def test_teeth_zero_padding():
    assert _changed({"pad": False}) > 0


GRID = [(v, n, L) for v in (B.SAB, B.ATIRE) for n, L in ((1, 64), (2, 1), (9, 64), (10, 2), (11, 64), (700, 64), (700, 7))]


@needs_ref
@pytest.mark.parametrize("variant,n,L", GRID)
def test_against_reference(variant, n, L):
    docs, voc = S.gen_lead_corpus(300 + n + L, n)
    queries = S.gen_lead_queries(400 + n, voc, 12)
    cfg = B.Config(variant=variant)
    X = S.Index(cfg, docs, L)
    ref = S.RefStrategy(cfg, docs, L, CCFG)
    K = R.Concepts(docs, docs, CCFG)
    for t in docs[:50]:
        assert S.lead(t, L) == S.ref_lead(t, L)
    for f in range(4):
        assert np.array_equal(X.doc_lengths(f), ref.doc_lengths(f)), f
        st = ref.field_stats(f)
        assert st["docs"] == len(X.field(f).lengths) and st["avg"] == X.field(f).avg and st["terms"] == len(X.field(f).postings)
        for h in list(X.field(f).postings)[:20]:
            d, t, idf, ttf = ref.postings(f, h)
            xd, xt, xidf, xttf = X.field(f).postings[h]
            assert np.array_equal(d, xd) and np.array_equal(t, xt) and idf == xidf and ttf == xttf
    for q in queries:
        s, chosen = ref.score(3, q, None, chosen=True)
        assert chosen == S.route(X.score(q)) and s.tobytes() == S.score(X, 3, q).tobytes(), q
        for pool in (0, 1, 2):
            assert S.score(X, pool, q).tobytes() == ref.score(pool, q).tobytes(), (pool, q)
            assert S.score(X, pool, q, K, 0.5).tobytes() == ref.score(pool, q, 0.5).tobytes(), (pool, q)
