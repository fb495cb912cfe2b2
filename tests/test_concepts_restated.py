"""The restated word-bigram concept index (tests/concepts_restated.cpp) against the stored answers of simeon's own ConceptIndex
(tests/golden/ref_concepts.json) and, where oracle/_ref/libref_concepts.so exists, against that build on a grid of document
counts, min_ttf, PMI floors, caps (a tie across the cut included), blend weights and both BM25 variants.  The teeth checks show
that the two order-dependent steps matter: the blend's concept order and the tied subset kept at the cap."""
import hashlib
import json
import os

import numpy as np
import pytest

from tests import bm25_restated as B
from tests import concepts_restated as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_concepts.json")))["cases"]


def _digest(a):
    a = np.ascontiguousarray(a)
    return a.tobytes().hex() if a.size <= 64 and a.dtype == np.float32 else "sha256:" + hashlib.sha256(a.tobytes()).hexdigest()


def _bits(x):
    return int(np.array([x], np.float32).view(np.uint32)[0])


def golden_inputs(case):
    docs, voc, ph = R.gen_concept_corpus(case["seed"], case["n"], 30, 1500, 40, case["tie_groups"])
    queries = R.gen_concept_queries(case["seed"] + 1, voc, ph, case["nq"])
    return docs, queries, R.CCfg(**case["config"]), B.Config(variant=case["variant"])


@pytest.mark.parametrize("case", GOLDEN, ids=[c["name"] for c in GOLDEN])
def test_stored_answers(case):
    docs, queries, cfg, bcfg = golden_inputs(case)
    K = R.Concepts(docs, docs, cfg)
    st, want = K.stats(), case["stats"]
    assert (st["size"], st["doc_count"], _bits(st["avg_bigram_dl"]), st["sum_bigram_dl"]) == \
        (want["size"], want["doc_count"], want["avg_bits"], want["sum_bigram_dl"])
    assert _digest(K.bigram_lengths()) == case["bigram_lengths"] and _digest(K.hashes()) == case["hashes"]
    for c in case["concepts"]:
        e = K.find(int(c["hash"]))
        assert (_bits(e["pmi"]), _bits(e["idf"]), str(e["a_hash"]), str(e["b_hash"]), e["total_tf"]) == \
            (c["pmi_bits"], c["idf_bits"], c["a"], c["b"], c["total_tf"])
        assert e["docs"].tolist() == c["docs"] and e["tfs"].tolist() == c["tfs"]
    X = B.Index(bcfg, docs)
    for q, d in zip(queries, case["scores"]):
        assert _digest(R.blended(X, K, q, case["weight"])) == d, q
    if case["name"] == "cap_tie_straddles":
        assert st["replayed"]
    if case["name"] == "cap_no_tie":
        assert st["accepted"] > st["size"] and not st["replayed"]


def compare(F, K, X, docs, queries, weight):
    """the restatement K (with the restated BM25 X) equals the reference F: stats, lengths, kept hashes, every concept, scores"""
    st, fs = K.stats(), F.stats()
    assert (st["size"], st["doc_count"], _bits(st["avg_bigram_dl"]), st["sum_bigram_dl"]) == \
        (fs["size"], fs["doc_count"], _bits(fs["avg_bigram_dl"]), fs["sum_bigram_dl"])
    assert np.array_equal(K.bigram_lengths(), F.bigram_lengths())
    hs = K.hashes()
    assert np.array_equal(hs, F.hashes())
    for h in hs:
        a, b = K.find(int(h)), F.find(int(h))
        assert all(np.array_equal(a[k], b[k]) if k in ("docs", "tfs") else _bits(a[k]) == _bits(b[k]) if k in ("pmi", "idf") else a[k] == b[k]
                   for k in a), int(h)
    rng = np.random.default_rng(len(docs))
    base = rng.standard_normal(len(docs)).astype(np.float32)
    for q in queries:
        assert R.blended(X, K, q, weight).tobytes() == F.score_blended(q, weight).tobytes(), q
        assert K.blend(q, base, weight).tobytes() == F.blend(q, base, weight).tobytes(), q


needs_ref = pytest.mark.skipif(not R.have_ref(), reason="oracle/_ref/libref_concepts.so not built (no reference tree)")


@needs_ref
@pytest.mark.parametrize("n,variant,min_ttf,floor,cap,weight", R.GRID)
def test_against_reference(n, variant, min_ttf, floor, cap, weight):
    docs, queries, cfg = R.grid_case(n, variant, min_ttf, floor, cap)
    F = R.RefConcepts(B.Config(variant=variant), docs, docs, cfg)
    compare(F, R.Concepts(docs, docs, cfg), B.Index(B.Config(variant=variant), docs), docs, queries, weight)


@needs_ref
def test_concept_texts_differ_from_index_texts():
    """the backend mines its raw texts against an index of other texts; a document-count mismatch makes the blend a no-op"""
    docs, voc, ph = R.gen_concept_corpus(21, 400, 25, 800, 30, 4)
    other = [d.lower()[: len(d) // 2] for d in docs]
    queries = R.gen_concept_queries(22, voc, ph, 20)
    for ctexts in (docs, docs + [b"", b"tiea0 tieb0"]):
        F = R.RefConcepts(B.Config(), other, ctexts, R.CCfg(min_ttf=2))
        K = R.Concepts(other, ctexts, R.CCfg(min_ttf=2))
        st = K.stats()
        assert st["size"] == F.stats()["size"] > 0
        assert np.array_equal(K.hashes(), F.hashes())
        X = B.Index(B.Config(), other)
        for q in queries:
            assert R.blended(X, K, q, 0.5).tobytes() == F.score_blended(q, 0.5).tobytes(), q
        if len(ctexts) != len(other):
            assert all(R.blended(X, K, q, 0.5).tobytes() == X.score(q).tobytes() for q in queries)


def test_teeth_blend_order():
    """a document in several matched concepts: adding them by ascending hash instead of the reference's order changes a bit"""
    case = next(c for c in GOLDEN if c["name"] == "min_ttf_1_floor_0")
    docs, queries, cfg, bcfg = golden_inputs(case)
    K = R.Concepts(docs, docs, cfg)
    X = B.Index(bcfg, docs)
    hs = K.hashes()
    changed = 0
    rng = np.random.default_rng(3)
    for q in [docs[int(i)][:200] for i in rng.integers(0, len(docs), 40)]:
        base = X.score(q)
        changed += K.blend(q, base, 0.5).tobytes() != K.blend(q, base, 0.5, sorted_order=True).tobytes()
    assert len(hs) > 0 and changed > 0


def test_teeth_tied_subset():
    """at a cap inside a PMI tie, another tied subset gives another kept-hash digest"""
    case = next(c for c in GOLDEN if c["name"] == "cap_tie_straddles")
    docs, _, cfg, _ = golden_inputs(case)
    a, b = R.Concepts(docs, docs, cfg), R.Concepts(docs, docs, cfg, cap_mode=1)
    assert a.stats()["replayed"] and _digest(a.hashes()) == case["hashes"]
    assert _digest(b.hashes()) != case["hashes"]
