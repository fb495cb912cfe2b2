"""The BM25 restatement (tests/bm25_restated.py) against simeon's own Bm25Index: every stored answer of the reference build
(tests/golden/ref_bm25.json), and, where oracle/_ref/libref_bm25.so exists (oracle/bm25.mk), the reference build itself on a
random grid of corpora, configurations and queries.  Also: the device entry points fail loudly without a GPU."""
import hashlib
import json
import os

import numpy as np
import pytest

from tests import bm25_restated as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_bm25.json")))["cases"]


def vec_digest(a):
    a = np.asarray(a, np.float32)
    return a.tobytes().hex() if a.size <= 64 else "sha256:" + hashlib.sha256(a.tobytes()).hexdigest()


def f32_bits(x):
    return int(np.array([x], np.float32).view(np.uint32)[0])


def golden_case(c):
    docs, voc = B.gen_corpus(c["seed"], c["n"], c["mean_words"], c["vocab"])
    cfg = B.Config(variant=c["variant"], ngram_min=c["ngram_min"], ngram_max=c["ngram_max"], gamma=c["gamma"],
                   prune_ratio=c["prune_ratio"])
    return docs, B.gen_queries(c["seed"] + 100, voc, c["nq"]), cfg


@pytest.mark.parametrize("case", GOLDEN, ids=[c["name"] for c in GOLDEN])
def test_restatement_reproduces_stored_answers(case):
    docs, queries, cfg = golden_case(case)
    X = B.Index(cfg, docs)
    st, want = X.stats(), case["stats"]
    assert st["n_docs"] == want["n_docs"] and st["total_tokens"] == want["total_tokens"]
    assert f32_bits(st["avg_dl"]) == want["avg_dl_bits"] and f32_bits(st["ngram_avg_dl"]) == want["ngram_avg_dl_bits"]
    assert list(st["terms"]) == want["terms"] and list(st["postings"]) == want["postings"] and st["pruned"] == want["pruned"]
    assert vec_digest(X.words.lengths.view(np.float32)) == case["doc_lengths"]
    for q, d in zip(queries, case["scores"]):
        assert vec_digest(X.score(q)) == d, q
    for w, df, idf_bits, ttf in case["terms"]:
        p = X.words.postings.get(B.hash64(w.encode()))
        got = (0, 0, 0) if p is None else (len(p[0]), f32_bits(p[2]), p[3])
        assert got == (df, idf_bits, ttf), w
    for g, df, idf_bits, ttf in case["ngrams"]:
        p = X.ngrams.postings.get(B.hash64(g.encode()))
        got = (0, 0, 0) if p is None else (len(p[0]), f32_bits(p[2]), p[3])
        assert got == (df, idf_bits, ttf), g


GRID = [(v, n, k, g, r) for v in (B.SAB, B.ATIRE) for n in (0, 1, 2, 3, 50, 400)
        for k, g, r in [((3, 4), 5.0, 0.5), ((1, 1), 0.0, 0.5), ((2, 8), 1e-3, 0.0), ((3, 4), 1e6, 1e-4), ((1, 3), 1.0, 0.34)]]


@pytest.mark.skipif(not B.have_ref(), reason="oracle/_ref/libref_bm25.so not built (no reference tree)")
@pytest.mark.parametrize("variant,n,ngr,gamma,ratio", GRID)
def test_restatement_equals_reference_build(variant, n, ngr, gamma, ratio):
    docs, voc = B.gen_corpus(500 + n, n, 30, 300)
    docs = docs + [b"A" * 3000 + b" tf" * 1500, b"\x80\xff word_1 X y Z"] if n >= 50 else docs
    cfg = B.Config(variant=variant, ngram_min=ngr[0], ngram_max=ngr[1], gamma=gamma, prune_ratio=ratio)
    R, X = B.RefIndex(cfg, docs), B.Index(cfg, docs)
    for q in B.gen_queries(n + 7, voc, 40) + [b"", b"tf tf TF", b"a" * 3000, b"qqqzzz"]:
        assert R.score(q).tobytes() == X.score(q).tobytes(), q
    rs, xs = R.stats(), X.stats()
    for key in rs:
        assert rs[key] == xs[key], key
    assert np.array_equal(R.doc_lengths(0), X.words.lengths)
    if variant == B.SAB:
        assert np.array_equal(R.doc_lengths(1), X.ngrams.lengths)
    for w in voc[:20]:
        df, idf, ttf = R.term(w.lower())
        p = X.words.postings.get(B.hash64(w.lower()))
        assert (df, f32_bits(idf), ttf) == ((0, 0, 0) if p is None else (len(p[0]), f32_bits(p[2]), p[3]))


def test_entry_points_fail_without_a_gpu():
    Y = pytest.importorskip("yams_b200")
    if Y.device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(Y.YamsB200Error) as e:
        Y.Bm25Index([b"alpha beta", b"gamma"])
    assert e.value.status == 4   # YAMS_ERR_INTERNAL
    import ctypes as C
    L = Y.lib()
    stats = Y._lib.Bm25Stats()
    assert L.yams_b200_bm25_stats(None, C.byref(stats)) == 4
    assert L.yams_b200_bm25_score(None, None, None, 0, None, 0, None, None, None) == 4
    ms = (C.c_float * 8)()
    assert L.yams_b200_bm25_last_timings(None, ms) == 4
