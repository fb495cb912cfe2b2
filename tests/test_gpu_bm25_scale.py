"""yams_b200_bm25_* bit for bit against the restatement (tests/bm25_restated.py) on the paths the corpora of test_gpu_bm25.py
are too small to reach: a build cut into many document slices (YAMS_B200_BM25_SLICE_PAIRS) whose postings are merged, queries
scored in more than one batch (the 4096-query cap and the 1 GiB bound on score rows), score tiles cut at 4096-document
boundaries, and the fused top-k at its full width of 4096, where rows longer than 4096 documents take the radix select."""
import functools
import os

import numpy as np
import pytest

from tests import bm25_restated as B
from tests.test_gpu_bm25 import _bits, _check, _device

pytestmark = pytest.mark.gpu

SLICE_ENV = "YAMS_B200_BM25_SLICE_PAIRS"
TOPK_MAX = 4096


def _queries_per_batch(n, nq):
    """bm25_score's batch: min(2^30 bytes of score rows, nq, 4096) queries (bm25.cu qb_max)"""
    return max(1, min((1 << 30) // (4 * n), nq, 4096))


def _pairs(X):
    """the pairs a document adds to a slice: its words, plus its n-grams for SubwordAwareBackoff"""
    c = X.words.lengths.astype(np.int64)
    return c + X.ngrams.lengths if X.cfg.variant == B.SAB else c


def _slice_cuts(pairs, budget):
    """bm25_build's cut rule: a new slice starts before document d when the current one holds pairs and d's would take it over
    the budget.  Returns the first document of every slice."""
    cuts, acc = [0], 0
    for d, c in enumerate(pairs.tolist()):
        if acc and acc + c > budget:
            cuts.append(d)
            acc = 0
        acc += c
    return cuts


def _check_topk(got, i, want, k):
    """row i of the fused top-k against the restatement's score vector, padding included"""
    wd, ws = B.topk(want, k)
    c = int(got["counts"][i])
    assert c == len(wd), i
    assert np.array_equal(got["docs"][i, :c], wd) and got["topk_scores"][i, :c].tobytes() == ws.tobytes(), i
    assert np.all(got["docs"][i, c:] == 0xFFFFFFFF) and not got["topk_scores"][i, c:].view(np.uint32).any(), i


def _check_all_postings(D, X, sample=300):
    """every posting list of the restatement on the device (docs, tfs, idf bits, total_tf), and a sample of the n-grams the
    restatement pruned absent from the device"""
    fields = [(0, X.words)] + ([(1, X.ngrams)] if X.cfg.variant == B.SAB else [])
    for fld, F in fields:
        for h, (docs, tfs, idf, ttf) in F.postings.items():
            d, t, i, tt = D.postings(fld, h)
            assert np.array_equal(d, docs) and np.array_equal(t, tfs) and _bits(i) == _bits(idf) and tt == ttf, (fld, hex(h))
    if X.cfg.variant != B.SAB:
        return
    # the n-grams of the corpus's words (the restatement also memoises the words of the queries it scored: not in the index)
    grams = {g for w, gs in X._grams.items() if X.h(w) in X.words.postings for g in gs}
    pruned = sorted(grams - X.ngrams.postings.keys())
    assert len(pruned) == X.ngrams.pruned
    for j in np.random.default_rng(1).permutation(len(pruned))[:sample]:
        d, _, _, tt = D.postings(1, pruned[j])
        assert len(d) == 0 and tt == 0, hex(pruned[j])


# ---- the build cut into document slices ----
SLICE_CONFIGS = {
    "sab": B.Config(),
    "sab-gamma0-unigrams": B.Config(gamma=0.0, ngram_min=1, ngram_max=1),
    "sab-noprune": B.Config(prune_ratio=0.0),
    "atire": B.Config(variant=B.ATIRE),
}


@functools.lru_cache(maxsize=None)
def _sliced_corpus():
    """2 000 generated documents with documents of words shorter than 3 bytes (no n-grams of 3..4), a document of 4 000 words
    in the middle and one at the end (each more pairs than a slice of a twenty-fifth of the corpus), and empty and word-free
    documents after the last one"""
    docs, voc = B.gen_corpus(4242, 2000, 20, 1000)
    big = b" ".join(voc[i % 300] for i in range(4000))
    short = [b"a bb C dd", b"x yz Q_", b"i j"]
    docs = docs[:700] + short + [big] + docs[700:] + [big.upper(), b"", b" .,\xe2\x80\x94", b""]
    queries = B.gen_queries(4243, voc, 40) + [b"bb yz", b"a i j", b"dd " + voc[0], voc[299] + b" " + voc[5], voc[0] + b" " + voc[1]]
    return docs, queries


@functools.lru_cache(maxsize=None)
def _sliced_restated(name):
    return B.Index(SLICE_CONFIGS[name], _sliced_corpus()[0])


@pytest.mark.parametrize("budget", ["1", "mid", "total-1", "total"])
@pytest.mark.parametrize("name", list(SLICE_CONFIGS))
def test_sliced_build(name, budget):
    """slices of at most N pairs give the index of one slice: the slice count of the cut rule, every score bit, the top-k, stats,
    doc lengths and every posting list"""
    cfg = SLICE_CONFIGS[name]
    docs, queries = _sliced_corpus()
    X = _sliced_restated(name)
    n, pairs = len(docs), _pairs(X)
    total = int(pairs.sum())
    assert total < 1 << 20   # under the budget's floor: the override alone decides the cuts, whatever the device holds
    N = {"1": 1, "mid": total // 25, "total-1": total - 1, "total": total}[budget]
    cuts = _slice_cuts(pairs, N)
    bounds = list(zip(cuts, cuts[1:] + [n]))
    if budget == "total":
        assert len(cuts) == 1
    elif budget == "total-1":
        assert len(cuts) == 2
    else:
        assert len(cuts) >= 10 and pairs.max() > N   # a document over the budget on its own
        assert X.words.lengths[cuts[-1]:].sum() == 0   # a last slice without words
        if cfg.variant == B.SAB and cfg.ngram_min == 3 and budget == "1":   # a slice of words without n-grams
            assert any(X.words.lengths[a:b].sum() > 0 and X.ngrams.lengths[a:b].sum() == 0 for a, b in bounds)
        if cfg.variant == B.SAB and cfg.prune_ratio > 0:
            # n-grams over df_max overall are pruned, though no slice has more than df_max documents
            assert X.ngrams.pruned > 0 and max(b - a for a, b in bounds) <= int(float(np.float32(cfg.prune_ratio)) * n)
    os.environ[SLICE_ENV] = str(N)
    try:
        D = _check(cfg, docs, queries, k=10)
    finally:
        del os.environ[SLICE_ENV]
    assert D.last_timings()["build_slices"] == len(cuts)
    _check_all_postings(D, X)
    D1 = _device(cfg, docs)
    assert D1.last_timings()["build_slices"] == 1
    assert D.score(queries)["scores"].tobytes() == D1.score(queries)["scores"].tobytes()


def test_slice_override_zero_is_unset():
    """YAMS_B200_BM25_SLICE_PAIRS = 0 leaves the memory budget in charge (one slice here)"""
    docs, _ = _sliced_corpus()
    os.environ[SLICE_ENV] = "0"
    try:
        D = _device(B.Config(), docs)
    finally:
        del os.environ[SLICE_ENV]
    assert D.last_timings()["build_slices"] == 1


# ---- scoring in batches of queries ----
def test_batched_scoring_query_cap():
    """4 101 queries over 3 000 documents: batches of 4 096 and 5 queries, with full vectors and a top-k, the top-k alone, and
    full vectors alone"""
    cfg = B.Config()
    docs, voc = B.gen_corpus(3100, 3000, 12, 800)
    queries = B.gen_queries(3101, voc, 4096) + [voc[0] + b" " + voc[i] for i in range(1, 6)]
    n, nq = len(docs), len(queries)
    assert _queries_per_batch(n, nq) == 4096 and nq == 4096 + 5
    X = B.Index(cfg, docs)
    want = np.stack([X.score(q) for q in queries])
    for j in range(5):   # a row of the second batch cannot pass for the same row of the first
        assert not np.array_equal(want[4096 + j], want[j])
    D = _device(cfg, docs)
    got = D.score(queries, k=10)
    assert got["scores"].tobytes() == want.tobytes()
    for i in range(nq):
        _check_topk(got, i, want[i], 10)
    top = D.score(queries, k=10, full=False)
    assert "scores" not in top
    for key in ("docs", "topk_scores", "counts"):
        assert top[key].tobytes() == got[key].tobytes(), key
    full = D.score(queries, k=0)
    assert full["scores"].tobytes() == want.tobytes() and "docs" not in full


def test_batched_scoring_dense_bound():
    """1 000 queries over 270 000 documents: 1 GiB of score rows holds 994, so the last 6 are a second batch.  Every top-k and the
    full vectors around the batch boundary against the restatement; every row and top-k against one query per call."""
    cfg = B.Config()
    docs, voc = B.gen_corpus(2025, 270_000, 8, 20_000)
    queries = B.gen_queries(2026, voc, 994) + [voc[i] + b" " + voc[i + 10] for i in range(6)]
    n, nq = len(docs), len(queries)
    qb = _queries_per_batch(n, nq)
    assert qb == 994 and nq == qb + 6
    X = B.Index(cfg, docs)
    D = _device(cfg, docs)
    got = D.score(queries, k=100)   # 1.08 GB of full vectors
    rows = set(range(6)) | set(range(qb - 6, nq))
    want_rows = {}
    for i, q in enumerate(queries):
        want = X.score(q)
        _check_topk(got, i, want, 100)
        if i in rows:
            want_rows[i] = want
            assert got["scores"][i].tobytes() == want.tobytes(), i
    for j in range(6):
        assert not np.array_equal(want_rows[qb + j], want_rows[j])
    for i, q in enumerate(queries):
        one = D.score([q], k=100)
        assert one["scores"][0].tobytes() == got["scores"][i].tobytes(), i
        for key in ("docs", "topk_scores"):
            assert one[key][0].tobytes() == got[key][i].tobytes(), (i, key)
        assert one["counts"][0] == got["counts"][i], i


# ---- score tiles ----
EDGE_DOCS = (0, 4095, 4096, 8191, 8192)


@pytest.mark.parametrize("variant", [B.SAB, B.ATIRE], ids=["sab", "atire"])
@pytest.mark.parametrize("n", [4095, 4096, 4097, 8192, 8193])
def test_tile_edges(n, variant):
    """n at and around the 4096-document tiles of bm_score_kernel; a word in every document, and words only in the documents
    either side of a tile boundary"""
    base, voc = B.gen_corpus(5000 + n, n, 6, 500)
    docs = [t + b" everywhere" for t in base]
    for d in EDGE_DOCS:
        if d < n:
            docs[d] += b" rimword edge%d" % d
    queries = ([b"everywhere", b"rimword", b"rimword everywhere", b"edge0 edge8192 rimword"] + [b"edge%d" % d for d in EDGE_DOCS] +
               B.gen_queries(6000 + n, voc, 24))
    _check(B.Config(variant=variant), docs, queries, k=16)


# ---- the fused top-k at k = 4096 ----
@pytest.mark.parametrize("variant", [B.SAB, B.ATIRE], ids=["sab", "atire"])
@pytest.mark.parametrize("n", [4095, 4096, 10_000])
def test_topk_full_width(n, variant):
    """k = 4096 over rows of n documents, 60 % of them identical copies: at n = 10 000 the copies' equal scores straddle rank
    4096 in the radix select and go by ascending document.  Queries with fewer than 4096 positive scores are padded; a query of
    the whole 2 000-word vocabulary gives one CTA thousands of legs."""
    cfg = B.Config(variant=variant)
    rng = np.random.default_rng(n)
    base, voc = B.gen_corpus(7000 + n, n, 10, 2000)
    copy = b"tie tie breaker " + voc[0] + b" " + voc[3]
    docs = list(base)
    perm = rng.permutation(n)
    for d in perm[: n * 6 // 10]:
        docs[d] = copy
    for d in perm[-50:]:   # a word of 2 bytes has no n-grams of 3..4: 50 documents score > 0
        docs[d] += b" qj"
    everything = b" ".join(voc)
    queries = [b"tie", voc[3], b"tie " + voc[3], b"qj", b"breaker " + voc[1999], everything, b"!?"]
    X = B.Index(cfg, docs)
    want = [X.score(q) for q in queries]
    if n > TOPK_MAX:
        for i in (0, 1):
            ties = B.topk(want[i], n)[1]
            assert ties[TOPK_MAX - 1] == ties[TOPK_MAX], i   # equal scores straddle rank 4096
    assert np.count_nonzero(want[3] > 0) == 50
    D = _check(cfg, docs, queries, k=TOPK_MAX)
    got = D.score(queries, k=TOPK_MAX, full=False)
    for i in range(len(queries)):
        _check_topk(got, i, want[i], TOPK_MAX)
    assert got["counts"][3] == 50 and got["counts"][6] == 0
