"""yams_b200_bm25_* (simeon's Bm25Index on the device) bit for bit: against the stored answers of the reference build
(tests/golden/ref_bm25.json) and against the restatement (tests/bm25_restated.py) over document counts 0..200 000, gamma,
n-gram ranges, prune ratios (the df == df_max boundary and n = 1 included), hostile texts and queries, the fused top-k with
ties, the posting / stats accessors, and the C++ host adapter B200Bm25Index."""
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

import yams_b200 as Y
from tests import bm25_restated as B

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_bm25.json")))["cases"]


def _digest(a):
    a = np.asarray(a, np.float32)
    return a.tobytes().hex() if a.size <= 64 else "sha256:" + hashlib.sha256(a.tobytes()).hexdigest()


def _bits(x):
    return int(np.array([x], np.float32).view(np.uint32)[0])


def _device(cfg: B.Config, docs):
    return Y.Bm25Index(docs, k1=cfg.k1, b=cfg.b, delta=cfg.delta, subword_gamma=cfg.gamma, variant=cfg.variant,
                       ngram_min=cfg.ngram_min, ngram_max=cfg.ngram_max, ngram_df_prune_ratio=cfg.prune_ratio, hash_seed=cfg.hash_seed)


def _check(cfg, docs, queries, k=10, postings_of=()):
    """every score bit, the top-k, stats, doc lengths and the posting lists of some words against the restatement"""
    X = B.Index(cfg, docs)
    D = _device(cfg, docs)
    got = D.score(queries, k=k)
    for i, q in enumerate(queries):
        want = X.score(q)
        assert got["scores"][i].tobytes() == want.tobytes(), (i, q[:80])
        wd, ws = B.topk(want, k)
        c = int(got["counts"][i])
        assert c == len(wd), (i, q[:80])
        assert np.array_equal(got["docs"][i, :c], wd) and got["topk_scores"][i, :c].tobytes() == ws.tobytes(), (i, q[:80])
        assert np.all(got["docs"][i, c:] == 0xFFFFFFFF)
    st, xs = D.stats(), X.stats()
    for key in ("n_docs", "total_tokens", "terms", "postings", "pruned"):
        assert st[key] == xs[key], key
    assert _bits(st["avg_dl"]) == _bits(xs["avg_dl"]) and _bits(st["ngram_avg_dl"]) == _bits(xs["ngram_avg_dl"])
    assert np.array_equal(D.doc_lengths(0), X.words.lengths)
    if cfg.variant == B.SAB:
        assert np.array_equal(D.doc_lengths(1), X.ngrams.lengths)
    for w in postings_of:
        for fld, F, hs in ((0, X.words, [X.h(w)]), (1, X.ngrams, X.gram_hashes(w)[:4] if cfg.variant == B.SAB else [])):
            for h in hs:
                docs_, tfs, idf, ttf = D.postings(fld, h)
                p = F.postings.get(h)
                if p is None:
                    assert len(docs_) == 0 and ttf == 0
                else:
                    assert np.array_equal(docs_, p[0]) and np.array_equal(tfs, p[1]) and _bits(idf) == _bits(p[2]) and ttf == p[3]
    return D


@pytest.mark.parametrize("case", GOLDEN, ids=[c["name"] for c in GOLDEN])
def test_stored_answers(case):
    docs, voc = B.gen_corpus(case["seed"], case["n"], case["mean_words"], case["vocab"])
    queries = B.gen_queries(case["seed"] + 100, voc, case["nq"])
    cfg = B.Config(variant=case["variant"], ngram_min=case["ngram_min"], ngram_max=case["ngram_max"], gamma=case["gamma"],
                   prune_ratio=case["prune_ratio"])
    D = _device(cfg, docs)
    got = D.score(queries)["scores"]
    for i, d in enumerate(case["scores"]):
        assert _digest(got[i]) == d, i
    st, want = D.stats(), case["stats"]
    assert st["n_docs"] == want["n_docs"] and st["total_tokens"] == want["total_tokens"] and st["pruned"] == want["pruned"]
    assert _bits(st["avg_dl"]) == want["avg_dl_bits"] and _bits(st["ngram_avg_dl"]) == want["ngram_avg_dl_bits"]
    assert list(st["terms"]) == want["terms"] and list(st["postings"]) == want["postings"]
    assert _digest(D.doc_lengths(0).view(np.float32)) == case["doc_lengths"]
    for fld, rows in ((0, case["terms"]), (1, case["ngrams"])):
        for t, df, idf_bits, ttf in rows:
            d, _, idf, tt = D.postings(fld, B.hash64(t.encode()))
            assert (len(d), _bits(idf) if len(d) else 0, tt) == (df, idf_bits, ttf), t


GRID = [(v, n, g, ngr, r) for v in (B.SAB, B.ATIRE) for n in (0, 1, 2, 3, 1000)
        for g, ngr, r in [(5.0, (3, 4), 0.5), (0.0, (1, 1), 0.5), (1e-3, (2, 8), 0.0), (1e6, (3, 4), 1e-4), (5.0, (2, 8), 0.5),
                          (1e-3, (3, 4), 0.5)]]


@pytest.mark.parametrize("variant,n,gamma,ngr,ratio", GRID)
def test_against_restatement(variant, n, gamma, ngr, ratio):
    docs, voc = B.gen_corpus(900 + n, n, 30, 1500)
    queries = B.gen_queries(n + 1, voc, 48) + [b"", b"!!", voc[0] + b" " + voc[0] + b" " + voc[0].upper()]
    cfg = B.Config(variant=variant, ngram_min=ngr[0], ngram_max=ngr[1], gamma=gamma, prune_ratio=ratio)
    _check(cfg, docs, queries, k=7, postings_of=[w.lower() for w in voc[:8]])


def test_hostile_texts_and_queries():
    """empty and word-free documents, bytes >= 0x80, mixed case, 1- and 2-byte words, a 100 KB word, tf in the thousands, a 1 MB
    document; queries: empty, out-of-vocabulary (n-gram leg only), duplicated words, words whose n-grams were all pruned, and
    1 000 queries in one call"""
    rng = np.random.default_rng(5)
    docs, voc = B.gen_corpus(77, 2000, 20, 800)
    big_word = bytes(rng.integers(97, 123, 100_000).astype(np.uint8))
    mega = b" ".join(voc[int(i)] for i in rng.integers(0, 50, 150_000))[: 1 << 20]
    docs += [b"", b"\x80\x81\xfe\xff", b"...,,, --", b"A a B b Ab aB x", big_word, b"the " * 3000 + b"The THE",
             b"caf\xc3\xa9 na\xefve \xe2\x80\x9cquoted\xe2\x80\x9d", mega, b"\x00\x00word\x00", b"ab ab ab"]
    queries = B.gen_queries(3, voc, 990) + [b"", b"\xff\xfe", b"the the THE", b"zqxjvwkp", b"abzqx qqqq", big_word[:5000],
                                            b"the", b"a b ab", b"CAF\xc3\x89", b"word"]
    cfg = B.Config()
    D = _check(cfg, docs, queries, k=20, postings_of=[b"the", b"ab", b"a", big_word[:10], b"word"])
    assert D.stats()["pruned"] > 0


@pytest.mark.parametrize("n,ratio", [(5, 0.4), (1, 0.5), (4, 0.5), (9, 1.0 / 3.0), (6, 1e-9)])
def test_prune_boundary(n, ratio):
    """df == df_max stays, df_max + 1 goes; n = 1 drops every n-gram"""
    base = [b"abcd", b"abcd xyzw", b"xyzw", b"xyzw", b"abcd", b"xyzw efgh", b"efgh", b"abcd", b"xyzw"]
    docs = base[:n]
    queries = [b"abcd", b"xyzw", b"efgh abcd", b"bcdq", b"zzzz"]
    for gamma in (0.0, 5.0):
        _check(B.Config(prune_ratio=ratio, gamma=gamma), docs, queries, k=3, postings_of=[b"abcd", b"xyzw"])


def test_topk_ties_by_document():
    """identical documents score identically: the top-k takes them by document index"""
    docs = [b"red green", b"blue", b"red green", b"red green", b"green red", b"red", b"", b"red green"] * 40
    _check(B.Config(), docs, [b"red green", b"red", b"blue"], k=50)
    _check(B.Config(variant=B.ATIRE), docs, [b"red green", b"red", b"blue"], k=50)


def test_unsupported_variant_and_arguments():
    with pytest.raises(Y.YamsB200Error) as e:
        Y.Bm25Index([b"x"], variant=1)
    assert e.value.status == 5
    D = Y.Bm25Index([b"x y"])
    with pytest.raises(Y.YamsB200Error) as e:
        D.score([b"x"], k=4097)
    assert e.value.status == 1


def test_200k_documents():
    docs, voc = B.gen_corpus(2024, 200_000, 8, 20_000)
    queries = B.gen_queries(8, voc, 24)
    _check(B.Config(), docs, queries, k=100, postings_of=[w.lower() for w in voc[:3]])


def test_cpp_host_adapter(tmp_path):
    """B200Bm25Index (the stand-in for simeon::Bm25Index in SimeonLexicalBackend) over the C ABI against the restatement"""
    exe = str(tmp_path / "test_bm25")
    subprocess.check_call(["/usr/bin/g++", "-std=c++20", "-O1", os.path.join(ROOT, "tests", "host_cpp", "test_bm25.cpp"),
                           "-o", exe, "-L" + os.path.join(ROOT, "yams_b200"), "-lyams_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "yams_b200")])
    docs, voc = B.gen_corpus(31, 300, 20, 400)
    queries = B.gen_queries(32, voc, 16) + [b""]
    terms = [voc[0], voc[1].lower(), voc[2].upper(), b"notaword", b""]

    def texts(ts):
        return np.array([len(ts)], np.uint64).tobytes() + b"".join(np.array([len(t)], np.uint64).tobytes() + t for t in ts)

    for variant in (B.SAB, B.ATIRE):
        path = tmp_path / f"in{variant}.bin"
        path.write_bytes(np.array([variant], np.uint32).tobytes() + texts(docs) + texts(queries) + texts(terms))
        out = subprocess.run([exe, str(path)], capture_output=True, text=True, timeout=120)
        assert out.returncode == 0 and out.stdout.endswith("ALL OK\n"), out.stdout[-500:] + out.stderr
        lines = out.stdout.split("\n")
        X = B.Index(B.Config(variant=variant), docs)
        assert lines[0].split() == [str(len(docs)), str(_bits(X.words.avg)), str(X.total_tokens)]
        assert [int(v) for v in lines[1].split()] == X.words.lengths.tolist()
        for i, q in enumerate(queries):
            assert [int(v) for v in lines[2 + i].split()] == X.score(q).view(np.uint32).tolist(), q
        for j, t in enumerate(terms):
            p = X.words.postings.get(B.hash64(t)) if t else None   # df / idf / total_tf hash the raw term
            want = (0, 0, 0) if p is None else (len(p[0]), _bits(p[2]), p[3])
            assert tuple(int(v) for v in lines[2 + len(queries) + j].split()) == want, t
