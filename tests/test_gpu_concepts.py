"""The word-bigram concept index on the device (yams_b200_concepts_*, yams_b200_bm25_score_blended) bit for bit: against the
stored answers of simeon's own ConceptIndex (tests/golden/ref_concepts.json) and against the restatement
(tests/concepts_restated.cpp) on the shared grid, at caps that bind with and without a tie across the cut (the replay flag),
on hostile texts and queries, concept texts that differ from the index's, batches across the query cap, score-tile edges, the
4096-wide top-k with ties, the standalone blend, and 200 000 documents."""
import hashlib
import json
import os

import numpy as np
import pytest

import yams_b200 as Y
from tests import bm25_restated as B
from tests import concepts_restated as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_concepts.json")))["cases"]


def _digest(a):
    a = np.ascontiguousarray(a)
    return a.tobytes().hex() if a.size <= 64 and a.dtype == np.float32 else "sha256:" + hashlib.sha256(a.tobytes()).hexdigest()


def _bits(x):
    return int(np.array([x], np.float32).view(np.uint32)[0])


def _index(bcfg: B.Config, docs):
    return Y.Bm25Index(docs, k1=bcfg.k1, b=bcfg.b, delta=bcfg.delta, subword_gamma=bcfg.gamma, variant=bcfg.variant,
                       ngram_min=bcfg.ngram_min, ngram_max=bcfg.ngram_max, ngram_df_prune_ratio=bcfg.prune_ratio, hash_seed=bcfg.hash_seed)


def _check(bcfg, docs, ctexts, queries, cfg, weight, k=10, concepts_of=200, X=None):
    """stats, lengths, kept hashes, concepts, blended full vectors and top-k, and the standalone blend against the restatement"""
    X = X or B.Index(bcfg, docs)
    K = R.Concepts(docs, ctexts, cfg)
    D = _index(bcfg, docs)
    C = D.mine_concepts(ctexts, **cfg.kw())
    st, ks = C.stats(), K.stats()
    for key in ("size", "doc_count", "sum_bigram_dl", "distinct", "passed_min_ttf", "accepted", "replayed"):
        assert st[key] == ks[key], (key, st[key], ks[key])
    assert _bits(st["avg_bigram_dl"]) == _bits(ks["avg_bigram_dl"])
    assert np.array_equal(C.bigram_lengths(), K.bigram_lengths())
    hs = C.hashes()
    assert np.array_equal(hs, K.hashes())
    for h in hs[:: max(1, len(hs) // concepts_of)]:
        a, b = C.find(int(h)), K.find(int(h))
        for key in a:
            if key in ("docs", "tfs"):
                assert np.array_equal(a[key], b[key]), (int(h), key)
            elif key in ("pmi", "idf"):
                assert _bits(a[key]) == _bits(b[key]), (int(h), key)
            else:
                assert a[key] == b[key], (int(h), key)
    assert C.find(12345) is None
    got = D.score(queries, k=k, concepts=C, weight=weight)
    rng = np.random.default_rng(len(docs))
    base = rng.standard_normal(len(docs)).astype(np.float32)
    for i, q in enumerate(queries):
        want = R.blended(X, K, q, weight)
        assert got["scores"][i].tobytes() == want.tobytes(), (i, q[:80])
        wd, ws = B.topk(want, k)
        c = int(got["counts"][i])
        assert c == len(wd) and np.array_equal(got["docs"][i, :c], wd) and got["topk_scores"][i, :c].tobytes() == ws.tobytes(), (i, q[:80])
        if i < 64:
            assert C.blend(q, base, weight).tobytes() == K.blend(q, base, weight).tobytes(), (i, q[:80])
    return D, C, K


@pytest.mark.parametrize("case", GOLDEN, ids=[c["name"] for c in GOLDEN])
def test_stored_answers(case):
    docs, voc, ph = R.gen_concept_corpus(case["seed"], case["n"], 30, 1500, 40, case["tie_groups"])
    queries = R.gen_concept_queries(case["seed"] + 1, voc, ph, case["nq"])
    D = _index(B.Config(variant=case["variant"]), docs)
    C = D.mine_concepts(docs, **case["config"])
    st, want = C.stats(), case["stats"]
    assert (st["size"], st["doc_count"], _bits(st["avg_bigram_dl"]), st["sum_bigram_dl"]) == \
        (want["size"], want["doc_count"], want["avg_bits"], want["sum_bigram_dl"])
    assert _digest(C.bigram_lengths()) == case["bigram_lengths"] and _digest(C.hashes()) == case["hashes"]
    for c in case["concepts"]:
        e = C.find(int(c["hash"]))
        assert (_bits(e["pmi"]), _bits(e["idf"]), str(e["a_hash"]), str(e["b_hash"]), e["total_tf"]) == \
            (c["pmi_bits"], c["idf_bits"], c["a"], c["b"], c["total_tf"])
        assert e["docs"].tolist() == c["docs"] and e["tfs"].tolist() == c["tfs"]
    got = D.score(queries, concepts=C, weight=case["weight"])["scores"]
    for i, d in enumerate(case["scores"]):
        assert _digest(got[i]) == d, i
    assert st["replayed"] == (case["name"] == "cap_tie_straddles")


@pytest.mark.parametrize("n,variant,min_ttf,floor,cap,weight", R.GRID)
def test_grid(n, variant, min_ttf, floor, cap, weight):
    docs, queries, cfg = R.grid_case(n, variant, min_ttf, floor, cap)
    _check(B.Config(variant=variant), docs, docs, queries, cfg, weight, k=7)


@pytest.mark.parametrize("tie", [True, False])
def test_cap_binds(tie):
    """planted collocations with 40 tied pairs: a cap inside the tie replays the reference's selection, one past it does not"""
    docs, voc, ph = R.gen_concept_corpus(77, 5000, 30, 3000, 60, 40)
    queries = R.gen_concept_queries(78, voc, ph, 64) + [b"tiea%d tieb%d tiea%d tieb%d" % (i, i, i + 1, i + 1) for i in range(39)]
    pm = R.Concepts(docs, docs, R.CCfg()).accepted_pmi()
    c = R.tie_cap(pm)
    assert c > 0
    if not tie:
        c = next(j for j in range(c, len(pm)) if pm[j - 1] != pm[j])
    cfg = R.CCfg(max_concepts=c)
    _, C, K = _check(B.Config(), docs, docs, queries, cfg, 0.5)
    st = C.stats()
    assert st["accepted"] > st["size"] == c and st["replayed"] == tie == K.stats()["replayed"]
    assert (C.last_timings()["replay_ms"] > 0) == tie


def test_hostile_texts_and_queries():
    """empty, one-word, word-free and >= 0x80-separated documents, a 1 MB document, a bigram with tf in the thousands; queries
    under 2 words, repeated bigrams, upper case, and bigrams of unknown words; 1 000 queries in one call"""
    rng = np.random.default_rng(9)
    docs, voc, ph = R.gen_concept_corpus(31, 3000, 20, 1000, 30, 4)
    mega = b" ".join(voc[int(i)].lower() for i in rng.integers(0, 60, 200_000))[: 1 << 20]
    docs += [b"", b"word", b"... ,,, --", b"alpha\x80beta\xffgamma\xc3\xa9delta alpha\x80beta", mega, b"red fox " * 3000,
             b"Red Fox red fox RED FOX", b"\x00red\x00fox\x00"]
    queries = R.gen_concept_queries(32, voc, ph, 990) + [b"", b"red", b"red fox red fox red fox", b"RED FOX", b"Red fox",
                                                         b"zqxj qqqq", b"alpha beta", b"red\xfffox", b"fox red", b"tiea0 tieb0"]
    _check(B.Config(), docs, docs, queries, R.CCfg(min_ttf=2), 0.5, k=20)


def test_concept_texts_differ_and_doc_count_mismatch():
    docs, voc, ph = R.gen_concept_corpus(41, 2000, 25, 900, 30, 4)
    other = [d.lower()[: len(d) // 2] for d in docs]
    queries = R.gen_concept_queries(42, voc, ph, 40)
    _check(B.Config(), other, docs, queries, R.CCfg(min_ttf=2), 0.5)
    X = B.Index(B.Config(), other)
    D, C, _ = _check(B.Config(), other, docs + [b"tiea0 tieb0"], queries, R.CCfg(min_ttf=2), 0.5, X=X)
    plain = D.score(queries)["scores"]
    assert C.stats()["size"] > 0 and np.array_equal(D.score(queries, concepts=C)["scores"].view(np.uint32), plain.view(np.uint32))
    base = np.ones(len(other), np.float32)
    assert np.array_equal(C.blend(queries[-1], base, 0.5), base)   # another length than the concept index's: no-op


def test_batches_across_the_query_cap():
    """4 101 queries in one call (batches of 4 096 + 5)"""
    docs, voc, ph = R.gen_concept_corpus(51, 3000, 20, 1000, 30, 4)
    queries = R.gen_concept_queries(52, voc, ph, 4101)
    _check(B.Config(), docs, docs, queries, R.CCfg(min_ttf=2), 0.5, k=5)


@pytest.mark.parametrize("n", [4095, 4096, 4097, 8193])
def test_score_tile_edges(n):
    docs, voc, ph = R.gen_concept_corpus(60 + n, n, 15, 800, 30, 4)
    queries = R.gen_concept_queries(61, voc, ph, 40)
    _check(B.Config(variant=B.ATIRE if n % 2 else B.SAB), docs, docs, queries, R.CCfg(min_ttf=2), 0.5, k=9)


def test_topk_4096_with_ties():
    """10 000 documents, many identical: blended scores tie across rank 4 096"""
    docs = [b"red fox jumps", b"red fox", b"blue whale", b"red fox red fox", b"fox red", b"", b"red fox jumps high"] * 1430
    queries = [b"red fox", b"red fox jumps", b"blue whale red fox", b"fox"]
    _check(B.Config(), docs[:10_000], docs[:10_000], queries, R.CCfg(min_ttf=1, pmi_floor=-1e30), 0.5, k=4096)
    _check(B.Config(variant=B.ATIRE), docs[:10_000], docs[:10_000], queries, R.CCfg(min_ttf=1, pmi_floor=-1e30), 1.0, k=4096)


def test_arguments():
    D = Y.Bm25Index([b"a b", b"a b"])
    C = D.mine_concepts([b"a b", b"a b"], min_ttf=1, pmi_floor=-1e30)
    assert C.stats()["size"] == 1
    with pytest.raises(Y.YamsB200Error) as e:
        D.score([b"a b"], k=4097, concepts=C)
    assert e.value.status == 1
    D.close()
    assert C.blend(b"a b", np.zeros(2, np.float32), 1.0)[0] > 0   # the concept index outlives its BM25 index


def test_200k_documents():
    docs, voc, ph = R.gen_concept_corpus(2024, 200_000, 8, 20_000, 400, 20)
    queries = R.gen_concept_queries(8, voc, ph, 24)
    _check(B.Config(), docs, docs, queries, R.CCfg(), 0.5, k=100, concepts_of=100)


def test_cpp_host_adapter(tmp_path):
    """B200ConceptIndex and mine_concepts (the stand-ins for simeon's in SimeonLexicalBackend) over the C ABI"""
    import subprocess
    exe = str(tmp_path / "test_concepts")
    subprocess.check_call(["/usr/bin/g++", "-std=c++20", "-O1", os.path.join(ROOT, "tests", "host_cpp", "test_concepts.cpp"),
                           "-o", exe, "-L" + os.path.join(ROOT, "yams_b200"), "-lyams_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "yams_b200")])
    docs, voc, ph = R.gen_concept_corpus(71, 300, 20, 400, 20, 3)
    queries = R.gen_concept_queries(72, voc, ph, 16) + [b""]
    K = R.Concepts(docs, docs, R.CCfg(min_ttf=2))
    hashes = [int(h) for h in K.hashes()[:5]] + [12345]

    def texts(ts):
        return np.array([len(ts)], np.uint64).tobytes() + b"".join(np.array([len(t)], np.uint64).tobytes() + t for t in ts)

    path = tmp_path / "in.bin"
    path.write_bytes(texts(docs) + texts(queries) + np.array([len(hashes)] + hashes, np.uint64).tobytes())
    out = subprocess.run([exe, str(path)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and out.stdout.endswith("ALL OK\n"), out.stdout[-500:] + out.stderr
    lines = out.stdout.split("\n")
    st = K.stats()
    assert lines[0].split() == [str(st["size"]), str(len(docs)), str(_bits(st["avg_bigram_dl"]))] and st["size"] > 0
    X = B.Index(B.Config(), docs)
    for i, q in enumerate(queries):
        assert [int(v) for v in lines[1 + 2 * i].split()] == R.blended(X, K, q, 0.5).view(np.uint32).tolist(), q
        assert [int(v) for v in lines[2 + 2 * i].split()] == K.blend(q, np.zeros(len(docs), np.float32), 1.0).view(np.uint32).tolist(), q
    for j, h in enumerate(hashes):
        e = K.find(h)
        want = ["0"] * 5 if e is None else ["1", str(_bits(e["pmi"])), str(_bits(e["idf"])), str(e["total_tf"]), str(len(e["docs"]))]
        assert lines[1 + 2 * len(queries) + j].split() == want, h
