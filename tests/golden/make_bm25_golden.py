"""Writes tests/golden/ref_bm25.json: what simeon's own Bm25Index (oracle/_ref/libref_bm25.so, built by oracle/bm25.mk) answers
on generated corpora and queries, for the tests that run where the reference build does not exist.  Score vectors are stored
as raw float bits (hex) up to 64 documents and as SHA-256 digests of the bits above; stats, df / idf bits / total_tf of sampled
words and n-grams, and the number of n-grams pruned (the index built again without pruning, minus the index).
Run from the repository root: python tests/golden/make_bm25_golden.py"""
import hashlib
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tests import bm25_restated as B  # noqa: E402

# (name, variant, corpus seed, n docs, mean words, vocabulary, ngram range, gamma, prune ratio, queries)
CASES = [
    ("sab_default_1000", B.SAB, 1, 1000, 40, 3000, (3, 4), 5.0, 0.5, 64),
    ("atire_1000", B.ATIRE, 1, 1000, 40, 3000, (3, 4), 5.0, 0.5, 64),
    ("sab_small_3", B.SAB, 2, 3, 8, 30, (3, 4), 5.0, 0.5, 24),
    ("sab_one_doc", B.SAB, 3, 1, 20, 50, (3, 4), 5.0, 0.5, 16),
    ("sab_gamma0_unigrams", B.SAB, 4, 200, 20, 400, (1, 1), 0.0, 0.5, 32),
    ("sab_wide_ngrams_noprune", B.SAB, 5, 300, 30, 800, (2, 8), 1e-3, 0.0, 32),
    ("sab_big_gamma_tiny_prune", B.SAB, 6, 500, 25, 600, (3, 4), 1e6, 1e-3, 32),
    ("atire_empty", B.ATIRE, 7, 0, 10, 10, (3, 4), 5.0, 0.5, 4),
    ("sab_two_docs", B.SAB, 8, 2, 12, 20, (3, 4), 5.0, 0.5, 16),
]


def _bits(a):
    return a.astype(np.float32).view(np.uint32)


def vec_digest(a):
    return a.astype(np.float32).tobytes().hex() if a.size <= 64 else "sha256:" + hashlib.sha256(a.astype(np.float32).tobytes()).hexdigest()


def main():
    out = []
    for name, variant, seed, n, mw, voc_n, (kmin, kmax), gamma, ratio, nq in CASES:
        docs, voc = B.gen_corpus(seed, n, mw, voc_n)
        cfg = B.Config(variant=variant, ngram_min=kmin, ngram_max=kmax, gamma=gamma, prune_ratio=ratio)
        R = B.RefIndex(cfg, docs)
        queries = B.gen_queries(seed + 100, voc, nq)
        st = R.stats()
        unpruned = B.RefIndex(B.Config(variant=variant, ngram_min=kmin, ngram_max=kmax, gamma=gamma, prune_ratio=0.0), docs).stats()
        words = [w.lower() for w in voc[:40]] + [b"zzzznotaword"]
        terms = []
        for w in words:
            df, idf, ttf = R.term(w)
            terms.append([w.decode(), df, int(_bits(np.array([idf]))[0]), ttf])
        grams = []
        if variant == B.SAB:
            for w in words[:10]:
                for g in B.ngrams(w, kmin, kmax)[:3]:
                    h = R.hash(g)
                    d, t, idf, ttf = R.postings(1, h)
                    grams.append([g.decode(), len(d), int(_bits(np.array([idf]))[0]), ttf])
        out.append({
            "name": name, "variant": variant, "seed": seed, "n": n, "mean_words": mw, "vocab": voc_n, "ngram_min": kmin,
            "ngram_max": kmax, "gamma": gamma, "prune_ratio": ratio, "nq": nq,
            "stats": {"n_docs": st["n_docs"], "avg_dl_bits": int(_bits(np.array([st["avg_dl"]]))[0]),
                      "ngram_avg_dl_bits": int(_bits(np.array([st["ngram_avg_dl"]]))[0]), "total_tokens": st["total_tokens"],
                      "terms": list(st["terms"]), "postings": list(st["postings"]),
                      "pruned": unpruned["terms"][1] - st["terms"][1]},
            "doc_lengths": vec_digest(R.doc_lengths(0).view(np.float32)),
            "scores": [vec_digest(R.score(q)) for q in queries],
            "terms": terms, "ngrams": grams,
        })
        R.close()
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_bm25.json")
    with open(path, "w") as f:
        json.dump({"generator": "tests/golden/make_bm25_golden.py", "cases": out}, f, indent=0)
        f.write("\n")
    print("wrote", path, len(out), "cases")


if __name__ == "__main__":
    main()
