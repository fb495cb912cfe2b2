"""Writes tests/golden/ref_concepts.json: the answers of simeon's own ConceptIndex (oracle/_ref/libref_concepts.so, built by
oracle/concepts.mk from the reference tree) on generated corpora with planted collocations.  Run from the repository root:
    python tests/golden/make_concepts_golden.py
Each case records its configuration, the stats, a digest of the bigram lengths and of the sorted kept hashes, some concepts in
full (pmi / idf bits, a / b, total_tf, postings) and the blended score vector of every query (bits, or SHA-256 above 64
documents)."""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import bm25_restated as B  # noqa: E402
from tests import concepts_restated as R  # noqa: E402


def digest(a):
    a = np.ascontiguousarray(a)
    return a.tobytes().hex() if a.size <= 64 and a.dtype == np.float32 else "sha256:" + hashlib.sha256(a.tobytes()).hexdigest()


def bits(x):
    return int(np.array([x], np.float32).view(np.uint32)[0])


# name, seed, n, variant, ConceptConfig overrides, tie groups, weight, queries
CASES = [
    ("default_sab", 11, 1000, B.SAB, {}, 0, 0.5, 24),
    ("default_atire", 12, 1000, B.ATIRE, {}, 0, 0.5, 24),
    ("cap_tie_straddles", 13, 1000, B.SAB, {"max_concepts": 15}, 30, 0.5, 24),
    ("cap_no_tie", 13, 1000, B.SAB, {"max_concepts": 30}, 30, 0.5, 24),
    ("min_ttf_1_floor_0", 14, 300, B.SAB, {"min_ttf": 1, "pmi_floor": 0.0}, 0, 1.0, 16),
    ("small_n", 15, 40, B.ATIRE, {"min_ttf": 1}, 0, -0.5, 16),
]


def case(name, seed, n, variant, over, ties, weight, nq):
    docs, voc, ph = R.gen_concept_corpus(seed, n, 30, 1500, 40, ties)
    queries = R.gen_concept_queries(seed + 1, voc, ph, nq)
    cfg = R.CCfg(**over)
    F = R.RefConcepts(B.Config(variant=variant), docs, docs, cfg)
    st = F.stats()
    hs = F.hashes()
    sample = []
    for h in list(hs[:4]) + list(hs[-2:]):
        e = F.find(int(h))
        sample.append({"hash": str(int(h)), "pmi_bits": bits(e["pmi"]), "idf_bits": bits(e["idf"]), "a": str(e["a_hash"]),
                       "b": str(e["b_hash"]), "total_tf": e["total_tf"], "docs": e["docs"].tolist(), "tfs": e["tfs"].tolist()})
    return {"name": name, "seed": seed, "n": n, "variant": variant, "config": cfg.kw(), "tie_groups": ties, "weight": weight, "nq": nq,
            "stats": {"size": st["size"], "doc_count": st["doc_count"], "avg_bits": bits(st["avg_bigram_dl"]),
                      "sum_bigram_dl": st["sum_bigram_dl"]},
            "bigram_lengths": digest(F.bigram_lengths()), "hashes": digest(hs), "concepts": sample,
            "scores": [digest(F.score_blended(q, weight)) for q in queries]}


def main():
    assert R.have_ref(), "oracle/_ref/libref_concepts.so is missing: build it with make -f oracle/concepts.mk"
    out = {"source": "simeon ConceptIndex (third_party/simeon/src/concept_mining.cpp) over Bm25Index, via oracle/concepts.mk",
           "cases": [case(*c) for c in CASES]}
    with open(os.path.join(ROOT, "tests", "golden", "ref_concepts.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
