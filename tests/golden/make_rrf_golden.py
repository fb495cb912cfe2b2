"""Writes tests/golden/ref_rrf.json: the answers of simeon's own score_bm25_variants_rrf (oracle/_ref/libref_rrf.so, built by
oracle/rrf.mk from the reference tree), over its own Bm25Index variants and, blended, its own ConceptIndex mined against the
first variant (min_ttf 2).  Run from the repository root:
    python tests/golden/make_rrf_golden.py
Each case records its corpus, variants, k_rrf values and blend weights, and per (k_rrf, weight) the fused score vector of every
query (bits, or SHA-256 above 64 documents)."""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import concepts_restated as R  # noqa: E402
from tests import rrf_restated as F  # noqa: E402

CCFG = R.CCfg(min_ttf=2)

# name, corpus, seed, n, variants, k_rrf values, blend weights (None: plain), queries
CASES = [
    ("sab_atire", "concepts", 101, 800, ["sab", "atire"], [60.0, 0.0, 1.5, 1e6], [None, 0.5], "concepts", 24),
    ("three_configs", "concepts", 102, 800, ["sab", "atire", "other"], [60.0, 1.5], [None, 0.5], "concepts", 24),
    ("same_index_twice", "concepts", 103, 500, ["sab", "sab"], [60.0], [None, 0.5], "concepts", 16),
    ("one_variant", "concepts", 104, 500, ["atire"], [60.0], [None, 0.5], "concepts", 16),
    ("zero_variants", "concepts", 105, 300, [], [60.0], [None], "concepts", 8),
    ("score_ties", "ties", 106, 1000, ["sab", "atire", "other"], [60.0, 0.0], [None, 0.5], "concepts", 24),
    ("ngram_only", "concepts", 107, 800, ["sab", "atire"], [60.0], [None, 0.5], "ngram", 24),
    ("matches_nothing", "catch2", 0, 2, ["sab", "atire"], [60.0], [None], "catch2", 1),
]


def digest(a):
    a = np.ascontiguousarray(a)
    return a.tobytes().hex() if a.size <= 64 and a.dtype == np.float32 else "sha256:" + hashlib.sha256(a.tobytes()).hexdigest()


def case(name, corpus, seed, n, variants, ks, weights, queries, nq):
    c = {"name": name, "corpus": corpus, "seed": seed, "n": n, "variants": variants, "k_rrf": ks, "weights": weights,
         "queries": queries, "nq": nq}
    docs, qs, cfgs = F.case_inputs(c)
    ixs = [F.RefIndex(cfg, docs) for cfg in cfgs]
    K = F.RefConcepts(ixs[0] if ixs else F.RefIndex(F.SAB, docs), docs, CCFG) if any(w is not None for w in weights) else None
    c["scores"] = [{"k_rrf": k, "weight": w,
                    "digests": [digest(F.ref_score(ixs, q, k, K if w is not None else None, w or 0.0, n=len(docs))) for q in qs]}
                   for k in ks for w in weights]
    return c


def main():
    assert F.have_ref(), "oracle/_ref/libref_rrf.so is missing: build it with make -f oracle/rrf.mk"
    out = {"source": "simeon score_bm25_variants_rrf (third_party/simeon/src/fusion.cpp) over Bm25Index and ConceptIndex, via "
                     "oracle/rrf.mk", "concept_config": CCFG.kw(), "cases": [case(*c) for c in CASES]}
    with open(os.path.join(ROOT, "tests", "golden", "ref_rrf.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
