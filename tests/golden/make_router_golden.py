"""Writes tests/golden/ref_router.json: the answers of simeon's own QueryRouter and the lexical backend's routed dispatch
(oracle/_ref/libref_router.so, built by oracle/router.mk from the reference tree) over its own Bm25Index (a SubwordAwareBackoff
primary beside an Atire index, or an Atire primary alone) and, blended, its own ConceptIndex mined against the primary
(min_ttf 2).  Run from the repository root:
    python tests/golden/make_router_golden.py
Each case (tests/router_restated.py CASES) records per blend weight (None: plain) and query the recipe, the features (float
bits; n_terms as is), and the score row and candidate projection (bits, or SHA-256 above 64 values)."""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import concepts_restated as R  # noqa: E402
from tests import router_restated as T  # noqa: E402

CCFG = R.CCfg(min_ttf=2)


def digest(a):
    a = np.ascontiguousarray(a)
    return a.tobytes().hex() if a.size <= 64 and a.dtype == np.float32 else "sha256:" + hashlib.sha256(a.tobytes()).hexdigest()


def feature_bits(f):
    return [int(f[k]) if k == "n_terms" else int(np.float32(f[k]).view(np.uint32)) for k in T.FEATURES]


def case(name, seed, n, variant, overrides):
    docs, queries, cfg, rcfg = T.case_inputs(name, seed, n, variant, overrides)
    X = T.RefIndex(cfg, docs)
    A = T.RefIndex(T.atire_of(cfg), docs) if T.atire_of(cfg) else None
    K = T.RefConcepts(X, docs, CCFG)
    out = {"name": name, "seed": seed, "n": n, "variant": variant, "router": overrides, "answers": {}}
    for w in (None, 0.5):
        rows = []
        for i, q in enumerate(queries):
            r, f, row, proj = T.ref_score(X, A, q, rcfg, K if w is not None else None, w or 0.0, T.pool(seed, n, i))
            rows.append({"recipe": r, "features": feature_bits(f), "scores": digest(row), "pool": digest(proj)})
        out["answers"][str(w)] = rows
    return out


def main():
    assert T.have_ref(), "oracle/_ref/libref_router.so is missing: build it with make -f oracle/router.mk"
    out = {"source": "simeon QueryRouter (third_party/simeon/src/query_router.cpp) and scoreRouted's dispatch over Bm25Index and "
                     "ConceptIndex, via oracle/router.mk", "concept_config": CCFG.kw(), "cases": [case(*c) for c in T.CASES]}
    with open(os.path.join(ROOT, "tests", "golden", "ref_router.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
