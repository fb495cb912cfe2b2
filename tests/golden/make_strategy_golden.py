"""Writes tests/golden/ref_strategy.json: the answers of simeon's own lead-text field and BM25F strategies
(oracle/_ref/libref_strategy.so, built by oracle/strategy.mk from the reference tree): extract_lead_tokens of generated texts,
and, per case, the aux fields' statistics and every query's score vector from Bm25Strategy (pool 0), KeyphraseStrategy (pool 1),
LeadFieldStrategy (pool 2) and the backend's entropy route over them (3, with the pool it chose), plain and blended with a
ConceptIndex mined against the index (min_ttf 2, weight 0.5).  Run from the repository root:
    python tests/golden/make_strategy_golden.py
Score vectors are stored as bits, or SHA-256 above 64 documents."""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import bm25_restated as B  # noqa: E402
from tests import concepts_restated as R  # noqa: E402
from tests import strategy_restated as S  # noqa: E402

CCFG = R.CCfg(min_ttf=2)
# name, corpus seed, documents, variant, lead tokens, queries
CASES = [
    ("sab_lead64", 201, 600, "sab", 64, 24),
    ("atire_lead64", 202, 600, "atire", 64, 24),
    ("sab_lead3", 203, 300, "sab", 3, 16),
    ("sab_no_lead", 204, 300, "sab", 0, 12),
    ("atire_no_lead", 205, 300, "atire", 0, 12),
    ("all_leads_empty", 206, 40, "sab", 64, 8),
    ("one_doc", 207, 1, "sab", 64, 8),
    ("concepts", 208, 800, "sab", 64, 24),          # queries of mined concepts: the blend changes the strategies' scores
    ("concepts_atire", 209, 800, "atire", 64, 24),
    ("few_matches", 210, 60, "sab", 64, 8),         # words in 3 identical documents: the top-10's zero padding decides the gate
    ("many_docs", 211, 4097, "sab", 64, 24),        # z-scores over 4 097 documents: the order of the sums shows
]
VARIANTS = {"sab": B.SAB, "atire": B.ATIRE}


def digest(a):
    a = np.ascontiguousarray(a)
    return a.tobytes().hex() if a.size <= 64 and a.dtype == np.float32 else "sha256:" + hashlib.sha256(a.tobytes()).hexdigest()


def case_inputs(c):
    """the case's documents and queries (all_leads_empty: whitespace-only and empty documents)"""
    if c["name"].startswith("concepts"):
        docs, voc, ph = R.gen_concept_corpus(c["seed"], c["n"])
        return docs, R.gen_concept_queries(c["seed"] + 1000, voc, ph, c["nq"]) + [b"the of and", b"Zeta zeta's"]
    docs, voc = S.gen_lead_corpus(c["seed"], c["n"])
    if c["name"] == "all_leads_empty":
        docs = [S.WS[i % len(S.WS)] * (i % 3) for i in range(c["n"])]
    if c["name"] == "few_matches":
        docs = docs[:c["n"] - 3] + [b"zeta omega kappa"] * 3
        return docs, [b"zeta", b"Zeta kappa", b"omega the", b"kappa zeta omega", b"a an the", b"zz", b"", b"zeta?"]
    return docs, S.gen_lead_queries(c["seed"] + 1000, voc, c["nq"])


def main():
    assert S.have_ref(), "oracle/_ref/libref_strategy.so is missing: make -f oracle/strategy.mk"
    texts, _ = S.gen_lead_corpus(200, 200)
    leads = [{"L": L, "cuts": [len(S.ref_lead(t, L)) for t in texts], "digest": hashlib.sha256(b"\0".join(S.ref_lead(t, L) for t in texts)).hexdigest()}
             for L in (1, 2, 5, 64)]
    out = {"concept_config": vars(CCFG), "lead_corpus_seed": 200, "lead_corpus_n": 200, "leads": leads, "cases": []}
    for name, seed, n, var, lead, nq in CASES:
        c = {"name": name, "seed": seed, "n": n, "variant": var, "lead": lead, "nq": nq}
        docs, queries = case_inputs(c)
        X = S.RefStrategy(B.Config(variant=VARIANTS[var]), docs, lead, CCFG)
        c["aux"] = [{k: (float(v) if k == "avg" else v) for k, v in X.field_stats(f).items()} for f in (2, 3)]
        c["scores"] = {f"{pool}/{w}": [digest(X.score(pool, q, w)) for q in queries] for pool in (0, 1, 2, 3) for w in (None, 0.5)}
        c["routed"] = [X.score(3, q, None, chosen=True)[1] for q in queries]
        out["cases"].append(c)
    with open(os.path.join(ROOT, "tests", "golden", "ref_strategy.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
