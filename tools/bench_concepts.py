"""Times the device concept index (yams_b200_concepts_*, yams_b200_bm25_score_blended) at the lexical backend's cap: the Zipf
corpus of tools/bench_bm25.py (200 000 documents, about 256 MiB) with planted two-word collocations, enough that more bigrams
pass the PMI floor than the 200 000 the cap keeps, and the backend's configuration (SubwordAwareBackoff BM25, ConceptConfig
defaults, weight 0.5).  Prints one JSON line with the card (name, power limit, SM clock), the mining call's device phases and
host part (the replay timed on its own), the blended score call against the plain one for 1, 16 and 256 queries per call
(full vectors and top-10), and the reference's own mine_concepts and score + blend_into (oracle/_ref/libref_concepts.so, one
CPU thread) on the same data in the same run, labelled "reference_cpu_1_thread"."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import yams_b200 as Y  # noqa: E402
from tests import bm25_restated as B  # noqa: E402
from tests import concepts_restated as R  # noqa: E402
from tools.bench_bm25 import card, corpus  # noqa: E402


def plant(seed, docs, voc, phrases, copies):
    """appends `copies` occurrences of each of `phrases` two-word collocations of lowercase words to random documents"""
    rng = np.random.default_rng(seed)
    low = [w for w in voc[1000:] if w == w.lower()]
    a = rng.integers(0, len(low), phrases)
    b = rng.integers(0, len(low), phrases)
    text = [low[a[i]] + b" " + low[b[i]] for i in range(phrases)]
    at = rng.integers(0, len(docs), phrases * copies)
    extra = [[] for _ in docs]
    for j, d in enumerate(at):
        extra[d].append(text[j % phrases])
    out = [d + b". " + b". ".join(e) if e else d for d, e in zip(docs, extra)]
    return out, text


def timed_calls(D, queries, per_call, full, reps, concepts):
    walls = []
    for _ in range(reps):
        t0 = time.perf_counter()
        for s in range(0, len(queries), per_call):
            D.score(queries[s:s + per_call], k=10, full=full, concepts=concepts)
        walls.append((time.perf_counter() - t0) * 1e3 / (len(queries) // per_call))
    return float(np.median(walls))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=200_000)
    ap.add_argument("--mib", type=int, default=256)
    ap.add_argument("--phrases", type=int, default=300_000)
    ap.add_argument("--no-ref", action="store_true", help="skip the reference")
    ap.add_argument("--ref-queries", type=int, default=16)
    args = ap.parse_args()
    t0 = time.perf_counter()
    docs, voc = corpus(7, args.docs, args.mib << 20)
    docs, phrases = plant(8, docs, voc, args.phrases, 6)
    gen_s = time.perf_counter() - t0
    rng = np.random.default_rng(9)
    queries = [phrases[int(i)] + b" " + phrases[int(j)] for i, j in rng.integers(0, len(phrases), (512, 2))]
    res = {"card": card(), "docs": len(docs), "text_mib": round(sum(len(d) for d in docs) / 2**20, 1), "generate_s": round(gen_s, 1)}
    D = Y.Bm25Index(docs)
    D.mine_concepts(docs[:1000]).close()   # warm-up
    mines = []
    for _ in range(2):
        t0 = time.perf_counter()
        C = D.mine_concepts(docs)
        mines.append(((time.perf_counter() - t0) * 1e3, C.last_timings()))
        if len(mines) < 2:
            C.close()
    wall, tm = mines[-1]
    st = C.stats()
    res["mine"] = {"wall_ms": round(wall, 1), "first_wall_ms": round(mines[0][0], 1), **{k: round(v, 2) for k, v in tm.items()},
                   **{k: (bool(v) if k == "replayed" else int(v) if k != "avg_bigram_dl" else float(v)) for k, v in st.items()}}
    D.score(queries[:256], k=10, concepts=C)   # warm-up of every call shape
    res["score_ms_per_call"] = {}
    for per_call in (1, 16, 256):
        qs = queries[:max(per_call, 64)] if per_call < 256 else queries[:512]
        res["score_ms_per_call"][str(per_call)] = {
            "blended_full": round(timed_calls(D, qs, per_call, True, 3, C), 3), "plain_full": round(timed_calls(D, qs, per_call, True, 3, None), 3),
            "blended_top10": round(timed_calls(D, qs, per_call, False, 3, C), 3), "plain_top10": round(timed_calls(D, qs, per_call, False, 3, None), 3)}
    if not args.no_ref and R.have_ref():
        F = R.RefConcepts(B.Config(), docs, docs, R.CCfg())
        rq = queries[:args.ref_queries]
        t0 = time.perf_counter()
        ref_scores = [F.score_blended(q, 0.5) for q in rq]
        ref_q = (time.perf_counter() - t0) * 1e3 / len(rq)
        dev = D.score(rq, concepts=C)["scores"]
        same = all(dev[i].tobytes() == ref_scores[i].tobytes() for i in range(len(rq)))
        res["reference_cpu_1_thread"] = {"mine_ms": round(F.mine_ms(), 1), "score_plus_blend_ms_per_query": round(ref_q, 2),
                                         "size": F.stats()["size"], "kept_hashes_identical": bool(np.array_equal(F.hashes(), C.hashes())),
                                         "device_scores_bit_identical": same}
    C.close()
    D.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
