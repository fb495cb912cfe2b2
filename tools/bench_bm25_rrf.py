"""Times reciprocal-rank fusion of BM25 variants on the device (yams_b200_bm25_score_rrf) at the lexical backend's cap: the Zipf
corpus of tools/bench_bm25.py (200 000 documents, about 256 MiB) and the backend's configuration (a SubwordAwareBackoff primary
with gamma 5, its Atire index served as a view of it, concepts mined with ConceptConfig's defaults, weight 0.5, k_rrf 60).
Prints one JSON line with the card (name, power limit, SM clock); the device memory of the SubwordAwareBackoff index, of its
Atire view and of a separately built Atire index; the RRF call for 1, 16 and 256 queries per call (full vectors to the host and
top-10 only, with and without the blend) against plain score_blended; and the reference's own score_bm25_variants_rrf
(oracle/_ref/libref_rrf.so, one CPU thread) on the same data in the same run, labelled "reference_cpu_1_thread", with its scores
compared bit for bit on 16 queries."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import yams_b200 as Y  # noqa: E402
from tests import bm25_restated as B  # noqa: E402
from tests import rrf_restated as F  # noqa: E402
from tools.bench_bm25 import card, corpus  # noqa: E402


def device_bytes():
    return int(Y.health()["device_buffer_bytes"])


def timed(fn, queries, per_call, reps=3):
    walls = []
    for _ in range(reps):
        t0 = time.perf_counter()
        for s in range(0, len(queries), per_call):
            fn(queries[s:s + per_call])
        walls.append((time.perf_counter() - t0) * 1e3 / (len(queries) // per_call))
    return round(float(np.median(walls)), 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=200_000)
    ap.add_argument("--mib", type=int, default=256)
    ap.add_argument("--no-ref", action="store_true", help="skip the reference")
    ap.add_argument("--ref-queries", type=int, default=16)
    args = ap.parse_args()
    t0 = time.perf_counter()
    docs, voc = corpus(7, args.docs, args.mib << 20)
    gen_s = time.perf_counter() - t0
    queries = B.gen_queries(11, [w.lower() for w in voc[:5000]], 512)
    res = {"card": card(), "docs": len(docs), "text_mib": round(sum(len(d) for d in docs) / 2**20, 1), "generate_s": round(gen_s, 1)}
    m0 = device_bytes()
    S = Y.Bm25Index(docs)
    m1 = device_bytes()
    t0 = time.perf_counter()
    V = S.atire_view()
    view_ms = (time.perf_counter() - t0) * 1e3
    m2 = device_bytes()
    A = Y.Bm25Index(docs, variant=Y.BM25_ATIRE)
    m3 = device_bytes()
    res["device_bytes"] = {"sab_index": m1 - m0, "atire_view": m2 - m1, "atire_build": m3 - m2}
    res["atire_view_ms"] = round(view_ms, 3)
    res["atire_build_wall_ms"] = round(A.last_timings()["build_wall_ms"], 1)
    A.close()
    C = S.mine_concepts(docs)
    res["concepts"] = int(C.stats()["size"])
    pair = [S, V]
    Y.bm25_score_rrf(pair, queries[:256], k=10, concepts=C)   # warm-up of every call shape
    S.score(queries[:256], k=10, concepts=C)
    res["ms_per_call"] = {}
    for per_call in (1, 16, 256):
        qs = queries[:max(per_call, 64)] if per_call < 256 else queries[:512]
        row = {}
        for full in (True, False):
            tag = "full" if full else "top10"
            row["rrf_blended_" + tag] = timed(lambda q: Y.bm25_score_rrf(pair, q, k=10, full=full, concepts=C), qs, per_call)
            row["rrf_plain_" + tag] = timed(lambda q: Y.bm25_score_rrf(pair, q, k=10, full=full), qs, per_call)
            row["score_blended_" + tag] = timed(lambda q: S.score(q, k=10, full=full, concepts=C), qs, per_call)
        res["ms_per_call"][str(per_call)] = row
    Y.bm25_score_rrf(pair, queries[:256], k=10, full=False, concepts=C)
    res["rrf_device_ms_256_top10_blended"] = round(S.last_timings()["score_device_ms"], 3)
    if not args.no_ref and F.have_ref():
        t0 = time.perf_counter()
        RI = [F.RefIndex(F.SAB, docs), F.RefIndex(F.ATIRE, docs)]
        ref_build_s = time.perf_counter() - t0
        rq = queries[:args.ref_queries]
        t0 = time.perf_counter()
        ref = [F.ref_score(RI, q) for q in rq]
        ref_q = (time.perf_counter() - t0) * 1e3 / len(rq)
        dev = Y.bm25_score_rrf(pair, rq)["scores"]
        res["reference_cpu_1_thread"] = {"two_builds_s": round(ref_build_s, 1), "rrf_ms_per_query": round(ref_q, 2),
                                         "device_scores_bit_identical": all(dev[i].tobytes() == ref[i].tobytes() for i in range(len(rq)))}
    C.close()
    V.close()
    S.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
