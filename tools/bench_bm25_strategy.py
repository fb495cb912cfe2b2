"""Times the lead-text field and the strategy router's BM25F strategies on the device (yams_b200_bm25_build_lead,
yams_b200_bm25_score_strategy) on the Zipf corpus of tools/bench_bm25.py (200 000 documents, about 256 MiB) with the lexical
backend's configuration (SubwordAwareBackoff, gamma 5, lead length 64, concepts with ConceptConfig's defaults, weight 0.5).
Prints one JSON line with the card (name, power limit, SM clock); the build's wall time and device memory with and without
the lead field; Bm25Strategy (pool 0), KeyphraseStrategy (pool 1), LeadFieldStrategy (pool 2) and the routed choice for 1, 16
and 256 queries per call (full vectors to the host and top-10 only) against plain blended scoring, with the z-score kernel's
device time; and the reference's own build and strategies (oracle/_ref/
libref_strategy.so, one CPU thread) on the same data in the same run, labelled "reference_cpu_1_thread", with its scores
compared bit for bit on 16 queries."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import yams_b200 as Y  # noqa: E402
from tests import bm25_restated as B  # noqa: E402
from tests import strategy_restated as S  # noqa: E402
from tools.bench_bm25 import card, corpus  # noqa: E402
from tools.bench_bm25_rrf import device_bytes, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=200_000)
    ap.add_argument("--mib", type=int, default=256)
    ap.add_argument("--no-ref", action="store_true", help="skip the reference")
    ap.add_argument("--ref-queries", type=int, default=16)
    args = ap.parse_args()
    docs, voc = corpus(7, args.docs, args.mib << 20)
    queries = B.gen_queries(11, [w.lower() for w in voc[:5000]], 512)
    res = {"card": card(), "docs": len(docs), "text_mib": round(sum(len(d) for d in docs) / 2**20, 1)}
    Y.Bm25Index(docs[:1000], lead_tokens=64).close()   # warm-up of the build's kernels
    res["build"] = {}
    for lead in (0, 64):
        m0 = device_bytes()
        t0 = time.perf_counter()
        I = Y.Bm25Index(docs, lead_tokens=lead)
        call_ms = (time.perf_counter() - t0) * 1e3
        t = I.last_timings()
        # call_ms: the Python call, texts to ctypes arrays included (tools/bench_bm25.py's "build wall"); build_ms: the library's
        # own wall time of the build (last_timings [4]); the device split from CUDA events
        res["build"][f"lead_{lead}"] = {"device_bytes": device_bytes() - m0, "call_ms": round(call_ms, 1), "build_ms": round(t["build_wall_ms"], 1),
                                        "device_upload_tokenise_sort_postings_ms": [round(t[k], 1) for k in ("build_upload_ms", "build_tokenise_ms",
                                                                                                          "build_sort_ms", "build_postings_ms")]}
        if lead:
            res["aux_stats"] = {k: (float(v) if k.endswith("dl") else v) for k, v in I.aux_stats().items()}
            L = I
        else:
            I.close()
    C = L.mine_concepts(docs)
    for p in (0, 1, 2, 3):
        L.score_strategy(queries[:256], p, k=10, concepts=C)   # warm-up of every call shape
    L.score(queries[:256], k=10, concepts=C)
    res["ms_per_call"] = {}
    for per_call in (1, 16, 256):
        qs = queries[:max(per_call, 64)] if per_call < 256 else queries[:512]
        row = {}
        for full in (True, False):
            tag = "full" if full else "top10"
            for p, name in ((0, "bm25_pool0"), (1, "keyphrase_pool1"), (2, "lead_field_pool2"), (3, "routed")):
                row[f"{name}_blended_{tag}"] = timed(lambda q: L.score_strategy(q, p, k=10, full=full, concepts=C), qs, per_call)
            row["score_blended_" + tag] = timed(lambda q: L.score(q, k=10, full=full, concepts=C), qs, per_call)
        res["ms_per_call"][str(per_call)] = row
    for p, name in ((0, "pool0"), (1, "pool1"), (2, "pool2"), (3, "routed")):
        L.score_strategy(queries[:256], p, k=10, full=False, concepts=C)
        st = L.strategy_stats()
        res[f"{name}_256_top10_blended"] = {"device_ms": round(st["device_ms"], 3), "zscore_ms": round(st["zscore_ms"], 3),
                                            "queries_per_pool": st["queries"], "keyphrase_boosted": st["keyphrase_boosted"],
                                            "replayed": st["replayed"]}
    if not args.no_ref and S.have_ref():
        from tests import concepts_restated as R
        t0 = time.perf_counter()
        ref = S.RefStrategy(B.Config(), docs, 64, R.CCfg())
        build_s = time.perf_counter() - t0
        rq = queries[:args.ref_queries]
        out = {"build_with_concepts_s": round(build_s, 1)}
        ok = True
        for p in (0, 1, 2, 3):
            t0 = time.perf_counter()
            want = [ref.score(p, q, 0.5) for q in rq]
            out[f"pool{p}_ms_per_query"] = round((time.perf_counter() - t0) * 1e3 / len(rq), 2)
            got = L.score_strategy(rq, p, concepts=C, weight=0.5)["scores"]
            ok = ok and all(got[i].tobytes() == want[i].tobytes() for i in range(len(rq)))
        out["device_scores_bit_identical"] = ok
        res["reference_cpu_1_thread"] = out
        ref.close()
    C.close()
    L.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
