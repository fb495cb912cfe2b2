"""Times the query router on the device (yams_b200_bm25_score_routed) on the Zipf corpus of tools/bench_bm25.py (200 000
documents, about 256 MiB) with the lexical backend's configuration (SubwordAwareBackoff, gamma 5, concepts with ConceptConfig's
defaults, weight 0.5, the backend's router preset).  Prints one JSON line with the card (name, power limit, SM clock); routed
scoring for one query per call and for 256 queries with a top-10, against plain blended scoring; 256 queries with a 1 000-document
candidate pool each, the projection alone against full rows to the host plus a host gather; the recipes the queries took; and
the reference's own scoreRouted (oracle/_ref/libref_router.so, one CPU thread, over its two builds) on the same data in the same
run, labelled "reference_cpu_1_thread", with its scores and projections compared bit for bit."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import yams_b200 as Y  # noqa: E402
from tests import bm25_restated as B  # noqa: E402
from tests import router_restated as T  # noqa: E402
from tools.bench_bm25 import card, corpus  # noqa: E402
from tools.bench_bm25_rrf import timed  # noqa: E402

POOL = 1000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=200_000)
    ap.add_argument("--mib", type=int, default=256)
    ap.add_argument("--no-ref", action="store_true", help="skip the reference")
    ap.add_argument("--ref-queries", type=int, default=16)
    args = ap.parse_args()
    docs, voc = corpus(7, args.docs, args.mib << 20)
    queries = B.gen_queries(11, [w.lower() for w in voc[:5000]], 512)
    rng = np.random.default_rng(13)
    pools = [rng.integers(0, len(docs), POOL).astype(np.uint32) for _ in queries]
    res = {"card": card(), "docs": len(docs), "text_mib": round(sum(len(d) for d in docs) / 2**20, 1)}
    I = Y.Bm25Index(docs)
    C = I.mine_concepts(docs)
    # warm-up of every call shape
    I.score_routed(queries[:256], k=10, concepts=C)
    I.score_routed(queries[:256], full=False, concepts=C, candidates=pools[:256])
    I.score(queries[:256], k=10, concepts=C)
    got = I.score_routed(queries, full=False, concepts=C)
    res["recipes_of_512"] = np.bincount(got["recipe"], minlength=3).tolist()   # Bm25Atire, Bm25SabSmooth, CascadeLinearAlpha

    def gather_on_host(q):   # full rows to the host, then the pools picked there: what the projection replaces
        s = I.score_routed(q, concepts=C)["scores"]
        return [s[i][pools[i]] for i in range(len(q))]

    res["ms_per_call"] = {
        "1": {"routed_blended_full": timed(lambda q: I.score_routed(q, concepts=C), queries[:64], 1),
              "routed_blended_pool": timed(lambda q: I.score_routed(q, full=False, concepts=C, candidates=pools[:len(q)]), queries[:64], 1),
              "score_blended_full": timed(lambda q: I.score(q, concepts=C), queries[:64], 1)},
        "256": {"routed_blended_top10": timed(lambda q: I.score_routed(q, k=10, full=False, concepts=C), queries, 256),
                "score_blended_top10": timed(lambda q: I.score(q, k=10, full=False, concepts=C), queries, 256),
                f"routed_blended_pool{POOL}_projection_only": timed(
                    lambda q: I.score_routed(q, full=False, concepts=C, candidates=pools[:len(q)]), queries, 256),
                f"routed_blended_pool{POOL}_full_rows_host_gather": timed(gather_on_host, queries, 256)},
    }
    I.score_routed(queries[:256], full=False, concepts=C, candidates=pools[:256])
    t = I.last_timings()
    res["projection_only_256_device_ms"] = round(t["score_device_ms"], 3)
    I.score_routed(queries[:256], concepts=C)
    t = I.last_timings()
    res["full_rows_256_device_ms"] = round(t["score_device_ms"], 3)   # includes the rows' device-to-host copy
    if not args.no_ref and T.have_ref():
        from tests import concepts_restated as R
        t0 = time.perf_counter()
        RX = T.RefIndex(B.Config(), docs)
        RA = T.RefIndex(T.atire_of(B.Config()), docs)
        RK = T.RefConcepts(RX, docs, R.CCfg())
        out = {"builds_with_concepts_s": round(time.perf_counter() - t0, 1)}
        rq = queries[:args.ref_queries]
        t0 = time.perf_counter()
        want = [T.ref_score(RX, RA, q, T.RCfg(), RK, 0.5, pools[i]) for i, q in enumerate(rq)]
        out["scoreRouted_ms_per_query"] = round((time.perf_counter() - t0) * 1e3 / len(rq), 2)
        g = I.score_routed(rq, concepts=C, candidates=pools[:len(rq)])
        out["device_bit_identical"] = all(int(g["recipe"][i]) == w[0] and g["scores"][i].tobytes() == w[2].tobytes()
                                          and g["candidates"][i].tobytes() == w[3].tobytes() for i, w in enumerate(want))
        res["reference_cpu_1_thread"] = out
    C.close()
    I.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
