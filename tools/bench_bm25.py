"""Times the device BM25 index (yams_b200_bm25_*) at the lexical backend's cap: a synthetic Zipf-distributed corpus of 200 000
documents and about 256 MiB of text, the backend's configuration (SubwordAwareBackoff, gamma 5, n-grams 3..4).  Prints one JSON
line with the card (name, power limit, SM clock), the build's wall time and device split, the score call's wall time for 1, 16
and 256 queries per call (full score vectors to the host, as the backend uses them, and top-10 only), the posting bytes a query
reads with that traffic as a share of HBM bandwidth, and the reference's own Bm25Index (oracle/_ref/libref_bm25.so, one CPU
thread) built and scoring the same data in the same run, labelled "reference_cpu_1_thread"."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import yams_b200 as Y  # noqa: E402
from tests import bm25_restated as B  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def corpus(seed, n, target_bytes, vocab=100_000):
    """n documents of Zipf(1.1) words over a vocabulary of 2..12-letter words (some capitalised), with punctuation"""
    rng = np.random.default_rng(seed)
    lens = rng.integers(2, 13, vocab)
    letters = rng.integers(97, 123, int(lens.sum())).astype(np.uint8)
    offs = np.concatenate([[0], np.cumsum(lens)])
    voc = [bytes(letters[offs[i]:offs[i + 1]]) for i in range(vocab)]
    for i in rng.integers(0, vocab, vocab // 10):
        voc[i] = voc[i].capitalize()
    mean_words = target_bytes / n / 9.7   # ~9.7 bytes per word and separator
    sizes = np.maximum(1, rng.poisson(mean_words, n))
    ids = np.minimum(rng.zipf(1.1, int(sizes.sum())) - 1, vocab - 1)
    seps = [b" ", b" ", b" ", b", ", b". "]
    docs, at = [], 0
    for s in sizes:
        docs.append(seps[at % 5].join(voc[i] for i in ids[at:at + s]))
        at += s
    return docs, voc


def query_bytes(D, cfg, q):
    """bytes of postings (document + tf) and document lengths the query's legs read"""
    idx = B.Index.__new__(B.Index)
    idx.cfg = cfg
    idx._hash, idx._grams = {}, {}
    total = 0
    for t in B.words(q):
        docs, _, _, _ = D.postings(0, idx.h(t))
        df = len(docs)
        alpha = np.float32(df) / (np.float32(df) + np.float32(cfg.gamma)) if df else np.float32(0)
        if alpha > 0:
            total += df * 12
        if alpha < 1:
            for g in dict.fromkeys(idx.gram_hashes(t)):
                total += len(D.postings(1, g)[0]) * 12
    return total


def timed_calls(D, queries, per_call, full, reps):
    walls = []
    for _ in range(reps):
        t0 = time.perf_counter()
        for s in range(0, len(queries), per_call):
            D.score(queries[s:s + per_call], k=10, full=full)
        walls.append((time.perf_counter() - t0) * 1e3 / (len(queries) // per_call))
    return float(np.median(walls))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=200_000)
    ap.add_argument("--mib", type=int, default=256)
    ap.add_argument("--no-ref", action="store_true", help="skip the reference build")
    ap.add_argument("--ref-queries", type=int, default=16)
    args = ap.parse_args()
    t0 = time.perf_counter()
    docs, voc = corpus(7, args.docs, args.mib << 20)
    gen_s = time.perf_counter() - t0
    nbytes = sum(len(d) for d in docs)
    queries = B.gen_queries(11, [w.lower() for w in voc[:5000]], 512)
    cfg = B.Config()
    res = {"card": card(), "docs": len(docs), "text_mib": round(nbytes / 2**20, 1), "generate_s": round(gen_s, 1)}
    Y.Bm25Index(docs[:1000]).close()   # warm-up: module load, allocator
    builds = []
    for _ in range(2):
        t0 = time.perf_counter()
        D = Y.Bm25Index(docs)
        builds.append(((time.perf_counter() - t0) * 1e3, D.last_timings()))
        if len(builds) < 2:
            D.close()
    wall, tm = builds[-1]
    st = D.stats()
    res["build"] = {"wall_ms": round(wall, 1), "upload_ms": round(tm["build_upload_ms"], 1), "tokenise_ms": round(tm["build_tokenise_ms"], 1),
                    "sort_ms": round(tm["build_sort_ms"], 1), "postings_ms": round(tm["build_postings_ms"], 1), "slices": tm["build_slices"],
                    "first_wall_ms": round(builds[0][0], 1), "terms": list(st["terms"]), "postings": list(st["postings"]),
                    "pruned": st["pruned"], "avg_dl": float(st["avg_dl"])}
    D.score(queries[:256], k=10)   # warm-up of every call shape
    res["score_ms_per_call"] = {}
    for per_call in (1, 16, 256):
        qs = queries[:max(per_call, 64)] if per_call < 256 else queries[:512]
        res["score_ms_per_call"][str(per_call)] = {"full_vectors": round(timed_calls(D, qs, per_call, True, 3), 3),
                                                   "top10_only": round(timed_calls(D, qs, per_call, False, 3), 3)}
    qb = [query_bytes(D, cfg, q) for q in queries[:64]]
    per_q = float(np.mean(qb))
    t_256 = res["score_ms_per_call"]["256"]["top10_only"] / 256 / 1e3
    res["posting_bytes_per_query_mean"] = round(per_q)
    res["posting_read_share_of_hbm_at_256_per_call"] = round(per_q / t_256 / HBM_BYTES_PER_S, 4)
    # the scores of a sample against the restatement is the tests' job; here the reference itself is timed and compared
    if not args.no_ref and B.have_ref():
        t0 = time.perf_counter()
        R = B.RefIndex(cfg, docs)
        ref_build = (time.perf_counter() - t0) * 1e3
        rq = queries[:args.ref_queries]
        t0 = time.perf_counter()
        ref_scores = [R.score(q) for q in rq]
        ref_q = (time.perf_counter() - t0) * 1e3 / len(rq)
        dev = D.score(rq)["scores"]
        same = all(dev[i].tobytes() == ref_scores[i].tobytes() for i in range(len(rq)))
        res["reference_cpu_1_thread"] = {"build_ms": round(ref_build, 1), "score_ms_per_query": round(ref_q, 2),
                                         "device_scores_bit_identical": same}
        R.close()
    D.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
