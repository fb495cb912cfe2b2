"""Document-level top-k (CandidateFilterMode::DocumentTopK) and candidate-set PQ search on the C5 corpus: 1M x 768 fp16 rows, a PQ
index with m = 32 sub-quantisers of 256 centroids, 256 queries.  Each query gets its own documents:
  uniform  500 documents x 20 rows,
  skewed   5 documents of 2000 rows + 495 documents of 2 rows.
Per call: wall time around the synchronous host call (median of 5 after 2 warm-ups) and the algorithmic bytes it must read
(exact: pairs x d x 2 B; PQ candidates: candidates x m B of codes + the reranked rows x d x 2 B; PQ documents: the indexed pairs
x d x 2 B, every one is reranked).  The exact mode's answers are compared with search_all_matching per query + grouping on the
host (what an adapter without the document entry would do), which is timed as well.  Prints the card, its power limit and
one JSON line per measurement."""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import yams_b200 as Y
from oracle import oracle as O

N, D, Q, K, M, KC = 1_000_000, 768, 256, 10, 32, 256


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def timed(fn, reps=5, warm=2):
    for _ in range(warm):
        r = fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        r = fn()
        ts.append(time.perf_counter() - t0)
    return r, float(np.median(ts)) * 1e3


def host_grouped(c, queries, docs, k, threshold):
    """search_all_matching per query + retainBestRecordPerDocument on the host"""
    nq = len(docs)
    out_d = np.full((nq, k), -1, np.int64)
    out_r = np.full((nq, k), -1, np.int64)
    out_s = np.zeros((nq, k), np.float32)
    out_c = np.zeros(nq, np.uint32)
    for q in range(nq):
        flat = np.concatenate(docs[q])
        r, s = c.search_all_matching(queries[q], threshold, allowed=flat)
        sim = dict(zip(r.tolist(), s.tolist()))
        best = []
        for di, rows in enumerate(docs[q]):
            b = None
            for rid in rows.tolist():
                v = sim.get(rid)
                if v is not None and (b is None or v > b[0]):
                    b = (v, rid)
            if b is not None:
                best.append((b[0], di, b[1]))
        best.sort(key=lambda t: (-t[0], t[1]))
        best = best[:k]
        out_c[q] = len(best)
        for i, (v, di, rid) in enumerate(best):
            out_d[q, i], out_r[q, i], out_s[q, i] = di, rid, v
    return out_d, out_r, out_s, out_c


def main():
    assert Y.plugin_init() == 0, Y.health()
    print("card, power limit:", card())
    c = Y.Corpus(D, Y.F16, Y.COSINE, capacity_hint=N)
    c.append_synthetic(42, 0, N)
    rng = np.random.default_rng(7)
    codebooks = (rng.normal(size=(M, KC, D // M)) / np.sqrt(D)).astype(np.float32).reshape(-1)
    pq = Y.PqIndex(c, M, KC, codebooks)
    queries = O.gen_rows_f32(43, 0, Q, D)
    thr = -1.0
    for case, sizes in (("uniform", [20] * 500), ("skewed", [2000] * 5 + [2] * 495)):
        docs = []
        for _ in range(Q):
            rows = rng.choice(N, size=sum(sizes), replace=False).astype(np.int64)
            cuts = np.cumsum(sizes)[:-1]
            docs.append(np.split(rows, cuts))
        pairs = Q * sum(sizes)
        # the C ABI's CSR layout, built once: the timed call is the library call
        rid = np.concatenate([np.concatenate(ds) for ds in docs])
        doffs = np.concatenate([[0], np.cumsum(np.tile(sizes, Q))]).astype(np.uint64)
        qdocs = (np.arange(Q + 1) * len(sizes)).astype(np.uint64)
        exact, ms_exact = timed(lambda: c.search_documents_csr(queries, K, rid, doffs, qdocs, threshold=thr))
        pqd, ms_pq = timed(lambda: c.search_documents_csr(queries, K, rid, doffs, qdocs, threshold=thr, pq=pq))
        exact = (np.where(exact[0] >= 0, exact[0] - qdocs[:-1, None].astype(np.int64), -1),) + tuple(exact[1:])
        assert all(np.array_equal(a, b) for a, b in zip(exact, c.search_documents(queries, K, docs, threshold=thr)))
        allowed = [np.concatenate(ds) for ds in docs]
        _, ms_cand = timed(lambda: pq.search(queries, K, rerank_factor=4, threshold=thr, allowed=allowed))
        host, ms_host = timed(lambda: host_grouped(c, queries, docs, K, thr), reps=1, warm=0)
        equal = all(np.array_equal(a, b) for a, b in zip(exact, host))
        rec = {"case": case, "queries": Q, "pairs": pairs,
               "exact_ms": round(ms_exact, 3), "exact_GBps": round(pairs * D * 2 / ms_exact / 1e6, 1),
               "pq_documents_ms": round(ms_pq, 3), "pq_documents_GBps": round(pairs * D * 2 / ms_pq / 1e6, 1),
               "pq_candidates_ms": round(ms_cand, 3),
               "pq_candidates_bytes": pairs * M + Q * K * 4 * D * 2,
               "all_matching_plus_host_grouping_ms": round(ms_host, 1),
               "exact_equals_all_matching_grouping": bool(equal),
               "pq_documents_counts_mean": float(np.mean(pqd[3]))}
        print(json.dumps(rec))
        assert equal, case
    pq.close()
    c.close()


if __name__ == "__main__":
    main()
