"""Write tests/golden/ref_pq_candidates.json by EXECUTING THE REFERENCE: for the corpora and candidate lists of
tests/test_gpu_documents.pq_candidates_case (fp32 and fp16) and pq_order_case, simeon's own encode and ADC scores (oracle/_ref, built from the
reference sources by `make -C oracle ref`) around simeonPqSearchUnlocked's candidate branch (sqlite_vec_backend.cpp:3910-4051):
the distinct indexed candidates, approxK = min(candidateCount, max(k, k * rerank_factor)), the best approxK by (score desc,
tie-break key asc), computeCosineSimilarity of the original query, `sim < threshold` dropped, order (similarity desc, rowid
asc), k results.  Run where oracle/_ref exists:
    python tests/golden/make_ref_pq_candidates.py
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from oracle import oracle as O  # noqa: E402
from tests import ref_checks  # noqa: E402
from tests.test_gpu_documents import PQC_GOLDEN, PQC_SEARCHES, pq_candidates_case, pq_order_case  # noqa: E402


def answers(cs, k, rf, thr):
    held, rowids, tie_keys, cb, m, kc = cs["held"], cs["rowids"], cs["tie_keys"], cs["codebooks"], cs["m"], cs["kc"]
    n, d = held.shape
    normed, ok = O.normalize_like_reference(held)
    idx_rows = np.nonzero(ok)[0]
    codes = O.pq_encode_ref(cb, d, m, kc, normed)
    pos_of = {int(rowids[r]): j for j, r in enumerate(idx_rows)}   # rowid -> index position
    out = []
    for q, lst in zip(cs["queries"], cs["lists"]):
        qn, qok = O.normalize_like_reference(q[None, :])
        cand = sorted({pos_of[int(r)] for r in lst if int(r) in pos_of})
        if not qok[0] or not cand:
            out.append([0, ref_checks.digest(np.zeros(0, np.int64), np.zeros(0, np.float32))])
            continue
        scores, _ = O.pq_scores_ref(cb, d, m, kc, qn[0], codes[cand])
        approx = min(len(cand), max(k, k * rf))
        order = sorted(range(len(cand)), key=lambda i: (-float(scores[i]), int(tie_keys[idx_rows[cand[i]]])))[:approx]
        qq = np.ascontiguousarray(q, dtype=np.float32)
        recs = []
        for i in order:
            r = idx_rows[cand[i]]
            row = np.ascontiguousarray(held[r], dtype=np.float32)
            s = np.float32(O.lib().yo_cosine_similarity_f64(qq.ctypes.data_as(O.f32p), row.ctypes.data_as(O.f32p), d))
            if s == s and not s < np.float32(thr):
                recs.append((s, int(rowids[r])))
        recs.sort(key=lambda t: (-float(t[0]), t[1]))
        recs = recs[:k]
        out.append([len(recs), ref_checks.digest(np.array([r for _, r in recs], dtype=np.int64),
                                                 np.array([s for s, _ in recs], dtype=np.float32))])
    return out


def main():
    assert O.ref_available(), "build oracle/_ref first (make -C oracle ref)"
    result = {}
    for dtype in ("f32", "f16"):
        cs = pq_candidates_case(O, dtype)
        result[dtype] = {"inputs": ref_checks.digest(cs["held"], cs["queries"], *cs["lists"]),
                         "searches": [answers(cs, k, rf, thr) for k, rf, thr in PQC_SEARCHES]}
    cs = pq_order_case(O)
    n = len(cs["rows"])
    cs.update(held=cs["rows"], tie_keys=np.arange(n, dtype=np.uint64))
    assert np.array_equal(O.pq_encode_ref(cs["codebooks"], cs["rows"].shape[1], cs["m"], cs["kc"],
                                          O.normalize_like_reference(cs["rows"])[0]), cs["codes"])
    result["order"] = {"inputs": ref_checks.digest(cs["rows"], cs["queries"], *cs["lists"]), "searches": [answers(cs, 1, 1, -1.0)]}
    with open(PQC_GOLDEN, "w") as f:
        json.dump(result, f, separators=(",", ":"))
    print("wrote", PQC_GOLDEN, os.path.getsize(PQC_GOLDEN), "bytes")


if __name__ == "__main__":
    main()
