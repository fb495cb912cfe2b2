"""Add the key "l2_near_tie" to tests/golden/ref_checks.json by EXECUTING THE REFERENCE: for the corpora of
tests/ref_checks.l2_near_tie_case (fp16 and fp32), every query's nearest rows by the reference build's own l2_distance
(oracle/_ref, built from the reference sources by `make -C oracle ref`), ranked by (distance, rowid).  The other keys are
left as they are.  Run where oracle/_ref exists:  python tests/golden/make_ref_l2_near_tie.py
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
from oracle import oracle as O  # noqa: E402
from tests import ref_checks  # noqa: E402

TOP = 32   # stored per query; the tests compare the first k = 10


def main():
    assert O.ref_available(), "build oracle/_ref first (make -C oracle ref)"
    R = O.ref()
    out = {}
    for dtype in ("f16", "f32"):
        _, held, queries = ref_checks.l2_near_tie_case(O, dtype)
        n, d = held.shape
        ids, dists = [], []
        for q in queries:
            q = np.ascontiguousarray(q, dtype=np.float32)
            dist = np.array([R.ref_l2_distance(O._p(q, O.f32p), O._p(held[i], O.f32p), d) for i in range(n)], dtype=np.float32)
            order = np.lexsort((np.arange(n), dist))[:TOP]
            ids.append([int(i) for i in order])
            dists.append(ref_checks.pack_f32(dist[order]))
        out[dtype] = {"inputs": ref_checks.digest(held, queries), "rowids": ids, "dist": dists}
    path = os.path.join(HERE, "ref_checks.json")
    with open(path) as f:
        data = json.load(f)
    data["l2_near_tie"] = out
    with open(path, "w") as f:
        json.dump(data, f, separators=(",", ":"))
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
