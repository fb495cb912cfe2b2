"""Writes tests/golden/ref_topology_kmeans.json: the partitions the reference's own KMeansTopologyEngine::buildArtifacts
(oracle/_ref/libref_topology_kmeans.so, built by oracle/topology_kmeans.mk) gives on generated documents, for the GPU tests
where the reference build does not exist.  Run from the repository root: python tests/golden/make_topology_kmeans_golden.py"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tests import topology_kmeans_restated as T  # noqa: E402

CASES = [
    {"seed": 11, "n": 700, "d": 7, "dtype": "f32", "k": 0, "iters": 0},
    {"seed": 12, "n": 700, "d": 7, "dtype": "f16", "k": 0, "iters": 0},
    {"seed": 13, "n": 400, "d": 384, "dtype": "f16", "k": 0, "iters": 10},
    {"seed": 14, "n": 300, "d": 768, "dtype": "f32", "k": 2, "iters": 10},
    {"seed": 15, "n": 250, "d": 1024, "dtype": "f32", "k": 0, "iters": 1},
    {"seed": 16, "n": 500, "d": 1, "dtype": "f32", "k": 40, "iters": 10},
    {"seed": 17, "n": 120, "d": 24, "dtype": "f16", "k": 500, "iters": 10},
    {"seed": 18, "n": 600, "d": 24, "dtype": "f32", "k": 30, "iters": 10, "empty": [0, 20, 599], "short": [33, 34]},
    {"seed": 19, "n": 3, "d": 8, "dtype": "f32", "k": 0, "iters": 0, "empty": [1]},
]


def main():
    assert T.have_ref(), "needs oracle/_ref/libref_topology_kmeans.so (make -f oracle/topology_kmeans.mk)"
    out = []
    for case in CASES:
        labels = T.ref_partition(T.golden_documents(case), case["k"], case["iters"])
        out.append(dict(case, partition=labels))
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ref_topology_kmeans.json")
    with open(path, "w") as f:
        json.dump({"source": "KMeansTopologyEngine::buildArtifacts (src/topology/topology_alternate_engines.cpp:644-670), "
                             "partition by first appearance", "cases": out}, f, separators=(",", ":"))
        f.write("\n")


if __name__ == "__main__":
    main()
