"""The k-means restatement (topology_kmeans_restated.c) pinned to the reference's own KMeansTopologyEngine::buildArtifacts:
built from the reference tree into oracle/_ref by oracle/topology_kmeans.mk where that tree exists (skipped elsewhere), and
through the partitions stored from it in tests/golden/ref_topology_kmeans.json everywhere."""
import json
import os

import numpy as np
import pytest

from tests import topology_kmeans_restated as T

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_topology_kmeans.json")


def _documents(seed, n, d, zero_rows, dup_rows, unusable):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, d)).astype(np.float32)
    x[rng.integers(0, n, zero_rows)] = 0.0
    src = rng.integers(0, n, dup_rows)
    x[rng.integers(0, n, dup_rows)] = x[src]
    docs = [x[i] for i in range(n)]
    for i in rng.integers(0, n, unusable):
        docs[i] = docs[i][: int(rng.integers(0, d))]   # empty or shorter than the first embedding: not usable
    return docs


@pytest.mark.skipif(not T.have_ref(), reason="oracle/_ref/libref_topology_kmeans.so not built (no reference tree)")
@pytest.mark.parametrize("seed", range(24))
def test_restatement_partition_equals_reference_build(seed):
    rng = np.random.default_rng(1000 + seed)
    n = int(rng.integers(2, 500))
    d = int(rng.choice([1, 2, 5, 16, 40]))
    k = int(rng.choice([0, 0, 2, 7, 18, n + 3]))
    iters = int(rng.choice([0, 1, 3, 10]))
    docs = _documents(seed, n, d, int(rng.integers(0, 4)), int(rng.integers(0, n // 2 + 1)), int(rng.integers(0, 4)))
    assert T.partition(T.run_kmeans(docs, k, iters)) == T.ref_partition(docs, k, iters)


@pytest.mark.skipif(not T.have_ref(), reason="oracle/_ref/libref_topology_kmeans.so not built (no reference tree)")
def test_stored_partitions_are_the_reference_builds():
    for case in json.load(open(GOLDEN))["cases"]:
        assert T.ref_partition(T.golden_documents(case), case["k"], case["iters"]) == case["partition"], case["seed"]


def test_restatement_matches_the_stored_reference_partitions():
    for case in json.load(open(GOLDEN))["cases"]:
        got = T.run_kmeans(T.golden_documents(case), case["k"], case["iters"])
        assert T.partition(got) == case["partition"], case["seed"]
