"""yams_b200_topology_kmeans against the plain-C restatement of the reference's runKMeans (topology_kmeans_restated.c): every
assignment and every centroid bit, on fp32 and fp16 corpora, odd and wide dims, every k rule, duplicates that force (chained)
empty-cluster repairs, zero / NaN / tiny-norm rows and exact distance ties; partitions against those the reference's own
KMeansTopologyEngine gave (tests/golden/ref_topology_kmeans.json); and the C++ host adapter B200TopologyKMeans::assign."""
import json
import os
import subprocess

import numpy as np
import pytest

import yams_b200 as Y
from tests import topology_kmeans_restated as T

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "ref_topology_kmeans.json")))["cases"]


def _bits(a):
    """float bits with every NaN as one value: a NaN's payload is the arithmetic's (the device's is 0x7FFFFFFF), not a result"""
    b = a.view(np.uint32).copy()
    b[np.isnan(a)] = 0x7FFFFFFF
    return b


def _corpus(x, dtype):
    c = Y.Corpus(x.shape[1], dtype, Y.COSINE)
    c.append(x.astype(np.float16) if dtype == Y.F16 else x.astype(np.float32))
    return c


def _check(x, dtype, k=0, iters=0):
    rows = x.astype(np.float16).astype(np.float32) if dtype == Y.F16 else x.astype(np.float32)
    c = _corpus(x, dtype)
    try:
        asg, cent, kk, it = c.topology_kmeans(k, iters)
        t = c.topology_kmeans_last_timings()
    finally:
        c.close()
    wa, wc, wk, wi = T.kmeans(rows, k, iters)
    assert (kk, it) == (wk, wi)
    assert np.array_equal(asg, wa)
    assert np.array_equal(_bits(cent), _bits(wc))
    if len(rows) >= 2:
        assert t["init_ms"] > 0 and t["assign_ms"] > 0 and t["total_ms"] > 0
    return asg, it


@pytest.mark.parametrize("dtype", [Y.F32, Y.F16])
@pytest.mark.parametrize("d", [1, 7, 384, 768, 1024])
def test_dims_and_dtypes(dtype, d):
    _check(T.edge_rows(d, 700, d, np.float16 if dtype == Y.F16 else np.float32), dtype)


@pytest.mark.parametrize("dtype", [Y.F32, Y.F16])
@pytest.mark.parametrize("k,iters", [(0, 0), (0, 1), (2, 10), (2, 0), (37, 10), (5000, 1), (5000, 10)])
def test_k_rules_and_iteration_caps(dtype, k, iters):
    _check(T.edge_rows(k + iters, 1500, 24, np.float16 if dtype == Y.F16 else np.float32), dtype, k, iters)


def test_matches_the_transcription_on_a_small_corpus():
    x = T.edge_rows(3, 40, 5)
    asg, cent, k, it = (lambda c: (c.topology_kmeans(6, 10), c.close())[0])(_corpus(x, Y.F32))
    wa, wc, wk, wi = T.transcribed(x, 6, 10)
    assert asg.tolist() == wa and (k, it) == (wk, wi)
    assert np.array_equal(_bits(cent), _bits(np.array(wc, dtype=np.float32)))


@pytest.mark.parametrize("dtype", [Y.F32, Y.F16])
def test_duplicates_force_chained_repairs(dtype):
    x = np.array([[1, 0, 0]] * 300 + [[0, 1, 0]] * 20 + [[0, 0, 1]] * 2, dtype=np.float32)
    asg, _ = _check(x, dtype, 12, 10)
    assert len(set(asg.tolist())) == 12


def test_fixed_point_after_the_first_round():
    # memberships start at 0, so finite rows always move in round 1; well-separated clusters whose farthest-first seeds are
    # one per cluster are a fixed point from then on: round 2 changes nothing and ends the call
    rng = np.random.default_rng(9)
    x = np.repeat(np.eye(3, 16, dtype=np.float32) * 4, 50, axis=0) + np.float32(0.01) * rng.standard_normal((150, 16)).astype(np.float32)
    asg, it = _check(x, Y.F32, 3, 10)
    assert it == 2 and T.partition(asg) == np.repeat(np.arange(3), 50).tolist()


def test_one_iteration_convergence():
    # every distance is NaN: nobody moves, no repair qualifies, the first round changes nothing
    x = np.full((50, 8), np.nan, dtype=np.float32)
    _, it = _check(x, Y.F32, 4, 10)
    assert it == 1


@pytest.mark.parametrize("dtype", [Y.F32, Y.F16])
def test_zero_nan_and_tiny_rows(dtype):
    rng = np.random.default_rng(5)
    x = rng.standard_normal((400, 64)).astype(np.float32)
    x[::7] = 0.0
    x[3::11] = np.nan
    x[5::13] *= np.float32(1e-20) if dtype == Y.F32 else np.float32(1e-6)   # fp16: subnormal stored values
    x[9::17, 1:] = 0.0
    x[9::17, 0] = np.float32(6e-8)
    for k in (0, 2, 30):
        _check(x, dtype, k, 10)


def test_equidistant_documents_take_the_lowest_centroid():
    x = np.array([[1, 0], [0, 1], [1, 1]] * 40, dtype=np.float32)
    asg, _ = _check(x, Y.F32, 2, 10)
    assert asg[2] == 0


def test_fewer_than_two_rows():
    c = _corpus(np.ones((1, 16), dtype=np.float32), Y.F32)
    try:
        asg, cent, k, it = c.topology_kmeans(3, 10)
    finally:
        c.close()
    assert asg.tolist() == [0] and k == 0 and it == 0


def test_l2_corpus_is_rejected():
    c = Y.Corpus(8, Y.F32, Y.L2)
    c.append(np.ones((4, 8), dtype=np.float32))
    try:
        with pytest.raises(Y.YamsB200Error):
            c.topology_kmeans()
    finally:
        c.close()


def test_200k_x_768_against_the_restatement():
    rng = np.random.default_rng(200)
    centers = rng.standard_normal((400, 768)).astype(np.float32)
    x = centers[rng.integers(0, 400, 200_000)] + np.float32(0.5) * rng.standard_normal((200_000, 768)).astype(np.float32)
    _check(x, Y.F32, 0, 3)


def _device(rows, k, iters, dtype):
    c = _corpus(rows, dtype)
    try:
        asg, _, kk, _ = c.topology_kmeans(k, iters)
    finally:
        c.close()
    return asg, kk


@pytest.mark.parametrize("case", GOLDEN, ids=lambda c: f"seed{c['seed']}")
def test_partition_equals_the_reference_build(case):
    """the device clustering of the usable documents, with runKMeans's singletons, against the partition the reference's own
    KMeansTopologyEngine::buildArtifacts gave (tests/golden/make_topology_kmeans_golden.py)"""
    dtype = Y.F16 if case["dtype"] == "f16" else Y.F32
    got = T.run_kmeans(T.golden_documents(case), case["k"], case["iters"], cluster=lambda r, k, i: _device(r, k, i, dtype))
    assert T.partition(got) == case["partition"]


def test_cpp_host_adapter(tmp_path):
    """B200TopologyKMeans::assign (the host adapter replacing runKMeans) over the C ABI: usable-document rule, iota below two
    usable documents, singletons after the k clusters -- the exact runKMeans vector and the reference's partition"""
    exe = str(tmp_path / "test_topology_kmeans")
    subprocess.check_call(["/usr/bin/g++", "-std=c++20", "-O1", os.path.join(ROOT, "tests", "host_cpp", "test_topology_kmeans.cpp"),
                           "-o", exe, "-L" + os.path.join(ROOT, "yams_b200"), "-lyams_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "yams_b200")])
    for case in GOLDEN:
        docs = T.golden_documents(case)
        stride = max(len(e) for e in docs)
        rows = np.zeros((len(docs), stride), dtype=np.float32)
        for i, e in enumerate(docs):
            rows[i, :len(e)] = e
        path = tmp_path / f"docs{case['seed']}.bin"
        with open(path, "wb") as f:
            f.write(np.array([len(docs)], dtype=np.uint64).tobytes() + np.array([stride], dtype=np.uint32).tobytes()
                    + np.array([case["k"], case["iters"]], dtype=np.uint64).tobytes()
                    + np.array([len(e) for e in docs], dtype=np.uint32).tobytes() + rows.tobytes())
        out = subprocess.run([exe, str(path)], capture_output=True, text=True, timeout=120)
        assert out.returncode == 0 and out.stdout.endswith("ALL OK\n"), out.stdout[-500:] + out.stderr
        got = [int(v) for v in out.stdout.split()[:-2]]
        assert got == T.run_kmeans(docs, case["k"], case["iters"]).tolist(), case["seed"]
        assert T.partition(got) == case["partition"], case["seed"]
