"""yams_b200_semantic_neighbors (the semantic-neighbour graph) against the plain-C restatement of the reference loop
(semantic_graph_restated.c): rowids, counts and similarity bits, on both stage-1 engines, the sampled-threshold path, the
certificate's fallback levels and every row class the graph's row set rule distinguishes; the stage-1 error of the graph's
scales against float64; argument errors; and the C++ adapter B200SemanticGraph."""
import os
import subprocess

import numpy as np
import pytest

from tests import semantic_restated as S

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID_ARG = 1


@pytest.fixture(scope="module")
def Y():
    import yams_b200
    assert yams_b200.device_count() > 0
    assert yams_b200.plugin_init() == 0, yams_b200.health()
    return yams_b200


def _rowids(n):
    return 5 + 3 * np.arange(n, dtype=np.int64)      # ascending, not dense: rowid != row


def _corpus(Y, x, dtype):
    c = Y.Corpus(x.shape[1], dtype, Y.COSINE)
    if len(x):
        c.append(x.view(np.uint16) if x.dtype == np.float16 else np.ascontiguousarray(x, dtype=np.float32), _rowids(len(x)))
    return c


def _check(Y, c, x, k, threshold=None, sources=None, expect_fallback=None):
    """the graph of corpus c (rows x) against the oracle; sources are row indices (>= len(x): unknown rowids)"""
    rid = _rowids(max(len(x), 1) + 64)
    src_rowids = None if sources is None else rid[np.asarray(sources, dtype=np.int64)]
    thr = S.FLT_TRUE_MIN if threshold is None else threshold
    r, s, cnt, flags = c.semantic_neighbors(k, thr, src_rowids)
    wr, ws, wc, _ = S.semantic_neighbors(x.astype(np.float32), k, threshold, sources)
    assert np.array_equal(cnt, wc)
    want_rowids = np.where(wr >= 0, rid[np.maximum(wr, 0)], -1)
    assert np.array_equal(r, want_rowids)
    assert np.array_equal(s.view(np.uint32), ws.view(np.uint32))
    if expect_fallback is not None:
        assert ((flags & Y.FLAG_FALLBACK_PATH) != 0).any() == expect_fallback
    return flags


def _unit_rows(seed, n, d):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, d)).astype(np.float32)
    return x / np.linalg.norm(x, axis=1, keepdims=True).astype(np.float32)


@pytest.mark.parametrize("d", [384, 768, 1000])
@pytest.mark.parametrize("n", [0, 1, 2, 3, 2000])
def test_all_sources_f32(Y, d, n):
    x = _unit_rows(d + n, n, d)
    c = _corpus(Y, x, Y.F32)
    _check(Y, c, x, 8)
    c.close()


def test_cuda_core_engine_d30(Y):
    x = _unit_rows(30, 3000, 30)          # 120-byte rows are no 16-byte TMA pitch: the wgmma engine declines the shape
    c = _corpus(Y, x, Y.F32)
    _check(Y, c, x, 8)
    assert c.last_timings()["engine"] == "cuda-core"
    _check(Y, c, x, 8, threshold=0.3)
    c.close()


@pytest.mark.parametrize("dtype", ["f32", "f16"])
def test_sampled_threshold_path(Y, dtype):
    """70 000 rows: above the dense limit (65 536), stage 1 runs with sampled thresholds and the filter"""
    n, d = 70_000, 768
    x = _unit_rows(70, n, d)
    if dtype == "f16":
        x = x.astype(np.float16)
    c = _corpus(Y, x, Y.F16 if dtype == "f16" else Y.F32)
    r, s, cnt, _ = c.semantic_neighbors(8)
    assert (cnt == 8).all()
    pick = np.random.default_rng(1).choice(n, 200, replace=False)
    pick.sort()
    wr, ws, wc, _ = S.semantic_neighbors(x.astype(np.float32), 8, None, pick)
    rid = _rowids(n)
    assert np.array_equal(cnt[pick], wc)
    assert np.array_equal(r[pick], np.where(wr >= 0, rid[np.maximum(wr, 0)], -1))
    assert np.array_equal(s[pick].view(np.uint32), ws.view(np.uint32))
    _check(Y, c, x, 8, sources=pick[:64])
    c.close()


def test_source_subsets(Y):
    x = _unit_rows(3, 3000, 256)
    x[10] = 0.0                            # excluded row as a source
    x[11, 5] = np.nan
    c = _corpus(Y, x, Y.F32)
    flags = _check(Y, c, x, 8, sources=[0, 10, 11, 12, 2999, 3000, 3010])   # 3000, 3010: unknown rowids
    assert ((flags & Y.FLAG_NOT_A_SOURCE) != 0).tolist() == [False, True, True, False, False, True, True]
    _check(Y, c, x, 8, sources=[])
    _check(Y, c, x, 8, sources=list(range(0, 3000, 7)))
    c.close()


@pytest.mark.parametrize("dtype", ["f32", "f16"])
@pytest.mark.parametrize("threshold", [None, 0.0, 0.05, 1.0])
def test_row_classes(Y, dtype, threshold):
    """tiny-norm rows are neighbours here (search skips them); zero, inf and NaN rows are not; fp16 subnormal rows count"""
    n, d = 1500, 64
    x = _unit_rows(9, n, d)
    x[100:140] *= np.float32(1e-7)        # |r|^2 ~ 1e-14: in the graph
    x[140:150] = 0.0
    x[150:155, 3] = np.inf
    x[155:160, 7] = np.nan
    x[160:200] = x[0:40] * np.float32(3e-6)    # fp16: subnormal elements (below 2^-14)
    x[200:210] = x[5]                     # duplicates of row 5
    if dtype == "f16":
        x = x.astype(np.float16)
    c = _corpus(Y, x, Y.F16 if dtype == "f16" else Y.F32)
    _check(Y, c, x, 8, threshold)
    c.close()


@pytest.mark.parametrize("d,scale", [(30, 1e-23), (64, 1e-23), (64, 1e-37)])
def test_underflowing_products_are_not_certified(Y, d, scale):
    """fp32 rows A, B = scale * row 0: A.B underflows in stage 1 (the CUDA-core engine at d = 30, the tf32 engine at d = 64;
    1e-37 also puts the elements below FLT_MIN) while the exact similarity is 1.  The certificate's underflow term sends A to
    the exhaustive levels (level 1 runs the CUDA-core engine, so it cannot certify either), which find B."""
    x = _unit_rows(d, 3000, d)
    x[3000 - 2:] = x[0] * np.float32(scale)
    c = _corpus(Y, x, Y.F32)
    flags = _check(Y, c, x, 8, sources=[0, 1500, 2998, 2999])
    assert flags[2] & Y.FLAG_FALLBACK_PATH and flags[3] & Y.FLAG_FALLBACK_PATH
    if scale > 1e-30:                                  # ordinary sources stay certified while 1/|r| * 2^-126 is small
        assert not flags[1] & Y.FLAG_FALLBACK_PATH
    assert c.last_timings()["resolved_full_pass"] >= 2
    _check(Y, c, x, 8)
    c.close()


def test_infinite_scale_rows(Y):
    """a row whose float 1/|r| overflows (every element 1e-45) is taken, with +-inf similarities; NaN ones (dot == 0) are dropped"""
    x = _unit_rows(8, 500, 64)
    x[17] = np.float32(1.4e-45)
    x[18, :] = 0.0
    x[18, :32] = np.float32(1.4e-45)
    x[18, 32:] = -np.float32(1.4e-45)              # dot with row 17 is 0: 0 * inf = NaN
    c = _corpus(Y, x, Y.F32)
    flags = _check(Y, c, x, 8)
    assert (flags & Y.FLAG_FALLBACK_PATH).all()     # no stage-1 bound holds with an infinite scale
    _check(Y, c, x, 8, threshold=0.0, sources=[0, 17, 18, 499])
    c.close()


def test_negative_zero_ties_by_row(Y):
    x = np.zeros((64, 4), dtype=np.float32)
    x[0] = [1, 0, 0, 0]
    x[1] = [-1.4e-45, 4, 0, 0]            # sim with row 0: -0.0
    x[2:] = _unit_rows(2, 62, 4)
    x[2:, 0] = 0.0                        # orthogonal to row 0: +0.0
    c = _corpus(Y, x, Y.F32)
    _check(Y, c, x, 16, threshold=0.0)
    _check(Y, c, x, 16)
    c.close()


def test_near_ties_fall_back(Y):
    """300 rows within 1e-4 of the k-th score: the certificate fails, the exhaustive level answers"""
    n, d = 4000, 128
    x = _unit_rows(4, n, d)
    rng = np.random.default_rng(5)
    base = x[0].copy()
    x[1:301] = base + rng.standard_normal((300, d)).astype(np.float32) * np.float32(3e-6)
    c = _corpus(Y, x, Y.F32)
    flags = _check(Y, c, x, 8, sources=[0, 1, 2, 500])
    assert flags[0] & Y.FLAG_FALLBACK_PATH
    c.close()


def test_duplicates_reach_level2(Y):
    """6 000 identical rows: neither stage 1 nor level 1 (4 096 survivors) can certify the top-8"""
    d = 64
    x = np.concatenate([np.tile(_unit_rows(6, 1, d), (6000, 1)), _unit_rows(7, 500, d)])
    c = _corpus(Y, x, Y.F32)
    flags = _check(Y, c, x, 8, sources=[0, 17, 5999, 6000, 6100])
    assert (flags[:3] & Y.FLAG_FALLBACK_PATH).all()
    assert c.last_timings()["resolved_full_pass"] >= 3
    c.close()


@pytest.mark.parametrize("k", [1, 8, 100, 3072])
def test_k(Y, k):
    x = _unit_rows(k, 4000, 64)
    x[300:310] = x[3]
    if k == 100:
        x = x.astype(np.float16)
    c = _corpus(Y, x, Y.F16 if k == 100 else Y.F32)
    _check(Y, c, x, k, sources=None if k <= 100 else list(range(0, 4000, 37)))
    c.close()


@pytest.mark.parametrize("engine", [1, 0])
@pytest.mark.parametrize("dtype", ["f32", "f16"])
def test_stage1_error_within_eps(Y, engine, dtype):
    """|stage-1 score - exact float score| <= eps (the certificate's bound, the score's float cast included), float64 check"""
    n, d = 20_000, 768
    x = _unit_rows(11, n, d) * np.float32(0.7)
    x[:200] *= np.float32(1e-4)
    if dtype == "f16":
        x = x.astype(np.float16)
    c = _corpus(Y, x, Y.F16 if dtype == "f16" else Y.F32)
    src = np.arange(0, n, 157)[:64]
    got, eps = c.debug_semantic_stage1(_rowids(n)[src], engine)
    xf = x.astype(np.float64)
    inv = np.array([np.float32(1.0 / np.sqrt(np.dot(r, r))) for r in xf], dtype=np.float32).astype(np.float64)
    exact = ((xf[src] @ xf.T) * inv[src][:, None] * inv[None, :]).astype(np.float32).astype(np.float64)
    err = np.abs(got.astype(np.float64) - exact)
    assert np.isfinite(got).all()
    assert (err <= eps[:, None]).all(), float((err - eps[:, None]).max())
    c.close()


def test_300k_f16_sources(Y):
    n, d = 300_000, 768
    x = _unit_rows(300, n, d).astype(np.float16)
    c = _corpus(Y, x, Y.F16)
    _check(Y, c, x, 8, sources=np.sort(np.random.default_rng(2).choice(n, 64, replace=False)))
    c.close()


def test_argument_errors(Y):
    x = _unit_rows(1, 100, 16)
    l2 = Y.Corpus(16, Y.F32, Y.L2)
    l2.append(x, _rowids(100))
    with pytest.raises(Y.YamsB200Error) as e:
        l2.semantic_neighbors(8)
    assert e.value.status == INVALID_ARG
    l2.close()
    c = _corpus(Y, x, Y.F32)
    for call in (lambda: c.semantic_neighbors(3073),
                 lambda: c.semantic_neighbors(8, sources=_rowids(100)[[3, 2]]),
                 lambda: c.semantic_neighbors(8, sources=_rowids(100)[[3, 3]])):
        with pytest.raises(Y.YamsB200Error) as e:
            call()
        assert e.value.status == INVALID_ARG
    import ctypes as C
    out_c = np.zeros(99, dtype=np.uint32)
    assert Y.lib().yams_b200_semantic_neighbors(c._h, None, 99, 8, Y.FLT_TRUE_MIN, None, None,
                                                out_c.ctypes.data_as(C.POINTER(C.c_uint32)), None) == INVALID_ARG
    r, s, cnt, _ = c.semantic_neighbors(0)
    assert r.shape == (100, 0) and (cnt == 0).all()
    c.close()


def test_cpp_semantic_graph(Y, tmp_path):
    """B200SemanticGraph::neighbors (the host adapter the daemon calls) over the C ABI"""
    exe = str(tmp_path / "test_semantic_graph")
    subprocess.check_call(["/usr/bin/g++", "-std=c++20", "-O1", os.path.join(ROOT, "tests", "host_cpp", "test_semantic_graph.cpp"),
                           "-o", exe, "-L" + os.path.join(ROOT, "yams_b200"), "-lyams_b200",
                           "-Wl,-rpath," + os.path.join(ROOT, "yams_b200")])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0 and "ALL OK" in out.stdout, out.stdout + out.stderr
