"""Stage 1 of the vector scan as a unit: the wgmma engine (csrc/knn_umma.cu) and the CUDA-core engine (csrc/knn.cu) against a
float64 evaluation of the values the corpus holds.

The exactness certificate (DESIGN.md §4.2) rests on two properties of stage 1, checked here element by element:
  * every stage-1 score is within eps[q] of the exact score, at every query-tile width (64 or 256 columns, partial last
    tiles), K-block tail, row-tile count and row sampling the scan uses, and on data built to stress fp16 / tf32 operand
    rounding and the fp32 accumulation inside the tensor core;
  * the filter epilogue lists exactly the rows whose stage-1 score is > tau[q] (and that are allowed), with the score the
    dense pass computes.  The certificate bounds a row that never reached the list by tau + eps, so a row the filter drops
    is lost without any check noticing.

Exact scores: cosine x.r / (|x| |r|), L2 2 q.r - |r|^2; rows the reference skips (non-finite, or sum r^2 <= 1e-12 for cosine;
non-finite for L2) score exactly -inf."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ENGINES = {"wgmma": 1, "cuda-core": 0}
UNSUPPORTED = 5                 # YAMS_ERR_UNSUPPORTED
WGMMA_MAX_NQ = 4096             # the wgmma engine keeps every query tile's thresholds in shared memory
ROWS = 132 * 128 + 1277         # 142 row tiles, the last one partial: more tiles than an H100 SXM has SMs (132)
MAC_BUDGET = 1.5e8              # float64 reference work per engine call

NQS = [1, 63, 64, 65, 255, 256, 257, 1024, WGMMA_MAX_NQ]   # 64-column query tiles up to 64 queries, 256-column tiles above
F16_DIMS = [8, 72, 200, 768, 1000]                          # K blocks of 64 fp16 elements: one partial, several + a tail
F32_DIMS = [4, 36, 100, 772]                                # K blocks of 32 tf32 elements
SHAPES = sorted(set(
    [("f16", 72, nq) for nq in NQS] + [("f32", 36, nq) for nq in NQS]
    + [("f16", d, nq) for d in F16_DIMS for nq in (64, 257)] + [("f32", d, nq) for d in F32_DIMS for nq in (64, 257)]
    + [("f16", 4096, 1), ("f16", 4096, 300), ("f32", 2048, 65)]))


@pytest.fixture(scope="module")
def Y():
    import yams_b200
    assert yams_b200.device_count() > 0
    assert yams_b200.plugin_init() == 0, yams_b200.health()
    return yams_b200


def make_corpus(Y, rows, metric):
    dt = Y.F16 if rows.dtype == np.float16 else Y.F32
    c = Y.Corpus(rows.shape[1], dt, Y.L2 if metric == "l2" else Y.COSINE)
    c.append(rows)
    return c


def exact_scores(rows, queries, metric):
    """float64 scores of the values the corpus holds -> (scores [nq, n], valid rows [n])"""
    r = rows.astype(np.float64)
    x = np.asarray(queries, dtype=np.float32).astype(np.float64)
    finite = np.isfinite(r).all(axis=1)
    r[~finite] = 0.0
    ss = np.einsum("ij,ij->i", r, r)
    dots = x @ r.T
    if metric == "cosine":
        valid = finite & (ss > 1e-12)
        with np.errstate(divide="ignore", invalid="ignore"):
            s = dots / (np.linalg.norm(x, axis=1)[:, None] * np.sqrt(ss)[None, :])
    else:
        valid = finite
        s = 2.0 * dots - ss[None, :]
    s[:, ~valid] = -np.inf
    return s, valid


def check_within_eps(got, want, valid, eps, where):
    """|got - want| <= eps[q] everywhere, no NaN, skipped rows exactly -inf -> the largest err / eps"""
    assert got.shape == want.shape, where
    assert not np.isnan(got).any(), where
    assert np.all(got[:, ~valid] == -np.inf), where
    assert np.all(eps > 0) and not np.isnan(eps).any(), where
    if not valid.any():
        return 0.0
    err = np.abs(got[:, valid].astype(np.float64) - want[:, valid]).max(axis=1)
    bad = np.nonzero(err > eps)[0]
    assert bad.size == 0, f"{where}: queries {bad[:5]} err {err[bad[:5]]} > eps {eps[bad[:5]]}"
    return float((err / eps).max())


def stage1(c, q, engine, row_start=0, row_stride=1, nrows=0):
    got = c.debug_stage1_scores(q, ENGINES[engine], row_start=row_start, row_stride=row_stride, nrows=nrows)
    return got, c.debug_last_eps(len(q))


def row_plans(n, nq, d):
    """(row_start, row_stride, nrows) of the calls that fit the reference budget: rows from 0 (the whole corpus where
    affordable), and the strided sampling pass starting past row 0"""
    span = min(n, max(256, int(MAC_BUDGET // (nq * d))))
    m = max(16, min(n // 7, span))
    stride = max(2, (n - 5) // m)
    return [(0, 1, span), (5, stride, min(m, (n - 6) // stride + 1))]


# ---------------------------------------------------------------------------------------------------------------------
# error bound over the scan's shapes
# ---------------------------------------------------------------------------------------------------------------------
_CORPORA = {}


def sweep_corpus(Y, dtype, d, metric):
    """Gaussian rows of norms spread over 2.5 decades, a zero row, rows with inf / NaN -> (corpus, held float64 values)"""
    key = (dtype, d, metric)
    if key not in _CORPORA:
        rng = np.random.default_rng(1000 + d)
        n = ROWS if d <= 256 else 4000 + 77
        scale = np.exp(rng.uniform(np.log(0.05), np.log(20.0), size=(n, 1))) / np.sqrt(d)
        r = (rng.standard_normal((n, d)) * scale).astype(np.float32)
        r[7] = 0.0
        r[11, d // 2] = np.inf
        r[13, 0] = np.nan
        rows = r.astype(np.float16 if dtype == "f16" else np.float32)
        _CORPORA[key] = (make_corpus(Y, rows, metric), rows)
    return _CORPORA[key]


@pytest.fixture(scope="module", autouse=True)
def _close_corpora():
    yield
    for c, _ in _CORPORA.values():
        c.close()
    _CORPORA.clear()


def sweep_queries(rows, nq, rng):
    q = (rng.standard_normal((nq, rows.shape[1])) * 3.0).astype(np.float32)
    k = min(nq, 8)
    src = rng.choice(np.arange(20, rows.shape[0]), size=k, replace=False)
    q[:k] = rows[src].astype(np.float32) * np.float32(1.5) + (rng.standard_normal((k, rows.shape[1])) * 1e-3).astype(np.float32)
    return q


@pytest.mark.parametrize("engine", list(ENGINES))
@pytest.mark.parametrize("metric", ["cosine", "l2"])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"{t}-d{d}-nq{nq}" for t, d, nq in SHAPES])
def test_stage1_within_eps_over_shapes(Y, shape, metric, engine, record_property):
    dtype, d, nq = shape
    c, rows = sweep_corpus(Y, dtype, d, metric)
    q = sweep_queries(rows, nq, np.random.default_rng(nq * 7 + d))
    worst = 0.0
    for start, stride, nrows in row_plans(rows.shape[0], nq, d):
        sel = rows[start:start + stride * nrows:stride]
        assert len(sel) == nrows
        want, valid = exact_scores(sel, q, metric)
        got, eps = stage1(c, q, engine, start, stride, nrows)
        worst = max(worst, check_within_eps(got, want, valid, eps, (engine, start, stride, nrows)))
    record_property("err_over_eps", worst)


def test_more_queries_than_the_wgmma_engine_takes(Y, oracle):
    """4097 queries: the wgmma engine declines, the search runs on the CUDA-core engine, reports it and stays exact."""
    O = oracle
    n, d, k = 3000, 64, 10
    rows = O.f16_from_float(O.gen_rows_f32(42, 0, n, d)).reshape(n, d)
    c = Y.Corpus(d, Y.F16, Y.COSINE)
    c.append(rows.view(np.float16))
    q = O.gen_rows_f32(43, 0, WGMMA_MAX_NQ + 1, d)
    with pytest.raises(Y.YamsB200Error) as e:
        c.debug_stage1_scores(q, ENGINES["wgmma"], nrows=256)
    assert e.value.status == UNSUPPORTED
    got = c.search(q, k)
    assert c.last_timings()["engine"] == "cuda-core"
    sub = [0, 1, 255, 256, 4095, 4096]
    rc, wr, ws, wc = O.exact_scan_cosine_batch(rows, q[sub], k)
    assert rc == 0 and np.array_equal(got[0][sub], wr) and np.array_equal(got[1][sub], ws)
    c.search(q[:WGMMA_MAX_NQ], k)
    assert c.last_timings()["engine"] == "wgmma"
    c.close()


@pytest.mark.parametrize("shape", [(1000, 128, 16), (5000, 768, 300), (777, 72, 5), (40000, 64, 257)])
def test_engines_agree_on_synthetic_rows(Y, oracle, shape, record_property):
    """The library's synthetic fp16 corpus and non-unit queries (1/|q| folding): both engines within eps of float64 and of
    each other, over all rows and over the strided sampling pass."""
    O = oracle
    n, d, nq = shape
    rows16 = O.f16_from_float(O.gen_rows_f32(42, 0, n, d)).reshape(n, d).view(np.float16)
    c = make_corpus(Y, rows16, "cosine")
    q = O.gen_rows_f32(43, 0, nq, d) * np.float32(3.0)
    want, valid = exact_scores(rows16, q, "cosine")
    got = {}
    for engine in ENGINES:
        got[engine] = stage1(c, q, engine)
        record_property(f"err_over_eps_{engine}", check_within_eps(*got[engine][:1], want, valid, got[engine][1], engine))
        ts, eps = stage1(c, q[:3], engine, row_start=0, row_stride=7, nrows=n // 7)
        check_within_eps(ts, want[:3, 0:7 * (n // 7):7], valid[0:7 * (n // 7):7], eps, (engine, "strided"))
    (tc, eps_tc), (cc, eps_cc) = got["wgmma"], got["cuda-core"]
    assert np.all(np.abs(tc.astype(np.float64) - cc) <= (eps_tc + eps_cc)[:, None])
    c.close()


# ---------------------------------------------------------------------------------------------------------------------
# error bound on adversarial data
# ---------------------------------------------------------------------------------------------------------------------
def _f16(x):
    return np.asarray(x, dtype=np.float32).astype(np.float16)


def adv_all_positive(rng, dtype, metric):
    """all-positive rows and queries: sum |y_i r_i| = y.r, the accumulation bound has no cancellation to hide in"""
    n, d = 2000, 768 if dtype == "f16" else 772
    r = rng.uniform(0.0, 1.0, size=(n, d)).astype(np.float32)
    rows = r.astype(np.float16) if dtype == "f16" else r
    q = np.concatenate([rng.uniform(0.0, 1.0, size=(24, d)).astype(np.float32), rows[:40].astype(np.float32)])
    return rows, q


def adv_sub_ulp(rng, dtype, metric):
    """fp16 d = 4096 rows: 16 elements 1.0, the other 4080 equal to b, queries equal to the rows.  The accumulator then sits
    just above a power of two for the whole K loop while every later product y_i r_i lies just below or above its ulp: an
    accumulation that aligns products to the accumulator and truncates loses almost one ulp per element -- the worst case
    of the 2^-23 (d + 4) term (d ulps of a value just above a power of two)."""
    d = 4096
    # |r| ~ 4 (cosine: x = r / |r|, acc = |r|, products b^2 / 4) and |r|^2 ~ 16 (L2: x = r, acc = |r|^2, products b^2): both
    # products equal the accumulator's ulp (2^-21 at 4, 2^-19 at 16) for b = 4 * 2^-11.5
    b0 = 4.0 * np.sqrt(np.ldexp(1.0, -23))
    b = np.unique(_f16(np.linspace(0.85 * b0, 1.15 * b0, 400)))
    rows = np.empty((len(b), d), dtype=np.float16)
    rows[:] = b[:, None]
    rows[:, :16] = 1.0
    q = np.concatenate([rows.astype(np.float32), rng.uniform(0.0, 1.0, size=(8, d)).astype(np.float32)])
    return rows, q


def adv_big_and_tiny(rng, dtype, metric):
    """fp16 d = 4096: in every 16-element K chunk one element 1.0 and fifteen tiny ones (2^-4 .. 2^-24, subnormals
    included): the tensor core aligns each chunk to its large product and truncates the small ones"""
    n, d = 256, 4096
    t = _f16(np.exp2(-rng.uniform(4.0, 24.0, size=n)))
    rows = np.empty((n, d), dtype=np.float16)
    rows[:] = t[:, None]
    for i in range(n):
        rows[i, (i % 16)::16] = 1.0
    q = np.concatenate([rows[:48].astype(np.float32), rows[48:64, ::-1].astype(np.float32),
                        rng.uniform(0.0, 1.0, size=(8, d)).astype(np.float32)])
    return rows, q


def adv_tiny_rows_extreme_queries(rng, dtype, metric):
    """fp16 rows with subnormal elements and rows whose sum r^2 lies just above / below the 1e-12 skip cutoff; queries with
    one dominant component and queries whose scaled components underflow fp16"""
    d = 64
    sub = _f16(rng.integers(1, 1024, size=(64, d)) * np.ldexp(1.0, -24))            # fp16 subnormals
    lo, hi = np.float16(np.ldexp(2.0, -24)), np.float16(np.ldexp(3.0, -24))         # 64 lo^2 < 1e-12 < 64 hi^2
    cut = np.full((65, d), lo, dtype=np.float16)
    for k in range(65):
        cut[k, :k] = hi
    normal = (rng.standard_normal((300, d)) * 0.2).astype(np.float16)
    rows = np.concatenate([sub, cut, normal])
    ss = (rows.astype(np.float64) ** 2).sum(axis=1)
    assert (np.abs(ss[64:129] / 1e-12 - 1.0) < 0.05).sum() >= 3 and (ss[64:129] <= 1e-12).any()
    q = (rng.standard_normal((40, d))).astype(np.float32)
    q[:8] = 1e-4
    q[np.arange(8), np.arange(8)] = 1.0                                              # one dominant component
    q[8:16] = 1e-9 * np.sign(q[8:16])                                                # scaled: underflow fp16 ...
    q[np.arange(8, 16), np.arange(8)] = 1.0                                          # ... next to a unit component
    q[16:24] = rows[129:137].astype(np.float32)
    q[24:32] = rows[64 + 4:64 + 12].astype(np.float32) * np.float32(2.0 ** 20)     # the cutoff rows' directions (a valid
    return rows, q                                                                  # query has |q|^2 >= 1e-10)


def adv_tf32_low_bits(rng, dtype, metric):
    """fp32 rows and queries with bits set in the 13 mantissa bits tf32 drops (all set, or random)"""
    n, d = 3000, 100 if metric == "cosine" else 772
    r = (rng.standard_normal((n, d)) * np.exp(rng.uniform(-3, 3, size=(n, 1)))).astype(np.float32)
    bits = r.view(np.uint32)
    bits[: n // 2] |= np.uint32(0x1FFF)
    bits[n // 2:] = (bits[n // 2:] & np.uint32(0xFFFFE000)) | rng.integers(0, 0x2000, size=(n - n // 2, d), dtype=np.uint32)
    q = (rng.standard_normal((40, d))).astype(np.float32)
    q.view(np.uint32)[:20] |= np.uint32(0x1FFF)
    q[20:30] = r[:10]
    return r, q


def adv_l2_cancellation(rng, dtype, metric):
    """L2 rows of norm ~1e3 and queries at or next to a row: 2 q.r and |r|^2 (~1e6) cancel to the squared distance"""
    n, d = 3000, 768 if dtype == "f16" else 128
    r = (rng.standard_normal((n, d)) * (1e3 / np.sqrt(d)) * rng.uniform(0.9, 1.1, size=(n, 1))).astype(np.float32)
    rows = r.astype(np.float16) if dtype == "f16" else r
    held = rows.astype(np.float32)
    q = np.concatenate([held[:16], held[16:32] + (rng.standard_normal((16, d)) * 1e-2).astype(np.float32),
                        (rng.standard_normal((8, d)) * 30.0).astype(np.float32)])
    return rows, q


ADVERSARIAL = [
    ("all_positive", adv_all_positive, [("f16", "cosine"), ("f16", "l2"), ("f32", "cosine"), ("f32", "l2")]),
    ("sub_ulp_accumulation", adv_sub_ulp, [("f16", "cosine"), ("f16", "l2")]),
    ("big_and_tiny_per_chunk", adv_big_and_tiny, [("f16", "cosine"), ("f16", "l2")]),
    ("tiny_rows_extreme_queries", adv_tiny_rows_extreme_queries, [("f16", "cosine")]),
    ("tf32_low_bits", adv_tf32_low_bits, [("f32", "cosine"), ("f32", "l2")]),
    ("l2_cancellation", adv_l2_cancellation, [("f16", "l2"), ("f32", "l2")]),
]
ADV_CASES = [(name, fn, dt, m, e) for name, fn, combos in ADVERSARIAL for dt, m in combos for e in ENGINES]


@pytest.mark.parametrize("case", ADV_CASES, ids=[f"{c[0]}-{c[2]}-{c[3]}-{c[4]}" for c in ADV_CASES])
def test_stage1_within_eps_on_adversarial_data(Y, case, record_property):
    name, build, dtype, metric, engine = case
    rows, q = build(np.random.default_rng(7), dtype, metric)
    c = make_corpus(Y, rows, metric)
    want, valid = exact_scores(rows, q, metric)
    got, eps = stage1(c, q, engine)
    record_property("err_over_eps", check_within_eps(got, want, valid, eps, (name, dtype, metric, engine)))
    c.close()


def test_f16_l2_query_outside_the_f16_range(Y, oracle):
    """An L2 query component beyond 65504 has no fp16 operand: its wgmma error bound must be +inf (never NaN), so the
    certificate sends the query to the exhaustive levels, which return the exact answer.  Other queries are unaffected."""
    O = oracle
    n, d, k = 20_000, 40, 10
    rows16 = O.f16_from_float(O.gen_rows_f32(42, 0, n, d) * np.float32(3.0)).reshape(n, d)
    rows = O.f16_to_float(rows16).reshape(n, d)
    c = Y.Corpus(d, Y.F16, Y.L2)
    c.append(rows16.view(np.float16))
    q = O.gen_rows_f32(43, 0, 6, d) * np.float32(2.0)
    q[2, 5] = 1e5
    q[4, 0] = -7e4
    got, eps = stage1(c, q, "wgmma")
    assert eps[2] == np.inf and eps[4] == np.inf, eps
    ok = [0, 1, 3, 5]
    want, valid = exact_scores(rows, q[ok], "l2")
    check_within_eps(got[ok], want, valid, eps[ok], "finite queries")
    rid, dist, cnt, flags = c.search(q, k)
    assert c.last_timings()["engine"] == "wgmma"
    assert [bool(f & Y.FLAG_FALLBACK_PATH) for f in flags] == [False, False, True, False, True, False]
    ex = c.search_exhaustive(q, k)
    assert np.array_equal(rid, ex[0]) and np.array_equal(dist, ex[1])
    for qi in range(len(q)):
        wr, wd = O.vec0_exact(rows, q[qi], k=k)
        assert np.allclose(dist[qi], wd, rtol=1e-6), qi
    c.close()


# ---------------------------------------------------------------------------------------------------------------------
# filter epilogue: the candidate lists are exactly {row : dense score > tau[q] (and allowed)}
# ---------------------------------------------------------------------------------------------------------------------
def filter_corpus_rows(dtype, metric, rng):
    """ROWS rows (142 row tiles), with the pre-filter's edge rows: cosine rows of norm ~1e-6 (1/|r| ~ 1e6) and rows just
    below the skip cutoff; L2 rows of norm ~1e3 (|r|^2 ~ 1e6); zero, inf and NaN rows"""
    d = 72 if dtype == "f16" else 100
    r = (rng.standard_normal((ROWS, d)) * np.exp(rng.uniform(-1.5, 1.5, size=(ROWS, 1)))).astype(np.float32)
    special = np.arange(100, ROWS, 997)[:16]
    for j, i in enumerate(special):
        if metric == "cosine":
            v = np.ldexp(3.0, -24) if dtype == "f16" else 1.3e-6 / np.sqrt(d)   # sum r^2 ~ 1.1e-12 .. 1.7e-12
            r[i] = v * np.where(rng.uniform(size=d) < 0.5, -1.0, 1.0)
            r[i, : j % 4] *= 1.0 if dtype == "f16" else 0.9
        else:
            r[i] = rng.standard_normal(d) * (1e3 / np.sqrt(d))
    r[3] = 0.0
    r[5, 1] = np.inf
    r[9, 2] = np.nan
    if metric == "cosine":
        r[17] = np.ldexp(1.0, -24) if dtype == "f16" else 1e-7 / np.sqrt(d)   # below the cutoff: skipped
    rows = r.astype(np.float16) if dtype == "f16" else r
    return rows, special


def check_lists(dense, counts, lists, tau, cap, row_start, row_stride, valid, allowed=None):
    nq, nrows = dense.shape
    grow = row_start + row_stride * np.arange(nrows, dtype=np.int64)
    for qi in range(nq):
        keep = dense[qi] > tau[qi]
        if allowed is not None:
            keep &= np.isin(grow, np.asarray(allowed[qi], dtype=np.int64))
        want = grow[keep]
        assert counts[qi] == want.size, (qi, int(counts[qi]), want.size)
        m = min(int(counts[qi]), cap)
        ent = lists[qi, :m]
        rows = ent["row"].astype(np.int64)
        assert np.unique(rows).size == m, qi                          # every listed row once ...
        assert np.isin(rows, want).all(), qi                          # ... and only rows above tau: with the count, the set
        assert valid[rows].all(), qi                                  # a skipped row never appears
        idx = (rows - row_start) // row_stride
        assert np.array_equal(ent["score"].view(np.uint32), dense[qi, idx].view(np.uint32)), qi   # the dense score, bit for bit


def below(x):
    return np.nextafter(np.float32(x), np.float32(-np.inf), dtype=np.float32)


FILTER_SCENARIOS = ["strict_greater", "just_above_tau", "all_pass_overflow", "none_pass", "mixed_thresholds", "masks"]
FILTER_CASES = [(dt, m, s) for dt in ("f16", "f32") for m in ("cosine", "l2") for s in FILTER_SCENARIOS
                if not (s == "masks" and m == "l2")]


@pytest.mark.parametrize("engine", list(ENGINES))
@pytest.mark.parametrize("case", FILTER_CASES, ids=["-".join(c) for c in FILTER_CASES])
def test_filter_lists_exactly_the_rows_above_tau(Y, case, engine):
    dtype, metric, scenario = case
    rng = np.random.default_rng(5)
    rows, special = filter_corpus_rows(dtype, metric, rng)
    n, d = rows.shape
    valid = np.isfinite(rows.astype(np.float64)).all(axis=1)
    if metric == "cosine":
        valid &= (rows.astype(np.float64) ** 2).sum(axis=1) > 1e-12
    c = make_corpus(Y, rows, metric)
    eng = ENGINES[engine]

    def run(q, tau, cap, start=0, stride=1, nrows=n, allowed=None):
        dense = c.debug_stage1_scores(q, eng, row_start=start, row_stride=stride, nrows=nrows)
        counts, lists = c.debug_stage1_candidates(q, eng, tau, cap, row_start=start, row_stride=stride, nrows=nrows,
                                                  allowed=allowed)
        check_lists(dense, counts, lists, tau, cap, start, stride, valid, allowed)
        return dense, counts, lists

    def near(i, nq):
        """nq copies of a query next to row i: its score is the largest of the row's tile, so the row-level pre-filter
        decides with no slack from other columns"""
        r = rows[i].astype(np.float64)
        base = r / np.linalg.norm(r) if metric == "cosine" else r      # a cosine query of norm ~1e-6 would be rejected
        x = (base * 1.3 + rng.standard_normal(d) * 1e-3 * np.abs(base).max()).astype(np.float32)
        return np.repeat(x[None, :], nq, axis=0)

    q_rand = (rng.standard_normal((65, d)) * 2.0).astype(np.float32)
    if scenario == "strict_greater":
        # tau equal to a dense score: that row and its equals are NOT listed
        dense = c.debug_stage1_scores(q_rand, eng)
        tau = np.sort(dense, axis=1)[:, -50].copy()
        run(q_rand, tau, n)
        for i in (int(special[0]), 1000):
            for nq in (1, 65):
                q = near(i, nq)
                s = c.debug_stage1_scores(q, eng)[:, i]
                _, counts, lists = run(q, s.copy(), n)
                assert not np.isin(i, lists[0, :counts[0]]["row"])
    elif scenario == "just_above_tau":
        # rows scoring one float step above tau sit inside the pre-filter's slack (several score units for |r|^2 ~ 1e6)
        for i in [int(x) for x in special[:4]] + [1000, 2001]:
            for nq in (1, 65):
                q = near(i, nq)
                s = c.debug_stage1_scores(q, eng)[:, i]
                _, counts, lists = run(q, below(s), n)
                assert np.isin(i, lists[0, :counts[0]]["row"]), (i, nq)
    elif scenario == "all_pass_overflow":
        cap = 100
        _, counts, _ = run(q_rand, np.full(len(q_rand), -np.inf, np.float32), cap)
        assert np.all(counts == valid.sum()) and counts[0] > cap
    elif scenario == "none_pass":
        _, counts, _ = run(q_rand, np.full(len(q_rand), np.inf, np.float32), n)
        assert not counts.any()
    elif scenario == "mixed_thresholds":
        # one query tile of very different thresholds (its minimum is far below most columns) + a partial second tile,
        # over the strided sampling pass
        q = (rng.standard_normal((257, d)) * 2.0).astype(np.float32)
        q[::9] = near(1000, 1)[0]
        start, stride = 3, 5
        nrows = (n - 1 - start) // stride + 1
        dense = c.debug_stage1_scores(q, eng, row_start=start, row_stride=stride, nrows=nrows)
        srt = np.sort(dense, axis=1)
        pick = [np.full(257, -np.inf), np.full(257, np.inf), srt[:, -3], below(srt[:, -20]), srt[:, nrows // 2],
                np.full(257, 1e30), np.full(257, -1e30), below(srt[:, -1])]
        tau = np.array([pick[(i + 2) % len(pick)][i] for i in range(257)], dtype=np.float32)
        run(q, tau, nrows, start, stride, nrows)
    else:
        allowed = [np.zeros(0, np.int64), np.array([1000], np.int64), np.arange(n, dtype=np.int64),
                   np.sort(rng.choice(n, n // 2, replace=False)).astype(np.int64),
                   np.array([3, 5, 9, 17, 1000, n + 3, n + 70], np.int64)]
        q = q_rand[:5].copy()
        q[1] = near(1000, 1)[0]
        for tau in (np.full(5, -np.inf, np.float32), np.median(c.debug_stage1_scores(q, eng), axis=1).astype(np.float32)):
            run(q, tau, n, allowed=allowed)
    c.close()
