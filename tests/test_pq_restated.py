"""The numpy restatement of the SimeonPqAdc engine (tests/pq_restated.py) anchored to the reference, without a GPU:

* its float32 FMA against exact rational arithmetic, on random triples and on the triples where rounding the float64 sum
  twice goes wrong, subnormal and overflowing results included;
* on the inputs of the PQ parity tests (tests/test_gpu_pq.py, tests/test_gpu_documents.py) it reproduces the reference
  engine's stored codes and answers (tests/golden/ref_checks.json, ref_pq_candidates.json), which makes it a stand-in for
  the reference at shapes no stored answer covers;
* where the reference build exists (oracle/_ref), its encoder, lookup table and ADC sums equal simeon's own on a grid of
  subspace widths and centroid counts with duplicate, huge and NaN centroids and rows at the edges of normalisation."""
import json
from fractions import Fraction

import numpy as np
import pytest

from tests import pq_restated as R
from tests import ref_checks
from tests import test_gpu_documents as TD
from tests import test_gpu_pq as TP

F32 = np.float32


def round_f32(x: Fraction) -> float:
    """x rounded to nearest-even float32 (subnormals, overflow to inf), as a Python float"""
    if x == 0:
        return 0.0
    sign = -1.0 if x < 0 else 1.0
    a = abs(x)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if Fraction(2) ** e > a:
        e -= 1
    q = Fraction(2) ** (max(e, -126) - 23)
    n = a / q
    fl = n.numerator // n.denominator
    rem = n - fl
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and fl % 2 == 1):
        fl += 1
    v = fl * q
    if v >= Fraction(2) ** 128:
        return sign * float("inf")
    return sign * float(v)


def exact_fma(a, b, c) -> np.ndarray:
    return np.array([round_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))) for x, y, z in zip(a, b, c)], dtype=F32)


def same_bits(a, b) -> np.ndarray:
    """elementwise: equal bit patterns, or both NaN"""
    a = np.asarray(a, dtype=F32)
    b = np.asarray(b, dtype=F32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def rand_f32(rng, n, lo, hi):
    """random float32 of random sign with exponents uniform in [lo, hi)"""
    return (rng.choice([-1.0, 1.0], n) * rng.uniform(1, 2, n) * 2.0 ** rng.integers(lo, hi, n)).astype(F32)


def test_fma_emulation_random_triples():
    rng = np.random.default_rng(1)
    n = 4000
    cases = [
        (rand_f32(rng, n, -20, 20), rand_f32(rng, n, -20, 20), rand_f32(rng, n, -40, 40)),
        (rand_f32(rng, n, -80, -60), rand_f32(rng, n, -80, -60), rand_f32(rng, n, -150, -126)),   # subnormal products and sums
        (rand_f32(rng, n, 60, 64), rand_f32(rng, n, 60, 66), rand_f32(rng, n, 120, 128)),        # near and past the overflow
    ]
    for a, b, c in cases:
        got = R.fma32(a, b, c)
        want = exact_fma(a, b, c)
        assert np.all(same_bits(got, want)), np.nonzero(~same_bits(got, want))[0][:5]
    sub = R.fma32(*cases[1])
    assert np.any((sub != 0) & (np.abs(sub) < np.finfo(F32).tiny))
    assert np.any(np.isinf(R.fma32(*cases[2])))


def test_fma_emulation_where_double_rounding_fails():
    """Triples whose float64 sum lands on a float32 halfway point that the exact sum is not on: rounding twice picks the
    wrong neighbour there; the emulator must not."""
    # 8384513 * 8392705 = 2^46 + 1: with a = 8384513 * 2^(s-35), b = 8392705 * 2^-35, c = 2^s the exact sum is
    # 2^s (1 + 2^-24 + 2^-70), a hair above a float32 halfway point; its float64 rounding is the halfway point itself
    A, B = 8384513, 8392705
    assert A * B == 2 ** 46 + 1
    s = np.arange(-100, 100)
    sign = np.where(s % 2 == 0, 1.0, -1.0)
    a = (sign * A * 2.0 ** (s - 35)).astype(F32)
    b = np.full(len(s), B * 2.0 ** -35, dtype=F32)
    c = (sign * 2.0 ** s).astype(F32)
    want = exact_fma(a, b, c)
    naive = (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(F32)
    assert not np.any(same_bits(naive, want))
    assert np.all(same_bits(R.fma32(a, b, c), want))
    assert np.all(np.abs(want) == np.abs(c) * F32(1 + 2.0 ** -23))
    # the same just below a halfway point (a negative product): the exact sum rounds down, the twice-rounded one up
    c2 = c * F32(1 + 2.0 ** -22)
    want = exact_fma(-a, b, c2)
    naive = ((-a).astype(np.float64) * b.astype(np.float64) + c2.astype(np.float64)).astype(F32)
    assert not np.any(same_bits(naive, want))
    assert np.all(same_bits(R.fma32(-a, b, c2), want))
    assert np.all(np.abs(want) == np.abs(c) * F32(1 + 2.0 ** -23))
    # exact halfway points: 1 + 2^-24 is a tie (to even: 1), a hair above / below it is not
    one, h = F32(1.0), F32(2.0 ** -24)
    got = R.fma32([h, h, h, -h], [F32(1.0), F32(1 + 2.0 ** -23), F32(1 - 2.0 ** -24), F32(1.0)], [one, one, one, F32(2.0)])
    assert list(got) == [F32(1.0), np.nextafter(one, F32(2)), F32(1.0), F32(2.0)]
    # signed zeros, infinities and NaN follow IEEE
    z = R.fma32([F32(-0.0), F32(np.inf), F32(np.inf), F32(1.0)], [F32(1.0), F32(0.0), F32(1.0), F32(np.nan)],
                [F32(-0.0), F32(1.0), F32(-np.inf), F32(1.0)])
    assert np.signbit(z[0]) and z[0] == 0 and np.isnan(z[1]) and np.isnan(z[2]) and np.isnan(z[3])


# ---- the restatement reproduces the reference's stored answers ------------------------------------------------------------

def check_answers(index, queries, k, rf, thr, want):
    for qi, q in enumerate(queries):
        r, s, cnt, _ = index.search(q, k, rf, thr)
        assert cnt == want[qi][0], (qi, k)
        assert ref_checks.digest(r[:cnt], s[:cnt]) == want[qi][1], (qi, k)


@pytest.mark.parametrize("cfg", TP.PQ_CFGS)
def test_restatement_reproduces_the_reference_pq_answers(oracle, cfg):
    want = ref_checks.load()["pq"][ref_checks.key(cfg)]
    cs = TP.pq_case(oracle, cfg)
    index = R.Index(cs["rows"], cs["rowids"], cs["m"], cs["kc"], cs["codebooks"], cs["tie_keys"])
    assert ref_checks.digest(index.codes) == want["codes"]
    for (k, rf, thr), results in zip(TP.PQ_SEARCHES, want["searches"]):
        check_answers(index, cs["queries"], k, rf, thr, results)


def test_restatement_reproduces_the_reference_fp16_large_and_overflow_answers(oracle):
    g = ref_checks.load()
    cs = TP.pq_fp16_case(oracle)
    index = R.Index(cs["held"], np.arange(len(cs["held"]), dtype=np.int64), cs["m"], cs["kc"], cs["codebooks"])
    check_answers(index, cs["queries"], *TP.PQ_FP16_SEARCH, g["pq_fp16"])
    cs = TP.pq_large_case(oracle)
    index = R.Index(cs["rows"], cs["rowids"], cs["m"], cs["kc"], cs["codebooks"], cs["tie_keys"])
    for (k, rf, thr), results in zip(TP.PQ_LARGE_SEARCHES, g["pq_large"]):
        check_answers(index, cs["queries"], k, rf, thr, results)
    cs = TP.pq_overflow_case(oracle)
    index = R.Index(cs["rows"], cs["rowids"], cs["m"], cs["kc"], cs["codebooks"], cs["tie_keys"])
    check_answers(index, cs["query"], *TP.PQ_OVERFLOW_SEARCH, g["pq_overflow"])


def test_restatement_reproduces_the_reference_summation_order_answers(oracle):
    """the candidate-set "order" case: approximate scores equal in exact arithmetic, decided by the float order of the sum"""
    with open(TD.PQC_GOLDEN) as f:
        want = json.load(f)["order"]
    cs = TD.pq_order_case(oracle)
    n = len(cs["rows"])
    index = R.Index(cs["rows"], cs["rowids"], cs["m"], cs["kc"], cs["codebooks"], np.arange(n, dtype=np.uint64))
    assert np.array_equal(index.codes, cs["codes"])
    pos_of = {int(r): j for j, r in enumerate(cs["rowids"][index.idx_rows])}
    for qi, (q, lst) in enumerate(zip(cs["queries"], cs["lists"])):
        r, s, cnt, _ = index.search(q, 1, 1, -1.0, positions=np.array(sorted(pos_of[int(x)] for x in lst)))
        assert [cnt, ref_checks.digest(r[:cnt], s[:cnt])] == want["searches"][0][qi], qi


# ---- the restatement against simeon's own encoder and lookup table ---------------------------------------------------------

GRID_K = (2, 3, 33, 100, 255, 256)
GRID_DSUB = (1, 3, 15, 16, 17, 31, 32, 33, 48, 768)


def grid_case(O, k: int, dsub: int, n: int = 96):
    """A small index at (k centroids, dsub) whose edges the encoder and the lookup table must get right.
    m = 3 subspaces (m = 1 at dsub = 768): subspace 0 holds duplicate centroids (1 and k - 1; 0 and 1 when k = 2) and
    centroids at +-1e20 (squared distances overflow to inf); subspace 1 (m = 3) is NaN everywhere, so every row's code there
    is 0; the last subspace holds the duplicates again and one NaN entry in centroid k // 2 (not at m = 1, k < 5, where
    it would hit a duplicate).  Rows: Gaussian rows, rows at
    centroid dup[0] (ties between the duplicates), one-element rows whose squared norm is just above / at most 1e-20, a zero row,
    a row with an inf and one with a NaN element.  -> dict(rows f32[n, d], codebooks, m, queries f32[5, d])"""
    m = 1 if dsub == 768 else 3
    d = m * dsub
    rng = np.random.default_rng(1000 * k + dsub)
    cb = (rng.normal(size=(m, k, dsub)) / np.sqrt(d)).astype(F32)
    dup = (0, 1) if k == 2 else (1, k - 1)
    base = rng.normal(size=d)
    base = (base / np.linalg.norm(base)).astype(F32)              # a unit row: normalising it changes (almost) nothing
    for mi in {0, m - 1}:
        cb[mi, dup[0]] = cb[mi, dup[1]] = base[mi * dsub:(mi + 1) * dsub]
    if k >= 4:
        cb[0, 2] = F32(1e20)
        cb[0, 3] = F32(-1e20)
    if m == 3:
        cb[1] = np.nan
    if m == 3 or k >= 5:
        cb[m - 1, k // 2, 0] = np.nan
    rows = (rng.normal(size=(n, d)) / np.sqrt(d)).astype(F32)
    rows[10:22] = base[None, :] + (rng.normal(size=(12, d)) * 1e-4 / np.sqrt(d)).astype(F32)
    v = F32(1e-10)
    while float(v) ** 2 <= 1e-20:
        v = np.nextafter(v, F32(1))
    rows[30] = 0
    rows[30, 0] = v                                   # |r|^2 just above 1e-20: indexed
    rows[31] = 0
    rows[31, d - 1] = np.nextafter(v, F32(0))         # |r|^2 <= 1e-20: left out
    rows[32] = 0                                      # left out
    rows[33, 0] = np.inf                              # indexed: normalises to NaN and zeros
    rows[34, d // 2] = np.nan                         # indexed: normalises to NaN everywhere, code 0
    rows[35] *= F32(1e-9)                             # small but normal
    queries = (rng.normal(size=(5, d)) / np.sqrt(d)).astype(F32)
    queries[1] = F32(1e30)                             # |q|^2 overflows float: inv = 0, a table of zeros (NaN at NaN centroids)
    queries[2] = rows[12]
    queries[3] *= F32(1e-12)
    return dict(rows=rows, codebooks=cb.reshape(-1), m=m, queries=queries)


def test_grid_normalisation_edges(oracle):
    cs = grid_case(oracle, 33, 17)
    _, ok = R.normalise(cs["rows"])
    assert ok[30] and not ok[31] and not ok[32] and ok[33] and ok[34] and ok[35]


@pytest.mark.parametrize("k", GRID_K)
def test_restatement_matches_simeon_encode_lut_and_adc(oracle, k):
    O = oracle
    if not O.ref_available():
        pytest.skip("the reference build (oracle/_ref) is not present")
    for dsub in GRID_DSUB:
        cs = grid_case(O, k, dsub)
        rows, cb, m = cs["rows"], cs["codebooks"], cs["m"]
        d = rows.shape[1]
        normed, ok = R.normalise(rows)
        codes = R.encode(normed, cb, m, k)
        assert np.array_equal(codes, O.pq_encode_ref(cb, d, m, k, normed)), (k, dsub)
        if m == 3:
            assert np.all(codes[:, 1] == 0)
        assert np.all(codes[np.count_nonzero(ok[:34])] == 0)          # the NaN row: code 0 everywhere
        dup = (0, 1) if k == 2 else (1, k - 1)
        ties = codes[10:22, 0]
        assert np.all(ties != dup[1]) and np.any(ties == dup[0]), (k, dsub)   # duplicates: the lower index wins
        qn, qok = R.normalise(cs["queries"])
        for q in qn:
            want_scores, want_lut = O.pq_scores_ref(cb, d, m, k, q, codes)
            table = R.lut(q, cb, m, k)
            assert np.all(same_bits(table.reshape(-1), want_lut)), (k, dsub)
            assert np.all(same_bits(R.adc(codes, table), want_scores)), (k, dsub)
