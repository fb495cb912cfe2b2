"""The exact scan's chain after stage 1 (DESIGN.md §4.2), each link against a plain float64 / numpy restatement:

  * top-K' selection (topk_select_kernel): the selected (score, row) pairs, their number and the certificate's `bound`;
  * the threshold calibration (the same kernel in tau_only mode): exact K-th best, the 12-bit histogram with its radix
    fallback, and the one-pass fast_tau restated thread share by thread share;
  * final ordering and the exactness certificate (final_kernel): order, rowid mapping, padding, TIE_AT_K and the
    certified / queued decision, including the L2 rule's rounding margin as a function of d;
  * the direct path's stage-1 engine (gather_score_kernel) within eps of float64, with the skip rule;
  * end to end: a query the certificate rejects is resolved exhaustively inside its candidate set, on every path.

Order of (score, row) pairs everywhere: score descending in the kernels' key order (-0 below +0, NaN below -inf), then row
ascending."""
import numpy as np
import pytest

from yams_b200._lib import CAND_DTYPE, EXACT_DTYPE

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
NO_ROW = 0xFFFFFFFF


@pytest.fixture(scope="module")
def Y():
    import yams_b200
    assert yams_b200.device_count() > 0
    assert yams_b200.plugin_init() == 0, yams_b200.health()
    return yams_b200


@pytest.fixture(scope="module")
def ws(Y):
    """an empty corpus: the workspace of the selection diagnostics"""
    c = Y.Corpus(8, Y.F32, Y.COSINE)
    yield c
    c.close()


# ---------------------------------------------------------------------------------------------------------------------
# float keys and the reference order
# ---------------------------------------------------------------------------------------------------------------------
def fkey(s):
    """the kernels' monotone 32-bit key of a float32 score (NaN -> 0, the lowest)"""
    s = np.asarray(s, dtype=np.float32)
    b = s.view(np.uint32).astype(np.uint64)
    k = np.where(b >> 31, (~b) & 0xFFFFFFFF, b | 0x80000000)
    return np.where(np.isnan(s), 0, k).astype(np.uint64)


def from_key(k):
    k = np.asarray(k, dtype=np.uint64)
    return np.where(k & 0x80000000, k & 0x7FFFFFFF, (~k) & 0xFFFFFFFF).astype(np.uint32).view(np.float32)


def ref_order(scores, rows):
    """indices sorted by (score desc in key order, row asc)"""
    return np.lexsort((np.asarray(rows, dtype=np.int64), -fkey(scores).astype(np.int64)))


def same_bits(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and bool(np.all((a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))))


def spread_rows(L, rng):
    """L distinct row indices spread over [0, 2^32 - 2] (0xFFFFFFFF is the 'no row' value)"""
    return ((rng.permutation(L).astype(np.uint64) * 2654435761 + 12345) % NO_ROW).astype(np.uint32)


# ---------------------------------------------------------------------------------------------------------------------
# 1-2. selection: exact top-K and bound
# ---------------------------------------------------------------------------------------------------------------------
DISTRIBUTIONS = ["random", "all_equal", "two_values", "straddle", "ulp_apart", "signed_zeros", "subnormal", "inf_nan"]


def scores_of(name, L, K, rng):
    if name == "random":
        return rng.standard_normal(L).astype(np.float32)
    if name == "all_equal":
        return np.full(L, 0.5, np.float32)
    if name == "two_values":
        return np.where(rng.uniform(size=L) < 0.5, 1.0, -1.0).astype(np.float32)
    if name == "straddle":
        # K // 2 clear winners, then one score shared by the rest: the K-th place falls inside the group, which the
        # selection must cut by row
        s = np.full(L, 0.25, np.float32)
        s[rng.permutation(L)[: K // 2]] = 2.0 + rng.uniform(size=min(K // 2, L)).astype(np.float32)
        return s
    if name == "ulp_apart":
        return (np.float32(0.7).view(np.uint32) + rng.permutation(L).astype(np.uint32)).view(np.float32)
    if name == "signed_zeros":
        v = np.array([-0.0, 0.0, -1e-30, 1e-30, -0.5, 0.5], np.float32)
        return v[rng.integers(0, len(v), L)]
    if name == "subnormal":
        b = rng.integers(1, 1 << 23, L).astype(np.uint32) | (rng.integers(0, 2, L).astype(np.uint32) << 31)
        return b.view(np.float32)
    assert name == "inf_nan"
    s = rng.standard_normal(L).astype(np.float32)
    u = rng.uniform(size=L)
    s[u < 0.3] = -np.inf
    s[(u >= 0.3) & (u < 0.4)] = np.nan
    s[(u >= 0.4) & (u < 0.45)] = np.inf
    return s


def straddle_rows(L, rng):
    """the straddle case's rows: half of them near 0, half near 2^32 - 2 (the low key word decides the cut)"""
    lo = np.arange(L // 2, dtype=np.uint64)
    hi = NO_ROW - 1 - np.arange(L - L // 2, dtype=np.uint64)
    return rng.permutation(np.concatenate([lo, hi])).astype(np.uint32)


def check_selection(sel, n, bound, scores, rows, K, want_bound, where):
    order = ref_order(scores, rows)
    m = min(K, len(scores))
    assert n == m, (where, int(n), m)
    top = order[:m]
    assert np.array_equal(sel["row"][:m], rows[top]), where
    assert same_bits(sel["score"][:m], scores[top]), where
    assert same_bits(bound, want_bound), (where, bound, want_bound)
    rest = scores[order[m:]]
    rest = rest[~np.isnan(rest)]
    assert not (rest > bound).any(), where                 # every unselected score is covered by the bound


def select_lengths(K):
    return sorted({L for L in (0, 1, K - 1, K, K + 1, 4095, 4096, 4097, 8192, 65536) if L >= 0})


SELECT_CASES = [(K, L) for K in (1, 31, 32, 64, 3840, 4096) for L in select_lengths(K)]


@pytest.mark.parametrize("K,L", SELECT_CASES, ids=[f"K{K}-L{L}" for K, L in SELECT_CASES])
def test_select_exact_top_k(ws, K, L):
    """Every distribution at once (one query each): dense input over three row layouts (rows 0.., row_start > 0 with
    row_stride 7, rows ending at 2^32 - 2), and candidate lists of scattered rows with a list threshold."""
    rng = np.random.default_rng(K * 100_003 + L)
    S = np.stack([scores_of(name, L, K, rng) for name in DISTRIBUTIONS]) if L else np.zeros((len(DISTRIBUTIONS), 0), np.float32)
    nq = len(DISTRIBUTIONS)
    for start, stride in ((0, 1), (123, 7), (NO_ROW - 1 - max(L - 1, 0), 1)):
        rows = (start + stride * np.arange(L, dtype=np.uint64)).astype(np.uint32)
        sel, n, bound = ws.debug_select(K, dense=S, row_start=start, row_stride=stride)
        for q in range(nq):
            want = S[q][ref_order(S[q], rows)[K - 1]] if L > K else np.float32(-np.inf)
            check_selection(sel[q], n[q], bound[q], S[q], rows, K, want, ("dense", DISTRIBUTIONS[q], start, stride))
    if L > 8192:
        return
    cands = np.zeros((nq, max(L, 1)), CAND_DTYPE)
    R = np.empty((nq, L), np.uint32)
    for q, name in enumerate(DISTRIBUTIONS):
        R[q] = straddle_rows(L, rng) if name == "straddle" else spread_rows(L, rng)
        cands[q, :L]["score"], cands[q, :L]["row"] = S[q], R[q]
    tau = np.full(nq, -0.125, np.float32)
    sel, n, bound = ws.debug_select(K, cands=cands, counts=np.full(nq, L, np.uint32), tau=tau)
    for q in range(nq):
        want = S[q][ref_order(S[q], R[q])[K - 1]] if L > K else tau[q]
        check_selection(sel[q], n[q], bound[q], S[q], R[q], K, want, ("lists", DISTRIBUTIONS[q]))


@pytest.mark.parametrize("K", [1, 32, 3840])
def test_select_bound_rules(ws, K):
    """bound: the K-th score when the input is longer than K, tau when a list is not, -inf for a dense input or a list
    without tau that is not, +inf when a list overflowed its capacity (the rows it lost are unknown)"""
    rng = np.random.default_rng(K)
    for L in (0, K - 1, K, K + 1, 5000):
        if L < 0:
            continue
        s = rng.standard_normal((3, L)).astype(np.float32)
        rows = np.stack([spread_rows(L, rng) for _ in range(3)])
        cands = np.zeros((3, max(L, 1)), CAND_DTYPE)
        cands[:, :L]["score"], cands[:, :L]["row"] = s, rows
        kth = [s[q][ref_order(s[q], rows[q])[K - 1]] if L > K else None for q in range(3)]
        tau = np.array([-0.5, -np.inf, 3.0], np.float32)
        _, _, b = ws.debug_select(K, cands=cands, counts=np.full(3, L, np.uint32), tau=tau)
        assert same_bits(b, [kth[q] if L > K else tau[q] for q in range(3)]), (L, b)
        _, _, b = ws.debug_select(K, cands=cands, counts=np.full(3, L, np.uint32))
        assert same_bits(b, [kth[q] if L > K else -np.inf for q in range(3)]), (L, b)
        _, _, b = ws.debug_select(K, dense=s)
        assert same_bits(b, [kth[q] if L > K else -np.inf for q in range(3)]), (L, b)
        # overflow: counts beyond cap -> +inf, whatever the list holds; the selection is over the cap entries it has
        counts = np.array([L + 1, L + 1000, 0xFFFFFFFF], np.uint32)
        sel, n, b = ws.debug_select(K, cands=cands[:, :L] if L else cands[:, :0], counts=counts, tau=tau)
        assert np.all(b == np.inf), (L, b)
        for q in range(3):
            check_selection(sel[q], n[q], np.float32(np.inf), s[q], rows[q], K, np.float32(np.inf), ("overflow", L, q))


# ---------------------------------------------------------------------------------------------------------------------
# 3. thresholds (tau_only)
# ---------------------------------------------------------------------------------------------------------------------
def kth_best(s, K):
    return np.sort(fkey(s))[::-1][K - 1]


def fast_tau_ref(s, K, aligned, threads=256):
    """the one-pass threshold restated: thread t keeps the largest key of float4 units i = t (mod 256) plus its share of the
    scalar tail (aligned rows), or of elements i = t (mod 256); the K-th largest of the 256 maxima"""
    L = len(s)
    keys = fkey(s)
    if aligned:
        n4 = L // 4
        owner = np.concatenate([(np.arange(n4 * 4) // 4) % threads, np.arange(L - n4 * 4) % threads])
    else:
        owner = np.arange(L) % threads
    mx = np.zeros(threads, np.uint64)
    np.maximum.at(mx, owner, keys)
    return np.sort(mx)[::-1][K - 1]


def tau_of(key, margin):
    return from_key(key) - np.float32(margin)


def test_thresholds_short_and_exact_paths(ws):
    rng = np.random.default_rng(3)
    margin = np.float32(2e-3)
    # fewer items than K -> -inf; exactly K -> their minimum - margin (dense and lists)
    s = rng.standard_normal((2, 50)).astype(np.float32)
    assert np.all(ws.debug_select(51, dense=s, tau_only=True, tau_margin=margin) == -np.inf)
    t = ws.debug_select(50, dense=s, tau_only=True, tau_margin=margin)
    assert same_bits(t, s.min(axis=1) - margin)
    cands = np.zeros((2, 64), CAND_DTYPE)
    cands[:, :50]["score"], cands[:, :50]["row"] = s, np.arange(50)
    t = ws.debug_select(50, cands=cands, counts=np.array([50, 49], np.uint32), tau_only=True, tau_margin=margin)
    assert same_bits(t, [s[0].min() - margin, -np.inf])
    # the 12-bit histogram: exactly the K-th best - margin
    for L in (5000, 32768):
        S = np.stack([scores_of(name, L, 8, rng) for name in ("random", "ulp_apart", "subnormal", "signed_zeros")])
        for K in (1, 8, 17, 100, 3000):
            t = ws.debug_select(K, dense=S, tau_only=True, tau_margin=margin)
            assert same_bits(t, [tau_of(kth_best(S[q], K), margin) for q in range(len(S))]), (L, K)
    # a crowded boundary bin (> 2048 keys share the top 12 bits: scores in [1, 1.125)) -> the radix fallback
    L = 8192
    S = rng.uniform(-1.0, 0.9, size=(3, L)).astype(np.float32)
    S[0, :3000] = rng.uniform(1.0, 1.125, size=3000).astype(np.float32)
    S[1, :2100] = (np.float32(1.0).view(np.uint32) + rng.permutation(2100).astype(np.uint32)).view(np.float32)
    S[2, :] = 1.0625                                                   # one value: the whole input in one bin
    S = np.stack([rng.permutation(x) for x in S])
    for K in (1, 1500, 2099, 2100, 2101, 5000):
        t = ws.debug_select(K, dense=S, tau_only=True, tau_margin=margin)
        assert same_bits(t, [tau_of(kth_best(S[q], K), margin) for q in range(3)]), K


@pytest.mark.parametrize("shift", [0, 1, 2, 3])
def test_fast_tau_per_thread_shares(ws, shift):
    """fast_tau (K <= 16, L >= 4096): equal to the restated per-thread maxima, on 16-byte aligned rows (float4 loads + scalar
    tail) and unaligned ones (scalar loads); never above the true K-th best"""
    rng = np.random.default_rng(10 + shift)
    for L in (4096, 4099, 10001, 65536):
        S = np.stack([scores_of(n, L, 8, rng) for n in ("random", "ulp_apart", "signed_zeros", "two_values", "inf_nan")])
        S[0, :16] = 5.0 + np.arange(16, dtype=np.float32)              # the top 16 in a few thread shares
        S[1, ::256] = 7.0                                               # all in thread 0's share
        for K in (1, 2, 8, 16):
            for margin in (0.0, 2e-3):
                t = ws.debug_select(K, dense=S, dense_shift=shift, tau_only=True, tau_margin=margin, fast_tau=True)
                want = [tau_of(fast_tau_ref(S[q], K, (shift + q * L) % 4 == 0), margin) for q in range(len(S))]
                assert same_bits(t, want), (L, K, margin)
                if margin == 0.0:
                    assert all(fkey(t[q]) <= kth_best(S[q], K) for q in range(len(S))), (L, K)
    # below the fast path's size or above its K the exact threshold is used even when fast_tau is asked for
    S = rng.standard_normal((2, 4095)).astype(np.float32)
    assert same_bits(ws.debug_select(8, dense=S, dense_shift=shift, tau_only=True, fast_tau=True),
                     [from_key(kth_best(S[q], 8)) for q in range(2)])
    S = rng.standard_normal((2, 5000)).astype(np.float32)
    assert same_bits(ws.debug_select(17, dense=S, dense_shift=shift, tau_only=True, fast_tau=True),
                     [from_key(kth_best(S[q], 17)) for q in range(2)])


# ---------------------------------------------------------------------------------------------------------------------
# 4. final ordering and the certificate
# ---------------------------------------------------------------------------------------------------------------------
FINAL_ROWS = 5000
FINAL_ROWIDS = 1_000_003 + 7 * np.arange(FINAL_ROWS, dtype=np.int64)


@pytest.fixture(scope="module")
def fin(Y):
    c = Y.Corpus(8, Y.F32, Y.COSINE)
    c.append(np.ones((FINAL_ROWS, 8), np.float32), rowids=FINAL_ROWIDS)
    yield c
    c.close()


def ref_final(ex, ex_n, k, negate):
    """-> (rowids, scores, count, tie flag, sorted valid sims) of one query"""
    m = len(ex) if ex_n is None else int(ex_n)
    e = ex[:m]
    e = e[~np.isnan(e["sim"])]
    order = ref_order(e["sim"], e["row"])
    sims, rows = e["sim"][order], e["row"][order]
    nout = min(len(e), k)
    pad = np.float32(np.inf if negate else -np.inf)
    rid = np.full(k, -1, np.int64)
    sc = np.full(k, pad, np.float32)
    rid[:nout] = FINAL_ROWIDS[rows[:nout]]
    sc[:nout] = -sims[:nout] if negate else sims[:nout]
    tie = len(e) > k and fkey(sims[k - 1]) == fkey(sims[k])
    return rid, sc, nout, tie, sims


def random_exact(rng, nq, Kp):
    ex = np.zeros((nq, Kp), EXACT_DTYPE)
    vals = np.array([0.9, 0.5, 0.5, 0.25, -0.0, 0.0, -0.75, np.nan], np.float32)
    for q in range(nq):
        ex[q]["sim"] = vals[rng.integers(0, len(vals), Kp)] if q % 2 else rng.standard_normal(Kp).astype(np.float32)
        ex[q]["row"] = rng.choice(FINAL_ROWS, Kp, replace=False)
    return ex


@pytest.mark.parametrize("metric", ["cosine", "l2"])
def test_final_order_mapping_padding_ties(Y, fin, metric):
    rng = np.random.default_rng(5)
    m = Y.L2 if metric == "l2" else Y.COSINE
    for Kp, k in ((64, 1), (64, 10), (64, 64), (64, 100), (4096, 3000), (1, 1)):
        nq = 6
        ex = random_exact(rng, nq, Kp)
        ex_n = np.array([Kp, Kp // 2, 0, Kp, max(Kp - 3, 0), Kp], np.uint32)
        # query 5: the k-th and (k+1)-th equal (tie); query 3: equal except for the sign of zero (not a tie)
        if Kp > k:
            ex[5]["sim"] = 0.125
            ex[5]["sim"][: k - 1] = 0.5
            ex[3]["sim"] = 0.0
            ex[3]["sim"][k:] = -0.0
        for use_n in (False, True):
            got = fin.debug_final(ex, k, bound=np.full(nq, -np.inf), eps=np.full(nq, 1e-6), metric=m,
                                  ex_n=ex_n if use_n else None)
            rid, sc, cnt, flags, queued = got
            assert queued.size == 0 and not np.any(flags & Y.FLAG_FALLBACK_PATH)
            for q in range(nq):
                wr, ws_, wc, tie, _ = ref_final(ex[q], ex_n[q] if use_n else None, k, metric == "l2")
                assert np.array_equal(rid[q], wr), (Kp, k, q)
                assert same_bits(sc[q], ws_), (Kp, k, q)
                assert cnt[q] == wc, (Kp, k, q)
                assert bool(flags[q] & Y.FLAG_TIE_AT_K) == tie, (Kp, k, q)
            if Kp > k:
                assert flags[5] & Y.FLAG_TIE_AT_K and not flags[3] & Y.FLAG_TIE_AT_K


def cert_ref(sims, k, bd, e, thr):
    """the cosine certificate restated in float32: bound + eps < (k-th exact score, or the threshold with < k of them)"""
    if bd == -np.inf:
        return True
    lvl = sims[k - 1] if len(sims) >= k else np.float32(thr)
    return bool(np.float32(bd) + np.float32(e) < lvl)


def run_cert_cases(Y, fin, cases, k, Kp, thr, level):
    """cases: (sims list, bound, eps) -> checks flags and the queue against cert_ref"""
    nq = len(cases)
    ex = np.zeros((nq, Kp), EXACT_DTYPE)
    ex["sim"] = np.nan
    for q, (sims, _, _) in enumerate(cases):
        ex[q, : len(sims)]["sim"] = sims
        ex[q, : len(sims)]["row"] = np.arange(len(sims)) + 10 * q
    bd = np.array([c[1] for c in cases], np.float32)
    e = np.array([c[2] for c in cases], np.float32)
    rid, sc, cnt, flags, queued = fin.debug_final(ex, k, bound=bd, eps=e, threshold=thr, level=level)
    want = np.array([cert_ref(ref_final(ex[q], None, k, False)[4], k, bd[q], e[q], thr) for q in range(nq)])
    fb = (flags & Y.FLAG_FALLBACK_PATH) != 0
    assert np.array_equal(fb, ~want if level == 0 else np.ones(nq, bool)), (fb, want)
    assert sorted(queued.tolist()) == list(np.nonzero(~want)[0]), (queued, want)
    return want


def test_cosine_certificate_decision(Y, fin):
    f = np.float32
    half, e10 = f(0.5), f(2.0 ** -10)
    sims = [f(0.9), f(0.7), half, f(0.3)]
    cases = [
        (sims, -np.inf, 1.0),                         # nothing outside the survivors
        (sims, np.inf, 1e-6),                         # a list overflowed: never certified
        (sims, f(0.4), f(1e-3)),                      # clear
        (sims, half - e10, e10),                      # bound + eps lands exactly on the k-th score: not certified
        (sims, half - e10 - f(2.0 ** -24), e10),      # one float step below it: certified
        (sims, half, f(0.0)),                         # bound equal to the k-th score, eps 0
        ([f(0.9), f(0.8)], f(0.2), f(0.05)),          # fewer than k valid: the threshold 0.3 decides, 0.25 < 0.3
        ([f(0.9), f(0.8)], f(0.25), f(0.05)),         # 0.3 == threshold: not certified
        ([f(0.9)], -np.inf, f(0.05)),
        ([], f(-0.5), f(0.1)),                        # no survivor at all, -0.4 < 0.3
        ([], f(0.5), f(0.1)),
    ]
    want = run_cert_cases(Y, fin, cases, 3, 8, 0.3, 0)
    assert list(want) == [True, False, True, False, True, False, True, False, True, True, False]
    # level 1 always flags; its failures go to the second queue
    run_cert_cases(Y, fin, cases, 3, 8, 0.3, 1)
    # randomised around the boundary: bound + eps within a few float steps of the k-th score
    rng = np.random.default_rng(9)
    cases = []
    for _ in range(400):
        s = np.sort(rng.uniform(-1, 1, 12).astype(np.float32))[::-1]
        e = f(rng.choice([0.0, 2.0 ** -20, 1e-5, 3e-4]))
        bd = f(s[4] - e)
        bd = (bd.view(np.uint32) + np.uint32(rng.integers(0, 5)) - np.uint32(2)).view(np.float32) if bd > 0 else bd
        cases.append((list(s[: rng.integers(3, 12)]), bd, e))
    run_cert_cases(Y, fin, cases, 5, 16, -1.0, 0)


def l2_rounding_factor(d):
    """The worst-case factor between dist_k^2 and the exact squared distance an unscored row needs to be certainly farther.
    The reference's float distance sums d terms fl(fl(q_i - r_i)^2): three roundings per term before the sum, then one per
    later addition -- d - 1 in the scalar loop, d/8 - 1 within an AVX lane plus 7 across lanes (d >= 16, d % 16 == 0) --
    and one more for the square root, which enters squared.  t roundings below 1 each: (1 - u)^-(t + 2)."""
    t = (d / 8 + 9) if (d >= 16 and d % 16 == 0) else (d + 2)
    return (1.0 - U) ** -(t + 2)


@pytest.mark.parametrize("d", [3, 16, 128, 1000, 1680, 1700, 4095, 4096, 65535])
def test_l2_certificate_margin_covers_float_rounding(Y, d):
    """The L2 rule |q|^2 - bound - eps > dist_k^2 * margin.  A row is left out safely only if its exact squared distance
    is above dist_k^2 * l2_rounding_factor(d): at 0.99 of that excess the kernel must not certify (scalar order, d >= 1674,
    needs more than the flat 1e-4 margin); above max(factor, 1 + 1e-4) it must.  The factor is checked against numpy float32
    sums in both orders on data made of equal terms (every addition rounds)."""
    # the stated bound holds for the reference's float arithmetic
    rng = np.random.default_rng(d)
    diff = (np.float32(1.0) + rng.integers(0, 1 << 20, size=(16, min(d, 4096))).astype(np.float32) * np.float32(U)).astype(np.float32)
    sq = (diff * diff).astype(np.float32)
    exact = (diff.astype(np.float64) ** 2).sum(axis=1)
    dd = sq.shape[1]
    if dd >= 16 and dd % 16 == 0:
        lanes = np.cumsum(sq.reshape(16, dd // 8, 8), axis=1, dtype=np.float32)[:, -1, :]
        fsum = np.cumsum(lanes, axis=1, dtype=np.float32)[:, -1]
    else:
        fsum = np.cumsum(sq, axis=1, dtype=np.float32)[:, -1]
    dist = np.sqrt(fsum).astype(np.float32).astype(np.float64)
    assert np.all(dist ** 2 * l2_rounding_factor(dd) >= exact)
    # the kernel's decision at both sides of the factor
    c = Y.Corpus(d, Y.F32, Y.L2)
    c.append(np.zeros((1, d), np.float32))
    dk = np.float32(2.0)
    need = l2_rounding_factor(d)
    used = max(need, 1.0001)
    targets = [1.0 + 0.99 * (need - 1.0), 1.0 + 1.01 * (used - 1.0), 1.5, 1.0]
    ex = np.zeros((len(targets), 1), EXACT_DTYPE)
    ex["sim"], ex["row"] = -dk, 0
    bd = np.array([-(float(dk) ** 2) * t for t in targets], np.float32)         # |q| = 0, eps = 0: the lower bound is -bound
    got = c.debug_final(ex, 1, bound=bd, eps=np.zeros(len(targets)), qnorm=np.zeros(len(targets)))
    fb = (got[3] & Y.FLAG_FALLBACK_PATH) != 0
    assert list(fb) == [True, False, False, True], (d, need, fb)
    # fewer than k survivors: never certified (the L2 rule has no threshold branch), however low the bound
    got = c.debug_final(ex[:1], 2, bound=np.full(1, -1e30), eps=np.zeros(1), qnorm=np.zeros(1))
    assert got[3][0] & Y.FLAG_FALLBACK_PATH and list(got[4]) == [0]
    c.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. the gather engine (direct path stage 1)
# ---------------------------------------------------------------------------------------------------------------------
GATHER_CASES = [(dt, d) for dt in ("f16", "f32") for d in (20, 30, 36, 64, 768)]


@pytest.mark.parametrize("dt,d", GATHER_CASES, ids=[f"{dt}-d{d}" for dt, d in GATHER_CASES])
def test_gather_engine_within_eps_and_skip_rule(Y, dt, d):
    """fp16 with d % 8 == 0 and fp32 with d % 4 == 0 take 16-byte loads, the rest the scalar loop.  Every listed row
    scores within eps of float64; zero, tiny-norm (sum r^2 <= 1e-12), inf and NaN rows score exactly -inf; unknown and
    repeated rowids give (-inf, 0xFFFFFFFF); an empty list gives nothing."""
    rng = np.random.default_rng(d * 7 + len(dt))
    n = 3000
    r = (rng.standard_normal((n, d)) * np.exp(rng.uniform(-2, 2, size=(n, 1)))).astype(np.float32)
    skipped = [0, 11, 12, 13, 2999]
    r[0] = 0.0
    r[11] = 0.0
    r[11, :8] = 1e-7 if dt == "f32" else 2.0 ** -24                                    # sum r^2 <= 1e-12
    r[12, d // 2] = np.inf
    r[13, 1] = np.nan
    r[2999, :] = np.inf
    rows = r.astype(np.float16) if dt == "f16" else r
    held = rows.astype(np.float64)
    rowids = 10 + 2 * np.arange(n, dtype=np.int64)                                         # odd rowids are unknown
    c = Y.Corpus(d, Y.F16 if dt == "f16" else Y.F32, Y.COSINE)
    c.append(rows, rowids=rowids)
    nq = 5
    q = (rng.standard_normal((nq, d)) * 3.0).astype(np.float32)
    q[1] = held[7].astype(np.float32) * np.float32(0.01)
    lists = [np.sort(np.concatenate([rowids[rng.choice(n, 700, replace=False)], rowids[skipped]])),
             np.sort(np.concatenate([rowids[:40], rowids[:40:3], [11, 13, 10**9, -5]])),             # repeats, unknown
             np.zeros(0, np.int64),
             rowids.copy(),
             np.array([rowids[5]] * 4 + [rowids[6]], np.int64)]
    cap = max(len(a) for a in lists)
    counts, cands = c.debug_stage1_candidates(q, 2, np.zeros(nq, np.float32), cap, allowed=lists)
    eps = c.debug_last_eps(nq)
    assert np.all(eps > 0)
    finite = np.isfinite(held).all(axis=1)
    ss = np.where(finite, (np.where(finite[:, None], held, 0.0) ** 2).sum(axis=1), 0.0)
    valid = finite & (ss > 1e-12)
    assert set(np.nonzero(~valid)[0]) == set(skipped)
    for qi, al in enumerate(lists):
        assert counts[qi] == len(al), qi
        ent = cands[qi, : len(al)]
        assert not np.isnan(ent["score"]).any(), qi
        idx = np.searchsorted(rowids, al)
        known = (idx < n) & (rowids[np.minimum(idx, n - 1)] == al)
        first = np.concatenate([[True], al[1:] != al[:-1]])
        take = known & first
        assert np.all(ent["row"][~take] == NO_ROW) and np.all(ent["score"][~take] == -np.inf), qi
        rows_t = idx[take]
        assert np.array_equal(ent["row"][take], rows_t), qi
        sc = ent["score"][take]
        v = valid[rows_t]
        assert np.all(sc[~v] == -np.inf), qi                                           # the skip rule
        x = q[qi].astype(np.float64)
        want = held[rows_t[v]] @ x / (np.sqrt(ss[rows_t[v]]) * np.linalg.norm(x))
        err = np.abs(sc[v].astype(np.float64) - want)
        assert np.all(err <= eps[qi]), (qi, err.max(), eps[qi])
    c.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6. end to end: exhaustive fallback inside candidate sets
# ---------------------------------------------------------------------------------------------------------------------
N_E2E, D_E2E, K_E2E = 100_000, 64, 10
N_DENSE = 50_000


def e2e_corpus(O, n, seed):
    """fp32 rows with (a) 600 rows whose cosine with q_tie lies within 2e-6 of 1 (far inside the stage-1 error bound),
    (b) 10000 copies of one row (more than exhaustive level 1 re-scores), (c) 40 zero rows and 20 rows opposite q_neg,
    (d) 600 rows whose cosine with q_low lies within 2e-6 of 0.5, while the 10000 copies score 0.9 against q_low"""
    d = D_E2E
    rng = np.random.default_rng(seed)
    rows = O.gen_rows_f32(seed, 0, n, d)
    perm = rng.permutation(n)
    tie_pos, dup_pos, zero_pos, neg_pos = np.sort(perm[:600]), np.sort(perm[600:10600]), np.sort(perm[10600:10640]), \
        np.sort(perm[10640:10660])
    q_tie = O.gen_rows_f32(seed + 1, 0, 1, d)[0]
    qn = q_tie / np.linalg.norm(q_tie)
    for p in tie_pos:
        delta = rng.normal(size=d).astype(np.float32)
        delta -= qn * float(delta @ qn)
        delta *= np.float32(np.sqrt(2.0 * 2e-6 * rng.uniform(0.0, 1.0)) / np.linalg.norm(delta))
        rows[p] = (qn + delta) * np.float32(rng.uniform(0.5, 2.0))
    rows[dup_pos] = rows[dup_pos[0]]
    q_dup = rows[dup_pos[0]] * np.float32(2.5)
    rows[zero_pos] = 0.0
    q_neg = O.gen_rows_f32(seed + 2, 0, 1, d)[0]
    rows[neg_pos] = -q_neg[None, :] * rng.uniform(0.5, 1.0, size=(20, 1)).astype(np.float32) + \
        rng.standard_normal((20, d)).astype(np.float32) * np.float32(0.01)
    low_pos = np.sort(perm[10660:11260])
    dn = rows[dup_pos[0]].astype(np.float64) / np.linalg.norm(rows[dup_pos[0]])
    q_low = 0.9 * dn + np.sqrt(0.19) * unit_orthogonal(rng.normal(size=d), dn)
    for p in low_pos:
        cos = 0.5 - 2e-6 * rng.uniform(0.0, 1.0)
        rows[p] = (cos * q_low + np.sqrt(1.0 - cos * cos) * unit_orthogonal(rng.normal(size=d), q_low)) * rng.uniform(0.5, 2.0)
    pos = dict(tie=tie_pos, dup=dup_pos, zero=zero_pos, neg=neg_pos, low=low_pos)
    return rows, pos, q_tie, q_dup, q_neg, q_low.astype(np.float32)


def unit_orthogonal(x, u):
    x = x - u * float(x @ u)
    return x / np.linalg.norm(x)


@pytest.fixture(scope="module")
def e2e(Y, oracle):
    O = oracle
    rows, pos, *qs = e2e_corpus(O, N_E2E, 61)
    rowids = 5 + 2 * np.arange(N_E2E, dtype=np.int64)
    c = Y.Corpus(D_E2E, Y.F32, Y.COSINE)
    c.append(rows, rowids=rowids)
    yield O, c, rows, rowids, pos, qs
    c.close()


# batch layout: rejected queries at non-adjacent positions.  LOW_AT: near ties of the candidate set that rank below more
# than 4096 rows outside it -- level 1 certifies them only if it applies the candidate set before its selection.
LEVEL1_AT, LEVEL2_AT, LOW_AT, ZERO_AT, NQ_E2E = (1, 6), (3,), 8, 4, 10


def e2e_batch(O, rows, pos, qs, rowids, path, rng):
    """NQ_E2E queries and their candidate sets.  The near-tie and duplicate queries may only use every other one of their
    rows, so an answer taken from the whole corpus is visibly wrong."""
    q_tie, q_dup, q_neg, q_low = qs
    n = len(rows)
    queries = O.gen_rows_f32(99, 0, NQ_E2E, D_E2E) * np.float32(1.3)
    for i in LEVEL1_AT:
        queries[i] = q_tie
    for i in LEVEL2_AT:
        queries[i] = q_dup
    queries[ZERO_AT] = q_neg
    if path == "dense":                  # no candidate set: q_low would simply rank the copies first
        return queries, None
    queries[LOW_AT] = q_low
    big = path == "masked-big"
    lists = []
    for i in range(NQ_E2E):
        base = rng.choice(n, 40_000 if big else 800, replace=False)
        if i in LEVEL1_AT:
            base = np.concatenate([base[:20_000 if big else 100], pos["tie"][i % 2::2]])
        elif i in LEVEL2_AT:
            base = np.concatenate([base[:20_000 if big else 300], pos["dup"][::2]])
        elif i == LOW_AT:
            base = np.concatenate([np.setdiff1d(base[:20_000 if big else 100], pos["dup"]), pos["low"][::2]])
        elif i == ZERO_AT:
            base = np.concatenate([base if big else base[:0], pos["zero"], pos["neg"]])
        al = np.unique(rowids[base])
        al = np.concatenate([al, [4, rowids[-1] + 2]])                       # ids that are not in the corpus
        al.sort()
        lists.append(al[::-1].copy() if path == "masked-small" else al)
    return queries, lists


@pytest.mark.parametrize("path", ["direct", "masked-small", "masked-big", "dense"])
def test_fallback_stays_inside_the_candidate_set(Y, oracle, e2e, path):
    """Queries the certificate rejects are resolved by exhaustive level 1 (near ties) or level 2 (more duplicates than
    level 1 re-scores), on each path a candidate set can take -- direct lists, the masked pass with few or many allowed rows
    -- and on the dense path without one.  Every answer is the reference scan restricted to the query's set: ids in order,
    scores bit for bit; exactly the rejected queries are flagged, and only the duplicates need the full exact pass.  A
    direct list of 40 zero rows and 20 rows scoring below 0 is certified on the fast path: the skipped rows score -inf in
    stage 1."""
    if path == "dense":
        O = oracle
        rows, pos, *qs = e2e_corpus(O, N_DENSE, 62)
        rowids = 5 + 2 * np.arange(N_DENSE, dtype=np.int64)
        c = Y.Corpus(D_E2E, Y.F32, Y.COSINE)
        c.append(rows, rowids=rowids)
    else:
        O, c, rows, rowids, pos, qs = e2e
    rng = np.random.default_rng(7)
    queries, lists = e2e_batch(O, rows, pos, qs, rowids, path, rng)
    rid, sc, cnt, flags = c.search(queries, K_E2E, threshold=-1.0, allowed=lists)
    for qi in range(len(queries)):
        al = None if lists is None else np.unique(lists[qi])
        rc, wr, ws_ = O.exact_scan_cosine(rows, queries[qi], K_E2E, threshold=-1.0, rowids=rowids, allowed=al)
        assert rc == 0
        got = rid[qi, : cnt[qi]]
        if al is not None:
            assert np.isin(got, al).all(), (path, qi, got[~np.isin(got, al)])
        assert cnt[qi] == len(wr) and np.array_equal(got, wr), (path, qi)
        assert np.array_equal(sc[qi, : len(wr)].view(np.uint32), ws_.view(np.uint32)), (path, qi)
    rejected = sorted(LEVEL1_AT + LEVEL2_AT + (() if path == "dense" else (LOW_AT,)))
    fb = list(np.nonzero(flags & Y.FLAG_FALLBACK_PATH)[0])
    assert fb == rejected, (path, fb)
    t = c.last_timings()
    assert t["resolved_exhaustively"] == len(rejected) and t["resolved_full_pass"] == len(LEVEL2_AT), (path, t)
    for i in LEVEL2_AT:
        assert flags[i] & Y.FLAG_TIE_AT_K
    if path == "dense":
        c.close()
