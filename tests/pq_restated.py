"""A plain numpy restatement of the SimeonPqAdc engine (yams_b200/csrc/pq.cu), bit for bit.

Written from the semantics the engine documents (ProductQuantizer::encode, PQInnerProductQuery with simd::dot of the AVX2
tier, inner_product_from_lut, simeonPqSearchUnlocked's selection and computeCosineSimilarity rerank), not from its code.
Every float operation is float32 and correctly rounded unless stated; numpy float32 arithmetic is, and nothing here mixes
dtypes in one operation.  tests/test_pq_restated.py anchors it to the reference's stored answers; tests/test_gpu_pq_scan.py
judges the device against it at shapes the stored answers do not cover."""
import numpy as np

F32 = np.float32
F64 = np.float64
FLAG_TIE_AT_K = 1


def normalise(rows):
    """normalizeEmbeddingInPlace -> (normalised rows of the accepted, accepted mask)"""
    from oracle import oracle as O
    return O.normalize_like_reference(rows)


# ---- float32 FMA ----------------------------------------------------------------------------------------------------------

def fma32(a, b, c):
    """fmaf(a, b, c) rounded once to float32, elementwise.  a*b of two floats is exact in float64; s = p + c is rounded to
    float64 and TwoSum gives its error e.  Rounding s to odd (step one float64 ulp towards e when s is inexact and its last
    bit is even) and then to float32 rounds the exact sum correctly, because 53 >= 24 + 2."""
    a = np.asarray(a, dtype=F32)
    b = np.asarray(b, dtype=F32)
    c = np.asarray(c, dtype=F32)
    with np.errstate(invalid="ignore", over="ignore"):
        p = a.astype(F64) * b.astype(F64)
        c64 = c.astype(F64)
        s = p + c64
        bb = s - p
        e = (p - (s - bb)) + (c64 - bb)
        odd_step = np.isfinite(s) & np.isfinite(e) & (e != 0) & ((s.view(np.uint64) & np.uint64(1)) == 0)
        s = np.where(odd_step, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
        return s.astype(F32)


# ---- index build ----------------------------------------------------------------------------------------------------------

def encode(rows_normalised, codebooks, m: int, k: int, chunk: int = 2048) -> np.ndarray:
    """ProductQuantizer::encode: per subspace l2_sq = sequential float loop of acc += (x - c) * (x - c) (separate multiply and
    add) against every centroid, code = the first index of the smallest distance; NaN never wins, all inf / NaN -> 0."""
    x = np.ascontiguousarray(rows_normalised, dtype=F32)
    n, d = x.shape
    dsub = d // m
    cb = np.ascontiguousarray(codebooks, dtype=F32).reshape(m, k, dsub)
    codes = np.zeros((n, m), dtype=np.uint8)
    with np.errstate(invalid="ignore", over="ignore"):
        for r0 in range(0, n, chunk):
            xs = x[r0:r0 + chunk]
            for mi in range(m):
                acc = np.zeros((len(xs), k), dtype=F32)
                for e in range(dsub):
                    df = xs[:, mi * dsub + e][:, None] - cb[mi, :, e][None, :]
                    acc = acc + df * df
                acc = np.where(np.isnan(acc), F32(np.inf), acc)
                best = np.argmin(acc, axis=1)                       # first index of the minimum
                best[np.isinf(acc[np.arange(len(xs)), best])] = 0   # nothing below +inf: the reference keeps 0
                codes[r0:r0 + len(xs), mi] = best
    return codes


def lut(query_normalised, codebooks, m: int, k: int) -> np.ndarray:
    """PQInnerProductQuery's table [m][k]: dot(q_sub, centroid).  dsub < 16: the scalar loop (separate multiply and add);
    dsub >= 16: simd::dot of the AVX2 tier (two 8-lane FMA accumulators over 16-element blocks, lanes summed as
    (a0[0] + a1[0]) + (a0[1] + a1[1]) + ... + (a0[7] + a1[7]) left to right, FMA over the tail)."""
    q = np.ascontiguousarray(query_normalised, dtype=F32).reshape(-1)
    dsub = q.size // m
    qs = q.reshape(m, 1, dsub)
    cb = np.ascontiguousarray(codebooks, dtype=F32).reshape(m, k, dsub)
    with np.errstate(invalid="ignore", over="ignore"):
        if dsub < 16:
            acc = np.zeros((m, k), dtype=F32)
            for i in range(dsub):
                acc = acc + qs[:, :, i] * cb[:, :, i]
            return acc
        a0 = np.zeros((m, k, 8), dtype=F32)
        a1 = np.zeros((m, k, 8), dtype=F32)
        i = 0
        while i + 16 <= dsub:
            a0 = fma32(np.broadcast_to(qs[:, :, i:i + 8], a0.shape), cb[:, :, i:i + 8], a0)
            a1 = fma32(np.broadcast_to(qs[:, :, i + 8:i + 16], a1.shape), cb[:, :, i + 8:i + 16], a1)
            i += 16
        s = a0[:, :, 0] + a1[:, :, 0]
        for l in range(1, 8):
            s = s + (a0[:, :, l] + a1[:, :, l])
        for j in range(i, dsub):
            s = fma32(np.broadcast_to(qs[:, :, j], s.shape), cb[:, :, j], s)
        return s


def adc(codes, table) -> np.ndarray:
    """inner_product_from_lut: the sequential float sum over mi of table[mi, code[mi]]"""
    cd = np.asarray(codes)
    t = np.asarray(table, dtype=F32)
    acc = np.zeros(len(cd), dtype=F32)
    with np.errstate(invalid="ignore", over="ignore"):
        for mi in range(t.shape[0]):
            acc = acc + t[mi][cd[:, mi]]
    return acc


# ---- search ---------------------------------------------------------------------------------------------------------------

def fkey(x) -> np.ndarray:
    """monotone uint32 key of float32 values (-0 below +0, NaN -> 0, below -inf): the engine's sort order"""
    b = np.asarray(x, dtype=F32).reshape(-1).view(np.uint32).astype(np.uint64)
    k = np.where(b & 0x80000000, ~b & np.uint64(0xFFFFFFFF), b | np.uint64(0x80000000))
    return np.where(np.isnan(np.asarray(x, dtype=F32).reshape(-1)), np.uint64(0), k)


def approx_k(n_idx: int, k: int, rerank_factor: int) -> int:
    return min(n_idx, max(k, k * max(rerank_factor, 1)))


def tie_rank(tie_keys, n_idx: int) -> np.ndarray:
    """rank of every index position by (tie-break key asc, position asc) (the host's stable sort); no keys: the position"""
    if tie_keys is None:
        return np.arange(n_idx, dtype=np.int64)
    order = np.argsort(np.asarray(tie_keys, dtype=np.uint64), kind="stable")
    rank = np.empty(n_idx, dtype=np.int64)
    rank[order] = np.arange(n_idx)
    return rank


def select(scores, ranks, approx: int) -> np.ndarray:
    """indexes of the best `approx` of (scores[i], ranks[i]) by (score desc, tie rank asc), NaN last, best first"""
    key = (fkey(scores) << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - np.asarray(ranks, dtype=np.uint64))
    if approx < len(key):
        part = np.argpartition(key, len(key) - approx)[len(key) - approx:]
    else:
        part = np.arange(len(key))
    return part[np.argsort(key[part], kind="stable")[::-1]]


def cosine_f32(query, rows) -> np.ndarray:
    """computeCosineSimilarity of the ORIGINAL query against held rows: sequential float64 sums, float cast, 0 for a zero norm"""
    q = np.asarray(query, dtype=F32).astype(F64)
    r = np.asarray(rows, dtype=F32).reshape(-1, q.size).astype(F64)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        dp = np.cumsum(r * q[None, :], axis=1)[:, -1] if q.size else np.zeros(len(r))
        na = np.sqrt(np.cumsum(q * q)[-1])
        nb = np.sqrt(np.cumsum(r * r, axis=1)[:, -1])
        sim = dp / (na * nb)
        sim = np.where((na == 0.0) | (nb == 0.0), 0.0, sim)
    return sim.astype(F32)


def final(query, survivors_rows, held_rows, rowids, k: int, threshold: float):
    """rerank + final order of one query: survivors_rows are corpus rows, held_rows[i] their stored values.
    -> (rowids i64[k] padded with -1, scores f32[k] padded with -inf, count, flags)"""
    out_r = np.full(k, -1, dtype=np.int64)
    out_s = np.full(k, -np.inf, dtype=F32)
    rows = np.asarray(survivors_rows, dtype=np.int64)
    if len(rows) == 0 or k == 0:
        return out_r, out_s, 0, 0
    sim = cosine_f32(query, held_rows)
    keep = ~np.isnan(sim) & ~(sim < F32(threshold))
    sim, rows = sim[keep], rows[keep]
    key = (fkey(sim) << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - rows.astype(np.uint64))
    o = np.argsort(key, kind="stable")[::-1]
    sim, rows, key = sim[o], rows[o], key[o]
    cnt = min(len(rows), k)
    out_r[:cnt] = np.asarray(rowids, dtype=np.int64)[rows[:cnt]]
    out_s[:cnt] = sim[:cnt]
    flags = FLAG_TIE_AT_K if len(rows) > k and (key[k - 1] >> np.uint64(32)) == (key[k] >> np.uint64(32)) else 0
    return out_r, out_s, cnt, flags


class Index:
    """The restated index over a corpus: held float32 row values (fp16 rows: their float values), rowids, m, k, codebooks,
    tie-break keys (one per corpus row or None).  codes: the index's code rows when already known (e.g. the device's, checked
    on a sample), else encoded here.  held may be a callable rows -> values for corpora too large to hold on the host."""

    def __init__(self, held, rowids, m, k, codebooks, tie_keys=None, codes=None, idx_rows=None):
        self.held = held
        self.rowids = np.asarray(rowids, dtype=np.int64)
        self.m, self.k = m, k
        self.codebooks = np.ascontiguousarray(codebooks, dtype=F32).reshape(-1)
        if idx_rows is None:
            _, ok = normalise(held)
            idx_rows = np.nonzero(ok)[0]
        self.idx_rows = np.asarray(idx_rows, dtype=np.int64)
        if codes is None:
            codes = encode(normalise(held[self.idx_rows])[0], self.codebooks, m, k)
        self.codes = codes
        tk = None if tie_keys is None else np.asarray(tie_keys, dtype=np.uint64)[self.idx_rows]
        self.ranks = tie_rank(tk, len(self.idx_rows))

    def rows_of(self, corpus_rows):
        return self.held(corpus_rows) if callable(self.held) else np.asarray(self.held)[corpus_rows]

    def query_table(self, query):
        """-> (lut [m][k], valid) of one query; an invalid query's table is not used"""
        qn, ok = normalise(np.asarray(query, dtype=F32)[None, :])
        if not ok[0]:
            return None, False
        return lut(qn[0], self.codebooks, self.m, self.k), True

    def survivors(self, query, approx: int, positions=None):
        """corpus rows of the best `approx` ADC scores (best first); [] for a query that cannot be normalised"""
        t, ok = self.query_table(query)
        if not ok:
            return np.zeros(0, dtype=np.int64)
        pos = np.arange(len(self.codes)) if positions is None else np.asarray(positions, dtype=np.int64)
        sel = select(adc(self.codes[pos], t), self.ranks[pos], approx)
        return self.idx_rows[pos[sel]]

    def search(self, query, k: int, rerank_factor: int, threshold: float, positions=None):
        """pq_search of one query (positions: the candidate index positions of pq_search_candidates) -> (rowids, scores,
        count, flags) padded to k"""
        n = len(self.idx_rows) if positions is None else len(positions)
        if k == 0 or n == 0:
            return np.full(k, -1, np.int64), np.full(k, -np.inf, F32), 0, 0
        surv = self.survivors(query, approx_k(n, k, rerank_factor), positions)
        return final(query, surv, self.rows_of(surv), self.rowids, k, threshold)
