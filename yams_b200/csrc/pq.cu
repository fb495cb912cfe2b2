// pq.cu -- the SimeonPqAdc engine scan (SURVEY.md §8f N3): product-quantised asymmetric-distance scan + exact rerank.
//
// Reference (paths under /root/reference):
//   simeonPqSearchUnlocked                src/vector/sqlite_vec_backend.cpp:3868-4056
//   index build (normalise, encode)       src/vector/sqlite_vec_backend.cpp:3540-3690, normalizeEmbeddingInPlace :213-226
//   ProductQuantizer::encode / PQInnerProductQuery / inner_product_from_lut
//                                         third_party/simeon/src/pq.cpp:31-57,218-235,391-414
//   simd::dot (AVX2 tier on x86 builds)   third_party/simeon/src/arch/avx2.cpp:63-84, include/simeon/simd.hpp:187-201
//   computeCosineSimilarity (rerank)      src/vector/vector_database.cpp:1786-1810
//
// What the reference does per query: normalise q; LUT[mi][ki] = q_sub . centroid[mi][ki]; for EVERY indexed row the score is
// the sequential float sum of m LUT entries selected by the row's m code bytes; the best approxK = max(k, k * rerank_factor)
// rows by (score desc, tie-break key asc) are re-scored exactly (double cosine against the stored embedding), filtered by
// the threshold, ordered (similarity desc, chunk_id asc) and cut to k.
//
// Device layout: codes [n_idx][m] bytes (32 B per row at the default m = 32: 320 MB per 10 M rows, 1/48 of the fp16 corpus),
// the LUT of the query in shared memory (m * k floats = 32 KiB), one CTA per 4096-row tile: scores -> shared memory ->
// tile-local top-approxK by a bitonic network -> one short list per query -> the exact selection / rerank kernels of the exact
// scan (knn.cu).  Every float operation is in the reference's order, so the approximate scores, the survivor set and the final
// scores are bit-identical to the CPU engine (tests/test_gpu_pq.py pins them against simeon's own pq.cpp compiled in place).
// The scan is HBM-bound at m bytes per row per query; it is the LATENCY engine -- for batches beyond ~150 queries the exact
// tensor-core scan of the same corpus is faster and exact (DESIGN.md §4.6).
#include <cuda_fp16.h>

#include <algorithm>
#include <memory>
#include <new>
#include <vector>

#include "cosine.cuh"
#include "knn.cuh"

namespace yb {

constexpr int PQ_TILE = 4096;        // rows per CTA
constexpr int PQ_THREADS = 256;
constexpr uint32_t PQ_MAX_APPROX = 1024;

// normalizeEmbeddingInPlace (sqlite_vec_backend.cpp:213-226): double sum of squares, float reciprocal square root, float scale
__device__ __forceinline__ bool normalize_factor(double norm_sq, float* inv) {
    if (norm_sq <= 1e-20) return false;
    *inv = __fdiv_rn(1.0f, sqrtf((float)norm_sq));
    return true;
}

// one thread per corpus row: is it indexable (the rule of normalize_factor: not norm_sq <= 1e-20)?  keep[row] = 1/0.  A row
// with a NaN element has a NaN norm: the reference indexes it (it encodes to code 0 everywhere and re-scores to NaN).
__global__ void pq_keep_kernel(const void* __restrict__ rows, int dtype, uint32_t d, uint64_t n, uint32_t* __restrict__ keep) {
    uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    double ss = 0.0;
    walk_row(rows, dtype, d, r, [&](float v) { ss += (double)v * v; });
    keep[r] = ss <= 1e-20 ? 0u : 1u;
}
__global__ void pq_compact_kernel(const uint32_t* __restrict__ keep, const uint32_t* __restrict__ pos, uint64_t n, uint32_t* __restrict__ idx_rows) {
    uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r < n && keep[r]) idx_rows[pos[r]] = (uint32_t)r;
}

// ProductQuantizer::encode (pq.cpp:218-235) of one normalised row per CTA: thread ki owns centroid ki of every subspace,
// l2_sq is the reference's sequential float loop (separate multiply and add), argmin with the first index winning ties.
__global__ void __launch_bounds__(256) pq_encode_kernel(const void* __restrict__ rows, int dtype, uint32_t d, const uint32_t* __restrict__ idx_rows,
                                                        uint64_t n_idx, const float* __restrict__ codebooks, uint32_t m, uint32_t k,
                                                        uint8_t* __restrict__ codes) {
    extern __shared__ float xs[];                    // the normalised row, d floats
    __shared__ double s_norm;
    __shared__ float s_best[8];
    __shared__ uint32_t s_arg[8];
    const uint64_t j = blockIdx.x;
    if (j >= n_idx) return;
    const uint64_t row = idx_rows[j];
    const uint32_t dsub = d / m;
    for (uint32_t c = threadIdx.x; c < d; c += blockDim.x) xs[c] = load_elem(rows, dtype, row * d + c);
    __syncthreads();
    if (threadIdx.x == 0) {
        double ss = 0.0;
        for (uint32_t c = 0; c < d; ++c) ss += (double)xs[c] * (double)xs[c];
        s_norm = ss;
    }
    __syncthreads();
    float inv = 0.f;
    normalize_factor(s_norm, &inv);
    for (uint32_t c = threadIdx.x; c < d; c += blockDim.x) xs[c] = __fmul_rn(xs[c], inv);
    __syncthreads();
    const uint32_t ki = threadIdx.x;
    for (uint32_t mi = 0; mi < m; ++mi) {
        float dist = INFINITY;
        if (ki < k) {
            const float* cb = codebooks + ((size_t)mi * k + ki) * dsub;
            const float* x = xs + mi * dsub;
            float acc = 0.f;
            for (uint32_t e = 0; e < dsub; ++e) {
                const float df = __fsub_rn(x[e], cb[e]);
                acc = __fadd_rn(acc, __fmul_rn(df, df));
            }
            dist = acc;
        }
        // argmin over ki with `d < best_d` semantics: smallest distance, lowest index on equality; NaN never wins
        float bd = dist == dist ? dist : INFINITY;
        uint32_t bi = ki;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float od = __shfl_xor_sync(0xffffffffu, bd, o);
            const uint32_t oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (od < bd || (od == bd && oi < bi)) { bd = od; bi = oi; }
        }
        if ((threadIdx.x & 31) == 0) { s_best[threadIdx.x >> 5] = bd; s_arg[threadIdx.x >> 5] = bi; }
        __syncthreads();
        if (threadIdx.x == 0) {
            float fb = s_best[0];
            uint32_t fi = s_arg[0];
            for (int w = 1; w < 8; ++w)
                if (s_best[w] < fb || (s_best[w] == fb && s_arg[w] < fi)) { fb = s_best[w]; fi = s_arg[w]; }
            // every distance +inf / NaN: the reference keeps best = 0
            codes[j * m + mi] = (uint8_t)(fb < INFINITY ? fi : 0u);
        }
        __syncthreads();
    }
}

// simd::dot of the AVX2 tier (avx2.cpp:63-84) for n >= 16, the scalar loop of pq.cpp:42-48 below that
__device__ __forceinline__ float pq_dot(const float* __restrict__ a, const float* __restrict__ b, uint32_t n) {
    if (n < 16) {
        float acc = 0.f;
        for (uint32_t i = 0; i < n; ++i) acc = __fadd_rn(acc, __fmul_rn(a[i], b[i]));
        return acc;
    }
    float a0[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, a1[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    uint32_t i = 0;
    for (; i + 16 <= n; i += 16) {
#pragma unroll
        for (int l = 0; l < 8; ++l) {
            a0[l] = __fmaf_rn(a[i + l], b[i + l], a0[l]);
            a1[l] = __fmaf_rn(a[i + 8 + l], b[i + 8 + l], a1[l]);
        }
    }
    float s = __fadd_rn(a0[0], a1[0]);
#pragma unroll
    for (int l = 1; l < 8; ++l) s = __fadd_rn(s, __fadd_rn(a0[l], a1[l]));
    for (; i < n; ++i) s = __fmaf_rn(a[i], b[i], s);
    return s;
}

// one CTA per query: normalised query + LUT[mi][ki] = dot(q_sub, centroid) (PQInnerProductQuery, pq.cpp:391-403);
// valid[q] = 0 when the query cannot be normalised (the reference returns no results)
__global__ void __launch_bounds__(256) pq_lut_kernel(const float* __restrict__ q32, uint32_t d, const float* __restrict__ codebooks, uint32_t m,
                                                     uint32_t k, float* __restrict__ lut, uint32_t* __restrict__ valid) {
    extern __shared__ float qs[];
    __shared__ double s_norm;
    const uint32_t q = blockIdx.x;
    const uint32_t dsub = d / m;
    for (uint32_t c = threadIdx.x; c < d; c += blockDim.x) qs[c] = q32[(size_t)q * d + c];
    __syncthreads();
    if (threadIdx.x == 0) {
        double ss = 0.0;
        for (uint32_t c = 0; c < d; ++c) ss += (double)qs[c] * (double)qs[c];
        s_norm = ss;
    }
    __syncthreads();
    float inv = 0.f;
    const bool ok = normalize_factor(s_norm, &inv);
    if (threadIdx.x == 0) valid[q] = ok ? 1u : 0u;
    for (uint32_t c = threadIdx.x; c < d; c += blockDim.x) qs[c] = __fmul_rn(qs[c], inv);
    __syncthreads();
    for (uint32_t e = threadIdx.x; e < m * k; e += blockDim.x) {
        const uint32_t mi = e / k;
        lut[(size_t)q * m * k + e] = pq_dot(qs + mi * dsub, codebooks + (size_t)e * dsub, dsub);
    }
}

// inner_product_from_lut (pq.cpp:50-57): the sequential float sum of LUT[mi][code[mi]] over the row's m code bytes.  The ADC
// scan and the candidate gather both call this one function, so their scores are the same floats.  vec: m % 16 == 0 (the
// code row is then 16-byte aligned and read 16 bytes at a time).
__device__ __forceinline__ float pq_adc_sum(const uint8_t* __restrict__ cd, const float* __restrict__ lut, uint32_t m, uint32_t k, bool vec) {
    float acc = 0.f;
    if (vec) {
        for (uint32_t mi = 0; mi < m; mi += 16) {
            const uint4 w = *reinterpret_cast<const uint4*>(cd + mi);
            const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
            for (int u = 0; u < 4; ++u)
#pragma unroll
                for (int b = 0; b < 4; ++b) acc = __fadd_rn(acc, lut[(mi + u * 4 + b) * k + ((ws[u] >> (8 * b)) & 0xFFu)]);
        }
    } else {
        for (uint32_t mi = 0; mi < m; ++mi) acc = __fadd_rn(acc, lut[mi * k + cd[mi]]);
    }
    return acc;
}

// ADC scan: CTA (tile, q).  score = pq_adc_sum of the row's codes;
// key = (score, tie rank) packed so that a descending sort is (score desc, tie-break key asc); the tile's best `approx`
// keys are written to the query's list.
__global__ void __launch_bounds__(PQ_THREADS) pq_adc_kernel(const uint8_t* __restrict__ codes, uint64_t n_idx, uint32_t m, uint32_t k,
                                                            const float* __restrict__ lut_all, const uint32_t* __restrict__ tie_rank,
                                                            uint32_t approx, Cand* __restrict__ lists, uint32_t list_cap,
                                                            uint32_t* __restrict__ counts, uint32_t tile_stride) {
    extern __shared__ unsigned char sm[];
    float* lut = reinterpret_cast<float*>(sm);                                     // m * k floats
    uint64_t* keys = reinterpret_cast<uint64_t*>(sm + (((size_t)m * k * 4 + 7) & ~(size_t)7));   // PQ_TILE keys
    const uint32_t q = blockIdx.y;
    const uint64_t r0 = (uint64_t)blockIdx.x * tile_stride * PQ_TILE;
    const float* lq = lut_all + (size_t)q * m * k;
    for (uint32_t e = threadIdx.x; e < m * k; e += PQ_THREADS) lut[e] = lq[e];
    __syncthreads();
    const bool vec = (m % 16) == 0;
    for (uint32_t t = threadIdx.x; t < PQ_TILE; t += PQ_THREADS) {
        const uint64_t j = r0 + t;
        uint64_t key = 0;
        if (j < n_idx) {
            const float acc = pq_adc_sum(codes + j * m, lut, m, k, vec);
            key = score_key(acc, tie_rank[j]);
            if (key == 0) key = 1;
        }
        keys[t] = key;
    }
    __syncthreads();
    block_sort_desc<PQ_THREADS>(keys, PQ_TILE);
    const uint64_t in_tile = n_idx > r0 ? min((uint64_t)PQ_TILE, n_idx - r0) : 0;
    const uint32_t nout = (uint32_t)min((uint64_t)approx, in_tile);
    __shared__ uint32_t s_base;
    if (threadIdx.x == 0) s_base = atomicAdd(&counts[q], nout);
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < nout; i += PQ_THREADS) {
        const uint64_t key = keys[i];
        Cand c;
        c.score = key_score(key);
        c.row = key_row(key);     // tie rank: topk_select orders equal scores by ascending `row`
        if (s_base + i < list_cap) lists[(size_t)q * list_cap + s_base + i] = c;
    }
}

// Threshold of the filtered scan: the approx-th best key of the sampled tiles (any lower bound of the global approx-th best
// key keeps the selection exact); 0 = accept every row (fewer than approx sampled rows).
__global__ void pq_tau_kernel(const Cand* __restrict__ sel, const uint32_t* __restrict__ sel_n, uint32_t approx, uint32_t nq,
                              uint64_t* __restrict__ tau, uint32_t* __restrict__ counts) {
    uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nq) return;
    uint64_t t = 0;
    if (sel_n[q] >= approx) {
        const Cand c = sel[(size_t)q * approx + approx - 1];
        t = score_key(c.score, c.row);
    }
    tau[q] = t;
    counts[q] = 0;
}

// Filtered ADC scan: CTA (row range, group of QG queries) with the QG lookup tables in shared memory; every row's code bytes
// are read once per group; rows whose key reaches the query's threshold are appended to its list.  Same float order as
// pq_adc_kernel (sequential sum over the m sub-quantisers).
template <int QG>
__global__ void __launch_bounds__(PQ_THREADS) pq_adc_filter_kernel(const uint8_t* __restrict__ codes, uint64_t n_idx, uint32_t m, uint32_t k,
                                                                   const float* __restrict__ lut_all, const uint32_t* __restrict__ tie_rank,
                                                                   const uint64_t* __restrict__ tau, uint32_t nq, uint64_t rows_per_cta,
                                                                   Cand* __restrict__ lists, uint32_t list_cap, uint32_t* __restrict__ counts) {
    extern __shared__ unsigned char sm[];
    float* lut = reinterpret_cast<float*>(sm);   // QG x m x k
    const uint32_t q0 = blockIdx.y * QG;
    const uint32_t lut_len = m * k;
    for (uint32_t e = threadIdx.x; e < lut_len * QG; e += PQ_THREADS) {
        const uint32_t g = e / lut_len;
        lut[e] = (q0 + g < nq) ? lut_all[(size_t)(q0 + g) * lut_len + (e - g * lut_len)] : 0.f;
    }
    uint64_t tq[QG];
#pragma unroll
    for (int g = 0; g < QG; ++g) tq[g] = (q0 + g < nq) ? tau[q0 + g] : ~0ull;
    __syncthreads();
    const uint64_t r0 = (uint64_t)blockIdx.x * rows_per_cta;
    const uint64_t r1 = min(n_idx, r0 + rows_per_cta);
    const bool vec = (m % 16) == 0;
    const unsigned lane = threadIdx.x & 31u;
    for (uint64_t base = r0; base < r1; base += PQ_THREADS) {     // block-uniform trip count (warp collectives below)
        const uint64_t j = base + threadIdx.x;
        const bool valid = j < r1;
        float acc[QG];
#pragma unroll
        for (int g = 0; g < QG; ++g) acc[g] = 0.f;
        if (valid) {
            const uint8_t* cd = codes + j * m;
            if (vec) {
                for (uint32_t mi = 0; mi < m; mi += 16) {
                    const uint4 w = *reinterpret_cast<const uint4*>(cd + mi);
                    const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
                    for (int u = 0; u < 4; ++u)
#pragma unroll
                        for (int b = 0; b < 4; ++b) {
                            const uint32_t e = (mi + u * 4 + b) * k + ((ws[u] >> (8 * b)) & 0xFFu);
#pragma unroll
                            for (int g = 0; g < QG; ++g) acc[g] = __fadd_rn(acc[g], lut[g * lut_len + e]);
                        }
                }
            } else {
                for (uint32_t mi = 0; mi < m; ++mi) {
                    const uint32_t e = mi * k + cd[mi];
#pragma unroll
                    for (int g = 0; g < QG; ++g) acc[g] = __fadd_rn(acc[g], lut[g * lut_len + e]);
                }
            }
        }
#pragma unroll
        for (int g = 0; g < QG; ++g) {
            const uint32_t b = fkey(acc[g]);
            const uint32_t th = (uint32_t)(tq[g] >> 32);
            bool pass = valid && b >= th;           // tq = ~0 for the padding queries of the last group: never passes
            uint32_t rank = 0;
            if (pass) {
                rank = tie_rank[j];
                uint64_t key = word_key(b, rank);
                if (key == 0) key = 1;
                pass = key >= tq[g] && tq[g] != ~0ull;
            }
            const unsigned mask = __ballot_sync(0xffffffffu, pass);
            if (mask) {
                const int leader = __ffs(mask) - 1;
                uint32_t pos = 0;
                if ((int)lane == leader) pos = atomicAdd(&counts[q0 + g], (uint32_t)__popc(mask));
                pos = __shfl_sync(0xffffffffu, pos, leader) + __popc(mask & ((1u << lane) - 1u));
                if (pass && pos < list_cap) {
                    Cand c;
                    c.score = acc[g];
                    c.row = rank;
                    lists[(size_t)(q0 + g) * list_cap + pos] = c;
                }
            }
        }
    }
}

// counts[q] > cap: the filtered list dropped rows (a sample that misjudged the data): the caller re-runs the unfiltered scan
__global__ void pq_overflow_kernel(const uint32_t* __restrict__ counts, uint32_t nq, uint32_t cap, uint32_t* __restrict__ flag) {
    uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q < nq && counts[q] > cap) atomicExch(flag, 1u);
}

// survivors carry tie ranks: back to corpus rows (rank -> indexed row -> corpus row)
__global__ void pq_rank_to_row_kernel(Cand* __restrict__ sel, const uint32_t* __restrict__ sel_n, uint32_t K, uint32_t nq,
                                      const uint32_t* __restrict__ rank_to_idx, const uint32_t* __restrict__ idx_rows) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nq * K) return;
    uint32_t q = t / K, j = t % K;
    if (j < sel_n[q]) {
        Cand c = sel[t];
        c.row = idx_rows[rank_to_idx[c.row]];
        sel[t] = c;
    }
}

// compute_cosine_similarity of the ORIGINAL query a against corpus row `row`, float cast, NaN and `similarity < threshold`
// dropped (sqlite_vec_backend.cpp:4022-4037).  -> true and *out = sim when kept.
__device__ __forceinline__ bool pq_rerank_sim(const void* __restrict__ rows, int dtype, uint32_t d, uint32_t row, const float* __restrict__ a,
                                              float threshold, float* out) {
    const float sim = (float)compute_cosine_similarity(rows, dtype, d, row, a);
    if (sim == sim && !(sim < threshold)) {
        *out = sim;
        return true;
    }
    return false;
}
__global__ void pq_rerank_kernel(const void* __restrict__ rows, int dtype, uint32_t d, const float* __restrict__ q32, const Cand* __restrict__ sel,
                                 const uint32_t* __restrict__ sel_n, const uint32_t* __restrict__ valid, uint32_t K, uint32_t nq,
                                 float threshold, Exact* __restrict__ out) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nq * K) return;
    uint32_t q = t / K, j = t % K;
    Exact e;
    e.sim = __int_as_float(0x7FC00000);
    e.row = 0xFFFFFFFFu;
    if (valid[q] && j < sel_n[q]) {
        const uint32_t row = sel[t].row;
        float sim;
        if (pq_rerank_sim(rows, dtype, d, row, q32 + (size_t)q * d, threshold, &sim)) {
            e.sim = sim;
            e.row = row;
        }
    }
    out[t] = e;
}

// ---- candidate sets and the document pass ------------------------------------------------------------------------------
// corpus row -> index position (0xFFFFFFFF: not in the index); the caller pre-fills the table with 0xFF bytes
__global__ void pq_row_to_idx_kernel(const uint32_t* __restrict__ idx_rows, uint64_t n_idx, uint32_t* __restrict__ row_to_idx) {
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n_idx; j += (uint64_t)gridDim.x * blockDim.x)
        row_to_idx[idx_rows[j]] = (uint32_t)j;
}

// CTA (x, q): the mapped entries of query q's list -> index positions; an entry counts when its row is in the index and the
// query's bit for that position was not yet set (a rowid listed twice counts once).  The distinct positions are appended to
// cidx[offs[q] ..], their number to counts[q].
__global__ void pq_cand_index_kernel(const Cand* __restrict__ mapped, const uint64_t* __restrict__ offs, const uint32_t* __restrict__ row_to_idx,
                                     uint32_t* __restrict__ bits, uint64_t bits_ld, uint32_t* __restrict__ cidx, uint32_t* __restrict__ counts) {
    const uint32_t q = blockIdx.y;
    const uint64_t lo = offs[q], hi = offs[q + 1];
    const unsigned lane = threadIdx.x & 31u;
    for (uint64_t base = lo + (uint64_t)blockIdx.x * blockDim.x; base < hi; base += (uint64_t)gridDim.x * blockDim.x) {   // warp-uniform trips
        const uint64_t i = base + threadIdx.x;
        bool take = false;
        uint32_t idx = 0xFFFFFFFFu;
        if (i < hi) {
            const uint32_t row = mapped[i].row;
            if (row != 0xFFFFFFFFu) idx = row_to_idx[row];
            if (idx != 0xFFFFFFFFu) {
                const uint32_t bit = 1u << (idx & 31);
                take = !(atomicOr(&bits[(uint64_t)q * bits_ld + (idx >> 5)], bit) & bit);
            }
        }
        const unsigned mask = __ballot_sync(0xffffffffu, take);
        if (mask) {
            const int leader = __ffs(mask) - 1;
            uint32_t pos = 0;
            if ((int)lane == leader) pos = atomicAdd(&counts[q], (uint32_t)__popc(mask));
            pos = __shfl_sync(0xffffffffu, pos, leader) + __popc(mask & ((1u << lane) - 1u));
            if (take) cidx[lo + pos] = idx;
        }
    }
}

// ADC scores of the candidate positions: CTA (slice of per_cta candidates, q) with the query's LUT in shared memory;
// lists[q * cap + j] = (pq_adc_sum, tie rank) for j < counts[q], the input of the top-approx selection
__global__ void __launch_bounds__(PQ_THREADS) pq_adc_gather_kernel(const uint8_t* __restrict__ codes, uint32_t m, uint32_t k,
                                                                   const float* __restrict__ lut_all, const uint32_t* __restrict__ tie_rank,
                                                                   const uint32_t* __restrict__ cidx, const uint64_t* __restrict__ offs,
                                                                   const uint32_t* __restrict__ counts, uint32_t per_cta,
                                                                   Cand* __restrict__ lists, uint32_t cap) {
    extern __shared__ float lut[];   // m * k floats
    const uint32_t q = blockIdx.y;
    const uint32_t cnt = counts[q];
    const uint32_t j0 = blockIdx.x * per_cta;
    if (j0 >= cnt) return;
    const uint32_t j1 = min(cnt, j0 + per_cta);
    const float* lq = lut_all + (size_t)q * m * k;
    for (uint32_t e = threadIdx.x; e < m * k; e += PQ_THREADS) lut[e] = lq[e];
    __syncthreads();
    const bool vec = (m % 16) == 0;
    const uint32_t* ci = cidx + offs[q];
    for (uint32_t j = j0 + threadIdx.x; j < j1; j += PQ_THREADS) {
        const uint32_t idx = ci[j];
        Cand c;
        c.score = pq_adc_sum(codes + (uint64_t)idx * m, lut, m, k, vec);
        c.row = tie_rank[idx];
        lists[(uint64_t)q * cap + j] = c;
    }
}

// valid[q] = 1 when the query can be normalised (normalizeEmbeddingInPlace, the rule of pq_lut_kernel)
__global__ void pq_query_valid_kernel(const float* __restrict__ q32, uint32_t nq, uint32_t d, uint32_t* __restrict__ valid) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nq) return;
    double ss = 0.0;
    walk_row(q32, YAMS_B200_F32, d, q, [&](float v) { ss += (double)v * v; });
    float inv;
    valid[q] = normalize_factor(ss, &inv) ? 1u : 0u;
}

// index of the segment holding element p: the last s with starts[s] <= p (starts ascending, starts[0] <= p)
__device__ __forceinline__ uint32_t segment_of(const uint64_t* __restrict__ starts, uint32_t nseg, uint64_t p) {
    uint32_t a = 0, b = nseg;
    while (b - a > 1) {
        const uint32_t mid = (a + b) >> 1;
        if (starts[mid] <= p) a = mid; else b = mid;
    }
    return a;
}

// Document pass, step 1: one thread per (query, candidate row) pair.  pairs[p].row is the corpus row (0xFFFFFFFF: unknown
// rowid); pairs[p].score becomes its similarity, NaN when the row is no result.
//   exact (row_to_idx == NULL): exact_cosine_sim against qnorm[q] (the exact scan's arithmetic, skip rules and threshold);
//   PQ: rows in the index only, pq_rerank_sim (the PQ engine's rerank arithmetic and threshold), nothing for a query that
//       cannot be normalised.
__global__ void doc_score_kernel(const void* __restrict__ rows, int dtype, uint32_t d, const float* __restrict__ q32, const double* __restrict__ qnorm,
                                 const uint32_t* __restrict__ valid, const uint32_t* __restrict__ row_to_idx, const uint64_t* __restrict__ qpair,
                                 uint32_t nq, uint64_t npairs, float threshold, Cand* __restrict__ pairs) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= npairs) return;
    const uint32_t q = segment_of(qpair, nq, p);
    const uint32_t row = pairs[p].row;
    float sim = __int_as_float(0x7FC00000), s;
    if (row != 0xFFFFFFFFu) {
        const float* qv = q32 + (size_t)q * d;
        if (row_to_idx) {
            if (valid[q] && row_to_idx[row] != 0xFFFFFFFFu && pq_rerank_sim(rows, dtype, d, row, qv, threshold, &s)) sim = s;
        } else if (exact_cosine_sim(rows, dtype, d, row, qv, qnorm[q], threshold, &s)) {
            sim = s;
        }
    }
    pairs[p].score = sim;
}

// Document pass, step 2: one warp per document, the arg-max of its rows by (sim desc, position in the document asc).  A document
// with a surviving row is appended to its query's list as (best sim, document index), the row index it came from is kept in
// best_row[doc].
__global__ void doc_argmax_kernel(const Cand* __restrict__ pairs, const uint64_t* __restrict__ doff, uint32_t ndocs, const uint64_t* __restrict__ qdocs,
                                  uint32_t nq, Cand* __restrict__ lists, uint32_t cap, uint32_t* __restrict__ counts, uint32_t* __restrict__ best_row) {
    const uint64_t doc = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const unsigned lane = threadIdx.x & 31u;
    if (doc >= ndocs) return;
    const uint64_t lo = doff[doc], hi = doff[doc + 1];
    uint64_t best = 0;
    for (uint64_t i = lo + lane; i < hi; i += 32) {
        const float s = pairs[i].score;
        if (s == s) best = max(best, score_key(s, (uint32_t)(i - lo)));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = max(best, (uint64_t)__shfl_xor_sync(0xffffffffu, best, o));
    if (lane == 0 && best) {
        const uint32_t q = segment_of(qdocs, nq, doc);
        best_row[doc] = pairs[lo + key_row(best)].row;
        Cand c;
        c.score = key_score(best);
        c.row = (uint32_t)doc;
        const uint32_t pos = atomicAdd(&counts[q], 1u);
        lists[(uint64_t)q * cap + pos] = c;
    }
}

// Document pass, step 4: the k best documents of every query (sel, from the top-k selection) -> document index, its best row's
// rowid and score; unused slots -1 / -1 / 0
__global__ void doc_emit_kernel(const Cand* __restrict__ sel, const uint32_t* __restrict__ sel_n, uint32_t k, uint32_t nq, uint64_t doc_base,
                                const uint32_t* __restrict__ best_row, const int64_t* __restrict__ rowids, int64_t* __restrict__ o_docs,
                                int64_t* __restrict__ o_rowids, float* __restrict__ o_scores, uint32_t* __restrict__ o_counts) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (uint64_t)nq * k) return;
    const uint32_t q = (uint32_t)(t / k), i = (uint32_t)(t % k);
    if (i < sel_n[q]) {
        const Cand c = sel[t];
        o_docs[t] = (int64_t)(doc_base + c.row);
        o_rowids[t] = rowids[best_row[c.row]];
        o_scores[t] = c.score;
    } else {
        o_docs[t] = -1;
        o_rowids[t] = -1;
        o_scores[t] = 0.f;
    }
    if (i == 0) o_counts[q] = sel_n[q];
}

// Host staging of ONE host-to-device copy: the pieces of a call's input at 16-byte aligned offsets
struct Staging {
    std::vector<unsigned char> h;
    size_t add(const void* src, size_t bytes) {
        const size_t off = (h.size() + 15) & ~(size_t)15;
        h.resize(off + bytes);
        if (bytes) memcpy(h.data() + off, src, bytes);
        return off;
    }
};

}  // namespace yb

using namespace yb;

struct yams_b200_pq {
    yams_b200_corpus* corpus = nullptr;
    uint64_t corpus_generation = 0;
    uint32_t m = 0, k = 0, dim = 0;
    uint64_t n_idx = 0;
    DevBuf codebooks, codes, idx_rows, tie_rank, rank_to_idx;
    DevBuf row_to_idx;          // corpus row -> index position, built by the first call that needs it (the index is immutable)
    bool row_to_idx_ready = false;
    // search workspace
    DevBuf q32, lut, valid, lists, counts, sel, exact, dout, tau;
    DevBuf cin, mapped, cidx, bits;   // candidate-set search: staged input, mapped rows, distinct positions, per-query seen bits
    uint32_t last_path[4] = {0, 0, 0, 0};   // the path of the last pq_search batch (yams_b200_debug_pq_last_path)
    std::mutex mu;
};

extern "C" {

yams_status_t yams_b200_pq_build(yams_b200_corpus* c, uint32_t m, uint32_t k, const float* codebooks, const uint64_t* tie_break_keys,
                                 yams_b200_pq** out) {
    YB_TRY
    YB_ARG(c && out && codebooks, "null argument");
    *out = nullptr;
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_BIND(c);
    YB_ARG(m >= 1 && k >= 2 && k <= 256, "m must be >= 1 and k in 2..256");            // sqlite_vec_backend.cpp:3552-3553
    YB_ARG(c->dim % m == 0, "m must divide the dimension");                            // :3549-3551
    YB_ARG((size_t)m * k * 4 + PQ_TILE * 8 + 64 <= 200 * 1024, "m * k too large for the shared-memory lookup table");
    const uint64_t n = c->n;
    YB_ARG(n < 0xFFFFFFFFull, "too many rows");
    std::unique_ptr<yams_b200_pq> p(new (std::nothrow) yams_b200_pq());
    if (!p) return YAMS_ERR_INTERNAL;
    p->corpus = c;
    p->corpus_generation = c->generation;
    p->m = m; p->k = k; p->dim = c->dim;
    cudaStream_t st = c->st;
    yams_status_t rc;
    const uint32_t dsub = c->dim / m;
    const size_t cb_bytes = (size_t)m * k * dsub * 4;
    if ((rc = p->codebooks.reserve(cb_bytes)) != YAMS_OK) return rc;
    YB_CUDA(cudaMemcpyAsync(p->codebooks.p, codebooks, cb_bytes, cudaMemcpyHostToDevice, st));
    if (n) {
        // rows the index holds: those normalizeEmbeddingInPlace accepts (:3569-3577)
        DevBuf keep, pos, scratch, total;
        if ((rc = keep.reserve(n * 4)) != YAMS_OK || (rc = pos.reserve(n * 4)) != YAMS_OK || (rc = total.reserve(8)) != YAMS_OK) return rc;
        pq_keep_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(c->rows.p, c->dtype, c->dim, n, keep.as<uint32_t>());
        if ((rc = exclusive_scan_u32(keep.as<uint32_t>(), pos.as<uint32_t>(), n, total.as<uint64_t>(), scratch, st)) != YAMS_OK) return rc;
        uint64_t n_idx = 0;
        YB_CUDA(cudaMemcpyAsync(&n_idx, total.p, 8, cudaMemcpyDeviceToHost, st));
        YB_CUDA(cudaStreamSynchronize(st));
        p->n_idx = n_idx;
        if ((rc = p->idx_rows.reserve(std::max<uint64_t>(n_idx, 1) * 4)) != YAMS_OK) return rc;
        pq_compact_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(keep.as<uint32_t>(), pos.as<uint32_t>(), n, p->idx_rows.as<uint32_t>());
        if ((rc = p->codes.reserve(std::max<uint64_t>(n_idx, 1) * m + 64)) != YAMS_OK) return rc;
        if (n_idx) {
            YB_CUDA(cudaFuncSetAttribute(pq_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(c->dim * 4)));
            pq_encode_kernel<<<(unsigned)n_idx, 256, c->dim * 4, st>>>(c->rows.p, c->dtype, c->dim, p->idx_rows.as<uint32_t>(), n_idx,
                                                                      p->codebooks.as<float>(), m, k, p->codes.as<uint8_t>());
        }
        YB_CUDA(cudaGetLastError());
        // tie-break order (sqlite_vec_backend.cpp:3985-3990): rank of every indexed row by (tie_break_key, position)
        std::vector<uint32_t> h_idx(n_idx), rank(n_idx), order(n_idx);
        if (n_idx) YB_CUDA(cudaMemcpyAsync(h_idx.data(), p->idx_rows.p, n_idx * 4, cudaMemcpyDeviceToHost, st));
        YB_CUDA(cudaStreamSynchronize(st));
        for (uint64_t j = 0; j < n_idx; ++j) order[j] = (uint32_t)j;
        if (tie_break_keys)
            std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return tie_break_keys[h_idx[a]] < tie_break_keys[h_idx[b]]; });
        for (uint64_t r = 0; r < n_idx; ++r) rank[order[r]] = (uint32_t)r;
        if ((rc = p->tie_rank.reserve(std::max<uint64_t>(n_idx, 1) * 4)) != YAMS_OK) return rc;
        if ((rc = p->rank_to_idx.reserve(std::max<uint64_t>(n_idx, 1) * 4)) != YAMS_OK) return rc;
        if (n_idx) {
            YB_CUDA(cudaMemcpyAsync(p->tie_rank.p, rank.data(), n_idx * 4, cudaMemcpyHostToDevice, st));
            YB_CUDA(cudaMemcpyAsync(p->rank_to_idx.p, order.data(), n_idx * 4, cudaMemcpyHostToDevice, st));
        }
        YB_CUDA(cudaStreamSynchronize(st));
    }
    *out = p.release();
    return YAMS_OK;
    YB_CATCH
}

void yams_b200_pq_destroy(yams_b200_pq* p) { delete p; }

yams_status_t yams_b200_pq_codes(yams_b200_pq* p, uint8_t* out_codes, int64_t* out_rowids, uint64_t* out_n) {
    YB_TRY
    YB_ARG(p && out_n, "null argument");
    std::lock_guard<std::mutex> lk(p->mu);
    std::lock_guard<std::mutex> corpus_lock(p->corpus->mu);
    YB_BIND(p->corpus);
    *out_n = p->n_idx;
    cudaStream_t st = p->corpus->st;
    if (p->n_idx && out_codes) YB_CUDA(cudaMemcpyAsync(out_codes, p->codes.p, p->n_idx * p->m, cudaMemcpyDeviceToHost, st));
    if (p->n_idx && out_rowids) {
        std::vector<uint32_t> h_idx(p->n_idx);
        std::vector<int64_t> h_rid(p->corpus->n);
        YB_CUDA(cudaMemcpyAsync(h_idx.data(), p->idx_rows.p, p->n_idx * 4, cudaMemcpyDeviceToHost, st));
        YB_CUDA(cudaMemcpyAsync(h_rid.data(), p->corpus->rowids.p, p->corpus->n * 8, cudaMemcpyDeviceToHost, st));
        YB_CUDA(cudaStreamSynchronize(st));
        for (uint64_t j = 0; j < p->n_idx; ++j) out_rowids[j] = h_rid[h_idx[j]];
    }
    YB_CUDA(cudaStreamSynchronize(st));
    return YAMS_OK;
    YB_CATCH
}

}  // extern "C"

// a public search entry reports no results until a batch has written them
static void zero_outputs(uint32_t nq, uint32_t* out_counts, uint64_t* out_flags) {
    for (uint32_t q = 0; q < nq; ++q) out_counts[q] = 0;
    if (out_flags) for (uint32_t q = 0; q < nq; ++q) out_flags[q] = 0;
}

// rows the reference re-scores exactly, before the cut to the rows there are: max(k, k * max(1, rerank_factor)) (:3670, :3956-3959)
static uint64_t pq_rerank_budget(uint32_t k, uint32_t rerank_factor) {
    return std::max<uint64_t>(k, (uint64_t)k * std::max<uint32_t>(rerank_factor, 1));
}

// The query-table stage: p->lut and p->valid (pq_lut_kernel) of the nq queries at d_q, which are on the device already
static yams_status_t pq_build_luts(yams_b200_pq* p, const float* d_q, uint32_t nq, cudaStream_t st) {
    yams_status_t rc;
    const uint32_t m = p->m, kc = p->k, d = p->dim;
    if ((rc = p->lut.reserve((size_t)nq * m * kc * 4)) != YAMS_OK) return rc;
    if ((rc = p->valid.reserve((size_t)nq * 4)) != YAMS_OK) return rc;
    YB_CUDA(cudaFuncSetAttribute(pq_lut_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(d * 4)));
    pq_lut_kernel<<<nq, 256, d * 4, st>>>(d_q, d, p->codebooks.as<float>(), m, kc, p->lut.as<float>(), p->valid.as<uint32_t>());
    YB_CUDA(cudaGetLastError());
    return YAMS_OK;
}

// The tail of a search: the <= K selected (ADC score, tie rank) entries of every query -> corpus rows -> exact rerank against the
// queries at d_q -> final order -> the copies to the caller's arrays, enqueued.  The caller enqueues what else it reads back
// and waits for the stream, so a batch costs one host synchronisation.
static yams_status_t pq_rerank_and_emit(yams_b200_pq* p, const float* d_q, Cand* d_sel, const uint32_t* d_sel_n, uint32_t K, uint32_t nq, uint32_t k,
                                        float threshold, int64_t* out_rowids, float* out_scores, uint32_t* out_counts, uint64_t* out_flags) {
    yams_b200_corpus* c = p->corpus;
    cudaStream_t st = c->st;
    yams_status_t rc;
    DeviceResults r;
    if ((rc = p->exact.reserve((size_t)nq * K * sizeof(Exact))) != YAMS_OK) return rc;
    if ((rc = reserve_results(p->dout, nq, k, &r)) != YAMS_OK) return rc;
    const uint32_t tot = nq * K;
    pq_rank_to_row_kernel<<<(tot + 255) / 256, 256, 0, st>>>(d_sel, d_sel_n, K, nq, p->rank_to_idx.as<uint32_t>(), p->idx_rows.as<uint32_t>());
    pq_rerank_kernel<<<(tot + 127) / 128, 128, 0, st>>>(c->rows.p, c->dtype, p->dim, d_q, d_sel, d_sel_n, p->valid.as<uint32_t>(), K, nq, threshold,
                                                        p->exact.as<Exact>());
    launch_final_plain(p->exact.as<Exact>(), K, k, nq, c->rowids.as<int64_t>(), r, st);
    YB_CUDA(cudaGetLastError());
    return enqueue_results(r, nq, k, out_rowids, out_scores, out_counts, out_flags, st);
}

// the per-query lists (32 k entries each on the filtered path) bound the batch one pass can take: larger batches are sliced
static constexpr uint32_t kPqMaxBatch = 512;

// one batch of <= kPqMaxBatch queries; the caller holds both locks and has bound the device
static yams_status_t pq_search_batch(yams_b200_pq* p, const float* queries, uint32_t nq, uint32_t k, uint32_t rerank_factor, float threshold,
                                     int64_t* out_rowids, float* out_scores, uint32_t* out_counts, uint64_t* out_flags) {
    YB_TRY
    yams_b200_corpus* c = p->corpus;
    const uint32_t approx = (uint32_t)std::min<uint64_t>(p->n_idx, pq_rerank_budget(k, rerank_factor));   // :3956-3959
    YB_ARG(approx <= PQ_MAX_APPROX, "k * rerank_factor > 1024 is not supported by the PQ engine (use the exact scan)");
    cudaStream_t st = c->st;
    yams_status_t rc;
    const uint32_t m = p->m, kc = p->k, d = p->dim;
    const uint32_t tiles = (uint32_t)((p->n_idx + PQ_TILE - 1) / PQ_TILE);
    // Two ways to the same exact top-approx by (score, tie-break key):
    //   unfiltered: every tile keeps its own top-approx (bitonic network in shared memory) -> lists of tiles * approx entries;
    //   filtered  : a strided sample of tiles goes through the unfiltered path and yields the sample's approx-th best key tau
    //               (<= the global approx-th best key), then ONE pass over all rows appends the rows with key >= tau.
    // The filtered pass does no sorting (the unfiltered kernel spends ~10x its lookup work in the network); it is used when
    // the expected survivors (approx * tiles / sample tiles) fit the list with a 4x margin, and falls back when a list overflows.
    static const int force_unfiltered = [] { const char* e = getenv("YAMS_B200_PQ_UNFILTERED"); return e ? atoi(e) : 0; }();
    const uint32_t kFilterCap = 32768;
    uint32_t sample_tiles = 16;
    while ((uint64_t)approx * 4 * tiles > (uint64_t)kFilterCap * sample_tiles && sample_tiles < tiles) sample_tiles *= 2;
    const bool filtered = !force_unfiltered && tiles >= 4 * sample_tiles;
    const uint32_t cap_unf = tiles * approx;
    const uint32_t cap = filtered ? std::max<uint32_t>(kFilterCap, sample_tiles * approx) : cap_unf;
    if ((rc = p->q32.reserve((size_t)nq * d * 4)) != YAMS_OK) return rc;
    if ((rc = p->lists.reserve((size_t)nq * cap * sizeof(Cand))) != YAMS_OK) return rc;
    if ((rc = p->counts.reserve((size_t)nq * 4 + 16)) != YAMS_OK) return rc;
    if ((rc = p->sel.reserve((size_t)nq * approx * sizeof(Cand) + (size_t)nq * 4)) != YAMS_OK) return rc;
    if ((rc = p->tau.reserve((size_t)nq * 8)) != YAMS_OK) return rc;
    Cand* d_sel = p->sel.as<Cand>();
    uint32_t* d_sel_n = reinterpret_cast<uint32_t*>(d_sel + (size_t)nq * approx);
    uint32_t* d_counts = p->counts.as<uint32_t>();
    uint32_t* d_overflow = d_counts + nq;
    YB_CUDA(cudaMemcpyAsync(p->q32.p, queries, (size_t)nq * d * 4, cudaMemcpyHostToDevice, st));
    if ((rc = pq_build_luts(p, p->q32.as<float>(), nq, st)) != YAMS_OK) return rc;
    const size_t lut_bytes = (size_t)m * kc * 4;
    const size_t smem = ((lut_bytes + 7) & ~(size_t)7) + (size_t)PQ_TILE * 8;
    YB_CUDA(cudaFuncSetAttribute(pq_adc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    auto unfiltered = [&](uint32_t ntiles, uint32_t stride, uint32_t list_cap) {
        cudaMemsetAsync(d_counts, 0, (size_t)nq * 4 + 16, st);
        pq_adc_kernel<<<dim3(ntiles, nq), PQ_THREADS, smem, st>>>(p->codes.as<uint8_t>(), p->n_idx, m, kc, p->lut.as<float>(), p->tie_rank.as<uint32_t>(),
                                                                  approx, p->lists.as<Cand>(), list_cap, d_counts, stride);
        launch_topk_lists(p->lists.as<Cand>(), d_counts, list_cap, nq, approx, d_sel, d_sel_n, st);
    };
    p->last_path[0] = filtered ? 1u : 0u;
    p->last_path[1] = p->last_path[2] = p->last_path[3] = 0;
    if (filtered) {
        const uint32_t stride = tiles / sample_tiles;
        unfiltered(sample_tiles, stride, cap);
        pq_tau_kernel<<<(nq + 127) / 128, 128, 0, st>>>(d_sel, d_sel_n, approx, nq, p->tau.as<uint64_t>(), d_counts);
        int qg = nq >= 4 ? 4 : (nq >= 2 ? 2 : 1);
        while (qg > 1 && (size_t)qg * lut_bytes > 200 * 1024) qg >>= 1;
        p->last_path[1] = (uint32_t)qg;
        p->last_path[2] = sample_tiles;
        const uint32_t groups = (nq + qg - 1) / qg;
        uint64_t chunks = std::max<uint64_t>(1, (uint64_t)c->dev->sm_count * 6 / groups);
        chunks = std::min<uint64_t>(chunks, (p->n_idx + 2047) / 2048);
        uint64_t rows_per_cta = ((p->n_idx + chunks - 1) / chunks + PQ_THREADS - 1) / PQ_THREADS * PQ_THREADS;
        chunks = (p->n_idx + rows_per_cta - 1) / rows_per_cta;
#define YB_PQF(G)                                                                                                                              \
        YB_CUDA(cudaFuncSetAttribute(pq_adc_filter_kernel<G>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(G * lut_bytes)));             \
        pq_adc_filter_kernel<G><<<dim3((unsigned)chunks, groups), PQ_THREADS, G * lut_bytes, st>>>(                                            \
            p->codes.as<uint8_t>(), p->n_idx, m, kc, p->lut.as<float>(), p->tie_rank.as<uint32_t>(), p->tau.as<uint64_t>(), nq, rows_per_cta,   \
            p->lists.as<Cand>(), cap, d_counts)
        if (qg == 4) { YB_PQF(4); } else if (qg == 2) { YB_PQF(2); } else { YB_PQF(1); }
#undef YB_PQF
        pq_overflow_kernel<<<(nq + 127) / 128, 128, 0, st>>>(d_counts, nq, cap, d_overflow);
        launch_topk_lists(p->lists.as<Cand>(), d_counts, cap, nq, approx, d_sel, d_sel_n, st);
    } else {
        unfiltered(tiles, 1, cap);
    }
    auto tail = [&] {
        return pq_rerank_and_emit(p, p->q32.as<float>(), d_sel, d_sel_n, approx, nq, k, threshold, out_rowids, out_scores, out_counts, out_flags);
    };
    if ((rc = tail()) != YAMS_OK) return rc;
    uint32_t h_overflow = 0;
    if (filtered) YB_CUDA(cudaMemcpyAsync(&h_overflow, d_overflow, 4, cudaMemcpyDeviceToHost, st));
    YB_CUDA(cudaStreamSynchronize(st));
    if (!h_overflow) return YAMS_OK;
    // a filtered list overflowed: redo the selection without the filter
    p->last_path[3] = 1;
    if ((rc = p->lists.reserve((size_t)nq * cap_unf * sizeof(Cand))) != YAMS_OK) return rc;
    unfiltered(tiles, 1, cap_unf);
    if ((rc = tail()) != YAMS_OK) return rc;
    YB_CUDA(cudaStreamSynchronize(st));
    return YAMS_OK;
    YB_CATCH
}

extern "C" {

yams_status_t yams_b200_pq_search(yams_b200_pq* p, const float* queries, uint32_t nq, uint32_t k, uint32_t rerank_factor, float threshold,
                                  int64_t* out_rowids, float* out_scores, uint32_t* out_counts, uint64_t* out_flags) {
    YB_TRY
    YB_ARG(p && out_counts, "null argument");
    std::lock_guard<std::mutex> lk(p->mu);
    yams_b200_corpus* c = p->corpus;
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_BIND(c);
    zero_outputs(nq, out_counts, out_flags);
    for (uint32_t& v : p->last_path) v = 0;
    if (nq == 0 || k == 0 || p->n_idx == 0) return YAMS_OK;                           // :3873-3881
    YB_ARG(queries && out_rowids && out_scores, "null argument");
    YB_ARG(c->generation == p->corpus_generation, "the corpus changed after the PQ index was built: rebuild it (the reference marks the index dirty)");
    for (uint32_t q0 = 0; q0 < nq; q0 += kPqMaxBatch) {
        const uint32_t nb = std::min<uint32_t>(kPqMaxBatch, nq - q0);
        yams_status_t rc = pq_search_batch(p, queries + (size_t)q0 * p->dim, nb, k, rerank_factor, threshold, out_rowids + (size_t)q0 * k,
                                           out_scores + (size_t)q0 * k, out_counts + q0, out_flags ? out_flags + q0 : nullptr);
        if (rc != YAMS_OK) return rc;
    }
    return YAMS_OK;
    YB_CATCH
}

yams_status_t yams_b200_debug_pq_lut(yams_b200_pq* p, const float* queries, uint32_t nq, float* out_lut, uint32_t* out_valid) {
    YB_TRY
    YB_ARG(p && (nq == 0 || (queries && out_lut && out_valid)), "null argument");
    std::lock_guard<std::mutex> lk(p->mu);
    yams_b200_corpus* c = p->corpus;
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_BIND(c);
    if (nq == 0) return YAMS_OK;
    cudaStream_t st = c->st;
    yams_status_t rc;
    const uint32_t m = p->m, kc = p->k, d = p->dim;
    if ((rc = p->q32.reserve((size_t)nq * d * 4)) != YAMS_OK) return rc;
    YB_CUDA(cudaMemcpyAsync(p->q32.p, queries, (size_t)nq * d * 4, cudaMemcpyHostToDevice, st));
    if ((rc = pq_build_luts(p, p->q32.as<float>(), nq, st)) != YAMS_OK) return rc;
    YB_CUDA(cudaMemcpyAsync(out_lut, p->lut.p, (size_t)nq * m * kc * 4, cudaMemcpyDeviceToHost, st));
    YB_CUDA(cudaMemcpyAsync(out_valid, p->valid.p, (size_t)nq * 4, cudaMemcpyDeviceToHost, st));
    YB_CUDA(cudaStreamSynchronize(st));
    return YAMS_OK;
    YB_CATCH
}

yams_status_t yams_b200_debug_pq_last_path(yams_b200_pq* p, uint32_t* out) {
    YB_TRY
    YB_ARG(p && out, "null argument");
    std::lock_guard<std::mutex> lk(p->mu);
    for (int i = 0; i < 4; ++i) out[i] = p->last_path[i];
    return YAMS_OK;
    YB_CATCH
}

}  // extern "C"

// corpus row -> index position table of the handle (the caller holds both locks)
static yams_status_t ensure_row_to_idx(yams_b200_pq* p, cudaStream_t st) {
    if (p->row_to_idx_ready) return YAMS_OK;
    const uint64_t n = p->corpus->n;
    yams_status_t rc;
    if ((rc = p->row_to_idx.reserve(std::max<uint64_t>(n, 1) * 4)) != YAMS_OK) return rc;
    YB_CUDA(cudaMemsetAsync(p->row_to_idx.p, 0xFF, std::max<uint64_t>(n, 1) * 4, st));
    if (p->n_idx)
        pq_row_to_idx_kernel<<<(unsigned)std::min<uint64_t>((p->n_idx + 255) / 256, 65535), 256, 0, st>>>(p->idx_rows.as<uint32_t>(), p->n_idx,
                                                                                                         p->row_to_idx.as<uint32_t>());
    YB_CUDA(cudaGetLastError());
    p->row_to_idx_ready = true;
    return YAMS_OK;
}

// one batch of <= kPqMaxBatch queries of pq_search_candidates; offs: the batch's nq + 1 offsets into `allowed` (absolute)
static yams_status_t pq_candidates_batch(yams_b200_pq* p, const float* queries, uint32_t nq, uint32_t k, uint32_t rerank_factor, float threshold,
                                         const int64_t* allowed, const uint64_t* offs, int64_t* out_rowids, float* out_scores, uint32_t* out_counts,
                                         uint64_t* out_flags) {
    YB_TRY
    yams_b200_corpus* c = p->corpus;
    cudaStream_t st = c->st;
    yams_status_t rc;
    const uint32_t m = p->m, kc = p->k, d = p->dim;
    const uint64_t want = pq_rerank_budget(k, rerank_factor);
    const uint64_t base = offs[0], total = offs[nq] - base;
    uint64_t maxlen = 0;
    for (uint32_t q = 0; q < nq; ++q) maxlen = std::max(maxlen, offs[q + 1] - offs[q]);
    YB_ARG(maxlen < 0xFFFFFFFFull, "candidate list too long");
    // approxK = min(candidateCount, max(k, k * rerank_factor)) (:3956-3959).  candidateCount (distinct indexed candidates) is
    // known on the device only: list lengths bound it; when the bound allows approxK > 1024 the selection keeps one more and
    // the limit is checked on the selected counts.
    uint32_t K = (uint32_t)std::max<uint64_t>(1, std::min(want, maxlen));
    const bool check_after = K > PQ_MAX_APPROX;
    if (check_after) K = PQ_MAX_APPROX + 1;
    const uint32_t cap = (uint32_t)std::max<uint64_t>(maxlen, 1);
    const uint64_t bits_ld = (p->n_idx + 31) / 32;
    if ((rc = ensure_row_to_idx(p, st)) != YAMS_OK) return rc;
    Staging in;
    const size_t o_q = in.add(queries, (size_t)nq * d * 4);
    const size_t o_al = in.add(allowed ? allowed + base : nullptr, (size_t)total * 8);
    std::vector<uint64_t> roffs(nq + 1);
    for (uint32_t q = 0; q <= nq; ++q) roffs[q] = offs[q] - base;
    const size_t o_of = in.add(roffs.data(), (size_t)(nq + 1) * 8);
    if ((rc = p->cin.reserve(in.h.size())) != YAMS_OK) return rc;
    if ((rc = p->mapped.reserve(std::max<uint64_t>(total, 1) * sizeof(Cand))) != YAMS_OK) return rc;
    if ((rc = p->cidx.reserve(std::max<uint64_t>(total, 1) * 4)) != YAMS_OK) return rc;
    if ((rc = p->bits.reserve((size_t)nq * bits_ld * 4 + 4)) != YAMS_OK) return rc;
    if ((rc = p->lists.reserve((size_t)nq * cap * sizeof(Cand))) != YAMS_OK) return rc;
    if ((rc = p->counts.reserve((size_t)nq * 4 + 16)) != YAMS_OK) return rc;
    if ((rc = p->sel.reserve((size_t)nq * K * sizeof(Cand) + (size_t)nq * 4)) != YAMS_OK) return rc;
    unsigned char* din = p->cin.as<unsigned char>();
    const float* d_q = reinterpret_cast<const float*>(din + o_q);
    const int64_t* d_al = reinterpret_cast<const int64_t*>(din + o_al);
    const uint64_t* d_of = reinterpret_cast<const uint64_t*>(din + o_of);
    uint32_t* d_counts = p->counts.as<uint32_t>();
    Cand* d_sel = p->sel.as<Cand>();
    uint32_t* d_sel_n = reinterpret_cast<uint32_t*>(d_sel + (size_t)nq * K);
    YB_CUDA(cudaMemcpyAsync(din, in.h.data(), in.h.size(), cudaMemcpyHostToDevice, st));
    YB_CUDA(cudaMemsetAsync(p->bits.p, 0, (size_t)nq * bits_ld * 4 + 4, st));
    YB_CUDA(cudaMemsetAsync(d_counts, 0, (size_t)nq * 4, st));
    if ((rc = pq_build_luts(p, d_q, nq, st)) != YAMS_OK) return rc;
    launch_map_rowids(d_al, total, c->rowids.as<int64_t>(), c->n, p->mapped.as<Cand>(), st);
    if (total) {
        const unsigned gx = (unsigned)std::min<uint64_t>((maxlen + 255) / 256, 256);
        pq_cand_index_kernel<<<dim3(gx, nq), 256, 0, st>>>(p->mapped.as<Cand>(), d_of, p->row_to_idx.as<uint32_t>(), p->bits.as<uint32_t>(), bits_ld,
                                                           p->cidx.as<uint32_t>(), d_counts);
        const uint32_t per_cta = 2048;
        const size_t lut_bytes = (size_t)m * kc * 4;
        YB_CUDA(cudaFuncSetAttribute(pq_adc_gather_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lut_bytes));
        pq_adc_gather_kernel<<<dim3((unsigned)((maxlen + per_cta - 1) / per_cta), nq), PQ_THREADS, lut_bytes, st>>>(
            p->codes.as<uint8_t>(), m, kc, p->lut.as<float>(), p->tie_rank.as<uint32_t>(), p->cidx.as<uint32_t>(), d_of, d_counts, per_cta,
            p->lists.as<Cand>(), cap);
    }
    launch_topk_lists(p->lists.as<Cand>(), d_counts, cap, nq, K, d_sel, d_sel_n, st);
    if ((rc = pq_rerank_and_emit(p, d_q, d_sel, d_sel_n, K, nq, k, threshold, out_rowids, out_scores, out_counts, out_flags)) != YAMS_OK) return rc;
    std::vector<uint32_t> sel_n(check_after ? nq : 0);
    if (check_after) YB_CUDA(cudaMemcpyAsync(sel_n.data(), d_sel_n, (size_t)nq * 4, cudaMemcpyDeviceToHost, st));
    YB_CUDA(cudaStreamSynchronize(st));
    for (uint32_t q = 0; q < (check_after ? nq : 0); ++q) {
        if (sel_n[q] > PQ_MAX_APPROX) {
            for (uint32_t i = 0; i < nq; ++i) out_counts[i] = 0;
            YB_ARG(false, "k * rerank_factor > 1024 is not supported by the PQ engine (use the exact scan)");
        }
    }
    return YAMS_OK;
    YB_CATCH
}

// every rowid of one query's documents at most once: a stamp table over the rowid range when it is small, else a sort per query
static bool rowids_unique_per_query(const int64_t* rid, const uint64_t* doc_offsets, const uint64_t* query_docs, uint32_t nq) {
    const uint64_t p0 = doc_offsets[query_docs[0]], p1 = doc_offsets[query_docs[nq]];
    if (p1 == p0) return true;
    int64_t lo = INT64_MAX, hi = INT64_MIN;
    for (uint64_t i = p0; i < p1; ++i) { lo = std::min(lo, rid[i]); hi = std::max(hi, rid[i]); }
    const uint64_t range = (uint64_t)hi - (uint64_t)lo + 1;
    if (range != 0 && range <= std::max<uint64_t>(16 * (p1 - p0), 1ull << 22)) {
        std::vector<uint32_t> stamp(range, 0u);
        for (uint32_t q = 0; q < nq; ++q)
            for (uint64_t i = doc_offsets[query_docs[q]]; i < doc_offsets[query_docs[q + 1]]; ++i) {
                uint32_t& s = stamp[(uint64_t)rid[i] - (uint64_t)lo];
                if (s == q + 1) return false;
                s = q + 1;
            }
        return true;
    }
    std::vector<int64_t> v;
    for (uint32_t q = 0; q < nq; ++q) {
        v.assign(rid + doc_offsets[query_docs[q]], rid + doc_offsets[query_docs[q + 1]]);
        std::sort(v.begin(), v.end());
        if (std::adjacent_find(v.begin(), v.end()) != v.end()) return false;
    }
    return true;
}

// one slice of search_documents: queries [q0, q1); the caller holds the locks, has checked the input and bound the device
static yams_status_t documents_slice(yams_b200_corpus* c, yams_b200_pq* pq, const float* queries, uint32_t q0, uint32_t q1, uint32_t k,
                                     float threshold, const int64_t* doc_rowids, const uint64_t* doc_offsets, const uint64_t* query_docs,
                                     int64_t* out_docs, int64_t* out_rowids, float* out_scores, uint32_t* out_counts) {
    YB_TRY
    cudaStream_t st = c->st;
    yams_status_t rc;
    const uint32_t nq = q1 - q0, d = c->dim;
    const uint64_t sd0 = query_docs[q0], ndocs = query_docs[q1] - sd0;
    const uint64_t p0 = doc_offsets[sd0], np = doc_offsets[query_docs[q1]] - p0;
    uint64_t cap = 1;
    for (uint32_t q = q0; q < q1; ++q) cap = std::max<uint64_t>(cap, query_docs[q + 1] - query_docs[q]);
    Staging in;
    const size_t o_q = in.add(queries + (size_t)q0 * d, (size_t)nq * d * 4);
    const size_t o_rid = in.add(np ? doc_rowids + p0 : nullptr, (size_t)np * 8);
    std::vector<uint64_t> v(ndocs + 1);
    for (uint64_t i = 0; i <= ndocs; ++i) v[i] = doc_offsets[sd0 + i] - p0;
    const size_t o_doff = in.add(v.data(), (size_t)(ndocs + 1) * 8);
    v.resize(nq + 1);
    for (uint32_t q = 0; q <= nq; ++q) v[q] = query_docs[q0 + q] - sd0;
    const size_t o_qdocs = in.add(v.data(), (size_t)(nq + 1) * 8);
    for (uint32_t q = 0; q <= nq; ++q) v[q] = doc_offsets[query_docs[q0 + q]] - p0;
    const size_t o_qpair = in.add(v.data(), (size_t)(nq + 1) * 8);
    // device workspace of the corpus (its lock is held): staged input, pairs, document lists, selection, outputs
    const size_t lists_b = (size_t)nq * cap * sizeof(Cand);
    const size_t out_b = (size_t)nq * k * 20 + (size_t)nq * 4 + 4;
    if ((rc = c->mask.reserve(in.h.size())) != YAMS_OK) return rc;
    if ((rc = c->sel.reserve(std::max<uint64_t>(np, 1) * sizeof(Cand))) != YAMS_OK) return rc;
    if ((rc = c->cands.reserve(lists_b + (size_t)nq * 4 + std::max<uint64_t>(ndocs, 1) * 4)) != YAMS_OK) return rc;
    if ((rc = c->outbuf.reserve((size_t)nq * k * sizeof(Cand) + (size_t)nq * 4)) != YAMS_OK) return rc;
    if ((rc = c->misc.reserve((size_t)nq * 16)) != YAMS_OK) return rc;
    if ((rc = c->status.reserve(16)) != YAMS_OK) return rc;
    if ((rc = c->dout.reserve(out_b)) != YAMS_OK) return rc;
    unsigned char* din = c->mask.as<unsigned char>();
    const float* d_q = reinterpret_cast<const float*>(din + o_q);
    const int64_t* d_rid = reinterpret_cast<const int64_t*>(din + o_rid);
    const uint64_t* d_doff = reinterpret_cast<const uint64_t*>(din + o_doff);
    const uint64_t* d_qdocs = reinterpret_cast<const uint64_t*>(din + o_qdocs);
    const uint64_t* d_qpair = reinterpret_cast<const uint64_t*>(din + o_qpair);
    Cand* d_pairs = c->sel.as<Cand>();
    Cand* d_lists = c->cands.as<Cand>();
    uint32_t* d_counts = reinterpret_cast<uint32_t*>(c->cands.as<unsigned char>() + lists_b);
    uint32_t* d_best = d_counts + nq;
    Cand* d_sel = c->outbuf.as<Cand>();
    uint32_t* d_sel_n = reinterpret_cast<uint32_t*>(d_sel + (size_t)nq * k);
    double* d_qnorm = c->misc.as<double>();
    float* d_qinv = reinterpret_cast<float*>(d_qnorm + nq);
    uint32_t* d_valid = reinterpret_cast<uint32_t*>(d_qinv + nq);
    int64_t* o_docs = c->dout.as<int64_t>();
    int64_t* o_rows = o_docs + (size_t)nq * k;
    float* o_sc = reinterpret_cast<float*>(o_rows + (size_t)nq * k);
    uint32_t* o_cnt = reinterpret_cast<uint32_t*>(o_sc + (size_t)nq * k);
    uint32_t* o_invalid = o_cnt + nq;
    YB_CUDA(cudaMemcpyAsync(din, in.h.data(), in.h.size(), cudaMemcpyHostToDevice, st));
    YB_CUDA(cudaMemsetAsync(d_counts, 0, (size_t)nq * 4, st));
    YB_CUDA(cudaMemsetAsync(c->status.p, 0, 16, st));
    if (pq) {
        if ((rc = ensure_row_to_idx(pq, st)) != YAMS_OK) return rc;
        pq_query_valid_kernel<<<(nq + 127) / 128, 128, 0, st>>>(d_q, nq, d, d_valid);
    } else {
        launch_query_prep(d_q, nq, d, d_qnorm, d_qinv, c->status.p, st);
    }
    launch_map_rowids(d_rid, np, c->rowids.as<int64_t>(), c->n, d_pairs, st);
    if (np)
        doc_score_kernel<<<(unsigned)((np + 127) / 128), 128, 0, st>>>(c->rows.p, c->dtype, d, d_q, d_qnorm, d_valid,
                                                                      pq ? pq->row_to_idx.as<uint32_t>() : nullptr, d_qpair, nq, np, threshold, d_pairs);
    if (ndocs)
        doc_argmax_kernel<<<(unsigned)((ndocs * 32 + 255) / 256), 256, 0, st>>>(d_pairs, d_doff, (uint32_t)ndocs, d_qdocs, nq, d_lists, (uint32_t)cap,
                                                                               d_counts, d_best);
    launch_topk_lists(d_lists, d_counts, (uint32_t)cap, nq, k, d_sel, d_sel_n, st);
    doc_emit_kernel<<<(unsigned)(((uint64_t)nq * k + 255) / 256), 256, 0, st>>>(d_sel, d_sel_n, k, nq, sd0, d_best, c->rowids.as<int64_t>(), o_docs,
                                                                                o_rows, o_sc, o_cnt);
    YB_CUDA(cudaMemcpyAsync(o_invalid, c->status.p, 4, cudaMemcpyDeviceToDevice, st));
    YB_CUDA(cudaGetLastError());
    std::vector<unsigned char> h(out_b);
    YB_CUDA(cudaMemcpyAsync(h.data(), c->dout.p, out_b, cudaMemcpyDeviceToHost, st));
    YB_CUDA(cudaStreamSynchronize(st));
    const unsigned char* hp = h.data();
    uint32_t n_invalid = 0;
    memcpy(&n_invalid, hp + (size_t)nq * k * 20 + (size_t)nq * 4, 4);
    YB_ARG(pq || n_invalid == 0, "exact vector search requires a finite, non-zero query embedding");   // :4127-4130
    memcpy(out_docs + (size_t)q0 * k, hp, (size_t)nq * k * 8);
    memcpy(out_rowids + (size_t)q0 * k, hp + (size_t)nq * k * 8, (size_t)nq * k * 8);
    memcpy(out_scores + (size_t)q0 * k, hp + (size_t)nq * k * 16, (size_t)nq * k * 4);
    memcpy(out_counts + q0, hp + (size_t)nq * k * 20, (size_t)nq * 4);
    return YAMS_OK;
    YB_CATCH
}

extern "C" {

yams_status_t yams_b200_pq_search_candidates(yams_b200_pq* p, const float* queries, uint32_t nq, uint32_t k, uint32_t rerank_factor, float threshold,
                                             const int64_t* allowed_rowids, const uint64_t* allowed_offsets, int64_t* out_rowids, float* out_scores,
                                             uint32_t* out_counts, uint64_t* out_flags) {
    YB_TRY
    YB_ARG(p && out_counts, "null argument");
    std::lock_guard<std::mutex> lk(p->mu);
    yams_b200_corpus* c = p->corpus;
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_BIND(c);
    zero_outputs(nq, out_counts, out_flags);
    if (nq == 0 || k == 0 || p->n_idx == 0) return YAMS_OK;
    YB_ARG(queries && out_rowids && out_scores && allowed_offsets, "null argument");
    for (uint32_t q = 0; q < nq; ++q) YB_ARG(allowed_offsets[q] <= allowed_offsets[q + 1], "allowed_offsets must be non-decreasing");
    YB_ARG(allowed_rowids || allowed_offsets[nq] == allowed_offsets[0], "allowed_rowids missing");
    YB_ARG(c->generation == p->corpus_generation, "the corpus changed after the PQ index was built: rebuild it (the reference marks the index dirty)");
    for (uint32_t q0 = 0; q0 < nq; q0 += kPqMaxBatch) {
        const uint32_t nb = std::min<uint32_t>(kPqMaxBatch, nq - q0);
        yams_status_t rc = pq_candidates_batch(p, queries + (size_t)q0 * p->dim, nb, k, rerank_factor, threshold, allowed_rowids, allowed_offsets + q0,
                                               out_rowids + (size_t)q0 * k, out_scores + (size_t)q0 * k, out_counts + q0,
                                               out_flags ? out_flags + q0 : nullptr);
        if (rc != YAMS_OK) {
            for (uint32_t q = 0; q < nq; ++q) out_counts[q] = 0;
            return rc;
        }
    }
    return YAMS_OK;
    YB_CATCH
}

yams_status_t yams_b200_search_documents(yams_b200_corpus* c, yams_b200_pq* pq, const float* queries, uint32_t nq, uint32_t k, float threshold,
                                         const int64_t* doc_rowids, const uint64_t* doc_offsets, const uint64_t* query_docs, int64_t* out_docs,
                                         int64_t* out_rowids, float* out_scores, uint32_t* out_counts) {
    YB_TRY
    YB_ARG(c && out_counts, "null argument");
    std::unique_lock<std::mutex> pq_lock;
    if (pq) pq_lock = std::unique_lock<std::mutex>(pq->mu);
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_BIND(c);
    settle_pending(c);
    zero_outputs(nq, out_counts, nullptr);
    if (nq == 0) return YAMS_OK;
    YB_ARG(queries && query_docs && out_docs && out_rowids && out_scores, "null argument");
    YB_ARG(c->metric == YAMS_B200_COSINE, "document search is defined for the cosine scan");
    if (pq) {
        YB_ARG(pq->corpus == c, "the PQ index belongs to another corpus");
        YB_ARG(c->generation == pq->corpus_generation, "the corpus changed after the PQ index was built: rebuild it (the reference marks the index dirty)");
    }
    YB_ARG(k <= 4096, "k > 4096 documents per query is not supported");
    for (uint32_t q = 0; q < nq; ++q) YB_ARG(query_docs[q] <= query_docs[q + 1], "query_docs must be non-decreasing");
    const uint64_t d0 = query_docs[0], d1 = query_docs[nq];
    YB_ARG(d1 - d0 < 0xFFFFFFFFull, "too many documents in one call");
    YB_ARG(doc_offsets, "null argument");
    for (uint64_t i = d0; i < d1; ++i) {
        YB_ARG(doc_offsets[i] <= doc_offsets[i + 1], "doc_offsets must be non-decreasing");
        YB_ARG(doc_offsets[i + 1] - doc_offsets[i] < 0xFFFFFFFFull, "document too long");
    }
    const uint64_t total = doc_offsets[d1] - doc_offsets[d0];
    YB_ARG(total == 0 || doc_rowids, "doc_rowids missing");
    YB_ARG(total == 0 || rowids_unique_per_query(doc_rowids, doc_offsets, query_docs, nq),
           "a rowid appears twice among one query's documents (documents are disjoint row sets)");
    if (k == 0) return YAMS_OK;
    // slices of <= kPqMaxBatch queries and a bounded number of (query, row) pairs; one host synchronisation each
    const uint64_t kMaxPairs = 1ull << 26;
    for (uint32_t q0 = 0; q0 < nq;) {
        uint32_t q1 = q0 + 1;
        while (q1 < nq && q1 - q0 < kPqMaxBatch && doc_offsets[query_docs[q1 + 1]] - doc_offsets[query_docs[q0]] <= kMaxPairs) ++q1;
        yams_status_t rc = documents_slice(c, pq, queries, q0, q1, k, threshold, doc_rowids, doc_offsets, query_docs, out_docs, out_rowids, out_scores,
                                           out_counts);
        if (rc != YAMS_OK) {
            for (uint32_t q = 0; q < nq; ++q) out_counts[q] = 0;
            return rc;
        }
        q0 = q1;
    }
    return YAMS_OK;
    YB_CATCH
}

}  // extern "C"
