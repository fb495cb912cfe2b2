// cosine.cuh -- device building blocks shared by the exact scan (knn.cu), the PQ engine (pq.cu), k-means (kmeans.cu) and the
// sqlite-vec operators (operators.cu): the double-precision element walk over a row and the exact similarities built on it, the
// score keys every ordered path ranks by, the in-block key sort and the rowid -> row lookup.
#pragma once
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"

namespace yb {

__device__ __forceinline__ float load_elem(const void* rows, int dtype, uint64_t idx) {
    if (dtype == YAMS_B200_F16) return __half2float(reinterpret_cast<const __half*>(rows)[idx]);
    return reinterpret_cast<const float*>(rows)[idx];
}

// monotone 32-bit key of a score (a descending key sort is a descending score sort); NaN ranks last
__device__ __forceinline__ uint32_t fkey(float f) {
    if (f != f) return 0u;
    uint32_t b = __float_as_uint(f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float fkey_inv(uint32_t k) {
    uint32_t b = (k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k;
    return __uint_as_float(b);
}

// The sort key of an entry: (fkey(score) << 32) | (0xFFFFFFFF - row).  Descending key order is score descending, then row
// ascending; key 0 marks "no entry".  word_key takes the score word fkey(score) of a caller that has already tested it.
// knn.cu's sel_key writes this format out on purpose, to keep topk_select_kernel's machine code (see there).
__device__ __forceinline__ uint64_t word_key(uint32_t w, uint32_t row) { return ((uint64_t)w << 32) | (uint64_t)(0xFFFFFFFFu - row); }
__device__ __forceinline__ uint64_t score_key(float s, uint32_t row) { return word_key(fkey(s), row); }
__device__ __forceinline__ float key_score(uint64_t key) { return fkey_inv((uint32_t)(key >> 32)); }
__device__ __forceinline__ uint32_t key_row(uint64_t key) { return 0xFFFFFFFFu - (uint32_t)key; }

// bitonic sort, descending, of buf[0, n) in shared memory (n a power of two) by the block's NT threads; ends with a barrier
template <int NT, typename T>
__device__ __forceinline__ void block_sort_desc(T* buf, uint32_t n) {
    for (uint32_t size = 2; size <= n; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t t = threadIdx.x; t < n / 2; t += NT) {
                const uint32_t lo = (t / stride) * (stride * 2) + (t % stride), hi = lo + stride;
                const bool desc = ((lo & size) == 0);
                const T x = buf[lo], y = buf[hi];
                if ((x < y) == desc) { buf[lo] = y; buf[hi] = x; }
            }
            __syncthreads();
        }
    }
}

// index of `want` in the ascending rowid table rowids[0, n), or n when it is not there
__device__ __forceinline__ uint64_t find_row(const int64_t* __restrict__ rowids, uint64_t n, int64_t want) {
    uint64_t a = 0, b = n;
    while (a < b) {
        const uint64_t m = a + ((b - a) >> 1);
        if (rowids[m] < want) a = m + 1; else b = m;
    }
    return (a < n && rowids[a] == want) ? a : n;
}

// f(x) for each element x of the N-element 16-byte chunk `raw` (fp16: N = 8, fp32: N = 4) that starts at element c; PAIR:
// f(x, y), y the matching element of the fp32 vector v, read one element at a time: where the threads of a warp share the vector
// (the re-scoring kernels, the k-means init) these reads are broadcasts, and 16-byte reads of it take pq_rerank_kernel past the
// 32 registers of full occupancy
template <bool PAIR, int N, typename F>
__device__ __forceinline__ void visit_chunk(const uint4& raw, const float* __restrict__ v, uint32_t c, F& f) {
    float x[N];
    if constexpr (N == 8) {
        const __half2* h2 = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 p = __half22float2(h2[e]);
            x[2 * e] = p.x;
            x[2 * e + 1] = p.y;
        }
    } else {
        x[0] = __uint_as_float(raw.x); x[1] = __uint_as_float(raw.y); x[2] = __uint_as_float(raw.z); x[3] = __uint_as_float(raw.w);
    }
    if constexpr (PAIR) {
#pragma unroll
        for (int e = 0; e < N; ++e) f(x[e], __ldg(v + c + e));
    } else {
#pragma unroll
        for (int e = 0; e < N; ++e) f(x[e]);
    }
}

// the d / N chunks of a row (d % N == 0), G per trip with their loads issued together, then the rest one per trip
template <bool PAIR, int G, int N, typename F>
__device__ __forceinline__ void walk_chunks(const uint4* __restrict__ rp, uint32_t d, const float* __restrict__ v, F& f) {
    uint32_t c = 0;
#pragma unroll 1
    for (; c + G * N <= d; c += G * N) {
        uint4 raw[G];
#pragma unroll
        for (int g = 0; g < G; ++g) raw[g] = __ldg(rp + c / N + g);
#pragma unroll
        for (int g = 0; g < G; ++g) visit_chunk<PAIR, N>(raw[g], v, c + g * N, f);
    }
#pragma unroll 1
    for (; c < d; c += N) visit_chunk<PAIR, N>(__ldg(rp + c / N), v, c, f);
}

template <bool PAIR, int G, typename F>
__device__ __forceinline__ void walk_elems(const void* __restrict__ rows, int dtype, uint32_t d, uint64_t row, const float* __restrict__ v,
                                           F& f) {
    const uint64_t base = row * d;
    if (dtype == YAMS_B200_F16 && d % 8 == 0) {
        walk_chunks<PAIR, G, 8>(reinterpret_cast<const uint4*>(static_cast<const __half*>(rows) + base), d, v, f);
    } else if (dtype == YAMS_B200_F32 && d % 4 == 0) {
        walk_chunks<PAIR, G, 4>(reinterpret_cast<const uint4*>(static_cast<const float*>(rows) + base), d, v, f);
    } else {
#pragma unroll 1
        for (uint32_t c = 0; c < d; ++c) {
            const float x = load_elem(rows, dtype, base + c);
            if constexpr (PAIR) f(x, v[c]);
            else f(x);
        }
    }
}

// The element walk of every exact path (the reference sums floats into a double in element order): f(x) for each element x of
// row `row` of the [rows][d] fp16/fp32 array, widened exactly to float, in element order.  An fp32 query row is walked with
// dtype F32.  Loads are 16 bytes wide where d keeps every row 16-byte aligned (fp16: d % 8 == 0, fp32: d % 4 == 0), and one
// element at a time otherwise.  G > 1 issues the loads of G 16-byte chunks together, for callers whose kernels have the
// registers to spare (one dependent load per trip leaves a thread latency-bound).  There is no early exit: f sees every
// element and does the accumulating and any finiteness tracking.
template <int G = 1, typename F>
__device__ __forceinline__ void walk_row(const void* __restrict__ rows, int dtype, uint32_t d, uint64_t row, F&& f) {
    walk_elems<false, G>(rows, dtype, d, row, nullptr, f);
}
// ... f(x, y) with y the matching element of the fp32 vector v
template <int G = 1, typename F>
__device__ __forceinline__ void walk_row_pair(const void* __restrict__ rows, int dtype, uint32_t d, uint64_t row, const float* __restrict__ v,
                                              F&& f) {
    walk_elems<true, G>(rows, dtype, d, row, v, f);
}

// Sequential double sums of corpus row `row` against qv (fp32): *norm_sq = sum r^2, *dot = sum r q, in the reference's element
// order; -> false when the row holds a non-finite element (the sums then mean nothing).  Four chunks per trip: the re-scoring
// kernels stay within the registers of their occupancy.
__device__ __forceinline__ bool row_dot(const void* __restrict__ rows, int dtype, uint32_t d, uint32_t row, const float* __restrict__ qv,
                                        double* norm_sq_out, double* dot_out) {
    double norm_sq = 0.0, dot = 0.0;
    bool finite = true;
    walk_row_pair<4>(rows, dtype, d, row, qv, [&](float x, float y) {
        if (!isfinite(x)) finite = false;
        norm_sq += (double)x * x;
        dot += (double)x * y;
    });
    *norm_sq_out = norm_sq;
    *dot_out = dot;
    return finite;
}

// VectorDatabase::computeCosineSimilarity (vector_database.cpp:1786-1810) of the fp32 vector a against row `row`: double sums
// of a.b, a^2 and b^2 in element order, 0 when either norm is 0, else dot / (|a| |b|)
__device__ __forceinline__ double compute_cosine_similarity(const void* __restrict__ rows, int dtype, uint32_t d, uint64_t row,
                                                            const float* __restrict__ a) {
    double dp = 0.0, na = 0.0, nb = 0.0;
    walk_row_pair(rows, dtype, d, row, a, [&](float y, float x) {   // the reference's names: x of a, y of the row (its b)
        dp += (double)x * y;
        na += (double)x * x;
        nb += (double)y * y;
    });
    na = sqrt(na);
    nb = sqrt(nb);
    return (na == 0.0 || nb == 0.0) ? 0.0 : dp / (na * nb);
}

// bruteForceSearchUnlocked's cosine (sqlite_vec_backend.cpp:4253-4279) of corpus row `row` against the query qv (fp32, 16-byte
// aligned) of double norm qnorm: sequential double accumulation, skip rules (a non-finite element or |row|^2 <= 1e-12), float
// cast of dot / (|row| * |q|), `sim < threshold` dropped.  -> true and *out = sim when the row is a result.
__device__ __forceinline__ bool exact_cosine_sim(const void* __restrict__ rows, int dtype, uint32_t d, uint32_t row, const float* __restrict__ qv,
                                                 double qnorm, float threshold, float* out) {
    double norm_sq, dot;
    const bool finite = row_dot(rows, dtype, d, row, qv, &norm_sq, &dot);
    if (finite && norm_sq > 1e-12) {
        double denom = sqrt(norm_sq) * qnorm;
        double simd = denom > 0.0 ? dot / denom : 0.0;
        if (isfinite(simd)) {
            float sim = (float)simd;
            if (!(sim < threshold)) {
                *out = sim;
                return true;
            }
        }
    }
    return false;
}

// the semantic-neighbour graph's cosineSimilarity (EmbeddingService.cpp:417-431) of corpus row `row` (graph scale inv_n > 0)
// against the source qv (graph scale inv_s > 0): float((dot * (double)inv_s) * (double)inv_n), the loads and element order of
// exact_cosine_sim; `sim < threshold` dropped.  -> true and *out = sim when the row is a result.
__device__ __forceinline__ bool semantic_sim(const void* __restrict__ rows, int dtype, uint32_t d, uint32_t row, const float* __restrict__ qv,
                                             float inv_s, float inv_n, float threshold, float* out) {
    double norm_sq, dot;
    row_dot(rows, dtype, d, row, qv, &norm_sq, &dot);
    const float sim = (float)((dot * (double)inv_s) * (double)inv_n);
    if (sim < threshold) return false;
    *out = sim;
    return true;
}

}  // namespace yb
