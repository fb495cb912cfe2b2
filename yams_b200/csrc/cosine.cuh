// cosine.cuh -- device building blocks shared by the exact scan (knn.cu), the PQ engine (pq.cu) and the sqlite-vec operators
// (operators.cu): the exact per-row similarity, the score keys every ordered path ranks by, the in-block key sort and the
// rowid -> row lookup.
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

// Sequential double sums of corpus row `row` against qv (fp32, 16-byte aligned): *norm_sq = sum r^2, *dot = sum r q, in the
// reference's element order; -> false when the row holds a non-finite element (the sums are then partial).
__device__ __forceinline__ bool row_dot(const void* __restrict__ rows, int dtype, uint32_t d, uint32_t row, const float* __restrict__ qv,
                                        double* norm_sq_out, double* dot_out) {
    const uint64_t base = (uint64_t)row * d;
    double norm_sq = 0.0, dot = 0.0;
    bool finite = true;
    // same element order as the reference's loop; only the loads are widened (16-byte row and query chunks)
    uint32_t c = 0;
    if (dtype == YAMS_B200_F16 && d % 8 == 0) {
        const uint4* rp = reinterpret_cast<const uint4*>(static_cast<const __half*>(rows) + base);
        const float4* qp = reinterpret_cast<const float4*>(qv);
        for (; c < d; c += 8) {
            const uint4 raw = __ldg(rp + (c >> 3));
            const float4 q0 = __ldg(qp + (c >> 2)), q1 = __ldg(qp + (c >> 2) + 1);
            const __half2* h2 = reinterpret_cast<const __half2*>(&raw);
            const float2 f0 = __half22float2(h2[0]), f1 = __half22float2(h2[1]), f2 = __half22float2(h2[2]), f3 = __half22float2(h2[3]);
            const float rv[8] = {f0.x, f0.y, f1.x, f1.y, f2.x, f2.y, f3.x, f3.y};
            const float qq[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                if (!isfinite(rv[e])) finite = false;
                const double sv = (double)rv[e];
                norm_sq += sv * sv;
                dot += sv * (double)qq[e];
            }
        }
    } else if (dtype == YAMS_B200_F32 && d % 4 == 0) {
        const float4* rp = reinterpret_cast<const float4*>(static_cast<const float*>(rows) + base);
        const float4* qp = reinterpret_cast<const float4*>(qv);
        for (; c < d; c += 4) {
            const float4 r4 = __ldg(rp + (c >> 2)), q4 = __ldg(qp + (c >> 2));
            const float rv[4] = {r4.x, r4.y, r4.z, r4.w};
            const float qq[4] = {q4.x, q4.y, q4.z, q4.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                if (!isfinite(rv[e])) finite = false;
                const double sv = (double)rv[e];
                norm_sq += sv * sv;
                dot += sv * (double)qq[e];
            }
        }
    }
    for (; c < d; ++c) {
        float v = load_elem(rows, dtype, base + c);
        if (!isfinite(v)) { finite = false; break; }
        double sv = (double)v, qd = (double)qv[c];
        norm_sq += sv * sv;
        dot += sv * qd;
    }
    *norm_sq_out = norm_sq;
    *dot_out = dot;
    return finite;
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
