// cosine.cuh -- the exact scan's per-row similarity, shared by its re-scoring kernel (knn.cu) and the document pass (pq.cu),
// and the score keys both order by.
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

// bruteForceSearchUnlocked's cosine (sqlite_vec_backend.cpp:4253-4279) of corpus row `row` against the query qv (fp32, 16-byte
// aligned) of double norm qnorm: sequential double accumulation, skip rules (a non-finite element or |row|^2 <= 1e-12), float
// cast of dot / (|row| * |q|), `sim < threshold` dropped.  -> true and *out = sim when the row is a result.
__device__ __forceinline__ bool exact_cosine_sim(const void* __restrict__ rows, int dtype, uint32_t d, uint32_t row, const float* __restrict__ qv,
                                                 double qnorm, float threshold, float* out) {
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

}  // namespace yb
