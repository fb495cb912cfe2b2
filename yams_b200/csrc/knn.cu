// knn.cu -- exact brute-force vector scan: CUDA-core stage-1 engine, top-K' selection, fp64
// rescoring, final ordering, the device key sort, corpus mirror and the vector_scan_v1 entry points.  The stateless
// sqlite-vec operators live in operators.cu.
//
// Reference semantics matched (paths under /root/reference):
//   bruteForceSearchUnlocked fast path   src/vector/sqlite_vec_backend.cpp:4203-4331
//   isFinite / isZeroNorm query checks   src/vector/sqlite_vec_backend.cpp:204-235, 4127-4130
//   vec0_run_exact_query                 third_party/sqlite-vec-cpp/.../sqlite/vec0_module.hpp:376-430
//   float16_t::from_float (truncating)   third_party/sqlite-vec-cpp/.../utils/float16.hpp:20-40
//
// Pipeline (DESIGN.md §scan):
//   stage 1  approximate fp32/fp16 scores of every row against every query (GEMM-shaped; this file
//            holds the CUDA-core engine, knn_umma.cu the wgmma engine) with a fused per-query
//            threshold filter -> short candidate lists; thresholds come from a strided row sample;
//   select   exact top-K' (K' = k + slack) of each candidate list (radix select + bitonic sort);
//   stage 2  the K' survivors are re-scored exactly like the reference (sequential double
//            accumulation, skip rules, float cast) -> scores are bit-identical to the CPU path;
//   final    order by (similarity desc, rowid asc), apply the threshold, keep k, flag ties at k.
#include <cuda_fp16.h>
#include <math.h>

#include <algorithm>
#include <memory>
#include <new>
#include <vector>

#include "cosine.cuh"
#include "knn.cuh"
#include "ref_order.cuh"

namespace yb {

// ---------------------------------------------------------------------------------------------------
// element helpers (load_elem: cosine.cuh)
// ---------------------------------------------------------------------------------------------------

// reference truncating fp32 -> fp16 (utils/float16.hpp:20-40), restated on integer bits
__host__ __device__ __forceinline__ uint16_t f16_from_float_trunc(float f) {
    uint32_t x;
#if defined(__CUDA_ARCH__)
    x = __float_as_uint(f);
#else
    memcpy(&x, &f, 4);
#endif
    uint32_t sign = (x >> 16) & 0x8000u;
    int32_t e = (int32_t)((x >> 23) & 0xFFu) - 127 + 15;
    uint32_t m = x & 0x7FFFFFu;
    if (e <= 0) {
        if (e < -10) return (uint16_t)sign;
        m = (m | 0x800000u) >> (1 - e);
        return (uint16_t)(sign | (m >> 13));
    }
    if (e >= 31) return (uint16_t)(sign | 0x7C00u);
    return (uint16_t)(sign | ((uint32_t)e << 10) | (m >> 13));
}

__global__ void convert_f32_to_f16_trunc_kernel(const float* __restrict__ in, uint16_t* __restrict__ out, uint64_t n) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        out[i] = f16_from_float_trunc(in[i]);
}

// SURVEY.md §8d generator: x = (splitmix64(seed ^ (row*d + c)) >> 40) * 2^-23 - 1
__device__ __forceinline__ float synth_value(uint64_t seed, uint64_t row, uint32_t d, uint32_t c) {
    uint64_t u = splitmix64(seed ^ (row * (uint64_t)d + (uint64_t)c));
    return (float)(u >> 40) * 1.1920928955078125e-07f - 1.0f;
}

// one thread per row: sequential double sum of squares (bit-identical to oracle yo_gen_rows_f32)
__global__ void synth_rownorm_kernel(uint64_t seed, uint64_t first_row, uint64_t n, uint32_t d, float* __restrict__ inv) {
    uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    double ss = 0.0;
    for (uint32_t c = 0; c < d; ++c) {
        float x = synth_value(seed, first_row + r, d, c);
        ss += (double)x * (double)x;
    }
    inv[r] = ss > 0.0 ? (float)(1.0 / sqrt(ss)) : 0.0f;
}

__global__ void synth_fill_kernel(uint64_t seed, uint64_t first_row, uint64_t n, uint32_t d, const float* __restrict__ inv,
                                  void* __restrict__ out, int dtype) {
    uint64_t total = n * (uint64_t)d;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t r = i / d;
        uint32_t c = (uint32_t)(i - r * d);
        float v = synth_value(seed, first_row + r, d, c) * inv[r];
        if (dtype == YAMS_B200_F16) reinterpret_cast<uint16_t*>(out)[i] = f16_from_float_trunc(v);
        else reinterpret_cast<float*>(out)[i] = v;
    }
}

// nonnegative floats order like their bit patterns: atomic max through the integer view
__device__ __forceinline__ void atomic_max_nonneg(float* addr, float v) {
    if (v == v) atomicMax(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
}

// per-row validity + 1/|row| exactly as the reference evaluates it (sqlite_vec_backend.cpp:4253-4269):
// sequential double accumulation; rows with a non-finite element or |row|^2 <= min_sq get 0 -- min_sq = 1e-12 for the search,
// 0 for the semantic graph (EmbeddingService.cpp:405-415), whose 1/|row| overflows to +inf below |row|^2 = 2^-256.
// L2 corpora (vec0 surface, no skip rules) keep |row|^2 in the same slot instead: stage 1 ranks by 2 q.r - |row|^2.
// stats[0] = max |row|, stats[1] = max |row - tf32(row)| (fp32 corpora read by the tf32 tensor-core engine),
// stats[2] = max of that residual relative to |row|, stats[3] = max 1/|row| of the rows cosine scores: the inputs of the
// stage-1 error bound (DESIGN.md §4.2)
__global__ void row_stats_kernel(const void* __restrict__ rows, int dtype, uint32_t d, uint64_t first, uint64_t n,
                                 float* __restrict__ inv_norm, int metric, float* __restrict__ stats, double min_sq) {
    uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    double ss = 0.0, res = 0.0;
    bool finite = true;
    walk_row(rows, dtype, d, first + r, [&](float v) {
        if (!isfinite(v)) finite = false;
        ss += (double)v * v;
        if (dtype == YAMS_B200_F32) {
            float t = v - __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
            res += (double)t * t;
        }
    });
    if (metric == YAMS_B200_L2) inv_norm[first + r] = finite ? (float)ss : INFINITY;
    else inv_norm[first + r] = (finite && ss > min_sq) ? (float)(1.0 / sqrt(ss)) : 0.0f;
    if (finite && ss > 0.0) {
        float nrm = (float)sqrt(ss), rs = (float)sqrt(res);
        atomic_max_nonneg(&stats[0], nrm * 1.0000002f);
        atomic_max_nonneg(&stats[1], rs * 1.0000002f);
        if (ss > min_sq) {
            atomic_max_nonneg(&stats[2], (rs / nrm) * 1.0000002f);
            atomic_max_nonneg(&stats[3], (float)(1.0 / sqrt(ss)) * 1.0000002f);
        }
    }
}

// Device-side status of one search call (read by the host once, after everything is enqueued)
struct ScanStatus {
    uint32_t n_invalid;   // queries the reference rejects (non-finite or zero norm, sqlite_vec_backend.cpp:4127-4130)
    uint32_t n_bad;       // queries whose fast-path result could not be certified exact -> resolved by the exhaustive levels
    uint32_t n_bad2;      // ... of which level 1 could not certify either -> full exact pass
    uint32_t pad;
    // followed by uint32_t bad[nq], bad2[nq]
};

// queries: invalid if non-finite or (cosine) |q|^2 < 1e-10 (sqlite_vec_backend.cpp:204-235,4127);
// qnorm[q] = sqrt(sum (double)q^2) (:4204-4209), qinv[q] = 1/qnorm as float (1 for L2: queries stay unscaled)
constexpr int QP_THREADS = 32;
__global__ void __launch_bounds__(QP_THREADS) query_prep_kernel(const float* __restrict__ q, uint32_t nq, uint32_t d, double* __restrict__ qnorm,
                                                                float* __restrict__ qinv, int metric, ScanStatus* __restrict__ status) {
    // thread = query, the reference's sequential double sum (sqlite_vec_backend.cpp:4140-4150).  The walk keeps four 16-byte
    // loads in flight (one 4-byte load per dependent trip cost 64 us for 1024 x 768 queries).
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    double ss = 0.0;
    bool finite = true;
    walk_row<4>(q, YAMS_B200_F32, d, i, [&](float v) {
        if (!isfinite(v)) finite = false;
        ss += (double)v * v;
    });
    bool bad = !finite || (metric == YAMS_B200_COSINE && ss < 1e-10);
    if (bad) atomicAdd(&status->n_invalid, 1u);
    double nrm = sqrt(ss);
    qnorm[i] = nrm;
    qinv[i] = metric == YAMS_B200_L2 ? 1.0f : (bad ? 0.0f : (float)(1.0 / nrm));
}

// error bound of the CUDA-core engine's stage-1 score (fp32 FMA chain over d products, Cauchy-Schwarz on sum |q_i r_i|;
// the float roundings of 1/|row|, 1/|q| or |row|^2 are covered by the +4):
//   cosine: |s~ - s| <= 2^-24 (d + 4);   L2 (s = 2 q.r - |r|^2): <= 2^-23 (d + 4) |q| Rmax + 2^-22 Rmax^2
__global__ void eps_cc_kernel(const double* __restrict__ qnorm, uint32_t nq, uint32_t d, int metric, float r_max,
                              float* __restrict__ eps, int keep_larger) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq) return;
    const float u = 5.9604645e-08f;   // 2^-24
    float e;
    if (metric == YAMS_B200_L2) e = 2.f * u * (float)(d + 4) * (float)qnorm[i] * r_max + 4.f * u * r_max * r_max + 1e-30f;
    else e = u * (float)(d + 4) + 1e-7f;
    eps[i] = keep_larger ? fmaxf(eps[i], e) : e;
}

// ---------------------------------------------------------------------------------------------------
// stage 1, CUDA-core engine: tiled fp32 GEMM [rows x dim] x [dim x queries] with fused epilogue
// ---------------------------------------------------------------------------------------------------
constexpr int CC_BM = 128, CC_BN = 64, CC_BK = 32, CC_THREADS = 256;
constexpr int CC_AS = CC_BM + 1;  // padded k-major A tile: conflict-free transposed stores

template <bool FILTER>
__global__ void __launch_bounds__(CC_THREADS, 2) stage1_cc_kernel(Stage1Args a, uint32_t nqt) {
    __shared__ float As[CC_BK][CC_AS];
    __shared__ __align__(16) float Bs[CC_BK][CC_BN];
    const uint32_t qt = blockIdx.x % nqt;
    const uint64_t rt = blockIdx.x / nqt;
    const uint64_t row0 = rt * CC_BM;   // tile-local row index base (within this launch)
    const uint32_t q0 = qt * CC_BN;
    const int tid = threadIdx.x;
    const int ty = tid >> 4, tx = tid & 15;
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    const bool vec_ok = a.dtype == YAMS_B200_F16 ? (a.dim % 8 == 0) : (a.dim % 4 == 0);
    for (uint32_t k0 = 0; k0 < a.dim; k0 += CC_BK) {
        // ---- A tile: CC_BM rows x CC_BK k, transposed into As[k][m] ----
        if (a.dtype == YAMS_B200_F16) {
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                int idx = tid + CC_THREADS * j;  // 512 segments of 8 halves
                int m = idx >> 2, seg = idx & 3;
                uint64_t li = row0 + m;
                uint32_t kk = k0 + seg * 8;
                float v[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) v[e] = 0.f;
                if (li < a.nrows) {
                    uint64_t grow = a.row_start + li * a.row_stride;
                    const __half* src = reinterpret_cast<const __half*>(a.rows) + grow * a.dim + kk;
                    if (vec_ok && kk + 8 <= a.dim) {
                        uint4 raw = *reinterpret_cast<const uint4*>(src);
                        const __half2* h2 = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            float2 f = __half22float2(h2[e]);
                            v[2 * e] = f.x;
                            v[2 * e + 1] = f.y;
                        }
                    } else {
#pragma unroll
                        for (int e = 0; e < 8; ++e)
                            if (kk + e < a.dim) v[e] = __half2float(src[e]);
                    }
                }
#pragma unroll
                for (int e = 0; e < 8; ++e) As[seg * 8 + e][m] = v[e];
            }
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                int idx = tid + CC_THREADS * j;  // 1024 segments of 4 floats
                int m = idx >> 3, seg = idx & 7;
                uint64_t li = row0 + m;
                uint32_t kk = k0 + seg * 4;
                float v[4] = {0.f, 0.f, 0.f, 0.f};
                if (li < a.nrows) {
                    uint64_t grow = a.row_start + li * a.row_stride;
                    const float* src = reinterpret_cast<const float*>(a.rows) + grow * a.dim + kk;
                    if (vec_ok && kk + 4 <= a.dim) {
                        float4 f = *reinterpret_cast<const float4*>(src);
                        v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
                    } else {
#pragma unroll
                        for (int e = 0; e < 4; ++e)
                            if (kk + e < a.dim) v[e] = src[e];
                    }
                }
#pragma unroll
                for (int e = 0; e < 4; ++e) As[seg * 4 + e][m] = v[e];
            }
        }
        // ---- B tile: CC_BK k x CC_BN queries (queries are row-major [q][dim]) ----
#pragma unroll
        for (int j = 0; j < (CC_BK * CC_BN) / CC_THREADS; ++j) {
            int idx = tid + CC_THREADS * j;
            int kk = idx & (CC_BK - 1), qn = idx / CC_BK;
            uint32_t q = q0 + qn, k = k0 + kk;
            Bs[kk][qn] = (q < a.nq && k < a.dim) ? a.q32[(uint64_t)q * a.dim + k] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < CC_BK; ++kk) {
            float av[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) av[i] = As[kk][ty * 8 + i];
            float4 b4 = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
            float bv[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }
    // ---- epilogue ----
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        uint64_t li = row0 + ty * 8 + i;
        if (li >= a.nrows) continue;
        uint64_t grow = a.row_start + li * a.row_stride;
        float inr = a.inv_norm[grow];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            uint32_t q = q0 + tx * 4 + j;
            if (q >= a.nq) continue;
            float s;
            // L2: 2 q.r - |r|^2 (slot holds |r|^2; +inf marks a non-finite row, whose dot product may be NaN)
            if (a.metric == YAMS_B200_L2) s = inr < INFINITY ? fmaf(2.f, acc[i][j], -inr) : -INFINITY;
            else s = inr > 0.f ? acc[i][j] * inr * a.qinv[q] : -INFINITY;
            if (FILTER) {
                bool pass = s > a.tau[q];
                if (pass && a.mask) pass = (a.mask[(uint64_t)q * a.mask_ld + (grow >> 5)] >> (grow & 31)) & 1u;
                if (pass) {
                    uint32_t pos = atomicAdd(&a.counts[q], 1u);
                    if (pos < a.cap) {
                        Cand c;
                        c.score = s;
                        c.row = (uint32_t)grow;
                        a.cands[(uint64_t)q * a.cap + pos] = c;
                    }
                }
            } else {
                a.out_scores[(uint64_t)q * a.ld + li] = s;
            }
        }
    }
}

yams_status_t stage1_cuda_core(const Stage1Args& a, bool filter, cudaStream_t st) {
    if (a.nrows == 0 || a.nq == 0) return YAMS_OK;
    uint32_t nqt = (a.nq + CC_BN - 1) / CC_BN;
    uint64_t nrt = (a.nrows + CC_BM - 1) / CC_BM;
    uint64_t grid = nrt * nqt;
    YB_ARG(grid < (1ull << 31), "scan too large for one launch");
    if (filter) stage1_cc_kernel<true><<<(unsigned)grid, CC_THREADS, 0, st>>>(a, nqt);
    else stage1_cc_kernel<false><<<(unsigned)grid, CC_THREADS, 0, st>>>(a, nqt);
    YB_CUDA(cudaGetLastError());
    return YAMS_OK;
}

// ---------------------------------------------------------------------------------------------------
// top-K selection (one CTA per query): radix select on monotone keys, gather, bitonic sort
// ---------------------------------------------------------------------------------------------------
// fkey / fkey_inv: cosine.cuh
constexpr int SEL_THREADS = 256;
constexpr int SEL_MAXK = 4096;       // survivors per query the select / final kernels can order in shared memory
static_assert(TOPK_MAX == SEL_MAXK, "launch_topk_dense takes K <= TOPK_MAX");

struct SelectIn {
    const float* dense;     // mode dense: scores[q * ld + i], row = row_start + i * row_stride
    uint64_t ld;
    uint64_t row_start, row_stride;
    uint64_t dense_len;
    const Cand* cands;      // mode list: cands[q * cap + i], length min(counts[q], cap)
    const uint32_t* counts;
    uint32_t cap;
    const uint32_t* qmap;   // nullable: CTA b handles query qmap[b] for the list/out side
    const float* tau;       // nullable (list mode): rows that never reached the list scored <= tau[q]
    float tau_margin;       // tau_only: subtracted from the selected score
    int fast_tau;           // tau_only, K <= 16: one pass, the K-th largest of the per-thread maxima (a lower bound of the K-th
                            // largest score: a threshold need not be exact, only close -- the certificate covers what it lets go)
};

__device__ __forceinline__ uint64_t sel_key(const SelectIn& in, uint32_t qsrc, uint64_t i) {
    float s;
    uint32_t row;
    if (in.dense) {
        s = in.dense[(uint64_t)qsrc * in.ld + i];
        row = (uint32_t)(in.row_start + i * in.row_stride);
    } else {
        Cand c = in.cands[(uint64_t)qsrc * in.cap + i];
        s = c.score;
        row = c.row;
    }
    // score_key (cosine.cuh) written out on purpose: through score_key, topk_select_kernel compiles to different machine code
    // (4960 -> 5120 SASS instructions, nvcc 12.9, sm_90a); with this line as it is, the kernel's code is unchanged
    return ((uint64_t)fkey(s) << 32) | (uint64_t)(0xFFFFFFFFu - row);
}

// tau_only: writes the K-th largest score to out_tau[q] (-inf when fewer than K items)
// else    : writes the top-K (sorted desc; ties -> smaller row first) to out_sel[b*K ..], count to out_n[b], and
//           out_bound[b] = an upper bound of the stage-1 score of every row that was NOT selected (the input of the
//           exactness certificate in final_kernel): the K-th selected score when the list was longer than K, else the
//           list threshold tau (rows that never reached the list), -inf when no other row exists, +inf when the list
//           overflowed its capacity (unknown rows were dropped)
__global__ void __launch_bounds__(SEL_THREADS) topk_select_kernel(SelectIn in, uint32_t K, int tau_only, float* __restrict__ out_tau,
                                                                  Cand* __restrict__ out_sel, uint32_t* __restrict__ out_n,
                                                                  float* __restrict__ out_bound) {
    __shared__ uint32_t hist[256];
    __shared__ uint64_t s_prefix;
    __shared__ uint32_t s_want;
    __shared__ uint32_t s_cnt;
    __shared__ uint64_t buf[SEL_MAXK];
    const uint32_t b = blockIdx.x;
    const uint32_t qdst = in.qmap ? in.qmap[b] : b;   // tau_only output slot / list-side query
    const uint32_t qsrc = in.dense ? b : qdst;
    uint64_t L = in.dense ? in.dense_len : (uint64_t)min(in.counts[qsrc], in.cap);
    // radix select of the K-th largest key among L > K items; result in s_prefix
    auto radix_select = [&](int npass) {
        if (threadIdx.x == 0) { s_prefix = 0; s_want = K; }
        __syncthreads();
        for (int p = 0; p < npass; ++p) {
            const int shift = 56 - 8 * p;
            for (int i = threadIdx.x; i < 256; i += SEL_THREADS) hist[i] = 0;
            __syncthreads();
            const uint64_t prefix = s_prefix;
            for (uint64_t i = threadIdx.x; i < L; i += SEL_THREADS) {
                uint64_t key = sel_key(in, qsrc, i);
                if (p == 0 || (key >> (shift + 8)) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                uint32_t want = s_want, cum = 0;
                int bsel = 0;
                for (int bk = 255; bk >= 0; --bk) {
                    uint32_t h = hist[bk];
                    if (cum + h >= want) { bsel = bk; break; }
                    cum += h;
                }
                s_want = want - cum;
                s_prefix = (prefix << 8) | (uint64_t)bsel;
            }
            __syncthreads();
        }
    };
    if (tau_only) {
        if (L < K || K == 0) {
            if (threadIdx.x == 0) out_tau[qdst] = -INFINITY;
        } else if (L == K) {
            if (threadIdx.x == 0) s_want = 0xFFFFFFFFu;
            __syncthreads();
            uint32_t mn = 0xFFFFFFFFu;
            for (uint64_t i = threadIdx.x; i < L; i += SEL_THREADS) mn = min(mn, (uint32_t)(sel_key(in, qsrc, i) >> 32));
            atomicMin(&s_want, mn);
            __syncthreads();
            if (threadIdx.x == 0) out_tau[qdst] = fkey_inv(s_want) - in.tau_margin;
        } else if (in.fast_tau && K <= 16 && L >= 16 * SEL_THREADS) {
            // One pass, no atomics: every thread keeps the best key of its strided share, the 256 maxima are sorted, the K-th of
            // them is the threshold.  It equals the K-th best score unless two of the top K fall into one thread's share (11 % for
            // K = 8), in which case it is the next one down: a slightly lower threshold, a few more survivors.
            uint32_t* arr = reinterpret_cast<uint32_t*>(buf);
            uint32_t mx = 0;
            const float* base = in.dense ? in.dense + (uint64_t)qsrc * in.ld : nullptr;
            if (base && (reinterpret_cast<uintptr_t>(base) & 15u) == 0) {
                // dense scores: 16-byte loads, four of them in flight per thread (one 4-byte load per trip was latency-bound:
                // 1.2 TB/s over the Q x S score matrix)
                const float4* b4 = reinterpret_cast<const float4*>(base);
                const uint64_t n4 = L / 4;
                uint64_t i = threadIdx.x;
                for (; i + 3 * SEL_THREADS < n4; i += 4 * SEL_THREADS) {
                    const float4 v0 = b4[i], v1 = b4[i + SEL_THREADS], v2 = b4[i + 2 * SEL_THREADS], v3 = b4[i + 3 * SEL_THREADS];
                    mx = max(mx, max(max(fkey(v0.x), fkey(v0.y)), max(fkey(v0.z), fkey(v0.w))));
                    mx = max(mx, max(max(fkey(v1.x), fkey(v1.y)), max(fkey(v1.z), fkey(v1.w))));
                    mx = max(mx, max(max(fkey(v2.x), fkey(v2.y)), max(fkey(v2.z), fkey(v2.w))));
                    mx = max(mx, max(max(fkey(v3.x), fkey(v3.y)), max(fkey(v3.z), fkey(v3.w))));
                }
                for (; i < n4; i += SEL_THREADS) {
                    const float4 v = b4[i];
                    mx = max(mx, max(max(fkey(v.x), fkey(v.y)), max(fkey(v.z), fkey(v.w))));
                }
                for (uint64_t j = n4 * 4 + threadIdx.x; j < L; j += SEL_THREADS) mx = max(mx, fkey(base[j]));
            } else {
                for (uint64_t i = threadIdx.x; i < L; i += SEL_THREADS) mx = max(mx, (uint32_t)(sel_key(in, qsrc, i) >> 32));
            }
            arr[threadIdx.x] = mx;
            __syncthreads();
            // block_sort_desc written out on purpose: as block_sort_desc<SEL_THREADS>(arr, SEL_THREADS) this kernel ran 33.0 -> 35.9 us
            // per call (H100 80GB HBM3, 700 W, nvcc 12.9)
            for (uint32_t size = 2; size <= SEL_THREADS; size <<= 1) {
                for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
                    const uint32_t t = threadIdx.x;
                    if (t < SEL_THREADS / 2) {
                        uint32_t lo = (t / stride) * (stride * 2) + (t % stride), hi = lo + stride;
                        bool desc = ((lo & size) == 0);
                        uint32_t x = arr[lo], y = arr[hi];
                        if ((x < y) == desc) { arr[lo] = y; arr[hi] = x; }
                    }
                    __syncthreads();
                }
            }
            if (threadIdx.x == 0) out_tau[qdst] = fkey_inv(arr[K - 1]) - in.tau_margin;
        } else {
            // Two passes instead of four: a 4096-bin histogram of the top 12 key bits locates the bin that holds the K-th
            // best score; its (few) members are collected and sorted in shared memory.  A crowded bin (> 2048 members,
            // e.g. constant scores) falls back to the plain 4-pass radix select.
            uint32_t* h12 = reinterpret_cast<uint32_t*>(buf);            // [4096] counters
            uint32_t* members = h12 + 4096;                               // [4096] score keys of the boundary bin
            for (int i = threadIdx.x; i < 4096; i += SEL_THREADS) h12[i] = 0;
            __syncthreads();
            for (uint64_t i = threadIdx.x; i < L; i += SEL_THREADS) atomicAdd(&h12[(uint32_t)(sel_key(in, qsrc, i) >> 52)], 1u);
            __syncthreads();
            if (threadIdx.x == 0) {
                uint32_t cum = 0;
                int bsel = 0;
                for (int bk = 4095; bk >= 0; --bk) {
                    uint32_t h = h12[bk];
                    if (cum + h >= K) { bsel = bk; break; }
                    cum += h;
                }
                s_want = K - cum;               // rank inside the boundary bin (1-based)
                s_prefix = (uint64_t)bsel;
                s_cnt = 0;
            }
            __syncthreads();
            const uint32_t bsel = (uint32_t)s_prefix, pop = h12[bsel];
            if (pop <= 2048) {
                const uint32_t np2 = pow2_at_least(pop);
                __syncthreads();
                for (uint32_t i = threadIdx.x; i < np2; i += SEL_THREADS) members[i] = 0;
                __syncthreads();
                for (uint64_t i = threadIdx.x; i < L; i += SEL_THREADS) {
                    uint32_t fk = (uint32_t)(sel_key(in, qsrc, i) >> 32);
                    if ((fk >> 20) == bsel) members[atomicAdd(&s_cnt, 1u)] = fk;
                }
                __syncthreads();
                block_sort_desc<SEL_THREADS>(members, np2);
                if (threadIdx.x == 0) out_tau[qdst] = fkey_inv(members[s_want - 1]) - in.tau_margin;
            } else {
                __syncthreads();
                radix_select(4);
                if (threadIdx.x == 0) out_tau[qdst] = fkey_inv((uint32_t)s_prefix) - in.tau_margin;
            }
        }
        return;
    }
    uint64_t kth = 0;  // keys >= kth are selected
    constexpr int KPT = SEL_MAXK / SEL_THREADS;   // 16 keys per thread
    if (L <= SEL_MAXK) {
        // The normal case (a candidate list of 1-3 k entries): the keys are read ONCE into registers and the K-th largest is found
        // bit by bit from the top -- 64 block-wide counts (compare, warp reduce, one barrier each), ~8 k cycles, where eight
        // histogram passes over the list or a 4096-key sorting network cost 150-300 us per 1024 queries.
        uint64_t kreg[KPT];
#pragma unroll
        for (int j = 0; j < KPT; ++j) {
            const uint64_t i = (uint64_t)threadIdx.x + (uint64_t)j * SEL_THREADS;
            kreg[j] = i < L ? sel_key(in, qsrc, i) : 0ull;          // 0 is no key (a real key carries 0xFFFFFFFF - row != 0 below)
        }
        if (L > K && K > 0) {
            // Block-wide helpers over 8 warps: one barrier per call, partials double-buffered by `slot`.
            uint32_t* part = reinterpret_cast<uint32_t*>(hist);      // [4][8]
            int slot = 0;
            auto block_sum = [&](uint32_t v) {
                const uint32_t w = __reduce_add_sync(0xffffffffu, v);
                uint32_t* pb = part + (slot & 3) * 8;
                ++slot;
                if ((threadIdx.x & 31) == 0) pb[threadIdx.x >> 5] = w;
                __syncthreads();
                uint32_t t = 0;
#pragma unroll
                for (int x = 0; x < SEL_THREADS / 32; ++x) t += pb[x];
                return t;
            };
            // score words first (32-bit compares); the bits every valid key shares are skipped
            uint32_t a_and = 0xFFFFFFFFu, a_or = 0u;
#pragma unroll
            for (int j = 0; j < KPT; ++j)
                if (kreg[j] != 0ull) { a_and &= (uint32_t)(kreg[j] >> 32); a_or |= (uint32_t)(kreg[j] >> 32); }
            {
                const uint32_t wa = __reduce_and_sync(0xffffffffu, a_and), wo = __reduce_or_sync(0xffffffffu, a_or);
                uint32_t* pb = part + 16;                              // slots 2,3 of the table: [8] ands, [8] ors
                if ((threadIdx.x & 31) == 0) { pb[threadIdx.x >> 5] = wa; pb[8 + (threadIdx.x >> 5)] = wo; }
                __syncthreads();
                a_and = 0xFFFFFFFFu; a_or = 0u;
#pragma unroll
                for (int x = 0; x < SEL_THREADS / 32; ++x) { a_and &= pb[x]; a_or |= pb[8 + x]; }
                __syncthreads();                                       // the table is reused by block_sum below
            }
            const uint32_t diff = a_and ^ a_or;
            uint32_t want = K;
            uint32_t shi = a_or;                                       // all scores equal: that score
            if (diff) {
                const int top = 31 - __clz(diff);
                shi = top == 31 ? 0u : (a_or & ~((2u << top) - 1u));   // the shared leading bits
                for (int bit = top; bit >= 0; --bit) {
                    const uint32_t cand = shi | (1u << bit);
                    const uint32_t himask = ~((1u << bit) - 1u);
                    uint32_t c = 0;
#pragma unroll
                    for (int j = 0; j < KPT; ++j) c += (kreg[j] != 0ull && ((uint32_t)(kreg[j] >> 32) & himask) == cand) ? 1u : 0u;
                    const uint32_t tot = block_sum(c);
                    if (tot >= want) shi = cand; else want -= tot;    // block-uniform
                }
            }
            // `want` of the keys whose score word equals shi are needed (those with the largest low words, i.e. the smallest rows)
            uint32_t g = 0;
#pragma unroll
            for (int j = 0; j < KPT; ++j) g += (kreg[j] != 0ull && (uint32_t)(kreg[j] >> 32) == shi) ? 1u : 0u;
            const uint32_t group = block_sum(g);
            uint32_t slo = 0;                                          // group == want: the whole group is selected
            if (group > want) {                                        // equal scores straddle the K-th place: resolve by the low words
                for (int bit = 31; bit >= 0; --bit) {
                    const uint32_t cand = slo | (1u << bit);
                    const uint32_t lomask = ~((1u << bit) - 1u);
                    uint32_t c = 0;
#pragma unroll
                    for (int j = 0; j < KPT; ++j)
                        c += (kreg[j] != 0ull && (uint32_t)(kreg[j] >> 32) == shi && ((uint32_t)kreg[j] & lomask) == cand) ? 1u : 0u;
                    const uint32_t tot = block_sum(c);
                    if (tot >= want) slo = cand; else want -= tot;
                }
            }
            kth = ((uint64_t)shi << 32) | (uint64_t)slo;
        }
        if (threadIdx.x == 0) s_cnt = 0;
        for (int i = threadIdx.x; i < SEL_MAXK; i += SEL_THREADS) buf[i] = 0;
        __syncthreads();
#pragma unroll
        for (int j = 0; j < KPT; ++j) {
            if (kreg[j] != 0ull && kreg[j] >= kth) {
                uint32_t pos = atomicAdd(&s_cnt, 1u);
                if (pos < SEL_MAXK) buf[pos] = kreg[j];
            }
        }
        __syncthreads();
    } else {
    if (L > K) {
        radix_select(8);
        kth = s_prefix;
    }
    if (threadIdx.x == 0) s_cnt = 0;
    for (int i = threadIdx.x; i < SEL_MAXK; i += SEL_THREADS) buf[i] = 0;
    __syncthreads();
    for (uint64_t i = threadIdx.x; i < L; i += SEL_THREADS) {
        uint64_t key = sel_key(in, qsrc, i);
        if (key >= kth) {
            uint32_t pos = atomicAdd(&s_cnt, 1u);
            if (pos < SEL_MAXK) buf[pos] = key;
        }
    }
    __syncthreads();
    }
    uint32_t cnt = min(s_cnt, (uint32_t)SEL_MAXK);
    block_sort_desc<SEL_THREADS>(buf, pow2_at_least(cnt));
    uint32_t nout = min(cnt, K);
    for (uint32_t i = threadIdx.x; i < nout; i += SEL_THREADS) {
        uint64_t key = buf[i];
        Cand c;
        c.score = key_score(key);
        c.row = key_row(key);
        out_sel[(uint64_t)b * K + i] = c;
    }
    if (threadIdx.x == 0) {
        out_n[b] = nout;
        if (out_bound) {
            float bd;
            if (!in.dense && in.counts[qsrc] > in.cap) bd = INFINITY;
            else if (L > K && K > 0) bd = key_score(buf[K - 1]);
            else if (L > K) bd = INFINITY;
            else bd = (!in.dense && in.tau) ? in.tau[qsrc] : -INFINITY;
            out_bound[b] = bd;
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// stage 2: exact re-scoring + final ordering
// ---------------------------------------------------------------------------------------------------
// one thread per (query, survivor).
// cosine: sqlite_vec_backend.cpp:4253-4279 evaluated in the same order (sequential double accumulation, skip rules, float cast)
// L2    : distances::l2_distance<float> as the reference BUILD evaluates it (YAMS compiles sqlite-vec-cpp with AVX,
//         src/vector/meson.build:79-87): dim >= 16 && dim % 16 == 0 -> simd/avx.hpp:20-66 (eight lane-strided float partial
//         sums, separate multiply and add, lanes summed left to right), else the scalar loop l2.hpp:108-118; sim = -dist.
// Entry b of sel/out belongs to query qmap[b] (or b).
// Semantic graph (graph.inv non-null): the graph's score (semantic_sim) of the rows it takes, the source's own row skipped, and
// -0.0 stored as +0.0 so that the two zeros order as one score (restore_zero_signs_kernel gives the results their sign back).
__global__ void rescore_kernel(const void* __restrict__ rows, int dtype, uint32_t d, const float* __restrict__ q32,
                               const double* __restrict__ qnorm, const Cand* __restrict__ sel, const uint32_t* __restrict__ sel_n,
                               uint32_t Kp, uint32_t nq, float threshold, Exact* __restrict__ out, int metric,
                               const uint32_t* __restrict__ qmap, const uint32_t* __restrict__ mask, uint64_t mask_ld, GraphRows graph) {
    uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (uint64_t)nq * Kp) return;
    uint32_t b = (uint32_t)(t / Kp), j = (uint32_t)(t % Kp);
    const uint32_t q = qmap ? qmap[b] : b;
    Exact e;
    e.sim = __int_as_float(0x7FC00000);
    e.row = 0xFFFFFFFFu;
    bool take = j < sel_n[b] && sel[(uint64_t)b * Kp + j].row != 0xFFFFFFFFu;
    if (take && mask) {   // candidate-set mode: a row outside the allowed set is never a result
        uint32_t row = sel[(uint64_t)b * Kp + j].row;
        take = (mask[(uint64_t)q * mask_ld + (row >> 5)] >> (row & 31)) & 1u;
    }
    if (take) {
        uint32_t row = sel[(uint64_t)b * Kp + j].row;
        uint64_t base = (uint64_t)row * d;
        const float* qv = q32 + (uint64_t)q * d;
        if (graph.inv) {
            const float inv_n = graph.inv[row];
            float sim;
            if (inv_n > 0.f && row != graph.src_row[q] &&
                semantic_sim(rows, dtype, d, row, qv, graph.inv[graph.src_row[q]], inv_n, threshold, &sim)) {
                e.sim = sim == 0.f ? 0.f : sim;
                e.row = row;
            }
        } else if (metric == YAMS_B200_L2) {
            auto row_at = [&](uint32_t c) { return load_elem(rows, dtype, base + c); };
            auto q_at = [&](uint32_t c) { return qv[c]; };
            float dist = ref_l2_distance(q_at, row_at, d);
            if (dist == dist) {
                e.sim = -dist;
                e.row = row;
            }
        } else {
            float sim;
            if (exact_cosine_sim(rows, dtype, d, row, qv, qnorm[q], threshold, &sim)) {
                e.sim = sim;
                e.row = row;
            }
        }
    }
    out[(uint64_t)b * Kp + j] = e;
}

// semantic graph: a batch's sources as the queries of the scan.  q32[q] = corpus row src_row[q] (fp16 widened exactly),
// qinv[q] = its graph scale; the search's query preparation (norms, validity) does not run.
__global__ void gather_sources_kernel(const void* __restrict__ rows, int dtype, uint32_t d, GraphRows graph, uint32_t nq,
                                      float* __restrict__ q32, float* __restrict__ qinv) {
    const uint64_t total = (uint64_t)nq * d;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t q = (uint32_t)(i / d), c = (uint32_t)(i - (uint64_t)q * d);
        const uint32_t row = graph.src_row[q];
        q32[i] = load_elem(rows, dtype, (uint64_t)row * d + c);
        if (c == 0) qinv[q] = graph.inv[row];
    }
}

// semantic graph: the results of a batch with similarity 0 are re-scored to give them their sign (rescore_kernel orders -0.0 as
// +0.0).  Only a call with threshold <= 0 can return a zero.
__global__ void restore_zero_signs_kernel(const void* __restrict__ rows, int dtype, uint32_t d, const float* __restrict__ q32,
                                          GraphRows graph, const int64_t* __restrict__ rowids, uint64_t n, DeviceResults out,
                                          uint32_t nq, uint32_t k) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (uint64_t)nq * k || out.rowids[t] < 0 || out.scores[t] != 0.f) return;
    const uint32_t q = (uint32_t)(t / k);
    const uint32_t row = (uint32_t)find_row(rowids, n, out.rowids[t]);
    float sim;
    if (semantic_sim(rows, dtype, d, row, q32 + (uint64_t)q * d, graph.inv[graph.src_row[q]], graph.inv[row], -INFINITY, &sim))
        out.scores[t] = sim;
}

// The semantic graph's certificate adds to eps[q] (DESIGN.md §4.9)
//   * the exact score's own rounding: it is float((dot inv_s) inv_n) with the same float scales stage 1 multiplies by, so
//     only the float cast (2^-24 |v|, |v| <= (1 + 2^-23)^2), the double products and the double sum (below 2^-32 for
//     d < 2^20) remain -- at most 2^-23;
//   * underflow: an fp32 product or partial sum below 2^-126 may be flushed or rounded to the subnormal grid, an absolute error
//     eps's relative terms do not cover.  Each of the d + 4 steps loses at most 2^-126 of the dot product of the engine's
//     operands (the raw source on the CUDA-core engine, the source scaled by 1/|s| on the wgmma engine), which the scales then
//     multiply by at most max(1/|s|, 1) * max 1/|r|: uf = (d + 4) 2^-126 max 1/|r| per unit of max(inv_s, 1).  It is negligible
//     unless rows or sources have norms below ~1e-30, and +inf (nothing certified, the exhaustive levels answer) when a
//     scale overflowed.
constexpr float kGraphEps = 1.1920929e-07f;
__host__ __device__ inline float graph_eps(float inv_s, float uf) { return kGraphEps + uf * fmaxf(inv_s, 1.f); }

// The exactness certificate (DESIGN.md §4.2).  Stage 1 ranks rows by an approximate score s~ with |s~ - s| <= eps[q];
// only the top-K' by s~ are re-scored exactly.  Every row that was NOT re-scored has s~ <= bound (topk_select_kernel), hence
// a true score <= bound + eps.  The emitted top-k is provably the reference's top-k iff no such row can reach the k-th exact
// score (or, with fewer than k valid survivors, the caller's threshold):
//   cosine:  bound + eps <  (valid >= k ? sim_k : threshold)
//   L2    :  |q|^2 - bound - eps > dist_k^2          (s~ = 2 q.r - |r|^2, so d^2 = |q|^2 - s)
// Otherwise the query is queued for the exhaustive levels (status->bad / bad2) and flagged.
struct CertArgs {
    const float* bound;       // per CTA
    const float* eps;         // per query
    const double* qnorm;      // per query (L2)
    float threshold;
    int metric;
    double l2_margin;         // L2: dist_k^2 factor covering the float rounding of the reference's distances (l2_cert_margin)
    ScanStatus* status;       // nullable: no certificate (results already exhaustive)
    int level;                // 0: failures go to bad[], 1: to bad2[]
    uint32_t nq_total;        // capacity of each list
    const float* graph_qinv;  // semantic graph: its sources' scales -> eps[q] + graph_eps(graph_qinv[q], graph_uf); null: search
    float graph_uf;
};

// one CTA per query: order survivors by (sim desc, row asc), emit k, certify.  CTA b serves query qmap[b] (or b).
__global__ void __launch_bounds__(SEL_THREADS) final_kernel(const Exact* __restrict__ ex, const uint32_t* __restrict__ ex_n,
                                                            uint32_t Kp, uint32_t k,
                                                            const int64_t* __restrict__ rowids, int negate,
                                                            int64_t* __restrict__ out_rowids, float* __restrict__ out_scores,
                                                            uint32_t* __restrict__ out_counts, uint64_t* __restrict__ out_flags,
                                                            float pad_score, const uint32_t* __restrict__ qmap, CertArgs cert) {
    __shared__ uint64_t buf[SEL_MAXK];
    const uint32_t b = blockIdx.x;
    const uint32_t q = qmap ? qmap[b] : b;
    const uint32_t np2 = pow2_at_least(Kp);
    for (uint32_t i = threadIdx.x; i < np2; i += SEL_THREADS) {
        uint64_t key = 0;
        if (i < Kp && (!ex_n || i < ex_n[b])) {
            Exact e = ex[(uint64_t)b * Kp + i];
            if (e.sim == e.sim) key = score_key(e.sim, e.row);
        }
        buf[i] = key;
    }
    __syncthreads();
    block_sort_desc<SEL_THREADS>(buf, np2);
    // valid entries are the non-zero keys at the front
    __shared__ uint32_t s_valid;
    if (threadIdx.x == 0) s_valid = 0;
    __syncthreads();
    uint32_t local = 0;
    for (uint32_t i = threadIdx.x; i < np2; i += SEL_THREADS) local += buf[i] != 0 ? 1u : 0u;
    atomicAdd(&s_valid, local);
    __syncthreads();
    uint32_t valid = s_valid;
    uint32_t nout = min(valid, k);
    for (uint32_t i = threadIdx.x; i < k; i += SEL_THREADS) {
        if (i < nout) {
            uint64_t key = buf[i];
            float s = key_score(key);
            out_rowids[(uint64_t)q * k + i] = rowids[key_row(key)];
            out_scores[(uint64_t)q * k + i] = negate ? -s : s;
        } else {
            out_rowids[(uint64_t)q * k + i] = -1;
            out_scores[(uint64_t)q * k + i] = pad_score;
        }
    }
    if (threadIdx.x == 0) {
        if (out_counts) out_counts[q] = nout;
        uint64_t f = 0;
        if (valid > k && k > 0 && (buf[k - 1] >> 32) == (buf[k] >> 32)) f |= YAMS_B200_FLAG_TIE_AT_K;
        if (cert.status && k > 0) {
            const float bd = cert.bound[b];
            const float extra = cert.graph_qinv ? graph_eps(cert.graph_qinv[q], cert.graph_uf) : 0.f;
            // a graph bound of 1 or more certifies nothing: its scales may have made stage-1 scores NaN, which no bound sees
            bool certified = extra < 1.f;
            if (bd > -INFINITY) {
                const float e = cert.eps[q];
                if (cert.metric == YAMS_B200_L2) {
                    certified = false;
                    if (valid >= k) {
                        const float dk = -key_score(buf[k - 1]);
                        const double qq = cert.qnorm[q] * cert.qnorm[q];
                        // distances are floats of a float sum: allow their own rounding
                        const double dk2 = (double)dk * (double)dk * cert.l2_margin + 1e-30;
                        certified = qq - (double)bd - (double)e > dk2;
                    }
                } else {
                    const float lvl = valid >= k ? key_score(buf[k - 1]) : cert.threshold;
                    certified = bd + e + extra < lvl;
                }
            }
            if (!certified) {
                f |= YAMS_B200_FLAG_FALLBACK_PATH;
                uint32_t* cnt = cert.level == 0 ? &cert.status->n_bad : &cert.status->n_bad2;
                uint32_t* list = reinterpret_cast<uint32_t*>(cert.status + 1) + (cert.level == 0 ? 0u : cert.nq_total);
                uint32_t pos = atomicAdd(cnt, 1u);
                if (pos < cert.nq_total) list[pos] = q;
            }
        }
        if (cert.level >= 1) f |= YAMS_B200_FLAG_FALLBACK_PATH;   // answered by an exhaustive level
        if (out_flags) out_flags[q] = f;
    }
}

// level 2 (full exact pass): keys sorted descending -> the k best of ONE query
__global__ void emit_sorted_kernel(const uint64_t* __restrict__ keys, uint64_t nkeys, uint32_t k, uint32_t q,
                                   const int64_t* __restrict__ rowids, int negate, float pad_score, int64_t* __restrict__ out_rowids,
                                   float* __restrict__ out_scores, uint32_t* __restrict__ out_counts, uint64_t* __restrict__ out_flags) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < k) {
        uint64_t key = i < nkeys ? keys[i] : 0;
        if (key) {
            float s = key_score(key);
            out_rowids[(uint64_t)q * k + i] = rowids[key_row(key)];
            out_scores[(uint64_t)q * k + i] = negate ? -s : s;
        } else {
            out_rowids[(uint64_t)q * k + i] = -1;
            out_scores[(uint64_t)q * k + i] = pad_score;
        }
    }
    if (i == 0) {
        uint32_t cnt = 0;
        while (cnt < k && cnt < nkeys && keys[cnt]) ++cnt;
        if (out_counts) out_counts[q] = cnt;
        uint64_t f = YAMS_B200_FLAG_FALLBACK_PATH;
        if (cnt == k && k < nkeys && keys[k] && (keys[k - 1] >> 32) == (keys[k] >> 32)) f |= YAMS_B200_FLAG_TIE_AT_K;
        if (out_flags) out_flags[q] = f;
    }
}

// ---------------------------------------------------------------------------------------------------
// candidate-set mask: bit (q, row) set when rowids[row] is in query q's allowed list
// ---------------------------------------------------------------------------------------------------
__global__ void build_mask_kernel(const int64_t* __restrict__ allowed, const uint64_t* __restrict__ offsets, uint32_t nq,
                                  const int64_t* __restrict__ rowids, uint64_t n, uint32_t* __restrict__ mask, uint64_t mask_ld) {
    uint32_t q = blockIdx.y;
    uint64_t lo = offsets[q], hi = offsets[q + 1];
    for (uint64_t i = lo + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t a = find_row(rowids, n, allowed[i]);
        if (a < n) atomicOr(&mask[(uint64_t)q * mask_ld + (a >> 5)], 1u << (a & 31));
    }
}

// scores of rows outside query q's allowed set become -inf (threshold calibration sample / exhaustive fallback).
// scores[b * ld + i] belongs to query (qmap ? qmap[b] : b) and row row_start + i * row_stride.
__global__ void mask_scores_kernel(float* __restrict__ scores, uint64_t ld, uint64_t len, uint64_t row_stride,
                                   const uint32_t* __restrict__ mask, uint64_t mask_ld, const uint32_t* __restrict__ qmap) {
    const uint32_t b = blockIdx.y;
    const uint32_t q = qmap ? qmap[b] : b;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t row = i * row_stride;
        if (!((mask[(uint64_t)q * mask_ld + (row >> 5)] >> (row & 31)) & 1u)) scores[(uint64_t)b * ld + i] = -INFINITY;
    }
}

// Small candidate sets: no corpus pass at all.  One warp per (query, allowed rowid) pair: rowid -> row by binary
// search, stage-1 score by a coalesced fp32 dot product of that one row, Cand written at the pair's list position
// (unknown or repeated rowids become (-inf, 0xFFFFFFFF) and are skipped downstream).  Lists must be ascending.
template <int VEC>   // 8: fp16 rows, dim % 8 == 0; 4: fp32 rows, dim % 4 == 0; 0: scalar
__global__ void gather_score_kernel(const void* __restrict__ rows, int dtype, uint32_t d, const float* __restrict__ inv_norm,
                                    const int64_t* __restrict__ rowids, uint64_t n, const float* __restrict__ q32,
                                    const float* __restrict__ qinv, const int64_t* __restrict__ allowed,
                                    const uint64_t* __restrict__ offsets, uint32_t nq, uint64_t total, Cand* __restrict__ cands,
                                    uint32_t cap) {
    const uint64_t pair = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31;
    if (pair >= total) return;
    uint32_t qa = 0, qb = nq;   // last q with offsets[q] <= pair
    while (qb - qa > 1) {
        uint32_t m = (qa + qb) >> 1;
        if (offsets[m] <= pair) qa = m; else qb = m;
    }
    const uint32_t q = qa;
    const uint64_t j = pair - offsets[q];
    const int64_t want = allowed[pair];
    const uint64_t a = find_row(rowids, n, want);
    const bool valid = !(j > 0 && allowed[pair - 1] == want) && a < n;
    Cand out;
    out.score = -INFINITY;
    out.row = 0xFFFFFFFFu;
    if (valid) {
        const float* qv = q32 + (uint64_t)q * d;
        float s = 0.f;
        if (VEC == 8) {
            const uint4* r = reinterpret_cast<const uint4*>(static_cast<const __half*>(rows) + a * d);
            for (uint32_t u = lane; u < d / 8; u += 32) {
                uint4 v = __ldg(r + u);
                const __half2* h = reinterpret_cast<const __half2*>(&v);
                const float4 q0 = *reinterpret_cast<const float4*>(qv + u * 8), q1 = *reinterpret_cast<const float4*>(qv + u * 8 + 4);
                float2 f0 = __half22float2(h[0]), f1 = __half22float2(h[1]), f2 = __half22float2(h[2]), f3 = __half22float2(h[3]);
                s = fmaf(f0.x, q0.x, s); s = fmaf(f0.y, q0.y, s); s = fmaf(f1.x, q0.z, s); s = fmaf(f1.y, q0.w, s);
                s = fmaf(f2.x, q1.x, s); s = fmaf(f2.y, q1.y, s); s = fmaf(f3.x, q1.z, s); s = fmaf(f3.y, q1.w, s);
            }
        } else if (VEC == 4) {
            const float4* r = reinterpret_cast<const float4*>(static_cast<const float*>(rows) + a * d);
            for (uint32_t u = lane; u < d / 4; u += 32) {
                float4 v = __ldg(r + u);
                const float4 qq = *reinterpret_cast<const float4*>(qv + u * 4);
                s = fmaf(v.x, qq.x, s); s = fmaf(v.y, qq.y, s); s = fmaf(v.z, qq.z, s); s = fmaf(v.w, qq.w, s);
            }
        } else {
            for (uint32_t cidx = lane; cidx < d; cidx += 32) s = fmaf(load_elem(rows, dtype, a * d + cidx), qv[cidx], s);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        // rows the reference skips (inv_norm 0) score -inf like in the other engines: their s may be inf or NaN
        const float inr = inv_norm[a];
        out.score = inr > 0.f ? s * inr * qinv[q] : -INFINITY;
        out.row = (uint32_t)a;
    }
    if (lane == 0) cands[(uint64_t)q * cap + j] = out;
}
__global__ void list_lengths_kernel(const uint64_t* __restrict__ offsets, uint32_t nq, uint32_t* __restrict__ counts) {
    uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q < nq) counts[q] = (uint32_t)(offsets[q + 1] - offsets[q]);
}

// ---------------------------------------------------------------------------------------------------
// device key sort (knn.cuh), shared by the exact paths below and the sqlite-vec operators (operators.cu)
// ---------------------------------------------------------------------------------------------------
// global-memory bitonic sort (descending) of 64-bit keys, n a power of two
__global__ void bitonic_step_kernel(uint64_t* __restrict__ keys, uint64_t n, uint64_t size, uint64_t stride) {
    for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n / 2; t += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t lo = (t / stride) * (stride * 2) + (t % stride);
        uint64_t hi = lo + stride;
        bool desc = ((lo & size) == 0);
        uint64_t x = keys[lo], y = keys[hi];
        if ((x < y) == desc) { keys[lo] = y; keys[hi] = x; }
    }
}
__global__ void count_nonzero_kernel(const uint64_t* __restrict__ keys, uint64_t n, unsigned long long* __restrict__ out) {
    unsigned long long c = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) c += keys[i] != 0;
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}
__global__ void unpack_keys_kernel(const uint64_t* __restrict__ keys, uint64_t m, const int64_t* __restrict__ rowids, int negate,
                                   int64_t* __restrict__ out_rowids, float* __restrict__ out_scores) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t key = keys[i];
        uint32_t row = key_row(key);
        float s = key_score(key);
        out_rowids[i] = rowids ? rowids[row] : (int64_t)row;
        out_scores[i] = negate ? -s : s;
    }
}

void sort_keys_desc(uint64_t* keys, uint64_t np2, cudaStream_t st) {
    const unsigned g = key_grid(np2);
    for (uint64_t size = 2; size <= np2; size <<= 1)
        for (uint64_t stride = size >> 1; stride > 0; stride >>= 1) bitonic_step_kernel<<<g, 256, 0, st>>>(keys, np2, size, stride);
}
void count_nonzero_keys(const uint64_t* keys, uint64_t n, unsigned long long* d_count, cudaStream_t st) {
    count_nonzero_kernel<<<key_grid(n), 256, 0, st>>>(keys, n, d_count);
}
void unpack_keys(const uint64_t* keys, uint64_t m, const int64_t* rowids, bool negate, int64_t* out_rowids, float* out_scores,
                 cudaStream_t st) {
    unpack_keys_kernel<<<key_grid(m), 256, 0, st>>>(keys, m, rowids, negate ? 1 : 0, out_rowids, out_scores);
}

// ---------------------------------------------------------------------------------------------------
// multi-GPU: merge R partial top-k lists per query
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SEL_THREADS) merge_partials_kernel(const int64_t* __restrict__ rowids, const float* __restrict__ scores,
                                                                     uint64_t rank_stride_r, uint64_t rank_stride_s,
                                                                     uint32_t R, uint32_t nq, uint32_t k, int l2,
                                                                     int64_t* __restrict__ out_rowids, float* __restrict__ out_scores,
                                                                     uint32_t* __restrict__ out_counts) {
    extern __shared__ unsigned char smraw[];
    float* ks = reinterpret_cast<float*>(smraw);                 // np2 scores (as "bigger is better")
    int64_t* kr = reinterpret_cast<int64_t*>(smraw + 0);         // placed after scores, see below
    const uint32_t q = blockIdx.x;
    const uint32_t total = R * k, np2 = pow2_at_least(total);
    kr = reinterpret_cast<int64_t*>(smraw + (((size_t)np2 * 4 + 7) & ~(size_t)7));
    for (uint32_t i = threadIdx.x; i < np2; i += SEL_THREADS) {
        float s = -INFINITY;
        int64_t r = INT64_MAX;
        if (i < total) {
            uint32_t rk = i / k, j = i % k;
            size_t idx = (size_t)q * k + j;
            r = rowids[(size_t)rk * rank_stride_r + idx];
            s = scores[(size_t)rk * rank_stride_s + idx];
            if (l2) s = -s;
            if (r < 0) { s = -INFINITY; r = INT64_MAX; }
        }
        ks[i] = s;
        kr[i] = r;
    }
    __syncthreads();
    for (uint32_t size = 2; size <= np2; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t t = threadIdx.x; t < np2 / 2; t += SEL_THREADS) {
                uint32_t lo = (t / stride) * (stride * 2) + (t % stride);
                uint32_t hi = lo + stride;
                bool desc = ((lo & size) == 0);
                float xs = ks[lo], ys = ks[hi];
                int64_t xr = kr[lo], yr = kr[hi];
                // "x is worse than y": lower score, or equal score and larger rowid
                bool x_worse = (xs < ys) || (xs == ys && xr > yr);
                if (x_worse == desc) { ks[lo] = ys; ks[hi] = xs; kr[lo] = yr; kr[hi] = xr; }
            }
            __syncthreads();
        }
    }
    __shared__ uint32_t s_valid;
    if (threadIdx.x == 0) s_valid = 0;
    __syncthreads();
    uint32_t local = 0;
    for (uint32_t i = threadIdx.x; i < np2; i += SEL_THREADS) local += (kr[i] != INT64_MAX) ? 1u : 0u;
    atomicAdd(&s_valid, local);
    __syncthreads();
    uint32_t nout = min(s_valid, k);
    for (uint32_t i = threadIdx.x; i < k; i += SEL_THREADS) {
        if (i < nout) {
            out_rowids[(size_t)q * k + i] = kr[i];
            out_scores[(size_t)q * k + i] = l2 ? -ks[i] : ks[i];
        } else {
            out_rowids[(size_t)q * k + i] = -1;
            out_scores[(size_t)q * k + i] = l2 ? INFINITY : -INFINITY;
        }
    }
    if (threadIdx.x == 0 && out_counts) out_counts[q] = nout;
}

// candidate rowids -> row indices (binary search in the ascending device rowid table); misses get 0xFFFFFFFF
__global__ void map_rowids_kernel(const int64_t* __restrict__ allowed, uint64_t na, const int64_t* __restrict__ rowids, uint64_t n,
                                  Cand* __restrict__ sel) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < na; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t a = find_row(rowids, n, allowed[i]);
        Cand c;
        c.score = 0.f;
        c.row = a < n ? (uint32_t)a : 0xFFFFFFFFu;
        sel[i] = c;
    }
}
__global__ void iota_sel_kernel(Cand* sel, uint64_t n) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        Cand c;
        c.score = 0.f;
        c.row = (uint32_t)i;
        sel[i] = c;
    }
}
// Exact results -> sortable keys (skipped entries sort last as 0)
__global__ void exact_keys_kernel(const Exact* __restrict__ ex, uint64_t n, uint64_t np2, uint64_t* __restrict__ keys) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < np2; i += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t key = 0;
        if (i < n) {
            Exact e = ex[i];
            if (e.sim == e.sim) key = score_key(e.sim, e.row);
        }
        keys[i] = key;
    }
}

// ---- corpus_remove: stable compaction ------------------------------------------------------------------
__global__ void fill_u32_kernel(uint32_t* p, uint64_t n, uint32_t v) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) p[i] = v;
}
__global__ void mark_removed_kernel(const int64_t* __restrict__ gone, uint64_t ng, const int64_t* __restrict__ rowids, uint64_t n,
                                    uint32_t* __restrict__ keep) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < ng; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t a = find_row(rowids, n, gone[i]);
        if (a < n) keep[a] = 0u;
    }
}
// kept rows of [b0, b1) -> tmp[dst[row] - dst[b0]]; one warp per row, UNIT-byte elements
template <typename UNIT>
__global__ void compact_gather_kernel(const UNIT* __restrict__ src, uint64_t units_per_row, uint64_t b0, uint64_t b1,
                                      const uint32_t* __restrict__ keep, const uint32_t* __restrict__ dst, UNIT* __restrict__ tmp) {
    uint64_t row = b0 + (((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    uint32_t lane = threadIdx.x & 31;
    if (row >= b1 || !keep[row] || dst[row] == row) return;
    const UNIT* s = src + row * units_per_row;
    UNIT* t = tmp + (uint64_t)(dst[row] - dst[b0]) * units_per_row;
    for (uint64_t u = lane; u < units_per_row; u += 32) t[u] = s[u];
}
template <typename UNIT>
__global__ void compact_scatter_kernel(UNIT* __restrict__ rows, uint64_t units_per_row, uint64_t b0, uint64_t b1,
                                       const uint32_t* __restrict__ keep, const uint32_t* __restrict__ dst, const UNIT* __restrict__ tmp) {
    uint64_t row = b0 + (((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    uint32_t lane = threadIdx.x & 31;
    if (row >= b1 || !keep[row] || dst[row] == row) return;
    UNIT* d = rows + (uint64_t)dst[row] * units_per_row;
    const UNIT* t = tmp + (uint64_t)(dst[row] - dst[b0]) * units_per_row;
    for (uint64_t u = lane; u < units_per_row; u += 32) d[u] = t[u];
}

// per-query state of one scan: survivor counts, certificate bounds, candidate-list counters
__global__ void scan_init_kernel(uint32_t nq, uint32_t* __restrict__ sel_n, float* __restrict__ bound, uint32_t* __restrict__ counts) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nq) {
        sel_n[i] = 0;
        bound[i] = -INFINITY;
        counts[i] = 0;
    }
}
__global__ void iota_rowids_kernel(int64_t* p, uint64_t n, int64_t first) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        p[i] = first + (int64_t)i;
}

}  // namespace yb

// ===================================================================================================
// host side: corpus mirror + search orchestration
// ===================================================================================================

namespace yb {

// wgmma engine (knn_umma.cu); returns YAMS_ERR_UNSUPPORTED when the shape is not covered
yams_status_t stage1_wgmma(Corpus* c, const Stage1Args& a, bool filter, cudaStream_t st, unsigned long long* prof = nullptr);
bool wgmma_supported(const Corpus* c, uint32_t nq);

constexpr uint32_t kMaxK = 3072;          // K' = k + max(16, k/4) rounded to 32 must fit SEL_MAXK
constexpr uint32_t kSampleRows = 32768;   // strided sample that calibrates the per-query thresholds (dense fp32 scores: Q x 128 KiB)
constexpr uint32_t kSampleRank = 8;       // threshold = 8th best score of the sample
constexpr float kTauMargin = 2e-3f;       // cosine: keeps the candidate lists comfortably longer than K' (not needed for
                                          // exactness -- the certificate covers rows below the threshold)
constexpr uint32_t kCandCap = 8192;       // candidate list capacity per query
constexpr uint32_t kDenseLimit = 65536;   // corpora up to this many rows are scored densely
constexpr uint32_t kLevel1K = SEL_MAXK;   // survivors re-scored per query by exhaustive level 1
constexpr uint32_t kLevel1Group = 8;      // queries per level-1 group: group * n floats of scratch
constexpr uint32_t kGraphBatch = 1024;    // semantic-graph sources per scan (the C2 shape the wgmma engine is tuned for)

static uint32_t survivors_for(uint32_t k) {
    uint32_t slack = std::max<uint32_t>(16, k / 4);
    uint32_t kp = ((k + slack + 31) / 32) * 32;
    return std::min<uint32_t>(kp, SEL_MAXK);
}

// dist_k^2 factor of the L2 certificate (final_kernel).  The reference's float distance of a row with exact squared distance
// D^2 sums d terms fl(fl(q_i - r_i)^2): one term meets three roundings before the sum and one per later addition, t of them
// in all -- d + 2 for the scalar loop, d/8 + 9 for the AVX order (d/8 - 1 lane additions, 7 across lanes).  So the float sum
// is >= D^2 (1-u)^t and its rounded square root s >= sqrt(D^2 (1-u)^t) (1-u).  A row whose D^2 exceeds dist_k^2 (1-u)^-(t+2)
// therefore has a distance > dist_k.  The factor never drops below the 1 + 1e-4 the certificate used before it depended on d
// (enough up to d ~ 1670 in the scalar order).
static double l2_cert_margin(uint32_t d) {
    const double u = 0x1p-24;
    const double t = (d >= 16 && d % 16 == 0) ? d / 8.0 + 9.0 : d + 2.0;
    return std::max(1.0001, pow(1.0 - u, -(t + 2.0)) * (1.0 + 1e-12));
}

static yams_status_t corpus_reserve(Corpus* c, uint64_t n_total) {
    yams_status_t rc;
    if ((rc = c->rows.reserve((size_t)n_total * c->dim * c->elem() + 256, true, c->st)) != YAMS_OK) return rc;
    if ((rc = c->rowids.reserve((size_t)n_total * 8 + 256, true, c->st)) != YAMS_OK) return rc;
    if ((rc = c->inv_norm.reserve((size_t)n_total * 4 + 256, true, c->st)) != YAMS_OK) return rc;
    if (!c->stats.p) {
        if ((rc = c->stats.reserve(16)) != YAMS_OK) return rc;
        YB_CUDA(cudaMemsetAsync(c->stats.p, 0, 16, c->st));
    }
    return YAMS_OK;
}

// row statistics of the n_new rows already copied behind the current end + commit of the append.
// Nothing of the corpus state changes unless every check passed (a rejected batch leaves the corpus as it was).
static yams_status_t corpus_finish_append(Corpus* c, uint64_t n_new, const int64_t* rowids_host, int64_t first_synthetic = -1) {
    int64_t* d_rid = c->rowids.as<int64_t>() + c->n;
    int64_t last = c->last_rowid;
    bool dense = c->rowids_dense;
    if (rowids_host) {
        for (uint64_t i = 0; i < n_new; ++i) {
            YB_ARG(rowids_host[i] >= 0, "rowids must be non-negative (-1 marks an unused result slot)");
            YB_ARG(rowids_host[i] > last, "rowids must be appended in strictly ascending order");
            if (c->n + i > 0 && rowids_host[i] != last + 1) dense = false;
            last = rowids_host[i];
        }
        YB_CUDA(cudaMemcpyAsync(d_rid, rowids_host, (size_t)n_new * 8, cudaMemcpyHostToDevice, c->st));
    } else {
        int64_t first = first_synthetic >= 0 ? first_synthetic : (c->n == 0 ? 0 : last + 1);
        YB_ARG(first > last || c->n == 0, "rowids must be appended in strictly ascending order");
        if (c->n > 0 && first != last + 1) dense = false;
        iota_rowids_kernel<<<(unsigned)std::min<uint64_t>((n_new + 255) / 256, 4096), 256, 0, c->st>>>(d_rid, n_new, first);
        last = first + (int64_t)n_new - 1;
    }
    row_stats_kernel<<<(unsigned)((n_new + 127) / 128), 128, 0, c->st>>>(c->rows.p, c->dtype, c->dim, c->n, n_new,
                                                                       c->inv_norm.as<float>(), c->metric, c->stats.as<float>(), 1e-12);
    YB_CUDA(cudaGetLastError());
    float h_stats[4] = {0, 0, 0, 0};
    YB_CUDA(cudaMemcpyAsync(h_stats, c->stats.p, 16, cudaMemcpyDeviceToHost, c->st));
    YB_CUDA(cudaStreamSynchronize(c->st));
    c->r_max = h_stats[0];
    c->dr_abs_max = h_stats[1];
    c->dr_rel_max = h_stats[2];
    c->inv_max = h_stats[3];
    c->last_rowid = last;
    c->rowids_dense = dense;
    c->n += n_new;
    ++c->generation;
    return YAMS_OK;
}

// stage 1 of the direct path: cands[q * cap + j] = (score, row) of list entry j (cap >= the longest list)
static yams_status_t gather_scores(Corpus* c, const DirectLists& L, uint32_t nq, const float* q32, const float* qinv, Cand* cands,
                                   uint32_t cap, cudaStream_t st) {
    if (L.total) {
        const unsigned grid = (unsigned)((L.total * 32 + 255) / 256);
        const bool v8 = c->dtype == YAMS_B200_F16 && c->dim % 8 == 0, v4 = c->dtype == YAMS_B200_F32 && c->dim % 4 == 0;
#define YB_GATHER(V)                                                                                                              \
    gather_score_kernel<V><<<grid, 256, 0, st>>>(c->rows.p, c->dtype, c->dim, c->inv_norm.as<float>(), c->rowids.as<int64_t>(), c->n, \
                                                 q32, qinv, L.d_allowed, L.d_offsets, nq, L.total, cands, cap)
        if (v8) YB_GATHER(8); else if (v4) YB_GATHER(4); else YB_GATHER(0);
#undef YB_GATHER
    }
    YB_CUDA(cudaGetLastError());
    return YAMS_OK;
}

static ScanStatus* status_of(Corpus* c) { return c->status.as<ScanStatus>(); }

// the CUDA-core engine's stage-1 error bound of the nq prepared queries -> dst[nq] (keep_larger: the max with dst's values)
static void launch_eps_cc(Corpus* c, uint32_t nq, float* dst, bool keep_larger) {
    eps_cc_kernel<<<(nq + 255) / 256, 256, 0, c->st>>>(c->qnorm.as<double>(), nq, c->dim, c->metric, c->r_max, dst, keep_larger ? 1 : 0);
}

// The stage-1 engine of a search (tensor = wgmma_supported, fall_back) or of a diagnostic call (one engine forced).  The
// wgmma engine prepares its operand-typed queries on its first run of the call; with fall_back, a shape it declines goes to
// the CUDA-core engine.
struct Stage1Engine {
    Corpus* c;
    bool tensor, fall_back;
    bool qprep_done = false, tensor_used = false, cc_used = false;
    yams_status_t run(Stage1Args a, bool filter, unsigned long long* prof = nullptr) {
        if (tensor) {
            a.skip_qprep = qprep_done;
            yams_status_t r = stage1_wgmma(c, a, filter, c->st, prof);
            if (r == YAMS_OK) qprep_done = tensor_used = true;
            if (r != YAMS_ERR_UNSUPPORTED || !fall_back) return r;
        }
        cc_used = true;
        return stage1_cuda_core(a, filter, c->st);
    }
    // eps[] of the engine(s) that ran: the CUDA-core bound (also that of the direct path's gathered fp32 dot products),
    // max-combined with the wgmma engine's when both ran
    void launch_eps(uint32_t nq) {
        if (cc_used || !tensor_used) launch_eps_cc(c, nq, c->eps.as<float>(), tensor_used);
    }
};

// the certificate of stage 2 (final_kernel) in the corpus's metric; failures are queued in the status block (level 0: bad[],
// level 1: bad2[])
static CertArgs cert_args(Corpus* c, const ScanPlan& p, const float* bound, const float* eps, int level) {
    CertArgs cert{};
    cert.bound = bound; cert.eps = eps; cert.qnorm = c->qnorm.as<double>(); cert.threshold = p.threshold;
    cert.metric = c->metric; cert.l2_margin = l2_cert_margin(c->dim); cert.status = status_of(c); cert.level = level;
    cert.nq_total = p.nq;
    cert.graph_qinv = p.graph ? c->qinv.as<float>() : nullptr;
    cert.graph_uf = p.graph ? p.graph->uf : 0.f;
    return cert;
}

// final_kernel over `grid` CTAs in the result convention of cert.metric (L2: distances = negated scores, padding +inf)
static void launch_final(const Exact* ex, const uint32_t* ex_n, uint32_t Kp, uint32_t k, const int64_t* rowids, const DeviceResults& out,
                         uint32_t grid, const uint32_t* qmap, const CertArgs& cert, cudaStream_t st) {
    const bool l2 = cert.metric == YAMS_B200_L2;
    final_kernel<<<grid, SEL_THREADS, 0, st>>>(ex, ex_n, Kp, k, rowids, l2 ? 1 : 0, out.rowids, out.scores, out.counts, out.flags,
                                               l2 ? INFINITY : -INFINITY, qmap, cert);
}

// Stage 2 of `grid` queries (CTA b serves query qmap[b], or b): exact re-scoring of the Kp survivors of each (sel, sel_n) into
// ex, ordering, the k results into p.out and the certificate of `level` against bound[b] and eps[query].  Level 1 hands its
// survivor counts to final_kernel; level 0 orders all Kp entries (rescore_kernel marks the missing ones skipped).
static yams_status_t rescore_and_certify(Corpus* c, const ScanPlan& p, const Cand* sel, const uint32_t* sel_n, uint32_t Kp, uint32_t grid,
                                         const uint32_t* qmap, Exact* ex, const float* bound, const float* eps, int level) {
    const uint64_t tot = (uint64_t)grid * Kp;
    rescore_kernel<<<(unsigned)((tot + 127) / 128), 128, 0, c->st>>>(c->rows.p, c->dtype, c->dim, c->q32.as<float>(), c->qnorm.as<double>(),
                                                                     sel, sel_n, Kp, grid, p.threshold, ex, c->metric, qmap, p.d_mask,
                                                                     p.mask_ld, p.graph ? *p.graph : GraphRows{});
    launch_final(ex, level ? sel_n : nullptr, Kp, p.k, c->rowids.as<int64_t>(), p.out, grid, qmap, cert_args(c, p, bound, eps, level), c->st);
    YB_CUDA(cudaGetLastError());
    return YAMS_OK;
}

// the stage-1 inputs shared by every call: the corpus, the prepared queries and the row scales with their statistics (the
// cached ones of the search, or those of the semantic graph g)
static void fill_stage1_common(Corpus* c, Stage1Args& a, uint32_t nq, const GraphRows* g = nullptr) {
    a.rows = c->rows.p;
    a.inv_norm = g ? g->inv : c->inv_norm.as<float>();
    a.dim = c->dim;
    a.dtype = c->dtype;
    a.q32 = c->q32.as<float>();
    a.qinv = c->qinv.as<float>();
    a.nq = nq;
    a.metric = c->metric;
    a.eps = c->eps.as<float>();
    a.r_max = g ? g->r_max : c->r_max;
    a.dr_abs_max = g ? g->dr_abs_max : c->dr_abs_max;
    a.dr_rel_max = g ? g->dr_rel_max : c->dr_rel_max;
    a.inv_max = g ? g->inv_max : c->inv_max;
}

// Enqueues the whole pipeline for the nq queries already prepared on the device (prepare_queries) and writes the padded
// [nq][k] result into p.out.  NO host synchronisation: list overflow, short lists and stage-1 rounding are all caught by
// the certificate in final_kernel, which queues such queries in the ScanStatus block for resolve_uncertain().
static yams_status_t scan_enqueue(Corpus* c, const ScanPlan& p) {
    yams_status_t rc;
    cudaStream_t st = c->st;
    const uint32_t nq = p.nq;
    const uint32_t Kp = survivors_for(p.k);
    const uint64_t n = c->n;
    const bool l2 = c->metric == YAMS_B200_L2;
    c->scan_timed = false;
    uint32_t* d_counts = c->counts.as<uint32_t>();
    if ((rc = c->sel.reserve((size_t)nq * Kp * sizeof(Cand) + (size_t)nq * 4)) != YAMS_OK) return rc;
    if ((rc = c->bound.reserve((size_t)nq * 4)) != YAMS_OK) return rc;
    if ((rc = c->eps.reserve((size_t)nq * 4)) != YAMS_OK) return rc;
    Stage1Args a{};
    fill_stage1_common(c, a, nq, p.graph);
    Stage1Engine s1{c, wgmma_supported(c, nq), true};
    Cand* d_sel = c->sel.as<Cand>();
    uint32_t* d_sel_n = reinterpret_cast<uint32_t*>(d_sel + (size_t)nq * Kp);
    float* d_bound = c->bound.as<float>();
    scan_init_kernel<<<(nq + 255) / 256, 256, 0, st>>>(nq, d_sel_n, d_bound, d_counts);

    if (n == 0) {
        // nothing to score: every list is empty, bound = -inf
    } else if (p.direct) {
        // ---- small candidate sets: score the listed rows only ----
        const uint32_t cap = std::max<uint32_t>(p.lists.max_len, 1);
        if ((rc = c->cands.reserve((size_t)nq * cap * sizeof(Cand))) != YAMS_OK) return rc;
        list_lengths_kernel<<<(nq + 255) / 256, 256, 0, st>>>(p.lists.d_offsets, nq, d_counts);
        if (p.lists.total) YB_CUDA(cudaEventRecord(c->ev_scan[0], st));
        if ((rc = gather_scores(c, p.lists, nq, a.q32, a.qinv, c->cands.as<Cand>(), cap, st)) != YAMS_OK) return rc;
        if (p.lists.total) {
            YB_CUDA(cudaEventRecord(c->ev_scan[1], st));
            c->scan_timed = true;
        }
        SelectIn in{};
        in.cands = c->cands.as<Cand>(); in.counts = d_counts; in.cap = cap;
        topk_select_kernel<<<nq, SEL_THREADS, 0, st>>>(in, Kp, 0, nullptr, d_sel, d_sel_n, d_bound);
    } else if (!p.d_mask && n <= kDenseLimit) {
        // ---- dense: every score materialised, exact top-K' straight from the matrix ----
        if ((rc = c->dense.reserve((size_t)nq * n * 4)) != YAMS_OK) return rc;
        a.row_start = 0; a.row_stride = 1; a.nrows = n;
        a.out_scores = c->dense.as<float>(); a.ld = n;
        if ((rc = s1.run(a, false)) != YAMS_OK) return rc;
        SelectIn in{};
        in.dense = c->dense.as<float>(); in.ld = n; in.row_start = 0; in.row_stride = 1; in.dense_len = n;
        topk_select_kernel<<<nq, SEL_THREADS, 0, st>>>(in, Kp, 0, nullptr, d_sel, d_sel_n, d_bound);
    } else {
        uint32_t cap;
        if ((rc = c->tau.reserve((size_t)nq * 4)) != YAMS_OK) return rc;
        float* d_tau = c->tau.as<float>();
        {
            // ---- thresholds from a strided sample (candidate-set mode: of the ALLOWED sample rows, so that ~4*K'
            //      allowed rows are expected above it; -inf when the sample holds fewer than m allowed rows) ----
            uint64_t S = std::min<uint64_t>(n, kSampleRows);
            uint64_t stride = n / S;
            // the sample rank is chosen so that ~4*K' rows are expected above the threshold
            uint32_t m = (uint32_t)std::max<uint64_t>(kSampleRank, (4ull * Kp + stride - 1) / stride);
            uint64_t expected = (uint64_t)m * stride;
            cap = (uint32_t)std::max<uint64_t>(kCandCap, ((3 * expected + 1023) / 1024) * 1024);
            if ((rc = c->sample_scores.reserve((size_t)nq * S * 4)) != YAMS_OK) return rc;
            Stage1Args s = a;
            s.row_start = 0; s.row_stride = stride; s.nrows = S;
            s.out_scores = c->sample_scores.as<float>(); s.ld = S;
            if ((rc = s1.run(s, false)) != YAMS_OK) return rc;
            if (p.d_mask)
                mask_scores_kernel<<<dim3((unsigned)((S + 255) / 256), nq), 256, 0, st>>>(c->sample_scores.as<float>(), S, S, stride,
                                                                                         p.d_mask, p.mask_ld, nullptr);
            SelectIn in{};
            in.dense = c->sample_scores.as<float>(); in.ld = S; in.row_start = 0; in.row_stride = stride; in.dense_len = S;
            in.tau_margin = l2 ? 0.f : kTauMargin;
            in.fast_tau = p.d_mask ? 0 : 1;   // candidate sets: masked sample rows are -inf, the exact rank matters there
            topk_select_kernel<<<nq, SEL_THREADS, 0, st>>>(in, m, 1, d_tau, nullptr, nullptr, nullptr);
        }
        if ((rc = c->cands.reserve((size_t)nq * cap * sizeof(Cand))) != YAMS_OK) return rc;
        Stage1Args f = a;
        f.row_start = 0; f.row_stride = 1; f.nrows = n;
        f.tau = d_tau; f.cands = c->cands.as<Cand>(); f.cap = cap; f.counts = d_counts;
        f.mask = p.d_mask; f.mask_ld = p.mask_ld;
        YB_CUDA(cudaEventRecord(c->ev_scan[0], st));
        if ((rc = s1.run(f, true)) != YAMS_OK) return rc;
        YB_CUDA(cudaEventRecord(c->ev_scan[1], st));
        c->scan_timed = true;
        SelectIn in{};
        in.cands = c->cands.as<Cand>(); in.counts = d_counts; in.cap = cap; in.tau = d_tau;
        topk_select_kernel<<<nq, SEL_THREADS, 0, st>>>(in, Kp, 0, nullptr, d_sel, d_sel_n, d_bound);
    }
    s1.launch_eps(nq);
    c->last_ms[4] = s1.tensor_used ? 1.f : 0.f;   // the engine that ran: wgmma declines shapes it does not take (nq > 4096)
    YB_CUDA(cudaEventRecord(c->ev[1], st));
    // ---- stage 2: exact re-scoring, ordering, certificate ----
    if ((rc = c->outbuf.reserve((size_t)nq * Kp * sizeof(Exact))) != YAMS_OK) return rc;
    return rescore_and_certify(c, p, d_sel, d_sel_n, Kp, nq, nullptr, c->outbuf.as<Exact>(), d_bound, c->eps.as<float>(), 0);
}

// entry points for the other engines (pq.cu): exact top-K of per-query candidate lists, and the plain final ordering
void launch_topk_lists(const Cand* lists, const uint32_t* counts, uint32_t cap, uint32_t nq, uint32_t K, Cand* out_sel, uint32_t* out_n,
                       cudaStream_t st) {
    SelectIn in{};
    in.cands = lists; in.counts = counts; in.cap = cap;
    topk_select_kernel<<<nq, SEL_THREADS, 0, st>>>(in, K, 0, nullptr, out_sel, out_n, nullptr);
}
// top-K of dense score rows: row q of `dense` holds the n scores of documents 0..n-1; out_sel[q * K ..] best first (score
// descending, then document ascending), out_n[q] = min(n, K)
void launch_topk_dense(const float* dense, uint64_t n, uint32_t nq, uint32_t K, Cand* out_sel, uint32_t* out_n, cudaStream_t st) {
    SelectIn in{};
    in.dense = dense; in.ld = n; in.row_start = 0; in.row_stride = 1; in.dense_len = n;
    topk_select_kernel<<<nq, SEL_THREADS, 0, st>>>(in, K, 0, nullptr, out_sel, out_n, nullptr);
}
void launch_final_plain(const Exact* exact, uint32_t Kp, uint32_t k, uint32_t nq, const int64_t* rowids, const DeviceResults& out,
                        cudaStream_t st) {
    // status == nullptr: no certificate (the caller's survivors are what the reference re-ranks, too); cosine results
    launch_final(exact, nullptr, Kp, k, rowids, out, nq, nullptr, CertArgs{}, st);
}
// rowids -> corpus rows (out[i].row, 0xFFFFFFFF for unknown rowids), any order
void launch_map_rowids(const int64_t* rowids_in, uint64_t n_in, const int64_t* corpus_rowids, uint64_t n, Cand* out, cudaStream_t st) {
    if (n_in) map_rowids_kernel<<<(unsigned)std::min<uint64_t>((n_in + 255) / 256, 65535), 256, 0, st>>>(rowids_in, n_in, corpus_rowids, n, out);
}
// the search's query preparation (cosine): qnorm[q] = sqrt of the sequential double sum of squares; the first uint32 of the
// zeroed 16-byte block `status` counts the queries the reference rejects (non-finite, |q|^2 < 1e-10)
void launch_query_prep(const float* q, uint32_t nq, uint32_t d, double* qnorm, float* qinv, void* status, cudaStream_t st) {
    query_prep_kernel<<<(nq + QP_THREADS - 1) / QP_THREADS, QP_THREADS, 0, st>>>(q, nq, d, qnorm, qinv, YAMS_B200_COSINE,
                                                                                static_cast<ScanStatus*>(status));
}

// DeviceResults (knn.cuh) in `buf`, the results buffer of the caller's handle
yams_status_t reserve_results(DevBuf& buf, uint32_t nq, uint32_t k, DeviceResults* r) {
    yams_status_t rc = buf.reserve((size_t)nq * k * 12 + (size_t)nq * 12 + 64);
    if (rc != YAMS_OK) return rc;
    r->rowids = buf.as<int64_t>();
    r->flags = reinterpret_cast<uint64_t*>(r->rowids + (size_t)nq * k);
    r->scores = reinterpret_cast<float*>(r->flags + nq);
    r->counts = reinterpret_cast<uint32_t*>(r->scores + (size_t)nq * k);
    return YAMS_OK;
}
yams_status_t enqueue_results(const DeviceResults& r, uint32_t nq, uint32_t k, int64_t* out_rowids, float* out_scores, uint32_t* out_counts,
                              uint64_t* out_flags, cudaStream_t st) {
    YB_CUDA(cudaMemcpyAsync(out_rowids, r.rowids, (size_t)nq * k * 8, cudaMemcpyDeviceToHost, st));
    YB_CUDA(cudaMemcpyAsync(out_scores, r.scores, (size_t)nq * k * 4, cudaMemcpyDeviceToHost, st));
    YB_CUDA(cudaMemcpyAsync(out_counts, r.counts, (size_t)nq * 4, cudaMemcpyDeviceToHost, st));
    if (out_flags) YB_CUDA(cudaMemcpyAsync(out_flags, r.flags, (size_t)nq * 8, cudaMemcpyDeviceToHost, st));
    return YAMS_OK;
}
yams_status_t copy_results(const DeviceResults& r, uint32_t nq, uint32_t k, int64_t* out_rowids, float* out_scores, uint32_t* out_counts,
                           uint64_t* out_flags, cudaStream_t st) {
    yams_status_t rc = enqueue_results(r, nq, k, out_rowids, out_scores, out_counts, out_flags, st);
    if (rc != YAMS_OK) return rc;
    YB_CUDA(cudaStreamSynchronize(st));
    return YAMS_OK;
}

// Exact scores of m corpus rows for query q (rescore_kernel; with a mask, rows outside it are skipped) as keys sorted
// descending into c->dense[0, np2), np2 = pow2_at_least(max(m, 1)); skipped rows and the padding are zero keys at the end.
// The rows are those of the m rowids at d_allowed (map_rowids_kernel, unknown rowids skipped) or, without a list, rows
// 0 .. m-1.  Workspace: c->sel (row list), c->outbuf (exact scores), c->lvl[0, 8) ({m, q}) and c->dense (keys); c->lvl past
// its first 8 bytes is left alone.
static yams_status_t exact_sorted_keys(Corpus* c, uint32_t q, uint64_t m, const int64_t* d_allowed, float threshold,
                                       const uint32_t* mask, uint64_t mask_ld, const GraphRows* graph = nullptr) {
    yams_status_t rc;
    cudaStream_t st = c->st;
    const uint64_t np2 = pow2_at_least(std::max<uint64_t>(m, 1));
    if ((rc = c->sel.reserve((size_t)m * sizeof(Cand) + 64)) != YAMS_OK) return rc;
    if ((rc = c->outbuf.reserve((size_t)m * sizeof(Exact) + 64)) != YAMS_OK) return rc;
    if ((rc = c->dense.reserve((size_t)np2 * 8 + 64)) != YAMS_OK) return rc;
    if ((rc = c->lvl.reserve(64)) != YAMS_OK) return rc;
    Cand* d_sel = c->sel.as<Cand>();
    uint32_t* d_small = c->lvl.as<uint32_t>();     // [0] = survivors (m), [1] = query index
    uint32_t h_small[2] = {(uint32_t)m, q};
    YB_CUDA(cudaMemcpyAsync(d_small, h_small, 8, cudaMemcpyHostToDevice, st));
    const unsigned g = key_grid(np2);
    if (m) {
        if (d_allowed) map_rowids_kernel<<<g, 256, 0, st>>>(d_allowed, m, c->rowids.as<int64_t>(), c->n, d_sel);
        else iota_sel_kernel<<<g, 256, 0, st>>>(d_sel, m);
        rescore_kernel<<<(unsigned)((m + 127) / 128), 128, 0, st>>>(c->rows.p, c->dtype, c->dim, c->q32.as<float>(), c->qnorm.as<double>(), d_sel, d_small,
                                                                   (uint32_t)m, 1, threshold, c->outbuf.as<Exact>(), c->metric, d_small + 1,
                                                                   mask, mask_ld, graph ? *graph : GraphRows{});
    }
    exact_keys_kernel<<<g, 256, 0, st>>>(c->outbuf.as<Exact>(), m, np2, c->dense.as<uint64_t>());
    sort_keys_desc(c->dense.as<uint64_t>(), np2, st);
    YB_CUDA(cudaGetLastError());
    return YAMS_OK;
}

// Level 2: exact score of EVERY row for one query (the reference's own loop, row-parallel) + a global sort.
static yams_status_t exact_all_rows(Corpus* c, const ScanPlan& p, uint32_t q) {
    yams_status_t rc;
    cudaStream_t st = c->st;
    const bool l2 = c->metric == YAMS_B200_L2;
    if ((rc = exact_sorted_keys(c, q, c->n, nullptr, p.threshold, p.d_mask, p.mask_ld, p.graph)) != YAMS_OK) return rc;
    emit_sorted_kernel<<<(p.k + 255) / 256, 256, 0, st>>>(c->dense.as<uint64_t>(), c->n, p.k, q, c->rowids.as<int64_t>(), l2 ? 1 : 0,
                                                          l2 ? INFINITY : -INFINITY, p.out.rowids, p.out.scores, p.out.counts, p.out.flags);
    YB_CUDA(cudaGetLastError());
    YB_CUDA(cudaStreamSynchronize(st));   // h_small / scratch reuse
    return YAMS_OK;
}

// Blocking: answers the queries the certificate rejected.
//   level 1: dense stage-1 scores of ALL rows with the CUDA-core engine (error bound eps_cc, ~1e-5), exact re-scoring of the
//            best kLevel1K (4096) rows instead of K', same certificate;
//   level 2: whatever level 1 cannot certify either (more than ~4000 rows within eps of the k-th score: a corpus of
//            duplicates) is answered by the exact score of every row.
static yams_status_t resolve_uncertain(Corpus* c, const ScanPlan& p, const uint32_t* bad, uint32_t n_bad, uint32_t* out_full) {
    yams_status_t rc;
    cudaStream_t st = c->st;
    const uint64_t n = c->n;
    const uint32_t G = kLevel1Group, K1 = kLevel1K;
    if ((rc = c->dense.reserve((size_t)G * n * 4 + (size_t)G * c->dim * 4 + (size_t)G * 8 + 64)) != YAMS_OK) return rc;
    if ((rc = c->lvl.reserve((size_t)G * K1 * (sizeof(Cand) + sizeof(Exact)) + (size_t)G * 16 + 64)) != YAMS_OK) return rc;
    if ((rc = c->eps2.reserve((size_t)p.nq * 4)) != YAMS_OK) return rc;
    float* d_scores = c->dense.as<float>();
    float* d_qg = d_scores + (size_t)G * n;
    float* d_qinv_g = d_qg + (size_t)G * c->dim;
    uint32_t* d_qmap = reinterpret_cast<uint32_t*>(d_qinv_g + G);
    Cand* d_sel1 = c->lvl.as<Cand>();
    Exact* d_ex1 = reinterpret_cast<Exact*>(d_sel1 + (size_t)G * K1);
    uint32_t* d_sel1_n = reinterpret_cast<uint32_t*>(d_ex1 + (size_t)G * K1);
    float* d_bound1 = reinterpret_cast<float*>(d_sel1_n + G);
    launch_eps_cc(c, p.nq, c->eps2.as<float>(), false);
    Stage1Args a{};
    fill_stage1_common(c, a, p.nq, p.graph);
    for (uint32_t g0 = 0; g0 < n_bad; g0 += G) {
        uint32_t g = std::min<uint32_t>(G, n_bad - g0);
        for (uint32_t i = 0; i < g; ++i) {
            YB_CUDA(cudaMemcpyAsync(d_qg + (size_t)i * c->dim, a.q32 + (size_t)bad[g0 + i] * c->dim, (size_t)c->dim * 4,
                                    cudaMemcpyDeviceToDevice, st));
            YB_CUDA(cudaMemcpyAsync(d_qinv_g + i, a.qinv + bad[g0 + i], 4, cudaMemcpyDeviceToDevice, st));
        }
        YB_CUDA(cudaMemcpyAsync(d_qmap, bad + g0, (size_t)g * 4, cudaMemcpyHostToDevice, st));
        Stage1Args e = a;
        e.q32 = d_qg; e.qinv = d_qinv_g; e.nq = g;
        e.row_start = 0; e.row_stride = 1; e.nrows = n; e.out_scores = d_scores; e.ld = n;
        if ((rc = stage1_cuda_core(e, false, st)) != YAMS_OK) return rc;
        if (p.d_mask)
            mask_scores_kernel<<<dim3((unsigned)std::min<uint64_t>((n + 255) / 256, 65535), g), 256, 0, st>>>(d_scores, n, n, 1, p.d_mask,
                                                                                                             p.mask_ld, d_qmap);
        SelectIn in{};
        in.dense = d_scores; in.ld = n; in.row_start = 0; in.row_stride = 1; in.dense_len = n;
        topk_select_kernel<<<g, SEL_THREADS, 0, st>>>(in, K1, 0, nullptr, d_sel1, d_sel1_n, d_bound1);
        if ((rc = rescore_and_certify(c, p, d_sel1, d_sel1_n, K1, g, d_qmap, d_ex1, d_bound1, c->eps2.as<float>(), 1)) != YAMS_OK) return rc;
        YB_CUDA(cudaStreamSynchronize(st));  // d_qmap / bad reuse
    }
    // level 2 for what is left
    uint32_t n_bad2 = 0;
    YB_CUDA(cudaMemcpyAsync(&n_bad2, &status_of(c)->n_bad2, 4, cudaMemcpyDeviceToHost, st));
    YB_CUDA(cudaStreamSynchronize(st));
    if (n_bad2) {
        n_bad2 = std::min(n_bad2, p.nq);
        *out_full = n_bad2;
        std::vector<uint32_t> bad2(n_bad2);
        const uint32_t* d_list2 = reinterpret_cast<const uint32_t*>(status_of(c) + 1) + p.nq;
        YB_CUDA(cudaMemcpyAsync(bad2.data(), d_list2, (size_t)n_bad2 * 4, cudaMemcpyDeviceToHost, st));
        YB_CUDA(cudaStreamSynchronize(st));
        for (uint32_t q : bad2)
            if ((rc = exact_all_rows(c, p, q)) != YAMS_OK) return rc;
    }
    return YAMS_OK;
}

}  // namespace yb

using namespace yb;

template <typename UNIT>
static yams_status_t compact_array(Corpus* c, void* base, uint64_t row_bytes, const uint32_t* d_keep, const uint32_t* d_dst,
                                   DevBuf& tmp) {
    const uint64_t units = row_bytes / sizeof(UNIT);
    // batches of <= 256 MiB: destinations never pass sources, so batch i only overwrites rows that batches <= i
    // have already moved (or staged in tmp)
    uint64_t batch = std::max<uint64_t>(1, (256ull << 20) / row_bytes);
    yams_status_t rc = tmp.reserve((size_t)std::min<uint64_t>(batch, c->n) * row_bytes);
    if (rc != YAMS_OK) return rc;
    for (uint64_t b0 = 0; b0 < c->n; b0 += batch) {
        uint64_t b1 = std::min<uint64_t>(c->n, b0 + batch);
        unsigned grid = (unsigned)(((b1 - b0) * 32 + 255) / 256);
        compact_gather_kernel<UNIT><<<grid, 256, 0, c->st>>>(static_cast<const UNIT*>(base), units, b0, b1, d_keep, d_dst, tmp.as<UNIT>());
        compact_scatter_kernel<UNIT><<<grid, 256, 0, c->st>>>(static_cast<UNIT*>(base), units, b0, b1, d_keep, d_dst, tmp.as<UNIT>());
    }
    YB_CUDA(cudaGetLastError());
    return YAMS_OK;
}

extern "C" {

yams_status_t yams_b200_corpus_create(void* self, uint32_t dim, int dtype, int metric, uint64_t capacity_hint,
                                      yams_b200_corpus** out) {
    YB_TRY
    (void)self;
    YB_ARG(out, "out is null");
    *out = nullptr;
    YB_ARG(dim > 0 && dim <= 65536, "dim must be in 1..65536");  // vec0_module.hpp:109
    YB_ARG(dtype == YAMS_B200_F32 || dtype == YAMS_B200_F16, "unknown dtype");
    YB_ARG(metric == YAMS_B200_COSINE || metric == YAMS_B200_L2, "unknown metric");
    DeviceCtx* dev = nullptr;
    yams_status_t rc = ensure_device(&dev);
    if (rc != YAMS_OK) return rc;
    std::unique_ptr<yams_b200_corpus> c(new (std::nothrow) yams_b200_corpus());
    if (!c) return YAMS_ERR_INTERNAL;
    c->dev = dev;
    c->dim = dim;
    c->dtype = dtype;
    c->metric = metric;
    if (cudaStreamCreateWithFlags(&c->st, cudaStreamNonBlocking) != cudaSuccess) {
        set_last_error("cudaStreamCreate failed");
        return YAMS_ERR_INTERNAL;
    }
    for (auto& e : c->ev) cudaEventCreate(&e);
    for (auto& e : c->ev_scan) cudaEventCreate(&e);
    if (capacity_hint && (rc = corpus_reserve(c.get(), capacity_hint)) != YAMS_OK) return rc;
    *out = c.release();
    return YAMS_OK;
    YB_CATCH
}

void yams_b200_corpus_destroy(yams_b200_corpus* c) { delete c; }

yams_status_t yams_b200_corpus_append(yams_b200_corpus* c, const void* rows, uint64_t n, const int64_t* rowids) {
    YB_TRY
    YB_ARG(c, "corpus is null");
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_BIND(c);
    settle_pending(c);
    if (n == 0) return YAMS_OK;
    YB_ARG(rows, "rows is null");
    YB_ARG(c->n + n < 0xFFFFFFFFull, "corpus is limited to 2^32-1 rows per GPU");
    yams_status_t rc = corpus_reserve(c, c->n + n);
    if (rc != YAMS_OK) return rc;
    size_t rb = (size_t)c->dim * c->elem();
    YB_CUDA(cudaMemcpyAsync(c->rows.as<uint8_t>() + (size_t)c->n * rb, rows, (size_t)n * rb, cudaMemcpyHostToDevice, c->st));
    return corpus_finish_append(c, n, rowids);
    YB_CATCH
}

yams_status_t yams_b200_corpus_append_f32_as_f16(yams_b200_corpus* c, const float* rows, uint64_t n, const int64_t* rowids) {
    YB_TRY
    YB_ARG(c, "corpus is null");
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_BIND(c);
    settle_pending(c);
    YB_ARG(c->dtype == YAMS_B200_F16, "corpus is not fp16");
    if (n == 0) return YAMS_OK;
    YB_ARG(rows, "rows is null");
    YB_ARG(c->n + n < 0xFFFFFFFFull, "corpus is limited to 2^32-1 rows per GPU");
    yams_status_t rc = corpus_reserve(c, c->n + n);
    if (rc != YAMS_OK) return rc;
    size_t cnt = (size_t)n * c->dim;
    if ((rc = c->dense.reserve(cnt * 4)) != YAMS_OK) return rc;
    YB_CUDA(cudaMemcpyAsync(c->dense.p, rows, cnt * 4, cudaMemcpyHostToDevice, c->st));
    convert_f32_to_f16_trunc_kernel<<<(unsigned)std::min<size_t>((cnt + 255) / 256, 65535), 256, 0, c->st>>>(
        c->dense.as<float>(), c->rows.as<uint16_t>() + (size_t)c->n * c->dim, cnt);
    return corpus_finish_append(c, n, rowids);
    YB_CATCH
}

yams_status_t yams_b200_corpus_append_synthetic(yams_b200_corpus* c, uint64_t seed, uint64_t first_row, uint64_t n) {
    YB_TRY
    YB_ARG(c, "corpus is null");
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_BIND(c);
    settle_pending(c);
    if (n == 0) return YAMS_OK;
    YB_ARG(c->n + n < 0xFFFFFFFFull, "corpus is limited to 2^32-1 rows per GPU");
    yams_status_t rc = corpus_reserve(c, c->n + n);
    if (rc != YAMS_OK) return rc;
    if ((rc = c->misc.reserve((size_t)n * 4)) != YAMS_OK) return rc;
    float* d_inv = c->misc.as<float>();
    synth_rownorm_kernel<<<(unsigned)((n + 127) / 128), 128, 0, c->st>>>(seed, first_row, n, c->dim, d_inv);
    size_t rb = (size_t)c->dim * c->elem();
    synth_fill_kernel<<<c->dev->sm_count * 16, 256, 0, c->st>>>(seed, first_row, n, c->dim, d_inv,
                                                               c->rows.as<uint8_t>() + (size_t)c->n * rb, c->dtype);
    YB_CUDA(cudaGetLastError());
    // rowid = first_row + i
    return corpus_finish_append(c, n, nullptr, (int64_t)first_row);
    YB_CATCH
}

yams_status_t yams_b200_corpus_remove(yams_b200_corpus* c, const int64_t* rowids, uint64_t n, uint64_t* out_removed) {
    YB_TRY
    YB_ARG(c, "corpus is null");
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_BIND(c);
    settle_pending(c);
    if (out_removed) *out_removed = 0;
    if (n == 0 || c->n == 0) return YAMS_OK;
    YB_ARG(rowids, "rowids is null");
    yams_status_t rc;
    cudaStream_t st = c->st;
    if ((rc = c->mask.reserve((size_t)n * 8)) != YAMS_OK) return rc;
    if ((rc = c->sel.reserve((size_t)c->n * 4 + 16)) != YAMS_OK) return rc;
    if ((rc = c->outbuf.reserve((size_t)c->n * 4 + 16)) != YAMS_OK) return rc;
    if ((rc = c->tau.reserve(8)) != YAMS_OK) return rc;
    uint32_t* d_keep = c->sel.as<uint32_t>();
    uint32_t* d_dst = c->outbuf.as<uint32_t>();
    uint64_t* d_total = reinterpret_cast<uint64_t*>(c->tau.p);
    YB_CUDA(cudaMemcpyAsync(c->mask.p, rowids, (size_t)n * 8, cudaMemcpyHostToDevice, st));
    unsigned g = (unsigned)std::min<uint64_t>((c->n + 255) / 256, 65535);
    fill_u32_kernel<<<g, 256, 0, st>>>(d_keep, c->n, 1u);
    mark_removed_kernel<<<(unsigned)std::min<uint64_t>((n + 255) / 256, 65535), 256, 0, st>>>(c->mask.as<int64_t>(), n, c->rowids.as<int64_t>(),
                                                                                              c->n, d_keep);
    if ((rc = exclusive_scan_u32(d_keep, d_dst, c->n, d_total, c->misc, st)) != YAMS_OK) return rc;
    uint64_t kept = 0;
    YB_CUDA(cudaMemcpyAsync(&kept, d_total, 8, cudaMemcpyDeviceToHost, st));
    YB_CUDA(cudaStreamSynchronize(st));
    if (kept == c->n) return YAMS_OK;
    const uint64_t row_bytes = (uint64_t)c->dim * c->elem();
    if (row_bytes % 16 == 0) rc = compact_array<uint4>(c, c->rows.p, row_bytes, d_keep, d_dst, c->dense);
    else if (row_bytes % 4 == 0) rc = compact_array<uint32_t>(c, c->rows.p, row_bytes, d_keep, d_dst, c->dense);
    else rc = compact_array<uint16_t>(c, c->rows.p, row_bytes, d_keep, d_dst, c->dense);
    if (rc == YAMS_OK) rc = compact_array<uint64_t>(c, c->rowids.p, 8, d_keep, d_dst, c->dense);
    if (rc == YAMS_OK) rc = compact_array<uint32_t>(c, c->inv_norm.p, 4, d_keep, d_dst, c->dense);
    if (rc != YAMS_OK) return rc;
    int64_t last = INT64_MIN;
    if (kept) YB_CUDA(cudaMemcpyAsync(&last, c->rowids.as<int64_t>() + (kept - 1), 8, cudaMemcpyDeviceToHost, st));
    YB_CUDA(cudaStreamSynchronize(st));
    if (out_removed) *out_removed = c->n - kept;
    c->n = kept;
    ++c->generation;
    c->last_rowid = last;
    c->rowids_dense = false;
    return YAMS_OK;
    YB_CATCH
}

yams_status_t yams_b200_corpus_clear(yams_b200_corpus* c) {
    YB_TRY
    YB_ARG(c, "corpus is null");
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_BIND(c);
    settle_pending(c);
    c->n = 0;
    ++c->generation;
    c->last_rowid = INT64_MIN;
    c->rowids_dense = true;
    c->r_max = c->dr_abs_max = c->dr_rel_max = c->inv_max = 0.f;
    if (c->stats.p) YB_CUDA(cudaMemsetAsync(c->stats.p, 0, 16, c->st));
    return YAMS_OK;
    YB_CATCH
}

yams_status_t yams_b200_corpus_size(const yams_b200_corpus* c, uint64_t* out_n) {
    YB_ARG(c && out_n, "null argument");
    *out_n = c->n;
    return YAMS_OK;
}

yams_status_t yams_b200_corpus_sync(yams_b200_corpus* c) {
    YB_TRY
    YB_ARG(c, "corpus is null");
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_BIND(c);
    YB_CUDA(cudaStreamSynchronize(c->st));
    return YAMS_OK;
    YB_CATCH
}

void* yams_b200_corpus_stream(yams_b200_corpus* c) { return c ? (void*)c->st : nullptr; }

// uploads the queries and enqueues their preparation: q32, qinv, qnorm on the device, status block zeroed,
// invalid queries counted in status->n_invalid (read by the host together with the results -- no synchronisation here)
static yams_status_t reserve_queries(yams_b200_corpus* c, uint32_t nq) {
    yams_status_t rc;
    if ((rc = c->q32.reserve((size_t)nq * c->dim * 4)) != YAMS_OK) return rc;
    if ((rc = c->qinv.reserve((size_t)nq * 4)) != YAMS_OK) return rc;
    if ((rc = c->qnorm.reserve((size_t)nq * 8)) != YAMS_OK) return rc;
    if ((rc = c->counts.reserve((size_t)nq * 4)) != YAMS_OK) return rc;
    if ((rc = c->status.reserve(sizeof(ScanStatus) + (size_t)nq * 8)) != YAMS_OK) return rc;
    if ((rc = c->h_pin.reserve(sizeof(ScanStatus) + (size_t)nq * 8 + 64)) != YAMS_OK) return rc;
    YB_CUDA(cudaMemsetAsync(c->status.p, 0, sizeof(ScanStatus), c->st));
    return YAMS_OK;
}
static yams_status_t prepare_queries(yams_b200_corpus* c, const float* q_src, bool src_is_device, uint32_t nq) {
    yams_status_t rc;
    size_t qb = (size_t)nq * c->dim * 4;
    if ((rc = reserve_queries(c, nq)) != YAMS_OK) return rc;
    YB_CUDA(cudaMemcpyAsync(c->q32.p, q_src, qb, src_is_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, c->st));
    query_prep_kernel<<<(nq + QP_THREADS - 1) / QP_THREADS, QP_THREADS, 0, c->st>>>(c->q32.as<float>(), nq, c->dim, c->qnorm.as<double>(),
                                                                                  c->qinv.as<float>(), c->metric, status_of(c));
    YB_CUDA(cudaGetLastError());
    return YAMS_OK;
}
// the semantic-graph form: the sources of batch p (all of them taken) as queries; the status block zeroed
static yams_status_t prepare_sources(yams_b200_corpus* c, const ScanPlan& p) {
    yams_status_t rc;
    if ((rc = reserve_queries(c, p.nq)) != YAMS_OK) return rc;
    gather_sources_kernel<<<key_grid((uint64_t)p.nq * c->dim), 256, 0, c->st>>>(c->rows.p, c->dtype, c->dim, *p.graph, p.nq,
                                                                               c->q32.as<float>(), c->qinv.as<float>());
    YB_CUDA(cudaGetLastError());
    return YAMS_OK;
}

// [0..2] and [5] of search_last_timings from the events of the last scan; the caller has seen them complete
static void time_scan_events(yams_b200_corpus* c) {
    cudaEventElapsedTime(&c->last_ms[0], c->ev[0], c->ev[1]);
    cudaEventElapsedTime(&c->last_ms[1], c->ev[1], c->ev[2]);
    cudaEventElapsedTime(&c->last_ms[2], c->ev[0], c->ev[2]);
    c->last_ms[5] = 0.f;
    if (c->scan_timed) cudaEventElapsedTime(&c->last_ms[5], c->ev_scan[0], c->ev_scan[1]);
}
// candidate sets as a bit matrix [nq][mask_ld * 32] of allowed corpus rows (allowed_offsets[nq + 1] into allowed_rowids)
static yams_status_t upload_mask(yams_b200_corpus* c, uint32_t nq, const int64_t* allowed_rowids, const uint64_t* allowed_offsets,
                                 const uint32_t** out_mask, uint64_t* out_mask_ld) {
    yams_status_t rc;
    const uint64_t total = allowed_offsets[nq];
    const uint64_t mask_ld = (c->n + 31) / 32;
    const size_t mb = (size_t)nq * mask_ld * 4;
    if ((rc = c->mask.reserve(mb + (size_t)total * 8 + (size_t)(nq + 1) * 8 + 64)) != YAMS_OK) return rc;
    uint32_t* dm = c->mask.as<uint32_t>();
    int64_t* d_allowed = reinterpret_cast<int64_t*>(c->mask.as<uint8_t>() + ((mb + 7) & ~(size_t)7));
    uint64_t* d_offs = reinterpret_cast<uint64_t*>(d_allowed + total);
    YB_CUDA(cudaMemsetAsync(dm, 0, mb, c->st));
    if (total) YB_CUDA(cudaMemcpyAsync(d_allowed, allowed_rowids, (size_t)total * 8, cudaMemcpyHostToDevice, c->st));
    YB_CUDA(cudaMemcpyAsync(d_offs, allowed_offsets, (size_t)(nq + 1) * 8, cudaMemcpyHostToDevice, c->st));
    dim3 grid(64, nq);
    build_mask_kernel<<<grid, 256, 0, c->st>>>(d_allowed, d_offs, nq, c->rowids.as<int64_t>(), c->n, dm, mask_ld);
    *out_mask = dm;
    *out_mask_ld = mask_ld;
    return YAMS_OK;
}

// candidate sets as ascending device lists for the direct path (gather_score_kernel); they live in c->mask until the scan is done
static yams_status_t upload_direct_lists(yams_b200_corpus* c, uint32_t nq, const int64_t* allowed_rowids, const uint64_t* allowed_offsets,
                                         DirectLists* lists) {
    yams_status_t rc;
    const uint64_t total = allowed_offsets[nq];
    if ((rc = c->mask.reserve((size_t)total * 8 + (size_t)(nq + 1) * 8 + 64)) != YAMS_OK) return rc;
    int64_t* d_allowed = c->mask.as<int64_t>();
    uint64_t* d_offs = reinterpret_cast<uint64_t*>(d_allowed + total);
    if (total) YB_CUDA(cudaMemcpyAsync(d_allowed, allowed_rowids, (size_t)total * 8, cudaMemcpyHostToDevice, c->st));
    YB_CUDA(cudaMemcpyAsync(d_offs, allowed_offsets, (size_t)(nq + 1) * 8, cudaMemcpyHostToDevice, c->st));
    lists->d_allowed = d_allowed;
    lists->d_offsets = d_offs;
    lists->total = total;
    return YAMS_OK;
}

static yams_status_t enqueue_status_readback(yams_b200_corpus* c, uint32_t nq) {
    YB_CUDA(cudaMemcpyAsync(c->h_pin.p, c->status.p, sizeof(ScanStatus) + (size_t)nq * 4, cudaMemcpyDeviceToHost, c->st));
    return YAMS_OK;
}

// Enqueues search p on the queries at q_src (a semantic-graph batch: on its sources): their preparation, the candidate sets
// (host allowed_rowids / allowed_offsets, nullable) as p's device lists or mask, the scan and the read-back of its status
// block.  No host synchronisation.
static yams_status_t enqueue_search(yams_b200_corpus* c, ScanPlan& p, const float* q_src, bool src_is_device, const int64_t* allowed_rowids,
                                    const uint64_t* allowed_offsets) {
    yams_status_t rc;
    if ((rc = p.graph ? prepare_sources(c, p) : prepare_queries(c, q_src, src_is_device, p.nq)) != YAMS_OK) return rc;
    YB_CUDA(cudaEventRecord(c->ev[0], c->st));
    if (p.direct) rc = upload_direct_lists(c, p.nq, allowed_rowids, allowed_offsets, &p.lists);
    else if (allowed_offsets && c->n) rc = upload_mask(c, p.nq, allowed_rowids, allowed_offsets, &p.d_mask, &p.mask_ld);
    if (rc != YAMS_OK) return rc;
    if ((rc = scan_enqueue(c, p)) != YAMS_OK) return rc;
    YB_CUDA(cudaEventRecord(c->ev[2], c->st));
    return enqueue_status_readback(c, p.nq);
}

// After the stream of search p has been synchronised: its status block (pinned copy) -> an invalid query is an error, the
// queries the certificate rejected (*out_resolved of them) are answered by the exhaustive levels, patching p.out in place.
// allowed_rowids / allowed_offsets: the host candidate sets of a direct-path search.
static yams_status_t finish_search(yams_b200_corpus* c, ScanPlan& p, const int64_t* allowed_rowids, const uint64_t* allowed_offsets,
                                   uint32_t* out_resolved) {
    const ScanStatus* hs = c->h_pin.as<ScanStatus>();
    const uint32_t n_bad = std::min(hs->n_bad, p.nq);
    time_scan_events(c);
    c->last_ms[6] = c->last_ms[7] = 0.f;
    *out_resolved = 0;
    YB_ARG(hs->n_invalid == 0, "exact vector search requires a finite, non-zero query embedding");
    if (n_bad == 0) return YAMS_OK;
    std::vector<uint32_t> bad(reinterpret_cast<const uint32_t*>(hs + 1), reinterpret_cast<const uint32_t*>(hs + 1) + n_bad);
    std::sort(bad.begin(), bad.end());
    yams_status_t rc;
    if (p.direct) {
        // The direct path scored the listed rows without a bit mask, but the exhaustive levels score every row: they need the
        // candidate sets as a mask.  The scan is finished, so its lists in c->mask may be overwritten.
        p.direct = false;
        if ((rc = upload_mask(c, p.nq, allowed_rowids, allowed_offsets, &p.d_mask, &p.mask_ld)) != YAMS_OK) return rc;
    }
    *out_resolved = n_bad;
    c->last_ms[6] = (float)n_bad;
    uint32_t full = 0;
    rc = resolve_uncertain(c, p, bad.data(), n_bad, &full);
    c->last_ms[7] = (float)full;   // queries answered by the full exact pass (level 2)
    return rc;
}

}  // extern "C"

void yb::settle_pending(Corpus* c) {
    if (!c->pending.active) return;
    c->pending.active = false;
    uint32_t resolved = 0;
    yams_status_t rc = YAMS_ERR_INTERNAL;
    const cudaError_t e = cudaStreamSynchronize(c->st);
    if (e == cudaSuccess) rc = finish_search(static_cast<yams_b200_corpus*>(c), c->pending.plan, nullptr, nullptr, &resolved);
    else set_last_error("cudaStreamSynchronize failed: %s", cudaGetErrorString(e));
    c->pending.settled = true;
    c->pending.status = rc;
    c->pending.resolved = resolved;
    c->pending.error = rc == YAMS_OK ? "" : last_error();
}

extern "C" {

// the blocking paths: prepare the queries and reject an invalid one before any search work is enqueued
static yams_status_t prepare_valid_queries(yams_b200_corpus* c, const float* queries, uint32_t nq) {
    yams_status_t rc;
    if ((rc = prepare_queries(c, queries, false, nq)) != YAMS_OK) return rc;
    if ((rc = enqueue_status_readback(c, 0)) != YAMS_OK) return rc;
    YB_CUDA(cudaStreamSynchronize(c->st));
    YB_ARG(c->h_pin.as<ScanStatus>()->n_invalid == 0,
           "exact vector search requires a finite, non-zero query embedding");   // InvalidArgument for a bad query (:4127)
    return YAMS_OK;
}

yams_status_t yams_b200_search(yams_b200_corpus* c, const float* queries, uint32_t nq, uint32_t k, float threshold,
                               const int64_t* allowed_rowids, const uint64_t* allowed_offsets, int64_t* out_rowids,
                               float* out_scores, uint32_t* out_counts, uint64_t* out_flags) {
    YB_TRY
    YB_ARG(c, "corpus is null");
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_BIND(c);
    settle_pending(c);
    if (nq == 0) return YAMS_OK;
    YB_ARG(queries && out_counts, "null argument");
    YB_ARG(!allowed_rowids || allowed_offsets, "allowed_offsets missing");
    YB_ARG(!allowed_offsets || allowed_rowids || allowed_offsets[nq] == 0, "allowed_rowids missing");
    for (uint32_t q = 0; q < nq; ++q) out_counts[q] = 0;
    if (out_flags) for (uint32_t q = 0; q < nq; ++q) out_flags[q] = 0;
    // the reference looks at k before it validates the query (sqlite_vec_backend.cpp:4123-4130: k == 0 returns
    // empty first): mirror that order
    if (k == 0) return YAMS_OK;
    YB_ARG(out_rowids && out_scores, "null output");
    YB_ARG(k <= kMaxK, "k > 3072 is not supported by the fused top-k path (page larger requests)");
    YB_ARG(nq <= 65535, "at most 65535 queries per call (split larger batches)");   // per-query grid dimensions
    YB_ARG(!allowed_offsets || c->metric == YAMS_B200_COSINE, "candidate sets are only supported for the cosine metric");
    yams_status_t rc;
    ScanPlan plan;
    plan.nq = nq; plan.k = k; plan.threshold = threshold;
    if ((rc = reserve_results(c->dout, nq, k, &plan.out)) != YAMS_OK) return rc;
    if (allowed_offsets && c->n) {
        // small ascending lists: score the listed rows directly instead of passing over the corpus.  Break-even
        // (DESIGN.md §4.4): a corpus pass costs ~max(1, nq/400) row reads per row, a gathered row about two.
        const uint64_t total = allowed_offsets[nq];
        plan.direct = total <= std::max<uint64_t>(c->n / 2, c->n / 400 * nq) && total < (1ull << 31);
        for (uint32_t q = 0; q < nq && plan.direct; ++q) {
            uint64_t lo = allowed_offsets[q], hi = allowed_offsets[q + 1];
            plan.direct = hi >= lo && hi - lo < 0xFFFFFFFFull;
            for (uint64_t i = lo + 1; i < hi && plan.direct; ++i) plan.direct = allowed_rowids[i - 1] <= allowed_rowids[i];
            if (plan.direct) plan.lists.max_len = std::max<uint32_t>(plan.lists.max_len, (uint32_t)(hi - lo));
        }
    }
    if ((rc = enqueue_search(c, plan, queries, false, allowed_rowids, allowed_offsets)) != YAMS_OK) return rc;
    const DeviceResults& r = plan.out;
    if ((rc = copy_results(r, nq, k, out_rowids, out_scores, out_counts, out_flags, c->st)) != YAMS_OK) return rc;
    uint32_t resolved = 0;
    if ((rc = finish_search(c, plan, allowed_rowids, allowed_offsets, &resolved)) != YAMS_OK) {
        for (uint32_t q = 0; q < nq; ++q) out_counts[q] = 0;
        return rc;
    }
    if (resolved) return copy_results(r, nq, k, out_rowids, out_scores, out_counts, out_flags, c->st);
    return YAMS_OK;
    YB_CATCH
}

// The full exact pass (level 2 of the fallback chain) for EVERY query: the reference's own loop evaluated for all rows,
// no stage 1, no thresholds, no certificate needed.  It is what bench.py and the tests check the fast path against at
// sizes the CPU oracle cannot reach; ~3 ms per query per 10 M rows.
yams_status_t yams_b200_search_exhaustive(yams_b200_corpus* c, const float* queries, uint32_t nq, uint32_t k, float threshold,
                                          int64_t* out_rowids, float* out_scores, uint32_t* out_counts, uint64_t* out_flags) {
    YB_TRY
    YB_ARG(c, "corpus is null");
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_BIND(c);
    settle_pending(c);
    if (nq == 0) return YAMS_OK;
    YB_ARG(queries && out_counts && out_rowids && out_scores, "null argument");
    YB_ARG(k > 0 && k <= kMaxK, "k must be in 1..3072");
    YB_ARG(nq <= 65535, "at most 65535 queries per call");
    yams_status_t rc;
    if ((rc = prepare_valid_queries(c, queries, nq)) != YAMS_OK) return rc;
    ScanPlan plan;
    plan.nq = nq; plan.k = k; plan.threshold = threshold;
    if ((rc = reserve_results(c->dout, nq, k, &plan.out)) != YAMS_OK) return rc;
    for (uint32_t q = 0; q < nq; ++q)
        if ((rc = exact_all_rows(c, plan, q)) != YAMS_OK) return rc;
    return copy_results(plan.out, nq, k, out_rowids, out_scores, out_counts, out_flags, c->st);
    YB_CATCH
}

yams_status_t yams_b200_search_all_matching(yams_b200_corpus* c, const float* query, float threshold,
                                            const int64_t* allowed_rowids, uint64_t n_allowed, int64_t* out_rowids,
                                            float* out_scores, uint64_t* out_count) {
    YB_TRY
    YB_ARG(c && query && out_count, "null argument");
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_BIND(c);
    settle_pending(c);
    *out_count = 0;
    YB_ARG(c->metric == YAMS_B200_COSINE, "all-matching selection is defined for the cosine scan");
    // the reference gathers the candidate rowids into a set (:4412-4448): duplicates count once
    std::vector<int64_t> uniq;
    if (allowed_rowids) {
        bool ascending = true;
        for (uint64_t i = 1; i < n_allowed && ascending; ++i) ascending = allowed_rowids[i - 1] < allowed_rowids[i];
        if (!ascending) {
            uniq.assign(allowed_rowids, allowed_rowids + n_allowed);
            std::sort(uniq.begin(), uniq.end());
            uniq.erase(std::unique(uniq.begin(), uniq.end()), uniq.end());
            allowed_rowids = uniq.data();
            n_allowed = uniq.size();
        }
    }
    const uint64_t m = allowed_rowids ? n_allowed : c->n;
    yams_status_t rc;
    if ((rc = prepare_valid_queries(c, query, 1)) != YAMS_OK) return rc;
    if (m == 0 || c->n == 0) return YAMS_OK;
    YB_ARG(out_rowids && out_scores, "null output");
    YB_ARG(m < (1ull << 31), "candidate set too large");
    cudaStream_t st = c->st;
    const uint64_t np2 = pow2_at_least(m);
    // dense: the sorted keys, then the unpacked rowids and scores
    if ((rc = c->dense.reserve((size_t)np2 * 8 + (size_t)m * 12 + 64)) != YAMS_OK) return rc;
    uint64_t* d_keys = c->dense.as<uint64_t>();
    int64_t* d_or = reinterpret_cast<int64_t*>(d_keys + np2);
    float* d_os = reinterpret_cast<float*>(d_or + m);
    int64_t* d_allowed = nullptr;
    if (allowed_rowids) {
        if ((rc = c->mask.reserve((size_t)m * 8 + 64)) != YAMS_OK) return rc;
        d_allowed = c->mask.as<int64_t>();
        YB_CUDA(cudaMemcpyAsync(d_allowed, allowed_rowids, (size_t)m * 8, cudaMemcpyHostToDevice, st));
    }
    if ((rc = exact_sorted_keys(c, 0, m, d_allowed, threshold, nullptr, 0)) != YAMS_OK) return rc;
    if ((rc = c->tau.reserve(8)) != YAMS_OK) return rc;
    unsigned long long* d_cnt = reinterpret_cast<unsigned long long*>(c->tau.p);
    YB_CUDA(cudaMemsetAsync(d_cnt, 0, 8, st));
    count_nonzero_keys(d_keys, np2, d_cnt, st);
    unsigned long long h_cnt = 0;
    YB_CUDA(cudaMemcpyAsync(&h_cnt, d_cnt, 8, cudaMemcpyDeviceToHost, st));
    YB_CUDA(cudaStreamSynchronize(st));
    if (h_cnt) {
        unpack_keys(d_keys, h_cnt, c->rowids.as<int64_t>(), false, d_or, d_os, st);
        YB_CUDA(cudaMemcpyAsync(out_rowids, d_or, (size_t)h_cnt * 8, cudaMemcpyDeviceToHost, st));
        YB_CUDA(cudaMemcpyAsync(out_scores, d_os, (size_t)h_cnt * 4, cudaMemcpyDeviceToHost, st));
        YB_CUDA(cudaStreamSynchronize(st));
    }
    *out_count = h_cnt;
    return YAMS_OK;
    YB_CATCH
}

// The semantic graph's rows (GraphRows): its scales and statistics over its own row set, one row_stats_kernel pass with the
// reference's inv > 0 rule, in c->graph; *h_inv = the scales on the host (the valid sources), *h_rowids = the corpus rowids.
// g->src_row has room for kGraphBatch sources.
static yams_status_t graph_rows(yams_b200_corpus* c, GraphRows* g, std::vector<float>* h_inv, std::vector<int64_t>* h_rowids) {
    yams_status_t rc;
    const uint64_t n = c->n;
    if ((rc = c->graph.reserve((size_t)n * 4 + 16 + (size_t)kGraphBatch * 4 + 64)) != YAMS_OK) return rc;
    float* inv = c->graph.as<float>();
    float* stats = inv + n;
    YB_CUDA(cudaMemsetAsync(stats, 0, 16, c->st));
    if (n) row_stats_kernel<<<(unsigned)((n + 127) / 128), 128, 0, c->st>>>(c->rows.p, c->dtype, c->dim, 0, n, inv, YAMS_B200_COSINE, stats, 0.0);
    YB_CUDA(cudaGetLastError());
    float h_stats[4];
    h_inv->resize(n);
    h_rowids->resize(n);
    YB_CUDA(cudaMemcpyAsync(h_stats, stats, 16, cudaMemcpyDeviceToHost, c->st));
    YB_CUDA(cudaMemcpyAsync(h_inv->data(), inv, (size_t)n * 4, cudaMemcpyDeviceToHost, c->st));
    YB_CUDA(cudaMemcpyAsync(h_rowids->data(), c->rowids.p, (size_t)n * 8, cudaMemcpyDeviceToHost, c->st));
    YB_CUDA(cudaStreamSynchronize(c->st));
    g->inv = inv;
    g->r_max = h_stats[0]; g->dr_abs_max = h_stats[1]; g->dr_rel_max = h_stats[2]; g->inv_max = h_stats[3];
    g->uf = (float)((c->dim + 4.0) * 0x1p-126 * (double)g->inv_max);   // +inf with a row whose scale is +inf
    g->src_row = reinterpret_cast<const uint32_t*>(stats + 4);
    return YAMS_OK;
}

yams_status_t yams_b200_semantic_neighbors(yams_b200_corpus* c, const int64_t* source_rowids, uint64_t n_sources, uint32_t k,
                                           float threshold, int64_t* out_rowids, float* out_sims, uint32_t* out_counts,
                                           uint64_t* out_flags) {
    YB_TRY
    YB_ARG(c, "corpus is null");
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_BIND(c);
    settle_pending(c);
    YB_ARG(c->metric == YAMS_B200_COSINE, "the semantic graph needs a cosine corpus");
    YB_ARG(source_rowids || n_sources == c->n, "without source_rowids, n_sources must equal the corpus size");
    YB_ARG(k <= kMaxK, "k > 3072 is not supported by the fused top-k path");
    YB_ARG(threshold == threshold, "threshold is NaN");
    if (n_sources == 0) return YAMS_OK;
    YB_ARG(out_counts, "null argument");
    if (source_rowids)
        for (uint64_t i = 1; i < n_sources; ++i) YB_ARG(source_rowids[i - 1] < source_rowids[i], "source_rowids must be strictly ascending");
    for (uint64_t i = 0; i < n_sources; ++i) out_counts[i] = 0;
    if (out_flags) for (uint64_t i = 0; i < n_sources; ++i) out_flags[i] = 0;
    if (k == 0) return YAMS_OK;
    YB_ARG(out_rowids && out_sims, "null output");
    if (out_flags) for (uint64_t i = 0; i < n_sources; ++i) out_flags[i] = YAMS_B200_FLAG_NOT_A_SOURCE;   // until answered
    for (uint64_t i = 0; i < n_sources * k; ++i) { out_rowids[i] = -1; out_sims[i] = 0.f; }
    yams_status_t rc;
    GraphRows g;
    std::vector<float> h_inv;
    std::vector<int64_t> h_rowids;
    if ((rc = graph_rows(c, &g, &h_inv, &h_rowids)) != YAMS_OK) return rc;
    // the valid sources: their corpus rows and output slots (unknown rowids and rows the graph does not take keep count 0)
    std::vector<uint32_t> src_row;
    std::vector<uint64_t> slot;
    for (uint64_t i = 0, r = 0; i < n_sources; ++i) {
        if (source_rowids) {
            while (r < c->n && h_rowids[r] < source_rowids[i]) ++r;
            if (r == c->n || h_rowids[r] != source_rowids[i]) continue;
        } else {
            r = i;
        }
        if (h_inv[r] > 0.f) { src_row.push_back((uint32_t)r); slot.push_back(i); }
    }
    const uint64_t nv = src_row.size();
    if (nv == 0) return YAMS_OK;
    DeviceResults all;
    if ((rc = reserve_results(c->dout, (uint32_t)nv, k, &all)) != YAMS_OK) return rc;   // nv <= rows < 2^32
    for (uint64_t b0 = 0; b0 < nv; b0 += kGraphBatch) {
        const uint32_t nb = (uint32_t)std::min<uint64_t>(kGraphBatch, nv - b0);
        YB_CUDA(cudaMemcpyAsync(const_cast<uint32_t*>(g.src_row), src_row.data() + b0, (size_t)nb * 4, cudaMemcpyHostToDevice, c->st));
        ScanPlan p;
        p.nq = nb; p.k = k; p.threshold = threshold; p.graph = &g;
        p.out.rowids = all.rowids + b0 * k; p.out.flags = all.flags + b0;
        p.out.scores = all.scores + b0 * k; p.out.counts = all.counts + b0;
        if ((rc = enqueue_search(c, p, nullptr, false, nullptr, nullptr)) != YAMS_OK) return rc;
        YB_CUDA(cudaStreamSynchronize(c->st));
        uint32_t resolved = 0;
        if ((rc = finish_search(c, p, nullptr, nullptr, &resolved)) != YAMS_OK) return rc;
        if (threshold <= 0.f)
            restore_zero_signs_kernel<<<(unsigned)(((uint64_t)nb * k + 255) / 256), 256, 0, c->st>>>(
                c->rows.p, c->dtype, c->dim, c->q32.as<float>(), g, c->rowids.as<int64_t>(), c->n, p.out, nb, k);
        YB_CUDA(cudaGetLastError());
    }
    std::vector<int64_t> rid(nv * k);
    std::vector<float> sim(nv * k);
    std::vector<uint32_t> cnt(nv);
    std::vector<uint64_t> flg(nv);
    if ((rc = copy_results(all, (uint32_t)nv, k, rid.data(), sim.data(), cnt.data(), flg.data(), c->st)) != YAMS_OK) return rc;
    for (uint64_t i = 0; i < nv; ++i) {
        const uint64_t s = slot[i];
        out_counts[s] = cnt[i];
        if (out_flags) out_flags[s] = flg[i];
        for (uint32_t j = 0; j < cnt[i]; ++j) {
            out_rowids[s * k + j] = rid[i * k + j];
            out_sims[s * k + j] = sim[i * k + j];
        }
    }
    return YAMS_OK;
    YB_CATCH
}

yams_status_t yams_b200_debug_semantic_stage1(yams_b200_corpus* c, const int64_t* source_rowids, uint32_t n_sources, int engine,
                                              float* out_scores, float* out_eps) {
    YB_TRY
    YB_ARG(c && source_rowids && out_scores && out_eps && n_sources > 0 && n_sources <= kGraphBatch, "bad argument");
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_ARG(c->metric == YAMS_B200_COSINE && c->n > 0, "needs a non-empty cosine corpus");
    yams_status_t rc;
    YB_BIND(c);
    settle_pending(c);
    GraphRows g;
    std::vector<float> h_inv;
    std::vector<int64_t> h_rowids;
    if ((rc = graph_rows(c, &g, &h_inv, &h_rowids)) != YAMS_OK) return rc;
    std::vector<uint32_t> src_row(n_sources);
    for (uint32_t i = 0; i < n_sources; ++i) {
        const auto it = std::lower_bound(h_rowids.begin(), h_rowids.end(), source_rowids[i]);
        YB_ARG(it != h_rowids.end() && *it == source_rowids[i] && h_inv[it - h_rowids.begin()] > 0.f, "every source must be a taken row");
        src_row[i] = (uint32_t)(it - h_rowids.begin());
    }
    YB_CUDA(cudaMemcpyAsync(const_cast<uint32_t*>(g.src_row), src_row.data(), (size_t)n_sources * 4, cudaMemcpyHostToDevice, c->st));
    ScanPlan p;
    p.nq = n_sources; p.graph = &g;
    if ((rc = prepare_sources(c, p)) != YAMS_OK) return rc;
    if ((rc = c->dense.reserve((size_t)n_sources * c->n * 4)) != YAMS_OK) return rc;
    if ((rc = c->eps.reserve((size_t)n_sources * 4)) != YAMS_OK) return rc;
    Stage1Args a{};
    fill_stage1_common(c, a, n_sources, &g);
    a.row_start = 0; a.row_stride = 1; a.nrows = c->n;
    a.out_scores = c->dense.as<float>(); a.ld = c->n;
    Stage1Engine s1{c, engine == 1, false};
    if ((rc = s1.run(a, false)) != YAMS_OK) return rc;
    s1.launch_eps(n_sources);
    YB_CUDA(cudaMemcpyAsync(out_scores, c->dense.p, (size_t)n_sources * c->n * 4, cudaMemcpyDeviceToHost, c->st));
    YB_CUDA(cudaMemcpyAsync(out_eps, c->eps.p, (size_t)n_sources * 4, cudaMemcpyDeviceToHost, c->st));
    YB_CUDA(cudaStreamSynchronize(c->st));
    for (uint32_t i = 0; i < n_sources; ++i) out_eps[i] += graph_eps(h_inv[src_row[i]], g.uf);   // as final_kernel adds it
    return YAMS_OK;
    YB_CATCH
}

yams_status_t yams_b200_search_device(yams_b200_corpus* c, const float* d_queries, uint32_t nq, uint32_t k, float threshold,
                                      int64_t* d_out_rowids, float* d_out_scores) {
    YB_TRY
    YB_ARG(c && d_queries && d_out_rowids && d_out_scores, "null argument");
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_BIND(c);
    YB_ARG(k > 0 && k <= 768, "k must be in 1..768");
    YB_ARG(nq <= 65535, "at most 65535 queries per call (split larger batches)");
    if (nq == 0) return YAMS_OK;
    // supersedes a pending search without waiting for it (a pipelined caller enqueues its next batch before the last is done)
    c->pending.active = c->pending.settled = false;
    ScanPlan plan;
    plan.nq = nq; plan.k = k; plan.threshold = threshold;
    plan.out.rowids = d_out_rowids; plan.out.scores = d_out_scores;
    yams_status_t rc = enqueue_search(c, plan, d_queries, true, nullptr, nullptr);
    if (rc != YAMS_OK) return rc;
    c->pending.plan = plan;
    c->pending.active = true;
    return YAMS_OK;
    YB_CATCH
}

yams_status_t yams_b200_search_device_finish(yams_b200_corpus* c, uint32_t* out_resolved) {
    YB_TRY
    YB_ARG(c, "corpus is null");
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_BIND(c);
    if (out_resolved) *out_resolved = 0;
    settle_pending(c);
    if (!c->pending.settled) return YAMS_OK;
    c->pending.settled = false;
    if (out_resolved) *out_resolved = c->pending.resolved;
    if (c->pending.status != YAMS_OK) set_last_error("%s", c->pending.error.c_str());
    return c->pending.status;
    YB_CATCH
}

static yams_status_t merge_launch(yams_b200_corpus* c, const int64_t* d_rowids, const float* d_scores, uint64_t rank_stride_r,
                                  uint64_t rank_stride_s, uint32_t nranks, uint32_t nq, uint32_t k, int64_t* d_out_rowids,
                                  float* d_out_scores, uint32_t* d_out_counts, cudaStream_t st) {
    YB_ARG(nranks >= 1 && k >= 1, "bad shape");
    const uint32_t np2 = pow2_at_least(nranks * k);
    YB_ARG(np2 <= 4096, "nranks * k too large to merge in one CTA");
    size_t smem = (((size_t)np2 * 4 + 7) & ~(size_t)7) + (size_t)np2 * 8;
    merge_partials_kernel<<<nq, SEL_THREADS, smem, st>>>(d_rowids, d_scores, rank_stride_r, rank_stride_s, nranks, nq, k,
                                                         c->metric == YAMS_B200_L2, d_out_rowids, d_out_scores, d_out_counts);
    YB_CUDA(cudaGetLastError());
    return YAMS_OK;
}

yams_status_t yams_b200_merge_partials_device(yams_b200_corpus* c, const int64_t* d_rowids, const float* d_scores,
                                              uint32_t nranks, uint32_t nq, uint32_t k, int64_t* d_out_rowids,
                                              float* d_out_scores, uint32_t* d_out_counts) {
    YB_TRY
    YB_ARG(c && d_rowids && d_scores && d_out_rowids && d_out_scores, "null argument");
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_BIND(c);
    return merge_launch(c, d_rowids, d_scores, (uint64_t)nq * k, (uint64_t)nq * k, nranks, nq, k, d_out_rowids, d_out_scores,
                        d_out_counts, c->st);
    YB_CATCH
}

yams_status_t yams_b200_merge_packed_device(yams_b200_corpus* c, const void* d_packed, uint32_t nranks, uint32_t nq, uint32_t k,
                                            int64_t* d_out_rowids, float* d_out_scores, uint32_t* d_out_counts, void* stream) {
    YB_ARG(c && d_packed && d_out_rowids && d_out_scores, "null argument");
    YB_BIND(c);
    // one rank's record: [nq*k int64 rowids][nq*k float scores] = 12 * nq * k bytes
    const uint8_t* base = static_cast<const uint8_t*>(d_packed);
    const uint64_t rec = (uint64_t)nq * k * 12;
    YB_ARG(rec % 8 == 0, "nq * k must be even for the packed layout");
    return merge_launch(c, reinterpret_cast<const int64_t*>(base), reinterpret_cast<const float*>(base + (uint64_t)nq * k * 8),
                        rec / 8, rec / 4, nranks, nq, k, d_out_rowids, d_out_scores, d_out_counts,
                        stream ? static_cast<cudaStream_t>(stream) : c->st);
}

yams_status_t yams_b200_search_last_timings(yams_b200_corpus* c, float out_ms[8]) {
    YB_ARG(c && out_ms, "null argument");
    // a search_device whose work is done reports its device times before (or without) its finish
    if (c->pending.active && cudaEventQuery(c->ev[2]) == cudaSuccess) time_scan_events(c);
    for (int i = 0; i < 8; ++i) out_ms[i] = c->last_ms[i];
    return YAMS_OK;
}

// diagnostics: dense stage-1 scores of rows [row_start + i*row_stride, i < nrows) against the queries with the
// chosen engine (0 cuda-core, 1 wgmma) -> out[q * nrows + i] (HOST). Used by the tests to compare engines.
yams_status_t yams_b200_debug_stage1_scores(yams_b200_corpus* c, const float* queries, uint32_t nq, int engine,
                                            uint64_t row_start, uint64_t row_stride, uint64_t nrows, float* out) {
    YB_TRY
    YB_ARG(c && queries && out && nq > 0 && nrows > 0 && row_stride > 0, "bad argument");
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_ARG(row_start + (nrows - 1) * row_stride < c->n, "rows out of range");
    yams_status_t rc;
    YB_BIND(c);
    settle_pending(c);
    if ((rc = prepare_queries(c, queries, false, nq)) != YAMS_OK) return rc;
    if ((rc = c->dense.reserve((size_t)nq * nrows * 4)) != YAMS_OK) return rc;
    if ((rc = c->eps.reserve((size_t)nq * 4)) != YAMS_OK) return rc;
    YB_CUDA(cudaMemsetAsync(c->dense.p, 0xFF, (size_t)nq * nrows * 4, c->st));
    Stage1Args a{};
    fill_stage1_common(c, a, nq);
    a.row_start = row_start; a.row_stride = row_stride; a.nrows = nrows;
    a.out_scores = c->dense.as<float>(); a.ld = nrows;
    Stage1Engine s1{c, engine == 1, false};
    if ((rc = s1.run(a, false)) != YAMS_OK) return rc;
    s1.launch_eps(nq);
    YB_CUDA(cudaMemcpyAsync(out, c->dense.p, (size_t)nq * nrows * 4, cudaMemcpyDeviceToHost, c->st));
    YB_CUDA(cudaStreamSynchronize(c->st));
    return YAMS_OK;
    YB_CATCH
}

// the filter-mode set-up of the stage-1 diagnostics: the queries prepared, tau[nq] uploaded, the list counters zeroed and `a`
// filled for lists of cap entries (the caller sets the rows)
static yams_status_t debug_filter_setup(yams_b200_corpus* c, const float* queries, uint32_t nq, const float* tau, uint32_t cap,
                                        Stage1Args& a) {
    yams_status_t rc;
    if ((rc = prepare_queries(c, queries, false, nq)) != YAMS_OK) return rc;
    if ((rc = c->eps.reserve((size_t)nq * 4)) != YAMS_OK) return rc;
    if ((rc = c->tau.reserve((size_t)nq * 4)) != YAMS_OK) return rc;
    if ((rc = c->cands.reserve((size_t)nq * cap * sizeof(Cand) + 8)) != YAMS_OK) return rc;
    YB_CUDA(cudaMemcpyAsync(c->tau.p, tau, (size_t)nq * 4, cudaMemcpyHostToDevice, c->st));
    YB_CUDA(cudaMemsetAsync(c->counts.p, 0, (size_t)nq * 4, c->st));
    fill_stage1_common(c, a, nq);
    a.tau = c->tau.as<float>(); a.cands = c->cands.as<Cand>(); a.cap = cap; a.counts = c->counts.as<uint32_t>();
    return YAMS_OK;
}

// diagnostics: the same rows and engines in FILTER mode -- the candidate lists the search builds from per-query thresholds
// (and candidate sets) -> out_counts[q] (raw, may exceed cap), out_cands[q * cap + j] = (float score, uint32 row) (HOST)
yams_status_t yams_b200_debug_stage1_candidates(yams_b200_corpus* c, const float* queries, uint32_t nq, int engine,
                                                uint64_t row_start, uint64_t row_stride, uint64_t nrows, const float* tau, uint32_t cap,
                                                const int64_t* allowed_rowids, const uint64_t* allowed_offsets, uint32_t* out_counts,
                                                void* out_cands) {
    YB_TRY
    YB_ARG(c && queries && tau && out_counts && (out_cands || cap == 0) && nq > 0 && nrows > 0 && row_stride > 0, "bad argument");
    YB_ARG(!allowed_rowids || allowed_offsets, "allowed_offsets missing");
    YB_ARG(!allowed_offsets || allowed_rowids || allowed_offsets[nq] == 0, "allowed_rowids missing");
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_ARG(row_start + (nrows - 1) * row_stride < c->n, "rows out of range");
    yams_status_t rc;
    YB_BIND(c);
    settle_pending(c);
    Stage1Args a{};
    if ((rc = debug_filter_setup(c, queries, nq, tau, cap, a)) != YAMS_OK) return rc;
    const size_t cb = (size_t)nq * cap * sizeof(Cand);
    YB_CUDA(cudaMemsetAsync(c->cands.p, 0xFF, cb, c->st));
    a.row_start = row_start; a.row_stride = row_stride; a.nrows = nrows;
    Stage1Engine s1{c, engine == 1, false};
    if (engine == 2) {
        // the direct path's engine: every listed rowid is scored, tau and the row range do not apply
        YB_ARG(allowed_offsets && c->metric == YAMS_B200_COSINE, "engine 2 scores cosine candidate-set lists");
        for (uint32_t q = 0; q < nq; ++q) {
            YB_ARG(allowed_offsets[q + 1] >= allowed_offsets[q] && allowed_offsets[q + 1] - allowed_offsets[q] <= cap,
                   "a list is longer than cap");
            for (uint64_t i = allowed_offsets[q] + 1; i < allowed_offsets[q + 1]; ++i)
                YB_ARG(allowed_rowids[i - 1] <= allowed_rowids[i], "engine 2 takes ascending lists");
        }
        DirectLists lists;
        if ((rc = upload_direct_lists(c, nq, allowed_rowids, allowed_offsets, &lists)) != YAMS_OK) return rc;
        list_lengths_kernel<<<(nq + 255) / 256, 256, 0, c->st>>>(lists.d_offsets, nq, a.counts);
        rc = gather_scores(c, lists, nq, a.q32, a.qinv, a.cands, cap, c->st);
    } else {
        if (allowed_offsets && (rc = upload_mask(c, nq, allowed_rowids, allowed_offsets, &a.mask, &a.mask_ld)) != YAMS_OK) return rc;
        rc = s1.run(a, true);
    }
    if (rc != YAMS_OK) return rc;
    s1.launch_eps(nq);
    YB_CUDA(cudaMemcpyAsync(out_counts, c->counts.p, (size_t)nq * 4, cudaMemcpyDeviceToHost, c->st));
    if (cb) YB_CUDA(cudaMemcpyAsync(out_cands, c->cands.p, cb, cudaMemcpyDeviceToHost, c->st));
    YB_CUDA(cudaStreamSynchronize(c->st));
    return YAMS_OK;
    YB_CATCH
}

// diagnostics: one pass of the profiling instantiation of the wgmma scan in filter mode over every row (the search's corpus
// pass) -> per-CTA cycle counters, the launch's layout and its device time (HOST out), see include/yams_b200.h
yams_status_t yams_b200_debug_stage1_profile(yams_b200_corpus* c, const float* queries, uint32_t nq, const float* tau, uint32_t cap,
                                             uint32_t max_ctas, uint64_t* out_cycles, uint32_t* out_info, float* out_ms) {
    YB_TRY
    YB_ARG(c && queries && tau && out_cycles && out_info && out_ms && nq > 0, "bad argument");
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_ARG(c->n > 0, "empty corpus");
    yams_status_t rc;
    YB_BIND(c);
    settle_pending(c);
    Stage1Args a{};
    if ((rc = debug_filter_setup(c, queries, nq, tau, cap, a)) != YAMS_OK) return rc;
    const size_t pb = (size_t)c->dev->sm_count * 4 * sizeof(unsigned long long);
    if ((rc = c->dense.reserve(pb)) != YAMS_OK) return rc;
    YB_CUDA(cudaMemsetAsync(c->dense.p, 0, pb, c->st));
    a.row_start = 0; a.row_stride = 1; a.nrows = c->n;
    Stage1Engine s1{c, true, false};
    YB_CUDA(cudaEventRecord(c->ev_scan[0], c->st));
    if ((rc = s1.run(a, true, reinterpret_cast<unsigned long long*>(c->dense.p))) != YAMS_OK) return rc;
    YB_CUDA(cudaEventRecord(c->ev_scan[1], c->st));
    const uint32_t ctas = c->wg_launch[1];
    YB_ARG(ctas <= max_ctas, "max_ctas is below the launch's CTA count");
    YB_CUDA(cudaMemcpyAsync(out_cycles, c->dense.p, (size_t)ctas * 4 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->st));
    YB_CUDA(cudaStreamSynchronize(c->st));
    YB_CUDA(cudaEventElapsedTime(out_ms, c->ev_scan[0], c->ev_scan[1]));
    out_info[0] = c->wg_launch[0]; out_info[1] = c->wg_launch[1];
    return YAMS_OK;
    YB_CATCH
}

// diagnostics: the top-K selection (topk_select_kernel) on caller-supplied scores, see include/yams_b200.h
yams_status_t yams_b200_debug_select(yams_b200_corpus* c, uint32_t nq, const float* dense, uint64_t ld, uint64_t len, uint64_t row_start,
                                     uint64_t row_stride, uint32_t dense_shift, const void* cands, const uint32_t* counts, uint32_t cap,
                                     const float* tau, uint32_t K, int tau_only, float tau_margin, int fast_tau, void* out_sel,
                                     uint32_t* out_n, float* out_bound) {
    YB_TRY
    YB_ARG(c && nq > 0 && out_bound && (tau_only || (out_sel && out_n)), "bad argument");
    YB_ARG(dense ? (ld >= len && dense_shift < 4) : (counts && (cands || cap == 0)), "bad input");
    YB_ARG(tau_only || K <= SEL_MAXK, "K > 4096");
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_BIND(c);
    settle_pending(c);
    yams_status_t rc;
    cudaStream_t st = c->st;
    SelectIn in{};
    if (dense) {
        const size_t nb = (size_t)nq * ld * 4;
        if ((rc = c->dense.reserve(nb + 16)) != YAMS_OK) return rc;
        float* d = c->dense.as<float>() + dense_shift;    // the allocation is 256-byte aligned: dense_shift sets the alignment
        if (nb) YB_CUDA(cudaMemcpyAsync(d, dense, nb, cudaMemcpyHostToDevice, st));
        in.dense = d; in.ld = ld; in.dense_len = len; in.row_start = row_start; in.row_stride = row_stride;
    } else {
        const size_t cb = (size_t)nq * cap * sizeof(Cand);
        if ((rc = c->cands.reserve(cb + 8)) != YAMS_OK) return rc;
        if ((rc = c->counts.reserve((size_t)nq * 4)) != YAMS_OK) return rc;
        if (cb) YB_CUDA(cudaMemcpyAsync(c->cands.p, cands, cb, cudaMemcpyHostToDevice, st));
        YB_CUDA(cudaMemcpyAsync(c->counts.p, counts, (size_t)nq * 4, cudaMemcpyHostToDevice, st));
        in.cands = c->cands.as<Cand>(); in.counts = c->counts.as<uint32_t>(); in.cap = cap;
        if (tau) {
            if ((rc = c->tau.reserve((size_t)nq * 4)) != YAMS_OK) return rc;
            YB_CUDA(cudaMemcpyAsync(c->tau.p, tau, (size_t)nq * 4, cudaMemcpyHostToDevice, st));
            in.tau = c->tau.as<float>();
        }
    }
    in.tau_margin = tau_margin;
    in.fast_tau = fast_tau;
    if ((rc = c->bound.reserve((size_t)nq * 4)) != YAMS_OK) return rc;
    float* d_bound = c->bound.as<float>();
    if (tau_only) {
        topk_select_kernel<<<nq, SEL_THREADS, 0, st>>>(in, K, 1, d_bound, nullptr, nullptr, nullptr);
    } else {
        if ((rc = c->sel.reserve((size_t)nq * K * sizeof(Cand) + (size_t)nq * 4 + 8)) != YAMS_OK) return rc;
        Cand* d_sel = c->sel.as<Cand>();
        uint32_t* d_n = reinterpret_cast<uint32_t*>(d_sel + (size_t)nq * K);
        topk_select_kernel<<<nq, SEL_THREADS, 0, st>>>(in, K, 0, nullptr, d_sel, d_n, d_bound);
        if (K) YB_CUDA(cudaMemcpyAsync(out_sel, d_sel, (size_t)nq * K * sizeof(Cand), cudaMemcpyDeviceToHost, st));
        YB_CUDA(cudaMemcpyAsync(out_n, d_n, (size_t)nq * 4, cudaMemcpyDeviceToHost, st));
    }
    YB_CUDA(cudaGetLastError());
    YB_CUDA(cudaMemcpyAsync(out_bound, d_bound, (size_t)nq * 4, cudaMemcpyDeviceToHost, st));
    YB_CUDA(cudaStreamSynchronize(st));
    return YAMS_OK;
    YB_CATCH
}

// diagnostics: the final ordering and the exactness certificate (final_kernel) on caller-supplied exact scores, see
// include/yams_b200.h
yams_status_t yams_b200_debug_final(yams_b200_corpus* c, uint32_t nq, uint32_t Kp, uint32_t k, const void* exact, const uint32_t* ex_n,
                                    const float* bound, const float* eps, const double* qnorm, float threshold, int metric, int level,
                                    int64_t* out_rowids, float* out_scores, uint32_t* out_counts, uint64_t* out_flags,
                                    uint32_t* out_queued, uint32_t* out_n_queued) {
    YB_TRY
    YB_ARG(c && nq > 0 && Kp > 0 && Kp <= SEL_MAXK && k > 0 && k <= SEL_MAXK && exact && bound && eps && qnorm, "bad argument");
    YB_ARG(out_rowids && out_scores && out_counts && out_flags && out_queued && out_n_queued, "null output");
    YB_ARG(metric == YAMS_B200_COSINE || metric == YAMS_B200_L2, "unknown metric");
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_BIND(c);
    settle_pending(c);
    const Exact* ex = static_cast<const Exact*>(exact);
    for (uint32_t b = 0; b < nq; ++b) {   // entries final_kernel reads must index the rowid table
        const uint32_t m = ex_n ? std::min(ex_n[b], Kp) : Kp;
        for (uint32_t i = 0; i < m; ++i) {
            const Exact& e = ex[(size_t)b * Kp + i];
            YB_ARG(e.sim != e.sim || e.row < c->n, "row out of range");
        }
    }
    yams_status_t rc;
    cudaStream_t st = c->st;
    const size_t eb = (size_t)nq * Kp * sizeof(Exact);
    if ((rc = c->outbuf.reserve(eb + (size_t)nq * 4 + 8)) != YAMS_OK) return rc;
    if ((rc = c->bound.reserve((size_t)nq * 4)) != YAMS_OK) return rc;
    if ((rc = c->eps.reserve((size_t)nq * 4)) != YAMS_OK) return rc;
    if ((rc = c->qnorm.reserve((size_t)nq * 8)) != YAMS_OK) return rc;
    if ((rc = c->status.reserve(sizeof(ScanStatus) + (size_t)nq * 8)) != YAMS_OK) return rc;
    DeviceResults r;
    if ((rc = reserve_results(c->dout, nq, k, &r)) != YAMS_OK) return rc;
    Exact* d_ex = c->outbuf.as<Exact>();
    uint32_t* d_ex_n = reinterpret_cast<uint32_t*>(d_ex + (size_t)nq * Kp);
    YB_CUDA(cudaMemcpyAsync(d_ex, ex, eb, cudaMemcpyHostToDevice, st));
    if (ex_n) YB_CUDA(cudaMemcpyAsync(d_ex_n, ex_n, (size_t)nq * 4, cudaMemcpyHostToDevice, st));
    YB_CUDA(cudaMemcpyAsync(c->bound.p, bound, (size_t)nq * 4, cudaMemcpyHostToDevice, st));
    YB_CUDA(cudaMemcpyAsync(c->eps.p, eps, (size_t)nq * 4, cudaMemcpyHostToDevice, st));
    YB_CUDA(cudaMemcpyAsync(c->qnorm.p, qnorm, (size_t)nq * 8, cudaMemcpyHostToDevice, st));
    YB_CUDA(cudaMemsetAsync(c->status.p, 0, sizeof(ScanStatus) + (size_t)nq * 8, st));
    ScanPlan p;
    p.nq = nq; p.threshold = threshold;
    CertArgs cert = cert_args(c, p, c->bound.as<float>(), c->eps.as<float>(), level);
    cert.metric = metric;   // either result convention on any corpus
    launch_final(d_ex, ex_n ? d_ex_n : nullptr, Kp, k, c->rowids.as<int64_t>(), r, nq, nullptr, cert, st);
    YB_CUDA(cudaGetLastError());
    std::vector<uint32_t> h_status(sizeof(ScanStatus) / 4 + (size_t)nq * 2);
    YB_CUDA(cudaMemcpyAsync(h_status.data(), c->status.p, h_status.size() * 4, cudaMemcpyDeviceToHost, st));
    if ((rc = copy_results(r, nq, k, out_rowids, out_scores, out_counts, out_flags, c->st)) != YAMS_OK) return rc;
    const ScanStatus* hs = reinterpret_cast<const ScanStatus*>(h_status.data());
    const uint32_t nqd = std::min(level == 0 ? hs->n_bad : hs->n_bad2, nq);
    const uint32_t* list = h_status.data() + sizeof(ScanStatus) / 4 + (level == 0 ? 0 : nq);
    for (uint32_t i = 0; i < nqd; ++i) out_queued[i] = list[i];
    *out_n_queued = nqd;
    return YAMS_OK;
    YB_CATCH
}

// bench / test utility: n synthetic rows of the SURVEY.md §8d generator (bit-identical to oracle yo_gen_rows_f32) as fp32
// into a DEVICE buffer -- the query batches of bench.py are produced by the library itself, not by the checker
yams_status_t yams_b200_synth_rows_device(uint64_t seed, uint64_t first_row, uint64_t n, uint32_t dim, float* d_out) {
    YB_TRY
    YB_ARG(d_out && dim > 0, "bad argument");
    if (n == 0) return YAMS_OK;
    DeviceCtx* dev = nullptr;
    yams_status_t rc = ensure_device(&dev);
    if (rc != YAMS_OK) return rc;
    DevBuf inv;
    if ((rc = inv.reserve((size_t)n * 4)) != YAMS_OK) return rc;
    synth_rownorm_kernel<<<(unsigned)((n + 127) / 128), 128>>>(seed, first_row, n, dim, inv.as<float>());
    synth_fill_kernel<<<dev->sm_count * 16, 256>>>(seed, first_row, n, dim, inv.as<float>(), d_out, YAMS_B200_F32);
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) {
        set_last_error("synth_rows_device failed: %s", cudaGetErrorString(e));
        return YAMS_ERR_INTERNAL;
    }
    return YAMS_OK;
    YB_CATCH
}

// diagnostics: the per-query stage-1 error bound eps[q] (certificate input) computed by the last search /
// debug_stage1_scores call on this corpus
yams_status_t yams_b200_debug_last_eps(yams_b200_corpus* c, uint32_t nq, float* out) {
    YB_TRY
    YB_ARG(c && out && nq > 0, "bad argument");
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_BIND(c);
    YB_ARG(c->eps.cap >= (size_t)nq * 4, "no search with that many queries has run");
    YB_CUDA(cudaMemcpyAsync(out, c->eps.p, (size_t)nq * 4, cudaMemcpyDeviceToHost, c->st));
    YB_CUDA(cudaStreamSynchronize(c->st));
    return YAMS_OK;
    YB_CATCH
}

}  // extern "C"
