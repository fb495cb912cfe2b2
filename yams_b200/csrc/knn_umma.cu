// knn_umma.cu -- stage-1 scan engine on the Hopper tensor cores (wgmma + TMA + mbarrier), sm_90a.
//
// Same contract as the CUDA-core engine in knn.cu (Stage1Args): approximate cosine scores of corpus rows
// against a query batch with a fused epilogue (store, or per-query threshold filter -> candidate lists).
// The scan of `rows x dim` fp16 against `nq x dim` queries is a dense GEMM (tensor-bound for large query
// batches, HBM-bound for small ones), so it runs as a warp-specialised, persistent kernel, one CTA per SM:
//
//   warpgroup 0     TMA producer : cp.async.bulk.tensor 2D loads of a 128-row corpus tile (A, K-major, 128B swizzle)
//                                   and an N-query tile (B) per 128-byte K block into a multi-stage smem ring
//   warpgroups 1-2  consumers    : each owns 64 of the 128 rows; wgmma.mma_async m64nNk16 (fp16) / m64nNk8 (tf32)
//                                   accumulates fp32 in registers, then the epilogue scales by 1/|row|, compares
//                                   with the per-query threshold and appends survivors
//
// A CTA owns whole row tiles and runs every query tile against each: the corpus tile comes from HBM once and is
// re-read from L2 by the same SM; the next row tile is prefetched into L2 during the last query tile.
//
// Queries are pre-scaled by 1/|q| and rounded to fp16; the resulting ~1e-5 score error only affects which
// rows reach stage 2, where the survivors are re-scored exactly in fp64 (knn.cu).
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdlib.h>

#include <algorithm>

#include "knn.cuh"

namespace yb {

constexpr int UM_BLOCK_M = 128;
constexpr int UM_BLOCK_K_BYTES = 128;    // one swizzle row of K per stage: 64 fp16 or 32 fp32 (tf32) elements
constexpr int UM_MMAS_PER_KBLOCK = 4;    // 4 x 32 bytes of K: 4 x (K=16 fp16) or 4 x (K=8 tf32)
constexpr int UM_THREADS = 384;          // 3 warpgroups: TMA producer + 2 x (wgmma + epilogue)
constexpr uint32_t UM_A_STAGE = UM_BLOCK_M * UM_BLOCK_K_BYTES;   // 16 KiB
constexpr uint32_t UM_SMEM_LIMIT = 227 * 1024;                   // opt-in shared memory per block on sm_90
// query columns per threshold group of the epilogue's pre-filter: 32 for fp16; the whole tile for tf32, whose MMAs take twice
// as long (the finer groups measured no faster there)
constexpr int UM_TAU_GROUP = 32;
constexpr int UM_MAX_TAU_GROUPS = 4096 / UM_TAU_GROUP;
constexpr long long UM_WAIT_LIMIT_CYCLES = 4000000000ll;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
// the same load with an L2 eviction policy (createpolicy) for the lines it reads
__device__ __forceinline__ void tma_load_2d_hint(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1,
                                                 uint64_t policy) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], [%2], %5;"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "l"(policy)
        : "memory");
}
// pull a tile into L2 ahead of time (no shared-memory destination, no barrier)
__device__ __forceinline__ void tma_prefetch_2d(const CUtensorMap* map, int c0, int c1) {
    asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];"
                 ::"l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1) : "memory");
}

// K-major operand tile, 128-byte swizzle: rows of 128 B, 8-row groups 1024 B apart (SBO)
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr >> 4) & 0x3FFFu);   // start address, 16-byte units
    d |= (uint64_t)1 << 16;                        // leading byte offset (unused for swizzled K-major)
    d |= (uint64_t)(1024 >> 4) << 32;              // stride byte offset between 8-row core groups
    d |= (uint64_t)1 << 62;                        // SWIZZLE_128B
    return d;
}

// m64nNk16 (fp16) / m64nNk8 (tf32), both operands K-major in shared memory, fp32 accumulators in registers.
// Accumulator layout (per warpgroup): thread t = 32 w + l holds rows 16 w + l / 4 (+8) and, for j < N / 8, columns
// 8 j + 2 (l % 4) (+1): d[4 j + 0] = (row, col), d[4 j + 1] = (row, col + 1), d[4 j + 2] = (row + 8, col), d[4 j + 3] = (row + 8, col + 1).
#define WG_REGS32 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}"
#define WG_REGS128 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}"
#define WG_F8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
#define WG_ACC32 WG_F8(0), WG_F8(8), WG_F8(16), WG_F8(24)
#define WG_ACC128 WG_ACC32, WG_F8(32), WG_F8(40), WG_F8(48), WG_F8(56), WG_F8(64), WG_F8(72), WG_F8(80), WG_F8(88), WG_F8(96), \
                  WG_F8(104), WG_F8(112), WG_F8(120)

template <int N, bool TF32>
__device__ __forceinline__ void wgmma_tile(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
    if constexpr (N == 256) {
        if constexpr (TF32)
            asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
                         "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 " WG_REGS128 ", %128, %129, p, 1, 1;\n\t}"
                         : WG_ACC128 : "l"(da), "l"(db), "r"(scale_d));
        else
            asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
                         "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 " WG_REGS128 ", %128, %129, p, 1, 1, 0, 0;\n\t}"
                         : WG_ACC128 : "l"(da), "l"(db), "r"(scale_d));
    } else {
        static_assert(N == 64, "query tile of 64 or 256 columns");
        if constexpr (TF32)
            asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                         "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 " WG_REGS32 ", %32, %33, p, 1, 1;\n\t}"
                         : WG_ACC32 : "l"(da), "l"(db), "r"(scale_d));
        else
            asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                         "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " WG_REGS32 ", %32, %33, p, 1, 1, 0, 0;\n\t}"
                         : WG_ACC32 : "l"(da), "l"(db), "r"(scale_d));
    }
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ bool mbar_try(uint32_t addr, uint32_t parity) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
    return done != 0;
}
// fast path: one try_wait, no clock reads; the slow path keeps the "never hang the GPU" limit (checked every 1024 spins)
template <bool PROF>
__device__ __forceinline__ void mbar_wait_u(uint32_t addr, uint32_t parity, long long* waited) {
    if (PROF) {
        const long long t_begin = clock64();
        while (!mbar_try(addr, parity))
            if (clock64() - t_begin > UM_WAIT_LIMIT_CYCLES) __trap();
        *waited += clock64() - t_begin;
    } else {
        if (mbar_try(addr, parity)) return;
        long long t_begin = 0;
        uint32_t spins = 0;
        while (!mbar_try(addr, parity)) {
            if ((++spins & 1023u) == 0) {
                const long long now = clock64();
                if (t_begin == 0) t_begin = now;
                else if (now - t_begin > UM_WAIT_LIMIT_CYCLES) __trap();
            }
        }
    }
}
__device__ __forceinline__ void mbar_expect_tx_u(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive_u(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}

// inlined: a call from the filter epilogue would have to save the live accumulators around it
__device__ __forceinline__ void append_candidate(uint32_t* counts, Cand* cands, uint32_t cap, uint32_t q, uint32_t row, float sc) {
    uint32_t pos = atomicAdd(&counts[q], 1u);
    if (pos < cap) {
        Cand cd;
        cd.score = sc;
        cd.row = row;
        cands[(uint64_t)q * cap + pos] = cd;
    }
}

struct WgArgs {
    Stage1Args a;
    uint32_t nqt;         // query tiles of N columns
    uint32_t nrt;         // corpus row tiles of UM_BLOCK_M rows
    uint32_t kblocks;     // ceil(dim / block_k)
    uint32_t stages;
    unsigned long long* prof;   // PROF: per CTA {consumer full-barrier wait, producer empty-barrier wait, epilogue, total} cycles
};

template <bool FILTER, int N, bool TF32, bool PROF>
__global__ void __launch_bounds__(UM_THREADS, 1)
stage1_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, WgArgs u) {
    const long long t_start = PROF ? clock64() : 0;
    constexpr int TG = TF32 ? N : UM_TAU_GROUP;
    constexpr uint32_t B_STAGE = N * UM_BLOCK_K_BYTES;
    constexpr uint32_t STAGE = UM_A_STAGE + B_STAGE;
    extern __shared__ uint8_t smem_raw[];
    // 1024-byte alignment for the 128B-swizzled tiles
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)u.stages * STAGE);
    float* tmin_s = reinterpret_cast<float*>(bars + 2 * u.stages);   // smallest threshold of each group of 32 query columns
    float* tau_all = tmin_s + UM_MAX_TAU_GROUPS;                      // [nqt * N] thresholds (+inf past nq)
    const uint32_t tiles_u = smem_u32(smem);
    const uint32_t full_u = smem_u32(bars), empty_u = full_u + 8u * u.stages;

    const uint32_t wg = threadIdx.x >> 7;
    const uint32_t lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmB)) : "memory");
        for (uint32_t s = 0; s < u.stages; ++s) {
            mbar_init(&bars[s], 1);                // full: the producer's expect_tx arrive
            mbar_init(&bars[u.stages + s], 8);     // empty: one arrive per consumer warp
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    if (FILTER) {
        const uint32_t nqpad = u.nqt * N;
        for (uint32_t i = threadIdx.x; i < nqpad; i += UM_THREADS) tau_all[i] = i < u.a.nq ? __ldg(&u.a.tau[i]) : INFINITY;
        __syncthreads();
        for (uint32_t t = threadIdx.x; t < nqpad / TG; t += UM_THREADS) {
            float m = INFINITY;
            for (uint32_t c = 0; c < TG; ++c) m = fminf(m, tau_all[t * TG + c]);
            tmin_s[t] = m;
        }
    }
    __syncthreads();

    if (wg == 0) {
        // ===================== TMA producer =====================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (threadIdx.x == 0) {
            long long w_empty = 0;
            uint32_t s = 0, ph = 0;
            const int block_k = UM_BLOCK_K_BYTES / (TF32 ? 4 : 2);
            // A corpus tile is read from L2 once per query tile.  Its last read marks its lines evict-first: with every
            // CTA's current and prefetched next tile (~50 MB at C2) the L2 is full, and a dead tile should leave before a
            // live one is pushed out and fetched from HBM again.  The next tile is prefetched during the current tile's last
            // query tile, not its first: from the first on, it would share the L2 with the current tile for the whole tile.
            uint64_t last_use;
            asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(last_use));
            for (uint32_t rt = blockIdx.x; rt < u.nrt; rt += gridDim.x) {
                const int a_row = (int)(rt * UM_BLOCK_M);
                const int a_next = (int)((rt + gridDim.x) * UM_BLOCK_M);
                const bool have_next = rt + gridDim.x < u.nrt;
                for (uint32_t qt = 0; qt < u.nqt; ++qt) {
                    const int b_row = (int)(qt * N);
                    const bool pf = qt + 1 == u.nqt && have_next;
                    const bool a_last = qt + 1 == u.nqt;
                    int kc = 0;
                    for (uint32_t kb = 0; kb < u.kblocks; ++kb, kc += block_k) {
                        mbar_wait_u<PROF>(empty_u + 8u * s, ph ^ 1u, &w_empty);
                        uint8_t* sa = smem + (size_t)s * STAGE;
                        mbar_expect_tx_u(full_u + 8u * s, STAGE);
                        if (a_last) tma_load_2d_hint(sa, &tmA, &bars[s], kc, a_row, last_use);
                        else tma_load_2d(sa, &tmA, &bars[s], kc, a_row);
                        tma_load_2d(sa + UM_A_STAGE, &tmB, &bars[s], kc, b_row);
                        if (pf) tma_prefetch_2d(&tmA, kc, a_next);
                        if (++s == u.stages) { s = 0; ph ^= 1u; }
                    }
                }
            }
            if (PROF) u.prof[4 * blockIdx.x + 1] = (unsigned long long)w_empty;
        }
    } else {
        // ===================== consumers: wgmma + epilogue =====================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        const uint32_t cw = wg - 1;                          // which 64-row half of the tile
        const uint32_t wq = (threadIdx.x >> 5) & 3;          // warp within the warpgroup
        const uint32_t row_in_tile = cw * 64 + wq * 16 + (lane >> 2);
        const uint32_t col0 = 2 * (lane & 3);
        const bool direct = u.a.mask != nullptr;             // candidate-set mode: most allowed rows survive
        const bool l2 = u.a.metric == YAMS_B200_L2;
        const uint64_t desc_hi = make_smem_desc(0);
        float acc[N / 2];
#pragma unroll
        for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
        long long w_full = 0, t_epi = 0;
        uint32_t s = 0, ph = 0;
        for (uint32_t rt = blockIdx.x; rt < u.nrt; rt += gridDim.x) {
            // per-row data of this thread's two rows (row_in_tile and row_in_tile + 8)
            uint64_t li[2], grow[2];
            float alpha[2], beta[2], ialpha[2], ealpha[2];
            bool rvalid[2], rowok[2];
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                li[r] = (uint64_t)rt * UM_BLOCK_M + row_in_tile + 8 * r;
                rvalid[r] = li[r] < u.a.nrows;
                grow[r] = u.a.row_start + li[r] * u.a.row_stride;
                const float inr = rvalid[r] ? __ldg(&u.a.inv_norm[grow[r]]) : 0.f;
                // score = acc * alpha + beta.  cosine: alpha = 1/|row| (0 marks a row the reference skips), beta = 0;
                // L2: alpha = 2, beta = -|row|^2 (the row slot holds |row|^2; +inf marks a non-finite row)
                alpha[r] = l2 ? 2.f : inr;
                beta[r] = l2 ? -inr : 0.f;
                rowok[r] = rvalid[r] && (l2 ? inr < INFINITY : inr > 0.f);
                ialpha[r] = 1.0f / alpha[r];
                ealpha[r] = 2e-6f / alpha[r];
            }
            for (uint32_t qt = 0; qt < u.nqt; ++qt) {
                const uint32_t q0 = qt * N;
                constexpr int G = N / TG;   // threshold groups per tile
                float bound[G][2];
                uint32_t prev = 0;
                for (uint32_t kb = 0; kb < u.kblocks; ++kb) {
                    mbar_wait_u<PROF>(full_u + 8u * s, ph, &w_full);
                    const uint32_t sa = tiles_u + s * STAGE;
                    const uint64_t adesc = desc_hi | (uint64_t)(((sa + cw * (UM_A_STAGE / 2)) >> 4) & 0x3FFFu);
                    const uint64_t bdesc = desc_hi | (uint64_t)(((sa + UM_A_STAGE) >> 4) & 0x3FFFu);
                    wgmma_fence();
                    // advance 32 bytes (16 fp16 / 8 tf32) along K inside the swizzle row: +2 in 16-byte units
#pragma unroll
                    for (uint32_t k = 0; k < UM_MMAS_PER_KBLOCK; ++k)
                        wgmma_tile<N, TF32>(acc, adesc + 2 * k, bdesc + 2 * k, (kb != 0 || k != 0) ? 1u : 0u);
                    wgmma_commit();
                    if (kb == 0) {
                        if (FILTER) {
                            // while the first K block's MMAs run: per group of TG query columns (TG / 4 of this thread's
                            // accumulators per row) and row, a conservative bound,
                            //   acc * alpha + beta > tau_q  =>  acc > (tmin - beta) / alpha (slightly relaxed),
                            // tmin = the group's smallest threshold.  Only groups whose maximum passes take the per-column test.
#pragma unroll
                            for (int h = 0; h < G; ++h) {
                                const float tmin = tmin_s[q0 / TG + h];
#pragma unroll
                                for (int r = 0; r < 2; ++r) {
                                    bound[h][r] = INFINITY;
                                    if (rowok[r]) {
                                        const float b0 = (tmin - beta[r]) * ialpha[r];
                                        bound[h][r] = b0 - (fabsf(tmin) + fabsf(beta[r])) * ealpha[r] - 1e-30f;
                                    }
                                }
                            }
                        }
                    } else {
                        // the previous K block's MMAs are done: its stage may be refilled
                        wgmma_wait<1>();
                        if (lane == 0) mbar_arrive_u(empty_u + 8u * prev);
                    }
                    prev = s;
                    if (++s == u.stages) { s = 0; ph ^= 1u; }
                }
                wgmma_wait<0>();
                if (lane == 0) mbar_arrive_u(empty_u + 8u * prev);

                const long long t_epi0 = PROF ? clock64() : 0;
                if (FILTER) {
                    // common path: the maximum of each (group, row) against its bound, one branch for the whole tile.  The
                    // outcomes are kept as one bit each (bit 2 h + r) for the cold path, not as 16 maxima in registers.
                    constexpr int J = TG / 8;   // accumulator column pairs per group
                    uint32_t pass = 0;
#pragma unroll
                    for (int h = 0; h < G; ++h) {
#pragma unroll
                        for (int r = 0; r < 2; ++r) {
                            float m = acc[4 * J * h + 2 * r];
#pragma unroll
                            for (int j = J * h; j < J * (h + 1); ++j) m = fmaxf(m, fmaxf(acc[4 * j + 2 * r], acc[4 * j + 2 * r + 1]));
                            pass |= (m > bound[h][r] ? 1u : 0u) << (2 * h + r);
                        }
                    }
                    if (pass) {   // rare: some column of a group of this thread may survive
                        const float* tau_t = tau_all + q0;
#pragma unroll
                        for (int h = 0; h < G; ++h) {
#pragma unroll
                            for (int r = 0; r < 2; ++r) {
                                if (!((pass >> (2 * h + r)) & 1u)) continue;
#pragma unroll
                                for (int j = J * h; j < J * (h + 1); ++j) {
#pragma unroll
                                    for (int e = 0; e < 2; ++e) {
                                        const uint32_t c = 8 * j + col0 + e;
                                        const float sc = fmaf(acc[4 * j + 2 * r + e], alpha[r], beta[r]);
                                        if (sc > tau_t[c]) {
                                            const uint32_t q = q0 + c;
                                            if (direct) {
                                                const uint32_t w = __ldg(&u.a.mask[(uint64_t)q * u.a.mask_ld + (grow[r] >> 5)]);
                                                if (!((w >> (grow[r] & 31)) & 1u)) continue;
                                            }
                                            append_candidate(u.a.counts, u.a.cands, u.a.cap, q, (uint32_t)grow[r], sc);
                                        }
                                    }
                                }
                            }
                        }
                    }
                } else {
#pragma unroll
                    for (int r = 0; r < 2; ++r) {
                        if (!rvalid[r]) continue;
#pragma unroll
                        for (int j = 0; j < N / 8; ++j) {
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                const uint32_t q = q0 + 8 * j + col0 + e;
                                if (q < u.a.nq)
                                    u.a.out_scores[(uint64_t)q * u.a.ld + li[r]] =
                                        rowok[r] ? fmaf(acc[4 * j + 2 * r + e], alpha[r], beta[r]) : -INFINITY;
                            }
                        }
                    }
                }
                if (PROF) t_epi += clock64() - t_epi0;
            }
        }
        if (PROF && threadIdx.x == 128) {   // the first consumer warp's view
            u.prof[4 * blockIdx.x + 0] = (unsigned long long)w_full;
            u.prof[4 * blockIdx.x + 2] = (unsigned long long)t_epi;
            u.prof[4 * blockIdx.x + 3] = (unsigned long long)(clock64() - t_start);
        }
    }
}

// Query preparation, one CTA per query: the operand-typed copy the tensor cores read (fp16, or fp32 read as tf32), pre-scaled
// by 1/|q| for the cosine metric, and the per-query stage-1 error bound eps[q] that the exactness certificate uses.
// With x = the scaled query, y = what the tensor core multiplies (fp16-rounded / tf32-truncated x), dq = |x - y|, and the
// rows r read as r' (exact for fp16 rows; tf32-truncated for fp32 rows, residual norms tracked per corpus):
//   |x.r - y.r'| <= dq |r'| + |x| |r - r'|            (Cauchy-Schwarz with the ACTUAL rounding residuals)
//   cosine (|x| = 1, score = x.r / |r|):  eps = 1.25 (dq + dr_rel_max) + 2^-23 (d + 4) Y R1
//   L2 (score = 2 x.r - |r|^2)         :  eps = 2.5 (dq Rmax + |x| dr_abs_max) + 2^-22 (d + 4) Y R2 + 2^-22 Rmax^2
// The 1.25 covers the second-order term and the fp32 accumulation inside the tensor core is the 2^-23 (d + 4) term.  The
// tensor core truncates products on alignment to the block's largest one.  With fp16 subnormal operands the error measured
// on an H100 reaches ~2^-13 of the largest true product, as if products were sized by exponent fields, where a subnormal
// counts as 2^-14.  So the accumulation term takes every fp16 operand element as at least 2^-14 (no floor for tf32),
// f = d 2^-28: Y = sqrt((|x| + dq)^2 + f) >= |y| with the floor,
// R1 = sqrt(1 + f max(1/|r|)^2) >= |r with the floor| / |r|, R2 = sqrt(Rmax^2 + f).  Both factors are 1 + O(1e-6) unless
// the corpus holds rows of norm ~1e-3 or less, whose 1/|r| amplifies the accumulator's absolute error.
template <bool TF32>
__global__ void __launch_bounds__(128) queries_prep_kernel(const float* __restrict__ q32, const float* __restrict__ qinv, uint32_t nq,
                                                           uint32_t d, void* __restrict__ out, int metric, float r_max, float dr_abs_max,
                                                           float dr_rel_max, float inv_max, float* __restrict__ eps) {
    const uint32_t q = blockIdx.x;
    const float scale = qinv[q];   // 1 for L2
    float ss = 0.f, xx = 0.f;
    for (uint32_t c = threadIdx.x; c < d; c += 128) {
        const float x = q32[(uint64_t)q * d + c] * scale;
        float y;
        if (TF32) {
            reinterpret_cast<float*>(out)[(uint64_t)q * d + c] = x;
            y = __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
        } else {
            const __half h = __float2half_rn(x);
            reinterpret_cast<__half*>(out)[(uint64_t)q * d + c] = h;
            y = __half2float(h);
        }
        const float r = x - y;
        ss = fmaf(r, r, ss);
        xx = fmaf(x, x, xx);
    }
    __shared__ float red[2][4];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        ss += __shfl_xor_sync(0xffffffffu, ss, o);
        xx += __shfl_xor_sync(0xffffffffu, xx, o);
    }
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = ss; red[1][threadIdx.x >> 5] = xx; }
    __syncthreads();
    if (threadIdx.x == 0) {
        const float dq = sqrtf(red[0][0] + red[0][1] + red[0][2] + red[0][3]) * 1.000001f;
        const float xn = sqrtf(red[1][0] + red[1][1] + red[1][2] + red[1][3]) * 1.000001f;
        const float u = 1.1920929e-07f;   // 2^-23
        const float f = TF32 ? 0.f : (float)d * 3.7252903e-09f;                  // d 2^-28
        const float yf = sqrtf((xn + dq) * (xn + dq) + f) * 1.000001f;
        float e;
        if (metric == YAMS_B200_L2)
            e = 2.5f * (dq * r_max + xn * dr_abs_max) + 2.f * u * (float)(d + 4) * yf * (sqrtf(r_max * r_max + f) * 1.000001f) +
                2.f * u * r_max * r_max + 1e-30f;
        else e = 1.25f * (dq + xn * dr_rel_max) + u * (float)(d + 4) * yf * (sqrtf(1.f + f * inv_max * inv_max) * 1.000001f) + 1e-7f;
        eps[q] = e;
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

static bool make_map_2d(CUtensorMap* m, const void* base, uint64_t inner, uint64_t outer, uint64_t outer_stride_bytes,
                        uint32_t box_inner, uint32_t box_outer, bool f32 = false) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) return false;
    cuuint64_t dims[2] = {inner, outer};
    cuuint64_t strides[1] = {outer_stride_bytes};
    cuuint32_t box[2] = {box_inner, box_outer};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(m, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

bool wgmma_supported(const Corpus* c, uint32_t nq) {
    (void)nq;
    if (getenv("YAMS_B200_DISABLE_WGMMA")) return false;
    if (get_encode_fn() == nullptr) return false;
    // fp16 rows: fp16 wgmma; fp32 rows (the reference's BLOB layout): tf32 wgmma.  TMA needs 16-byte row pitches.
    return c->dtype == YAMS_B200_F16 ? (c->dim % 8 == 0) : (c->dim % 4 == 0 && !getenv("YAMS_B200_DISABLE_TF32"));
}

template <bool FILTER, int N, bool TF32, bool PROF>
static yams_status_t launch_wgmma(const CUtensorMap& tmA, const CUtensorMap& tmB, const WgArgs& u, unsigned grid, size_t smem,
                                  cudaStream_t st) {
    YB_CUDA(cudaFuncSetAttribute(stage1_wgmma_kernel<FILTER, N, TF32, PROF>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    stage1_wgmma_kernel<FILTER, N, TF32, PROF><<<grid, UM_THREADS, smem, st>>>(tmA, tmB, u);
    YB_CUDA(cudaGetLastError());
    return YAMS_OK;
}

template <int N>
static yams_status_t launch_wgmma_n(const CUtensorMap& tmA, const CUtensorMap& tmB, const WgArgs& u, unsigned grid, size_t smem,
                                    bool filter, bool tf32, cudaStream_t st) {
    if (u.prof) {   // the profiling instantiation: filter mode, as the search's corpus pass runs it
        if (!filter) return YAMS_ERR_UNSUPPORTED;
        return tf32 ? launch_wgmma<true, N, true, true>(tmA, tmB, u, grid, smem, st) : launch_wgmma<true, N, false, true>(tmA, tmB, u, grid, smem, st);
    }
    if (filter)
        return tf32 ? launch_wgmma<true, N, true, false>(tmA, tmB, u, grid, smem, st) : launch_wgmma<true, N, false, false>(tmA, tmB, u, grid, smem, st);
    return tf32 ? launch_wgmma<false, N, true, false>(tmA, tmB, u, grid, smem, st) : launch_wgmma<false, N, false, false>(tmA, tmB, u, grid, smem, st);
}

yams_status_t stage1_wgmma(Corpus* c, const Stage1Args& a, bool filter, cudaStream_t st, unsigned long long* prof) {
    const bool tf32 = a.dtype == YAMS_B200_F32;
    const uint32_t esz = tf32 ? 4 : 2;
    if ((a.dim * esz) % 16 != 0 || a.nrows == 0 || a.nq == 0) return YAMS_ERR_UNSUPPORTED;
    if (tf32 && getenv("YAMS_B200_DISABLE_TF32")) return YAMS_ERR_UNSUPPORTED;
    if ((reinterpret_cast<uintptr_t>(a.rows) & 15) != 0) return YAMS_ERR_UNSUPPORTED;
    if (a.nrows >= (1ull << 32)) return YAMS_ERR_UNSUPPORTED;
    yams_status_t rc;
    // queries pre-scaled by 1/|q| (so the epilogue only multiplies by 1/|row|), in the operand type of the engine
    size_t qb = (size_t)a.nq * a.dim * esz;
    if ((rc = c->q16.reserve(qb + 256)) != YAMS_OK) return rc;
    void* d_q16 = c->q16.p;
    if (!a.skip_qprep) {
        if (!a.eps) return YAMS_ERR_UNSUPPORTED;
        if (tf32) queries_prep_kernel<true><<<a.nq, 128, 0, st>>>(a.q32, a.qinv, a.nq, a.dim, d_q16, a.metric, a.r_max, a.dr_abs_max,
                                                                   a.dr_rel_max, a.inv_max, a.eps);
        else queries_prep_kernel<false><<<a.nq, 128, 0, st>>>(a.q32, a.qinv, a.nq, a.dim, d_q16, a.metric, a.r_max, 0.f, 0.f, a.inv_max,
                                                               a.eps);
    }


    // Small batches (HBM-bound: the corpus stream sets the pace) take 64-column query tiles, everything else 256-column
    // tiles, the widest wgmma (half the corpus-operand shared-memory reads per MAC of a 128-column tile).
    const uint32_t n_tile = a.nq <= 64 ? 64 : 256;
    WgArgs u{};
    u.a = a;
    u.prof = prof;
    u.nqt = (a.nq + n_tile - 1) / n_tile;
    u.nrt = (uint32_t)((a.nrows + UM_BLOCK_M - 1) / UM_BLOCK_M);
    const uint32_t block_k = UM_BLOCK_K_BYTES / esz;
    u.kblocks = (a.dim + block_k - 1) / block_k;
    if (u.nqt > 32 || (size_t)u.nqt * n_tile > 4096) return YAMS_ERR_UNSUPPORTED;   // thresholds live in shared memory
    const uint32_t stage_bytes = UM_A_STAGE + n_tile * UM_BLOCK_K_BYTES;
    const size_t fixed = 1024 /*align slack*/ + UM_MAX_TAU_GROUPS * 4 + (size_t)u.nqt * n_tile * 4;
    u.stages = std::min<uint32_t>(8, (uint32_t)((UM_SMEM_LIMIT - fixed - 16 * 8) / (stage_bytes + 16)));
    if (u.stages < 2) return YAMS_ERR_UNSUPPORTED;
    const size_t smem = (size_t)u.stages * (stage_bytes + 16) + fixed;

    CUtensorMap tmA, tmB;
    const uint8_t* a_base = reinterpret_cast<const uint8_t*>(a.rows) + (size_t)a.row_start * a.dim * esz;
    if (!make_map_2d(&tmA, a_base, a.dim, a.nrows, (uint64_t)a.row_stride * a.dim * esz, block_k, UM_BLOCK_M, tf32))
        return YAMS_ERR_UNSUPPORTED;
    if (!make_map_2d(&tmB, d_q16, a.dim, a.nq, (uint64_t)a.dim * esz, block_k, n_tile, tf32)) return YAMS_ERR_UNSUPPORTED;

    const unsigned grid = (unsigned)std::min<uint64_t>(u.nrt, (uint64_t)c->dev->sm_count);
    c->wg_launch[0] = n_tile; c->wg_launch[1] = grid;
    if (n_tile == 64) return launch_wgmma_n<64>(tmA, tmB, u, grid, smem, filter, tf32, st);
    return launch_wgmma_n<256>(tmA, tmB, u, grid, smem, filter, tf32, st);
}

}  // namespace yb
