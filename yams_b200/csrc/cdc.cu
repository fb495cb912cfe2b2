// cdc.cu -- content-defined chunk boundary detection on the GPU (candidates + exact cut selection).
//
// Replaces the byte loops of the reference chunkers
//   /root/reference/src/chunking/rabin_chunker.cpp:63-152   (RabinChunker)
//   /root/reference/include/yams/chunking/streaming_chunker.h:146-204 (StreamingChunker)
// with a data-parallel formulation (DESIGN.md §ingest):
//   1. candidate scan   -- HBM-bound; every byte position is tested independently with the
//                          closed-form masked rolling value (cdc_logic.h is_candidate); a SIMD
//                          low-byte prefilter keeps the common case at ~1 instr/byte;
//   2. ordered compaction of candidate positions (count -> scan -> write);
//   3. next-cut per candidate and file root (parallel), block-wise chain resolution, chunk emission.
// All results are bit-identical to the sequential reference; the logic lives in cdc_logic.h so the
// same lines are unit-tested on the CPU against the oracle.
#include "cdc_kernels.cuh"

namespace yb {

// 16-bit mask of positions (within the 16 bytes at stream position p0) that pass the low-byte
// prefilter.  word i covers bytes 4i..4i+3 (little endian).
__device__ __forceinline__ uint32_t prefilter16(const uint4& v, const CdcParams& P,
                                                const uint8_t* pass_s) {
    uint32_t wv[4] = {v.x, v.y, v.z, v.w};
    uint32_t mask = 0;
    if (P.nfast) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            uint32_t z = 0;
            for (uint32_t f = 0; f < P.nfast; ++f) {
                uint32_t m = wv[i] ^ (0x01010101u * P.fast[f]);
                // exact per-byte zero detect (no borrow false positives): bit7 of each byte set
                // iff that byte of m is zero
                uint32_t t = (m & 0x7f7f7f7fu) + 0x7f7f7f7fu;
                z |= ~(t | m | 0x7f7f7f7fu);
            }
            // compress 0x80 flags of 4 bytes into 4 bits
            uint32_t bits = ((z >> 7) & 1u) | ((z >> 14) & 2u) | ((z >> 21) & 4u) | ((z >> 28) & 8u);
            mask |= bits << (4 * i);
        }
    } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
#pragma unroll
            for (int b = 0; b < 4; ++b) {
                uint32_t byte = (wv[i] >> (8 * b)) & 0xffu;
                mask |= (uint32_t)pass_s[byte] << (4 * i + b);
            }
        }
    }
    return mask;
}

// Tests the 16-byte unit at stream position p0 (whose address is 16-byte aligned by construction
// of `origin`); positions outside [scan_lo, scan_hi) are masked.  Returns a 16-bit hit mask.
__device__ __forceinline__ uint32_t scan16(const ScanArgs& A, const uint64_t* T_s, const uint8_t* pass_s,
                                           uint64_t p0) {
    uint64_t lo = p0 > A.scan_lo ? p0 : A.scan_lo;
    uint64_t hi = p0 + 16 < A.scan_hi ? p0 + 16 : A.scan_hi;
    if (lo >= hi) return 0;
    uint4 v;
    uint32_t valid = 0xffffu;
    if (lo == p0 && hi == p0 + 16) {
        v = ldg_stream_u4(A.data + (p0 - A.base_pos));
    } else {
        // ragged first / last unit: byte loads of the in-range positions only
        uint32_t wv[4] = {0, 0, 0, 0};
        valid = 0;
        for (uint64_t q = lo; q < hi; ++q) {
            uint32_t b = (uint32_t)(q - p0);
            wv[b >> 2] |= (uint32_t)A.data[q - A.base_pos] << (8 * (b & 3));
            valid |= 1u << b;
        }
        v = make_uint4(wv[0], wv[1], wv[2], wv[3]);
    }
    uint32_t pre = prefilter16(v, A.P, pass_s) & valid;
    uint32_t hits = 0;
    ByteView view{A.data, A.base_pos, A.lowest};
    while (pre) {
        int b = __ffs(pre) - 1;
        pre &= pre - 1;
        if (is_candidate(view, T_s, A.P, p0 + (uint64_t)b)) hits |= 1u << b;
    }
    return hits;
}

__device__ __forceinline__ void load_tables(const ScanArgs& A, uint64_t* T_s, uint8_t* pass_s) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
        uint64_t t = A.table[i];
        T_s[i] = t;
        uint64_t m0 = A.P.mask & 0xffull;
        pass_s[i] = ((t & m0) == m0) ? 1 : 0;
    }
    __syncthreads();
}

// Candidates among the (< 16) positions [scan_lo, origin) that precede the first aligned unit (only when the
// buffer starts misaligned at the very beginning of a stream); returned as a bit mask, bit i = scan_lo + i.
__device__ __forceinline__ uint32_t scan_head(const ScanArgs& A, const uint64_t* T_s) {
    uint32_t hits = 0;
    ByteView view{A.data, A.base_pos, A.lowest};
    for (uint64_t p = A.scan_lo; p < A.origin && p < A.scan_hi; ++p)
        if (is_candidate(view, T_s, A.P, p)) hits |= 1u << (uint32_t)(p - A.scan_lo);
    return hits;
}

// pass 1: number of candidates per 16 KiB tile
__global__ void __launch_bounds__(kScanThreads) cdc_count_kernel(ScanArgs A, uint32_t ntiles,
                                                                 uint32_t* __restrict__ tile_counts) {
    __shared__ uint64_t T_s[256];
    __shared__ uint8_t pass_s[256];
    __shared__ uint32_t warp_sums[kScanThreads / 32];
    load_tables(A, T_s, pass_s);
    for (uint32_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        uint64_t tile_pos = A.origin + (uint64_t)tile * kTileBytes;
        uint32_t cnt = 0;
#pragma unroll
        for (int it = 0; it < kScanIters; ++it) {
            uint64_t p0 = tile_pos + ((uint64_t)it * kScanThreads + threadIdx.x) * 16;
            cnt += __popc(scan16(A, T_s, pass_s, p0));
        }
        if (tile == 0 && threadIdx.x == 0 && A.origin > A.scan_lo) cnt += __popc(scan_head(A, T_s));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = cnt;
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t s = 0;
#pragma unroll
            for (int w = 0; w < kScanThreads / 32; ++w) s += warp_sums[w];
            tile_counts[tile] = s;
        }
        __syncthreads();
    }
}

// pass 2: ordered write of candidate stream positions at the scanned tile offsets
__global__ void __launch_bounds__(kScanThreads) cdc_write_kernel(ScanArgs A, uint32_t ntiles,
                                                                 const uint32_t* __restrict__ tile_counts,
                                                                 const uint32_t* __restrict__ tile_offsets,
                                                                 uint64_t* __restrict__ cand) {
    __shared__ uint64_t T_s[256];
    __shared__ uint8_t pass_s[256];
    __shared__ uint32_t warp_sums[kScanThreads / 32];
    load_tables(A, T_s, pass_s);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (uint32_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        if (tile_counts[tile] == 0) continue;  // block-uniform
        uint64_t tile_pos = A.origin + (uint64_t)tile * kTileBytes;
        uint32_t running = tile_offsets[tile];
        for (int it = 0; it < kScanIters; ++it) {
            uint64_t p0 = tile_pos + ((uint64_t)it * kScanThreads + threadIdx.x) * 16;
            uint32_t hits = scan16(A, T_s, pass_s, p0);
            uint32_t head = 0;
            if (tile == 0 && it == 0 && threadIdx.x == 0 && A.origin > A.scan_lo) head = scan_head(A, T_s);
            uint32_t c = __popc(hits) + __popc(head);
            // block-wide exclusive prefix of c in thread order
            uint32_t incl = c;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                uint32_t nb = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += nb;
            }
            if (lane == 31) warp_sums[warp] = incl;
            __syncthreads();
            uint32_t wbase = 0, total = 0;
#pragma unroll
            for (int w = 0; w < kScanThreads / 32; ++w) {
                uint32_t s = warp_sums[w];
                if (w < warp) wbase += s;
                total += s;
            }
            uint32_t o = running + wbase + incl - c;
            while (head) {
                int b = __ffs(head) - 1;
                head &= head - 1;
                cand[o++] = A.scan_lo + (uint64_t)b;
            }
            while (hits) {
                int b = __ffs(hits) - 1;
                hits &= hits - 1;
                cand[o++] = p0 + (uint64_t)b;
            }
            running += total;
            __syncthreads();
        }
    }
}

// ---- single-pass scan: one contiguous byte range per WARP, tiles staged in shared memory by bulk async copies ----
//
// Every warp owns a contiguous range of the segment and walks it in 4 KiB tiles.  Lane 0 issues cp.async.bulk
// (TMA 1-D) copies of [64-byte look-behind | tile] into the warp's private 3-stage shared-memory ring (mbarrier
// complete_tx); the 32 lanes then read 16-byte units from shared memory (conflict-free LDS.128), run the SIMD
// low-byte prefilter and confirm the rare prefilter hits against bytes that are already in shared memory.
// Hits are written in position order (ballot + popc) to the warp's private slice of a global buffer; a second
// tiny kernel concatenates the slices.  No block-level synchronisation, no atomics; the input is read from HBM
// exactly once (+1.6% look-behind).  Anything exceptional (slice overflow on adversarial data) raises a flag
// and the host re-runs the segment through the exact two-pass kernels above.
constexpr int WS_WARPS = 16;
constexpr int WS_THREADS = WS_WARPS * 32;
constexpr uint32_t WS_TILE = 4096;
constexpr uint32_t WS_HALO = 64;      // >= kHistory (56), multiple of 16
constexpr int WS_STAGES = 3;
constexpr uint32_t WS_BUF = WS_HALO + WS_TILE;
constexpr uint32_t WS_LIST = 64;      // confirmed candidates of one tile kept in shared memory (expected 0.5)

struct SinglePassArgs {
    ScanArgs A;
    uint32_t ntiles;        // 4 KiB tiles in the segment (from A.origin)
    uint32_t tiles_per_warp;
    uint32_t slice_cap;     // candidate capacity of one warp slice
    uint32_t halo_ok;       // 1: the 64 bytes before A.origin are readable memory
    uint64_t end16;         // A.origin + floor16(A.scan_hi - A.origin): bulk copies stop here
    uint64_t* cand_tmp;     // [nwarps][slice_cap]
    uint32_t* slice_counts; // [nwarps]; 0xFFFFFFFF marks overflow
};

struct SmemView {
    const uint8_t* s;   // s[0] is stream position pos0
    uint64_t pos0;
    uint64_t lowest;
    __device__ __forceinline__ uint32_t at(int64_t pos) const {
        if (pos < (int64_t)lowest) return 0;
        return s[pos - (int64_t)pos0];
    }
};

__device__ __forceinline__ uint32_t sc_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// per-word "some byte equals one of the NFAST prefilter values" flags (bit 7 of each matching byte);
// pat[f] = 0x01010101 * value, held in registers
template <int NFAST>
__device__ __forceinline__ uint32_t fast_flags(uint32_t w, const uint32_t (&pat)[4]) {
    uint32_t z = 0;
#pragma unroll
    for (int f = 0; f < NFAST; ++f) {
        uint32_t m = w ^ pat[f];
        uint32_t t = (m & 0x7f7f7f7fu) + 0x7f7f7f7fu;
        z |= ~(t | m | 0x7f7f7f7fu);
    }
    return z;
}

// NFAST = number of byte values that pass the low-byte prefilter (1..4), or 0 for the generic table path
template <int NFAST>
__global__ void __launch_bounds__(WS_THREADS, 1) cdc_scan_single_pass_kernel(SinglePassArgs S) {
    extern __shared__ __align__(128) uint8_t sc_smem[];
    // warps per CTA is a launch parameter (16 when the scan runs alone, 8 when it shares the SMs with SHA-256 CTAs): the
    // warps never synchronise with each other after the table is loaded
    const int nwarps = (int)(blockDim.x >> 5);
    uint8_t* bufs = sc_smem;                                                        // nwarps x WS_STAGES x WS_BUF
    uint64_t* T_s = reinterpret_cast<uint64_t*>(bufs + (size_t)nwarps * WS_STAGES * WS_BUF);
    uint64_t* bars = T_s + 256;                                                     // nwarps x WS_STAGES
    uint8_t* pass_s = reinterpret_cast<uint8_t*>(bars + nwarps * WS_STAGES);        // 256
    uint16_t* T16_s = reinterpret_cast<uint16_t*>(pass_s + 256);                    // 256: low 16 bits of the table
    uint32_t* wlist_s = reinterpret_cast<uint32_t*>(T16_s + 256);                   // nwarps x WS_LIST confirmed candidates
    uint32_t* wcnt_s = wlist_s + nwarps * WS_LIST;                                  // nwarps counters
    uint8_t* wqueue_s = reinterpret_cast<uint8_t*>(wcnt_s + nwarps);                // nwarps x 256 flagged units
    const ScanArgs& A = S.A;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    for (int i = tid; i < 256; i += (int)blockDim.x) {
        uint64_t t = A.table[i];
        T_s[i] = t;
        uint64_t m0 = A.P.mask & 0xffull;
        pass_s[i] = ((t & m0) == m0) ? 1 : 0;
        T16_s[i] = (uint16_t)(t & 0xffffu);
    }
    // masks of <= 16 bits (every YAMS configuration) depend on exactly three bytes: b[p], b[p-1], b[p-W]
    const bool three_byte = A.P.steps <= 2;
    const uint32_t mask16 = (uint32_t)(A.P.mask & 0xffffu);
    const uint32_t W = A.P.window;
    uint8_t* my_bufs = bufs + (size_t)warp * WS_STAGES * WS_BUF;
    uint64_t* my_bars = bars + warp * WS_STAGES;
    if (lane == 0) {
        wcnt_s[warp] = 0;
        for (int s = 0; s < WS_STAGES; ++s)
            asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(sc_smem_u32(&my_bars[s])), "r"(1));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();

    const uint32_t gw = blockIdx.x * (uint32_t)nwarps + warp;
    const uint64_t t_begin64 = (uint64_t)gw * S.tiles_per_warp;
    const uint32_t t_begin = (uint32_t)(t_begin64 < S.ntiles ? t_begin64 : S.ntiles);
    const uint32_t t_end = (uint32_t)(t_begin64 + S.tiles_per_warp < S.ntiles ? t_begin64 + S.tiles_per_warp : S.ntiles);
    const uint32_t n_my = t_end > t_begin ? t_end - t_begin : 0;

    auto issue = [&](uint32_t i) {   // lane 0: start the copy of my i-th tile into stage i % WS_STAGES
        const uint32_t tile = t_begin + i;
        const uint32_t s = i % WS_STAGES;
        uint8_t* dst = my_bufs + (size_t)s * WS_BUF;
        const uint64_t tile_pos = A.origin + (uint64_t)tile * WS_TILE;
        uint64_t lo = (tile == 0 && !S.halo_ok) ? tile_pos : tile_pos - WS_HALO;
        uint64_t hi = tile_pos + WS_TILE < S.end16 ? tile_pos + WS_TILE : S.end16;
        uint32_t bytes = hi > lo ? (uint32_t)(hi - lo) : 0u;
        const uint32_t bar = sc_smem_u32(&my_bars[s]);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        if (bytes) {
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(sc_smem_u32(dst + (lo - (tile_pos - WS_HALO)))), "l"(A.data + (lo - A.base_pos)), "r"(bytes), "r"(bar)
                         : "memory");
        } else {
            asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
        }
    };
    if (lane == 0)
        for (uint32_t i = 0; i < n_my && i < (uint32_t)WS_STAGES; ++i) issue(i);

    uint32_t my_total = 0;          // candidates written by this warp so far (uniform across lanes)
    bool overflow = false;
    uint64_t* my_out = S.cand_tmp + (size_t)gw * S.slice_cap;
    uint32_t pat[4];
#pragma unroll
    for (int f = 0; f < 4; ++f) pat[f] = 0x01010101u * (uint32_t)A.P.fast[f];

    for (uint32_t i = 0; i < n_my; ++i) {
        const uint32_t tile = t_begin + i;
        const uint32_t s = i % WS_STAGES;
        const uint32_t parity = (i / WS_STAGES) & 1;
        uint8_t* buf = my_bufs + (size_t)s * WS_BUF;
        const uint64_t tile_pos = A.origin + (uint64_t)tile * WS_TILE;
        // bytes the bulk copy cannot bring in: look-behind of the very first tile, ragged tail (< 16 B)
        if (tile == 0 && !S.halo_ok) {
            for (uint32_t j = lane; j < WS_HALO; j += 32) {
                int64_t pos = (int64_t)tile_pos - WS_HALO + j;
                buf[j] = (pos >= (int64_t)A.lowest && pos >= 0) ? A.data[pos - (int64_t)A.base_pos] : 0;
            }
        }
        if (S.end16 < A.scan_hi && S.end16 >= tile_pos && S.end16 < tile_pos + WS_TILE) {
            uint64_t q = S.end16 + lane;
            if (q < A.scan_hi) buf[WS_HALO + (q - tile_pos)] = A.data[q - A.base_pos];
        }
        {   // wait for the bulk copy of this stage
            const uint32_t bar = sc_smem_u32(&my_bars[s]);
            uint32_t done = 0;
            long long t0 = 0;
            while (!done) {
                asm volatile(
                    "{\n\t.reg .pred p;\n\t"
                    "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                    "selp.u32 %0, 1, 0, p;\n\t}"
                    : "=r"(done) : "r"(bar), "r"(parity) : "memory");
                if (!done) {   // a wait longer than ~2 s of SM clocks aborts the kernel instead of hanging the GPU
                    long long now = clock64();
                    if (t0 == 0) t0 = now;
                    else if (now - t0 > 4000000000ll) __trap();
                }
            }
        }
        __syncwarp();
        uint32_t* my_list = wlist_s + warp * WS_LIST;
        uint32_t* my_cnt = wcnt_s + warp;
        uint8_t* my_queue = wqueue_s + warp * 256;
        // positions of a misaligned stream head that precede the first aligned unit (global tile 0 only);
        // list entries are offsets from tile_pos biased by 16, so the head sorts before every in-tile entry
        if (tile == 0 && A.origin > A.scan_lo) {
            uint64_t p = A.scan_lo + lane;
            if (p < A.origin && p < A.scan_hi) {
                ByteView gview{A.data, A.base_pos, A.lowest};
                if (is_candidate(gview, T_s, A.P, p)) {
                    uint32_t idx = atomicAdd(my_cnt, 1u);
                    if (idx < WS_LIST) my_list[idx] = 16u - (uint32_t)(A.origin - p);
                }
            }
        }
        SmemView view{buf, tile_pos - WS_HALO, A.lowest};
        const bool inside = tile_pos >= A.scan_lo && tile_pos + WS_TILE <= A.scan_hi;   // warp-uniform
        // ---- phase 1: which of my 8 units contain a byte that passes the low-byte prefilter? (~6% of units) ----
        uint32_t fm = 0;
#pragma unroll
        for (int j = 0; j < (int)(WS_TILE / 16 / 32); ++j) {
            const uint4 v = *reinterpret_cast<const uint4*>(buf + WS_HALO + (j * 32 + lane) * 16);
            uint32_t any;
            if (NFAST > 0) any = fast_flags<NFAST>(v.x, pat) | fast_flags<NFAST>(v.y, pat) | fast_flags<NFAST>(v.z, pat) | fast_flags<NFAST>(v.w, pat);
            else any = prefilter16(v, A.P, pass_s);
            fm |= (any != 0 ? 1u : 0u) << j;
        }
        // ---- compaction: flagged (lane, unit) pairs -> a dense queue, so phase 2 runs once per 32 flagged units ----
        const uint32_t c = __popc(fm);
        uint32_t incl = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t nb = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += nb;
        }
        const uint32_t nflag = __shfl_sync(0xffffffffu, incl, 31);
        {
            uint32_t o = incl - c;
            while (fm) {
                int j = __ffs(fm) - 1;
                fm &= fm - 1;
                my_queue[o++] = (uint8_t)(j * 32 + lane);   // unit index 0..255
            }
        }
        __syncwarp();
        // ---- phase 2: one lane per flagged unit: exact byte positions, 3-byte (or generic) confirm ----
        for (uint32_t qi = lane; qi < ((nflag + 31u) & ~31u); qi += 32) {
            if (qi < nflag) {
                const uint32_t u = my_queue[qi];
                const uint64_t p0 = tile_pos + (uint64_t)u * 16;
                const uint4 v = *reinterpret_cast<const uint4*>(buf + WS_HALO + u * 16);
                uint32_t pre;
                if (NFAST > 0) {
                    uint32_t zz[4] = {fast_flags<NFAST>(v.x, pat), fast_flags<NFAST>(v.y, pat), fast_flags<NFAST>(v.z, pat),
                                      fast_flags<NFAST>(v.w, pat)};
                    pre = 0;
#pragma unroll
                    for (int w = 0; w < 4; ++w)
                        pre |= (((zz[w] >> 7) & 1u) | ((zz[w] >> 14) & 2u) | ((zz[w] >> 21) & 4u) | ((zz[w] >> 28) & 8u)) << (4 * w);
                } else {
                    pre = prefilter16(v, A.P, pass_s);
                }
                if (!inside) {
                    uint64_t lo = p0 > A.scan_lo ? p0 : A.scan_lo;
                    uint64_t hi = p0 + 16 < A.scan_hi ? p0 + 16 : A.scan_hi;
                    uint32_t valid = 0;
                    if (lo < hi) valid = ((hi - p0 >= 16) ? 0xffffu : ((1u << (uint32_t)(hi - p0)) - 1u)) & ~((1u << (uint32_t)(lo - p0)) - 1u);
                    pre &= valid;
                }
                const uint8_t* ub = buf + WS_HALO + u * 16;
                while (pre) {
                    int b = __ffs(pre) - 1;
                    pre &= pre - 1;
                    bool hit;
                    if (three_byte) {
                        // h_p & 0xffff = ((T[b[p-1]] - T[b[p-W]]) & 0xff) << 8  ^  (T[b[p]] & 0xffff); the look-behind bytes
                        // are in this tile's buffer (the 64-byte halo holds zeros before the stream start)
                        uint32_t t0 = T16_s[ub[b]], t1 = T16_s[ub[b - 1]], tw = T16_s[ub[b - (int)W]];
                        uint32_t h = (((t1 - tw) & 0xffu) << 8) ^ t0;
                        hit = (h & mask16) == mask16;
                    } else {
                        hit = is_candidate(view, T_s, A.P, p0 + (uint64_t)b);
                    }
                    if (hit) {
                        uint32_t idx = atomicAdd(my_cnt, 1u);
                        if (idx < WS_LIST) my_list[idx] = u * 16 + (uint32_t)b + 16u;
                    }
                }
            }
        }
        __syncwarp();
        // ---- ordered write-out: rank order == position order (entries are unique) ----
        const uint32_t ncand = *my_cnt;
        if (ncand) {
            if (overflow || ncand > WS_LIST || my_total + ncand > S.slice_cap) {
                overflow = true;
            } else {
                for (uint32_t j = lane; j < ncand; j += 32) {
                    uint32_t mine = my_list[j], rank = 0;
                    for (uint32_t t = 0; t < ncand; ++t) rank += my_list[t] < mine ? 1u : 0u;
                    my_out[my_total + rank] = tile_pos + mine - 16u;
                }
                my_total += ncand;
            }
            __syncwarp();
            if (lane == 0) *my_cnt = 0;
        }
        __syncwarp();
        if (lane == 0 && i + WS_STAGES < n_my) issue(i + WS_STAGES);
    }
    if (lane == 0) S.slice_counts[gw] = overflow ? 0xFFFFFFFFu : my_total;
}

// concatenates the warp slices in warp order; scalars[0] = total candidates, scalars[2] = overflow flag.
// One block: a parallel exclusive scan of the slice counts (4 per thread), then a warp-per-slice copy.
__global__ void __launch_bounds__(1024) cdc_compact_kernel(const uint64_t* __restrict__ cand_tmp, const uint32_t* __restrict__ slice_counts,
                                                           uint32_t nslices, uint32_t slice_cap, uint64_t* __restrict__ cand,
                                                           uint64_t* __restrict__ scalars) {
    extern __shared__ uint64_t offs[];   // nslices + 1 (nslices <= 4096)
    __shared__ uint64_t warp_tot[32];
    __shared__ uint32_t bad;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) bad = 0;
    __syncthreads();
    uint32_t c[4];
    uint64_t local = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        uint32_t s = tid * 4 + j;
        uint32_t n = s < nslices ? slice_counts[s] : 0u;
        if (n == 0xFFFFFFFFu) { bad = 1; n = 0; }
        c[j] = n;
        local += n;
    }
    uint64_t incl = local;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint64_t nb = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= (uint32_t)o) incl += nb;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint64_t w = warp_tot[lane];
        uint64_t wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint64_t nb = __shfl_up_sync(0xffffffffu, wi, o);
            if (lane >= (uint32_t)o) wi += nb;
        }
        warp_tot[lane] = wi - w;   // exclusive
        if (lane == 31) {
            scalars[0] = wi;
            offs[nslices] = wi;
        }
    }
    __syncthreads();
    uint64_t run = warp_tot[warp] + incl - local;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        uint32_t s = tid * 4 + j;
        if (s < nslices) offs[s] = run;
        run += c[j];
    }
    __syncthreads();
    if (tid == 0) scalars[2] = bad;
    if (bad) return;
    const uint32_t nw = blockDim.x >> 5;
    for (uint32_t s = warp; s < nslices; s += nw) {
        uint32_t n = (uint32_t)(offs[s + 1] - offs[s]);
        for (uint32_t j = lane; j < n; j += 32) cand[offs[s] + j] = cand_tmp[(size_t)s * slice_cap + j];
    }
}

yams_status_t launch_scan_single_pass(const ScanArgs& A, uint32_t ntiles, uint64_t* cand_tmp, uint32_t* slice_counts,
                                      uint32_t slice_cap, uint32_t nslices, uint64_t* cand, uint64_t* scalars, cudaStream_t st) {
    const int W = WS_WARPS;
    SinglePassArgs S{};
    S.A = A;
    S.ntiles = ntiles;
    S.tiles_per_warp = (ntiles + nslices - 1) / nslices;
    S.slice_cap = slice_cap;
    S.halo_ok = (A.origin >= A.lowest + WS_HALO) ? 1u : 0u;
    S.end16 = A.scan_hi > A.origin ? A.origin + ((A.scan_hi - A.origin) & ~15ull) : A.origin;
    S.cand_tmp = cand_tmp;
    S.slice_counts = slice_counts;
    size_t smem = (size_t)W * WS_STAGES * WS_BUF + 256 * 8 + (size_t)W * WS_STAGES * 8 + 256 + 512 +
                  (size_t)W * (WS_LIST * 4 + 4 + 256) + 64;
    unsigned nctas = (nslices + W - 1) / W;
#define YB_LAUNCH_SCAN(NF)                                                                                                  \
    do {                                                                                                                    \
        YB_CUDA(cudaFuncSetAttribute(cdc_scan_single_pass_kernel<NF>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        cdc_scan_single_pass_kernel<NF><<<nctas, W * 32, smem, st>>>(S);                                                \
    } while (0)
    switch (A.P.nfast) {
        case 1: YB_LAUNCH_SCAN(1); break;
        case 2: YB_LAUNCH_SCAN(2); break;
        case 3: YB_LAUNCH_SCAN(3); break;
        case 4: YB_LAUNCH_SCAN(4); break;
        default: YB_LAUNCH_SCAN(0); break;
    }
#undef YB_LAUNCH_SCAN
    cdc_compact_kernel<<<1, 1024, (size_t)(nslices + 1) * 8, st>>>(cand_tmp, slice_counts, nslices, slice_cap, cand, scalars);
    YB_CUDA(cudaGetLastError());
    return YAMS_OK;
}

// ---- cut selection ----------------------------------------------------------------------------

// one warp per block of kNodeBlock nodes; lanes load coalesced, lane 0 does the backward pass
__global__ void __launch_bounds__(32) cdc_exit_kernel(const uint32_t* __restrict__ next, uint32_t nnodes,
                                                      uint32_t* __restrict__ exit_out) {
    __shared__ uint32_t nx[kNodeBlock];
    __shared__ uint32_t ex[kNodeBlock];
    uint32_t blk_start = blockIdx.x * kNodeBlock;
    uint32_t blk_end = min(blk_start + kNodeBlock, nnodes);
    for (uint32_t i = threadIdx.x; i < blk_end - blk_start; i += 32) nx[i] = next[blk_start + i];
    __syncwarp();
    if (threadIdx.x == 0) block_exit_seq(nx, blk_start, blk_end, ex);
    __syncwarp();
    for (uint32_t i = threadIdx.x; i < blk_end - blk_start; i += 32) exit_out[blk_start + i] = ex[i];
}

// single thread: hop block to block from the root, recording where the chain enters each block
__global__ void cdc_walk_kernel(const uint32_t* __restrict__ exit_in, uint32_t nnodes,
                                uint32_t* __restrict__ entry) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    uint32_t cur = 0;
    while (cur < nnodes) {
        entry[cur / kNodeBlock] = cur;
        cur = exit_in[cur];
    }
}

__global__ void __launch_bounds__(32) cdc_mark_kernel(const uint32_t* __restrict__ next, uint32_t nnodes,
                                                      const uint32_t* __restrict__ entry,
                                                      uint8_t* __restrict__ onchain) {
    __shared__ uint32_t nx[kNodeBlock];
    __shared__ uint8_t oc[kNodeBlock];
    uint32_t blk_start = blockIdx.x * kNodeBlock;
    uint32_t blk_end = min(blk_start + kNodeBlock, nnodes);
    uint32_t ent = entry[blockIdx.x];
    for (uint32_t i = threadIdx.x; i < blk_end - blk_start; i += 32) {
        nx[i] = next[blk_start + i];
        oc[i] = 0;
    }
    __syncwarp();
    if (threadIdx.x == 0 && ent != kNoEntry) block_mark_seq(nx, blk_start, blk_end, ent, oc);
    __syncwarp();
    for (uint32_t i = threadIdx.x; i < blk_end - blk_start; i += 32) onchain[blk_start + i] = oc[i];
}

// ---- cut selection over a layout of files (a streaming feed or chunk_and_hash_batch): thin wrappers over cdc_logic.h ----
// one thread per item (a candidate or a file root); it fills the entries of the item's node
__global__ void batch_next_kernel(BatchArgs B, uint64_t* __restrict__ npos, uint32_t* __restrict__ next, uint32_t* __restrict__ forced,
                                  uint32_t* __restrict__ cnt) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B.L.ncand + B.L.nfiles) return;
    BatchNext r = batch_next(B.L, B.P, i);
    npos[r.node] = r.pos;
    next[r.node] = r.next;
    forced[r.node] = r.forced;
    cnt[r.node] = r.count;
}

__global__ void batch_mask_counts_kernel(const uint8_t* __restrict__ onchain, uint32_t* __restrict__ cnt, uint32_t nnodes) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nnodes && !onchain[i]) cnt[i] = 0;
}

// *open_start = where the chunk after the last node of the chain starts
__global__ void batch_emit_kernel(BatchArgs B, const uint64_t* __restrict__ npos, const uint32_t* __restrict__ next,
                                  const uint32_t* __restrict__ forced, const uint8_t* __restrict__ onchain,
                                  const uint32_t* __restrict__ offsets, yams_chunk_desc* __restrict__ out,
                                  uint64_t* __restrict__ open_start) {
    const uint32_t nnodes = B.L.ncand + B.L.nfiles;
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nnodes || !onchain[i]) return;
    yams_chunk_desc* o = out + offsets[i];
    const uint32_t nx = next[i];
    const uint64_t end = batch_emit(B.L, B.P, npos[i], forced[i], nx < nnodes ? npos[nx] : 0ull, [o](uint64_t k, uint64_t off, uint64_t size) {
        o[k].offset = off;
        o[k].size = size;
    });
    if (nx == nnodes) *open_start = end;
}

__global__ void batch_first_kernel(BatchArgs B, const uint32_t* __restrict__ offsets, const uint64_t* __restrict__ total,
                                   uint64_t* __restrict__ first) {
    uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f < B.L.nfiles) first[f] = offsets[batch_node_of_root(B.L, f)];
    if (f == B.L.nfiles) first[f] = *total;
}

__global__ void batch_rebase_kernel(BatchArgs B, yams_chunk_desc* __restrict__ descs, uint64_t n) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) descs[i].offset = batch_file_offset(B.L, descs[i].offset);
}

// ---- generic exclusive scan (u32) ----------------------------------------------------------------
constexpr int kScanBlock = 256;
constexpr int kScanItems = 8;
constexpr int kScanChunk = kScanBlock * kScanItems;

__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* warp_s, uint32_t* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t nb = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += nb;
    }
    if (lane == 31) warp_s[warp] = incl;
    __syncthreads();
    uint32_t wbase = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < kScanBlock / 32; ++w) {
        uint32_t s = warp_s[w];
        if (w < warp) wbase += s;
        tot += s;
    }
    __syncthreads();
    *total = tot;
    return wbase + incl - v;
}

__global__ void __launch_bounds__(kScanBlock) scan_reduce_kernel(const uint32_t* __restrict__ in, size_t n,
                                                                 uint64_t* __restrict__ block_sums) {
    __shared__ uint32_t warp_s[kScanBlock / 32];
    size_t base = (size_t)blockIdx.x * kScanChunk + (size_t)threadIdx.x * kScanItems;
    uint32_t s = 0;
#pragma unroll
    for (int i = 0; i < kScanItems; ++i)
        if (base + i < n) s += in[base + i];
    uint32_t tot;
    block_exclusive_scan(s, warp_s, &tot);
    if (threadIdx.x == 0) block_sums[blockIdx.x] = tot;
}

// single block: exclusive scan of block_sums (u64) in place, total to *d_total
__global__ void __launch_bounds__(kScanBlock) scan_sums_kernel(uint64_t* __restrict__ block_sums, size_t nb,
                                                               uint64_t* __restrict__ d_total) {
    __shared__ uint64_t sh[kScanBlock];
    __shared__ uint64_t carry_s;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    for (size_t base = 0; base < nb; base += kScanBlock) {
        size_t i = base + threadIdx.x;
        uint64_t v = i < nb ? block_sums[i] : 0;
        sh[threadIdx.x] = v;
        __syncthreads();
        // Hillis-Steele inclusive scan in shared memory
        for (int o = 1; o < kScanBlock; o <<= 1) {
            uint64_t add = threadIdx.x >= o ? sh[threadIdx.x - o] : 0;
            __syncthreads();
            sh[threadIdx.x] += add;
            __syncthreads();
        }
        uint64_t carry = carry_s;
        if (i < nb) block_sums[i] = carry + sh[threadIdx.x] - v;
        __syncthreads();
        if (threadIdx.x == kScanBlock - 1) carry_s = carry + sh[kScanBlock - 1];
        __syncthreads();
    }
    if (threadIdx.x == 0) *d_total = carry_s;
}

__global__ void __launch_bounds__(kScanBlock) scan_apply_kernel(const uint32_t* __restrict__ in,
                                                                uint32_t* __restrict__ out, size_t n,
                                                                const uint64_t* __restrict__ block_sums) {
    __shared__ uint32_t warp_s[kScanBlock / 32];
    size_t base = (size_t)blockIdx.x * kScanChunk + (size_t)threadIdx.x * kScanItems;
    uint32_t v[kScanItems];
    uint32_t s = 0;
#pragma unroll
    for (int i = 0; i < kScanItems; ++i) {
        v[i] = base + i < n ? in[base + i] : 0;
        s += v[i];
    }
    uint32_t tot;
    uint32_t ex = block_exclusive_scan(s, warp_s, &tot);
    uint32_t run = (uint32_t)block_sums[blockIdx.x] + ex;
#pragma unroll
    for (int i = 0; i < kScanItems; ++i) {
        if (base + i < n) out[base + i] = run;
        run += v[i];
    }
}

yams_status_t exclusive_scan_u32(const uint32_t* d_in, uint32_t* d_out, size_t n, uint64_t* d_total,
                                 DevBuf& scratch, cudaStream_t st) {
    if (n == 0) {
        YB_CUDA(cudaMemsetAsync(d_total, 0, sizeof(uint64_t), st));
        return YAMS_OK;
    }
    size_t nb = (n + kScanChunk - 1) / kScanChunk;
    yams_status_t rc = scratch.reserve(nb * sizeof(uint64_t));
    if (rc != YAMS_OK) return rc;
    uint64_t* sums = scratch.as<uint64_t>();
    scan_reduce_kernel<<<(unsigned)nb, kScanBlock, 0, st>>>(d_in, n, sums);
    scan_sums_kernel<<<1, kScanBlock, 0, st>>>(sums, nb, d_total);
    scan_apply_kernel<<<(unsigned)nb, kScanBlock, 0, st>>>(d_in, d_out, n, sums);
    YB_CUDA(cudaGetLastError());
    return YAMS_OK;
}

// ---- calculateDeduplication (/root/reference/src/chunking/rabin_chunker.cpp:224-239) ----------------------
// Open-addressing set of chunk indices keyed by the digest: the thread that claims a slot owns the first
// occurrence of that digest; later chunks with an identical 32-byte digest are duplicates.
__global__ void dedup_stats_kernel(const yams_chunk_desc* __restrict__ descs, uint32_t n, uint32_t* __restrict__ table,
                                   uint64_t slots, unsigned long long* __restrict__ out /* total, unique, count, uniq */) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned long long tot = 0, usz = 0, ucnt = 0, cnt = 0;
    if (i < n) {
        const uint64_t* dg = reinterpret_cast<const uint64_t*>(descs[i].digest);
        const uint64_t d0 = dg[0], d1 = dg[1], d2 = dg[2], d3 = dg[3];
        const uint64_t size = descs[i].size;
        uint64_t slot = splitmix64(d0 ^ (d1 << 1)) & (slots - 1);
        bool unique = false;
        for (;;) {
            uint32_t cur = atomicCAS(&table[slot], 0xFFFFFFFFu, i);
            if (cur == 0xFFFFFFFFu) { unique = true; break; }   // claimed: first occurrence
            const uint64_t* og = reinterpret_cast<const uint64_t*>(descs[cur].digest);
            if (og[0] == d0 && og[1] == d1 && og[2] == d2 && og[3] == d3) break;   // duplicate of chunk `cur`
            slot = (slot + 1) & (slots - 1);
        }
        tot = size;
        cnt = 1;
        if (unique) { usz = size; ucnt = 1; }
    }
    // warp-level reduction, one atomic per warp and counter
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        tot += __shfl_xor_sync(0xffffffffu, tot, o);
        usz += __shfl_xor_sync(0xffffffffu, usz, o);
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        ucnt += __shfl_xor_sync(0xffffffffu, ucnt, o);
    }
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(&out[0], tot);
        atomicAdd(&out[1], usz);
        atomicAdd(&out[2], cnt);
        atomicAdd(&out[3], ucnt);
    }
}

yams_status_t launch_dedup_stats(const yams_chunk_desc* d_descs, uint32_t n, uint32_t* d_table, uint64_t slots,
                                 unsigned long long* d_out, cudaStream_t st) {
    dedup_stats_kernel<<<(n + 255) / 256, 256, 0, st>>>(d_descs, n, d_table, slots, d_out);
    YB_CUDA(cudaGetLastError());
    return YAMS_OK;
}

// ---- synthetic byte stream (SURVEY.md §8d): byte[i] = (splitmix64(seed ^ (i>>3)) >> (8*(i&7))) ----
__global__ void synth_bytes_kernel(uint64_t seed, uint64_t start, uint64_t n, uint8_t* __restrict__ out) {
    // one thread per aligned 8-byte group of the STREAM
    uint64_t g0 = start >> 3;
    uint64_t ngroups = ((start + n + 7) >> 3) - g0;
    for (uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; g < ngroups;
         g += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t grp = g0 + g;
        uint64_t v = splitmix64(seed ^ grp);
        uint64_t pos = grp << 3;
        if (pos >= start && pos + 8 <= start + n && (((uintptr_t)(out + (pos - start))) & 7) == 0) {
            *reinterpret_cast<uint64_t*>(out + (pos - start)) = v;
        } else {
            for (int b = 0; b < 8; ++b) {
                uint64_t q = pos + b;
                if (q >= start && q < start + n) out[q - start] = (uint8_t)(v >> (8 * b));
            }
        }
    }
}

yams_status_t launch_synth_bytes(uint64_t seed, uint64_t start, uint64_t n, uint8_t* d_out, int sm_count,
                                 cudaStream_t st) {
    if (n == 0) return YAMS_OK;
    synth_bytes_kernel<<<sm_count * 8, 256, 0, st>>>(seed, start, n, d_out);
    YB_CUDA(cudaGetLastError());
    return YAMS_OK;
}

// ---- host orchestration ---------------------------------------------------------------------------

yams_status_t resolve_params(const yams_cdc_config* cfg, CdcParams* P, uint64_t table[256]) {
    YB_ARG(cfg != nullptr, "cfg is null");
    YB_ARG(cfg->variant == YAMS_CDC_STREAMING || cfg->variant == YAMS_CDC_RABIN, "unknown cdc variant");
    YB_ARG(cfg->window_size <= (uint64_t)kMaxWindow,
           "window_size must be <= 48 (the reference ring buffer is a fixed 48-byte array)");
    memset(P, 0, sizeof(*P));
    uint64_t poly = cfg->polynomial ? cfg->polynomial : kDefaultPoly;
    for (int b = 0; b < 256; ++b) table[b] = table_entry(poly, (uint32_t)b);
    P->mask = cfg->mask;
    P->window = cfg->window_size ? (uint32_t)cfg->window_size : 1u;  // streaming_chunker.cpp:44-46
    P->steps = mask_steps(cfg->mask);
    uint64_t force = cfg->min_chunk > cfg->max_chunk ? cfg->min_chunk : cfg->max_chunk;
    if (cfg->variant == YAMS_CDC_STREAMING) {
        P->lo = (cfg->min_chunk > 1 ? cfg->min_chunk : 1) - 1;
        if (force == 0) force = 1;
    } else {
        P->lo = cfg->min_chunk;
        YB_ARG(force != 0, "RabinChunker with min_chunk == max_chunk == 0 never terminates");
    }
    P->force = force;
    // low-byte prefilter: byte values whose table entry has all of (mask & 0xff) set
    uint64_t m0 = cfg->mask & 0xffull;
    uint32_t npass = 0;
    uint8_t vals[4] = {0, 0, 0, 0};
    for (int b = 0; b < 256; ++b) {
        if ((table[b] & m0) == m0) {
            if (npass < 4) vals[npass] = (uint8_t)b;
            ++npass;
        }
    }
    if (npass >= 1 && npass <= 4) {
        P->nfast = npass;
        memcpy(P->fast, vals, 4);
    } else {
        P->nfast = 0;
    }
    return YAMS_OK;
}

}  // namespace yb
