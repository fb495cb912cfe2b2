// sha256.cu -- SHA-256 (FIPS 180-4) over a table of chunks, one chunk per LANE, bytes staged by the
// whole warp through shared memory with coalesced 128-bit loads.
//
// Replaces SHA256Hasher::hash as called per chunk by the reference chunkers
// (/root/reference/src/chunking/rabin_chunker.cpp:140,
//  /root/reference/include/yams/chunking/streaming_chunker.h:190; hasher
//  /root/reference/src/crypto/sha256_hasher.cpp:167-195 -> OpenSSL EVP_sha256).
//
// Design (DESIGN.md §sha256): the compression function is a 64-round dependent chain, so the only
// parallelism is across chunks.  Each lane owns one chunk at a time (persistent lanes pulling chunk
// indices from a global counter, so variable chunk lengths do not idle lanes).  Every WINDOW of
// kWinBlocks 64-byte blocks the warp cooperatively copies, for each of its 32 lane-chunks, the next
// <=192 bytes (13 x 16-byte units from the 16-byte-aligned-down address) into that lane's shared
// memory row: one ld.global.v4 instruction covers two rows x 13 units, i.e. two contiguous 208-byte
// spans.  Lanes then read their row word-by-word; the byte misalignment of the chunk start and the
// big-endian word order are both absorbed by ONE prmt per message word.
// The kernel is INT32-ALU bound (~22 instr/byte), not HBM bound (SURVEY.md §8d).
#include <algorithm>

#include "common.cuh"

namespace yb {

constexpr int kShaWarpsPerCta = 4;
constexpr int kWinBlocks = 3;       // 64-byte blocks consumed per staging window
constexpr int kRowUnits = 13;       // 16-byte units per lane row: ceil((15 + 192) / 16)
constexpr int kRowWords = kRowUnits * 4;

__device__ __constant__ uint32_t kSha256K[64] = {
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5,
    0xd807aa98, 0x12835b01, 0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174,
    0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da,
    0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967,
    0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
    0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070,
    0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3,
    0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};

__device__ __forceinline__ uint32_t rotr(uint32_t x, int n) { return __funnelshift_r(x, x, n); }

// With `one` an opaque runtime 1, x * one + y compiles to IMAD, which runs on the FMA pipe and takes
// the additions off the INT32 ALU pipe where the SHF/LOP3 of the round function already saturate issue
// (DESIGN.md §sha256: ALU-pipe instructions per block drop from ~1330 to ~1030).
__device__ __forceinline__ uint32_t add2(uint32_t x, uint32_t y, uint32_t one) {
    return x * one + y;
}

__device__ __forceinline__ void sha256_compress(uint32_t (&st)[8], uint32_t (&w)[16], uint32_t one) {
    uint32_t a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
#pragma unroll
    for (int i = 0; i < 64; ++i) {
        if (i >= 16) {
            uint32_t w15 = w[(i - 15) & 15], w2 = w[(i - 2) & 15];
            uint32_t s0 = rotr(w15, 7) ^ rotr(w15, 18) ^ (w15 >> 3);
            uint32_t s1 = rotr(w2, 17) ^ rotr(w2, 19) ^ (w2 >> 10);
            w[i & 15] = add2(add2(add2(w[i & 15], s0, one), w[(i - 7) & 15], one), s1, one);
        }
        uint32_t S1 = rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25);
        uint32_t ch = (e & f) ^ (~e & g);
        uint32_t kw = add2(w[i & 15], kSha256K[i], one);
        uint32_t t1 = add2(add2(add2(h, S1, one), ch, one), kw, one);
        uint32_t S0 = rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22);
        uint32_t mj = (a & b) ^ (a & c) ^ (b & c);
        uint32_t t2 = add2(S0, mj, one);
        h = g; g = f; f = e; e = add2(d, t1, one); d = c; c = b; b = a; a = add2(t1, t2, one);
    }
    st[0] += a; st[1] += b; st[2] += c; st[3] += d; st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}

constexpr int kShaCtasPerSm = 4;   // resident CTAs per SM: the register budget of the launch bounds and the grid's cap

// data[0] is stream position base_pos; desc.offset is a stream position.
__global__ void __launch_bounds__(kShaWarpsPerCta * 32, kShaCtasPerSm)
sha256_chunks_kernel(const uint8_t* __restrict__ data, uint64_t base_pos,
                     yams_chunk_desc* __restrict__ descs, uint32_t first, uint32_t n,
                     unsigned int* __restrict__ counter, uint32_t one, const uint32_t* __restrict__ order) {
    __shared__ __align__(16) uint32_t smem[kShaWarpsPerCta][32 * kRowWords];
    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    uint32_t* rows = smem[warp];
    uint32_t* myrow = rows + lane * kRowWords;
    const unsigned full = 0xffffffffu;

    bool has = false, exhausted = false;
    uint64_t ptr = 0, rem = 0, total = 0;
    uint32_t idx = 0;
    int fin = 0;  // 1: data consumed, the length-only padding block is still due
    uint32_t st[8];

    for (;;) {
        // ---- idle lanes pull the next chunk index -------------------------------------------
        bool want = !has && !exhausted;
        unsigned m = __ballot_sync(full, want);
        if (m) {
            int leader = __ffs(m) - 1;
            unsigned int base = 0;
            if (lane == leader) base = atomicAdd(counter, (unsigned)__popc(m));
            base = __shfl_sync(full, base, leader);
            if (want) {
                uint32_t k = base + __popc(m & ((1u << lane) - 1u));
                if (k < n) {
                    idx = order ? order[k] : first + k;
                    uint64_t off = descs[idx].offset;
                    uint64_t sz = descs[idx].size;
                    ptr = (uint64_t)data + (off - base_pos);
                    rem = sz;
                    total = sz;
                    fin = 0;
                    st[0] = 0x6a09e667u; st[1] = 0xbb67ae85u; st[2] = 0x3c6ef372u; st[3] = 0xa54ff53au;
                    st[4] = 0x510e527fu; st[5] = 0x9b05688cu; st[6] = 0x1f83d9abu; st[7] = 0x5be0cd19u;
                    has = true;
                } else {
                    exhausted = true;
                }
            }
        }
        if (!__any_sync(full, has)) break;

        // ---- cooperative staging of this window ------------------------------------------------
        // lane-row r needs bytes [ptr_r, ptr_r + wl_r), wl_r = min(rem_r, 192)
        uint32_t wl = (has && !fin) ? (uint32_t)(rem < (uint64_t)(64 * kWinBlocks) ? rem : 64 * kWinBlocks) : 0u;
        uint64_t ubase = ptr & ~(uint64_t)15;
        uint32_t nunits = wl ? (uint32_t)(((ptr + wl - 1) >> 4) - (ptr >> 4) + 1) : 0u;
        const int half = lane >> 4, unit = lane & 15;
#pragma unroll
        for (int p = 0; p < 16; ++p) {
            int r = 2 * p + half;
            uint64_t rb = __shfl_sync(full, ubase, r);
            uint32_t rn = __shfl_sync(full, nunits, r);
            if ((uint32_t)unit < rn) {
                uint4 v = ldg_stream_u4(reinterpret_cast<const void*>(rb + (uint64_t)unit * 16));
                *reinterpret_cast<uint4*>(rows + r * kRowWords + unit * 4) = v;
            }
        }
        __syncwarp();

        const uint32_t a = (uint32_t)(ptr & 15);
        const uint32_t sh = a & 3;
        const uint32_t sel = (sh + 3) | ((sh + 2) << 4) | ((sh + 1) << 8) | (sh << 12);
#pragma unroll 1
        for (int blk = 0; blk < kWinBlocks; ++blk) {
            if (has) {
                uint32_t w[16];
                bool done = false;
                if (fin) {
                    // length-only block
#pragma unroll
                    for (int t = 0; t < 14; ++t) w[t] = 0;
                    uint64_t bits = total << 3;
                    w[14] = (uint32_t)(bits >> 32);
                    w[15] = (uint32_t)bits;
                    done = true;
                } else {
                    const uint32_t* src = myrow + (a >> 2) + 16 * blk;
                    uint32_t x[17];
#pragma unroll
                    for (int t = 0; t < 17; ++t) x[t] = src[t];
#pragma unroll
                    for (int t = 0; t < 16; ++t) w[t] = __byte_perm(x[t], x[t + 1], sel);
                    if (rem >= 64) {
                        rem -= 64;
                        ptr += 64;
                    } else {
                        // last data block: keep rem bytes, append 0x80, zero the rest
                        const uint32_t r = (uint32_t)rem;
#pragma unroll
                        for (int t = 0; t < 16; ++t) {
                            int kb = (int)r - 4 * t;  // bytes of word t that are message bytes
                            uint32_t keep = kb >= 4 ? 0xffffffffu : (kb <= 0 ? 0u : ~(0xffffffffu >> (8 * kb)));
                            uint32_t v = w[t] & keep;
                            if (kb >= 0 && kb < 4) v |= 0x80u << (24 - 8 * kb);
                            w[t] = v;
                        }
                        rem = 0;
                        if (r <= 55) {
                            uint64_t bits = total << 3;
                            w[14] = (uint32_t)(bits >> 32);
                            w[15] = (uint32_t)bits;
                            done = true;
                        } else {
                            fin = 1;
                        }
                    }
                }
                sha256_compress(st, w, one);
                if (done) {
                    uint4 lo, hi;
                    lo.x = __byte_perm(st[0], 0, 0x0123); lo.y = __byte_perm(st[1], 0, 0x0123);
                    lo.z = __byte_perm(st[2], 0, 0x0123); lo.w = __byte_perm(st[3], 0, 0x0123);
                    hi.x = __byte_perm(st[4], 0, 0x0123); hi.y = __byte_perm(st[5], 0, 0x0123);
                    hi.z = __byte_perm(st[6], 0, 0x0123); hi.w = __byte_perm(st[7], 0, 0x0123);
                    uint4* dg = reinterpret_cast<uint4*>(descs[idx].digest);
                    dg[0] = lo;
                    dg[1] = hi;
                    has = false;
                    fin = 0;
                }
            }
        }
        __syncwarp();
    }
}

// Longest-first order.  Every lane hashes whole chunks, so the launch ends when the lane that drew the last long chunk ends:
// in index order that tail is 39 % of the ideal time on a 16 GiB / 700 k-chunk table (10 % at 64 GiB), sorted by size it is
// 5 % / 1 % (simulation in DESIGN.md 3.3).  A 32-bucket counting sort by size (bucket = 6 * size / mean, largest first) is
// close enough to a full sort; the order inside a bucket is whatever the atomics produce -- digests land in descs[idx], so
// the result does not depend on it.
constexpr int kShaBuckets = 32;
__device__ __forceinline__ int sha_bucket(uint64_t size, uint64_t mean) {
    const uint64_t t = mean ? (size * 6u) / mean : 0u;
    return kShaBuckets - 1 - (int)(t < (uint64_t)(kShaBuckets - 1) ? t : (uint64_t)(kShaBuckets - 1));
}
__global__ void sha_order_count_kernel(const yams_chunk_desc* __restrict__ descs, uint32_t first, uint32_t n, uint64_t mean,
                                       uint32_t* __restrict__ counts) {
    __shared__ uint32_t h[kShaBuckets];
    if (threadIdx.x < kShaBuckets) h[threadIdx.x] = 0;
    __syncthreads();
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        atomicAdd(&h[sha_bucket(descs[first + i].size, mean)], 1u);
    __syncthreads();
    if (threadIdx.x < kShaBuckets && h[threadIdx.x]) atomicAdd(&counts[threadIdx.x], h[threadIdx.x]);
}
__global__ void sha_order_scatter_kernel(const yams_chunk_desc* __restrict__ descs, uint32_t first, uint32_t n, uint64_t mean,
                                         const uint32_t* __restrict__ counts, uint32_t* __restrict__ cursors,
                                         uint32_t* __restrict__ order) {
    __shared__ uint32_t base[kShaBuckets];
    __shared__ uint32_t h[kShaBuckets];
    __shared__ uint32_t got[kShaBuckets];
    if (threadIdx.x < kShaBuckets) h[threadIdx.x] = 0;
    if (threadIdx.x == 0) {
        uint32_t acc = 0;
        for (int b = 0; b < kShaBuckets; ++b) { base[b] = acc; acc += counts[b]; }
    }
    __syncthreads();
    // one tile of blockDim.x chunks per iteration: rank inside the CTA by shared atomics, one global atomic per bucket per tile
    for (uint32_t t0 = blockIdx.x * blockDim.x; t0 < n; t0 += gridDim.x * blockDim.x) {
        const uint32_t i = t0 + threadIdx.x;
        int b = -1;
        uint32_t r = 0;
        if (i < n) {
            b = sha_bucket(descs[first + i].size, mean);
            r = atomicAdd(&h[b], 1u);
        }
        __syncthreads();
        if (threadIdx.x < kShaBuckets) {
            got[threadIdx.x] = h[threadIdx.x] ? atomicAdd(&cursors[threadIdx.x], h[threadIdx.x]) : 0u;
            h[threadIdx.x] = 0;
        }
        __syncthreads();
        if (b >= 0) order[base[b] + got[b] + r] = first + i;
        __syncthreads();
    }
}

// Launch helper: hashes descs[first .. first+n). d_counter must point at a zeroed uint32.
yams_status_t launch_sha256_chunks(const uint8_t* d_data, uint64_t base_pos, yams_chunk_desc* d_descs,
                                   uint32_t first, uint32_t n, unsigned int* d_counter, int sm_count,
                                   cudaStream_t st, uint32_t* d_order_ws, uint64_t total_bytes) {
    if (n == 0) return YAMS_OK;
    YB_CUDA(cudaMemsetAsync(d_counter, 0, sizeof(unsigned int), st));
    // d_order_ws: 64 counters + n indices (sha256_order_ws_bytes); tables that leave every lane under ~2 chunks are not worth it
    const uint32_t* d_order = nullptr;
    if (n >= 4096) {
        const uint64_t mean = std::max<uint64_t>(1, total_bytes / n);
        YB_CUDA(cudaMemsetAsync(d_order_ws, 0, 64 * sizeof(uint32_t), st));
        const unsigned g = (unsigned)std::min<uint32_t>((n + 255) / 256, (uint32_t)sm_count * 8u);
        sha_order_count_kernel<<<g, 256, 0, st>>>(d_descs, first, n, mean, d_order_ws);
        sha_order_scatter_kernel<<<g, 256, 0, st>>>(d_descs, first, n, mean, d_order_ws, d_order_ws + 32, d_order_ws + 64);
        d_order = d_order_ws + 64;
    }
    uint32_t warps_needed = (n + 31) / 32;
    uint32_t ctas = (warps_needed + kShaWarpsPerCta - 1) / kShaWarpsPerCta;
    uint32_t max_ctas = (uint32_t)sm_count * (uint32_t)kShaCtasPerSm;
    if (ctas > max_ctas) ctas = max_ctas;
    sha256_chunks_kernel<<<ctas, kShaWarpsPerCta * 32, 0, st>>>(d_data, base_pos, d_descs, first, n, d_counter, 1u, d_order);
    YB_CUDA(cudaGetLastError());
    return YAMS_OK;
}

}  // namespace yb
