// digest_set.cu -- device-resident set of SHA-256 chunk digests: the batched form of the per-chunk
// `storage_->exists(hash)` / `storage_->store(hash, ...)` loop that follows chunking in the reference
// (/root/reference/src/api/content_store_impl.cpp:245-288; storage_engine.cpp:281-305), SURVEY.md §8f N1.
//
// Layout in HBM: `store` = every digest that was new when it was offered, 32 B each, append-only; `table` = open-addressing array of
// uint32 indices into `store` (0xFFFFFFFF = empty, load factor <= 0.5, linear probing from splitmix64 of the first
// 16 digest bytes).  One thread per digest; a probe is one 4-byte read plus, on a hit, one 32-byte compare.
//
// Batch semantics == the reference's sequential loop: digest i "existed" iff it was in the set before the call or an
// EARLIER digest of the same batch equals it (the loop stores chunk j before it looks at chunk i > j).  The claim
// kernel lets equal digests of one batch agree on their lowest index with atomicMin, so the answer is deterministic.
#include <memory>
#include <mutex>
#include <new>

#include "common.cuh"

namespace yb {

constexpr uint32_t kEmptySlot = 0xFFFFFFFFu;

struct Digest {
    uint4 lo, hi;
};
__device__ __forceinline__ bool digest_eq(const Digest& a, const Digest& b) {
    return a.lo.x == b.lo.x && a.lo.y == b.lo.y && a.lo.z == b.lo.z && a.lo.w == b.lo.w && a.hi.x == b.hi.x && a.hi.y == b.hi.y &&
           a.hi.z == b.hi.z && a.hi.w == b.hi.w;
}
__device__ __forceinline__ uint64_t mix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ULL;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
    return x ^ (x >> 31);
}
__device__ __forceinline__ uint64_t digest_slot(const Digest& d, uint64_t slots) {
    uint64_t a = ((uint64_t)d.lo.y << 32) | d.lo.x, b = ((uint64_t)d.lo.w << 32) | d.lo.z;
    return mix64(a ^ (b << 1)) & (slots - 1);
}

// staged input (stride bytes apart, 4-byte aligned or not) -> store[base + i]
__global__ void digest_stage_kernel(const uint8_t* __restrict__ in, uint64_t stride, uint32_t n, Digest* __restrict__ store, uint32_t base) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint8_t* p = in + (uint64_t)i * stride;
    uint32_t w[8];
#pragma unroll
    for (int k = 0; k < 8; ++k)
        w[k] = (uint32_t)p[4 * k] | ((uint32_t)p[4 * k + 1] << 8) | ((uint32_t)p[4 * k + 2] << 16) | ((uint32_t)p[4 * k + 3] << 24);
    Digest d;
    d.lo = make_uint4(w[0], w[1], w[2], w[3]);
    d.hi = make_uint4(w[4], w[5], w[6], w[7]);
    store[base + i] = d;
}

// claim: store[first .. first+n) enter the table; equal digests with index >= batch_base settle on the lowest index
__global__ void digest_claim_kernel(const Digest* __restrict__ store, uint32_t first, uint32_t n, uint32_t batch_base,
                                    uint32_t* __restrict__ table, uint64_t slots) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t idx = first + i;
    const Digest mine = store[idx];
    uint64_t slot = digest_slot(mine, slots);
    for (;;) {
        uint32_t cur = atomicCAS(&table[slot], kEmptySlot, idx);
        if (cur == kEmptySlot) return;
        if (digest_eq(store[cur], mine)) {
            if (cur >= batch_base && idx < cur) atomicMin(&table[slot], idx);
            return;
        }
        slot = (slot + 1) & (slots - 1);
    }
}

// read-only membership of staged digests (they sit in scratch, not in the store)
__global__ void digest_contains_kernel(const Digest* __restrict__ store, const Digest* __restrict__ probe, uint32_t n,
                                       const uint32_t* __restrict__ table, uint64_t slots, uint8_t* __restrict__ out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Digest mine = probe[i];
    uint64_t slot = digest_slot(mine, slots);
    uint8_t hit = 0;
    for (;;) {
        uint32_t cur = table[slot];
        if (cur == kEmptySlot) break;
        if (digest_eq(store[cur], mine)) { hit = 1; break; }
        slot = (slot + 1) & (slots - 1);
    }
    out[i] = hit;
}

// staged digests that are not in the table yet are appended to the store at base + pos[i] (pos = exclusive scan of
// fresh[]); slot_of[i] remembers the store index so that the resolve pass can tell "mine" from "an earlier twin"
__global__ void digest_fresh_flags_kernel(const uint8_t* __restrict__ present, uint32_t n, uint32_t* __restrict__ fresh) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) fresh[i] = present[i] ? 0u : 1u;
}
__global__ void digest_append_kernel(const Digest* __restrict__ probe, const uint32_t* __restrict__ fresh, const uint32_t* __restrict__ pos,
                                     uint32_t n, uint32_t base, Digest* __restrict__ store, uint32_t* __restrict__ index_of) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    if (fresh[i]) {
        store[base + pos[i]] = probe[i];
        index_of[i] = base + pos[i];
    } else {
        index_of[i] = kEmptySlot;
    }
}
// existed[i]: present before the call, or the table slot of its digest is owned by an earlier twin of this batch
__global__ void digest_resolve2_kernel(const Digest* __restrict__ store, const Digest* __restrict__ probe, const uint32_t* __restrict__ index_of,
                                       uint32_t n, const uint32_t* __restrict__ table, uint64_t slots, uint8_t* __restrict__ existed,
                                       unsigned long long* __restrict__ n_new) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    unsigned fresh = 0;
    if (i < n) {
        const uint32_t idx = index_of[i];
        if (idx != kEmptySlot) {
            const Digest mine = probe[i];
            uint64_t slot = digest_slot(mine, slots);
            for (;;) {
                uint32_t cur = table[slot];
                if (cur == idx) { fresh = 1; break; }
                if (cur == kEmptySlot) break;   // cannot happen after the claim pass
                if (digest_eq(store[cur], mine)) break;
                slot = (slot + 1) & (slots - 1);
            }
        }
        existed[i] = fresh ? 0 : 1;
    }
    unsigned m = __ballot_sync(0xffffffffu, fresh);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(n_new, (unsigned long long)__popc(m));
}

}  // namespace yb

using namespace yb;

struct yams_b200_digest_set {
    DeviceCtx* dev = nullptr;
    cudaStream_t st = nullptr;
    DevBuf store, table, stage, flags, probe, counter, fresh, pos, index_of, scan_scratch;
    HostBuf pin;
    uint64_t entries = 0;   // digests in `store`: every digest that was new when offered (+ twins inside one batch)
    uint64_t unique = 0;    // distinct digests == set size
    uint64_t slots = 0;
    float last_ms = 0.f;    // device time of the last insert/contains (staging + kernels, no PCIe)
    cudaEvent_t ev[2] = {nullptr, nullptr};
    std::mutex mu;
    // the stream is drained first, so the buffers may be freed in any order after it is destroyed
    ~yams_b200_digest_set() {
        if (st) cudaStreamSynchronize(st);
        for (auto& e : ev)
            if (e) cudaEventDestroy(e);
        if (st) cudaStreamDestroy(st);
    }
};

static yams_status_t set_grow(yams_b200_digest_set* s, uint64_t need_entries) {
    yams_status_t rc;
    YB_ARG(need_entries < 0xFFFFFFF0ull, "digest set is limited to 2^32 entries");
    if ((rc = s->store.reserve((size_t)need_entries * 32, true, s->st)) != YAMS_OK) return rc;
    uint64_t want = s->slots ? s->slots : 1024;
    while (want < 2 * need_entries) want <<= 1;
    if (want != s->slots) {
        // grow with headroom so that a stream of small batches rehashes O(log) times
        if (s->slots) want <<= 1;
        DevBuf nt;
        if ((rc = nt.reserve((size_t)want * 4)) != YAMS_OK) return rc;
        YB_CUDA(cudaMemsetAsync(nt.p, 0xFF, (size_t)want * 4, s->st));
        if (s->entries) {
            // batch_base = entries: no index is >= it, so equal digests simply keep whoever claimed first
            digest_claim_kernel<<<(unsigned)((s->entries + 255) / 256), 256, 0, s->st>>>(s->store.as<Digest>(), 0, (uint32_t)s->entries,
                                                                                        (uint32_t)s->entries, nt.as<uint32_t>(), want);
            YB_CUDA(cudaGetLastError());
        }
        YB_CUDA(cudaStreamSynchronize(s->st));
        s->table = std::move(nt);
        s->slots = want;
    }
    return YAMS_OK;
}

extern "C" {

yams_status_t yams_b200_digest_set_create(void* self, uint64_t capacity_hint, yams_b200_digest_set** out) {
    YB_TRY
    (void)self;
    YB_ARG(out, "out is null");
    *out = nullptr;
    DeviceCtx* dev = nullptr;
    yams_status_t rc = ensure_device(&dev);
    if (rc != YAMS_OK) return rc;
    std::unique_ptr<yams_b200_digest_set> s(new (std::nothrow) yams_b200_digest_set());
    YB_ARG(s, "out of memory");
    s->dev = dev;
    cudaError_t e = cudaStreamCreateWithFlags(&s->st, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreate(&s->ev[0]);
    if (e == cudaSuccess) e = cudaEventCreate(&s->ev[1]);
    if (e != cudaSuccess) {
        set_last_error("digest_set_create: %s", cudaGetErrorString(e));
        return YAMS_ERR_INTERNAL;
    }
    if ((rc = s->counter.reserve(8)) != YAMS_OK || (rc = set_grow(s.get(), capacity_hint ? capacity_hint : 1024)) != YAMS_OK) return rc;
    *out = s.release();
    return YAMS_OK;
    YB_CATCH
}

void yams_b200_digest_set_destroy(yams_b200_digest_set* s) { delete s; }

yams_status_t yams_b200_digest_set_size(yams_b200_digest_set* s, uint64_t* out) {
    YB_TRY
    YB_ARG(s && out, "null argument");
    std::lock_guard<std::mutex> lk(s->mu);
    *out = s->unique;
    return YAMS_OK;
    YB_CATCH
}

yams_status_t yams_b200_digest_set_insert(yams_b200_digest_set* s, const uint8_t* digests, size_t stride, size_t n,
                                          uint8_t* out_existed, uint64_t* out_new) {
    YB_TRY
    YB_ARG(s, "set is null");
    if (out_new) *out_new = 0;
    if (n == 0) return YAMS_OK;
    YB_ARG(digests && stride >= 32, "bad digests/stride");
    YB_ARG(n < (1ull << 31), "batch too large");
    std::lock_guard<std::mutex> lk(s->mu);
    YB_BIND(s);
    yams_status_t rc;
    // the store only ever receives digests that are not in the set yet, so re-offering known content (the common case
    // of a daily `yams add` over an unchanged tree) does not grow it
    if ((rc = set_grow(s, s->entries + n)) != YAMS_OK) return rc;
    const size_t in_bytes = (n - 1) * stride + 32;
    if ((rc = s->stage.reserve(in_bytes)) != YAMS_OK) return rc;
    if ((rc = s->probe.reserve(n * 32)) != YAMS_OK) return rc;
    if ((rc = s->flags.reserve(n)) != YAMS_OK) return rc;
    if ((rc = s->fresh.reserve(n * 4)) != YAMS_OK) return rc;
    if ((rc = s->pos.reserve(n * 4)) != YAMS_OK) return rc;
    if ((rc = s->index_of.reserve(n * 4)) != YAMS_OK) return rc;
    if ((rc = s->counter.reserve(16)) != YAMS_OK) return rc;
    cudaStream_t st = s->st;
    YB_CUDA(cudaMemcpyAsync(s->stage.p, digests, in_bytes, cudaMemcpyHostToDevice, st));
    unsigned long long* d_new = s->counter.as<unsigned long long>();
    uint64_t* d_total = reinterpret_cast<uint64_t*>(d_new + 1);
    YB_CUDA(cudaMemsetAsync(s->counter.p, 0, 16, st));
    const unsigned grid = (unsigned)((n + 255) / 256);
    const uint32_t base = (uint32_t)s->entries;
    YB_CUDA(cudaEventRecord(s->ev[0], st));
    digest_stage_kernel<<<grid, 256, 0, st>>>(s->stage.as<uint8_t>(), stride, (uint32_t)n, s->probe.as<Digest>(), 0);
    digest_contains_kernel<<<grid, 256, 0, st>>>(s->store.as<Digest>(), s->probe.as<Digest>(), (uint32_t)n, s->table.as<uint32_t>(),
                                                 s->slots, s->flags.as<uint8_t>());
    digest_fresh_flags_kernel<<<grid, 256, 0, st>>>(s->flags.as<uint8_t>(), (uint32_t)n, s->fresh.as<uint32_t>());
    if ((rc = exclusive_scan_u32(s->fresh.as<uint32_t>(), s->pos.as<uint32_t>(), n, d_total, s->scan_scratch, st)) != YAMS_OK) return rc;
    digest_append_kernel<<<grid, 256, 0, st>>>(s->probe.as<Digest>(), s->fresh.as<uint32_t>(), s->pos.as<uint32_t>(), (uint32_t)n, base,
                                               s->store.as<Digest>(), s->index_of.as<uint32_t>());
    uint64_t appended = 0;
    YB_CUDA(cudaMemcpyAsync(&appended, d_total, 8, cudaMemcpyDeviceToHost, st));
    YB_CUDA(cudaStreamSynchronize(st));
    if (appended) {
        digest_claim_kernel<<<(unsigned)((appended + 255) / 256), 256, 0, st>>>(s->store.as<Digest>(), base, (uint32_t)appended, base,
                                                                               s->table.as<uint32_t>(), s->slots);
    }
    digest_resolve2_kernel<<<grid, 256, 0, st>>>(s->store.as<Digest>(), s->probe.as<Digest>(), s->index_of.as<uint32_t>(), (uint32_t)n,
                                                 s->table.as<uint32_t>(), s->slots, s->flags.as<uint8_t>(), d_new);
    YB_CUDA(cudaEventRecord(s->ev[1], st));
    YB_CUDA(cudaGetLastError());
    unsigned long long fresh = 0;
    YB_CUDA(cudaMemcpyAsync(&fresh, d_new, 8, cudaMemcpyDeviceToHost, st));
    if (out_existed) YB_CUDA(cudaMemcpyAsync(out_existed, s->flags.p, n, cudaMemcpyDeviceToHost, st));
    YB_CUDA(cudaStreamSynchronize(st));
    cudaEventElapsedTime(&s->last_ms, s->ev[0], s->ev[1]);
    s->entries += appended;
    s->unique += fresh;
    if (out_new) *out_new = fresh;
    return YAMS_OK;
    YB_CATCH
}

yams_status_t yams_b200_digest_set_contains(yams_b200_digest_set* s, const uint8_t* digests, size_t stride, size_t n,
                                            uint8_t* out_exists) {
    YB_TRY
    YB_ARG(s, "set is null");
    if (n == 0) return YAMS_OK;
    YB_ARG(digests && stride >= 32 && out_exists, "bad argument");
    YB_ARG(n < (1ull << 31), "batch too large");
    std::lock_guard<std::mutex> lk(s->mu);
    YB_BIND(s);
    yams_status_t rc;
    const size_t in_bytes = (n - 1) * stride + 32;
    if ((rc = s->stage.reserve(in_bytes)) != YAMS_OK) return rc;
    if ((rc = s->probe.reserve(n * 32)) != YAMS_OK) return rc;
    if ((rc = s->flags.reserve(n)) != YAMS_OK) return rc;
    cudaStream_t st = s->st;
    YB_CUDA(cudaMemcpyAsync(s->stage.p, digests, in_bytes, cudaMemcpyHostToDevice, st));
    const unsigned grid = (unsigned)((n + 255) / 256);
    YB_CUDA(cudaEventRecord(s->ev[0], st));
    digest_stage_kernel<<<grid, 256, 0, st>>>(s->stage.as<uint8_t>(), stride, (uint32_t)n, s->probe.as<Digest>(), 0);
    digest_contains_kernel<<<grid, 256, 0, st>>>(s->store.as<Digest>(), s->probe.as<Digest>(), (uint32_t)n, s->table.as<uint32_t>(),
                                                 s->slots, s->flags.as<uint8_t>());
    YB_CUDA(cudaEventRecord(s->ev[1], st));
    YB_CUDA(cudaGetLastError());
    YB_CUDA(cudaMemcpyAsync(out_exists, s->flags.p, n, cudaMemcpyDeviceToHost, st));
    YB_CUDA(cudaStreamSynchronize(st));
    cudaEventElapsedTime(&s->last_ms, s->ev[0], s->ev[1]);
    return YAMS_OK;
    YB_CATCH
}

yams_status_t yams_b200_digest_set_last_ms(yams_b200_digest_set* s, float* out_ms) {
    YB_ARG(s && out_ms, "null argument");
    *out_ms = s->last_ms;
    return YAMS_OK;
}

}  // extern "C"
