// common.cuh -- shared helpers for libyams_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <atomic>
#include <exception>
#include <new>
#include <type_traits>
#include <utility>

#include <string>

#include "../../include/yams_b200.h"

namespace yb {

// thread-local last error text (exposed through yams_b200_last_error / health JSON)
void set_last_error(const char* fmt, ...);
const char* last_error();
void note_global_error(const char* text);  // remembered for yams_plugin_get_health_json

#define YB_CUDA(expr)                                                                        \
    do {                                                                                     \
        cudaError_t _e = (expr);                                                             \
        if (_e != cudaSuccess) {                                                             \
            ::yb::set_last_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),     \
                                 __FILE__, __LINE__);                                        \
            return YAMS_ERR_INTERNAL;                                                        \
        }                                                                                    \
    } while (0)

#define YB_ARG(cond, msg)                                   \
    do {                                                    \
        if (!(cond)) {                                      \
            ::yb::set_last_error("invalid argument: %s", msg); \
            return YAMS_ERR_INVALID_ARG;                    \
        }                                                   \
    } while (0)

// No exception may cross the C boundary (the reference catches at its C entry points too,
// third_party/sqlite-vec-cpp/src/sqlite_vec_c_api.cpp:30-53): host-side allocations (std::vector, std::thread) inside an
// extern "C" entry are wrapped by YB_TRY ... YB_CATCH.
#define YB_TRY try {
#define YB_CATCH                                                      \
    }                                                                 \
    catch (const std::bad_alloc&) {                                   \
        ::yb::set_last_error("out of host memory");                   \
        return YAMS_ERR_INTERNAL;                                     \
    }                                                                 \
    catch (const std::exception& e) {                                 \
        ::yb::set_last_error("unexpected host exception: %s", e.what()); \
        return YAMS_ERR_INTERNAL;                                     \
    }

// Bytes currently held by every DevBuf / HostBuf of the process (reported by yams_plugin_get_health_json): a GPU's free
// memory is shared with other processes, these counters are exact for this one.
extern std::atomic<uint64_t> g_device_buffer_bytes, g_pinned_buffer_bytes;

// Growable device buffer (never shrinks); contents are NOT preserved across growth unless asked.  It owns its allocation:
// freed on destruction, moved but never copied.
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
    DevBuf& operator=(DevBuf&& o) noexcept {
        if (this != &o) {
            release();
            p = o.p; cap = o.cap;
            o.p = nullptr; o.cap = 0;
        }
        return *this;
    }
    ~DevBuf() { release(); }
    yams_status_t reserve(size_t bytes, bool preserve = false, cudaStream_t st = 0) {
        if (bytes <= cap) return YAMS_OK;
        size_t ncap = cap ? cap : 256;
        while (ncap < bytes) ncap += ncap / 2 + 256;
        ncap = (ncap + 255) & ~size_t(255);
        void* np = nullptr;
        YB_CUDA(cudaMalloc(&np, ncap));
        g_device_buffer_bytes += ncap;
        DevBuf nb;   // frees the new allocation if the copy below fails
        nb.p = np;
        nb.cap = ncap;
        if (preserve && p && cap) {
            YB_CUDA(cudaMemcpyAsync(nb.p, p, cap, cudaMemcpyDeviceToDevice, st));
            YB_CUDA(cudaStreamSynchronize(st));
        }
        *this = std::move(nb);
        return YAMS_OK;
    }
    void release() {
        if (p) cudaFree(p);
        g_device_buffer_bytes -= cap;
        p = nullptr;
        cap = 0;
    }
    template <typename T> T* as() const { return reinterpret_cast<T*>(p); }
};

// Pinned host buffer; owns its allocation like DevBuf.
struct HostBuf {
    void* p = nullptr;
    size_t cap = 0;
    HostBuf() = default;
    HostBuf(HostBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
    HostBuf& operator=(HostBuf&& o) noexcept {
        if (this != &o) {
            release();
            p = o.p; cap = o.cap;
            o.p = nullptr; o.cap = 0;
        }
        return *this;
    }
    ~HostBuf() { release(); }
    yams_status_t reserve(size_t bytes) {
        if (bytes <= cap) return YAMS_OK;
        release();
        size_t ncap = (bytes + 4095) & ~size_t(4095);
        YB_CUDA(cudaMallocHost(&p, ncap));
        cap = ncap;
        g_pinned_buffer_bytes += ncap;
        return YAMS_OK;
    }
    void release() {
        if (p) cudaFreeHost(p);
        g_pinned_buffer_bytes -= cap;
        p = nullptr;
        cap = 0;
    }
    template <typename T> T* as() const { return reinterpret_cast<T*>(p); }
};

static_assert(!std::is_copy_constructible<DevBuf>::value && !std::is_copy_assignable<DevBuf>::value, "a DevBuf is never copied");
static_assert(std::is_nothrow_move_constructible<DevBuf>::value && std::is_nothrow_move_assignable<DevBuf>::value, "DevBuf moves");
static_assert(!std::is_copy_constructible<HostBuf>::value && !std::is_copy_assignable<HostBuf>::value, "a HostBuf is never copied");
static_assert(std::is_nothrow_move_constructible<HostBuf>::value && std::is_nothrow_move_assignable<HostBuf>::value, "HostBuf moves");

// Per-plugin device context: which GPU, SM count, init state.
struct DeviceCtx {
    int device = -1;
    int sm_count = 0;
    int cc_major = 0, cc_minor = 0;
    bool ok = false;
};
// Lazily initialises (cudaSetDevice) and validates sm_90; returns YAMS_ERR_INTERNAL when no
// usable GPU exists -- there is no CPU fallback.
yams_status_t ensure_device(DeviceCtx** out);
void set_requested_device(int dev);

// Every handle-based entry point binds the handle's device on the calling thread first (the header promises "any host
// thread"; a fresh thread starts on device 0 whatever the plugin was initialised with).
#define YB_BIND(h)                                                   \
    do {                                                             \
        if ((h)->dev) cudaSetDevice((h)->dev->device);               \
    } while (0)

// Pooled workspace of the small host-pointer operators (pairwise distances, computeCosineSimilarity, vec0_exact,
// batch_distance): a stream, a few growable device buffers and one pinned staging buffer, parked between calls so that
// no call pays cudaMalloc / cudaStreamCreate.  Concurrent callers get separate workspaces.
struct OpWs {
    cudaStream_t st = nullptr;
    DevBuf d[8];
    HostBuf h;
    // the stream is drained first, so the buffers may be freed after it is destroyed
    ~OpWs() {
        if (st) {
            cudaStreamSynchronize(st);
            cudaStreamDestroy(st);
        }
    }
};
OpWs* opws_acquire();             // nullptr (+ last error set) when no device / stream can be had
void opws_release(OpWs* w);
struct OpWsLease {
    OpWs* w;
    OpWsLease() : w(opws_acquire()) {}
    ~OpWsLease() { if (w) opws_release(w); }
    OpWsLease(const OpWsLease&) = delete;
    OpWsLease& operator=(const OpWsLease&) = delete;
};

// exclusive scan of n uint32 values (in may alias out); *d_total (device, uint64) receives the sum
yams_status_t exclusive_scan_u32(const uint32_t* d_in, uint32_t* d_out, size_t n, uint64_t* d_total,
                                 DevBuf& scratch, cudaStream_t st);

__device__ __forceinline__ uint4 ldg_stream_u4(const void* p) {
    // streaming 128-bit load: read once, do not pollute L1
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ULL;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ULL;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBULL;
    return x ^ (x >> 31);
}

}  // namespace yb
