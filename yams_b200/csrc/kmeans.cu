// kmeans.cu -- the k-means topology engine's spherical k-means on the device (yams_b200_topology_kmeans), bit-identical to
// the reference's runKMeans (src/topology/topology_alternate_engines.cpp:288-478, meanEmbedding topology_build_utils.h:27-56).
//
// Every distance is the reference's cosineDistance: dot, |a|^2 and |b|^2 accumulated in double in element order, 2.0 when a
// norm is <= 0, else 1 - clamp(dot / (sqrt(na) * sqrt(nb)), -1, 1) with a NaN kept.  Products of two floats are exact in
// double, so a fused multiply-add gives the same sums.  The assignment compares these doubles directly: two centroids whose
// distances differ below float resolution must still be told apart, so the float-ranked scan of knn.cu cannot serve it.
// Instead a CUDA-core fp64 tile kernel computes every (document, centroid) dot with its own sequential accumulator.
//
// Pipeline (DESIGN.md §4.10):
//   norms    |a|^2 of every document, once
//   init     farthest-first: k - 1 steps of (distance to the newest centroid, minDist update, (max, first index) reduction,
//            normalisation of the chosen document), enqueued back to back without a host synchronisation
//   iterate  assignment (fp64 tiles, first strictly smallest distance, NaN never chosen) -> stable partition of the documents
//            by cluster (device key sort) -> one float sum per (cluster, dim) in member order, the division and the
//            normalisation -> the first empty-cluster repair's exact pass -> one host synchronisation for the changed flag, the
//            cluster sizes and that pass's result -> the repairs, one exact pass per further empty cluster, in order
#include <cuda_fp16.h>
#include <float.h>
#include <math.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <vector>

#include "cosine.cuh"
#include "knn.cuh"

namespace yb {

constexpr uint32_t kNone = 0xFFFFFFFFu;
constexpr int kRedThreads = 256;   // argmax kernels
constexpr int kPickThreads = 1024;

// cosineDistance from its three sums (std::clamp keeps a NaN)
__device__ __forceinline__ double km_distance(double dot, double na, double nb) {
    if (na <= 0.0 || nb <= 0.0) return 2.0;
    const double cs = dot / (sqrt(na) * sqrt(nb));
    return 1.0 - (cs < -1.0 ? -1.0 : (1.0 < cs ? 1.0 : cs));
}

// (value, index) argmax with the first index on ties; value -1 with index kNone is "none" (the reference starts at -1.0 and
// compares with a strict >, so a NaN is never taken)
struct ArgMax {
    double v;
    uint32_t i;
};
__device__ __forceinline__ ArgMax better_of(ArgMax a, ArgMax b) {
    if (b.v > a.v || (b.v == a.v && b.i < a.i)) return b;
    return a;
}
template <int NT>
__device__ ArgMax block_argmax(ArgMax m) {
    __shared__ double sv[NT / 32];
    __shared__ uint32_t si[NT / 32];
    for (int o = 16; o > 0; o >>= 1) {
        ArgMax t;
        t.v = __shfl_xor_sync(0xFFFFFFFFu, m.v, o);
        t.i = __shfl_xor_sync(0xFFFFFFFFu, m.i, o);
        m = better_of(m, t);
    }
    const int w = threadIdx.x >> 5;
    __syncthreads();
    if ((threadIdx.x & 31) == 0) { sv[w] = m.v; si[w] = m.i; }
    __syncthreads();
    m = {sv[0], si[0]};
    for (int j = 1; j < NT / 32; ++j) m = better_of(m, ArgMax{sv[j], si[j]});
    return m;
}

// normalized(): out = v * float(1 / sqrt(sum (double)v^2)) (v unchanged when the sum is <= 0) and *out_norm = the sum of
// squares of out, both in element order.  v is the block's shared vector; every thread calls it.
__device__ void block_normalize(float* v, uint32_t d, float* __restrict__ out, double* __restrict__ out_norm) {
    __shared__ float s_inv;
    __shared__ int s_scale;
    __syncthreads();
    if (threadIdx.x == 0) {
        double norm = 0.0;
        for (uint32_t i = 0; i < d; ++i) norm += (double)v[i] * (double)v[i];
        s_scale = norm > 0.0;
        s_inv = (float)(1.0 / sqrt(norm));
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < d; i += blockDim.x) {
        const float x = s_scale ? v[i] * s_inv : v[i];
        v[i] = x;
        out[i] = x;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double nb = 0.0;
        for (uint32_t i = 0; i < d; ++i) nb += (double)v[i] * (double)v[i];
        *out_norm = nb;
    }
}

__global__ void km_norms_kernel(const void* __restrict__ rows, int dtype, uint32_t d, uint32_t n, double* __restrict__ na) {
    const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= n) return;
    double a = 0.0;
    walk_row(rows, dtype, d, u, [&](float x) { a += (double)x * x; });
    na[u] = a;
}

// Farthest-first step against centroid `cent` (norm cnorm): minDist[u] = min(minDist[u], d) (strict <) for the unselected
// documents, and per block the first unselected u with the largest minDist -> part[blockIdx]
__global__ void __launch_bounds__(kRedThreads) km_far_step_kernel(const void* __restrict__ rows, int dtype, uint32_t d, uint32_t n,
                                                                  const double* __restrict__ na, const uint8_t* __restrict__ selected,
                                                                  const float* __restrict__ cent, const double* __restrict__ cnorm,
                                                                  double* __restrict__ min_dist, ArgMax* __restrict__ part) {
    const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
    ArgMax m{-1.0, kNone};
    if (u < n && !selected[u]) {
        double dot = 0.0;
        walk_row_pair(rows, dtype, d, u, cent, [&](float x, float y) { dot += (double)x * y; });
        const double dist = km_distance(dot, na[u], *cnorm);
        double md = min_dist[u];
        if (dist < md) { md = dist; min_dist[u] = md; }
        m = {md, u};
    }
    m = block_argmax<kRedThreads>(m);
    if (threadIdx.x == 0) part[blockIdx.x] = m;
}

// the block-wide (max, first index) of nparts partial results
__device__ ArgMax reduce_parts(const ArgMax* __restrict__ part, uint32_t nparts) {
    ArgMax m{-1.0, kNone};
    for (uint32_t j = threadIdx.x; j < nparts; j += kPickThreads) m = better_of(m, part[j]);
    return block_argmax<kPickThreads>(m);
}

// Farthest-first pick: centroid slot s = normalized(document f), f the reduction of the step's partials (nparts == 0: f = 0,
// the first centroid); f becomes selected
__global__ void __launch_bounds__(kPickThreads) km_far_pick_kernel(const void* __restrict__ rows, int dtype, uint32_t d,
                                                                   const ArgMax* __restrict__ part, uint32_t nparts,
                                                                   uint8_t* __restrict__ selected, float* __restrict__ cent,
                                                                   double* __restrict__ cnorm) {
    extern __shared__ float km_vec[];
    __shared__ uint32_t s_f;
    const ArgMax m = nparts ? reduce_parts(part, nparts) : ArgMax{0.0, 0};
    if (threadIdx.x == 0) { s_f = m.i; selected[m.i] = 1; }
    __syncthreads();
    const uint32_t f = s_f;
    for (uint32_t i = threadIdx.x; i < d; i += kPickThreads) km_vec[i] = load_elem(rows, dtype, (uint64_t)f * d + i);
    block_normalize(km_vec, d, cent, cnorm);
}

// Assignment: nearestCentroid of every document -- the first centroid with the strictly smallest distance, 0 when every
// distance is NaN.  A 64 x 64 tile of (document, centroid) pairs per step, each pair's dot in its own double accumulator fed in
// element order from shared memory; the CTA walks every centroid tile for its 64 documents.  changed = 1 when a membership moves.
constexpr int AS_BM = 64, AS_BN = 64, AS_BK = 16, AS_T = 256;
__global__ void __launch_bounds__(AS_T) km_assign_kernel(const void* __restrict__ rows, int dtype, uint32_t d, uint32_t n,
                                                         const double* __restrict__ na, const float* __restrict__ cent,
                                                         const double* __restrict__ cnorm, uint32_t k, uint32_t* __restrict__ membership,
                                                         uint32_t* __restrict__ changed) {
    __shared__ double As[AS_BK][AS_BM];
    __shared__ double Bs[AS_BK][AS_BN];
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const uint64_t u0 = (uint64_t)blockIdx.x * AS_BM;
    double best[4];
    uint32_t bestc[4];
    double nau[4];
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        best[a] = DBL_MAX;
        bestc[a] = kNone;
        const uint64_t u = u0 + ty + 16 * a;
        nau[a] = u < n ? na[u] : 0.0;
    }
    for (uint32_t c0 = 0; c0 < k; c0 += AS_BN) {
        double acc[4][4];
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
        for (uint32_t k0 = 0; k0 < d; k0 += AS_BK) {
            const int kl = (int)min((uint32_t)AS_BK, d - k0);
            for (int e = threadIdx.x; e < AS_BM * AS_BK; e += AS_T) {
                const int r = e / AS_BK, kk = e % AS_BK;
                const uint64_t u = u0 + r;
                As[kk][r] = (u < n && kk < kl) ? (double)load_elem(rows, dtype, u * d + k0 + kk) : 0.0;
                const uint32_t c = c0 + r;
                Bs[kk][r] = (c < k && kk < kl) ? (double)cent[(uint64_t)c * d + k0 + kk] : 0.0;
            }
            __syncthreads();
            for (int kk = 0; kk < kl; ++kk) {
                double av[4], bv[4];
#pragma unroll
                for (int a = 0; a < 4; ++a) av[a] = As[kk][ty + 16 * a];
#pragma unroll
                for (int b = 0; b < 4; ++b) bv[b] = Bs[kk][tx + 16 * b];
#pragma unroll
                for (int a = 0; a < 4; ++a)
#pragma unroll
                    for (int b = 0; b < 4; ++b) acc[a][b] = fma(av[a], bv[b], acc[a][b]);   // the product is exact
            }
            __syncthreads();
        }
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            const uint32_t c = c0 + tx + 16 * b;
            if (c >= k) continue;
            const double nb = cnorm[c];
#pragma unroll
            for (int a = 0; a < 4; ++a) {
                const double dist = km_distance(acc[a][b], nau[a], nb);
                if (dist < best[a]) { best[a] = dist; bestc[a] = c; }
            }
        }
    }
    // the 16 threads of a row of the tile hold disjoint centroid subsets, each ascending: (smallest, first index) across them
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        double bd = best[a];
        uint32_t bc = bestc[a];
        for (int o = 8; o > 0; o >>= 1) {
            const double od = __shfl_xor_sync(0xFFFFFFFFu, bd, o);
            const uint32_t oc = __shfl_xor_sync(0xFFFFFFFFu, bc, o);
            if (oc != kNone && (bc == kNone || od < bd || (od == bd && oc < bc))) { bd = od; bc = oc; }
        }
        const uint64_t u = u0 + ty + 16 * a;
        if (tx == 0 && u < n) {
            const uint32_t c = bc == kNone ? 0u : bc;
            if (membership[u] != c) { membership[u] = c; *changed = 1u; }
        }
    }
}

// stable partition: key (~cluster, ~u) sorted descending is (cluster asc, u asc); padding keys are 0
__global__ void km_keys_kernel(const uint32_t* __restrict__ membership, uint32_t n, uint64_t np2, uint64_t* __restrict__ keys,
                               uint32_t* __restrict__ count) {
    for (uint64_t u = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; u < np2; u += (uint64_t)gridDim.x * blockDim.x) {
        if (u < n) {
            const uint32_t c = membership[u];
            keys[u] = ((uint64_t)~c << 32) | (uint64_t)(~(uint32_t)u);
            atomicAdd(count + c, 1u);
        } else {
            keys[u] = 0;
        }
    }
}
__device__ __forceinline__ uint32_t key_cluster(uint64_t key) { return ~(uint32_t)(key >> 32); }
__device__ __forceinline__ uint32_t key_doc(uint64_t key) { return ~(uint32_t)key; }
// start[c] = the first position of cluster c in the sorted keys
__global__ void km_starts_kernel(const uint64_t* __restrict__ keys, uint32_t n, uint32_t* __restrict__ start) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t c = key_cluster(keys[i]);
        if (i == 0 || key_cluster(keys[i - 1]) != c) start[c] = (uint32_t)i;
    }
}

// meanEmbedding() of cluster cl = *only (grid.x == 1), else blockIdx.x, one thread per dim: the cluster's partition range
// restricted to the documents still in cl (an empty-cluster repair takes one out), a float sum per dim in member order from
// +0, then / float(count) -> mean[cl][dim].  A cluster without members is skipped (it keeps its centroid).
constexpr int MEAN_T = 64;
__global__ void __launch_bounds__(MEAN_T) km_mean_kernel(const void* __restrict__ rows, int dtype, uint32_t d, const uint64_t* __restrict__ keys,
                                                         const uint32_t* __restrict__ start, const uint32_t* __restrict__ part_count,
                                                         const uint32_t* __restrict__ membership, const uint32_t* __restrict__ only,
                                                         float* __restrict__ mean) {
    const uint32_t cl = only ? *only : blockIdx.x;
    const uint32_t i = blockIdx.y * MEAN_T + threadIdx.x;
    if (cl == kNone || i >= d) return;
    const uint32_t cnt = part_count[cl];
    if (cnt == 0) return;
    const uint64_t* mk = keys + start[cl];
    float s = 0.f;
    uint32_t members = 0;
#pragma unroll 4
    for (uint32_t j = 0; j < cnt; ++j) {
        const uint32_t u = key_doc(mk[j]);
        if (only && membership[u] != cl) continue;
        s += load_elem(rows, dtype, (uint64_t)u * d + i);
        ++members;
    }
    mean[(uint64_t)cl * d + i] = s / (float)members;
}

// centroidOf() = normalized(mean[cl]) for the clusters km_mean_kernel wrote (same cl rule, one block each)
__global__ void km_normalize_kernel(const float* __restrict__ mean, uint32_t d, const uint32_t* __restrict__ part_count,
                                    const uint32_t* __restrict__ only, float* __restrict__ cent, double* __restrict__ cnorm) {
    extern __shared__ float km_vec[];
    const uint32_t cl = only ? *only : blockIdx.x;
    if (cl == kNone || part_count[cl] == 0) return;
    for (uint32_t i = threadIdx.x; i < d; i += blockDim.x) km_vec[i] = mean[(uint64_t)cl * d + i];
    block_normalize(km_vec, d, cent + (uint64_t)cl * d, cnorm + cl);
}

// Empty-cluster repair scan: per block, the first document with the strictly largest distance to its own centroid among
// clusters of more than one member -> part[blockIdx]
__global__ void __launch_bounds__(kRedThreads) km_repair_scan_kernel(const void* __restrict__ rows, int dtype, uint32_t d, uint32_t n,
                                                                     const double* __restrict__ na, const uint32_t* __restrict__ membership,
                                                                     const uint32_t* __restrict__ size, const float* __restrict__ cent,
                                                                     const double* __restrict__ cnorm, ArgMax* __restrict__ part) {
    const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
    ArgMax m{-1.0, kNone};
    if (u < n) {
        const uint32_t mc = membership[u];
        if (size[mc] > 1) {
            double dot = 0.0;
            walk_row_pair(rows, dtype, d, u, cent + (uint64_t)mc * d, [&](float x, float y) { dot += (double)x * y; });
            const double dist = km_distance(dot, na[u], cnorm[mc]);
            if (dist > -1.0) m = {dist, u};
        }
    }
    m = block_argmax<kRedThreads>(m);
    if (threadIdx.x == 0) part[blockIdx.x] = m;
}

// the (max, first index) of a repair scan's partials -> *worst
__global__ void __launch_bounds__(kPickThreads) km_reduce_kernel(const ArgMax* __restrict__ part, uint32_t nparts, ArgMax* __restrict__ worst) {
    const ArgMax m = reduce_parts(part, nparts);
    if (threadIdx.x == 0) *worst = m;
}

// Empty-cluster repair move: the worst document w joins the empty cluster c, whose centroid becomes normalized(w); *donor = its
// old cluster (kNone when no document qualifies, and nothing changes)
__global__ void __launch_bounds__(kPickThreads) km_repair_move_kernel(const void* __restrict__ rows, int dtype, uint32_t d, uint32_t c,
                                                                      const ArgMax* __restrict__ worst, uint32_t* __restrict__ membership,
                                                                      uint32_t* __restrict__ size, float* __restrict__ cent,
                                                                      double* __restrict__ cnorm, uint32_t* __restrict__ donor) {
    extern __shared__ float km_vec[];
    const ArgMax m = *worst;
    if (m.i == kNone) {
        if (threadIdx.x == 0) *donor = kNone;
        return;
    }
    if (threadIdx.x == 0) {
        const uint32_t from = membership[m.i];
        *donor = from;
        size[from] -= 1;
        size[c] = 1;
        membership[m.i] = c;
    }
    for (uint32_t i = threadIdx.x; i < d; i += kPickThreads) km_vec[i] = load_elem(rows, dtype, (uint64_t)m.i * d + i);
    block_normalize(km_vec, d, cent + (uint64_t)c * d, cnorm + c);
}

}  // namespace yb

using namespace yb;

yams_status_t yams_b200_topology_kmeans(yams_b200_corpus* c, uint32_t k_requested, uint32_t max_iterations, uint32_t* out_assignment,
                                        float* out_centroids, uint32_t* out_k, uint32_t* out_iterations) {
    YB_TRY
    YB_ARG(c && out_assignment && out_k && out_iterations, "null argument");
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    YB_BIND(c);
    settle_pending(c);
    YB_ARG(c->metric == YAMS_B200_COSINE, "k-means clusters a cosine corpus");
    YB_ARG(c->n < 0xFFFFFFFFull, "at most 2^32 - 2 documents");
    const uint32_t n = (uint32_t)c->n, d = c->dim;
    for (int i = 0; i < 4; ++i) c->kmeans_ms[i] = 0.f;
    *out_k = 0;
    *out_iterations = 0;
    if (n < 2) {   // runKMeans: fewer than 2 usable documents -> every document is its own cluster
        for (uint32_t i = 0; i < n; ++i) out_assignment[i] = i;
        return YAMS_OK;
    }
    const auto t0 = std::chrono::steady_clock::now();
    uint64_t k64 = k_requested ? k_requested : (uint64_t)std::llround(std::sqrt((double)n));
    const uint32_t k = (uint32_t)std::min<uint64_t>(std::max<uint64_t>(k64, 2), n);
    const uint32_t iterations = max_iterations == 0 ? 10 : max_iterations;
    const uint64_t np2 = pow2_at_least((uint64_t)n);
    const uint32_t nblk = (n + kRedThreads - 1) / kRedThreads;
    // workspace, 256-byte aligned pieces of c->kmeans
    size_t off = 0;
    auto carve = [&](size_t bytes) { const size_t o = off; off += (bytes + 255) & ~size_t(255); return o; };
    const size_t o_keys = carve(np2 * 8), o_na = carve((size_t)n * 8), o_min = carve((size_t)n * 8), o_mem = carve((size_t)n * 4),
                 o_sel = carve(n), o_cent = carve((size_t)k * d * 4), o_mean = carve((size_t)k * d * 4), o_cnorm = carve((size_t)k * 8),
                 o_cnt = carve((size_t)k * 4), o_size = carve((size_t)k * 4), o_start = carve((size_t)k * 4),
                 o_part = carve((size_t)nblk * sizeof(ArgMax)), o_worst = carve(sizeof(ArgMax)), o_flag = carve(16);
    yams_status_t rc;
    if ((rc = c->kmeans.reserve(off)) != YAMS_OK) return rc;
    char* base = c->kmeans.as<char>();
    uint64_t* keys = reinterpret_cast<uint64_t*>(base + o_keys);
    double* na = reinterpret_cast<double*>(base + o_na);
    double* min_dist = reinterpret_cast<double*>(base + o_min);
    uint32_t* membership = reinterpret_cast<uint32_t*>(base + o_mem);
    uint8_t* selected = reinterpret_cast<uint8_t*>(base + o_sel);
    float* cent = reinterpret_cast<float*>(base + o_cent);
    float* mean = reinterpret_cast<float*>(base + o_mean);
    double* cnorm = reinterpret_cast<double*>(base + o_cnorm);
    uint32_t* count = reinterpret_cast<uint32_t*>(base + o_cnt);   // partition sizes
    uint32_t* size = reinterpret_cast<uint32_t*>(base + o_size);   // live sizes during the repairs
    uint32_t* start = reinterpret_cast<uint32_t*>(base + o_start);
    ArgMax* part = reinterpret_cast<ArgMax*>(base + o_part);
    ArgMax* worst = reinterpret_cast<ArgMax*>(base + o_worst);
    uint32_t* flags = reinterpret_cast<uint32_t*>(base + o_flag);   // [0] changed, [1] repair donor
    // pinned read-back of a round: changed flag, the first repair's worst document, the partition sizes
    if ((rc = c->h_pin.reserve((size_t)k * 4 + 32)) != YAMS_OK) return rc;
    uint32_t* h_changed = c->h_pin.as<uint32_t>();
    ArgMax* h_worst = reinterpret_cast<ArgMax*>(c->h_pin.as<char>() + 16);
    uint32_t* h_count = reinterpret_cast<uint32_t*>(c->h_pin.as<char>() + 32);
    cudaStream_t st = c->st;
    const size_t vec_smem = (size_t)d * 4;
    if (vec_smem > 48 * 1024) {
        YB_CUDA(cudaFuncSetAttribute(km_far_pick_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)vec_smem));
        YB_CUDA(cudaFuncSetAttribute(km_normalize_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)vec_smem));
        YB_CUDA(cudaFuncSetAttribute(km_repair_move_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)vec_smem));
    }
    constexpr int kEv = 7;
    cudaEvent_t ev[kEv];
    for (auto& e : ev) YB_CUDA(cudaEventCreate(&e));
    struct EvGuard { cudaEvent_t* e; ~EvGuard() { for (int i = 0; i < kEv; ++i) cudaEventDestroy(e[i]); } } ev_guard{ev};
    const void* rows = c->rows.p;
    const int dt = c->dtype;
    const dim3 mean_grid(k, (d + MEAN_T - 1) / MEAN_T), one_mean_grid(1, (d + MEAN_T - 1) / MEAN_T);
    float ms = 0.f;

    // init: |a|^2, then farthest-first
    YB_CUDA(cudaEventRecord(ev[0], st));
    km_norms_kernel<<<nblk, kRedThreads, 0, st>>>(rows, dt, d, n, na);
    YB_CUDA(cudaMemsetAsync(selected, 0, n, st));
    YB_CUDA(cudaMemsetAsync(membership, 0, (size_t)n * 4, st));
    std::vector<double> dbl_max(n, DBL_MAX);
    YB_CUDA(cudaMemcpyAsync(min_dist, dbl_max.data(), (size_t)n * 8, cudaMemcpyHostToDevice, st));
    km_far_pick_kernel<<<1, kPickThreads, vec_smem, st>>>(rows, dt, d, part, 0, selected, cent, cnorm);
    for (uint32_t s = 1; s < k; ++s) {
        km_far_step_kernel<<<nblk, kRedThreads, 0, st>>>(rows, dt, d, n, na, selected, cent + (size_t)(s - 1) * d, cnorm + (s - 1),
                                                          min_dist, part);
        km_far_pick_kernel<<<1, kPickThreads, vec_smem, st>>>(rows, dt, d, part, nblk, selected, cent + (size_t)s * d, cnorm + s);
    }
    YB_CUDA(cudaGetLastError());
    YB_CUDA(cudaEventRecord(ev[1], st));

    // Rounds.  The round's one host synchronisation reads the changed flag, the cluster sizes and the first empty-cluster
    // repair's worst document, whose scan is enqueued before it on every round: repairs see the same state until one succeeds,
    // so when the first finds no document none does, and when it finds one the round has changed.
    bool repairs_timed = false;   // ev[5] -> ev[6] bracket repairs whose time is not yet added
    uint32_t iter = 0;
    while (iter < iterations) {
        ++iter;
        YB_CUDA(cudaMemsetAsync(flags, 0, 16, st));
        YB_CUDA(cudaEventRecord(ev[2], st));
        km_assign_kernel<<<(n + AS_BM - 1) / AS_BM, AS_T, 0, st>>>(rows, dt, d, n, na, cent, cnorm, k, membership, flags);
        YB_CUDA(cudaEventRecord(ev[3], st));
        YB_CUDA(cudaMemsetAsync(count, 0, (size_t)k * 4, st));
        km_keys_kernel<<<key_grid(np2), 256, 0, st>>>(membership, n, np2, keys, count);
        sort_keys_desc(keys, np2, st);
        km_starts_kernel<<<key_grid(n), 256, 0, st>>>(keys, n, start);
        km_mean_kernel<<<mean_grid, MEAN_T, 0, st>>>(rows, dt, d, keys, start, count, membership, nullptr, mean);
        km_normalize_kernel<<<k, 128, vec_smem, st>>>(mean, d, count, nullptr, cent, cnorm);
        YB_CUDA(cudaMemcpyAsync(size, count, (size_t)k * 4, cudaMemcpyDeviceToDevice, st));
        km_repair_scan_kernel<<<nblk, kRedThreads, 0, st>>>(rows, dt, d, n, na, membership, size, cent, cnorm, part);
        km_reduce_kernel<<<1, kPickThreads, 0, st>>>(part, nblk, worst);
        YB_CUDA(cudaGetLastError());
        YB_CUDA(cudaEventRecord(ev[4], st));
        YB_CUDA(cudaMemcpyAsync(h_changed, flags, 4, cudaMemcpyDeviceToHost, st));
        YB_CUDA(cudaMemcpyAsync(h_worst, worst, sizeof(ArgMax), cudaMemcpyDeviceToHost, st));
        YB_CUDA(cudaMemcpyAsync(h_count, count, (size_t)k * 4, cudaMemcpyDeviceToHost, st));
        YB_CUDA(cudaStreamSynchronize(st));
        if (iter == 1) YB_CUDA(cudaEventElapsedTime(&c->kmeans_ms[0], ev[0], ev[1]));
        YB_CUDA(cudaEventElapsedTime(&ms, ev[2], ev[3]));
        c->kmeans_ms[1] += ms;
        YB_CUDA(cudaEventElapsedTime(&ms, ev[3], ev[4]));
        c->kmeans_ms[2] += ms;
        if (repairs_timed) {
            YB_CUDA(cudaEventElapsedTime(&ms, ev[5], ev[6]));
            c->kmeans_ms[2] += ms;
            repairs_timed = false;
        }
        bool changed = h_changed[0] != 0;
        if (h_worst->i != kNone) {
            bool first = true;
            for (uint32_t e = 0; e < k; ++e) {
                if (h_count[e] != 0) continue;
                if (first) YB_CUDA(cudaEventRecord(ev[5], st));
                if (!first) {
                    km_repair_scan_kernel<<<nblk, kRedThreads, 0, st>>>(rows, dt, d, n, na, membership, size, cent, cnorm, part);
                    km_reduce_kernel<<<1, kPickThreads, 0, st>>>(part, nblk, worst);
                }
                km_repair_move_kernel<<<1, kPickThreads, vec_smem, st>>>(rows, dt, d, e, worst, membership, size, cent, cnorm, flags + 1);
                km_mean_kernel<<<one_mean_grid, MEAN_T, 0, st>>>(rows, dt, d, keys, start, count, membership, flags + 1, mean);
                km_normalize_kernel<<<1, 128, vec_smem, st>>>(mean, d, count, flags + 1, cent, cnorm);
                first = false;
                changed = true;
            }
            YB_CUDA(cudaGetLastError());
            if (!first) {
                YB_CUDA(cudaEventRecord(ev[6], st));
                repairs_timed = true;
            }
        }
        if (!changed) break;
    }
    YB_CUDA(cudaMemcpyAsync(out_assignment, membership, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
    if (out_centroids) YB_CUDA(cudaMemcpyAsync(out_centroids, cent, (size_t)k * d * 4, cudaMemcpyDeviceToHost, st));
    YB_CUDA(cudaStreamSynchronize(st));
    if (repairs_timed) {
        YB_CUDA(cudaEventElapsedTime(&ms, ev[5], ev[6]));
        c->kmeans_ms[2] += ms;
    }
    *out_k = k;
    *out_iterations = iter;
    c->kmeans_ms[3] = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return YAMS_OK;
    YB_CATCH
}

yams_status_t yams_b200_topology_kmeans_last_timings(yams_b200_corpus* c, float out_ms[4]) {
    YB_TRY
    YB_ARG(c && out_ms, "null argument");
    std::lock_guard<std::mutex> corpus_lock(c->mu);
    for (int i = 0; i < 4; ++i) out_ms[i] = c->kmeans_ms[i];
    return YAMS_OK;
    YB_CATCH
}
