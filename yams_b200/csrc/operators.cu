// operators.cu -- the stateless sqlite-vec-cpp operator surface of libyams_b200.so: pairwise distances
// (sqlite3_vec_distance_l2 / _cosine, yams_b200_vec_distance_l1), vec0_run_exact_query (yams_b200_vec0_exact), batch distances
// (yams_b200_batch_distance) and computeCosineSimilarity[_many].  None of them touches a corpus: every call runs on a pooled
// OpWs workspace (api.cu).
//
// Reference semantics matched:
//   pairwise C API                 third_party/sqlite-vec-cpp/src/sqlite_vec_c_api.cpp:57-105
//   vec0_run_exact_query           third_party/sqlite-vec-cpp/.../sqlite/vec0_module.hpp:376-430
//   batch distances                third_party/sqlite-vec-cpp/.../distances/batch.hpp:24-146
//   computeCosineSimilarity        src/vector/vector_database.cpp:1786-1810
#include <algorithm>
#include <vector>

#include "cosine.cuh"
#include "knn.cuh"
#include "ref_order.cuh"

namespace yb {

// pairwise operators of the sqlite-vec-cpp C API: one thread evaluates the pair in the reference build's operation order
__global__ void pair_distance_kernel(const float* __restrict__ a, const float* __restrict__ b, uint32_t d, int metric,
                                     float* __restrict__ out) {
    F32At fa{a}, fb{b};
    *out = metric == YAMS_B200_L2 ? ref_l2_distance(fa, fb, d) : (metric == 2 ? ref_l1_distance(fa, fb, d) : ref_cosine_distance(fa, fb, d));
}

static int pair_distance(const void* v1, size_t size1, const void* v2, size_t size2, float* result, int metric) {
    // sqlite_vec_c_api.cpp:57-105: SQLITE_OK 0 / SQLITE_ERROR 1
    if (!v1 || !v2 || !result) return 1;
    size_t d1 = size1 / sizeof(float), d2 = size2 / sizeof(float);
    if (d1 != d2) return 1;
    OpWsLease lease;
    OpWs* w = lease.w;
    if (!w) return 1;
    const size_t bytes = (2 * d1 + 4) * sizeof(float);
    if (w->d[0].reserve(bytes) != YAMS_OK || w->h.reserve(bytes) != YAMS_OK) return 1;
    float* hp = w->h.as<float>();
    memcpy(hp, v1, d1 * 4);
    memcpy(hp + d1, v2, d1 * 4);
    float* dp = w->d[0].as<float>();
    if (cudaMemcpyAsync(dp, hp, 2 * d1 * 4, cudaMemcpyHostToDevice, w->st) != cudaSuccess) return 1;
    pair_distance_kernel<<<1, 1, 0, w->st>>>(dp, dp + d1, (uint32_t)d1, metric, dp + 2 * d1);
    if (cudaMemcpyAsync(hp + 2 * d1, dp + 2 * d1, 4, cudaMemcpyDeviceToHost, w->st) != cudaSuccess) return 1;
    if (cudaStreamSynchronize(w->st) != cudaSuccess) return 1;
    *result = hp[2 * d1];
    return 0;
}

// vec0_run_exact_query and distances/batch.hpp: one thread per row evaluates the float distance in the reference build's own
// operation order (ref_order.cuh) -> bit-identical results.  NEGATED distance out so that the descending key sort yields
// ascending distances.
__global__ void batch_dist_kernel(const float* __restrict__ rows, uint32_t d, uint64_t n, const float* __restrict__ q, int metric,
                                  float* __restrict__ out_neg) {
    uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    F32At qa{q}, ra{rows + r * d};
    out_neg[r] = -(metric == YAMS_B200_L2 ? ref_l2_distance(qa, ra, d) : ref_cosine_distance(qa, ra, d));
}
// sort keys of np2 entries: row i < n gets score_key(-dist, i), so a NaN distance (fkey 0) still ranks after every finite one
// but above the zero padding.  filtered: only rows with dist < threshold get a key (NaN rows do not).
__global__ void dist_keys_kernel(const float* __restrict__ neg_dist, uint64_t n, uint64_t np2, int filtered, float threshold,
                                 uint64_t* __restrict__ keys) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < np2; i += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t key = 0;
        if (i < n && (!filtered || (-neg_dist[i]) < threshold))
            key = score_key(neg_dist[i], (uint32_t)i);
        keys[i] = key;
    }
}
__global__ void negate_kernel(float* p, uint64_t n) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) p[i] = -p[i];
}
// computeCosineSimilarity of pair p: row p of a_all against row p of b_all ([n][d] each, one after the other in a 256-byte-aligned
// buffer, so every row is 16-byte aligned when d % 4 == 0)
__global__ void cosine_similarity_f64_kernel(const float* __restrict__ a_all, const float* __restrict__ b_all, uint64_t n, uint32_t d,
                                             double* __restrict__ out_all) {
    const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p < n) out_all[p] = compute_cosine_similarity(b_all, YAMS_B200_F32, d, p, a_all + p * d);
}

// n pairs (a_i, b_i) of d floats each -> n doubles; one thread per pair, the reference's accumulation order
static yams_status_t cosine_similarity_pairs(const float* a, const float* b, size_t n, size_t d, double* out) {
    YB_ARG(d < 0x100000000ull, "dim must be below 2^32");
    OpWsLease lease;
    OpWs* w = lease.w;
    if (!w) return YAMS_ERR_INTERNAL;
    yams_status_t rc;
    const size_t vb = n * d * 4;
    if ((rc = w->d[0].reserve(2 * vb + n * 8 + 64)) != YAMS_OK) return rc;
    if ((rc = w->h.reserve(n * 8 + 64)) != YAMS_OK) return rc;
    float* da = w->d[0].as<float>();
    float* db = da + n * d;
    double* dout = reinterpret_cast<double*>(w->d[0].as<uint8_t>() + ((2 * vb + 7) & ~(size_t)7));
    YB_CUDA(cudaMemcpyAsync(da, a, vb, cudaMemcpyHostToDevice, w->st));
    YB_CUDA(cudaMemcpyAsync(db, b, vb, cudaMemcpyHostToDevice, w->st));
    cosine_similarity_f64_kernel<<<(unsigned)((n + 63) / 64), 64, 0, w->st>>>(da, db, n, (uint32_t)d, dout);
    YB_CUDA(cudaMemcpyAsync(w->h.p, dout, n * 8, cudaMemcpyDeviceToHost, w->st));
    YB_CUDA(cudaStreamSynchronize(w->st));
    memcpy(out, w->h.p, n * 8);
    return YAMS_OK;
}

// Distances of the n rows [n][dim] to the query (batch_dist_kernel), for vec0_exact and batch_distance.
//   BATCH_ALL: out_dist[i] = distance of row i;
//   otherwise ascending, equal distances by row ascending: the first min(k, n) rows (TOP_K) or every row with
//   distance < threshold (FILTERED) -> out_ids (rowids[i] of the host table, or i without one) and out_dist (nullable).
static yams_status_t sorted_distances(const char* what, int metric, const float* query, uint32_t dim, const float* rows, uint64_t n,
                                      int mode, uint64_t k, float threshold, const int64_t* rowids, int64_t* out_ids, float* out_dist,
                                      uint64_t* out_count) {
    OpWsLease lease;
    if (!lease.w) return YAMS_ERR_INTERNAL;
    cudaStream_t st = lease.w->st;
    const uint64_t np2 = pow2_at_least(n);
    const bool sorted = mode != YAMS_B200_BATCH_ALL;
    DevBuf &d_rows = lease.w->d[0], &d_q = lease.w->d[1], &d_dist = lease.w->d[2], &d_keys = lease.w->d[3], &d_oi = lease.w->d[4],
           &d_od = lease.w->d[5], &d_cnt = lease.w->d[6], &d_rid = lease.w->d[7];
    yams_status_t rc = d_rows.reserve((size_t)n * dim * 4);
    if (rc == YAMS_OK) rc = d_q.reserve((size_t)dim * 4);
    if (rc == YAMS_OK) rc = d_dist.reserve((size_t)n * 4);
    if (rc == YAMS_OK && sorted) {
        rc = d_keys.reserve((size_t)np2 * 8);
        if (rc == YAMS_OK) rc = d_oi.reserve((size_t)n * 8);
        if (rc == YAMS_OK) rc = d_od.reserve((size_t)n * 4);
        if (rc == YAMS_OK) rc = d_cnt.reserve(8);
        if (rc == YAMS_OK && rowids) rc = d_rid.reserve((size_t)n * 8);
    }
    if (rc != YAMS_OK) return rc;
    cudaError_t e = cudaMemcpyAsync(d_rows.p, rows, (size_t)n * dim * 4, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_q.p, query, (size_t)dim * 4, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess && sorted && rowids) e = cudaMemcpyAsync(d_rid.p, rowids, (size_t)n * 8, cudaMemcpyHostToDevice, st);
    batch_dist_kernel<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(d_rows.as<float>(), dim, n, d_q.as<float>(), metric, d_dist.as<float>());
    const unsigned g = key_grid(np2);
    uint64_t outn = n;
    if (!sorted) {
        negate_kernel<<<g, 256, 0, st>>>(d_dist.as<float>(), n);
        if (e == cudaSuccess) e = cudaMemcpyAsync(out_dist, d_dist.p, (size_t)n * 4, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    } else {
        const bool filtered = mode == YAMS_B200_BATCH_FILTERED;
        dist_keys_kernel<<<g, 256, 0, st>>>(d_dist.as<float>(), n, np2, filtered ? 1 : 0, threshold, d_keys.as<uint64_t>());
        sort_keys_desc(d_keys.as<uint64_t>(), np2, st);
        if (!filtered) {
            outn = std::min<uint64_t>(k, n);
        } else {
            unsigned long long h_cnt = 0;
            if (e == cudaSuccess) e = cudaMemsetAsync(d_cnt.p, 0, 8, st);
            count_nonzero_keys(d_keys.as<uint64_t>(), np2, d_cnt.as<unsigned long long>(), st);
            if (e == cudaSuccess) e = cudaMemcpyAsync(&h_cnt, d_cnt.p, 8, cudaMemcpyDeviceToHost, st);
            if (e == cudaSuccess) e = cudaStreamSynchronize(st);
            outn = h_cnt;
        }
        if (outn && e == cudaSuccess) {
            unpack_keys(d_keys.as<uint64_t>(), outn, rowids ? d_rid.as<int64_t>() : nullptr, true, d_oi.as<int64_t>(), d_od.as<float>(), st);
            e = cudaMemcpyAsync(out_ids, d_oi.p, (size_t)outn * 8, cudaMemcpyDeviceToHost, st);
            if (e == cudaSuccess && out_dist) e = cudaMemcpyAsync(out_dist, d_od.p, (size_t)outn * 4, cudaMemcpyDeviceToHost, st);
            if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        }
    }
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) {
        set_last_error("%s failed: %s", what, cudaGetErrorString(e));
        return YAMS_ERR_INTERNAL;
    }
    *out_count = outn;
    return YAMS_OK;
}

}  // namespace yb

using namespace yb;

extern "C" {

int sqlite3_vec_distance_l2(const void* vec1, size_t size1, const void* vec2, size_t size2, float* result) {
    return pair_distance(vec1, size1, vec2, size2, result, YAMS_B200_L2);
}
int sqlite3_vec_distance_cosine(const void* vec1, size_t size1, const void* vec2, size_t size2, float* result) {
    return pair_distance(vec1, size1, vec2, size2, result, YAMS_B200_COSINE);
}
int yams_b200_vec_distance_l1(const void* vec1, size_t size1, const void* vec2, size_t size2, float* result) {
    return pair_distance(vec1, size1, vec2, size2, result, 2);
}

yams_status_t yams_b200_vec0_exact(void* self, const float* query, uint32_t dim, const float* rows, const int64_t* rowids,
                                   uint64_t n, uint64_t k, int use_range, int64_t rowid_lo, int64_t rowid_hi,
                                   int64_t* out_rowids, float* out_dist, uint64_t* out_count) {
    YB_TRY
    (void)self;
    YB_ARG(out_count, "out_count is null");
    *out_count = 0;
    YB_ARG(query && dim > 0, "bad query");
    if (n == 0) return YAMS_OK;
    YB_ARG(rows && out_rowids && out_dist, "null argument");
    YB_ARG(n < 0xFFFFFFFFull, "too many rows");
    if (!use_range)
        return sorted_distances("vec0_exact", YAMS_B200_L2, query, dim, rows, n, YAMS_B200_BATCH_TOP_K, k ? k : n, 0.f, rowids,
                                out_rowids, out_dist, out_count);
    // rowid range filter (vec0_module.hpp:399-401) is applied on the host side of the copy: only the rows in range are
    // uploaded, packed into one copy (pure data movement, no arithmetic)
    std::vector<int64_t> rid_h;
    std::vector<float> packed;
    for (uint64_t i = 0; i < n; ++i) {
        int64_t rid = rowids ? rowids[i] : (int64_t)i;
        if (rid < rowid_lo || rid > rowid_hi) continue;
        rid_h.push_back(rid);
        packed.insert(packed.end(), rows + (size_t)i * dim, rows + (size_t)(i + 1) * dim);
    }
    const uint64_t m = rid_h.size();
    if (m == 0) return YAMS_OK;
    return sorted_distances("vec0_exact", YAMS_B200_L2, query, dim, packed.data(), m, YAMS_B200_BATCH_TOP_K, k ? k : m, 0.f,
                            rid_h.data(), out_rowids, out_dist, out_count);
    YB_CATCH
}

yams_status_t yams_b200_batch_distance(void* self, int metric, const float* query, uint32_t dim, const float* database,
                                       uint64_t n, int mode, uint64_t k, float threshold, uint64_t* out_idx, float* out_dist,
                                       uint64_t* out_count) {
    YB_TRY
    (void)self;
    YB_ARG(out_count, "out_count is null");
    *out_count = 0;
    YB_ARG(metric == YAMS_B200_COSINE || metric == YAMS_B200_L2, "unknown metric");
    YB_ARG(mode >= YAMS_B200_BATCH_ALL && mode <= YAMS_B200_BATCH_FILTERED, "unknown mode");
    YB_ARG(query && dim > 0, "bad query");
    if (n == 0 || (mode == YAMS_B200_BATCH_TOP_K && k == 0)) return YAMS_OK;
    YB_ARG(database, "database is null");
    YB_ARG(n < 0xFFFFFFFFull, "too many rows");
    YB_ARG(mode == YAMS_B200_BATCH_ALL ? out_dist != nullptr : out_idx != nullptr, "null output");
    YB_ARG(mode != YAMS_B200_BATCH_FILTERED || out_dist, "null output");
    // row indices come back as the int64 ids of the identity table: the same 8 bytes as uint64 for n < 2^32
    return sorted_distances("batch_distance", metric, query, dim, database, n, mode, k, threshold, nullptr,
                            reinterpret_cast<int64_t*>(out_idx), out_dist, out_count);
    YB_CATCH
}

yams_status_t yams_b200_compute_cosine_similarity(void* self, const float* a, size_t na, const float* b, size_t nb, double* out) {
    YB_TRY
    (void)self;
    YB_ARG(out, "out is null");
    *out = 0.0;
    if (na != nb || na == 0) return YAMS_OK;   // vector_database.cpp:1788-1790
    YB_ARG(a && b, "null vector");
    return cosine_similarity_pairs(a, b, 1, na, out);
    YB_CATCH
}

// The rerank loops that call computeCosineSimilarity once per candidate (sqlite_vec_backend.cpp:4025,4374,4507) as ONE device
// pass: n pairs, row-major a[n][dim] / b[n][dim] (pass the same query n times, or n different pairs).
yams_status_t yams_b200_compute_cosine_similarity_many(void* self, const float* a, const float* b, size_t n, size_t dim, double* out) {
    YB_TRY
    (void)self;
    YB_ARG(out || n == 0, "out is null");
    if (n == 0) return YAMS_OK;
    if (dim == 0) {
        for (size_t i = 0; i < n; ++i) out[i] = 0.0;
        return YAMS_OK;
    }
    YB_ARG(a && b, "null vector");
    return cosine_similarity_pairs(a, b, n, dim, out);
    YB_CATCH
}

}  // extern "C"
