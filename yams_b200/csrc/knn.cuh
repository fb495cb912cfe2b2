// knn.cuh -- shared declarations of the exact vector scan (vector_scan_v1).
#pragma once
#include <algorithm>
#include <mutex>
#include <string>

#include "common.cuh"

namespace yb {

// (score, row index) candidate produced by stage 1
struct __align__(8) Cand {
    float score;
    uint32_t row;
};

// exactly re-scored survivor of stage 2, the input of the final ordering
struct Exact {
    float sim;       // reference similarity (float cast of the double quotient); NaN marks "skipped"
    uint32_t row;
};

// the padded [nq][k] results of a search on the device: [nq*k rowids][nq flags][nq*k scores][nq counts] carved out of one buffer
// (reserve_results); search_device writes only rowids and scores, into the caller's buffers (counts, flags null)
struct DeviceResults {
    int64_t* rowids = nullptr;
    uint64_t* flags = nullptr;
    float* scores = nullptr;
    uint32_t* counts = nullptr;
};

// Small candidate sets (CandidateFilterMode::Exact): device lists (ascending rowids, d_offsets[nq+1]) short enough that
// scoring the listed rows one by one is cheaper than a corpus pass -> gather_score_kernel
struct DirectLists {
    const int64_t* d_allowed = nullptr;
    const uint64_t* d_offsets = nullptr;
    uint64_t total = 0;
    uint32_t max_len = 0;
};

// The semantic-neighbour graph's rows (yams_b200_semantic_neighbors): its own row set and scales, which replace the search's
// cached inv_norm and statistics in stage 1 and the exact score, and the source row of each query of a batch
struct GraphRows {
    const float* inv = nullptr;          // n: float(1 / sqrt(sum (double)r^2)) of the rows the graph takes, else 0
    float r_max = 0.f, dr_abs_max = 0.f, dr_rel_max = 0.f, inv_max = 0.f;   // row_stats_kernel over those rows
    float uf = 0.f;                      // the certificate's underflow term per unit of max(1/|s|, 1) (knn.cu graph_eps)
    const uint32_t* src_row = nullptr;   // nq: corpus row of source q (never its own neighbour)
};

// one exact search (knn.cu): the candidate-set form it scans and the device results it writes, from the enqueue to the finish
struct ScanPlan {
    uint32_t nq = 0, k = 0;
    float threshold = -1.f;
    bool direct = false;                // candidate sets as the lists below
    DirectLists lists;
    const uint32_t* d_mask = nullptr;   // else nullable: bit matrix [nq][mask_ld*32] of allowed rows -> masked corpus pass
    uint64_t mask_ld = 0;
    const GraphRows* graph = nullptr;   // a batch of semantic-graph sources instead of queries
    DeviceResults out;
};

struct Corpus {
    DeviceCtx* dev = nullptr;
    cudaStream_t st = nullptr;
    uint32_t dim = 0;
    int dtype = YAMS_B200_F16;
    int metric = YAMS_B200_COSINE;
    uint64_t n = 0;
    uint64_t generation = 0;   // bumped by every append / remove / clear: derived indexes (pq.cu) notice a stale corpus
    int64_t last_rowid = INT64_MIN;
    bool rowids_dense = true;  // rowid[i] == rowid[0] + i
    DevBuf rows;       // n x dim elements
    DevBuf rowids;     // n x int64
    DevBuf inv_norm;   // n x float. cosine: 1/|row| (double math), 0 for rows the reference skips; L2: |row|^2
    DevBuf stats;      // 4 floats: max |row|, max |row - tf32(row)|, max of that residual relative to |row|, max 1/|row|
                       // (row_stats_kernel)
    float r_max = 0.f, dr_abs_max = 0.f, dr_rel_max = 0.f, inv_max = 0.f;   // host copies of stats (upper bounds; removals keep them)
    // search workspace
    DevBuf q32, q16, qinv, tau, counts, cands, sample_scores, sel, outbuf, dense, mask, misc, dout;
    DevBuf qnorm;      // nq doubles: |q| of the search's queries, written by its query preparation only (misc is scratch that
                       // mutators overwrite while a search_device is still pending)
    DevBuf status;     // ScanStatus + bad[nq] + bad2[nq] of the call in flight
    DevBuf bound, eps, eps2;   // per query: certificate inputs (knn.cu final_kernel)
    DevBuf lvl;        // exhaustive level 1 workspace
    DevBuf graph;      // semantic graph: inv[n] + stats[4] + the batch's source rows
    DevBuf kmeans;     // topology k-means workspace (kmeans.cu)
    float kmeans_ms[4] = {0, 0, 0, 0};   // the last k-means call: device ms of init, assignment, update; host wall ms
    HostBuf h_pin;
    // the call enqueued by search_device and not yet finished (search_device_finish)
    struct Pending {
        ScanPlan plan;
        bool active = false;
        // finished by settle_pending before another call ran on the corpus: what search_device_finish reports
        bool settled = false;
        yams_status_t status = YAMS_OK;
        uint32_t resolved = 0;
        std::string error;
    } pending;
    cudaEvent_t ev[3] = {nullptr, nullptr, nullptr};
    cudaEvent_t ev_scan[2] = {nullptr, nullptr};  // around the full-corpus filtered scan launch
    bool scan_timed = false;
    float last_ms[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    uint32_t wg_launch[2] = {0, 0};   // the last wgmma scan launch: query-tile columns, CTAs
    std::mutex mu;   // public entry points on one corpus are serialised (the workspace buffers are per corpus)
    size_t elem() const { return dtype == YAMS_B200_F16 ? 2 : 4; }
    // the stream is drained first, so the buffers may be freed in any order after it is destroyed
    ~Corpus() {
        if (st) cudaStreamSynchronize(st);
        for (auto& e : ev)
            if (e) cudaEventDestroy(e);
        for (auto& e : ev_scan)
            if (e) cudaEventDestroy(e);
        if (st) cudaStreamDestroy(st);
    }
};

// Stage-1 engine interface: approximate scores of `nrows` corpus rows (row_start + i*row_stride) against nq queries.
//   cosine: score = q.r * inv_norm[row] * qinv[q]          (-inf for rows the reference skips)
//   L2    : score = 2 q.r - |row|^2  (inv_norm[] holds |row|^2; larger = closer; |q|^2 is constant per query)
//   STORE : out_scores[q * ld + i] = score
//   FILTER: rows with score > tau[q] (and mask bit set, if mask) are appended to cands[q][..cap)
struct Stage1Args {
    const void* rows;
    const float* inv_norm;
    uint32_t dim;
    int dtype;
    uint64_t row_start;
    uint64_t row_stride;
    uint64_t nrows;
    const float* q32;       // nq x dim fp32
    const float* qinv;      // nq: 1/|q|
    uint32_t nq;
    // STORE
    float* out_scores;
    uint64_t ld;
    // FILTER
    const float* tau;
    Cand* cands;
    uint32_t cap;
    uint32_t* counts;
    const uint32_t* mask;   // nullable: bit (q * mask_ld*32 + row)
    uint64_t mask_ld;       // words per query
    int metric;             // YAMS_B200_COSINE / YAMS_B200_L2
    // tensor engine: operand-typed queries + the per-query error bound eps[] (|score~ - score| <= eps[q], the input of the
    // exactness certificate) are prepared by the first call of a search and reused by the following ones
    bool skip_qprep;
    float* eps;             // nq floats, written by the engine's query preparation
    float r_max, dr_abs_max, dr_rel_max, inv_max;   // corpus norm statistics (Corpus)
};

yams_status_t stage1_cuda_core(const Stage1Args& a, bool filter, cudaStream_t st);

// Finishes a pending search_device (knn.cu) on the corpus it was enqueued on and keeps its outcome for search_device_finish.
// Every entry point on a corpus but search_device calls it first, under the corpus lock: a mutator would otherwise change the
// rows its exhaustive levels re-score, and any call reuses the workspace its finish reads.
void settle_pending(Corpus* c);

// Stages of the exact scan that the other engines (pq.cu) launch on their own lists; each is described at its definition in knn.cu
void launch_topk_lists(const Cand* lists, const uint32_t* counts, uint32_t cap, uint32_t nq, uint32_t K, Cand* out_sel, uint32_t* out_n,
                       cudaStream_t st);
void launch_topk_dense(const float* dense, uint64_t n, uint32_t nq, uint32_t K, Cand* out_sel, uint32_t* out_n, cudaStream_t st);
constexpr uint32_t TOPK_MAX = 4096;   // the largest K the selection orders in shared memory (knn.cu SEL_MAXK)
void launch_final_plain(const Exact* exact, uint32_t Kp, uint32_t k, uint32_t nq, const int64_t* rowids, const DeviceResults& out,
                        cudaStream_t st);
void launch_map_rowids(const int64_t* rowids_in, uint64_t n_in, const int64_t* corpus_rowids, uint64_t n, Cand* out, cudaStream_t st);
void launch_query_prep(const float* q, uint32_t nq, uint32_t d, double* qnorm, float* qinv, void* status, cudaStream_t st);

yams_status_t reserve_results(DevBuf& buf, uint32_t nq, uint32_t k, DeviceResults* r);
// device results -> the caller's arrays (out_flags nullable).  enqueue_results only enqueues the copies, for a caller with one
// more read-back to make before it waits; copy_results also waits for them.
yams_status_t enqueue_results(const DeviceResults& r, uint32_t nq, uint32_t k, int64_t* out_rowids, float* out_scores, uint32_t* out_counts,
                              uint64_t* out_flags, cudaStream_t st);
yams_status_t copy_results(const DeviceResults& r, uint32_t nq, uint32_t k, int64_t* out_rowids, float* out_scores, uint32_t* out_counts,
                           uint64_t* out_flags, cudaStream_t st);

// Device key sort of the exact paths (knn.cu) and the sqlite-vec operators (operators.cu); the keys are score_key (cosine.cuh).
// pow2_at_least computes in the type of n: the kernels size their shared-memory sorts in 32 bits.
template <typename T>
__host__ __device__ inline T pow2_at_least(T n) {
    T p = 1;
    while (p < n) p <<= 1;
    return p;
}
// grid of the 256-thread grid-stride key kernels over n keys
inline unsigned key_grid(uint64_t n) { return (unsigned)std::min<uint64_t>((n + 255) / 256, 65535); }
// bitonic sort, descending, of np2 keys (a power of two)
void sort_keys_desc(uint64_t* keys, uint64_t np2, cudaStream_t st);
// *d_count += the number of non-zero keys among n
void count_nonzero_keys(const uint64_t* keys, uint64_t n, unsigned long long* d_count, cudaStream_t st);
// the first m keys -> out_rowids[i] = rowids ? rowids[row] : row, out_scores[i] = negate ? -score : score
void unpack_keys(const uint64_t* keys, uint64_t m, const int64_t* rowids, bool negate, int64_t* out_rowids, float* out_scores,
                 cudaStream_t st);

}  // namespace yb

// the opaque handle of the C ABI
struct yams_b200_corpus : public yb::Corpus {};
