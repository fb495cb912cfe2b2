// bm25.cu -- simeon's Bm25Index on the device (yams_b200_bm25_*): the build and the scoring of the lexical backend
// (SimeonLexicalBackend), Atire and SubwordAwareBackoff, bit-identical to the reference.  DESIGN.md §4.11.
//
// Reference (paths under third_party/simeon):
//   Bm25Index::add_doc, collect_field_term_stats   src/bm25.cpp:563-656, :107-149 (words, lowercase, n-grams, dl, ngram_dl)
//   Bm25Index::finalize                            src/bm25.cpp:658-767 (avg_dl, n-gram pruning, idf, total_tf)
//   Bm25Index::score                               src/bm25.cpp:769-874 (SubwordAwareBackoff legs, Atire)
//   score_atire, score_bm25_plus                   src/bm25.cpp:163-188
//   splitmix64_hash                                src/hasher.cpp:33-47 (text_hash.cuh)
//
// Build: the texts are uploaded into one layout with a zero byte after every document, so no word crosses a document.  One
// pass counts dl / ngram_dl per document (integer atomics: exact), then the corpus is cut into document slices that fit the
// device.  Per slice: the word starts are selected, one pair (hash, document) is written per word and one per n-gram
// occurrence, both pair lists (document-major) are sorted by hash with CUB's stable radix sort, so every hash's pairs come out in
// document order, and the runs of (hash, document) become (hash, document, tf) postings.  The postings of all slices are
// merged by one more stable sort by hash (slice order is document order), the runs of hash give df and the dictionary, and
// n-grams over the df limit are dropped and the dictionary rebuilt.  IDF depends on (n, df) only: a table idf[0..n] is
// evaluated on the host with the reference's own float expression and C-library logf.
//
// Score: the host tokenises the queries (words, their hashes, each word's distinct n-gram hashes in emission order); a plan
// kernel looks each up in the sorted dictionaries and writes every query's ordered legs (posting range, weight, field).  One
// CTA per (query, tile of documents) keeps the tile's scores in shared memory and walks the legs in order; per leg it finds the
// part of the posting list inside the tile by binary search and adds each document's contribution -- a document appears once
// per leg, so no atomics, and each document receives its additions in the reference's order.  Every float operation is an
// explicit _rn intrinsic: the reference is compiled without -mfma, so nothing may be fused.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <memory>
#include <mutex>
#include <new>
#include <unordered_set>
#include <vector>

#include "common.cuh"
#include "knn.cuh"
#include "text_hash.cuh"
#include "upload.cuh"

namespace yb {

constexpr int BM_THREADS = 256;
constexpr uint32_t BM_TILE = 4096;                  // documents per scoring CTA: 16 KiB of shared scores
constexpr uint64_t BM_DENSE_BYTES = 1ull << 30;     // score rows per batch of queries

struct Bm25Field {
    DevBuf hashes;   // terms: sorted distinct hashes
    DevBuf offs;     // terms + 1: posting offsets
    DevBuf ttf;      // terms: total tf
    DevBuf docs;     // postings: document ids, ascending per term
    DevBuf tfs;      // postings: tf
    DevBuf dl;       // n_docs: dl / ngram_dl
    uint64_t terms = 0, posts = 0;
    float avg = 0.f;
    std::vector<uint32_t> h_dl;
};

// ---- build kernels ----
struct IsWordStart {
    const uint8_t* t;
    __device__ bool operator()(uint64_t i) const { return is_word_char(t[i]) && (i == 0 || !is_word_char(t[i - 1])); }
};

__host__ __device__ __forceinline__ uint64_t ngram_count(uint64_t L, uint32_t kmin, uint32_t kmax) {
    uint64_t c = 0;
    for (uint64_t k = kmin; k <= kmax && k <= L; ++k) c += L - k + 1;
    return c;
}

// index of the last element <= x in a[0, n) (a ascending, a[0] <= x)
template <typename T>
__device__ __forceinline__ uint64_t last_le(const T* a, uint64_t n, T x) {
    uint64_t lo = 0, hi = n;   // answer in [lo, hi)
    while (hi - lo > 1) {
        const uint64_t mid = lo + (hi - lo) / 2;
        if (a[mid] <= x) lo = mid; else hi = mid;
    }
    return lo;
}

__device__ __forceinline__ uint64_t word_end(const uint8_t* t, uint64_t i) {
    while (is_word_char(t[i])) ++i;   // the zero byte after every document ends the last word
    return i;
}

// dl and ngram_dl of every document: the thread at a word's first byte counts the word and its n-grams
__global__ void bm_doc_counts_kernel(const uint8_t* __restrict__ t, uint64_t len, const uint64_t* __restrict__ pos, uint64_t n,
                                     int sab, uint32_t kmin, uint32_t kmax, uint32_t* __restrict__ dl, uint32_t* __restrict__ gdl) {
    const IsWordStart ws{t};
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += (uint64_t)gridDim.x * blockDim.x) {
        if (!ws(i)) continue;
        const uint64_t d = last_le(pos, n + 1, i);
        atomicAdd(&dl[d], 1u);
        if (sab) atomicAdd(&gdl[d], (uint32_t)ngram_count(word_end(t, i) - i, kmin, kmax));
    }
}

// one word: its hash, document, length and n-gram count
__global__ void bm_words_kernel(const uint8_t* __restrict__ t, const uint64_t* __restrict__ wstart, uint64_t nw,
                                const uint64_t* __restrict__ pos, uint64_t n, uint64_t h0, uint32_t kmin, uint32_t kmax,
                                uint64_t* __restrict__ whash, uint32_t* __restrict__ wdoc, uint32_t* __restrict__ wlen,
                                uint64_t* __restrict__ gcnt) {
    for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < nw; w += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t s = wstart[w], L = word_end(t, s) - s;
        whash[w] = gram_hash<true>(t + s, L, h0);
        wdoc[w] = (uint32_t)last_le(pos, n + 1, s);
        wlen[w] = (uint32_t)L;
        if (gcnt) gcnt[w] = ngram_count(L, kmin, kmax);
    }
}

// one n-gram occurrence j (goff = exclusive scan of the words' n-gram counts): word, then k ascending, then position
__global__ void bm_ngrams_kernel(const uint8_t* __restrict__ t, const uint64_t* __restrict__ wstart, const uint32_t* __restrict__ wdoc,
                                 const uint32_t* __restrict__ wlen, const uint64_t* __restrict__ goff, uint64_t nw, uint64_t total,
                                 uint64_t h0, uint32_t kmin, uint64_t* __restrict__ ghash, uint32_t* __restrict__ gdoc) {
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < total; j += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t w = last_le(goff, nw, j);
        const uint64_t L = wlen[w];
        uint64_t r = j - goff[w], k = kmin;
        while (r >= L - k + 1) { r -= L - k + 1; ++k; }
        ghash[j] = gram_hash<true>(t + wstart[w] + r, k, h0);
        gdoc[j] = wdoc[w];
    }
}

// first pair of each (hash, document) run of the sorted pairs
struct NewPairRun {
    const uint64_t* h;
    const uint32_t* d;
    __device__ bool operator()(uint64_t i) const { return i == 0 || h[i] != h[i - 1] || d[i] != d[i - 1]; }
};
// first posting of each term
struct NewTerm {
    const uint64_t* h;
    __device__ bool operator()(uint64_t i) const { return i == 0 || h[i] != h[i - 1]; }
};

// runs of (hash, document) -> postings (hash, document << 32 | tf) at out + 0..nruns
__global__ void bm_runs_kernel(const uint64_t* __restrict__ h, const uint32_t* __restrict__ d, uint64_t m,
                               const uint64_t* __restrict__ starts, uint64_t nruns, uint64_t* __restrict__ ph, uint64_t* __restrict__ pv) {
    for (uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; r < nruns; r += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t s = starts[r], e = r + 1 < nruns ? starts[r + 1] : m;
        ph[r] = h[s];
        pv[r] = ((uint64_t)d[s] << 32) | (e - s);
    }
}

// the dictionary of the term runs: hash, posting offset, total tf
__global__ void bm_terms_kernel(const uint64_t* __restrict__ ph, const uint64_t* __restrict__ pv, uint64_t np,
                                const uint64_t* __restrict__ starts, uint64_t nterms, uint64_t* __restrict__ hashes,
                                uint64_t* __restrict__ offs, uint64_t* __restrict__ ttf) {
    for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < nterms; t += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t s = starts[t], e = t + 1 < nterms ? starts[t + 1] : np;
        uint64_t sum = 0;
        for (uint64_t i = s; i < e; ++i) sum += (uint32_t)pv[i];
        hashes[t] = ph[s];
        offs[t] = s;
        ttf[t] = sum;
        if (t + 1 == nterms) offs[nterms] = np;
    }
}

// postings of the terms whose df is at most df_max
struct KeepPosting {
    const uint64_t* offs;
    uint64_t nterms, df_max;
    __device__ bool operator()(uint64_t i) const {
        const uint64_t t = last_le(offs, nterms, i);
        return offs[t + 1] - offs[t] <= df_max;
    }
};

__global__ void bm_gather_kernel(const uint64_t* __restrict__ idx, uint64_t m, const uint64_t* __restrict__ ph,
                                 const uint64_t* __restrict__ pv, uint64_t* __restrict__ oh, uint64_t* __restrict__ ov) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (uint64_t)gridDim.x * blockDim.x) {
        oh[i] = ph[idx[i]];
        ov[i] = pv[idx[i]];
    }
}

__global__ void bm_unpack_kernel(const uint64_t* __restrict__ pv, uint64_t m, uint32_t* __restrict__ docs, uint32_t* __restrict__ tfs) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (uint64_t)gridDim.x * blockDim.x) {
        docs[i] = (uint32_t)(pv[i] >> 32);
        tfs[i] = (uint32_t)pv[i];
    }
}

// ---- score ----
struct RawLeg {        // one query word (field 0) or one distinct n-gram of it (field 1)
    uint64_t hash;
    uint64_t term_hash;
    uint32_t field;
    uint32_t pad;
};
struct Leg {           // an addition over documents docs[b, e) of `field`; empty when b == e
    uint64_t b, e;
    float w, idf;
    uint32_t field;
    uint32_t pad;
};
struct Dict {
    const uint64_t* hashes;
    const uint64_t* offs;
    uint64_t terms;
};

__device__ __forceinline__ bool dict_find(const Dict& D, uint64_t h, uint64_t* b, uint64_t* e) {
    if (D.terms == 0 || h < D.hashes[0]) return false;
    const uint64_t t = last_le(D.hashes, D.terms, h);
    if (D.hashes[t] != h) return false;
    *b = D.offs[t];
    *e = D.offs[t + 1];
    return true;
}

__global__ void bm_plan_kernel(const RawLeg* __restrict__ raw, uint64_t nlegs, Dict w, Dict g, const float* __restrict__ idf,
                               int sab, float gamma, Leg* __restrict__ legs) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nlegs; i += (uint64_t)gridDim.x * blockDim.x) {
        const RawLeg r = raw[i];
        Leg L{};
        L.field = r.field;
        uint64_t b = 0, e = 0;
        if (!sab) {
            if (dict_find(w, r.hash, &b, &e)) { L.b = b; L.e = e; L.idf = idf[e - b]; }
        } else {
            // alpha = float(df) / (float(df) + gamma), 0 when the word is unknown (bm25.cpp:805-807)
            const uint64_t df = dict_find(w, r.term_hash, &b, &e) ? e - b : 0;
            const float alpha = df > 0 ? __fdiv_rn(__ull2float_rn(df), __fadd_rn(__ull2float_rn(df), gamma)) : 0.0f;
            if (r.field == 0) {
                if (alpha > 0.0f) { L.b = b; L.e = e; L.w = alpha; L.idf = idf[df]; }
            } else if (alpha < 1.0f && dict_find(g, r.hash, &b, &e)) {
                L.b = b; L.e = e; L.w = __fsub_rn(1.0f, alpha); L.idf = idf[e - b];
            }
        }
        legs[i] = L;
    }
}

struct ScoreArgs {
    const Leg* legs;
    const uint64_t* qoff;     // legs of query q: [qoff[q], qoff[q + 1])
    uint32_t q0;              // first query of the batch
    const uint32_t* docs[2];
    const uint32_t* tfs[2];
    const uint32_t* dl[2];
    float avg[2];             // avg_dl > 0 ? avg_dl : 1
    uint64_t n;
    float k1, b, delta;
    int sab;
    float* out;               // [batch][n]
};

__device__ __forceinline__ uint64_t first_ge(const uint32_t* a, uint64_t lo, uint64_t hi, uint64_t x) {
    while (lo < hi) {
        const uint64_t mid = lo + (hi - lo) / 2;
        if (a[mid] < x) lo = mid + 1; else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(BM_THREADS) bm_score_kernel(ScoreArgs a) {
    __shared__ float s[BM_TILE];
    const uint32_t q = a.q0 + blockIdx.y;
    const uint64_t lo = (uint64_t)blockIdx.x * BM_TILE;
    const uint32_t len = (uint32_t)min((uint64_t)BM_TILE, a.n - lo);
    for (uint32_t i = threadIdx.x; i < len; i += BM_THREADS) s[i] = 0.0f;
    __syncthreads();
    const float k1p1 = __fadd_rn(a.k1, 1.0f), omb = __fsub_rn(1.0f, a.b);
    for (uint64_t l = a.qoff[q]; l < a.qoff[q + 1]; ++l) {
        const Leg g = a.legs[l];
        if (g.b == g.e) continue;
        const uint32_t* docs = a.docs[g.field];
        const uint64_t sb = first_ge(docs, g.b, g.e, lo), se = first_ge(docs, sb, g.e, lo + len);
        if (sb == se) continue;   // the same for every thread of the CTA
        const uint32_t* tfs = a.tfs[g.field];
        const uint32_t* dlv = a.dl[g.field];
        const float avg = a.avg[g.field];
        for (uint64_t i = sb + threadIdx.x; i < se; i += BM_THREADS) {
            const uint32_t d = docs[i];
            const float tf = __uint2float_rn(tfs[i]), dl = __uint2float_rn(dlv[d]);
            // tf + k1 * (1 - b + b * dl / avg)
            const float denom = __fadd_rn(tf, __fmul_rn(a.k1, __fadd_rn(omb, __fdiv_rn(__fmul_rn(a.b, dl), avg))));
            float add;
            if (a.sab)   // alpha * (idf * (tf * (k1 + 1) / denom + delta))
                add = __fmul_rn(g.w, __fmul_rn(g.idf, __fadd_rn(__fdiv_rn(__fmul_rn(tf, k1p1), denom), a.delta)));
            else         // idf * tf * (k1 + 1) / denom
                add = __fdiv_rn(__fmul_rn(__fmul_rn(g.idf, tf), k1p1), denom);
            s[d - lo] = __fadd_rn(s[d - lo], add);
        }
        __syncthreads();
    }
    float* out = a.out + (uint64_t)blockIdx.y * a.n + lo;
    for (uint32_t i = threadIdx.x; i < len; i += BM_THREADS) out[i] = s[i];
}

inline unsigned bm_grid(uint64_t n) { return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((n + BM_THREADS - 1) / BM_THREADS, 65535ull * 4)); }

// cub temp storage in a growable buffer
struct CubTmp {
    DevBuf buf;
    size_t bytes = 0;
    yams_status_t grow() { return buf.reserve(std::max<size_t>(bytes, 256)); }
};

template <typename Pred>
yams_status_t select_indices(CubTmp& tmp, uint64_t lo, uint64_t n, Pred pred, DevBuf& out, DevBuf& cnt, uint64_t* h_cnt, cudaStream_t st) {
    yams_status_t rc;
    if ((rc = out.reserve(std::max<uint64_t>(n, 1) * 8)) != YAMS_OK) return rc;
    if ((rc = cnt.reserve(8)) != YAMS_OK) return rc;
    thrust::counting_iterator<uint64_t> it(lo);
    tmp.bytes = 0;
    YB_CUDA(cub::DeviceSelect::If(nullptr, tmp.bytes, it, out.as<uint64_t>(), cnt.as<uint64_t>(), (int64_t)n, pred, st));
    if ((rc = tmp.grow()) != YAMS_OK) return rc;
    YB_CUDA(cub::DeviceSelect::If(tmp.buf.p, tmp.bytes, it, out.as<uint64_t>(), cnt.as<uint64_t>(), (int64_t)n, pred, st));
    YB_CUDA(cudaMemcpyAsync(h_cnt, cnt.p, 8, cudaMemcpyDeviceToHost, st));
    YB_CUDA(cudaStreamSynchronize(st));
    return YAMS_OK;
}

template <typename V>
yams_status_t sort_pairs(CubTmp& tmp, DevBuf& k, DevBuf& v, DevBuf& k2, DevBuf& v2, uint64_t m, cudaStream_t st) {
    yams_status_t rc;
    if ((rc = k2.reserve(std::max<uint64_t>(m, 1) * 8)) != YAMS_OK) return rc;
    if ((rc = v2.reserve(std::max<uint64_t>(m, 1) * sizeof(V))) != YAMS_OK) return rc;
    tmp.bytes = 0;
    YB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp.bytes, k.as<uint64_t>(), k2.as<uint64_t>(), v.as<V>(), v2.as<V>(), (int64_t)m, 0, 64, st));
    if ((rc = tmp.grow()) != YAMS_OK) return rc;
    YB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.buf.p, tmp.bytes, k.as<uint64_t>(), k2.as<uint64_t>(), v.as<V>(), v2.as<V>(), (int64_t)m, 0, 64, st));
    std::swap(k, k2);
    std::swap(v, v2);
    return YAMS_OK;
}

}  // namespace yb

using namespace yb;

struct yams_b200_bm25 {
    DeviceCtx* dev = nullptr;
    yams_bm25_config cfg{};
    uint64_t n = 0, total_tokens = 0, pruned = 0;
    Bm25Field f[2];
    DevBuf idf;                   // n + 1 floats: idf of df = 0..n
    cudaStream_t st = nullptr;
    cudaEvent_t ev[2] = {nullptr, nullptr};
    DevBuf raw, legs, qoff, dense, sel, seln;   // score workspace
    float ms[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    std::mutex mu;
    ~yams_b200_bm25() {
        if (st) cudaStreamSynchronize(st);
        for (auto& e : ev)
            if (e) cudaEventDestroy(e);
        if (st) cudaStreamDestroy(st);
    }
};

namespace yb {

static double wall_ms() {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// device ms of the work `fn` enqueues on the index's stream (waits for it)
template <typename F>
static yams_status_t timed(yams_b200_bm25* x, float* acc, F&& fn) {
    YB_CUDA(cudaEventRecord(x->ev[0], x->st));
    yams_status_t rc = fn();
    if (rc != YAMS_OK) return rc;
    YB_CUDA(cudaEventRecord(x->ev[1], x->st));
    YB_CUDA(cudaEventSynchronize(x->ev[1]));
    float ms = 0.f;
    YB_CUDA(cudaEventElapsedTime(&ms, x->ev[0], x->ev[1]));
    *acc += ms;
    return YAMS_OK;
}

// postings (hash, document << 32 | tf) of one field, slices appended in document order -> the field's dictionary and lists.
// N-grams over the df limit are dropped first (finalize_ngram_field).
static yams_status_t finish_field(yams_b200_bm25* x, Bm25Field& F, DevBuf& ph, DevBuf& pv, uint64_t np, bool merge, bool prune,
                                  CubTmp& tmp) {
    cudaStream_t st = x->st;
    yams_status_t rc;
    DevBuf ph2, pv2, starts, cnt;
    if (merge && np > 1 && (rc = sort_pairs<uint64_t>(tmp, ph, pv, ph2, pv2, np, st)) != YAMS_OK) return rc;
    for (int pass = 0; pass < 2; ++pass) {
        uint64_t nterms = 0;
        if (np && (rc = select_indices(tmp, 0, np, NewTerm{ph.as<uint64_t>()}, starts, cnt, &nterms, st)) != YAMS_OK) return rc;
        if ((rc = F.hashes.reserve(std::max<uint64_t>(nterms, 1) * 8)) != YAMS_OK) return rc;
        if ((rc = F.offs.reserve((nterms + 1) * 8)) != YAMS_OK) return rc;
        if ((rc = F.ttf.reserve(std::max<uint64_t>(nterms, 1) * 8)) != YAMS_OK) return rc;
        if (nterms)
            bm_terms_kernel<<<bm_grid(nterms), BM_THREADS, 0, st>>>(ph.as<uint64_t>(), pv.as<uint64_t>(), np, starts.as<uint64_t>(), nterms,
                                                                    F.hashes.as<uint64_t>(), F.offs.as<uint64_t>(), F.ttf.as<uint64_t>());
        else
            YB_CUDA(cudaMemsetAsync(F.offs.p, 0, 8, st));
        YB_CUDA(cudaGetLastError());
        F.terms = nterms;
        F.posts = np;
        if (pass == 1 || !prune) break;
        // finalize_ngram_field (bm25.cpp:704-708): df_max = size_t(double(ratio) * double(n)), only when ratio > 0 and n > 0
        const uint64_t df_max = (uint64_t)((double)x->cfg.ngram_df_prune_ratio * (double)x->n);
        uint64_t kept = 0;
        if (np && (rc = select_indices(tmp, 0, np, KeepPosting{F.offs.as<uint64_t>(), nterms, df_max}, starts, cnt, &kept, st)) != YAMS_OK)
            return rc;
        if (kept == np) break;
        if ((rc = ph2.reserve(std::max<uint64_t>(kept, 1) * 8)) != YAMS_OK || (rc = pv2.reserve(std::max<uint64_t>(kept, 1) * 8)) != YAMS_OK)
            return rc;
        if (kept)
            bm_gather_kernel<<<bm_grid(kept), BM_THREADS, 0, st>>>(starts.as<uint64_t>(), kept, ph.as<uint64_t>(), pv.as<uint64_t>(),
                                                                   ph2.as<uint64_t>(), pv2.as<uint64_t>());
        YB_CUDA(cudaGetLastError());
        std::swap(ph, ph2);
        std::swap(pv, pv2);
        np = kept;
        x->pruned = nterms;   // minus the terms left, below
    }
    if (prune && x->pruned) x->pruned -= F.terms;
    if ((rc = F.docs.reserve(std::max<uint64_t>(np, 1) * 4)) != YAMS_OK || (rc = F.tfs.reserve(std::max<uint64_t>(np, 1) * 4)) != YAMS_OK)
        return rc;
    if (np) bm_unpack_kernel<<<bm_grid(np), BM_THREADS, 0, st>>>(pv.as<uint64_t>(), np, F.docs.as<uint32_t>(), F.tfs.as<uint32_t>());
    YB_CUDA(cudaGetLastError());
    return YAMS_OK;
}

// appends src[0, m) of 8-byte elements to dst at element `at`, growing dst (contents kept)
static yams_status_t append_u64(DevBuf& dst, uint64_t at, const DevBuf& src, uint64_t m, cudaStream_t st) {
    yams_status_t rc = dst.reserve((at + m) * 8, true, st);
    if (rc != YAMS_OK) return rc;
    if (m) YB_CUDA(cudaMemcpyAsync(dst.as<uint64_t>() + at, src.p, m * 8, cudaMemcpyDeviceToDevice, st));
    return YAMS_OK;
}

// sorted pairs (hash, document) -> postings appended to (ph, pv) at *np
static yams_status_t pair_runs(CubTmp& tmp, DevBuf& k, DevBuf& v, uint64_t m, DevBuf& ph, DevBuf& pv, uint64_t* np, cudaStream_t st) {
    if (m == 0) return YAMS_OK;
    yams_status_t rc;
    DevBuf starts, cnt, rh, rv;
    uint64_t nruns = 0;
    if ((rc = select_indices(tmp, 0, m, NewPairRun{k.as<uint64_t>(), v.as<uint32_t>()}, starts, cnt, &nruns, st)) != YAMS_OK) return rc;
    if ((rc = rh.reserve(nruns * 8)) != YAMS_OK || (rc = rv.reserve(nruns * 8)) != YAMS_OK) return rc;
    bm_runs_kernel<<<bm_grid(nruns), BM_THREADS, 0, st>>>(k.as<uint64_t>(), v.as<uint32_t>(), m, starts.as<uint64_t>(), nruns,
                                                          rh.as<uint64_t>(), rv.as<uint64_t>());
    YB_CUDA(cudaGetLastError());
    if ((rc = append_u64(ph, *np, rh, nruns, st)) != YAMS_OK || (rc = append_u64(pv, *np, rv, nruns, st)) != YAMS_OK) return rc;
    YB_CUDA(cudaStreamSynchronize(st));   // rh / rv are freed on return
    *np += nruns;
    return YAMS_OK;
}

static yams_status_t bm25_build(yams_b200_bm25* x, const char* const* texts, const size_t* lens) {
    const double t0 = wall_ms();
    cudaStream_t st = x->st;
    const uint64_t n = x->n;
    const bool sab = x->cfg.variant == YAMS_BM25_SUBWORD_AWARE_BACKOFF;
    const uint32_t kmin = x->cfg.ngram_min, kmax = x->cfg.ngram_max;
    const uint64_t h0 = gram_hash_h0(x->cfg.hash_seed);
    yams_status_t rc;
    // ---- layout: document d at pos[d], one zero byte after it ----
    std::vector<uint64_t> pos(n + 1, 0);
    std::vector<LayoutPiece> pieces;
    pieces.reserve(n);
    for (uint64_t d = 0; d < n; ++d) {
        if (lens[d]) pieces.push_back({pos[d], (uint64_t)lens[d], reinterpret_cast<const uint8_t*>(texts[d])});
        pos[d + 1] = pos[d] + lens[d] + 1;
    }
    const uint64_t L = pos[n];
    DevBuf text, d_pos;
    if ((rc = text.reserve(L + 16)) != YAMS_OK || (rc = d_pos.reserve((n + 1) * 8)) != YAMS_OK) return rc;
    for (Bm25Field& F : x->f) {
        if ((rc = F.dl.reserve(std::max<uint64_t>(n, 1) * 4)) != YAMS_OK) return rc;
        YB_CUDA(cudaMemsetAsync(F.dl.p, 0, std::max<uint64_t>(n, 1) * 4, st));
        F.h_dl.assign(n, 0);
    }
    rc = timed(x, &x->ms[0], [&]() -> yams_status_t {
        HostBuf pin[2];
        cudaEvent_t done[2] = {nullptr, nullptr};
        for (auto& e : done) YB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        yams_status_t r = staged_upload(pin, done, text.as<uint8_t>(), L, pieces, st);
        if (r == YAMS_OK && cudaMemsetAsync(text.as<uint8_t>() + L, 0, 16, st) != cudaSuccess) r = YAMS_ERR_INTERNAL;
        if (r == YAMS_OK && cudaMemcpyAsync(d_pos.p, pos.data(), (n + 1) * 8, cudaMemcpyHostToDevice, st) != cudaSuccess) r = YAMS_ERR_INTERNAL;
        cudaStreamSynchronize(st);   // the pinned buffers are freed on return
        for (auto& e : done) cudaEventDestroy(e);
        if (r == YAMS_ERR_INTERNAL) set_last_error("bm25 upload failed");
        return r;
    });
    if (rc != YAMS_OK) return rc;
    // ---- dl / ngram_dl ----
    rc = timed(x, &x->ms[1], [&]() -> yams_status_t {
        if (L) bm_doc_counts_kernel<<<bm_grid(L), BM_THREADS, 0, st>>>(text.as<uint8_t>(), L, d_pos.as<uint64_t>(), n, sab, kmin, kmax,
                                                                       x->f[0].dl.as<uint32_t>(), x->f[1].dl.as<uint32_t>());
        YB_CUDA(cudaGetLastError());
        for (Bm25Field& F : x->f)
            if (n) YB_CUDA(cudaMemcpyAsync(F.h_dl.data(), F.dl.p, n * 4, cudaMemcpyDeviceToHost, st));
        return YAMS_OK;
    });
    if (rc != YAMS_OK) return rc;
    uint64_t sums[2] = {0, 0};
    for (int fi = 0; fi < 2; ++fi) {
        for (uint32_t v : x->f[fi].h_dl) sums[fi] += v;
        x->f[fi].avg = n == 0 ? 0.0f : (float)((double)sums[fi] / (double)n);   // finalize_word_field (bm25.cpp:668-676)
    }
    x->total_tokens = sums[0];
    // ---- document slices: pairs of one slice (words + n-grams) within what the device can hold ----
    size_t free_b = 0, total_b = 0;
    YB_CUDA(cudaMemGetInfo(&free_b, &total_b));
    // per pair of a slice: keys and values twice, run starts, the word arrays, postings and the sort's scratch: ~96 bytes.
    // YAMS_B200_BM25_SLICE_PAIRS = N >= 1 lowers the budget to N pairs, read at every build (the index is the same at any cut).
    uint64_t budget = std::max<uint64_t>(1ull << 20, std::min<uint64_t>((uint64_t)free_b / 2 / 96, 1ull << 31));
    if (const char* e = getenv("YAMS_B200_BM25_SLICE_PAIRS")) {
        const uint64_t cap = strtoull(e, nullptr, 10);
        if (cap) budget = std::min(budget, cap);
    }
    std::vector<uint64_t> cuts{0};
    uint64_t acc = 0;
    for (uint64_t d = 0; d < n; ++d) {
        const uint64_t c = (uint64_t)x->f[0].h_dl[d] + (sab ? (uint64_t)x->f[1].h_dl[d] : 0);
        if (acc && acc + c > budget) { cuts.push_back(d); acc = 0; }
        acc += c;
    }
    cuts.push_back(n);
    const uint64_t nslices = cuts.size() - 1;
    CubTmp tmp;
    DevBuf ph[2], pv[2];
    uint64_t np[2] = {0, 0};
    for (uint64_t si = 0; si < nslices; ++si) {
        const uint64_t lo = pos[cuts[si]], hi = pos[cuts[si + 1]];
        DevBuf wstart, cnt, whash, wdoc, wlen, gcnt, k2, v2;
        uint64_t nw = 0, ng = 0;
        rc = timed(x, &x->ms[1], [&]() -> yams_status_t {
            yams_status_t r;
            if ((r = select_indices(tmp, lo, hi - lo, IsWordStart{text.as<uint8_t>()}, wstart, cnt, &nw, st)) != YAMS_OK) return r;
            if ((r = whash.reserve(std::max<uint64_t>(nw, 1) * 8)) != YAMS_OK || (r = wdoc.reserve(std::max<uint64_t>(nw, 1) * 4)) != YAMS_OK ||
                (r = wlen.reserve(std::max<uint64_t>(nw, 1) * 4)) != YAMS_OK || (r = gcnt.reserve(std::max<uint64_t>(nw, 1) * 8)) != YAMS_OK)
                return r;
            if (nw)
                bm_words_kernel<<<bm_grid(nw), BM_THREADS, 0, st>>>(text.as<uint8_t>(), wstart.as<uint64_t>(), nw, d_pos.as<uint64_t>(), n, h0,
                                                                    kmin, kmax, whash.as<uint64_t>(), wdoc.as<uint32_t>(), wlen.as<uint32_t>(),
                                                                    sab ? gcnt.as<uint64_t>() : nullptr);
            YB_CUDA(cudaGetLastError());
            return YAMS_OK;
        });
        if (rc != YAMS_OK) return rc;
        // words: sort by hash (stable: document order within a hash), runs -> postings
        rc = timed(x, &x->ms[2], [&] { return sort_pairs<uint32_t>(tmp, whash, wdoc, k2, v2, nw, st); });
        if (rc != YAMS_OK) return rc;
        rc = timed(x, &x->ms[3], [&] { return pair_runs(tmp, whash, wdoc, nw, ph[0], pv[0], &np[0], st); });
        if (rc != YAMS_OK) return rc;
        if (!sab || nw == 0) continue;
        // the n-gram occurrences of the slice's words; the sort left the words' documents in word order in v2
        DevBuf goff, ghash, gdoc;
        rc = timed(x, &x->ms[1], [&]() -> yams_status_t {
            yams_status_t r;
            if ((r = goff.reserve(nw * 8)) != YAMS_OK) return r;
            tmp.bytes = 0;
            YB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp.bytes, gcnt.as<uint64_t>(), goff.as<uint64_t>(), (int64_t)nw, st));
            if ((r = tmp.grow()) != YAMS_OK) return r;
            YB_CUDA(cub::DeviceScan::ExclusiveSum(tmp.buf.p, tmp.bytes, gcnt.as<uint64_t>(), goff.as<uint64_t>(), (int64_t)nw, st));
            uint64_t last[2];
            YB_CUDA(cudaMemcpyAsync(&last[0], goff.as<uint64_t>() + nw - 1, 8, cudaMemcpyDeviceToHost, st));
            YB_CUDA(cudaMemcpyAsync(&last[1], gcnt.as<uint64_t>() + nw - 1, 8, cudaMemcpyDeviceToHost, st));
            YB_CUDA(cudaStreamSynchronize(st));
            ng = last[0] + last[1];
            if ((r = ghash.reserve(std::max<uint64_t>(ng, 1) * 8)) != YAMS_OK || (r = gdoc.reserve(std::max<uint64_t>(ng, 1) * 4)) != YAMS_OK)
                return r;
            if (ng)
                bm_ngrams_kernel<<<bm_grid(ng), BM_THREADS, 0, st>>>(text.as<uint8_t>(), wstart.as<uint64_t>(), v2.as<uint32_t>(),
                                                                     wlen.as<uint32_t>(), goff.as<uint64_t>(), nw, ng, h0, kmin,
                                                                     ghash.as<uint64_t>(), gdoc.as<uint32_t>());
            YB_CUDA(cudaGetLastError());
            return YAMS_OK;
        });
        if (rc != YAMS_OK) return rc;
        wstart = DevBuf(); whash = DevBuf(); wdoc = DevBuf(); wlen = DevBuf(); gcnt = DevBuf(); goff = DevBuf(); k2 = DevBuf(); v2 = DevBuf();
        rc = timed(x, &x->ms[2], [&] { return sort_pairs<uint32_t>(tmp, ghash, gdoc, k2, v2, ng, st); });
        if (rc != YAMS_OK) return rc;
        rc = timed(x, &x->ms[3], [&] { return pair_runs(tmp, ghash, gdoc, ng, ph[1], pv[1], &np[1], st); });
        if (rc != YAMS_OK) return rc;
    }
    text = DevBuf();
    for (int fi = 0; fi < (sab ? 2 : 1); ++fi) {
        rc = timed(x, &x->ms[3], [&] {
            return finish_field(x, x->f[fi], ph[fi], pv[fi], np[fi], nslices > 1, fi == 1 && x->cfg.ngram_df_prune_ratio > 0.0f && n > 0, tmp);
        });
        if (rc != YAMS_OK) return rc;
    }
    // ---- idf of df = 0..n: the reference's float expression and std::log(float) (bm25.cpp:680-682, 729-731) ----
    std::vector<float> idf(n + 1);
    const float nf = (float)n;
    for (uint64_t df = 0; df <= n; ++df) {
        const float d = (float)df;
        idf[df] = std::log((nf - d + 0.5f) / (d + 0.5f) + 1.0f);
    }
    if ((rc = x->idf.reserve((n + 1) * 4)) != YAMS_OK) return rc;
    YB_CUDA(cudaMemcpyAsync(x->idf.p, idf.data(), (n + 1) * 4, cudaMemcpyHostToDevice, st));
    YB_CUDA(cudaStreamSynchronize(st));
    x->ms[4] = (float)(wall_ms() - t0);
    x->ms[5] = (float)nslices;
    return YAMS_OK;
}

// the words of a query in order, lowercased (collect_field_term_stats / StringTermSink)
static void query_words(const uint8_t* p, size_t len, std::vector<std::pair<size_t, size_t>>& out) {
    out.clear();
    size_t i = 0;
    while (i < len) {
        while (i < len && !is_word_char(p[i])) ++i;
        const size_t s = i;
        while (i < len && is_word_char(p[i])) ++i;
        if (s < i) out.push_back({s, i - s});
    }
}

static yams_status_t bm25_score(yams_b200_bm25* x, const char* const* queries, const size_t* qlens, uint32_t nq, float* out_scores,
                                uint32_t k, uint32_t* out_docs, float* out_topk, uint32_t* out_counts) {
    const double t0 = wall_ms();
    cudaStream_t st = x->st;
    const uint64_t n = x->n;
    const bool sab = x->cfg.variant == YAMS_BM25_SUBWORD_AWARE_BACKOFF;
    const uint64_t h0 = gram_hash_h0(x->cfg.hash_seed);
    yams_status_t rc;
    // ---- host: the legs of every query, in the reference's order ----
    std::vector<RawLeg> raw;
    std::vector<uint64_t> qoff(nq + 1, 0);
    std::vector<std::pair<size_t, size_t>> ws;
    std::vector<uint8_t> low;
    std::unordered_set<uint64_t> seen;
    for (uint32_t q = 0; q < nq; ++q) {
        const uint8_t* p = reinterpret_cast<const uint8_t*>(queries[q]);
        query_words(p, qlens[q], ws);
        for (const auto& [s, l] : ws) {
            low.resize(l);
            for (size_t i = 0; i < l; ++i) low[i] = ascii_lower(p[s + i]);
            const uint64_t th = gram_hash(low.data(), l, h0);
            raw.push_back({th, th, 0, 0});
            if (!sab) continue;
            // collect_unique_query_ngrams (bm25.cpp:151-161): k ascending, position ascending, first occurrence of each hash
            seen.clear();
            for (uint64_t kk = x->cfg.ngram_min; kk <= x->cfg.ngram_max && kk <= l; ++kk)
                for (uint64_t i = 0; i + kk <= l; ++i) {
                    const uint64_t gh = gram_hash(low.data() + i, kk, h0);
                    if (seen.insert(gh).second) raw.push_back({gh, th, 1, 0});
                }
        }
        qoff[q + 1] = raw.size();
    }
    const uint64_t nlegs = raw.size();
    const uint32_t K = std::min<uint64_t>(k, n);
    if ((rc = x->raw.reserve(std::max<uint64_t>(nlegs, 1) * sizeof(RawLeg))) != YAMS_OK) return rc;
    if ((rc = x->legs.reserve(std::max<uint64_t>(nlegs, 1) * sizeof(Leg))) != YAMS_OK) return rc;
    if ((rc = x->qoff.reserve((nq + 1) * 8)) != YAMS_OK) return rc;
    const uint64_t qb_max = n ? std::max<uint64_t>(1, std::min<uint64_t>({BM_DENSE_BYTES / (n * 4), (uint64_t)nq, 4096})) : 0;
    if (n && (rc = x->dense.reserve(qb_max * n * 4)) != YAMS_OK) return rc;
    if (K && (rc = x->sel.reserve(qb_max * K * sizeof(Cand))) != YAMS_OK) return rc;
    if (K && (rc = x->seln.reserve(qb_max * 4)) != YAMS_OK) return rc;
    if (k) {
        for (uint64_t i = 0; i < (uint64_t)nq * k; ++i) { out_docs[i] = 0xFFFFFFFFu; out_topk[i] = 0.0f; }
        for (uint32_t q = 0; q < nq; ++q) out_counts[q] = 0;
    }
    if (n == 0) {
        x->ms[6] = 0.f;
        x->ms[7] = (float)(wall_ms() - t0);
        return YAMS_OK;
    }
    float dev_ms = 0.f;
    std::vector<Cand> h_sel;
    std::vector<uint32_t> h_n;
    rc = timed(x, &dev_ms, [&]() -> yams_status_t {
        if (nlegs) {
            YB_CUDA(cudaMemcpyAsync(x->raw.p, raw.data(), nlegs * sizeof(RawLeg), cudaMemcpyHostToDevice, st));
            Dict w{x->f[0].hashes.as<uint64_t>(), x->f[0].offs.as<uint64_t>(), x->f[0].terms};
            Dict g{x->f[1].hashes.as<uint64_t>(), x->f[1].offs.as<uint64_t>(), x->f[1].terms};
            bm_plan_kernel<<<bm_grid(nlegs), BM_THREADS, 0, st>>>(x->raw.as<RawLeg>(), nlegs, w, g, x->idf.as<float>(), sab,
                                                                  x->cfg.subword_gamma, x->legs.as<Leg>());
            YB_CUDA(cudaGetLastError());
        }
        YB_CUDA(cudaMemcpyAsync(x->qoff.p, qoff.data(), (nq + 1) * 8, cudaMemcpyHostToDevice, st));
        ScoreArgs a{};
        a.legs = x->legs.as<Leg>();
        a.qoff = x->qoff.as<uint64_t>();
        for (int fi = 0; fi < 2; ++fi) {
            a.docs[fi] = x->f[fi].docs.as<uint32_t>();
            a.tfs[fi] = x->f[fi].tfs.as<uint32_t>();
            a.dl[fi] = x->f[fi].dl.as<uint32_t>();
            a.avg[fi] = x->f[fi].avg > 0.0f ? x->f[fi].avg : 1.0f;
        }
        a.n = n;
        a.k1 = x->cfg.k1; a.b = x->cfg.b; a.delta = x->cfg.delta;
        a.sab = sab;
        a.out = x->dense.as<float>();
        const unsigned tiles = (unsigned)((n + BM_TILE - 1) / BM_TILE);
        for (uint32_t q0 = 0; q0 < nq; q0 += (uint32_t)qb_max) {
            const uint32_t qb = (uint32_t)std::min<uint64_t>(qb_max, nq - q0);
            a.q0 = q0;
            bm_score_kernel<<<dim3(tiles, qb), BM_THREADS, 0, st>>>(a);
            YB_CUDA(cudaGetLastError());
            if (out_scores)
                YB_CUDA(cudaMemcpyAsync(out_scores + (uint64_t)q0 * n, x->dense.p, (uint64_t)qb * n * 4, cudaMemcpyDeviceToHost, st));
            if (K) {
                launch_topk_dense(x->dense.as<float>(), n, qb, K, x->sel.as<Cand>(), x->seln.as<uint32_t>(), st);
                YB_CUDA(cudaGetLastError());
                h_sel.resize((uint64_t)qb * K);
                h_n.resize(qb);
                YB_CUDA(cudaMemcpyAsync(h_sel.data(), x->sel.p, (uint64_t)qb * K * sizeof(Cand), cudaMemcpyDeviceToHost, st));
                YB_CUDA(cudaMemcpyAsync(h_n.data(), x->seln.p, (uint64_t)qb * 4, cudaMemcpyDeviceToHost, st));
                YB_CUDA(cudaStreamSynchronize(st));
                // best first: the documents of score > 0 lead the selection
                for (uint32_t j = 0; j < qb; ++j) {
                    uint32_t c = 0;
                    const uint32_t m = std::min(h_n[j], K);
                    while (c < m && h_sel[(uint64_t)j * K + c].score > 0.0f) {
                        out_docs[(uint64_t)(q0 + j) * k + c] = h_sel[(uint64_t)j * K + c].row;
                        out_topk[(uint64_t)(q0 + j) * k + c] = h_sel[(uint64_t)j * K + c].score;
                        ++c;
                    }
                    out_counts[q0 + j] = c;
                }
            } else if (q0 + qb < nq) {
                YB_CUDA(cudaStreamSynchronize(st));   // the next batch overwrites the score rows
            }
        }
        return YAMS_OK;
    });
    if (rc != YAMS_OK) return rc;
    x->ms[6] = dev_ms;
    x->ms[7] = (float)(wall_ms() - t0);
    return YAMS_OK;
}

// a small kernel reads one term's dictionary entry
__global__ void bm_lookup_kernel(Dict D, const uint64_t* __restrict__ ttf, uint64_t h, uint64_t* __restrict__ out) {
    uint64_t b = 0, e = 0;
    const bool found = dict_find(D, h, &b, &e);
    out[0] = found ? b : 0;
    out[1] = found ? e : 0;
    out[2] = found ? ttf[last_le(D.hashes, D.terms, h)] : 0;
}

}  // namespace yb

extern "C" {

void yams_b200_bm25_default_config(yams_bm25_config* cfg) {
    if (!cfg) return;
    // Bm25Config defaults (include/simeon/bm25.hpp:85-107) with the lexical backend's variant and gamma
    cfg->k1 = 1.2f;
    cfg->b = 0.75f;
    cfg->delta = 1.0f;
    cfg->subword_gamma = 5.0f;
    cfg->variant = YAMS_BM25_SUBWORD_AWARE_BACKOFF;
    cfg->ngram_min = 3;
    cfg->ngram_max = 4;
    cfg->ngram_df_prune_ratio = 0.5f;
    cfg->hash_seed = 0xB252B252B252B252ULL;
}

yams_status_t yams_b200_bm25_build(void* self, const yams_bm25_config* cfg_in, const char* const* texts, const size_t* lens,
                                   uint64_t n_docs, yams_b200_bm25** out) {
    YB_TRY
    (void)self;
    DeviceCtx* dev = nullptr;
    yams_status_t rc = ensure_device(&dev);
    if (rc != YAMS_OK) return rc;
    YB_ARG(out, "out is null");
    *out = nullptr;
    yams_bm25_config cfg;
    if (cfg_in) cfg = *cfg_in; else yams_b200_bm25_default_config(&cfg);
    if (cfg.variant != YAMS_BM25_ATIRE && cfg.variant != YAMS_BM25_SUBWORD_AWARE_BACKOFF) {
        set_last_error("bm25 variant %u is not served (Atire = 0, SubwordAwareBackoff = 7)", cfg.variant);
        return YAMS_ERR_UNSUPPORTED;
    }
    YB_ARG(cfg.variant != YAMS_BM25_SUBWORD_AWARE_BACKOFF || cfg.ngram_max <= 64, "ngram_max must be <= 64");
    YB_ARG(n_docs < 0xFFFFFFFFull, "too many documents");
    YB_ARG(n_docs == 0 || (texts && lens), "null argument");
    for (uint64_t i = 0; i < n_docs; ++i) YB_ARG(texts[i] || lens[i] == 0, "null text");
    std::unique_ptr<yams_b200_bm25> x(new (std::nothrow) yams_b200_bm25());
    if (!x) return YAMS_ERR_INTERNAL;
    x->dev = dev;
    x->cfg = cfg;
    x->n = n_docs;
    YB_CUDA(cudaStreamCreateWithFlags(&x->st, cudaStreamNonBlocking));
    for (auto& e : x->ev) YB_CUDA(cudaEventCreate(&e));
    if ((rc = bm25_build(x.get(), texts, lens)) != YAMS_OK) return rc;
    *out = x.release();
    return YAMS_OK;
    YB_CATCH
}

yams_status_t yams_b200_bm25_score(yams_b200_bm25* idx, const char* const* queries, const size_t* qlens, uint32_t nq, float* out_scores,
                                   uint32_t k, uint32_t* out_docs, float* out_topk_scores, uint32_t* out_counts) {
    YB_TRY
    DeviceCtx* dev = nullptr;
    yams_status_t rc = ensure_device(&dev);
    if (rc != YAMS_OK) return rc;
    YB_ARG(idx, "index is null");
    YB_ARG(k <= TOPK_MAX, "k must be <= 4096");
    YB_ARG(k == 0 || (out_docs && out_topk_scores && out_counts), "null top-k output");
    if (nq == 0) return YAMS_OK;
    YB_ARG(queries && qlens, "null argument");
    for (uint32_t q = 0; q < nq; ++q) YB_ARG(queries[q] || qlens[q] == 0, "null query");
    YB_BIND(idx);
    std::lock_guard<std::mutex> g(idx->mu);
    return bm25_score(idx, queries, qlens, nq, out_scores, k, out_docs, out_topk_scores, out_counts);
    YB_CATCH
}

yams_status_t yams_b200_bm25_stats(yams_b200_bm25* idx, yams_bm25_stats* out) {
    DeviceCtx* dev = nullptr;
    yams_status_t rc = ensure_device(&dev);
    if (rc != YAMS_OK) return rc;
    YB_ARG(idx && out, "null argument");
    out->n_docs = idx->n;
    out->avg_dl = idx->f[0].avg;
    out->ngram_avg_dl = idx->f[1].avg;
    out->total_tokens = idx->total_tokens;
    for (int fi = 0; fi < 2; ++fi) {
        out->terms[fi] = idx->f[fi].terms;
        out->postings[fi] = idx->f[fi].posts;
    }
    out->pruned = idx->pruned;
    return YAMS_OK;
}

yams_status_t yams_b200_bm25_postings(yams_b200_bm25* idx, uint32_t field, uint64_t term_hash, uint32_t* out_df, float* out_idf,
                                      uint64_t* out_total_tf, uint32_t* out_docs, uint32_t* out_tfs, uint64_t cap) {
    YB_TRY
    DeviceCtx* dev = nullptr;
    yams_status_t rc = ensure_device(&dev);
    if (rc != YAMS_OK) return rc;
    YB_ARG(idx && out_df && out_idf && out_total_tf, "null argument");
    YB_ARG(field < 2, "field must be 0 (words) or 1 (n-grams)");
    YB_ARG(cap == 0 || (out_docs && out_tfs), "null posting output");
    YB_BIND(idx);
    std::lock_guard<std::mutex> g(idx->mu);
    const Bm25Field& F = idx->f[field];
    *out_df = 0;
    *out_idf = 0.0f;
    *out_total_tf = 0;
    if (F.terms == 0) return YAMS_OK;
    OpWsLease lease;
    OpWs* w = lease.w;
    if (!w) return YAMS_ERR_INTERNAL;
    if ((rc = w->d[0].reserve(24)) != YAMS_OK) return rc;
    bm_lookup_kernel<<<1, 1, 0, w->st>>>(Dict{F.hashes.as<uint64_t>(), F.offs.as<uint64_t>(), F.terms}, F.ttf.as<uint64_t>(), term_hash,
                                         w->d[0].as<uint64_t>());
    YB_CUDA(cudaGetLastError());
    uint64_t r[3];
    YB_CUDA(cudaMemcpyAsync(r, w->d[0].p, 24, cudaMemcpyDeviceToHost, w->st));
    YB_CUDA(cudaStreamSynchronize(w->st));
    const uint64_t df = r[1] - r[0];
    if (df == 0) return YAMS_OK;
    *out_df = (uint32_t)df;
    YB_CUDA(cudaMemcpy(out_idf, idx->idf.as<float>() + df, 4, cudaMemcpyDeviceToHost));
    *out_total_tf = r[2];
    const uint64_t m = std::min(df, cap);
    if (m) {
        YB_CUDA(cudaMemcpy(out_docs, F.docs.as<uint32_t>() + r[0], m * 4, cudaMemcpyDeviceToHost));
        YB_CUDA(cudaMemcpy(out_tfs, F.tfs.as<uint32_t>() + r[0], m * 4, cudaMemcpyDeviceToHost));
    }
    return YAMS_OK;
    YB_CATCH
}

yams_status_t yams_b200_bm25_doc_lengths(yams_b200_bm25* idx, uint32_t field, uint32_t* out) {
    DeviceCtx* dev = nullptr;
    yams_status_t rc = ensure_device(&dev);
    if (rc != YAMS_OK) return rc;
    YB_ARG(idx, "index is null");
    YB_ARG(field < 2, "field must be 0 (words) or 1 (n-grams)");
    YB_ARG(out || idx->n == 0, "out is null");
    if (idx->n) memcpy(out, idx->f[field].h_dl.data(), idx->n * 4);
    return YAMS_OK;
}

yams_status_t yams_b200_bm25_last_timings(yams_b200_bm25* idx, float out_ms[8]) {
    DeviceCtx* dev = nullptr;
    yams_status_t rc = ensure_device(&dev);
    if (rc != YAMS_OK) return rc;
    YB_ARG(idx && out_ms, "null argument");
    std::lock_guard<std::mutex> g(idx->mu);
    for (int i = 0; i < 8; ++i) out_ms[i] = idx->ms[i];
    return YAMS_OK;
}

void yams_b200_bm25_destroy(yams_b200_bm25* idx) { delete idx; }

}  // extern "C"
