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
// explicit _rn intrinsic: the reference is compiled without -mfma, so nothing may be fused.  Every score call takes one host
// path: its legs go into a host leg list (LegList, one appender per leg kind), one staging step uploads and plans a list
// (stage_legs) and one launches the score kernel over a batch's rows (score_rows), and one driver (run_batches) sizes the
// batches from the bytes a query's rows take, carves them from one arena, and emits each batch's rows and top-k.
//
// RRF (score_bm25_variants_rrf, fusion.cpp; DESIGN.md §4.13): the variants' score rows, their ranked entries as sortable keys,
// one segmented sort per batch, one scatter of 1 / (k + r) per variant in order.  An Atire view shares its parent's word field
// and idf table, which an Atire build of the same texts would reproduce exactly.
//
// Lead field and strategy router (extract_lead_tokens, add_doc(text, aux), score_bm25f, KeyphraseStrategy, the backend's entropy
// route; DESIGN.md §4.14): one warp per document cuts its lead prefix in the uploaded text, the build's own pipeline makes the aux
// fields 2 and 3 from the cut text, and BM25F is more legs: a body-scale leg, then aux legs whose weight is fl(wa * alpha).  The
// keyphrase strategy counts matches with presence legs and z-scores a row with one lane's sequential double sums; the route
// reduces each row's profile on the device with a bound on its distance from the reference's, replaying the row on the host
// when the bound cannot settle it.
//
// Query router (QueryRouter::features / choose, the backend's scoreRouted; DESIGN.md §4.15): one kernel looks up the unfolded
// query words' field-0 statistics, the host computes the features and the recipe in the reference's order, Bm25Atire rows of a
// SubwordAwareBackoff index score with BM_ATIRE legs in the same launch as the others, and the candidate pools are gathered from
// each batch's rows on the device.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <functional>
#include <limits>
#include <memory>
#include <mutex>
#include <new>
#include <unordered_map>
#include <string>
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
    uint64_t terms = 0, posts = 0, sum = 0;   // sum: of dl
    float avg = 0.f;
    std::vector<uint32_t> h_dl;
};

// ---- build kernels ----
__host__ __device__ __forceinline__ bool is_space(uint8_t c) { return c == ' ' || (c >= '\t' && c <= '\r'); }   // isspace, C locale

// The lead-text field (extract_lead_tokens(text, lead), corpus_adapter.cpp:16-39): one warp per document finds the whitespace
// byte that ends its lead-th whitespace-delimited token (none: the document's end) and zeroes the bytes from there to the
// document's end, so the field's words are the prefix's.  *active = 1 when some document's lead text is non-empty (a
// non-whitespace byte before its cut), which activates the reference's aux field.
__global__ void bm_lead_cut_kernel(uint8_t* __restrict__ t, const uint64_t* __restrict__ pos, uint64_t n, uint32_t lead,
                                   uint32_t* __restrict__ active) {
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t d = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; d < n; d += warps) {
        const uint64_t s = pos[d], e = pos[d + 1] - 1;   // the document's bytes; the zero byte after it is not one
        uint64_t cut = e;
        uint32_t count = 0;
        bool any = false;
        for (uint64_t c0 = s; c0 < e; c0 += 32) {
            const uint64_t i = c0 + lane;
            const bool in = i < e, sp = in && is_space(t[i]);
            const unsigned ends = __ballot_sync(0xFFFFFFFFu, sp && i > s && !is_space(t[i - 1]));   // a token ends at i
            const unsigned chars = __ballot_sync(0xFFFFFFFFu, in && !sp);
            const uint32_t m = __popc(ends);
            if (count + m >= lead) {
                const uint32_t bit = __fns(ends, 0, (int)(lead - count));
                cut = c0 + bit;
                any = any || (chars & ((1u << bit) - 1u)) != 0;
                break;
            }
            count += m;
            any = any || chars != 0;
        }
        for (uint64_t i = cut + lane; i < e; i += 32) t[i] = 0;
        if (lane == 0 && any) *active = 1;
    }
}

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

// ConceptIndex::hash_bigram: ordered (a, b) (concept_mining.cpp:40-44)
__host__ __device__ __forceinline__ uint64_t hash_bigram(uint64_t a, uint64_t b) { return sm64_mix(a ^ sm64_mix(b + 0x9E3779B97F4A7C15ULL)); }

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

// one word: its hash (FOLD: of the ASCII-lowercased bytes), document, length and n-gram count
template <bool FOLD>
__global__ void bm_words_kernel(const uint8_t* __restrict__ t, const uint64_t* __restrict__ wstart, uint64_t nw,
                                const uint64_t* __restrict__ pos, uint64_t n, uint64_t h0, uint32_t kmin, uint32_t kmax,
                                uint64_t* __restrict__ whash, uint32_t* __restrict__ wdoc, uint32_t* __restrict__ wlen,
                                uint64_t* __restrict__ gcnt) {
    for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < nw; w += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t s = wstart[w], L = word_end(t, s) - s;
        whash[w] = gram_hash<FOLD>(t + s, L, h0);
        wdoc[w] = (uint32_t)last_le(pos, n + 1, s);
        if (wlen) wlen[w] = (uint32_t)L;
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
// Field kinds of a leg: 0 the words, 1 the n-grams, 2 the lead-text words, 3 the lead-text n-grams (the index's four fields),
// 4 a mined concept (ConceptIndex, blended after the BM25 legs of its query), 5 BM25F's body scale (every score of the row
// times the leg's weight, between the body legs and the aux legs).
constexpr uint32_t BM_AUX = 2;
constexpr uint32_t BM_CONCEPT = 4;
constexpr uint32_t BM_SCALE = 5;
// A presence leg (RawLeg / Leg pad of a field-0 leg): adds 1.0f to each document of a keyphrase's word list whose single-term
// score (score_weighted_hashes with weight 1: bm25plus, or score_atire for Atire) is > 0, counting KeyphraseStrategy's matches.
constexpr uint32_t BM_PRESENCE = 1;
// An Atire leg (RawLeg / Leg pad of a word leg of a SubwordAwareBackoff index): scored as an Atire build of the same texts would
// score it (score_atire over the word's list), so rows of both variants share one launch (the query router's Bm25Atire rows).
constexpr uint32_t BM_ATIRE = 2;

struct RawLeg {        // one query word (field 0 / 2), one distinct n-gram of it (1 / 3), one matched concept, or a scale
    uint64_t hash;
    uint64_t term_hash;
    uint32_t field;
    uint32_t pad;      // BM_SCALE: the scale's float bits; BM_PRESENCE, BM_ATIRE: the leg's kind
};
struct Leg {           // an addition over documents docs[b, e) of `field`; empty when b == e
    uint64_t b, e;
    float w, idf;
    uint32_t field;
    uint32_t pad;      // BM_PRESENCE: a presence leg; BM_ATIRE: an Atire leg
};
struct Dict {
    const uint64_t* hashes;
    const uint64_t* offs;
    uint64_t terms;
};
struct ConceptDict {   // the kept concepts of a ConceptIndex: sorted hashes, posting offsets, pmi and idf; the blend's weight
    Dict d;
    const float* pmi;
    const float* idf;
    float weight;
};

__device__ __forceinline__ bool dict_find(const Dict& D, uint64_t h, uint64_t* b, uint64_t* e, uint64_t* t_out = nullptr) {
    if (D.terms == 0 || h < D.hashes[0]) return false;
    const uint64_t t = last_le(D.hashes, D.terms, h);
    if (D.hashes[t] != h) return false;
    *b = D.offs[t];
    *e = D.offs[t + 1];
    if (t_out) *t_out = t;
    return true;
}

struct FieldDicts {     // the index's fields 0..3
    Dict d[4];
};

// An aux leg's weight is fl(wa * alpha), fl(wa * (1 - alpha)) or wa (Atire), taken before the product with the score, as
// score_bm25f's `weight_aux * alpha * bm25plus` (bm25.cpp:1041-1060, 1087); alpha comes from the aux field's df.
__global__ void bm_plan_kernel(const RawLeg* __restrict__ raw, uint64_t nlegs, FieldDicts f, const float* __restrict__ idf,
                               int sab, float gamma, float wa, ConceptDict c, Leg* __restrict__ legs) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nlegs; i += (uint64_t)gridDim.x * blockDim.x) {
        const RawLeg r = raw[i];
        Leg L{};
        L.field = r.field;
        uint64_t b = 0, e = 0, t = 0;
        if (r.field == BM_SCALE) {
            L.w = __uint_as_float(r.pad);
        } else if (r.field == BM_CONCEPT) {
            // wpmi = weight * pmi (concept_mining.cpp:106); the host only emits concepts the index keeps
            if (dict_find(c.d, r.hash, &b, &e, &t)) { L.b = b; L.e = e; L.w = __fmul_rn(c.weight, c.pmi[t]); L.idf = c.idf[t]; }
        } else {
            const bool aux = r.field >= BM_AUX;
            const Dict& w = f.d[r.field & BM_AUX];
            if (r.pad == BM_PRESENCE) {   // a keyphrase's word list, whatever the variant
                if (dict_find(w, r.hash, &b, &e)) { L.b = b; L.e = e; L.idf = idf[e - b]; L.pad = BM_PRESENCE; }
            } else if (!sab || r.pad == BM_ATIRE) {
                if (dict_find(w, r.hash, &b, &e)) { L.b = b; L.e = e; L.w = aux ? wa : 0.0f; L.idf = idf[e - b]; L.pad = r.pad; }
            } else {
                // alpha = float(df) / (float(df) + gamma), 0 when the word is unknown (bm25.cpp:805-807)
                const uint64_t df = dict_find(w, r.term_hash, &b, &e) ? e - b : 0;
                const float alpha = df > 0 ? __fdiv_rn(__ull2float_rn(df), __fadd_rn(__ull2float_rn(df), gamma)) : 0.0f;
                if ((r.field & 1) == 0) {
                    if (alpha > 0.0f) { L.b = b; L.e = e; L.w = aux ? __fmul_rn(wa, alpha) : alpha; L.idf = idf[df]; }
                } else if (alpha < 1.0f && dict_find(f.d[r.field], r.hash, &b, &e)) {
                    const float w1 = __fsub_rn(1.0f, alpha);
                    L.b = b; L.e = e; L.w = aux ? __fmul_rn(wa, w1) : w1; L.idf = idf[e - b];
                }
            }
        }
        legs[i] = L;
    }
}

struct ScoreArgs {
    const Leg* legs;
    const uint64_t* qoff;     // legs of query q: [qoff[q], qoff[q + 1])
    uint32_t q0;              // first query of the batch
    const uint32_t* docs[5];
    const uint32_t* tfs[5];
    const uint32_t* dl[5];
    float avg[5];             // fields 0..3: avg_dl > 0 ? avg_dl : 1; concepts: avg_bigram_dl (> 0 whenever a concept exists)
    float k1[5], b[5];        // fields 0..3: Bm25Config's; concepts: ConceptConfig's
    uint64_t n;
    float delta;
    int sab;
    const float* init;        // nullable: [batch][n] starting scores (the standalone blend), else zeros
    float* out;               // [batch][n]; may be init
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
    const float* init = a.init ? a.init + (uint64_t)blockIdx.y * a.n + lo : nullptr;
    for (uint32_t i = threadIdx.x; i < len; i += BM_THREADS) s[i] = init ? init[i] : 0.0f;
    __syncthreads();
    for (uint64_t l = a.qoff[q]; l < a.qoff[q + 1]; ++l) {
        const Leg g = a.legs[l];
        if (g.field == BM_SCALE) {   // score_bm25f's `s *= weight_body` over the whole row (bm25.cpp:993-996)
            for (uint32_t i = threadIdx.x; i < len; i += BM_THREADS) s[i] = __fmul_rn(s[i], g.w);
            __syncthreads();
            continue;
        }
        if (g.b == g.e) continue;
        const uint32_t* docs = a.docs[g.field];
        const uint64_t sb = first_ge(docs, g.b, g.e, lo), se = first_ge(docs, sb, g.e, lo + len);
        if (sb == se) continue;   // the same for every thread of the CTA
        const uint32_t* tfs = a.tfs[g.field];
        const uint32_t* dlv = a.dl[g.field];
        const float avg = a.avg[g.field], k1 = a.k1[g.field], b = a.b[g.field];
        const float k1p1 = __fadd_rn(k1, 1.0f), omb = __fsub_rn(1.0f, b);
        const bool sab = a.sab && g.pad != BM_ATIRE;   // this leg's arithmetic
        for (uint64_t i = sb + threadIdx.x; i < se; i += BM_THREADS) {
            const uint32_t d = docs[i];
            const float tf = __uint2float_rn(tfs[i]), dl = __uint2float_rn(dlv[d]);
            // tf + k1 * (1 - b + b * dl / avg)
            const float denom = __fadd_rn(tf, __fmul_rn(k1, __fadd_rn(omb, __fdiv_rn(__fmul_rn(b, dl), avg))));
            // idf * tf * (k1 + 1) / denom: Atire, and a concept's score_atire (concept_mining.cpp:31-36)
            const float atire = __fdiv_rn(__fmul_rn(__fmul_rn(g.idf, tf), k1p1), denom);
            // idf * (tf * (k1 + 1) / denom + delta)
            const float plus = __fmul_rn(g.idf, __fadd_rn(__fdiv_rn(__fmul_rn(tf, k1p1), denom), a.delta));
            float add;
            if (g.pad == BM_PRESENCE)    // 1.0f * the single-term score > 0
                add = (sab ? plus : atire) > 0.0f ? 1.0f : 0.0f;
            else if (g.field == BM_CONCEPT || (!sab && g.field == BM_AUX))   // wpmi * score_atire; weight_aux * score_atire
                add = __fmul_rn(g.w, atire);
            else if (sab)                // alpha * bm25plus
                add = __fmul_rn(g.w, plus);
            else
                add = atire;
            s[d - lo] = __fadd_rn(s[d - lo], add);
        }
        __syncthreads();
    }
    float* out = a.out + (uint64_t)blockIdx.y * a.n + lo;
    for (uint32_t i = threadIdx.x; i < len; i += BM_THREADS) out[i] = s[i];
}

// The strategy router's entropy profile of one score row per block (SimeonLexicalBackend::scoreStrategyRouted,
// simeon_lexical_backend.cpp:1000-1017): out[3 * row] = max, [+1] = the documents of score > 0, [+2] = the sum over them of
// sn * -log(sn), sn = (double)(s / max), 0 when max <= 0.  The sum is a tree in double with the device's log; the host bounds
// its distance from the reference's sequential sum with glibc's log (route_pool).
__global__ void __launch_bounds__(BM_THREADS) bm_route_kernel(const float* __restrict__ rows, uint64_t n, double* __restrict__ out) {
    using RF = cub::BlockReduce<float, BM_THREADS>;
    using RD = cub::BlockReduce<double, BM_THREADS>;
    __shared__ union { typename RF::TempStorage f; typename RD::TempStorage d; } ts;
    __shared__ float top;
    const float* s = rows + (uint64_t)blockIdx.x * n;
    float m = 0.0f;
    for (uint64_t i = threadIdx.x; i < n; i += BM_THREADS) m = fmaxf(m, s[i]);
    m = RF(ts.f).Reduce(m, cub::Max());
    if (threadIdx.x == 0) top = m;
    __syncthreads();
    m = top;
    double sum = 0.0, cnt = 0.0;
    if (m > 0.0f)
        for (uint64_t i = threadIdx.x; i < n; i += BM_THREADS) {
            const float v = s[i];
            if (!(v > 0.0f)) continue;
            const double sn = (double)__fdiv_rn(v, m);
            if (sn > 0.0) sum = __dadd_rn(sum, __dmul_rn(sn, -log(sn)));
            cnt += 1.0;
        }
    sum = RD(ts.d).Sum(sum);
    __syncthreads();
    cnt = RD(ts.d).Sum(cnt);
    if (threadIdx.x == 0) {
        out[3 * blockIdx.x] = (double)m;
        out[3 * blockIdx.x + 1] = cnt;
        out[3 * blockIdx.x + 2] = sum;
    }
}

// KeyphraseStrategy's boost of one gated row per block (retrieval_strategy.cpp:17-30, 243-250): zscore_inplace's two sums in
// double over the n scores in document order -- one lane adds while its warp stages the row through shared memory (adding +0.0
// is exact, so the mean's pass skips zeros; the variance's may not) -- then every document's
// float((x - mean) / sd) + lw * (float(matches) / nkp).  zrow[b] is the row, zp[2 b] lw = fl(lam * 0.25f), zp[2 b + 1] nkp.
__global__ void __launch_bounds__(BM_THREADS) bm_zscore_kernel(float* __restrict__ rows, const float* __restrict__ counts, uint64_t n,
                                                               const uint32_t* __restrict__ zrow, const float* __restrict__ zp) {
    constexpr uint32_t CH = 1024;
    __shared__ float buf[CH];
    __shared__ double stat[2];
    float* x = rows + (uint64_t)zrow[blockIdx.x] * n;
    const float* cnt = counts + (uint64_t)zrow[blockIdx.x] * n;
    if (threadIdx.x < 32) {
        const uint32_t lane = threadIdx.x;
        double mean = 0.0;
        for (int pass = 0; pass < 2; ++pass) {
            double acc = 0.0;
            for (uint64_t c0 = 0; c0 < n; c0 += CH) {
                const uint32_t len = (uint32_t)min((uint64_t)CH, n - c0);
                for (uint32_t j = lane; j < len; j += 32) buf[j] = x[c0 + j];
                __syncwarp();
                if (lane == 0) {
                    if (pass == 0) {
                        for (uint32_t j = 0; j < len; ++j)
                            if (buf[j] != 0.0f) acc = __dadd_rn(acc, (double)buf[j]);
                    } else {
                        for (uint32_t j = 0; j < len; ++j) {
                            const double d = __dsub_rn((double)buf[j], mean);
                            acc = __dadd_rn(acc, __dmul_rn(d, d));
                        }
                    }
                }
                __syncwarp();
            }
            if (pass == 0) mean = __shfl_sync(0xFFFFFFFFu, __ddiv_rn(acc, (double)n), 0);
            else if (lane == 0) {
                stat[0] = mean;
                stat[1] = (double)__double2float_rn(__dadd_rn(__dsqrt_rn(__ddiv_rn(acc, (double)n)), 1e-12));
            }
        }
    }
    __syncthreads();
    const double mean = stat[0], sd = stat[1];
    const float lw = zp[2 * blockIdx.x], nkp = zp[2 * blockIdx.x + 1];
    for (uint64_t i = threadIdx.x; i < n; i += BM_THREADS)
        x[i] = __fadd_rn(__double2float_rn(__ddiv_rn(__dsub_rn((double)x[i], mean), sd)), __fmul_rn(lw, __fdiv_rn(cnt[i], nkp)));
}

// The query router's projection onto the caller's candidate pools (scoreRouted, simeon_lexical_backend.cpp:920-931): out[j] =
// the row's score of candidate j if finite, else 0; 0 for a candidate the index does not hold (any index >= n).  Block row y is
// query q0 + y of the batch; its pool is docs[off[q], off[q + 1]).
__global__ void __launch_bounds__(BM_THREADS) bm_pool_gather_kernel(const float* __restrict__ rows, uint64_t n, uint32_t q0,
                                                                    const uint64_t* __restrict__ off, const uint32_t* __restrict__ docs,
                                                                    float* __restrict__ out) {
    const uint32_t q = q0 + blockIdx.y;
    const float* row = rows + (uint64_t)blockIdx.y * n;
    for (uint64_t j = off[q] + (uint64_t)blockIdx.x * BM_THREADS + threadIdx.x; j < off[q + 1]; j += (uint64_t)gridDim.x * BM_THREADS) {
        const uint32_t d = docs[j];
        const float v = d < n ? row[d] : 0.0f;
        out[j] = isfinite(v) ? v : 0.0f;
    }
}

inline unsigned bm_grid(uint64_t n) { return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((n + BM_THREADS - 1) / BM_THREADS, 65535ull * 4)); }

// cub temp storage in a growable buffer
struct CubTmp {
    DevBuf buf;
    size_t bytes = 0;
    yams_status_t grow() { return buf.reserve(std::max<size_t>(bytes, 256)); }
};

// The score calls' workspace: the staged legs (raw, planned, per-query offsets), the arena of a batch's rows (and whatever a
// path carves from it) and the top-k selection
struct ScoreWs {
    DevBuf raw, legs, qoff, rows, sel, seln;
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
    uint64_t n = 0, total_tokens = 0, pruned = 0, aux_pruned = 0;
    uint32_t lead = 0;        // the lead-text field's token count (0: no lead field)
    bool aux_active = false;  // some document's lead text is non-empty: the reference's aux field exists for all n documents
    // Fields 0 words, 1 n-grams, 2 lead-text words, 3 lead-text n-grams.  The fields and the idf table are shared with the
    // index's Atire views (yams_b200_bm25_atire_view), which read the word fields and the table in place; whichever handle goes
    // last frees them.  Nothing writes them after the build.
    std::shared_ptr<Bm25Field> f[4] = {std::make_shared<Bm25Field>(), std::make_shared<Bm25Field>(), std::make_shared<Bm25Field>(),
                                       std::make_shared<Bm25Field>()};
    std::shared_ptr<DevBuf> idf = std::make_shared<DevBuf>();   // n + 1 floats: idf of df = 0..n
    cudaStream_t st = nullptr;
    cudaEvent_t ev[2] = {nullptr, nullptr};
    ScoreWs ws;
    DevBuf route, zrow, zp;                     // strategy workspace: route profiles, z-score rows
    cudaEvent_t zev[2] = {nullptr, nullptr};
    yams_bm25_strategy_stats sstats{};
    DevBuf cnt, base;                           // RRF workspace: ranked entries per tile, their scan (on the first variant's)
    DevBuf rwords, rstats, pool_off, pool_docs, pool_out;   // query-router workspace: word lookups, candidate pools
    CubTmp tmp;
    float ms[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    std::mutex mu;
    ~yams_b200_bm25() {
        if (st) cudaStreamSynchronize(st);
        for (auto& e : ev)
            if (e) cudaEventDestroy(e);
        for (auto& e : zev)
            if (e) cudaEventDestroy(e);
        if (st) cudaStreamDestroy(st);
    }
};

// simeon::ConceptIndex mined against an index (DESIGN.md §4.12).  It owns everything it scores with, the hash seed included, and
// may outlive the index.
struct yams_b200_concepts {
    DeviceCtx* dev = nullptr;
    yams_concept_config cfg{};
    uint64_t h0 = 0;                 // gram_hash_h0 of the index's hash seed
    uint64_t n = 0, sum_bdl = 0, distinct = 0, passed_ttf = 0, accepted = 0;
    float avg = 0.f;
    uint32_t replayed = 0;
    DevBuf bdl;                      // n: bigram_dl
    std::vector<uint32_t> h_bdl;
    // the kept concepts, by hash ascending: device dictionary and postings, host copies of what find() and the blend read
    uint64_t size = 0;
    DevBuf hashes, offs, docs, tfs, pmi, idf;
    std::vector<uint64_t> h_hashes, h_offs, h_ttf, h_a, h_b;
    std::vector<float> h_pmi, h_idf;
    cudaStream_t st = nullptr;
    cudaEvent_t ev[2] = {nullptr, nullptr};
    ScoreWs ws;                      // the standalone blend's
    float ms[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    std::mutex mu;
    ~yams_b200_concepts() {
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

// device ms of the work `fn` enqueues on the handle's stream (waits for it)
template <typename H, typename F>
static yams_status_t timed(H* x, float* acc, F&& fn) {
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
                                  uint64_t* pruned, CubTmp& tmp) {
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
        *pruned = nterms;   // minus the terms left, below
    }
    if (prune && *pruned) *pruned -= F.terms;
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

// texts -> one device layout, document d at pos[d] with one zero byte after it (so no word crosses a document), 16 more zero
// bytes at the end; d_pos = pos[0..n]
static yams_status_t upload_texts(const char* const* texts, const size_t* lens, uint64_t n, std::vector<uint64_t>& pos, DevBuf& text,
                                  DevBuf& d_pos, cudaStream_t st) {
    pos.assign(n + 1, 0);
    std::vector<LayoutPiece> pieces;
    pieces.reserve(n);
    for (uint64_t d = 0; d < n; ++d) {
        if (lens[d]) pieces.push_back({pos[d], (uint64_t)lens[d], reinterpret_cast<const uint8_t*>(texts[d])});
        pos[d + 1] = pos[d] + lens[d] + 1;
    }
    const uint64_t L = pos[n];
    yams_status_t r;
    if ((r = text.reserve(L + 16)) != YAMS_OK || (r = d_pos.reserve((n + 1) * 8)) != YAMS_OK) return r;
    HostBuf pin[2];
    cudaEvent_t done[2] = {nullptr, nullptr};
    for (auto& e : done) YB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    r = staged_upload(pin, done, text.as<uint8_t>(), L, pieces, st);
    if (r == YAMS_OK && cudaMemsetAsync(text.as<uint8_t>() + L, 0, 16, st) != cudaSuccess) r = YAMS_ERR_INTERNAL;
    if (r == YAMS_OK && cudaMemcpyAsync(d_pos.p, pos.data(), (n + 1) * 8, cudaMemcpyHostToDevice, st) != cudaSuccess) r = YAMS_ERR_INTERNAL;
    cudaStreamSynchronize(st);   // the pinned buffers and pos are read until here
    for (auto& e : done) cudaEventDestroy(e);
    if (r == YAMS_ERR_INTERNAL) set_last_error("text upload failed");
    return r;
}

// The word field fw and the n-gram field fw + 1 of the texts laid out in `text` (upload_texts): per-document lengths and
// averages, then the slices' pairs, sorts and runs, then each field's dictionary.  *pruned gets the n-grams the df rule drops,
// *nslices the document slices.  The last pass frees the text before the dictionaries, the build's most memory-hungry stage.
static yams_status_t build_fields(yams_b200_bm25* x, DevBuf& text, const DevBuf& d_pos, const std::vector<uint64_t>& pos, int fw,
                                  uint64_t* pruned, uint64_t* nslices_out, bool last) {
    cudaStream_t st = x->st;
    const uint64_t n = x->n;
    const bool sab = x->cfg.variant == YAMS_BM25_SUBWORD_AWARE_BACKOFF;
    const uint32_t kmin = x->cfg.ngram_min, kmax = x->cfg.ngram_max;
    const uint64_t h0 = gram_hash_h0(x->cfg.hash_seed);
    Bm25Field* fs[2] = {x->f[fw].get(), x->f[fw + 1].get()};
    yams_status_t rc;
    for (Bm25Field* pf : fs) {
        if ((rc = pf->dl.reserve(std::max<uint64_t>(n, 1) * 4)) != YAMS_OK) return rc;
        YB_CUDA(cudaMemsetAsync(pf->dl.p, 0, std::max<uint64_t>(n, 1) * 4, st));
        pf->h_dl.assign(n, 0);
    }
    const uint64_t L = pos[n];
    // ---- dl / ngram_dl ----
    rc = timed(x, &x->ms[1], [&]() -> yams_status_t {
        if (L) bm_doc_counts_kernel<<<bm_grid(L), BM_THREADS, 0, st>>>(text.as<uint8_t>(), L, d_pos.as<uint64_t>(), n, sab, kmin, kmax,
                                                                       fs[0]->dl.as<uint32_t>(), fs[1]->dl.as<uint32_t>());
        YB_CUDA(cudaGetLastError());
        for (Bm25Field* pf : fs)
            if (n) YB_CUDA(cudaMemcpyAsync(pf->h_dl.data(), pf->dl.p, n * 4, cudaMemcpyDeviceToHost, st));
        return YAMS_OK;
    });
    if (rc != YAMS_OK) return rc;
    for (Bm25Field* pf : fs) {
        pf->sum = 0;
        for (uint32_t v : pf->h_dl) pf->sum += v;
        pf->avg = n == 0 ? 0.0f : (float)((double)pf->sum / (double)n);   // finalize_word_field (bm25.cpp:668-676)
    }
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
        const uint64_t c = (uint64_t)fs[0]->h_dl[d] + (sab ? (uint64_t)fs[1]->h_dl[d] : 0);
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
                bm_words_kernel<true><<<bm_grid(nw), BM_THREADS, 0, st>>>(text.as<uint8_t>(), wstart.as<uint64_t>(), nw, d_pos.as<uint64_t>(), n, h0,
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
    if (last) text = DevBuf();
    for (int fi = 0; fi < (sab ? 2 : 1); ++fi) {
        rc = timed(x, &x->ms[3], [&] {
            return finish_field(x, *fs[fi], ph[fi], pv[fi], np[fi], nslices > 1, fi == 1 && x->cfg.ngram_df_prune_ratio > 0.0f && n > 0,
                                pruned, tmp);
        });
        if (rc != YAMS_OK) return rc;
    }
    *nslices_out = nslices;
    return YAMS_OK;
}

// Bm25Index::add_doc(text, aux) for every document, then finalize(): the body's fields, then, with a lead length, the same
// pipeline over the texts cut to their lead prefixes (bytes past the cut zeroed, so they separate words) for the aux fields.
// An inactive aux field has no words, hence no terms (nothing of it is read) and zero lengths, as the reference's.  The aux
// fields have the body's document count whenever they are active, so they share its idf table (which depends on n alone).
static yams_status_t bm25_build(yams_b200_bm25* x, const char* const* texts, const size_t* lens) {
    const double t0 = wall_ms();
    cudaStream_t st = x->st;
    const uint64_t n = x->n;
    yams_status_t rc;
    std::vector<uint64_t> pos;
    DevBuf text, d_pos;
    rc = timed(x, &x->ms[0], [&] { return upload_texts(texts, lens, n, pos, text, d_pos, st); });
    if (rc != YAMS_OK) return rc;
    uint64_t slices = 0, aux_slices = 0;
    if ((rc = build_fields(x, text, d_pos, pos, 0, &x->pruned, &slices, !(x->lead && n))) != YAMS_OK) return rc;
    x->total_tokens = x->f[0]->sum;
    for (int fi = 2; fi < 4; ++fi) x->f[fi]->h_dl.assign(n, 0);
    if (x->lead && n) {
        DevBuf flag;
        uint32_t active = 0;
        rc = timed(x, &x->ms[1], [&]() -> yams_status_t {
            yams_status_t r;
            if ((r = flag.reserve(4)) != YAMS_OK) return r;
            YB_CUDA(cudaMemsetAsync(flag.p, 0, 4, st));
            bm_lead_cut_kernel<<<(unsigned)std::min<uint64_t>((n + 7) / 8, 65535ull * 4), BM_THREADS, 0, st>>>(
                text.as<uint8_t>(), d_pos.as<uint64_t>(), n, x->lead, flag.as<uint32_t>());
            YB_CUDA(cudaGetLastError());
            YB_CUDA(cudaMemcpyAsync(&active, flag.p, 4, cudaMemcpyDeviceToHost, st));
            return YAMS_OK;
        });
        if (rc != YAMS_OK) return rc;
        x->aux_active = active != 0;
        if (x->aux_active && (rc = build_fields(x, text, d_pos, pos, 2, &x->aux_pruned, &aux_slices, true)) != YAMS_OK) return rc;
    }
    text = DevBuf();
    // ---- idf of df = 0..n: the reference's float expression and std::log(float) (bm25.cpp:680-682, 729-731) ----
    std::vector<float> idf(n + 1);
    const float nf = (float)n;
    for (uint64_t df = 0; df <= n; ++df) {
        const float d = (float)df;
        idf[df] = std::log((nf - d + 0.5f) / (d + 0.5f) + 1.0f);
    }
    if ((rc = x->idf->reserve((n + 1) * 4)) != YAMS_OK) return rc;
    YB_CUDA(cudaMemcpyAsync(x->idf->p, idf.data(), (n + 1) * 4, cudaMemcpyHostToDevice, st));
    YB_CUDA(cudaStreamSynchronize(st));
    x->ms[4] = (float)(wall_ms() - t0);
    x->ms[5] = (float)(slices + aux_slices);
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

// The end of the lead prefix of p[0, len): the whitespace byte that ends its lead-th token, else len (extract_lead_tokens,
// corpus_adapter.cpp:16-39).  The prefix's words are the lead text's: the reference only turns whitespace into ' ' and trims.
static size_t lead_cut(const uint8_t* p, size_t len, uint32_t lead) {
    uint32_t tokens = 0;
    bool in_token = false;
    for (size_t i = 0; i < len; ++i) {
        if (is_space(p[i])) {
            if (in_token) { ++tokens; in_token = false; }
            if (tokens >= lead) return i;
        } else {
            in_token = true;
        }
    }
    return len;
}

// The lexical backend's strategies over its primary index (SimeonLexicalBackend, simeon_lexical_backend.cpp:563-580): Bm25Strategy
// scores score_bm25f(q, lead(q, 64), 0.85, 0.15), or score(q) when that lead text is empty; LeadFieldStrategy scores
// score_bm25f(q, q, 0.85, 0.15) (retrieval_strategy.cpp:84-127).
constexpr uint32_t STRATEGY_LEAD = 64;
constexpr float STRATEGY_WB = 0.85f, STRATEGY_WA = 0.15f;

// The raw legs of a run of queries in the reference's order: query j's are raw[qoff[j], qoff[j + 1]).  Each appender adds one
// kind of leg to the open query; end_query closes it.
struct LegList {
    std::vector<RawLeg> raw;
    std::vector<uint64_t> qoff{0};
    std::vector<std::pair<size_t, size_t>> ws;   // the appenders' scratch
    std::vector<uint8_t> low;
    std::unordered_set<uint64_t> seen;
    std::vector<uint64_t> qw;

    void clear() {
        raw.clear();
        qoff.assign(1, 0);
    }
    void end_query() { qoff.push_back(raw.size()); }

    // The BM25 legs of the words of p[0, len) over fields fw (words) and fw + 1 (n-grams) of index x, in Bm25Index::score's
    // order; with atire, the legs an Atire build of the same texts would score (words only, as BM_ATIRE legs)
    void words(const yams_b200_bm25* x, const uint8_t* p, size_t len, uint32_t fw, bool atire = false) {
        const bool sab = x->cfg.variant == YAMS_BM25_SUBWORD_AWARE_BACKOFF && !atire;
        const uint64_t h0 = gram_hash_h0(x->cfg.hash_seed);
        query_words(p, len, ws);
        for (const auto& [s, l] : ws) {
            low.resize(l);
            for (size_t i = 0; i < l; ++i) low[i] = ascii_lower(p[s + i]);
            const uint64_t th = gram_hash(low.data(), l, h0);
            raw.push_back({th, th, fw, atire ? BM_ATIRE : 0u});
            if (!sab) continue;
            // collect_unique_query_ngrams (bm25.cpp:151-161): k ascending, position ascending, first occurrence of each hash
            seen.clear();
            for (uint64_t kk = x->cfg.ngram_min; kk <= x->cfg.ngram_max && kk <= l; ++kk)
                for (uint64_t i = 0; i + kk <= l; ++i) {
                    const uint64_t gh = gram_hash(low.data() + i, kk, h0);
                    if (seen.insert(gh).second) raw.push_back({gh, th, fw + 1, 0});
                }
        }
    }
    // score_bm25f's legs after the body's, for strategy pool 0 or 2: the body scale, then the aux query's legs over the aux
    // fields.  The aux query is the query's lead prefix (Bm25Strategy) or the query (LeadFieldStrategy); a lead prefix of
    // whitespace alone is no evidence, and the query scores as Bm25Index::score alone.
    void bm25f(const yams_b200_bm25* x, const uint8_t* p, size_t len, uint32_t pool) {
        size_t aux = len;
        if (pool == YAMS_BM25_STRATEGY_BM25) {
            aux = lead_cut(p, len, STRATEGY_LEAD);
            if (std::all_of(p, p + aux, [](uint8_t ch) { return is_space(ch); })) return;
        }
        uint32_t wb_bits;
        memcpy(&wb_bits, &STRATEGY_WB, 4);
        raw.push_back({0, 0, BM_SCALE, wb_bits});   // weight_body != 1 (bm25.cpp:993-996)
        words(x, p, aux, BM_AUX);
    }
    // one presence leg per keyphrase hash
    void presence(const std::vector<uint64_t>& kh) {
        for (uint64_t h : kh) raw.push_back({h, h, 0, BM_PRESENCE});
    }
    // The concepts of concept index c that p[0, len) matches, in ConceptIndex::blend_into's order: its unfolded words' adjacent
    // bigrams that are kept concepts, emplaced into an unordered_map reserved for the word count, in that map's iteration order
    // (concept_mining.cpp:82-104).  The additions of a document in several matched concepts are made in this order.
    void concepts(const yams_b200_concepts* c, const uint8_t* p, size_t len) {
        query_words(p, len, ws);
        if (c->size == 0 || ws.size() < 2) return;
        qw.resize(ws.size());
        for (size_t i = 0; i < ws.size(); ++i) qw[i] = gram_hash(p + ws[i].first, ws[i].second, c->h0);
        std::unordered_map<uint64_t, uint32_t> matched;
        matched.reserve(qw.size());
        for (size_t i = 1; i < qw.size(); ++i) {
            const uint64_t bh = hash_bigram(qw[i - 1], qw[i]);
            const auto it = std::lower_bound(c->h_hashes.begin(), c->h_hashes.end(), bh);
            if (it != c->h_hashes.end() && *it == bh) matched.emplace(bh, (uint32_t)(it - c->h_hashes.begin()));
        }
        for (const auto& m : matched) raw.push_back({m.first, m.first, BM_CONCEPT, 0});
    }
};

// What a leg list is planned and scored against: index x's fields and concept index c's concepts at the blend's weight.  Either
// may be null when the list has none of its legs.
struct Scorer {
    const yams_b200_bm25* x;
    const yams_b200_concepts* c;
    float weight;
};

// Uploads leg list L to w, one copy of its legs and one of its offsets, and plans it.  L's queries form ns blocks of equal count,
// block i planned against s[i] (RRF: one block per variant, each against its own dictionaries, then the concepts').
static yams_status_t stage_legs(ScoreWs& w, const LegList& L, const Scorer* s, uint32_t ns, cudaStream_t st) {
    const uint64_t nlegs = L.raw.size(), per = (L.qoff.size() - 1) / ns;
    if (nlegs == 0) return YAMS_OK;
    yams_status_t rc;
    if ((rc = w.raw.reserve(nlegs * sizeof(RawLeg))) != YAMS_OK || (rc = w.legs.reserve(nlegs * sizeof(Leg))) != YAMS_OK ||
        (rc = w.qoff.reserve(L.qoff.size() * 8)) != YAMS_OK)
        return rc;
    YB_CUDA(cudaMemcpyAsync(w.raw.p, L.raw.data(), nlegs * sizeof(RawLeg), cudaMemcpyHostToDevice, st));
    YB_CUDA(cudaMemcpyAsync(w.qoff.p, L.qoff.data(), L.qoff.size() * 8, cudaMemcpyHostToDevice, st));
    for (uint32_t i = 0; i < ns; ++i) {
        const uint64_t lb = L.qoff[i * per], le = L.qoff[(i + 1) * per];
        if (lb == le) continue;
        const yams_b200_bm25* x = s[i].x;
        FieldDicts f{};
        for (int fi = 0; x && fi < 4; ++fi) f.d[fi] = Dict{x->f[fi]->hashes.as<uint64_t>(), x->f[fi]->offs.as<uint64_t>(), x->f[fi]->terms};
        const yams_b200_concepts* c = s[i].c;
        const ConceptDict cd = c ? ConceptDict{Dict{c->hashes.as<uint64_t>(), c->offs.as<uint64_t>(), c->size}, c->pmi.as<float>(),
                                               c->idf.as<float>(), s[i].weight}
                                 : ConceptDict{};
        bm_plan_kernel<<<bm_grid(le - lb), BM_THREADS, 0, st>>>(w.raw.as<RawLeg>() + lb, le - lb, f, x ? x->idf->as<float>() : nullptr,
                                                               x && x->cfg.variant == YAMS_BM25_SUBWORD_AWARE_BACKOFF,
                                                               x ? x->cfg.subword_gamma : 0.0f, STRATEGY_WA, cd, w.legs.as<Leg>() + lb);
        YB_CUDA(cudaGetLastError());
    }
    return YAMS_OK;
}

// Scores queries [q0, q0 + qb) of the staged list L against s onto rows[qb][n]: from zero, or (in_place) onto the rows' own
// scores, each CTA reading and writing its tile
static yams_status_t score_rows(const ScoreWs& w, const LegList& L, const Scorer& s, uint64_t n, uint64_t q0, uint32_t qb, bool in_place,
                                float* rows, cudaStream_t st) {
    if (L.qoff[q0] == L.qoff[q0 + qb]) {   // no leg: zeros, or the rows as they are
        if (!in_place) YB_CUDA(cudaMemsetAsync(rows, 0, (uint64_t)qb * n * 4, st));
        return YAMS_OK;
    }
    ScoreArgs a{};
    if (const yams_b200_bm25* x = s.x) {
        for (int fi = 0; fi < 4; ++fi) {
            a.docs[fi] = x->f[fi]->docs.as<uint32_t>();
            a.tfs[fi] = x->f[fi]->tfs.as<uint32_t>();
            a.dl[fi] = x->f[fi]->dl.as<uint32_t>();
            a.avg[fi] = x->f[fi]->avg > 0.0f ? x->f[fi]->avg : 1.0f;
            a.k1[fi] = x->cfg.k1;
            a.b[fi] = x->cfg.b;
        }
        a.delta = x->cfg.delta;
        a.sab = x->cfg.variant == YAMS_BM25_SUBWORD_AWARE_BACKOFF;
    }
    if (const yams_b200_concepts* c = s.c) {
        a.docs[BM_CONCEPT] = c->docs.as<uint32_t>();
        a.tfs[BM_CONCEPT] = c->tfs.as<uint32_t>();
        a.dl[BM_CONCEPT] = c->bdl.as<uint32_t>();
        a.avg[BM_CONCEPT] = c->avg;
        a.k1[BM_CONCEPT] = c->cfg.k1;
        a.b[BM_CONCEPT] = c->cfg.b;
    }
    a.legs = w.legs.as<Leg>();
    a.qoff = w.qoff.as<uint64_t>() + q0;
    a.n = n;
    a.init = in_place ? rows : nullptr;
    a.out = rows;
    bm_score_kernel<<<dim3((unsigned)((n + BM_TILE - 1) / BM_TILE), qb), BM_THREADS, 0, st>>>(a);
    YB_CUDA(cudaGetLastError());
    return YAMS_OK;
}

// What a score call returns: the full score rows, and the best k (k <= 4096) of score > 0 of each query, best first
struct ScoreOut {
    float* scores;      // nullable: [nq][n]
    uint32_t k;
    uint32_t* docs;     // [nq][k], padded with 0xFFFFFFFF
    float* topk;        // [nq][k], padded with 0
    uint32_t* counts;   // [nq]
};

// The outputs of one batch: queries q0 .. q0 + qb, whose score rows are rows[qb][n] on x's stream -- the full vectors, and the
// best K (k <= 4096 asked) of score > 0 through x's selection workspace.  Returns with the rows free for the next batch.
static yams_status_t emit_batch(yams_b200_bm25* x, const float* rows, uint32_t q0, uint32_t qb, uint32_t nq, uint32_t K, const ScoreOut& o,
                                std::vector<Cand>& h_sel, std::vector<uint32_t>& h_n) {
    cudaStream_t st = x->st;
    const uint64_t n = x->n;
    if (o.scores) YB_CUDA(cudaMemcpyAsync(o.scores + (uint64_t)q0 * n, rows, (uint64_t)qb * n * 4, cudaMemcpyDeviceToHost, st));
    if (K) {
        launch_topk_dense(rows, n, qb, K, x->ws.sel.as<Cand>(), x->ws.seln.as<uint32_t>(), st);
        YB_CUDA(cudaGetLastError());
        h_sel.resize((uint64_t)qb * K);
        h_n.resize(qb);
        YB_CUDA(cudaMemcpyAsync(h_sel.data(), x->ws.sel.p, (uint64_t)qb * K * sizeof(Cand), cudaMemcpyDeviceToHost, st));
        YB_CUDA(cudaMemcpyAsync(h_n.data(), x->ws.seln.p, (uint64_t)qb * 4, cudaMemcpyDeviceToHost, st));
        YB_CUDA(cudaStreamSynchronize(st));
        // best first: the documents of score > 0 lead the selection
        for (uint32_t j = 0; j < qb; ++j) {
            uint32_t c = 0;
            const uint32_t m = std::min(h_n[j], K);
            while (c < m && h_sel[(uint64_t)j * K + c].score > 0.0f) {
                o.docs[(uint64_t)(q0 + j) * o.k + c] = h_sel[(uint64_t)j * K + c].row;
                o.topk[(uint64_t)(q0 + j) * o.k + c] = h_sel[(uint64_t)j * K + c].score;
                ++c;
            }
            o.counts[q0 + j] = c;
        }
    } else if (q0 + qb < nq) {
        YB_CUDA(cudaStreamSynchronize(st));   // the next batch overwrites the score rows
    }
    return YAMS_OK;
}

// the top-k outputs before any batch: padding, counts 0
static void clear_topk(uint32_t nq, const ScoreOut& o) {
    if (!o.k) return;
    for (uint64_t i = 0; i < (uint64_t)nq * o.k; ++i) { o.docs[i] = 0xFFFFFFFFu; o.topk[i] = 0.0f; }
    for (uint32_t q = 0; q < nq; ++q) o.counts[q] = 0;
}

// the next buffer carved from a row arena: the first 256-byte boundary at or after p
template <typename T>
static T* carve(const void* p) {
    return reinterpret_cast<T*>((reinterpret_cast<uintptr_t>(p) + 255) & ~uintptr_t(255));
}

// The batches of one score call on x's stream and workspace.  A query's rows take bytes_per_q, so a batch holds
// max(1, min(BM_DENSE_BYTES / bytes_per_q, nq, 4096)) queries, and the row arena one batch's rows with room to align three
// buffers carved from it.  The top-k is cleared first; an empty index scores nothing.  body(q0, qb, arena, &rows) computes
// queries q0 .. q0 + qb and sets the rows to emit; ksel is the widest top-k a body selects itself.  ms[6] gets the device time,
// ms[7] the wall time since t0.
template <typename Body>
static yams_status_t run_batches(yams_b200_bm25* x, double t0, uint32_t nq, uint64_t bytes_per_q, uint32_t ksel, const ScoreOut& o,
                                 Body&& body) {
    const uint64_t n = x->n;
    const uint32_t K = (uint32_t)std::min<uint64_t>(o.k, n);
    ksel = (uint32_t)std::min<uint64_t>(std::max(o.k, ksel), n);
    const uint64_t qb_max = n ? std::max<uint64_t>(1, std::min<uint64_t>({BM_DENSE_BYTES / bytes_per_q, (uint64_t)nq, 4096})) : 0;
    yams_status_t rc;
    if (n && (rc = x->ws.rows.reserve(qb_max * bytes_per_q + 3 * 256)) != YAMS_OK) return rc;
    if (ksel && ((rc = x->ws.sel.reserve(qb_max * ksel * sizeof(Cand))) != YAMS_OK || (rc = x->ws.seln.reserve(qb_max * 4)) != YAMS_OK))
        return rc;
    clear_topk(nq, o);
    float dev_ms = 0.f;
    if (n) {
        std::vector<Cand> h_sel;
        std::vector<uint32_t> h_n;
        rc = timed(x, &dev_ms, [&]() -> yams_status_t {
            for (uint32_t q0 = 0; q0 < nq; q0 += (uint32_t)qb_max) {
                const uint32_t qb = (uint32_t)std::min<uint64_t>(qb_max, nq - q0);
                const float* rows = nullptr;
                yams_status_t r;
                if ((r = body(q0, qb, x->ws.rows.p, &rows)) != YAMS_OK || (r = emit_batch(x, rows, q0, qb, nq, K, o, h_sel, h_n)) != YAMS_OK)
                    return r;
            }
            return YAMS_OK;
        });
        if (rc != YAMS_OK) return rc;
    }
    x->ms[6] = dev_ms;
    x->ms[7] = (float)(wall_ms() - t0);
    return YAMS_OK;
}

// The query router's part of a score call: rows scored as Atire, and the candidate pools projected from the rows
struct Routed {
    const uint8_t* atire;        // [nq]: 1 = the row scores as an Atire build of the same texts
    const uint64_t* cand_off;    // nullable: [nq + 1] pool offsets, cand_off[0] = 0
    const uint32_t* cand_docs;   // [cand_off[nq]]
    float* out_cand;             // [cand_off[nq]]
};

// Bm25Index::score of every query; with a concept index `c` of the same document count, then ConceptIndex::blend_into(query,
// scores, weight) of each (SimeonLexicalBackend::score).
// With strategy >= 0, the strategy's score_bm25f replaces Bm25Index::score (the strategy router's pools 0 and 2).  With rt, its
// Atire rows score as Atire and its pools are gathered from each batch's rows and copied back once.
static yams_status_t bm25_score(yams_b200_bm25* x, const yams_b200_concepts* c, float weight, const char* const* queries,
                                const size_t* qlens, uint32_t nq, const ScoreOut& o, int strategy = -1, const Routed* rt = nullptr) {
    const double t0 = wall_ms();
    cudaStream_t st = x->st;
    const uint64_t n = x->n;
    yams_status_t rc;
    // ---- host: the legs of every query, in the reference's order ----
    // the blend is a no-op when the concept index is empty or of another document count (blend_into's size test)
    const Scorer s{x, c && c->size && c->n == n ? c : nullptr, weight};
    LegList L;
    for (uint32_t q = 0; q < nq; ++q, L.end_query()) {
        const uint8_t* p = reinterpret_cast<const uint8_t*>(queries[q]);
        L.words(x, p, qlens[q], 0, rt && rt->atire[q]);
        if (strategy >= 0) L.bm25f(x, p, qlens[q], (uint32_t)strategy);
        if (s.c) L.concepts(s.c, p, qlens[q]);
    }
    const uint64_t npool = rt && rt->cand_off ? rt->cand_off[nq] : 0;
    if (npool && (rc = x->pool_off.reserve((nq + 1) * 8)) != YAMS_OK) return rc;
    if (npool && (rc = x->pool_docs.reserve(npool * 4)) != YAMS_OK) return rc;
    if (npool && (rc = x->pool_out.reserve(npool * 4)) != YAMS_OK) return rc;
    if (n == 0)
        for (uint64_t j = 0; j < npool; ++j) rt->out_cand[j] = 0.0f;   // no candidate is indexed
    return run_batches(x, t0, nq, n * 4, 0, o, [&](uint32_t q0, uint32_t qb, void* arena, const float** out) -> yams_status_t {
        float* rows = static_cast<float*>(arena);
        yams_status_t r;
        if (q0 == 0) {   // the call's pools and legs, staged once
            if (npool) {
                YB_CUDA(cudaMemcpyAsync(x->pool_off.p, rt->cand_off, (nq + 1) * 8, cudaMemcpyHostToDevice, st));
                YB_CUDA(cudaMemcpyAsync(x->pool_docs.p, rt->cand_docs, npool * 4, cudaMemcpyHostToDevice, st));
            }
            if ((r = stage_legs(x->ws, L, &s, 1, st)) != YAMS_OK) return r;
        }
        if ((r = score_rows(x->ws, L, s, n, q0, qb, false, rows, st)) != YAMS_OK) return r;
        if (npool && rt->cand_off[q0 + qb] > rt->cand_off[q0]) {
            uint64_t longest = 0;
            for (uint32_t j = q0; j < q0 + qb; ++j) longest = std::max(longest, rt->cand_off[j + 1] - rt->cand_off[j]);
            const unsigned gx = (unsigned)std::min<uint64_t>((longest + BM_THREADS - 1) / BM_THREADS, 64);
            bm_pool_gather_kernel<<<dim3(gx, qb), BM_THREADS, 0, st>>>(rows, n, q0, x->pool_off.as<uint64_t>(), x->pool_docs.as<uint32_t>(),
                                                                      x->pool_out.as<float>());
            YB_CUDA(cudaGetLastError());
        }
        if (npool && q0 + qb == nq) YB_CUDA(cudaMemcpyAsync(rt->out_cand, x->pool_out.p, npool * 4, cudaMemcpyDeviceToHost, st));
        *out = rows;
        return YAMS_OK;
    });
}

// ---- the keyphrase strategy and the entropy route (DESIGN.md §4.14) ----
// extract_keyphrases (retrieval_strategy.cpp:152-186): alphabetic runs (C locale) of >= 2 bytes, lowercased, stopwords dropped,
// sorted and de-duplicated; each hashed as Bm25Index::hash_term hashes it
static void keyphrase_hashes(const yams_b200_bm25* x, const uint8_t* p, size_t len, std::vector<uint64_t>& out) {
    static const std::unordered_set<std::string> stop = {
        "a", "an", "the", "and", "or", "but", "in", "on", "at", "to", "for", "of", "with", "by", "from", "is", "are", "was", "were",
        "be", "been", "being", "have", "has", "had", "do", "does", "did", "will", "would", "could", "should", "may", "might", "can",
        "shall", "this", "that", "these", "those", "it", "its", "they", "them", "we", "us", "he", "she", "his", "her", "their", "our",
        "my", "your", "not", "no", "nor", "so", "as", "if", "than", "then", "also", "very", "just", "about", "into", "over", "after",
        "before", "between", "under", "during", "without"};
    auto alpha = [](uint8_t c) { return (c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z'); };
    std::vector<std::string> kps;
    for (size_t i = 0; i < len;) {
        while (i < len && !alpha(p[i])) ++i;
        const size_t st = i;
        while (i < len && alpha(p[i])) ++i;
        if (i - st < 2) continue;
        std::string w(reinterpret_cast<const char*>(p + st), i - st);
        for (char& ch : w) ch = (char)ascii_lower((uint8_t)ch);
        if (!stop.count(w)) kps.push_back(std::move(w));
    }
    std::sort(kps.begin(), kps.end());
    kps.erase(std::unique(kps.begin(), kps.end()), kps.end());
    const uint64_t h0 = gram_hash_h0(x->cfg.hash_seed);
    out.clear();
    for (const auto& w : kps) out.push_back(gram_hash(reinterpret_cast<const uint8_t*>(w.data()), w.size(), h0));
}

// The route of one row: the backend's bm25_entropy < 0.05f -> pool 0, > 0.50f -> pool 2, else pool 1.  The device's profile
// (bm_route_kernel) differs from the reference's by the order of the sum and device against glibc log: every term
// sn * -log(sn) >= 0 is within 8u of the reference's (each log within 1 ulp, one rounding of the product on each side), and
// each order's rounding is within (count)u of the exact sum, so |S_dev - S_ref| <= S_dev (8u + 2 count u)(1 + 1%) (u = 2^-53).
// When every value in that interval, divided by count, rounds to a float on one side of both thresholds, the route is certain;
// otherwise the row is copied back and the backend's loop replayed with std::log.  `margin` widens the entropy's interval.
static int route_pool(const double* prof, const float* row_dev, uint64_t n, double margin, cudaStream_t st, bool* replayed) {
    *replayed = false;
    const double m = prof[0], cnt = prof[1], sum = prof[2];
    if (!(m > 0.0) || cnt == 0.0) return 0;   // bm25_entropy = 0
    const double u = 0x1p-53;
    const double E = sum * (8.0 * u + 2.0 * cnt * u) * 1.01;
    const double lo = (sum - E) / cnt * (1.0 - 4.0 * u) - margin, hi = (sum + E) / cnt * (1.0 + 4.0 * u) + margin;
    const double t0 = 0.05f, t1 = 0.50f;
    if (hi < (double)std::nextafter(0.05f, 0.0f)) return 0;
    if (lo >= t0 && hi <= t1) return 1;
    if (lo >= (double)std::nextafter(0.50f, 1.0f)) return 2;
    *replayed = true;
    std::vector<float> tmp(n);
    if (cudaMemcpyAsync(tmp.data(), row_dev, n * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
        return -1;
    const float top = *std::max_element(tmp.begin(), tmp.end());
    float e = 0.0f;
    if (top > 0.0f) {
        double acc = 0.0, positives = 0.0;
        for (float v : tmp) {
            if (v <= 0.0f) continue;
            const double sn = v / top;
            if (sn > 0.0) acc += sn * (-std::log(sn));
            positives += 1.0;
        }
        e = positives > 0.0 ? (float)(acc / positives) : 0.0f;
    }
    return e < 0.05f ? 0 : e > 0.50f ? 2 : 1;
}

// The strategy router's KEYPHRASE pool or its ROUTED choice for every query, then ConceptIndex::blend_into.  Per batch: the
// plain score rows; with ROUTED, each row's profile and pool; the BM25F legs of rows routed to pools 0 and 2 onto their rows; for
// rows of pool 1 the top-10 (padded with zero scores as simeon::top_k keeps them), the gate, the matches of each gated row's
// keyphrases and the z-score; the concept legs; the outputs.
static yams_status_t bm25_score_staged(yams_b200_bm25* x, const yams_b200_concepts* c, float weight, uint32_t strategy,
                                       const char* const* queries, const size_t* qlens, uint32_t nq, const ScoreOut& o,
                                       uint32_t* out_chosen) {
    const double t0 = wall_ms();
    cudaStream_t st = x->st;
    const uint64_t n = x->n;
    const Scorer plain{x, nullptr, 0.0f}, blend{x, c && c->size && c->n == n ? c : nullptr, weight};
    const uint32_t K10 = (uint32_t)std::min<uint64_t>(10, n);
    double margin = 0.0;   // YAMS_B200_BM25_ROUTE_MARGIN = w > 0 widens the certified interval by w, read at every call
    if (const char* e = getenv("YAMS_B200_BM25_ROUTE_MARGIN")) margin = std::max(0.0, strtod(e, nullptr));
    if (n == 0 && out_chosen) std::fill(out_chosen, out_chosen + nq, strategy == YAMS_BM25_STRATEGY_ROUTED ? 0u : strategy);
    // A batch's plain, BM25F, presence and concept legs: each list outlives its copy, and the next batch starts after emit_batch
    // has synchronised, so the sub-passes need no synchronisation of their own.
    LegList plain_legs, f_legs, kp_legs, concept_legs;
    std::vector<uint64_t> kh;
    std::vector<double> prof;
    std::vector<uint32_t> pool, zrow;
    std::vector<float> zp;
    std::vector<Cand> h_sel;
    std::vector<uint32_t> h_n;
    // per query: its score row and its row of keyphrase matches
    return run_batches(x, t0, nq, n * 8, 10, o, [&](uint32_t q0, uint32_t qb, void* arena, const float** out) -> yams_status_t {
        float* rows = static_cast<float*>(arena);
        float* counts = carve<float>(rows + (uint64_t)qb * n);
        auto qp = [&](uint32_t j) { return reinterpret_cast<const uint8_t*>(queries[q0 + j]); };
        yams_status_t r;
        if ((r = x->route.reserve((uint64_t)qb * 24)) != YAMS_OK || (r = x->zrow.reserve((uint64_t)qb * 4)) != YAMS_OK ||
            (r = x->zp.reserve((uint64_t)qb * 8)) != YAMS_OK)
            return r;
        // the plain scores
        plain_legs.clear();
        for (uint32_t j = 0; j < qb; ++j, plain_legs.end_query()) plain_legs.words(x, qp(j), qlens[q0 + j], 0);
        if ((r = stage_legs(x->ws, plain_legs, &plain, 1, st)) != YAMS_OK ||
            (r = score_rows(x->ws, plain_legs, plain, n, 0, qb, false, rows, st)) != YAMS_OK)
            return r;
        // the pools
        pool.assign(qb, strategy);
        if (strategy == YAMS_BM25_STRATEGY_ROUTED) {
            prof.resize((uint64_t)qb * 3);
            bm_route_kernel<<<qb, BM_THREADS, 0, st>>>(rows, n, x->route.as<double>());
            YB_CUDA(cudaGetLastError());
            YB_CUDA(cudaMemcpyAsync(prof.data(), x->route.p, (uint64_t)qb * 24, cudaMemcpyDeviceToHost, st));
            YB_CUDA(cudaStreamSynchronize(st));
            for (uint32_t j = 0; j < qb; ++j) {
                bool rep = false;
                const int p = route_pool(prof.data() + 3 * j, rows + (uint64_t)j * n, n, margin, st, &rep);
                if (p < 0) { set_last_error("route replay copy failed"); return YAMS_ERR_INTERNAL; }
                pool[j] = (uint32_t)p;
                x->sstats.replayed += rep;
            }
        }
        // pools 0 and 2: score_bm25f's body scale and aux legs onto the plain rows
        f_legs.clear();
        bool kp = false;
        for (uint32_t j = 0; j < qb; ++j, f_legs.end_query()) {
            ++x->sstats.queries[pool[j]];
            if (pool[j] == YAMS_BM25_STRATEGY_KEYPHRASE) kp = true;
            else f_legs.bm25f(x, qp(j), qlens[q0 + j], pool[j]);
        }
        if ((r = stage_legs(x->ws, f_legs, &plain, 1, st)) != YAMS_OK || (r = score_rows(x->ws, f_legs, plain, n, 0, qb, true, rows, st)) != YAMS_OK)
            return r;
        // pool 1: the entropy gate over the top-10 with its zeros, the matches, the z-score
        if (kp) {
            launch_topk_dense(rows, n, qb, K10, x->ws.sel.as<Cand>(), x->ws.seln.as<uint32_t>(), st);
            YB_CUDA(cudaGetLastError());
            h_sel.resize((uint64_t)qb * K10);
            h_n.resize(qb);
            YB_CUDA(cudaMemcpyAsync(h_sel.data(), x->ws.sel.p, (uint64_t)qb * K10 * sizeof(Cand), cudaMemcpyDeviceToHost, st));
            YB_CUDA(cudaMemcpyAsync(h_n.data(), x->ws.seln.p, (uint64_t)qb * 4, cudaMemcpyDeviceToHost, st));
            YB_CUDA(cudaStreamSynchronize(st));
            kp_legs.clear();
            zrow.clear();
            zp.clear();
            for (uint32_t j = 0; j < qb; ++j, kp_legs.end_query()) {
                if (pool[j] != 1) continue;
                // simeon::top_k(scores, 10): the positives best first, then zeros (every other score is 0)
                double vals[10];
                uint32_t m = 0;
                for (; m < std::min(h_n[j], K10) && h_sel[(uint64_t)j * K10 + m].score > 0.0f; ++m)
                    vals[m] = (double)h_sel[(uint64_t)j * K10 + m].score;
                for (; m < K10; ++m) vals[m] = 0.0;
                double ent = 0.0;
                if (K10 >= 2) {
                    double sum_exp = 0.0;
                    for (uint32_t i = 0; i < K10; ++i) sum_exp += std::exp(vals[i]);
                    for (uint32_t i = 0; i < K10; ++i) {
                        const double pr = std::exp(vals[i]) / sum_exp;
                        if (pr > 1e-12) ent -= pr * std::log(pr);
                    }
                    ent /= std::log((double)K10);
                }
                const float entropy = (float)ent;
                if (entropy < 0.30f) continue;
                keyphrase_hashes(x, qp(j), qlens[q0 + j], kh);
                if (kh.empty()) continue;
                kp_legs.presence(kh);
                const float lam = 1.0f / (1.0f + std::exp(-(entropy - 0.48f) * 8.0f));
                zrow.push_back(j);
                zp.push_back(lam * 0.25f);
                zp.push_back((float)kh.size());
            }
            if (!zrow.empty()) {
                x->sstats.keyphrase_boosted += (uint32_t)zrow.size();
                if ((r = stage_legs(x->ws, kp_legs, &plain, 1, st)) != YAMS_OK ||
                    (r = score_rows(x->ws, kp_legs, plain, n, 0, qb, false, counts, st)) != YAMS_OK)
                    return r;
                YB_CUDA(cudaMemcpyAsync(x->zrow.p, zrow.data(), zrow.size() * 4, cudaMemcpyHostToDevice, st));
                YB_CUDA(cudaMemcpyAsync(x->zp.p, zp.data(), zp.size() * 4, cudaMemcpyHostToDevice, st));
                YB_CUDA(cudaEventRecord(x->zev[0], st));
                bm_zscore_kernel<<<(unsigned)zrow.size(), BM_THREADS, 0, st>>>(rows, counts, n, x->zrow.as<uint32_t>(), x->zp.as<float>());
                YB_CUDA(cudaGetLastError());
                YB_CUDA(cudaEventRecord(x->zev[1], st));
                YB_CUDA(cudaEventSynchronize(x->zev[1]));
                float zms = 0.f;
                YB_CUDA(cudaEventElapsedTime(&zms, x->zev[0], x->zev[1]));
                x->sstats.zscore_ms += zms;
            }
        }
        // the concept blend onto the strategies' rows
        if (blend.c) {
            concept_legs.clear();
            for (uint32_t j = 0; j < qb; ++j, concept_legs.end_query()) concept_legs.concepts(blend.c, qp(j), qlens[q0 + j]);
            if ((r = stage_legs(x->ws, concept_legs, &blend, 1, st)) != YAMS_OK ||
                (r = score_rows(x->ws, concept_legs, blend, n, 0, qb, true, rows, st)) != YAMS_OK)
                return r;
        }
        if (out_chosen) std::copy(pool.begin(), pool.end(), out_chosen + q0);
        *out = rows;
        return YAMS_OK;
    });
}

// The strategy router's score call and its stats.  Pools 0 and 2 score every query in one pass: the body, the scale, the aux
// legs and the concepts.  KEYPHRASE and ROUTED are staged per batch and count the pool of each row they score, so an empty
// index counts none of their queries and reports no time.
static yams_status_t bm25_score_strategy(yams_b200_bm25* x, uint32_t strategy, const yams_b200_concepts* c, float weight,
                                         const char* const* queries, const size_t* qlens, uint32_t nq, const ScoreOut& o,
                                         uint32_t* out_chosen) {
    yams_status_t rc;
    x->sstats = yams_bm25_strategy_stats{};
    if (strategy == YAMS_BM25_STRATEGY_KEYPHRASE || strategy == YAMS_BM25_STRATEGY_ROUTED) {
        if ((rc = bm25_score_staged(x, c, weight, strategy, queries, qlens, nq, o, out_chosen)) != YAMS_OK || x->n == 0) return rc;
    } else {
        if ((rc = bm25_score(x, c, weight, queries, qlens, nq, o, (int)strategy)) != YAMS_OK) return rc;
        if (out_chosen) std::fill(out_chosen, out_chosen + nq, strategy);
        x->sstats.queries[strategy] = nq;
    }
    x->sstats.device_ms = x->ms[6];
    x->sstats.wall_ms = x->ms[7];
    return YAMS_OK;
}

// ---- reciprocal-rank fusion of BM25 variants (score_bm25_variants_rrf, fusion.cpp:24-63) ----
// A ranked entry: the key (~score_bits << 32) | document sorts ascending as the reference's ranking (score descending, then
// document ascending, fusion.cpp:14-20); only positive finite scores are ranked, whose bits order as their values.
__device__ __forceinline__ bool rrf_ranked(float s) { return __float_as_uint(s) - 1u < 0x7F7FFFFFu; }

// ranked entries of each (row, tile of BM_TILE documents); block b = row * tiles + tile
__global__ void __launch_bounds__(BM_THREADS) rrf_count_kernel(const float* __restrict__ rows, uint64_t n, uint32_t tiles,
                                                               uint32_t* __restrict__ cnt) {
    const uint64_t row = blockIdx.x / tiles, lo = (uint64_t)(blockIdx.x % tiles) * BM_TILE;
    const uint32_t len = (uint32_t)min((uint64_t)BM_TILE, n - lo);
    const float* s = rows + row * n + lo;
    uint32_t c = 0;
    for (uint32_t i0 = 0; i0 < len; i0 += BM_THREADS)
        c += __syncthreads_count(i0 + threadIdx.x < len && rrf_ranked(s[i0 + threadIdx.x]));
    if (threadIdx.x == 0) cnt[blockIdx.x] = c;
}

// the ranked entries' keys, each (row, tile) at its exclusive-scan base, in document order
__global__ void __launch_bounds__(BM_THREADS) rrf_keys_kernel(const float* __restrict__ rows, uint64_t n, uint32_t tiles,
                                                              const uint32_t* __restrict__ base, uint64_t* __restrict__ keys) {
    using Scan = cub::BlockScan<uint32_t, BM_THREADS>;
    __shared__ typename Scan::TempStorage ts;
    const uint64_t row = blockIdx.x / tiles, lo = (uint64_t)(blockIdx.x % tiles) * BM_TILE;
    const uint32_t len = (uint32_t)min((uint64_t)BM_TILE, n - lo);
    const float* s = rows + row * n + lo;
    uint32_t at = base[blockIdx.x];
    for (uint32_t i0 = 0; i0 < len; i0 += BM_THREADS) {
        const uint32_t i = i0 + threadIdx.x;
        const float v = i < len ? s[i] : 0.0f;
        const uint32_t f = rrf_ranked(v) ? 1u : 0u;
        uint32_t pre, total;
        Scan(ts).ExclusiveSum(f, pre, total);
        if (f) keys[at + pre] = ((uint64_t)~__float_as_uint(v) << 32) | (uint32_t)(lo + i);
        at += total;
        __syncthreads();   // ts is reused
    }
}

// segment r (a (variant, query) row) of the sorted keys: [base[r * tiles], base[(r + 1) * tiles])
struct RowStart {
    const uint32_t* base;
    uint32_t tiles;
    __host__ __device__ uint32_t operator()(uint64_t r) const { return base[r * tiles]; }
};

// one variant's contributions, in rank order r = 1, 2, ...: fused[q][doc] += 1.0f / (k + float(r)) (fusion.cpp:31-33), each
// operation rounded once.  A document appears once per segment and one launch serves one variant, so the additions of a
// document follow the variant order with no atomics.
__global__ void rrf_scatter_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ base, uint32_t tiles, uint64_t row0,
                                   float k_rrf, uint64_t n, float* __restrict__ fused) {
    const uint64_t r = row0 + blockIdx.y;
    const uint32_t b = base[r * tiles], e = base[(r + 1) * tiles];
    float* out = fused + (uint64_t)blockIdx.y * n;
    for (uint32_t i = b + blockIdx.x * blockDim.x + threadIdx.x; i < e; i += gridDim.x * blockDim.x) {
        const uint32_t d = (uint32_t)keys[i];
        out[d] = __fadd_rn(out[d], __fdiv_rn(1.0f, __fadd_rn(k_rrf, __ull2float_rn((uint64_t)(i - b) + 1))));
    }
}

// score_bm25_variants_rrf(v[0..nv), query, out, k_rrf) of every query, then, with a concept index c of the same document count,
// ConceptIndex::blend_into(query, out, weight) (SimeonLexicalBackend::score with bm25_variants_rrf), on v[0]'s stream and
// workspace.  Per batch of queries: every variant's score rows, their ranked keys, one segmented sort of the (variant, query)
// segments, one scatter per variant in order onto zeroed fused rows, the blend's concept legs, the outputs.
static yams_status_t bm25_score_rrf(const yams_b200_bm25* const* v, uint32_t nv, float k_rrf, const yams_b200_concepts* c, float weight,
                                    const char* const* queries, const size_t* qlens, uint32_t nq, const ScoreOut& o) {
    const double t0 = wall_ms();
    yams_b200_bm25* x = const_cast<yams_b200_bm25*>(v[0]);
    cudaStream_t st = x->st;
    const uint64_t n = x->n;
    // ---- host: each variant's legs of every query, then the concepts' ----
    std::vector<Scorer> s;
    for (uint32_t j = 0; j < nv; ++j) s.push_back({v[j], nullptr, 0.0f});
    if (c && c->size && c->n == n) s.push_back({nullptr, c, weight});
    LegList L;
    for (const Scorer& b : s)
        for (uint32_t q = 0; q < nq; ++q, L.end_query()) {
            const uint8_t* p = reinterpret_cast<const uint8_t*>(queries[q]);
            if (b.x) L.words(b.x, p, qlens[q], 0);
            else L.concepts(b.c, p, qlens[q]);
        }
    const uint64_t tiles = (n + BM_TILE - 1) / BM_TILE;
    // per query: nv score rows (4 bytes a document), at most n keys per row twice (the sort's double buffer), one fused row
    return run_batches(x, t0, nq, n * (20ull * nv + 4), 0, o, [&](uint32_t q0, uint32_t qb, void* arena, const float** out) -> yams_status_t {
        yams_status_t r;
        const uint64_t rows = (uint64_t)nv * qb, blocks = rows * tiles;
        if (q0 == 0 && (r = stage_legs(x->ws, L, s.data(), (uint32_t)s.size(), st)) != YAMS_OK) return r;   // the call's legs, once
        if ((r = x->cnt.reserve((blocks + 1) * 4)) != YAMS_OK || (r = x->base.reserve((blocks + 1) * 4)) != YAMS_OK) return r;
        float* dense = static_cast<float*>(arena);
        uint64_t* keys = carve<uint64_t>(dense + rows * n);
        uint64_t* keys2 = carve<uint64_t>(keys + rows * n);
        float* fused = carve<float>(keys2 + rows * n);
        // every variant's rows: variant j's queries at rows j * qb ..
        for (uint32_t j = 0; j < nv; ++j)
            if ((r = score_rows(x->ws, L, s[j], n, (uint64_t)j * nq + q0, qb, false, dense + (uint64_t)j * qb * n, st)) != YAMS_OK) return r;
        // the ranked keys of each row, the rows' segments, one segmented sort
        rrf_count_kernel<<<(unsigned)blocks, BM_THREADS, 0, st>>>(dense, n, (uint32_t)tiles, x->cnt.as<uint32_t>());
        YB_CUDA(cudaGetLastError());
        YB_CUDA(cudaMemsetAsync(x->cnt.as<uint32_t>() + blocks, 0, 4, st));
        x->tmp.bytes = 0;
        YB_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, x->tmp.bytes, x->cnt.as<uint32_t>(), x->base.as<uint32_t>(), (int64_t)blocks + 1, st));
        if ((r = x->tmp.grow()) != YAMS_OK) return r;
        YB_CUDA(cub::DeviceScan::ExclusiveSum(x->tmp.buf.p, x->tmp.bytes, x->cnt.as<uint32_t>(), x->base.as<uint32_t>(), (int64_t)blocks + 1, st));
        uint32_t items = 0;
        YB_CUDA(cudaMemcpyAsync(&items, x->base.as<uint32_t>() + blocks, 4, cudaMemcpyDeviceToHost, st));
        rrf_keys_kernel<<<(unsigned)blocks, BM_THREADS, 0, st>>>(dense, n, (uint32_t)tiles, x->base.as<uint32_t>(), keys);
        YB_CUDA(cudaGetLastError());
        YB_CUDA(cudaStreamSynchronize(st));   // items
        const uint64_t* sorted = keys;
        if (items) {
            cub::DoubleBuffer<uint64_t> db(keys, keys2);
            const auto begins = thrust::make_transform_iterator(thrust::counting_iterator<uint64_t>(0), RowStart{x->base.as<uint32_t>(), (uint32_t)tiles});
            x->tmp.bytes = 0;
            YB_CUDA(cub::DeviceSegmentedSort::SortKeys(nullptr, x->tmp.bytes, db, (int64_t)items, (int64_t)rows, begins, begins + 1, st));
            if ((r = x->tmp.grow()) != YAMS_OK) return r;
            YB_CUDA(cub::DeviceSegmentedSort::SortKeys(x->tmp.buf.p, x->tmp.bytes, db, (int64_t)items, (int64_t)rows, begins, begins + 1, st));
            sorted = db.Current();
        }
        // the fusion: zeros, then each variant's ranks in order
        YB_CUDA(cudaMemsetAsync(fused, 0, (uint64_t)qb * n * 4, st));
        const unsigned gx = (unsigned)std::min<uint64_t>((n + 4 * BM_THREADS - 1) / (4 * BM_THREADS), 64);
        for (uint32_t j = 0; items && j < nv; ++j) {
            rrf_scatter_kernel<<<dim3(gx, qb), BM_THREADS, 0, st>>>(sorted, x->base.as<uint32_t>(), (uint32_t)tiles, (uint64_t)j * qb, k_rrf, n,
                                                                    fused);
            YB_CUDA(cudaGetLastError());
        }
        // the blend adds onto the fused rows in place
        if (s.size() > nv && (r = score_rows(x->ws, L, s[nv], n, (uint64_t)nv * nq + q0, qb, true, fused, st)) != YAMS_OK) return r;
        *out = fused;
        return YAMS_OK;
    });
}

// ---- concept mining (mine_concepts, concept_mining.cpp:117-258) ----
// words per document (integer atomics: exact)
__global__ void cm_doc_words_kernel(const uint32_t* __restrict__ wdoc, uint64_t nw, uint32_t* __restrict__ cnt) {
    for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < nw; w += (uint64_t)gridDim.x * blockDim.x)
        atomicAdd(&cnt[wdoc[w]], 1u);
}

// word w starts a bigram: the next word is of the same document
struct StartsBigram {
    const uint32_t* wdoc;
    uint64_t nw;
    __device__ bool operator()(uint64_t w) const { return w + 1 < nw && wdoc[w + 1] == wdoc[w]; }
};

// pair j (first word pw[j]): its bigram hash, and j itself, which is its corpus position
__global__ void cm_pairs_kernel(const uint64_t* __restrict__ pw, uint64_t np, const uint64_t* __restrict__ whash,
                                uint64_t* __restrict__ key, uint32_t* __restrict__ val) {
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < np; j += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t w = pw[j];
        key[j] = hash_bigram(whash[w], whash[w + 1]);
        val[j] = (uint32_t)j;
    }
}

// the document of every sorted pair
__global__ void cm_pair_docs_kernel(const uint32_t* __restrict__ pj, uint64_t np, const uint64_t* __restrict__ pw,
                                    const uint32_t* __restrict__ wdoc, uint32_t* __restrict__ pdoc) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < np; i += (uint64_t)gridDim.x * blockDim.x)
        pdoc[i] = wdoc[pw[pj[i]]];
}

enum : uint8_t { CM_UNDER_TTF = 0, CM_NO_WORD = 1, CM_CANDIDATE = 2 };

// one distinct bigram (its pairs start at pstart[b] of the sorted pairs, a run of total_tf): the first occurrence (the run's
// first pair) gives (a, b); under min_ttf or with a word the index lacks it is dropped, else the PMI ratio
// p_ab / (p_a * p_b) is formed in double, each operation rounded once as the reference's (concept_mining.cpp:211-220)
__global__ void cm_bigrams_kernel(const uint64_t* __restrict__ pstart, uint64_t nb, uint64_t np, const uint32_t* __restrict__ pj,
                                  const uint64_t* __restrict__ pw, const uint64_t* __restrict__ whash, Dict words,
                                  const uint64_t* __restrict__ wttf, uint32_t min_ttf, double sum_bdl, double total_tokens,
                                  uint32_t* __restrict__ first, uint64_t* __restrict__ ab, uint8_t* __restrict__ status,
                                  double* __restrict__ ratio) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nb; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t s = pstart[i], e = i + 1 < nb ? pstart[i + 1] : np, ttf = e - s;
        const uint32_t j = pj[s];
        const uint64_t a = whash[pw[j]], b = whash[pw[j] + 1];
        first[i] = j;
        ab[2 * i] = a;
        ab[2 * i + 1] = b;
        ratio[i] = 0.0;
        if (ttf < min_ttf) { status[i] = CM_UNDER_TTF; continue; }
        uint64_t lo = 0, hi = 0, t = 0;
        const uint64_t tf_a = dict_find(words, a, &lo, &hi, &t) ? wttf[t] : 0;
        const uint64_t tf_b = dict_find(words, b, &lo, &hi, &t) ? wttf[t] : 0;
        if (tf_a == 0 || tf_b == 0) { status[i] = CM_NO_WORD; continue; }
        status[i] = CM_CANDIDATE;
        const double p_ab = __ddiv_rn((double)ttf, sum_bdl);
        const double p_a = __ddiv_rn((double)tf_a, total_tokens), p_b = __ddiv_rn((double)tf_b, total_tokens);
        ratio[i] = __ddiv_rn(p_ab, __dmul_rn(p_a, p_b));
    }
}

struct IsCandidate {
    const uint8_t* status;
    __device__ bool operator()(uint64_t i) const { return status[i] == CM_CANDIDATE; }
};
struct PassedTtf {
    const uint8_t* status;
    __device__ bool operator()(uint64_t i) const { return status[i] != CM_UNDER_TTF; }
};

__global__ void cm_candidates_kernel(const uint64_t* __restrict__ cand, uint64_t nc, const uint64_t* __restrict__ bhash,
                                     const double* __restrict__ ratio, uint64_t* __restrict__ ch, double* __restrict__ cr) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nc; i += (uint64_t)gridDim.x * blockDim.x) {
        ch[i] = bhash[cand[i]];
        cr[i] = ratio[cand[i]];
    }
}

// kept concept j (distinct bigram kb[j]): hash, total_tf, a, b, df
__global__ void cm_kept_kernel(const uint64_t* __restrict__ kb, uint64_t nk, const uint64_t* __restrict__ bhash,
                               const uint64_t* __restrict__ boffs, const uint64_t* __restrict__ bttf, const uint64_t* __restrict__ ab,
                               uint64_t* __restrict__ out) {
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < nk; j += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t b = kb[j];
        out[5 * j] = bhash[b];
        out[5 * j + 1] = bttf[b];
        out[5 * j + 2] = ab[2 * b];
        out[5 * j + 3] = ab[2 * b + 1];
        out[5 * j + 4] = boffs[b + 1] - boffs[b];
    }
}

// posting i of the kept concepts (koffs: their offsets) from the packed postings (document << 32 | tf) of every bigram
__global__ void cm_gather_kernel(const uint64_t* __restrict__ kb, const uint64_t* __restrict__ koffs, uint64_t nk, uint64_t total,
                                 const uint64_t* __restrict__ boffs, const uint64_t* __restrict__ pv, uint32_t* __restrict__ docs,
                                 uint32_t* __restrict__ tfs) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t j = last_le(koffs, nk, i);
        const uint64_t v = pv[boffs[kb[j]] + (i - koffs[j])];
        docs[i] = (uint32_t)(v >> 32);
        tfs[i] = (uint32_t)v;
    }
}

template <typename K, typename V>
static yams_status_t radix_sort(CubTmp& tmp, DevBuf& k, DevBuf& v, DevBuf& k2, DevBuf& v2, uint64_t m, cudaStream_t st) {
    yams_status_t rc;
    if ((rc = k2.reserve(std::max<uint64_t>(m, 1) * sizeof(K))) != YAMS_OK || (rc = v2.reserve(std::max<uint64_t>(m, 1) * sizeof(V))) != YAMS_OK)
        return rc;
    tmp.bytes = 0;
    YB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp.bytes, k.as<K>(), k2.as<K>(), v.as<V>(), v2.as<V>(), (int64_t)m, 0, 8 * (int)sizeof(K), st));
    if ((rc = tmp.grow()) != YAMS_OK) return rc;
    YB_CUDA(cub::DeviceRadixSort::SortPairs(tmp.buf.p, tmp.bytes, k.as<K>(), k2.as<K>(), v.as<V>(), v2.as<V>(), (int64_t)m, 0, 8 * (int)sizeof(K),
                                            st));
    std::swap(k, k2);
    std::swap(v, v2);
    return YAMS_OK;
}

// The cap (concept_mining.cpp:228-234) when a PMI tie crosses it.  The reference collects its accepted bigrams in the iteration
// order of unordered_map<uint64_t, RawEntry> raw, whose keys were inserted in first-occurrence order (the map's order depends
// on that sequence of keys alone), then keeps the first max_concepts after std::nth_element by PMI descending.  `order` is
// every distinct bigram hash by first occurrence; `acc` maps an accepted hash to its (PMI, distinct-bigram index).
static void replay_cap(const std::vector<uint64_t>& order, const std::unordered_map<uint64_t, std::pair<float, uint64_t>>& acc,
                       uint32_t max_concepts, std::vector<std::pair<uint64_t, float>>& kept) {
    std::unordered_map<uint64_t, char> raw;
    for (uint64_t h : order) raw[h];
    std::vector<std::pair<uint64_t, float>> accepted;   // (hash, PMI), as the reference's vector
    accepted.reserve(acc.size());
    for (const auto& [h, unused] : raw) {
        (void)unused;
        const auto it = acc.find(h);
        if (it != acc.end()) accepted.emplace_back(h, it->second.first);
    }
    std::nth_element(accepted.begin(), accepted.begin() + static_cast<std::ptrdiff_t>(max_concepts), accepted.end(),
                     [](const auto& x, const auto& y) { return x.second > y.second; });
    accepted.resize(max_concepts);
    kept.clear();
    for (const auto& [h, pmi] : accepted) kept.emplace_back(acc.at(h).second, pmi);
}

static yams_status_t concepts_mine(yams_b200_concepts* c, yams_b200_bm25* x, const char* const* texts, const size_t* lens) {
    const double t0 = wall_ms();
    cudaStream_t st = c->st;
    const uint64_t n = c->n;
    yams_status_t rc;
    c->h_bdl.assign(n, 0);
    if ((rc = c->bdl.reserve(std::max<uint64_t>(n, 1) * 4)) != YAMS_OK || (rc = c->offs.reserve(8)) != YAMS_OK) return rc;
    YB_CUDA(cudaMemsetAsync(c->bdl.p, 0, std::max<uint64_t>(n, 1) * 4, st));
    YB_CUDA(cudaMemsetAsync(c->offs.p, 0, 8, st));
    std::vector<uint64_t> pos;
    DevBuf text, d_pos;
    rc = timed(c, &c->ms[0], [&] { return upload_texts(texts, lens, n, pos, text, d_pos, st); });
    if (rc != YAMS_OK) return rc;
    const uint64_t L = pos[n];
    // ---- words (unfolded hashes), words per document, pairs of adjacent words of one document ----
    CubTmp tmp;
    DevBuf wstart, cnt, whash, wdoc, dcount, pw, key, val, k2, v2;
    uint64_t nw = 0, np = 0;
    rc = timed(c, &c->ms[1], [&]() -> yams_status_t {
        yams_status_t r;
        if ((r = select_indices(tmp, 0, L, IsWordStart{text.as<uint8_t>()}, wstart, cnt, &nw, st)) != YAMS_OK) return r;
        if ((r = whash.reserve(std::max<uint64_t>(nw, 1) * 8)) != YAMS_OK || (r = wdoc.reserve(std::max<uint64_t>(nw, 1) * 4)) != YAMS_OK ||
            (r = dcount.reserve(std::max<uint64_t>(n, 1) * 4)) != YAMS_OK)
            return r;
        YB_CUDA(cudaMemsetAsync(dcount.p, 0, std::max<uint64_t>(n, 1) * 4, st));
        if (nw) {
            bm_words_kernel<false><<<bm_grid(nw), BM_THREADS, 0, st>>>(text.as<uint8_t>(), wstart.as<uint64_t>(), nw, d_pos.as<uint64_t>(), n,
                                                                       c->h0, 0, 0, whash.as<uint64_t>(), wdoc.as<uint32_t>(), nullptr, nullptr);
            cm_doc_words_kernel<<<bm_grid(nw), BM_THREADS, 0, st>>>(wdoc.as<uint32_t>(), nw, dcount.as<uint32_t>());
        }
        YB_CUDA(cudaGetLastError());
        if (n) YB_CUDA(cudaMemcpyAsync(c->h_bdl.data(), dcount.p, n * 4, cudaMemcpyDeviceToHost, st));
        if (nw && (r = select_indices(tmp, 0, nw, StartsBigram{wdoc.as<uint32_t>(), nw}, pw, cnt, &np, st)) != YAMS_OK) return r;
        if (np >= 0xFFFFFFFFull) {
            set_last_error("concept mining: %llu word pairs, at most 2^32 - 2 are served", (unsigned long long)np);
            return YAMS_ERR_INVALID_ARG;
        }
        if ((r = key.reserve(std::max<uint64_t>(np, 1) * 8)) != YAMS_OK || (r = val.reserve(std::max<uint64_t>(np, 1) * 4)) != YAMS_OK) return r;
        if (np) cm_pairs_kernel<<<bm_grid(np), BM_THREADS, 0, st>>>(pw.as<uint64_t>(), np, whash.as<uint64_t>(), key.as<uint64_t>(), val.as<uint32_t>());
        YB_CUDA(cudaGetLastError());
        return YAMS_OK;
    });
    if (rc != YAMS_OK) return rc;
    text = DevBuf();
    wstart = DevBuf();
    dcount = DevBuf();
    // bigram_dl = words - 1 for documents of >= 2 words (concept_mining.cpp:154-159)
    for (uint64_t d = 0; d < n; ++d) {
        c->h_bdl[d] = c->h_bdl[d] >= 2 ? c->h_bdl[d] - 1 : 0;
        c->sum_bdl += c->h_bdl[d];
    }
    c->avg = n == 0 ? 0.0f : (float)((double)c->sum_bdl / (double)n);
    if (n) YB_CUDA(cudaMemcpyAsync(c->bdl.p, c->h_bdl.data(), n * 4, cudaMemcpyHostToDevice, st));
    // ---- stable sort by bigram hash: each hash's pairs in corpus order ----
    rc = timed(c, &c->ms[2], [&] { return np ? radix_sort<uint64_t, uint32_t>(tmp, key, val, k2, v2, np, st) : YAMS_OK; });
    if (rc != YAMS_OK) return rc;
    k2 = DevBuf();
    v2 = DevBuf();
    // ---- runs: (hash, document) -> postings; hash -> distinct bigrams (total_tf, first occurrence); the filter ----
    DevBuf ph, pv, bhash, boffs, bttf, pstart, first, ab, status, ratio, cand, ch, cr;
    uint64_t nposts = 0, nb = 0, nc = 0;
    const uint64_t T = x->total_tokens;
    std::vector<uint64_t> h_ch;
    std::vector<double> h_cr;
    rc = timed(c, &c->ms[3], [&]() -> yams_status_t {
        yams_status_t r;
        if (np == 0) return YAMS_OK;
        DevBuf pdoc, sc;
        if ((r = pdoc.reserve(np * 4)) != YAMS_OK) return r;
        cm_pair_docs_kernel<<<bm_grid(np), BM_THREADS, 0, st>>>(val.as<uint32_t>(), np, pw.as<uint64_t>(), wdoc.as<uint32_t>(), pdoc.as<uint32_t>());
        YB_CUDA(cudaGetLastError());
        if ((r = pair_runs(tmp, key, pdoc, np, ph, pv, &nposts, st)) != YAMS_OK) return r;
        if ((r = select_indices(tmp, 0, nposts, NewTerm{ph.as<uint64_t>()}, sc, cnt, &nb, st)) != YAMS_OK) return r;
        if ((r = bhash.reserve(nb * 8)) != YAMS_OK || (r = boffs.reserve((nb + 1) * 8)) != YAMS_OK || (r = bttf.reserve(nb * 8)) != YAMS_OK)
            return r;
        bm_terms_kernel<<<bm_grid(nb), BM_THREADS, 0, st>>>(ph.as<uint64_t>(), pv.as<uint64_t>(), nposts, sc.as<uint64_t>(), nb,
                                                            bhash.as<uint64_t>(), boffs.as<uint64_t>(), bttf.as<uint64_t>());
        YB_CUDA(cudaGetLastError());
        uint64_t nb2 = 0;
        if ((r = select_indices(tmp, 0, np, NewTerm{key.as<uint64_t>()}, pstart, cnt, &nb2, st)) != YAMS_OK) return r;
        if ((r = first.reserve(nb * 4)) != YAMS_OK || (r = ab.reserve(nb * 16)) != YAMS_OK || (r = status.reserve(nb)) != YAMS_OK ||
            (r = ratio.reserve(nb * 8)) != YAMS_OK)
            return r;
        const Dict words{x->f[0]->hashes.as<uint64_t>(), x->f[0]->offs.as<uint64_t>(), x->f[0]->terms};
        cm_bigrams_kernel<<<bm_grid(nb), BM_THREADS, 0, st>>>(pstart.as<uint64_t>(), nb, np, val.as<uint32_t>(), pw.as<uint64_t>(),
                                                              whash.as<uint64_t>(), words, x->f[0]->ttf.as<uint64_t>(), c->cfg.min_ttf,
                                                              (double)c->sum_bdl, (double)T, first.as<uint32_t>(), ab.as<uint64_t>(),
                                                              status.as<uint8_t>(), ratio.as<double>());
        YB_CUDA(cudaGetLastError());
        if ((r = select_indices(tmp, 0, nb, PassedTtf{status.as<uint8_t>()}, cand, cnt, &c->passed_ttf, st)) != YAMS_OK) return r;
        // the reference returns before the filter when the index has no tokens (concept_mining.cpp:193-195); sum_bdl > 0 here
        if (T == 0) return YAMS_OK;
        if ((r = select_indices(tmp, 0, nb, IsCandidate{status.as<uint8_t>()}, cand, cnt, &nc, st)) != YAMS_OK) return r;
        if ((r = ch.reserve(std::max<uint64_t>(nc, 1) * 8)) != YAMS_OK || (r = cr.reserve(std::max<uint64_t>(nc, 1) * 8)) != YAMS_OK) return r;
        if (nc) cm_candidates_kernel<<<bm_grid(nc), BM_THREADS, 0, st>>>(cand.as<uint64_t>(), nc, bhash.as<uint64_t>(), ratio.as<double>(),
                                                                         ch.as<uint64_t>(), cr.as<double>());
        YB_CUDA(cudaGetLastError());
        h_ch.resize(nc);
        h_cr.resize(nc);
        if (nc) {
            YB_CUDA(cudaMemcpyAsync(h_ch.data(), ch.p, nc * 8, cudaMemcpyDeviceToHost, st));
            YB_CUDA(cudaMemcpyAsync(h_cr.data(), cr.p, nc * 8, cudaMemcpyDeviceToHost, st));
        }
        return YAMS_OK;
    });
    if (rc != YAMS_OK) return rc;
    c->distinct = nb;
    key = DevBuf();
    // ---- host: std::log of each ratio, the finiteness and floor tests, float(pmi); the cap ----
    const double th = wall_ms();
    std::vector<uint64_t> h_cand(nc);
    if (nc) {
        YB_CUDA(cudaMemcpyAsync(h_cand.data(), cand.p, nc * 8, cudaMemcpyDeviceToHost, st));
        YB_CUDA(cudaStreamSynchronize(st));
    }
    std::vector<std::pair<uint64_t, float>> kept;   // (distinct-bigram index, PMI)
    std::vector<uint64_t> khash;                     // the hash of each
    std::vector<float> apmi;
    for (uint64_t i = 0; i < nc; ++i) {
        const double pmi = std::log(h_cr[i]);
        if (!std::isfinite(pmi) || pmi < (double)c->cfg.pmi_floor) continue;
        kept.emplace_back(h_cand[i], (float)pmi);
        khash.push_back(h_ch[i]);
    }
    c->accepted = kept.size();
    const uint64_t cap = c->cfg.max_concepts;
    double replay_ms = 0.0;
    if (kept.size() > cap) {
        apmi.resize(kept.size());
        for (size_t i = 0; i < kept.size(); ++i) apmi[i] = kept[i].second;
        std::nth_element(apmi.begin(), apmi.begin() + cap, apmi.end(), std::greater<float>());
        const float at_cut = apmi[cap];                                  // rank max_concepts
        const float last_in = cap ? *std::min_element(apmi.begin(), apmi.begin() + cap) : at_cut;   // rank max_concepts - 1
        if (cap == 0) {
            kept.clear();
        } else if (last_in != at_cut) {
            // no tie across the cut: the top max_concepts are the same in any order
            std::vector<std::pair<uint64_t, float>> top;
            top.reserve(cap);
            for (const auto& kv : kept)
                if (kv.second >= last_in) top.push_back(kv);
            kept.swap(top);
        } else {
            const double tr = wall_ms();
            std::vector<uint64_t> order(nb);
            DevBuf k1, v1, k3, v3;
            if ((rc = k1.reserve(nb * 4)) != YAMS_OK || (rc = v1.reserve(nb * 8)) != YAMS_OK) return rc;
            YB_CUDA(cudaMemcpyAsync(k1.p, first.p, nb * 4, cudaMemcpyDeviceToDevice, st));
            YB_CUDA(cudaMemcpyAsync(v1.p, bhash.p, nb * 8, cudaMemcpyDeviceToDevice, st));
            if ((rc = radix_sort<uint32_t, uint64_t>(tmp, k1, v1, k3, v3, nb, st)) != YAMS_OK) return rc;
            YB_CUDA(cudaMemcpyAsync(order.data(), v1.p, nb * 8, cudaMemcpyDeviceToHost, st));
            YB_CUDA(cudaStreamSynchronize(st));
            std::unordered_map<uint64_t, std::pair<float, uint64_t>> acc;
            acc.reserve(kept.size());
            for (size_t i = 0; i < kept.size(); ++i) acc.emplace(khash[i], std::make_pair(kept[i].second, kept[i].first));
            replay_cap(order, acc, c->cfg.max_concepts, kept);
            c->replayed = 1;
            replay_ms = wall_ms() - tr;
        }
    }
    std::sort(kept.begin(), kept.end());   // by distinct-bigram index: hash ascending
    const uint64_t nk = kept.size();
    c->size = nk;
    c->ms[5] = (float)(wall_ms() - th - replay_ms);
    c->ms[6] = (float)replay_ms;
    // ---- gather the kept concepts: dictionary, postings, pmi, idf ----
    rc = timed(c, &c->ms[4], [&]() -> yams_status_t {
        yams_status_t r;
        if (nk == 0) return YAMS_OK;
        std::vector<uint64_t> kb(nk), info(5 * nk);
        for (uint64_t j = 0; j < nk; ++j) kb[j] = kept[j].first;
        DevBuf d_kb, d_info;
        if ((r = d_kb.reserve(nk * 8)) != YAMS_OK || (r = d_info.reserve(nk * 40)) != YAMS_OK) return r;
        YB_CUDA(cudaMemcpyAsync(d_kb.p, kb.data(), nk * 8, cudaMemcpyHostToDevice, st));
        cm_kept_kernel<<<bm_grid(nk), BM_THREADS, 0, st>>>(d_kb.as<uint64_t>(), nk, bhash.as<uint64_t>(), boffs.as<uint64_t>(),
                                                           bttf.as<uint64_t>(), ab.as<uint64_t>(), d_info.as<uint64_t>());
        YB_CUDA(cudaGetLastError());
        YB_CUDA(cudaMemcpyAsync(info.data(), d_info.p, nk * 40, cudaMemcpyDeviceToHost, st));
        YB_CUDA(cudaStreamSynchronize(st));
        c->h_hashes.resize(nk); c->h_ttf.resize(nk); c->h_a.resize(nk); c->h_b.resize(nk);
        c->h_offs.assign(nk + 1, 0); c->h_pmi.resize(nk); c->h_idf.resize(nk);
        const float nf = (float)n;
        for (uint64_t j = 0; j < nk; ++j) {
            c->h_hashes[j] = info[5 * j];
            c->h_ttf[j] = info[5 * j + 1];
            c->h_a[j] = info[5 * j + 2];
            c->h_b[j] = info[5 * j + 3];
            c->h_offs[j + 1] = c->h_offs[j] + info[5 * j + 4];
            c->h_pmi[j] = kept[j].second;
            // the BM25 idf expression for this concept's df (concept_mining.cpp:252-253)
            const float df = (float)info[5 * j + 4];
            c->h_idf[j] = std::log((nf - df + 0.5f) / (df + 0.5f) + 1.0f);
        }
        const uint64_t total = c->h_offs[nk];
        if ((r = c->hashes.reserve(nk * 8)) != YAMS_OK || (r = c->offs.reserve((nk + 1) * 8)) != YAMS_OK ||
            (r = c->pmi.reserve(nk * 4)) != YAMS_OK || (r = c->idf.reserve(nk * 4)) != YAMS_OK ||
            (r = c->docs.reserve(total * 4)) != YAMS_OK || (r = c->tfs.reserve(total * 4)) != YAMS_OK)
            return r;
        YB_CUDA(cudaMemcpyAsync(c->hashes.p, c->h_hashes.data(), nk * 8, cudaMemcpyHostToDevice, st));
        YB_CUDA(cudaMemcpyAsync(c->offs.p, c->h_offs.data(), (nk + 1) * 8, cudaMemcpyHostToDevice, st));
        YB_CUDA(cudaMemcpyAsync(c->pmi.p, c->h_pmi.data(), nk * 4, cudaMemcpyHostToDevice, st));
        YB_CUDA(cudaMemcpyAsync(c->idf.p, c->h_idf.data(), nk * 4, cudaMemcpyHostToDevice, st));
        cm_gather_kernel<<<bm_grid(total), BM_THREADS, 0, st>>>(d_kb.as<uint64_t>(), c->offs.as<uint64_t>(), nk, total, boffs.as<uint64_t>(),
                                                                pv.as<uint64_t>(), c->docs.as<uint32_t>(), c->tfs.as<uint32_t>());
        YB_CUDA(cudaGetLastError());
        YB_CUDA(cudaStreamSynchronize(st));   // the host vectors and d_kb are read until here
        return YAMS_OK;
    });
    if (rc != YAMS_OK) return rc;
    YB_CUDA(cudaStreamSynchronize(st));
    c->ms[7] = (float)(wall_ms() - t0);
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

// ---- the query router (simeon::QueryRouter over the index's field 0, query_router.cpp; DESIGN.md §4.15) ----
struct TermStat {   // Bm25Index::df / idf / total_tf of one hash: 0, 0.0f, 0 when absent
    uint64_t ttf;
    uint32_t df;
    float idf;
};

// df, idf and total_tf of every word hash of a batch of queries
__global__ void bm_term_stats_kernel(Dict D, const uint64_t* __restrict__ ttf, const float* __restrict__ idf, const uint64_t* __restrict__ h,
                                     uint64_t m, TermStat* __restrict__ out) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t b = 0, e = 0, t = 0;
        out[i] = dict_find(D, h[i], &b, &e, &t) ? TermStat{ttf[t], (uint32_t)(e - b), idf[e - b]} : TermStat{0, 0, 0.0f};
    }
}

// QueryRouter::features (query_router.cpp:29-117) of one query from its words' lengths, unfolded hashes and field-0 statistics,
// every operation the reference's, in its order (double, glibc log)
static yams_bm25_query_features router_features(const uint64_t* wlen, const uint64_t* h, const TermStat* ts, uint32_t nw,
                                                uint64_t total_tokens) {
    yams_bm25_query_features f{};
    f.n_terms = nw;
    if (nw == 0) return f;
    uint32_t oov = 0, present = 0;
    double idf_sum = 0.0, idf_sq_sum = 0.0, scq = 0.0;
    uint64_t char_sum = 0;
    float min_idf_seen = std::numeric_limits<float>::infinity();
    std::unordered_map<uint64_t, uint32_t> q_count;
    for (uint32_t i = 0; i < nw; ++i) {
        char_sum += wlen[i];
        if (ts[i].df == 0) { ++oov; continue; }
        const float v = ts[i].idf;
        idf_sum += (double)v;
        idf_sq_sum += (double)v * (double)v;
        if (v > f.max_idf) f.max_idf = v;
        if (v < min_idf_seen) min_idf_seen = v;
        ++present;
        if (ts[i].ttf > 0) scq += (1.0 + std::log((double)ts[i].ttf)) * (double)v;
        ++q_count[h[i]];
    }
    f.oov_rate = (float)oov / (float)nw;
    if (present > 0) {
        f.avg_idf = (float)(idf_sum / present);
        f.min_idf = min_idf_seen;
        if (present > 1) {
            const double mean = idf_sum / present;
            const double var = (idf_sq_sum / present) - (mean * mean);
            f.idf_stddev = (float)(var > 0.0 ? std::sqrt(var) : 0.0);
        }
    }
    f.avg_term_chars = (float)((double)char_sum / (double)nw);
    f.scq_sum = (float)scq;
    if (!q_count.empty() && total_tokens > 0) {
        const double q_norm = (double)nw, c_norm = (double)total_tokens;
        double acc = 0.0;
        std::unordered_set<uint64_t> visited;
        for (uint32_t i = 0; i < nw; ++i) {   // distinct hashes in first-occurrence order
            if (!visited.insert(h[i]).second || ts[i].ttf == 0) continue;
            const double p_q = (double)q_count[h[i]] / q_norm, p_c = (double)ts[i].ttf / c_norm;
            acc += p_q * std::log(p_q / p_c);
        }
        f.simplified_clarity = (float)acc;
    }
    return f;
}

// QueryRouter::choose (query_router.cpp:222-238); features() leaves the pool signals at pool_overlap_jaccard 1, score_decay_rate 0
static uint32_t router_choose(const yams_bm25_query_features& f, const yams_bm25_router_config& c) {
    const float jaccard = 1.0f, decay = 0.0f;
    if (f.n_terms == 0 || f.oov_rate > c.oov_threshold) return YAMS_BM25_RECIPE_SAB_SMOOTH;
    if (f.avg_idf > c.high_idf_threshold && f.n_terms >= c.atire_min_terms && f.min_idf >= c.atire_min_idf_floor &&
        jaccard <= c.atire_max_pool_jaccard && decay >= c.atire_min_score_decay && f.scq_sum >= c.atire_min_scq &&
        f.simplified_clarity <= c.atire_max_clarity)
        return YAMS_BM25_RECIPE_ATIRE;
    if (f.n_terms >= c.cascade_min_terms && f.avg_idf <= c.cascade_max_idf) return YAMS_BM25_RECIPE_CASCADE;
    return YAMS_BM25_RECIPE_SAB_SMOOTH;
}

// SimeonLexicalBackend::scoreRouted with router_enabled: the router's words of every query (unfolded hashes) looked up on the
// device in one kernel, features and choose on the host, then one score call whose Bm25Atire rows score as Atire, the blend
// and the pools' projection
static yams_status_t bm25_score_routed(yams_b200_bm25* x, const yams_bm25_router_config& rc, const yams_b200_concepts* c, float weight,
                                      const char* const* queries, const size_t* qlens, uint32_t nq, const ScoreOut& o,
                                      const uint64_t* cand_off, const uint32_t* cand_docs, float* out_cand, uint32_t* out_recipe,
                                      yams_bm25_query_features* out_features) {
    const double t0 = wall_ms();
    cudaStream_t st = x->st;
    const uint64_t h0 = gram_hash_h0(x->cfg.hash_seed);
    std::vector<std::pair<size_t, size_t>> ws;
    std::vector<uint64_t> h, woff(nq + 1, 0);
    std::vector<uint64_t> wlen;
    for (uint32_t q = 0; q < nq; ++q) {
        const uint8_t* p = reinterpret_cast<const uint8_t*>(queries[q]);
        query_words(p, qlens[q], ws);
        for (const auto& [s, l] : ws) {
            h.push_back(gram_hash(p + s, l, h0));
            wlen.push_back(l);
        }
        woff[q + 1] = h.size();
    }
    std::vector<TermStat> ts(h.size());
    if (!h.empty()) {
        yams_status_t r;
        if ((r = x->rwords.reserve(h.size() * 8)) != YAMS_OK || (r = x->rstats.reserve(h.size() * sizeof(TermStat))) != YAMS_OK) return r;
        const Bm25Field& F = *x->f[0];
        YB_CUDA(cudaMemcpyAsync(x->rwords.p, h.data(), h.size() * 8, cudaMemcpyHostToDevice, st));
        bm_term_stats_kernel<<<bm_grid(h.size()), BM_THREADS, 0, st>>>(Dict{F.hashes.as<uint64_t>(), F.offs.as<uint64_t>(), F.terms},
                                                                       F.ttf.as<uint64_t>(), x->idf->as<float>(), x->rwords.as<uint64_t>(),
                                                                       h.size(), x->rstats.as<TermStat>());
        YB_CUDA(cudaGetLastError());
        YB_CUDA(cudaMemcpyAsync(ts.data(), x->rstats.p, h.size() * sizeof(TermStat), cudaMemcpyDeviceToHost, st));
        YB_CUDA(cudaStreamSynchronize(st));
    }
    std::vector<uint8_t> atire(nq);
    for (uint32_t q = 0; q < nq; ++q) {
        const uint64_t w0 = woff[q];
        const yams_bm25_query_features f =
            router_features(wlen.data() + w0, h.data() + w0, ts.data() + w0, (uint32_t)(woff[q + 1] - w0), x->total_tokens);
        const uint32_t recipe = router_choose(f, rc);
        atire[q] = recipe == YAMS_BM25_RECIPE_ATIRE;
        if (out_recipe) out_recipe[q] = recipe;
        if (out_features) out_features[q] = f;
    }
    if (!o.scores && o.k == 0 && !(cand_off && cand_off[nq])) {   // the route alone: nothing of the scores is asked for
        x->ms[6] = 0.f;
        x->ms[7] = (float)(wall_ms() - t0);
        return YAMS_OK;
    }
    const Routed rt{atire.data(), cand_off, cand_docs, out_cand};
    const yams_status_t r = bm25_score(x, c, weight, queries, qlens, nq, o, -1, &rt);
    x->ms[7] = (float)(wall_ms() - t0);
    return r;
}

// the argument checks every score call makes after its handles': k, the top-k outputs and, when there are queries, the queries
static yams_status_t check_score_args(const char* const* queries, const size_t* qlens, uint32_t nq, const ScoreOut& o) {
    YB_ARG(o.k <= TOPK_MAX, "k must be <= 4096");
    YB_ARG(o.k == 0 || (o.docs && o.topk && o.counts), "null top-k output");
    if (nq == 0) return YAMS_OK;
    YB_ARG(queries && qlens, "null argument");
    for (uint32_t q = 0; q < nq; ++q) YB_ARG(queries[q] || qlens[q] == 0, "null query");
    return YAMS_OK;
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
    return yams_b200_bm25_build_lead(self, cfg_in, texts, lens, n_docs, 0, out);
}

yams_status_t yams_b200_bm25_build_lead(void* self, const yams_bm25_config* cfg_in, const char* const* texts, const size_t* lens,
                                        uint64_t n_docs, uint32_t lead_tokens, yams_b200_bm25** out) {
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
    x->lead = lead_tokens;
    YB_CUDA(cudaStreamCreateWithFlags(&x->st, cudaStreamNonBlocking));
    for (auto& e : x->ev) YB_CUDA(cudaEventCreate(&e));
    for (auto& e : x->zev) YB_CUDA(cudaEventCreate(&e));
    if ((rc = bm25_build(x.get(), texts, lens)) != YAMS_OK) return rc;
    *out = x.release();
    return YAMS_OK;
    YB_CATCH
}

yams_status_t yams_b200_bm25_score(yams_b200_bm25* idx, const char* const* queries, const size_t* qlens, uint32_t nq, float* out_scores,
                                   uint32_t k, uint32_t* out_docs, float* out_topk_scores, uint32_t* out_counts) {
    return yams_b200_bm25_score_blended(idx, nullptr, 0.0f, queries, qlens, nq, out_scores, k, out_docs, out_topk_scores, out_counts);
}

yams_status_t yams_b200_bm25_stats(yams_b200_bm25* idx, yams_bm25_stats* out) {
    DeviceCtx* dev = nullptr;
    yams_status_t rc = ensure_device(&dev);
    if (rc != YAMS_OK) return rc;
    YB_ARG(idx && out, "null argument");
    out->n_docs = idx->n;
    out->avg_dl = idx->f[0]->avg;
    out->ngram_avg_dl = idx->f[1]->avg;
    out->total_tokens = idx->total_tokens;
    for (int fi = 0; fi < 2; ++fi) {
        out->terms[fi] = idx->f[fi]->terms;
        out->postings[fi] = idx->f[fi]->posts;
    }
    out->pruned = idx->pruned;
    return YAMS_OK;
}

yams_status_t yams_b200_bm25_aux_stats(yams_b200_bm25* idx, yams_bm25_stats* out) {
    DeviceCtx* dev = nullptr;
    yams_status_t rc = ensure_device(&dev);
    if (rc != YAMS_OK) return rc;
    YB_ARG(idx && out, "null argument");
    out->n_docs = idx->aux_active ? idx->n : 0;
    out->avg_dl = idx->f[2]->avg;
    out->ngram_avg_dl = idx->f[3]->avg;
    out->total_tokens = idx->f[2]->sum;
    for (int fi = 0; fi < 2; ++fi) {
        out->terms[fi] = idx->f[2 + fi]->terms;
        out->postings[fi] = idx->f[2 + fi]->posts;
    }
    out->pruned = idx->aux_pruned;
    return YAMS_OK;
}

yams_status_t yams_b200_bm25_postings(yams_b200_bm25* idx, uint32_t field, uint64_t term_hash, uint32_t* out_df, float* out_idf,
                                      uint64_t* out_total_tf, uint32_t* out_docs, uint32_t* out_tfs, uint64_t cap) {
    YB_TRY
    DeviceCtx* dev = nullptr;
    yams_status_t rc = ensure_device(&dev);
    if (rc != YAMS_OK) return rc;
    YB_ARG(idx && out_df && out_idf && out_total_tf, "null argument");
    YB_ARG(field < 4, "field must be 0 (words), 1 (n-grams), 2 (lead words) or 3 (lead n-grams)");
    YB_ARG(cap == 0 || (out_docs && out_tfs), "null posting output");
    YB_BIND(idx);
    std::lock_guard<std::mutex> g(idx->mu);
    const Bm25Field& F = *idx->f[field];
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
    YB_CUDA(cudaMemcpy(out_idf, idx->idf->as<float>() + df, 4, cudaMemcpyDeviceToHost));
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
    YB_ARG(field < 4, "field must be 0 (words), 1 (n-grams), 2 (lead words) or 3 (lead n-grams)");
    YB_ARG(out || idx->n == 0, "out is null");
    if (idx->n) memcpy(out, idx->f[field]->h_dl.data(), idx->n * 4);
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

yams_status_t yams_b200_bm25_atire_view(yams_b200_bm25* idx, yams_b200_bm25** out) {
    YB_TRY
    DeviceCtx* dev = nullptr;
    yams_status_t rc = ensure_device(&dev);
    if (rc != YAMS_OK) return rc;
    YB_ARG(idx && out, "null argument");
    *out = nullptr;
    YB_BIND(idx);
    std::unique_ptr<yams_b200_bm25> v(new (std::nothrow) yams_b200_bm25());
    if (!v) return YAMS_ERR_INTERNAL;
    // An Atire build of the same texts, k1, b and hash seed has exactly this word field (n-grams and their pruning never touch
    // words) and the same idf table (it depends on n alone); its n-gram field is empty.
    v->dev = idx->dev;
    v->cfg = idx->cfg;
    v->cfg.variant = YAMS_BM25_ATIRE;
    v->n = idx->n;
    v->total_tokens = idx->total_tokens;
    v->f[0] = idx->f[0];
    v->f[1]->h_dl.assign(idx->n, 0);
    v->f[2] = idx->f[2];   // the lead-text words, as an Atire build with the same lead length would have them
    v->f[3]->h_dl.assign(idx->n, 0);
    v->lead = idx->lead;
    v->aux_active = idx->aux_active;
    v->idf = idx->idf;
    YB_CUDA(cudaStreamCreateWithFlags(&v->st, cudaStreamNonBlocking));
    for (auto& e : v->ev) YB_CUDA(cudaEventCreate(&e));
    for (auto& e : v->zev) YB_CUDA(cudaEventCreate(&e));
    *out = v.release();
    return YAMS_OK;
    YB_CATCH
}

yams_status_t yams_b200_bm25_score_rrf(const yams_b200_bm25* const* variants, uint32_t nv, float k_rrf, const yams_b200_concepts* concepts,
                                       float weight, const char* const* queries, const size_t* qlens, uint32_t nq, float* out_scores,
                                       uint32_t k, uint32_t* out_docs, float* out_topk_scores, uint32_t* out_counts) {
    YB_TRY
    DeviceCtx* dev = nullptr;
    yams_status_t rc = ensure_device(&dev);
    if (rc != YAMS_OK) return rc;
    YB_ARG(nv == 0 || variants, "variants is null");
    for (uint32_t j = 0; j < nv; ++j) YB_ARG(variants[j], "an index is null");
    for (uint32_t j = 1; j < nv; ++j) YB_ARG(variants[j]->n == variants[0]->n, "the indexes differ in document count");
    for (uint32_t j = 1; j < nv; ++j)
        if (variants[j]->dev && variants[0]->dev && variants[j]->dev->device != variants[0]->dev->device) {
            set_last_error("the indexes are on different devices");
            return YAMS_ERR_UNSUPPORTED;
        }
    YB_ARG(std::isfinite(k_rrf) && k_rrf >= 0.0f, "k_rrf must be finite and >= 0");
    YB_ARG(nv == 0 || (uint64_t)nv * variants[0]->n < (1ull << 32), "more than 2^32 - 1 ranked entries per query");
    const ScoreOut o{out_scores, k, out_docs, out_topk_scores, out_counts};
    if ((rc = check_score_args(queries, qlens, nq, o)) != YAMS_OK || nq == 0) return rc;
    if (nv == 0) {   // nothing ranks a document; there is no document count, so no score row
        clear_topk(nq, o);
        return YAMS_OK;
    }
    YB_BIND(variants[0]);
    // every distinct index, locked in address order (the same index may be passed twice; callers may pass them in any order)
    std::vector<yams_b200_bm25*> hs;
    for (uint32_t j = 0; j < nv; ++j) hs.push_back(const_cast<yams_b200_bm25*>(variants[j]));
    std::sort(hs.begin(), hs.end());
    hs.erase(std::unique(hs.begin(), hs.end()), hs.end());
    std::vector<std::unique_lock<std::mutex>> locks;
    for (yams_b200_bm25* h : hs) locks.emplace_back(h->mu);
    return bm25_score_rrf(variants, nv, k_rrf, concepts, weight, queries, qlens, nq, o);
    YB_CATCH
}

void yams_b200_concepts_default_config(yams_concept_config* cfg) {
    if (!cfg) return;
    // ConceptConfig defaults (include/simeon/concept_mining.hpp:16-23)
    cfg->min_ttf = 5;
    cfg->pmi_floor = 2.0f;
    cfg->max_concepts = 200000;
    cfg->k1 = 1.2f;
    cfg->b = 0.75f;
}

yams_status_t yams_b200_concepts_mine(yams_b200_bm25* idx, const yams_concept_config* cfg_in, const char* const* texts, const size_t* lens,
                                      uint64_t n_docs, yams_b200_concepts** out) {
    YB_TRY
    DeviceCtx* dev = nullptr;
    yams_status_t rc = ensure_device(&dev);
    if (rc != YAMS_OK) return rc;
    YB_ARG(idx && out, "null argument");
    *out = nullptr;
    YB_ARG(n_docs < 0xFFFFFFFFull, "too many documents");
    YB_ARG(n_docs == 0 || (texts && lens), "null argument");
    for (uint64_t i = 0; i < n_docs; ++i) YB_ARG(texts[i] || lens[i] == 0, "null text");
    YB_BIND(idx);
    std::unique_ptr<yams_b200_concepts> c(new (std::nothrow) yams_b200_concepts());
    if (!c) return YAMS_ERR_INTERNAL;
    c->dev = dev;
    if (cfg_in) c->cfg = *cfg_in; else yams_b200_concepts_default_config(&c->cfg);
    c->n = n_docs;
    YB_CUDA(cudaStreamCreateWithFlags(&c->st, cudaStreamNonBlocking));
    for (auto& e : c->ev) YB_CUDA(cudaEventCreate(&e));
    std::lock_guard<std::mutex> g(idx->mu);
    c->h0 = gram_hash_h0(idx->cfg.hash_seed);
    if ((rc = concepts_mine(c.get(), idx, texts, lens)) != YAMS_OK) return rc;
    *out = c.release();
    return YAMS_OK;
    YB_CATCH
}

yams_status_t yams_b200_bm25_score_blended(yams_b200_bm25* idx, const yams_b200_concepts* concepts, float weight, const char* const* queries,
                                           const size_t* qlens, uint32_t nq, float* out_scores, uint32_t k, uint32_t* out_docs,
                                           float* out_topk_scores, uint32_t* out_counts) {
    YB_TRY
    DeviceCtx* dev = nullptr;
    yams_status_t rc = ensure_device(&dev);
    if (rc != YAMS_OK) return rc;
    YB_ARG(idx, "index is null");
    const ScoreOut o{out_scores, k, out_docs, out_topk_scores, out_counts};
    if ((rc = check_score_args(queries, qlens, nq, o)) != YAMS_OK || nq == 0) return rc;
    YB_BIND(idx);
    std::lock_guard<std::mutex> g(idx->mu);
    return bm25_score(idx, concepts, weight, queries, qlens, nq, o);
    YB_CATCH
}

yams_status_t yams_b200_bm25_score_strategy(yams_b200_bm25* idx, uint32_t strategy, const yams_b200_concepts* concepts, float weight,
                                            const char* const* queries, const size_t* qlens, uint32_t nq, float* out_scores, uint32_t k,
                                            uint32_t* out_docs, float* out_topk_scores, uint32_t* out_counts, uint32_t* out_chosen) {
    YB_TRY
    DeviceCtx* dev = nullptr;
    yams_status_t rc = ensure_device(&dev);
    if (rc != YAMS_OK) return rc;
    YB_ARG(idx, "index is null");
    YB_ARG(strategy <= YAMS_BM25_STRATEGY_ROUTED, "strategy must be 0 (BM25), 1 (KEYPHRASE), 2 (LEAD_FIELD) or 3 (ROUTED)");
    const ScoreOut o{out_scores, k, out_docs, out_topk_scores, out_counts};
    if ((rc = check_score_args(queries, qlens, nq, o)) != YAMS_OK || nq == 0) return rc;
    YB_BIND(idx);
    std::lock_guard<std::mutex> g(idx->mu);
    return bm25_score_strategy(idx, strategy, concepts, weight, queries, qlens, nq, o, out_chosen);
    YB_CATCH
}

void yams_b200_bm25_default_router_config(yams_bm25_router_config* cfg) {
    if (!cfg) return;
    // RouterConfig's defaults (include/simeon/query_router.hpp:14-65) under the backend's RouterPreset (passE_scq0_clar3,
    // simeon_lexical_backend.h:75-85, applied by toRouterConfig)
    cfg->oov_threshold = 0.0f;
    cfg->high_idf_threshold = 3.0f;
    cfg->atire_min_terms = 0;
    cfg->atire_min_idf_floor = 0.0f;
    cfg->atire_max_pool_jaccard = 1.0f;
    cfg->atire_min_score_decay = 0.0f;
    cfg->atire_min_scq = 0.0f;
    cfg->atire_max_clarity = 3.0f;
    cfg->cascade_min_terms = 4;
    cfg->cascade_max_idf = 5.0f;
}

yams_status_t yams_b200_bm25_score_routed(yams_b200_bm25* idx, const yams_bm25_router_config* rcfg, const yams_b200_concepts* concepts,
                                          float weight, const char* const* queries, const size_t* qlens, uint32_t nq, float* out_scores,
                                          uint32_t k, uint32_t* out_docs, float* out_topk_scores, uint32_t* out_counts,
                                          const uint64_t* cand_offsets, const uint32_t* cand_docs, float* out_cand_scores,
                                          uint32_t* out_recipe, yams_bm25_query_features* out_features) {
    YB_TRY
    DeviceCtx* dev = nullptr;
    yams_status_t rc = ensure_device(&dev);
    if (rc != YAMS_OK) return rc;
    YB_ARG(idx, "index is null");
    const ScoreOut o{out_scores, k, out_docs, out_topk_scores, out_counts};
    if ((rc = check_score_args(queries, qlens, nq, o)) != YAMS_OK || nq == 0) return rc;
    if (cand_offsets) {
        YB_ARG(cand_offsets[0] == 0, "cand_offsets[0] must be 0");
        for (uint32_t q = 0; q < nq; ++q) YB_ARG(cand_offsets[q + 1] >= cand_offsets[q], "cand_offsets must not decrease");
        YB_ARG(cand_offsets[nq] == 0 || (cand_docs && out_cand_scores), "null candidate pool");
        for (uint64_t j = 0; j < cand_offsets[nq]; ++j)
            YB_ARG(cand_docs[j] < idx->n || cand_docs[j] == 0xFFFFFFFFu, "a candidate index is >= n_docs (0xFFFFFFFF: not indexed)");
    }
    yams_bm25_router_config cfg;
    if (rcfg) cfg = *rcfg; else yams_b200_bm25_default_router_config(&cfg);
    YB_BIND(idx);
    std::lock_guard<std::mutex> g(idx->mu);
    return bm25_score_routed(idx, cfg, concepts, weight, queries, qlens, nq, o, cand_offsets, cand_docs, out_cand_scores, out_recipe,
                             out_features);
    YB_CATCH
}

yams_status_t yams_b200_bm25_strategy_stats(yams_b200_bm25* idx, yams_bm25_strategy_stats* out) {
    YB_ARG(idx && out, "null argument");
    std::lock_guard<std::mutex> g(idx->mu);
    *out = idx->sstats;
    return YAMS_OK;
}

yams_status_t yams_b200_concepts_blend(yams_b200_concepts* c, const char* query, size_t qlen, float weight, float* inout, uint64_t n) {
    YB_TRY
    DeviceCtx* dev = nullptr;
    yams_status_t rc = ensure_device(&dev);
    if (rc != YAMS_OK) return rc;
    YB_ARG(c, "concept index is null");
    YB_ARG(query || qlen == 0, "null query");
    YB_ARG(inout || n == 0, "null score vector");
    if (n != c->n || c->size == 0) return YAMS_OK;
    YB_BIND(c);
    std::lock_guard<std::mutex> g(c->mu);
    LegList L;
    L.concepts(c, reinterpret_cast<const uint8_t*>(query), qlen);
    L.end_query();
    if (L.raw.empty()) return YAMS_OK;
    const Scorer s{nullptr, c, weight};
    if ((rc = c->ws.rows.reserve(n * 4)) != YAMS_OK) return rc;
    float* row = c->ws.rows.as<float>();
    float dev_ms = 0.f;   // timed() also waits for the copy back
    return timed(c, &dev_ms, [&]() -> yams_status_t {
        yams_status_t r;
        YB_CUDA(cudaMemcpyAsync(row, inout, n * 4, cudaMemcpyHostToDevice, c->st));
        if ((r = stage_legs(c->ws, L, &s, 1, c->st)) != YAMS_OK || (r = score_rows(c->ws, L, s, n, 0, 1, true, row, c->st)) != YAMS_OK)
            return r;
        YB_CUDA(cudaMemcpyAsync(inout, row, n * 4, cudaMemcpyDeviceToHost, c->st));
        return YAMS_OK;
    });
    YB_CATCH
}

yams_status_t yams_b200_concepts_stats(yams_b200_concepts* c, yams_concepts_stats* out) {
    YB_ARG(c && out, "null argument");
    out->size = c->size;
    out->doc_count = c->n;
    out->avg_bigram_dl = c->avg;
    out->replayed = c->replayed;
    out->sum_bigram_dl = c->sum_bdl;
    out->distinct = c->distinct;
    out->passed_min_ttf = c->passed_ttf;
    out->accepted = c->accepted;
    return YAMS_OK;
}

yams_status_t yams_b200_concepts_find(yams_b200_concepts* c, uint64_t hash, uint32_t* found, float* pmi, float* idf, uint64_t* total_tf,
                                      uint64_t* a_hash, uint64_t* b_hash, uint32_t* df, uint32_t* out_docs, uint32_t* out_tfs, uint64_t cap) {
    YB_TRY
    DeviceCtx* dev = nullptr;
    yams_status_t rc = ensure_device(&dev);
    if (rc != YAMS_OK) return rc;
    YB_ARG(c && found && pmi && idf && total_tf && a_hash && b_hash && df, "null argument");
    YB_ARG(cap == 0 || (out_docs && out_tfs), "null posting output");
    *found = 0; *pmi = 0.0f; *idf = 0.0f; *total_tf = 0; *a_hash = 0; *b_hash = 0; *df = 0;
    const auto it = std::lower_bound(c->h_hashes.begin(), c->h_hashes.end(), hash);
    if (it == c->h_hashes.end() || *it != hash) return YAMS_OK;
    const uint64_t j = (uint64_t)(it - c->h_hashes.begin());
    *found = 1;
    *pmi = c->h_pmi[j];
    *idf = c->h_idf[j];
    *total_tf = c->h_ttf[j];
    *a_hash = c->h_a[j];
    *b_hash = c->h_b[j];
    *df = (uint32_t)(c->h_offs[j + 1] - c->h_offs[j]);
    const uint64_t m = std::min<uint64_t>(*df, cap);
    if (m) {
        YB_BIND(c);
        YB_CUDA(cudaMemcpy(out_docs, c->docs.as<uint32_t>() + c->h_offs[j], m * 4, cudaMemcpyDeviceToHost));
        YB_CUDA(cudaMemcpy(out_tfs, c->tfs.as<uint32_t>() + c->h_offs[j], m * 4, cudaMemcpyDeviceToHost));
    }
    return YAMS_OK;
    YB_CATCH
}

yams_status_t yams_b200_concepts_hashes(yams_b200_concepts* c, uint64_t* out) {
    YB_ARG(c && (out || c->size == 0), "null argument");
    if (c->size) memcpy(out, c->h_hashes.data(), c->size * 8);
    return YAMS_OK;
}

yams_status_t yams_b200_concepts_bigram_lengths(yams_b200_concepts* c, uint32_t* out) {
    YB_ARG(c && (out || c->n == 0), "null argument");
    if (c->n) memcpy(out, c->h_bdl.data(), c->n * 4);
    return YAMS_OK;
}

yams_status_t yams_b200_concepts_last_timings(yams_b200_concepts* c, float out_ms[8]) {
    YB_ARG(c && out_ms, "null argument");
    std::lock_guard<std::mutex> g(c->mu);
    for (int i = 0; i < 8; ++i) out_ms[i] = c->ms[i];
    return YAMS_OK;
}

void yams_b200_concepts_destroy(yams_b200_concepts* c) { delete c; }

}  // extern "C"
