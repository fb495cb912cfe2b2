// ref_bm25_shim.cpp -- C entry into simeon's own Bm25Index (third_party/simeon/src/bm25.cpp), compiled with it by
// oracle/bm25.mk into oracle/_ref/libref_bm25.so.  Test infrastructure only.
//
// The index keeps its n-gram field private; the shim reads it (avg length, posting lists) through `private` redefined as
// `public` for this one translation unit.  That changes access, not layout: the class is the one bm25.cpp was compiled with.
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <string_view>
#include <vector>

#define private public
#include "simeon/bm25.hpp"
#undef private

namespace {

struct ShimCfg {   // the layout of yams_bm25_config (include/yams_b200.h)
    float k1, b, delta, gamma;
    uint32_t variant, ngram_min, ngram_max;
    float prune_ratio;
    uint64_t hash_seed;
};

const simeon::FlatHashMapU64<simeon::Bm25Index::TermPostings>& field_map(const simeon::Bm25Index& ix, int field) {
    return field == 0 ? ix.postings_ : ix.ngram_postings_;
}

}  // namespace

extern "C" {

void* ref_bm25_build(const ShimCfg* c, const char* const* texts, const size_t* lens, size_t n) {
    simeon::Bm25Config cfg;
    cfg.k1 = c->k1;
    cfg.b = c->b;
    cfg.delta = c->delta;
    cfg.subword_gamma = c->gamma;
    cfg.variant = static_cast<simeon::Bm25Variant>(c->variant);
    cfg.ngram_min = c->ngram_min;
    cfg.ngram_max = c->ngram_max;
    cfg.ngram_df_prune_ratio = c->prune_ratio;
    cfg.hash_seed = c->hash_seed;
    auto* ix = new simeon::Bm25Index(cfg);
    for (size_t i = 0; i < n; ++i) ix->add_doc(std::string_view(lens[i] ? texts[i] : "", lens[i]));
    ix->finalize();
    return ix;
}

void ref_bm25_score(void* h, const char* q, size_t len, float* out) {
    auto* ix = static_cast<simeon::Bm25Index*>(h);
    ix->score(std::string_view(len ? q : "", len), std::span<float>(out, ix->doc_count()));
}

// out_f[0] avg_dl, [1] ngram avg_dl; out_u[0] n_docs, [1] total_tokens, [2..3] terms (word, n-gram), [4..5] postings
void ref_bm25_stats(void* h, float* out_f, uint64_t* out_u) {
    auto* ix = static_cast<simeon::Bm25Index*>(h);
    out_f[0] = ix->avg_dl_;
    out_f[1] = ix->ngram_avg_dl_;
    out_u[0] = ix->doc_count();
    out_u[1] = ix->total_tokens_;
    for (int f = 0; f < 2; ++f) {
        const auto& m = field_map(*ix, f);
        uint64_t terms = 0, posts = 0;
        for (const auto& [hash, tp] : m) {
            (void)hash;
            ++terms;
            posts += tp.docs.size();
        }
        out_u[2 + f] = terms;
        out_u[4 + f] = posts;
    }
}

// the posting list of term_hash in field 0 (words) or 1 (n-grams): returns df (0 when absent); docs/tfs get min(df, cap)
uint32_t ref_bm25_postings(void* h, int field, uint64_t term_hash, float* idf, uint64_t* total_tf, uint32_t* docs, uint32_t* tfs,
                           size_t cap) {
    auto* ix = static_cast<simeon::Bm25Index*>(h);
    const auto& m = field_map(*ix, field);
    auto it = m.find(term_hash);
    if (it == m.end()) return 0;
    *idf = it->second.idf;
    *total_tf = it->second.total_tf;
    const auto& d = it->second.docs;
    for (size_t i = 0; i < d.size() && i < cap; ++i) {
        docs[i] = d[i].first;
        tfs[i] = d[i].second;
    }
    return (uint32_t)d.size();
}

void ref_bm25_doc_lengths(void* h, int field, uint32_t* out) {
    auto* ix = static_cast<simeon::Bm25Index*>(h);
    const auto& v = field == 0 ? ix->doc_lengths_ : ix->ngram_doc_lengths_;
    if (!v.empty()) std::memcpy(out, v.data(), v.size() * 4);
}

uint64_t ref_bm25_hash(void* h, const char* term, size_t len) {
    return static_cast<simeon::Bm25Index*>(h)->hash_term(std::string_view(len ? term : "", len));
}

// Bm25Index::df / idf / total_tf of a raw term string (no tokenisation, no case folding)
void ref_bm25_term(void* h, const char* term, size_t len, uint32_t* df, float* idf, uint64_t* total_tf) {
    auto* ix = static_cast<simeon::Bm25Index*>(h);
    const std::string_view t(len ? term : "", len);
    *df = ix->df(t);
    *idf = ix->idf(t);
    *total_tf = ix->total_tf(t);
}

void ref_bm25_destroy(void* h) { delete static_cast<simeon::Bm25Index*>(h); }

}  // extern "C"
