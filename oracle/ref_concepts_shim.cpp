// ref_concepts_shim.cpp -- C entry into simeon's own ConceptIndex (third_party/simeon/src/concept_mining.cpp) and the Bm25Index
// it is mined against, compiled with them by oracle/concepts.mk into oracle/_ref/libref_concepts.so.  Test infrastructure only.
//
// The concept index keeps its state private; the shim reads it (lengths, average, entries) through `private` redefined as
// `public` for this one translation unit.  That changes access, not layout.
#include <algorithm>
#include <chrono>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <string_view>
#include <vector>

#define private public
#include "simeon/bm25.hpp"
#include "simeon/concept_mining.hpp"
#undef private

namespace {

struct ShimCfg {   // the layout of yams_bm25_config (include/yams_b200.h)
    float k1, b, delta, gamma;
    uint32_t variant, ngram_min, ngram_max;
    float prune_ratio;
    uint64_t hash_seed;
};
struct ShimConceptCfg {   // the layout of yams_concept_config
    uint32_t min_ttf;
    float pmi_floor;
    uint32_t max_concepts;
    float k1, b;
};

struct Pair {
    simeon::Bm25Index* ix;
    simeon::ConceptIndex ci;
    double mine_ms = 0.0;   // wall time of mine_concepts alone
};

std::vector<std::string_view> views(const char* const* texts, const size_t* lens, size_t n) {
    std::vector<std::string_view> v;
    for (size_t i = 0; i < n; ++i) v.emplace_back(lens[i] ? texts[i] : "", lens[i]);
    return v;
}

}  // namespace

extern "C" {

// a Bm25Index over texts, then mine_concepts(index, ctexts, cfg)
void* ref_concepts_build(const ShimCfg* c, const char* const* texts, const size_t* lens, size_t n, const ShimConceptCfg* cc,
                         const char* const* ctexts, const size_t* clens, size_t cn) {
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
    auto* p = new Pair{new simeon::Bm25Index(cfg), {}, 0.0};
    for (const auto& t : views(texts, lens, n)) p->ix->add_doc(t);
    p->ix->finalize();
    simeon::ConceptConfig ccfg;
    ccfg.min_ttf = cc->min_ttf;
    ccfg.pmi_floor = cc->pmi_floor;
    ccfg.max_concepts = cc->max_concepts;
    ccfg.k1 = cc->k1;
    ccfg.b = cc->b;
    const auto docs = views(ctexts, clens, cn);
    const auto t0 = std::chrono::steady_clock::now();
    p->ci = simeon::mine_concepts(*p->ix, docs, ccfg);
    p->mine_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return p;
}

double ref_concepts_mine_ms(void* h) { return static_cast<Pair*>(h)->mine_ms; }

// out_f[0] avg_bigram_dl; out_u[0] size, [1] doc_count, [2] sum of bigram lengths
void ref_concepts_stats(void* h, float* out_f, uint64_t* out_u) {
    const auto* p = static_cast<Pair*>(h);
    out_f[0] = p->ci.avg_dl();
    out_u[0] = p->ci.size();
    out_u[1] = p->ci.doc_count();
    uint64_t s = 0;
    for (uint32_t v : p->ci.bigram_doc_lengths_) s += v;
    out_u[2] = s;
}

void ref_concepts_bigram_lengths(void* h, uint32_t* out) {
    const auto& v = static_cast<Pair*>(h)->ci.bigram_doc_lengths_;
    if (!v.empty()) std::memcpy(out, v.data(), v.size() * 4);
}

// the kept hashes, ascending
void ref_concepts_hashes(void* h, uint64_t* out) {
    std::vector<uint64_t> v;
    for (const auto& kv : static_cast<Pair*>(h)->ci.concepts_) v.push_back(kv.first);
    std::sort(v.begin(), v.end());
    if (!v.empty()) std::memcpy(out, v.data(), v.size() * 8);
}

// ConceptIndex::find: -1 when absent, else df; ttf_ab = total_tf, a_hash, b_hash; the first min(df, cap) postings
int64_t ref_concepts_find(void* h, uint64_t hash, float* pmi, float* idf, uint64_t* ttf_ab, uint32_t* docs, uint32_t* tfs, size_t cap) {
    const simeon::ConceptEntry* e = static_cast<Pair*>(h)->ci.find(hash);
    if (!e) return -1;
    *pmi = e->pmi;
    *idf = e->idf;
    ttf_ab[0] = e->total_tf;
    ttf_ab[1] = e->a_hash;
    ttf_ab[2] = e->b_hash;
    for (size_t i = 0; i < e->docs.size() && i < cap; ++i) {
        docs[i] = e->docs[i].first;
        tfs[i] = e->docs[i].second;
    }
    return (int64_t)e->docs.size();
}

// ConceptIndex::blend_into(query, vec[n], weight)
void ref_concepts_blend(void* h, const char* q, size_t len, float weight, float* vec, size_t n) {
    static_cast<Pair*>(h)->ci.blend_into(std::string_view(len ? q : "", len), std::span<float>(vec, n), weight);
}

// the lexical backend's score: Bm25Index::score into zeros, then blend_into(query, scores, weight)
void ref_concepts_score_blended(void* h, const char* q, size_t len, float weight, float* out) {
    auto* p = static_cast<Pair*>(h);
    const std::string_view query(len ? q : "", len);
    const size_t n = p->ix->doc_count();
    std::fill(out, out + n, 0.0f);
    p->ix->score(query, std::span<float>(out, n));
    p->ci.blend_into(query, std::span<float>(out, n), weight);
}

void ref_concepts_destroy(void* h) {
    auto* p = static_cast<Pair*>(h);
    delete p->ix;
    delete p;
}

}  // extern "C"
