// ref_rrf_shim.cpp -- C entry into simeon's own score_bm25_variants_rrf (third_party/simeon/src/fusion.cpp), over its own
// Bm25Index variants and ConceptIndex, compiled with them by oracle/rrf.mk into oracle/_ref/libref_rrf.so.  Test
// infrastructure only.
#include <cstddef>
#include <cstdint>
#include <span>
#include <string_view>
#include <vector>

#include "simeon/bm25.hpp"
#include "simeon/concept_mining.hpp"
#include "simeon/fusion.hpp"

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

std::vector<std::string_view> views(const char* const* texts, const size_t* lens, size_t n) {
    std::vector<std::string_view> v;
    for (size_t i = 0; i < n; ++i) v.emplace_back(lens[i] ? texts[i] : "", lens[i]);
    return v;
}

}  // namespace

extern "C" {

// a Bm25Index over texts (add_doc each, finalize)
void* ref_rrf_index(const ShimCfg* c, const char* const* texts, const size_t* lens, size_t n) {
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
    for (const auto& t : views(texts, lens, n)) ix->add_doc(t);
    ix->finalize();
    return ix;
}

void ref_rrf_index_destroy(void* h) { delete static_cast<simeon::Bm25Index*>(h); }

// mine_concepts(index, texts, cfg)
void* ref_rrf_concepts(void* ix, const ShimConceptCfg* cc, const char* const* texts, const size_t* lens, size_t n) {
    simeon::ConceptConfig cfg;
    cfg.min_ttf = cc->min_ttf;
    cfg.pmi_floor = cc->pmi_floor;
    cfg.max_concepts = cc->max_concepts;
    cfg.k1 = cc->k1;
    cfg.b = cc->b;
    return new simeon::ConceptIndex(simeon::mine_concepts(*static_cast<simeon::Bm25Index*>(ix), views(texts, lens, n), cfg));
}

void ref_rrf_concepts_destroy(void* h) { delete static_cast<simeon::ConceptIndex*>(h); }

// SimeonLexicalBackend::score with bm25_variants_rrf: score_bm25_variants_rrf(variants, query, out[n], k_rrf), then, with a
// concept index, blend_into(query, out, weight)
void ref_rrf_score(void* const* variants, size_t nv, const char* q, size_t len, float k_rrf, void* concepts, float weight, float* out,
                   size_t n) {
    std::vector<const simeon::Bm25Index*> vs;
    for (size_t j = 0; j < nv; ++j) vs.push_back(static_cast<const simeon::Bm25Index*>(variants[j]));
    const std::string_view query(len ? q : "", len);
    simeon::score_bm25_variants_rrf(std::span<const simeon::Bm25Index* const>(vs.data(), vs.size()), query, std::span<float>(out, n), k_rrf);
    if (concepts) static_cast<const simeon::ConceptIndex*>(concepts)->blend_into(query, std::span<float>(out, n), weight);
}

}  // extern "C"
