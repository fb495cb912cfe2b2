// ref_router_shim.cpp -- C entry into simeon's own QueryRouter (third_party/simeon/src/query_router.cpp), over its own Bm25Index
// and ConceptIndex, compiled with them by oracle/router.mk into oracle/_ref/libref_router.so.  Test infrastructure only.
//
// ref_router_score restates SimeonLexicalBackend::scoreRouted with router_enabled (fragment geometry and RRF off,
// simeon_lexical_backend.cpp:836-934): the router over the Atire index when there is one, else the primary (:553); choose; the
// chosen index's score -- the Atire index for Bm25Atire when there is one, else the primary; the concept blend; the projection
// onto the candidate pool.
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <span>
#include <string_view>
#include <vector>

#include "simeon/bm25.hpp"
#include "simeon/concept_mining.hpp"
#include "simeon/query_router.hpp"

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
struct ShimRouterCfg {   // the layout of yams_bm25_router_config
    float oov_threshold, high_idf_threshold;
    uint32_t atire_min_terms;
    float atire_min_idf_floor, atire_max_pool_jaccard, atire_min_score_decay, atire_min_scq, atire_max_clarity;
    uint32_t cascade_min_terms;
    float cascade_max_idf;
};
struct ShimFeatures {   // the layout of yams_bm25_query_features
    float oov_rate, avg_idf, max_idf, min_idf, idf_stddev;
    uint32_t n_terms;
    float avg_term_chars, scq_sum, simplified_clarity;
};

std::vector<std::string_view> views(const char* const* texts, const size_t* lens, size_t n) {
    std::vector<std::string_view> v;
    for (size_t i = 0; i < n; ++i) v.emplace_back(lens[i] ? texts[i] : "", lens[i]);
    return v;
}

}  // namespace

extern "C" {

// a Bm25Index over texts (add_doc each, finalize)
void* ref_router_index(const ShimCfg* c, const char* const* texts, const size_t* lens, size_t n) {
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

void ref_router_index_destroy(void* h) { delete static_cast<simeon::Bm25Index*>(h); }

// mine_concepts(index, texts, cfg)
void* ref_router_concepts(void* ix, const ShimConceptCfg* cc, const char* const* texts, const size_t* lens, size_t n) {
    simeon::ConceptConfig cfg;
    cfg.min_ttf = cc->min_ttf;
    cfg.pmi_floor = cc->pmi_floor;
    cfg.max_concepts = cc->max_concepts;
    cfg.k1 = cc->k1;
    cfg.b = cc->b;
    return new simeon::ConceptIndex(simeon::mine_concepts(*static_cast<simeon::Bm25Index*>(ix), views(texts, lens, n), cfg));
}

void ref_router_concepts_destroy(void* h) { delete static_cast<simeon::ConceptIndex*>(h); }

// scoreRouted of one query over the primary and the Atire index (nullable: none, as when the primary is Atire): *recipe, the
// features, the full scores out[n] and, for ncand candidates (0xFFFFFFFF: not indexed), their projection out_cand[ncand]
void ref_router_score(void* primary, void* atire, const ShimRouterCfg* rc, const char* q, size_t len, void* concepts, float weight,
                      float* out, size_t n, const uint32_t* cand, size_t ncand, float* out_cand, uint32_t* recipe, ShimFeatures* feats) {
    const auto* idx = static_cast<const simeon::Bm25Index*>(primary);
    const auto* at = static_cast<const simeon::Bm25Index*>(atire);
    simeon::RouterConfig cfg;
    cfg.oov_threshold = rc->oov_threshold;
    cfg.high_idf_threshold = rc->high_idf_threshold;
    cfg.atire_min_terms = rc->atire_min_terms;
    cfg.atire_min_idf_floor = rc->atire_min_idf_floor;
    cfg.atire_max_pool_jaccard = rc->atire_max_pool_jaccard;
    cfg.atire_min_score_decay = rc->atire_min_score_decay;
    cfg.atire_min_scq = rc->atire_min_scq;
    cfg.atire_max_clarity = rc->atire_max_clarity;
    cfg.cascade_min_terms = rc->cascade_min_terms;
    cfg.cascade_max_idf = rc->cascade_max_idf;
    const std::string_view query(len ? q : "", len);
    const simeon::QueryRouter router(at ? *at : *idx, cfg);
    const simeon::QueryFeatures f = router.features(query);
    const simeon::Recipe r = router.choose(f);
    const simeon::Bm25Index* chosen = r == simeon::Recipe::Bm25Atire && at ? at : idx;
    std::vector<float> full(n, 0.0f);
    chosen->score(query, std::span<float>(full));
    if (concepts) static_cast<const simeon::ConceptIndex*>(concepts)->blend_into(query, std::span<float>(full), weight);
    for (size_t i = 0; i < n; ++i) out[i] = full[i];
    for (size_t j = 0; j < ncand; ++j)
        out_cand[j] = cand[j] == 0xFFFFFFFFu ? 0.0f : (std::isfinite(full[cand[j]]) ? full[cand[j]] : 0.0f);
    *recipe = static_cast<uint32_t>(r);
    *feats = ShimFeatures{f.oov_rate, f.avg_idf, f.max_idf, f.min_idf, f.idf_stddev, f.n_terms, f.avg_term_chars, f.scq_sum,
                          f.simplified_clarity};
}

}  // extern "C"
