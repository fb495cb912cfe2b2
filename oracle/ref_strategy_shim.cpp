// ref_strategy_shim.cpp -- C entry into simeon's own lead-text field and the lexical backend's strategy router: extract_lead_tokens
// (src/corpus_adapter.cpp), Bm25Index::add_doc(text, aux_text) and score_bm25f (src/bm25.cpp), Bm25Strategy, KeyphraseStrategy,
// LeadFieldStrategy and EntropyRouter (src/retrieval_strategy.cpp), and the concept blend after them (src/concept_mining.cpp).
// Compiled with them by oracle/strategy.mk into oracle/_ref/libref_strategy.so.  Test infrastructure only.
//
// The entropy profile the router routes on is the backend's own code (SimeonLexicalBackend::scoreStrategyRouted), not simeon's;
// ref_strategy_score restates it below.
//
// The index keeps its aux fields private; the shim reads them (lengths, averages, posting lists) through `private` redefined
// as `public` for bm25.hpp's own text only.  Every header it includes is included before the redefinition, so their include
// guards keep the macro out of the standard library.  That changes access, not layout.
#include <atomic>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <memory>
#include <mutex>
#include <span>
#include <string>
#include <string_view>
#include <utility>
#include <vector>

#include "simeon/flat_hash_map_u64.hpp"
#include "simeon/simeon.hpp"
#define private public
#include "simeon/bm25.hpp"
#undef private
#include "simeon/concept_mining.hpp"
#include "simeon/corpus_adapter.hpp"
#include "simeon/retrieval_strategy.hpp"

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

// what the backend builds with the strategy router on: the index with every document's lead text as its aux field, the lead
// texts themselves (LeadFieldStrategy's), and the three strategies over them
struct Built {
    simeon::Bm25Index ix;
    std::vector<std::string> leads;
    simeon::Bm25Strategy pool0;
    simeon::KeyphraseStrategy pool1;
    simeon::LeadFieldStrategy pool2;
    explicit Built(const simeon::Bm25Config& c, std::vector<std::string> l)
        : ix(c), leads(std::move(l)), pool0(ix), pool1(ix, 0.25f, 0.30f), pool2(ix, leads, 0.85f, 0.15f) {}
};

std::string_view view(const char* p, size_t len) { return std::string_view(len ? p : "", len); }

const simeon::FlatHashMapU64<simeon::Bm25Index::TermPostings>& field_map(const simeon::Bm25Index& ix, int field) {
    switch (field) {
        case 0: return ix.postings_;
        case 1: return ix.ngram_postings_;
        case 2: return ix.aux_postings_;
        default: return ix.aux_ngram_postings_;
    }
}
const std::vector<uint32_t>& lengths(const simeon::Bm25Index& ix, int field) {
    switch (field) {
        case 0: return ix.doc_lengths_;
        case 1: return ix.ngram_doc_lengths_;
        case 2: return ix.aux_doc_lengths_;
        default: return ix.aux_ngram_doc_lengths_;
    }
}

}  // namespace

extern "C" {

// extract_lead_tokens(text, max_tokens) -> out (capacity len); returns its length
size_t ref_strategy_lead(const char* text, size_t len, uint32_t max_tokens, char* out) {
    const std::string s = simeon::extract_lead_tokens(view(text, len), max_tokens);
    if (!s.empty()) std::memcpy(out, s.data(), s.size());
    return s.size();
}

// add_doc(text, lead_tokens ? extract_lead_tokens(text, lead_tokens) : "") for each text, then finalize()
void* ref_strategy_build(const ShimCfg* c, const char* const* texts, const size_t* lens, size_t n, uint32_t lead_tokens) {
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
    std::vector<std::string> leads;
    for (size_t i = 0; i < n; ++i) leads.push_back(lead_tokens ? simeon::extract_lead_tokens(view(texts[i], lens[i]), lead_tokens) : "");
    auto* b = new Built(cfg, leads);
    for (size_t i = 0; i < n; ++i) b->ix.add_doc(view(texts[i], lens[i]), b->leads[i]);
    b->ix.finalize();
    return b;
}

void ref_strategy_destroy(void* h) { delete static_cast<Built*>(h); }

void* ref_strategy_concepts(void* h, const ShimConceptCfg* cc, const char* const* texts, const size_t* lens, size_t n) {
    simeon::ConceptConfig cfg;
    cfg.min_ttf = cc->min_ttf;
    cfg.pmi_floor = cc->pmi_floor;
    cfg.max_concepts = cc->max_concepts;
    cfg.k1 = cc->k1;
    cfg.b = cc->b;
    std::vector<std::string_view> v;
    for (size_t i = 0; i < n; ++i) v.push_back(view(texts[i], lens[i]));
    return new simeon::ConceptIndex(simeon::mine_concepts(static_cast<Built*>(h)->ix, v, cfg));
}

void ref_strategy_concepts_destroy(void* h) { delete static_cast<simeon::ConceptIndex*>(h); }

// pool 0 (Bm25Strategy, evidence = TextAdapter::process_query's lead text), 1 (KeyphraseStrategy), 2 (LeadFieldStrategy) of the
// backend's strategy list, or 3: the router -- the entropy profile of the query's plain scores, then EntropyRouter::route over the
// three.  Then blend_into(query, out, weight) with a concept index.  Returns the pool that scored.
int ref_strategy_score(void* h, int pool, const char* q, size_t len, void* concepts, float weight, float* out) {
    auto* b = static_cast<Built*>(h);
    const std::string_view query = view(q, len);
    const size_t n = b->ix.doc_count();
    const std::span<float> s(out, n);
    simeon::TextAdapter adapter;
    const simeon::AdapterEvidence ev = adapter.process_query("query", query);
    simeon::RetrievalStrategy* pools[3] = {&b->pool0, &b->pool1, &b->pool2};
    int chosen = pool;
    if (pool == 3) {
        // The profile: over the documents of positive plain score, in document order, the mean of sn * -log(sn), sn = s / max
        // as a float quotient taken to double; 0 when no score is positive.
        std::vector<float> plain(n, 0.0f);
        b->ix.score(query, std::span<float>(plain));
        float top = 0.0f;
        for (float v : plain) top = v > top ? v : top;
        simeon::QueryProfile profile;
        if (top > 0.0f) {
            double acc = 0.0, positives = 0.0;
            for (float v : plain) {
                if (!(v > 0.0f)) continue;
                const double sn = v / top;
                if (sn > 0.0) acc += sn * (-std::log(sn));
                positives += 1.0;
            }
            profile.bm25_entropy = positives > 0.0 ? static_cast<float>(acc / positives) : 0.0f;
        }
        chosen = profile.bm25_entropy < 0.05f ? 0 : profile.bm25_entropy > 0.50f ? 2 : 1;
        simeon::EntropyRouter().route(query, profile, ev, std::span<simeon::RetrievalStrategy* const>(pools, 3), s);
    } else {
        pools[pool]->score(query, ev, s);
    }
    if (concepts) static_cast<const simeon::ConceptIndex*>(concepts)->blend_into(query, s, weight);
    return chosen;
}

// field 0..3 (words, n-grams, aux words, aux n-grams): out_f[0] avg length; out_u[0] documents of the field (0 for an aux field
// never activated), [1] sum of lengths, [2] terms, [3] postings
void ref_strategy_field_stats(void* h, int field, float* out_f, uint64_t* out_u) {
    const auto& ix = static_cast<Built*>(h)->ix;
    const float avgs[4] = {ix.avg_dl_, ix.ngram_avg_dl_, ix.aux_avg_dl_, ix.aux_ngram_avg_dl_};
    out_f[0] = avgs[field];
    const auto& l = lengths(ix, field);
    out_u[0] = l.size();
    out_u[1] = 0;
    for (uint32_t v : l) out_u[1] += v;
    out_u[2] = out_u[3] = 0;
    for (const auto& [hash, tp] : field_map(ix, field)) {
        (void)hash;
        ++out_u[2];
        out_u[3] += tp.docs.size();
    }
}

// the posting list of term_hash in field 0..3: returns df (0 when absent); docs / tfs get min(df, cap)
uint32_t ref_strategy_postings(void* h, int field, uint64_t term_hash, float* idf, uint64_t* total_tf, uint32_t* docs, uint32_t* tfs,
                               size_t cap) {
    const auto& m = field_map(static_cast<Built*>(h)->ix, field);
    auto it = m.find(term_hash);
    if (it == m.end()) return 0;
    *idf = it->second.idf;
    *total_tf = it->second.total_tf;
    const auto& d = it->second.docs;
    for (size_t i = 0; i < d.size() && i < cap; ++i) {
        docs[i] = d[i].first;
        tfs[i] = d[i].second;
    }
    return static_cast<uint32_t>(d.size());
}

// the lengths of field 0..3 -> out[doc_count] (zeros where the field has none)
void ref_strategy_doc_lengths(void* h, int field, uint32_t* out) {
    const auto& ix = static_cast<Built*>(h)->ix;
    const auto& v = lengths(ix, field);
    std::memset(out, 0, ix.doc_count() * 4);
    if (!v.empty()) std::memcpy(out, v.data(), v.size() * 4);
}

}  // extern "C"
