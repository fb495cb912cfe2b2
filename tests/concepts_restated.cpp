// concepts_restated.cpp -- a restatement of simeon's word-bigram concept mining and blend (ConceptIndex), written from the
// semantics in DESIGN.md §4.12; compiled at test time into a temporary shared library (tests/concepts_restated.py).
//
// C++ rather than numpy: two of the reference's results depend on the standard library's container order, and this file uses
// the same containers the same way.  The cap keeps the first max_concepts of the accepted bigrams -- collected in the iteration
// order of an unordered_map filled in first-occurrence order -- after std::nth_element by PMI descending; the blend adds the
// matched concepts in the iteration order of an unordered_map reserved for the query's word count.  The word statistics the
// mining needs (total_tf of a case-folded word, total_tokens) are computed here from the index's texts.
//
// Float arithmetic is plain float with one rounding per operation: build without -mfma (and with -ffp-contract=off).
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

namespace {

uint64_t mix(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
}

// SplitMix64 string hash of bytes p[0, n), optionally of their ASCII lowercase
uint64_t hash_bytes(const unsigned char* p, size_t n, uint64_t seed, bool fold) {
    auto byte = [&](size_t i) -> uint64_t {
        unsigned char c = p[i];
        if (fold && c >= 'A' && c <= 'Z') c = (unsigned char)(c | 0x20);
        return c;
    };
    uint64_t h = mix(seed ^ 0x9E3779B97F4A7C15ULL);
    size_t i = 0;
    for (; i + 8 <= n; i += 8) {
        uint64_t w = 0;
        for (int b = 0; b < 8; ++b) w |= byte(i + b) << (8 * b);
        h = mix(h ^ w);
    }
    if (i < n) {
        uint64_t w = 0;
        for (size_t j = 0; i + j < n; ++j) w |= byte(i + j) << (8 * j);
        h = mix(h ^ w ^ ((uint64_t)(n - i) << 56));
    }
    return mix(h ^ (uint64_t)n);
}

bool word_char(unsigned char c) { return (c >= '0' && c <= '9') || (c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z') || c == '_'; }

std::vector<uint64_t> word_hashes(const char* text, size_t len, uint64_t seed, bool fold) {
    std::vector<uint64_t> out;
    const auto* p = reinterpret_cast<const unsigned char*>(text);
    size_t i = 0;
    while (i < len) {
        if (!word_char(p[i])) { ++i; continue; }
        const size_t s = i;
        while (i < len && word_char(p[i])) ++i;
        out.push_back(hash_bytes(p + s, i - s, seed, fold));
    }
    return out;
}

uint64_t bigram(uint64_t a, uint64_t b) { return mix(a ^ mix(b + 0x9E3779B97F4A7C15ULL)); }

struct Concept {
    float pmi = 0.f, idf = 0.f;
    uint64_t total_tf = 0, a = 0, b = 0;
    std::vector<std::pair<uint32_t, uint32_t>> postings;   // (document, tf), document ascending
};

struct Cfg {
    uint32_t min_ttf;
    float pmi_floor;
    uint32_t max_concepts;
    float k1, b;
};

struct Mined {
    uint64_t seed = 0;
    Cfg cfg{};
    uint32_t n = 0;
    std::vector<uint32_t> bdl;
    uint64_t sum_bdl = 0, distinct = 0, passed = 0, accepted = 0;
    uint32_t tie_at_cap = 0;
    float avg = 0.f;
    std::vector<float> accepted_pmi;   // descending, before the cap
    std::unordered_map<uint64_t, Concept> concepts;
};

struct Bigram {   // one distinct bigram while mining
    uint64_t total_tf = 0, a = 0, b = 0;
    std::vector<std::pair<uint32_t, uint32_t>> postings;
};

// cap_mode 1 reverses the accepted list before the selection, which keeps another subset when a tie crosses the cap
Mined* mine(uint64_t seed, const char* const* itexts, const size_t* ilens, size_t in, const Cfg& cfg, const char* const* texts,
            const size_t* lens, size_t n, int cap_mode) {
    auto* m = new Mined();
    m->seed = seed;
    m->cfg = cfg;
    m->n = (uint32_t)n;
    m->bdl.assign(n, 0);
    // the index's word statistics: total tf of every case-folded word, and the token count
    std::unordered_map<uint64_t, uint64_t> word_tf;
    uint64_t tokens = 0;
    for (size_t d = 0; d < in; ++d)
        for (uint64_t h : word_hashes(itexts[d], ilens[d], seed, true)) {
            ++word_tf[h];
            ++tokens;
        }
    // every distinct bigram, inserted in order of first occurrence in the corpus
    std::unordered_map<uint64_t, Bigram> all;
    for (size_t d = 0; d < n; ++d) {
        const std::vector<uint64_t> w = word_hashes(texts[d], lens[d], seed, false);
        if (w.size() < 2) continue;
        m->bdl[d] = (uint32_t)(w.size() - 1);
        m->sum_bdl += w.size() - 1;
        std::vector<uint64_t> seen_order;
        std::unordered_map<uint64_t, uint32_t> tf;
        for (size_t i = 0; i + 1 < w.size(); ++i) {
            const uint64_t h = bigram(w[i], w[i + 1]);
            if (tf[h]++ == 0) seen_order.push_back(h);
            auto it = all.find(h);
            if (it == all.end()) {
                Bigram& g = all[h];
                g.a = w[i];
                g.b = w[i + 1];
            }
        }
        for (uint64_t h : seen_order) {
            Bigram& g = all[h];
            g.total_tf += tf[h];
            g.postings.emplace_back((uint32_t)d, tf[h]);
        }
    }
    m->distinct = all.size();
    for (const auto& kv : all) m->passed += kv.second.total_tf >= cfg.min_ttf;
    m->avg = n == 0 ? 0.0f : (float)((double)m->sum_bdl / (double)n);
    if (tokens == 0 || m->sum_bdl == 0) return m;
    // the PMI filter, in the map's iteration order
    std::vector<std::pair<uint64_t, float>> acc;
    const double T = (double)tokens, S = (double)m->sum_bdl;
    for (const auto& [h, g] : all) {
        if (g.total_tf < cfg.min_ttf) continue;
        const auto ia = word_tf.find(g.a), ib = word_tf.find(g.b);
        if (ia == word_tf.end() || ib == word_tf.end()) continue;
        const double ratio = ((double)g.total_tf / S) / (((double)ia->second / T) * ((double)ib->second / T));
        const double pmi = std::log(ratio);
        if (!std::isfinite(pmi) || pmi < (double)cfg.pmi_floor) continue;
        acc.emplace_back(h, (float)pmi);
    }
    m->accepted = acc.size();
    for (const auto& e : acc) m->accepted_pmi.push_back(e.second);
    std::sort(m->accepted_pmi.begin(), m->accepted_pmi.end(), [](float x, float y) { return x > y; });
    if (acc.size() > cfg.max_concepts) {
        const size_t c = cfg.max_concepts;
        m->tie_at_cap = c > 0 && m->accepted_pmi[c - 1] == m->accepted_pmi[c];
        if (cap_mode == 1) std::reverse(acc.begin(), acc.end());
        std::nth_element(acc.begin(), acc.begin() + (std::ptrdiff_t)c, acc.end(),
                         [](const std::pair<uint64_t, float>& x, const std::pair<uint64_t, float>& y) { return x.second > y.second; });
        acc.resize(c);
    }
    const float nf = (float)n;
    for (const auto& [h, pmi] : acc) {
        const Bigram& g = all.at(h);
        Concept& e = m->concepts[h];
        e.pmi = pmi;
        e.total_tf = g.total_tf;
        e.a = g.a;
        e.b = g.b;
        e.postings = g.postings;
        const float df = (float)e.postings.size();
        e.idf = std::log((nf - df + 0.5f) / (df + 0.5f) + 1.0f);
    }
    return m;
}

float atire(float tf, float dl, float idf, float k1, float b, float avg) {
    if (avg <= 0.0f) return 0.0f;
    const float denom = tf + k1 * (1.0f - b + b * dl / avg);
    return idf * tf * (k1 + 1.0f) / denom;
}

}  // namespace

extern "C" {

void* cr_mine(uint64_t seed, const char* const* itexts, const size_t* ilens, size_t in, uint32_t min_ttf, float pmi_floor,
              uint32_t max_concepts, float k1, float b, const char* const* texts, const size_t* lens, size_t n, int cap_mode) {
    return mine(seed, itexts, ilens, in, Cfg{min_ttf, pmi_floor, max_concepts, k1, b}, texts, lens, n, cap_mode);
}

// out_u: size, doc_count, sum_bdl, distinct, passed_min_ttf, accepted, tie_at_cap
void cr_stats(void* h, float* avg, uint64_t* out_u) {
    const auto* m = static_cast<Mined*>(h);
    *avg = m->avg;
    const uint64_t u[7] = {m->concepts.size(), m->n, m->sum_bdl, m->distinct, m->passed, m->accepted, m->tie_at_cap};
    std::memcpy(out_u, u, sizeof u);
}

void cr_bigram_lengths(void* h, uint32_t* out) {
    const auto* m = static_cast<Mined*>(h);
    if (!m->bdl.empty()) std::memcpy(out, m->bdl.data(), m->bdl.size() * 4);
}

void cr_accepted_pmi(void* h, float* out) {
    const auto* m = static_cast<Mined*>(h);
    if (!m->accepted_pmi.empty()) std::memcpy(out, m->accepted_pmi.data(), m->accepted_pmi.size() * 4);
}

void cr_hashes(void* h, uint64_t* out) {
    const auto* m = static_cast<Mined*>(h);
    std::vector<uint64_t> v;
    for (const auto& kv : m->concepts) v.push_back(kv.first);
    std::sort(v.begin(), v.end());
    if (!v.empty()) std::memcpy(out, v.data(), v.size() * 8);
}

// -1 when absent, else df; the first min(df, cap) postings
int64_t cr_find(void* h, uint64_t hash, float* pmi, float* idf, uint64_t* ttf_ab, uint32_t* docs, uint32_t* tfs, size_t cap) {
    const auto* m = static_cast<Mined*>(h);
    const auto it = m->concepts.find(hash);
    if (it == m->concepts.end()) return -1;
    const Concept& e = it->second;
    *pmi = e.pmi;
    *idf = e.idf;
    ttf_ab[0] = e.total_tf;
    ttf_ab[1] = e.a;
    ttf_ab[2] = e.b;
    for (size_t i = 0; i < e.postings.size() && i < cap; ++i) {
        docs[i] = e.postings[i].first;
        tfs[i] = e.postings[i].second;
    }
    return (int64_t)e.postings.size();
}

// blend_into(query, out[n], weight); order_mode 1 adds the matched concepts by ascending hash instead
void cr_blend(void* h, const char* q, size_t len, float weight, float* out, size_t n, int order_mode) {
    const auto* m = static_cast<Mined*>(h);
    if (m->concepts.empty() || n != m->n) return;
    const std::vector<uint64_t> w = word_hashes(q, len, m->seed, false);
    if (w.size() < 2) return;
    std::unordered_map<uint64_t, const Concept*> matched;
    matched.reserve(w.size());
    for (size_t i = 0; i + 1 < w.size(); ++i) {
        const uint64_t bh = bigram(w[i], w[i + 1]);
        const auto it = m->concepts.find(bh);
        if (it != m->concepts.end()) matched.emplace(bh, &it->second);
    }
    std::vector<std::pair<uint64_t, const Concept*>> order(matched.begin(), matched.end());
    if (order_mode == 1) std::sort(order.begin(), order.end());
    for (const auto& [bh, e] : order) {
        (void)bh;
        const float wpmi = weight * e->pmi;
        for (const auto& [d, tf] : e->postings)
            out[d] += wpmi * atire((float)tf, (float)m->bdl[d], e->idf, m->cfg.k1, m->cfg.b, m->avg);
    }
}

void cr_destroy(void* h) { delete static_cast<Mined*>(h); }

}  // extern "C"
