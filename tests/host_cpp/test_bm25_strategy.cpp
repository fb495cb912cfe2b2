// GPU test driver of B200Bm25Index built with the lead-text field and its score_strategy (yams_b200/host/b200_host.hpp), the
// device stand-ins for SimeonLexicalBackend's primary index with the strategy router on and its Bm25Strategy / LeadFieldStrategy.
// Reads a file: u64 n_docs and the texts, u64 n_queries and the queries (each text is u64 length + bytes).  Builds the default
// (SubwordAwareBackoff) index with add_doc for each text and lead length 64, mines concepts with min_ttf 2, and prints its
// doc_count; per query the bits of pool 0's and pool 2's scores, of pool 2's blended with weight 0.5, of pool 1's, and the routed
// pool followed by the routed scores blended with weight 0.5; then "ALL OK".
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../yams_b200/host/b200_host.hpp"

using namespace yams_b200::host;

static bool read_texts(std::FILE* f, std::vector<std::string>* out) {
    uint64_t n = 0;
    if (std::fread(&n, 8, 1, f) != 1) return false;
    for (uint64_t i = 0; i < n; ++i) {
        uint64_t len = 0;
        if (std::fread(&len, 8, 1, f) != 1) return false;
        std::string s(len, '\0');
        if (len && std::fread(s.data(), 1, len, f) != len) return false;
        out->push_back(std::move(s));
    }
    return true;
}

static void print_bits(const std::vector<float>& v) {
    for (size_t i = 0; i < v.size(); ++i) {
        uint32_t b;
        std::memcpy(&b, &v[i], 4);
        std::printf(i ? " %u" : "%u", b);
    }
    std::printf("\n");
}

int main(int argc, char** argv) {
    if (argc < 2) return 2;
    std::FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 2;
    std::vector<std::string> docs, queries;
    if (!read_texts(f, &docs) || !read_texts(f, &queries)) return 2;
    std::fclose(f);
    try {
        B200Bm25Index idx(nullptr, 64);
        for (const auto& d : docs) idx.add_doc(d);
        idx.finalize();
        yams_concept_config ccfg;
        yams_b200_concepts_default_config(&ccfg);
        ccfg.min_ttf = 2;
        std::vector<std::string_view> views(docs.begin(), docs.end());
        B200ConceptIndex concepts = mine_concepts(idx, views, ccfg);
        std::printf("%u\n", idx.doc_count());
        std::vector<float> s(idx.doc_count());
        for (const auto& q : queries) {
            idx.score_strategy(YAMS_BM25_STRATEGY_BM25, q, s);
            print_bits(s);
            idx.score_strategy(YAMS_BM25_STRATEGY_LEAD_FIELD, q, s);
            print_bits(s);
            idx.score_strategy(YAMS_BM25_STRATEGY_LEAD_FIELD, q, s, &concepts, 0.5f);
            print_bits(s);
            idx.score_strategy(YAMS_BM25_STRATEGY_KEYPHRASE, q, s);
            print_bits(s);
            std::printf("%u ", idx.score_strategy_routed(q, s, &concepts, 0.5f));
            print_bits(s);
        }
        bool threw = false;
        try {
            idx.score_strategy(4, queries.empty() ? std::string() : queries[0], s);
        } catch (const std::runtime_error&) {
            threw = true;
        }
        if (!threw) return 1;
    } catch (const std::exception& e) {
        std::printf("error: %s\n", e.what());
        return 1;
    }
    std::printf("ALL OK\n");
    return 0;
}
