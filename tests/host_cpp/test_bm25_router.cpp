// GPU test driver of B200Bm25Index::score_routed and router_features (yams_b200/host/b200_host.hpp), the device stand-ins for
// SimeonLexicalBackend::scoreRouted with router_enabled: no CPU index and no QueryRouter.  Reads a file: u64 n_docs and the
// texts, u64 n_queries and the queries (each text is u64 length + bytes).  Builds the default (SubwordAwareBackoff) index with
// add_doc for each text, mines concepts with min_ttf 2, and prints its doc_count; per query the recipe followed by the bits of the
// routed scores blended with weight 0.5, the recipe followed by the bits of the same scores projected onto a fixed candidate
// pool (documents 7j mod n for j < 40, then NOT_INDEXED, 3, 3), and the features (n_terms as is, the others' float bits); then
// "ALL OK".
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

static void print_bits(const float* v, size_t n) {
    for (size_t i = 0; i < n; ++i) {
        uint32_t b;
        std::memcpy(&b, &v[i], 4);
        std::printf(" %u", b);
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
        B200Bm25Index idx;
        for (const auto& d : docs) idx.add_doc(d);
        idx.finalize();
        yams_concept_config ccfg;
        yams_b200_concepts_default_config(&ccfg);
        ccfg.min_ttf = 2;
        std::vector<std::string_view> views(docs.begin(), docs.end());
        B200ConceptIndex concepts = mine_concepts(idx, views, ccfg);
        std::printf("%u\n", idx.doc_count());
        std::vector<uint32_t> cands;
        for (uint32_t j = 0; j < 40; ++j) cands.push_back((7 * j) % idx.doc_count());
        cands.insert(cands.end(), {B200Bm25Index::NOT_INDEXED, 3, 3});
        std::vector<float> s(idx.doc_count()), pool(cands.size());
        for (const auto& q : queries) {
            std::printf("%u", idx.score_routed(q, s, &concepts, 0.5f));
            print_bits(s.data(), s.size());
            std::printf("%u", idx.score_routed(q, cands, pool, &concepts, 0.5f));
            print_bits(pool.data(), pool.size());
            const yams_bm25_query_features ft = idx.router_features(q);
            const float fs[8] = {ft.oov_rate, ft.avg_idf, ft.max_idf, ft.min_idf, ft.idf_stddev, ft.avg_term_chars, ft.scq_sum,
                                 ft.simplified_clarity};
            uint32_t b[8];
            std::memcpy(b, fs, sizeof b);
            std::printf("%u %u %u %u %u %u %u %u %u\n", b[0], b[1], b[2], b[3], b[4], ft.n_terms, b[5], b[6], b[7]);
        }
        bool threw = false;
        try {
            const uint32_t bad[1] = {idx.doc_count()};
            float o[1];
            idx.score_routed(queries.empty() ? std::string() : queries[0], std::span<const uint32_t>(bad, 1), std::span<float>(o, 1));
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
