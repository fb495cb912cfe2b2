// GPU test driver of B200Bm25Index::atire_view and score_bm25_variants_rrf (yams_b200/host/b200_host.hpp), the device stand-ins
// for SimeonLexicalBackend's Atire index and simeon::score_bm25_variants_rrf.  Reads a file: u64 n_docs and the texts, u64
// n_queries and the queries (each text is u64 length + bytes).  Builds the default (SubwordAwareBackoff) index, its Atire view
// and concepts mined with min_ttf 2, destroys the primary only after the view's first use, and prints the view's doc_count and
// avg_dl bits; per query the bits of the view's score, of score_bm25_variants_rrf({primary, view}) and of the blended overload
// (weight 0.5); then "ALL OK".
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

static uint32_t bits(float x) {
    uint32_t b;
    std::memcpy(&b, &x, 4);
    return b;
}

static void print(const std::vector<float>& v) {
    for (float x : v) std::printf("%u ", bits(x));
    std::printf("\n");
}

int main(int argc, char** argv) {
    if (argc != 2) return 2;
    std::FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 2;
    std::vector<std::string> docs, queries;
    const bool ok = read_texts(f, &docs) && read_texts(f, &queries);
    std::fclose(f);
    if (!ok) return 2;
    auto primary = std::make_unique<B200Bm25Index>();
    for (const auto& d : docs) primary->add_doc(d);
    primary->finalize();
    const std::unique_ptr<B200Bm25Index> atire = primary->atire_view();
    std::vector<std::string_view> views(docs.begin(), docs.end());
    yams_concept_config cfg;
    yams_b200_concepts_default_config(&cfg);
    cfg.min_ttf = 2;
    const B200ConceptIndex ci = mine_concepts(*primary, views, cfg);
    std::printf("%u %u\n", atire->doc_count(), bits(atire->avg_dl()));
    std::vector<float> out(atire->doc_count());
    try {   // a span of the wrong size throws, as the reference's score does
        std::vector<float> bad(out.size() + 1);
        const B200Bm25Index* v[1] = {primary.get()};
        score_bm25_variants_rrf(v, "x", bad);
        return 3;
    } catch (const std::runtime_error&) {
    }
    for (size_t i = 0; i < queries.size(); ++i) {
        atire->score(queries[i], out);
        print(out);
        const B200Bm25Index* variants[2] = {primary.get(), atire.get()};
        score_bm25_variants_rrf(variants, queries[i], out);
        print(out);
        score_bm25_variants_rrf(variants, queries[i], out, &ci, 0.5f);
        print(out);
    }
    primary.reset();   // the view keeps the word field
    atire->score(queries.empty() ? std::string_view() : std::string_view(queries[0]), out);
    print(out);
    std::printf("ALL OK\n");
    return 0;
}
