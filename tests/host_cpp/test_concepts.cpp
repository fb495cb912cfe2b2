// GPU test driver of B200ConceptIndex and mine_concepts (yams_b200/host/b200_host.hpp), the device stand-ins for
// simeon::ConceptIndex in SimeonLexicalBackend.  Reads a file: u64 n_docs and the texts, u64 n_queries and the queries (each text
// is u64 length + bytes), then u64 count and that many concept hashes.  Mines with min_ttf 2 and prints size, doc_count and
// avg_dl bits; per query the bits of score(query, &concepts, 0.5) (BM25 + blend) and then of ConceptIndex::score (the blend
// alone, weight 1, into zeros); per hash "found pmi_bits idf_bits total_tf df"; then "ALL OK".
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

int main(int argc, char** argv) {
    if (argc != 2) return 2;
    std::FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 2;
    std::vector<std::string> docs, queries;
    uint64_t nh = 0;
    bool ok = read_texts(f, &docs) && read_texts(f, &queries) && std::fread(&nh, 8, 1, f) == 1;
    std::vector<uint64_t> hashes(nh);
    ok = ok && (nh == 0 || std::fread(hashes.data(), 8, nh, f) == nh);
    std::fclose(f);
    if (!ok) return 2;
    B200Bm25Index ix;
    for (const auto& d : docs) ix.add_doc(d);
    ix.finalize();
    std::vector<std::string_view> views(docs.begin(), docs.end());
    yams_concept_config cfg;
    yams_b200_concepts_default_config(&cfg);
    cfg.min_ttf = 2;
    const B200ConceptIndex ci = mine_concepts(ix, views, cfg);
    std::printf("%u %u %u\n", ci.size(), ci.doc_count(), bits(ci.avg_dl()));
    std::vector<float> out(ix.doc_count());
    for (const auto& q : queries) {
        ix.score(q, out, &ci, 0.5f);
        for (float v : out) std::printf("%u ", bits(v));
        std::printf("\n");
        std::fill(out.begin(), out.end(), 0.0f);
        ci.score(q, out);
        for (float v : out) std::printf("%u ", bits(v));
        std::printf("\n");
    }
    for (uint64_t h : hashes) {
        const auto e = ci.find(h);
        if (e)
            std::printf("1 %u %u %llu %zu\n", bits(e->pmi), bits(e->idf), (unsigned long long)e->total_tf, e->docs.size());
        else
            std::printf("0 0 0 0 0\n");
    }
    std::printf("ALL OK\n");
    return 0;
}
