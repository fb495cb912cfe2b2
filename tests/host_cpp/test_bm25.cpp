// GPU test driver of B200Bm25Index (yams_b200/host/b200_host.hpp), the device stand-in for simeon::Bm25Index in
// SimeonLexicalBackend.  Reads a file: u32 variant, u64 n_docs, then n_docs texts, u64 n_queries, then the queries (each text is
// u64 length + bytes), and a u64 count of raw terms with their bytes.  Prints doc_count, avg_dl bits, total_tokens, every
// doc_length, the score bits of every query (one line each), df / idf bits / total_tf of every raw term, then "ALL OK".
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
    uint32_t variant = 0;
    std::vector<std::string> docs, queries, terms;
    const bool ok = std::fread(&variant, 4, 1, f) == 1 && read_texts(f, &docs) && read_texts(f, &queries) && read_texts(f, &terms);
    std::fclose(f);
    if (!ok) return 2;
    yams_bm25_config cfg;
    yams_b200_bm25_default_config(&cfg);
    cfg.variant = variant;
    B200Bm25Index ix(&cfg);
    for (const auto& d : docs) ix.add_doc(d);
    std::vector<float> early(docs.size());
    try {
        ix.score("x", early);   // before finalize(): the reference throws
        std::fprintf(stderr, "score before finalize did not throw\n");
        return 1;
    } catch (const std::runtime_error&) {
    }
    ix.finalize();
    std::printf("%u %u %llu\n", ix.doc_count(), bits(ix.avg_dl()), (unsigned long long)ix.total_tokens());
    for (uint32_t d = 0; d < ix.doc_count(); ++d) std::printf("%u ", ix.doc_length(d));
    std::printf("\n");
    std::vector<float> out(ix.doc_count());
    for (const auto& q : queries) {
        ix.score(q, out);
        for (float v : out) std::printf("%u ", bits(v));
        std::printf("\n");
    }
    for (const auto& t : terms)
        std::printf("%u %u %llu\n", ix.df(t), bits(ix.idf(t)), (unsigned long long)ix.total_tf(t));
    try {
        ix.add_doc("late");
        std::fprintf(stderr, "add_doc after finalize did not throw\n");
        return 1;
    } catch (const std::runtime_error&) {
    }
    std::printf("ALL OK\n");
    return 0;
}
