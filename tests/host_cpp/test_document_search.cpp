// GPU test of B200VectorStore::searchDocumentCandidates (yams_b200/host/b200_host.hpp), the IDocumentCandidateVectorStore seam
// that CandidateFilterMode::DocumentTopK reaches (/root/reference/src/vector/vector_database.cpp:553-569): documents ordered by
// (best score desc, document_hash asc), each represented by its best chunk (score desc, chunk_id asc), string keys whose order
// differs from rowid order.  Prints "ALL OK" on success.
#include <cstdio>
#include <cstdlib>

#include "../../yams_b200/host/b200_host.hpp"

using namespace yams_b200::host;

#define CHECK(cond)                                                                  \
    do {                                                                             \
        if (!(cond)) {                                                               \
            std::fprintf(stderr, "CHECK failed %s:%d: %s\n", __FILE__, __LINE__, #cond); \
            std::exit(1);                                                            \
        }                                                                            \
    } while (0)

int main() {
    if (yams_plugin_init("{}", nullptr) != YAMS_PLUGIN_OK) {
        std::fprintf(stderr, "plugin init failed: %s\n", yams_b200_last_error());
        return 2;
    }
    B200VectorStore store(4);
    const std::vector<float> A = {1.f, 2.f, 3.f, 4.f}, B = {4.f, -1.f, 0.5f, 1.f}, Z = {0.f, 0.f, 0.f, 0.f};
    std::vector<float> rows;
    for (const auto* v : {&A, &A, &A, &B, &Z, &A, &B}) rows.insert(rows.end(), v->begin(), v->end());
    // rowid:              10       11       12       13       14       15       16
    const std::vector<int64_t> rowids = {10, 11, 12, 13, 14, 15, 16};
    const std::vector<std::string> chunks = {"b-2", "b-10", "a-1", "c-1", "z-1", "x-1", "c-0"};
    const std::vector<std::string> docs = {"doc-b", "doc-b", "doc-a", "doc-c", "doc-z", "doc-x", "doc-c"};
    store.insertVectorsBatch(rows, rowids, chunks, docs);

    // doc-a and doc-b tie on score: doc-a first (hash order); inside doc-b the identical rows tie: chunk "b-10" < "b-2" wins
    // although its rowid is larger; doc-c's two identical rows: "c-0" (rowid 16) wins; doc-z (zero row) and the unknown hash
    // are absent; doc-x is not a candidate
    const std::unordered_set<std::string> cand = {"doc-c", "doc-b", "doc-z", "doc-a", "doc-missing"};
    VectorSearchDiagnostics diag;
    auto hits = store.searchDocumentCandidates(A, 10, -1.0f, cand, nullptr, &diag);
    CHECK(hits.size() == 3);
    CHECK(hits[0].document_hash == "doc-a" && hits[0].rowid == 12 && hits[0].chunk_id == "a-1");
    CHECK(hits[1].document_hash == "doc-b" && hits[1].rowid == 11 && hits[1].chunk_id == "b-10");
    CHECK(hits[2].document_hash == "doc-c" && hits[2].rowid == 16 && hits[2].chunk_id == "c-0");
    CHECK(hits[0].relevance_score == hits[1].relevance_score && hits[1].relevance_score > hits[2].relevance_score);
    CHECK(diag.returnedRows == 3 && diag.rowsVisited == 6);
    auto top1 = store.searchDocumentCandidates(A, 1, -1.0f, cand);
    CHECK(top1.size() == 1 && top1[0].document_hash == "doc-a");
    CHECK(store.searchDocumentCandidates(A, 0, -1.0f, cand).empty());
    auto above = store.searchDocumentCandidates(A, 10, hits[2].relevance_score + 1e-3f, cand);
    CHECK(above.size() == 2);

    bool threw = false;
    try { store.searchDocumentCandidates(A, 10, -1.0f, {}); } catch (const std::invalid_argument&) { threw = true; }
    CHECK(threw);   // vector_database.cpp:554-557
    threw = false;
    try { store.searchDocumentCandidates(Z, 10, -1.0f, cand); } catch (const std::invalid_argument&) { threw = true; }
    CHECK(threw);   // the exact fallback rejects a zero query

    // the hits of the row-level search carry document_hash too
    auto sim = store.searchSimilar(B, 2, -1.0f);
    CHECK(sim.size() == 2 && sim[0].document_hash == "doc-c" && sim[0].chunk_id == "c-0");
    std::printf("ALL OK\n");
    return 0;
}
