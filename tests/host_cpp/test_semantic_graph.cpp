// GPU test of B200SemanticGraph::neighbors (yams_b200/host/b200_host.hpp), the call that replaces the pair loop of
// EmbeddingService::updateSemanticNeighborGraphUnlocked: first record per hash, hash order, zero-norm documents skipped,
// adaptive and explicit thresholds, the reference's similarity bits, and mixed dimensions refused.  Prints "ALL OK" on success.
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

// EmbeddingService.cpp:405-431
static float inverseNorm(const std::vector<float>& v) {
    double norm = 0.0;
    for (float x : v) norm += (double)x * (double)x;
    return norm <= 0.0 ? 0.0f : (float)(1.0 / std::sqrt(norm));
}
static float cosine(const std::vector<float>& a, const std::vector<float>& b) {
    double dot = 0.0;
    for (size_t i = 0; i < a.size(); ++i) dot += (double)a[i] * (double)b[i];
    return (float)(dot * inverseNorm(a) * inverseNorm(b));
}

int main() {
    if (yams_plugin_init("{}", nullptr) != YAMS_PLUGIN_OK) {
        std::fprintf(stderr, "plugin init failed: %s\n", yams_b200_last_error());
        return 2;
    }
    const std::vector<float> A = {1.f, 0.1f}, B = {0.9f, 0.5f}, Cv = {1.f, 0.f}, D = {0.f, 1.f}, F = {-1.f, 0.f};
    const std::vector<SemanticDoc> docs = {{"c", Cv}, {"a", A}, {"f", F}, {"b", B}, {"a", F}, {"e", {0.f, 0.f}}, {"d", D}, {"", A}};
    std::vector<std::pair<std::string, B200SemanticGraph::Neighbors>> out;

    // streaming form, adaptive: c's neighbours are a then b (d scores 0, f below 0: dropped)
    CHECK(B200SemanticGraph::neighbors(docs, {"c", "zz"}, 8, std::nullopt, &out) == YAMS_OK);
    CHECK(out.size() == 1 && out[0].first == "c" && out[0].second.size() == 2);
    CHECK(out[0].second[0].first == "a" && out[0].second[0].second == cosine(Cv, A));
    CHECK(out[0].second[1].first == "b" && out[0].second[1].second == cosine(Cv, B));

    // explicit threshold 0.9 keeps a only; a threshold above 1 is clamped to 1
    CHECK(B200SemanticGraph::neighbors(docs, {"c"}, 8, 0.9f, &out) == YAMS_OK);
    CHECK(out.size() == 1 && out[0].second.size() == 1 && out[0].second[0].first == "a");
    CHECK(B200SemanticGraph::neighbors(docs, {"c"}, 8, 7.f, &out) == YAMS_OK);
    CHECK(out.size() == 1 && out[0].second.empty());

    // the rebuild: every document with a positive norm, in hash order (e is skipped; a is the first record of "a")
    CHECK(B200SemanticGraph::neighbors(docs, {}, 1, std::nullopt, &out) == YAMS_OK);
    CHECK(out.size() == 5);
    const char* order[] = {"a", "b", "c", "d", "f"};
    for (size_t i = 0; i < 5; ++i) CHECK(out[i].first == order[i]);
    CHECK(out[0].second.size() == 1 && out[0].second[0].first == "c");
    CHECK(out[3].second.size() == 1 && out[3].second[0].first == "b" && out[3].second[0].second == cosine(D, B));
    CHECK(out[4].second.empty());   // f = -c: every similarity is <= 0

    // more than one dimension: the daemon keeps its own loop
    const std::vector<SemanticDoc> mixed = {{"a", A}, {"b", {1.f, 2.f, 3.f}}};
    CHECK(B200SemanticGraph::neighbors(mixed, {}, 8, std::nullopt, &out) == YAMS_ERR_UNSUPPORTED);
    std::printf("ALL OK\n");
    return 0;
}
