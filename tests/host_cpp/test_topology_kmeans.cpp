// GPU test driver of B200TopologyKMeans::assign (yams_b200/host/b200_host.hpp), the call that replaces runKMeans in
// KMeansTopologyEngine::buildArtifacts.  Reads documents from a file: u64 n, u32 stride, u64 k, u64 max_iterations,
// u32 dims[n], f32 rows[n][stride] (document i's embedding is its first dims[i] values; 0 = none), and prints the assignment
// vector, one value per line, then "ALL OK".
#include <cstdio>
#include <cstdlib>

#include "../../yams_b200/host/b200_host.hpp"

using namespace yams_b200::host;

int main(int argc, char** argv) {
    if (argc != 2) return 2;
    std::FILE* f = std::fopen(argv[1], "rb");
    if (!f) return 2;
    uint64_t n = 0, k = 0, iters = 0;
    uint32_t stride = 0;
    bool ok = std::fread(&n, 8, 1, f) == 1 && std::fread(&stride, 4, 1, f) == 1 && std::fread(&k, 8, 1, f) == 1 &&
              std::fread(&iters, 8, 1, f) == 1;
    std::vector<uint32_t> dims(n);
    std::vector<float> rows(n * stride);
    ok = ok && std::fread(dims.data(), 4, n, f) == n && std::fread(rows.data(), 4, n * stride, f) == n * stride;
    std::fclose(f);
    if (!ok) return 2;
    std::vector<std::span<const float>> embeddings;
    for (uint64_t i = 0; i < n; ++i) embeddings.emplace_back(rows.data() + i * stride, dims[i]);
    std::vector<int64_t> assignment;
    const yams_status_t st = B200TopologyKMeans::assign(embeddings, k, iters, &assignment);
    if (st != YAMS_OK || assignment.size() != n) {
        std::fprintf(stderr, "assign: status %d, %zu values\n", st, assignment.size());
        return 1;
    }
    for (int64_t v : assignment) std::printf("%lld\n", (long long)v);
    std::printf("ALL OK\n");
    return 0;
}
