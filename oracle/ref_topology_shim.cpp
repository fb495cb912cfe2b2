// ref_topology_shim.cpp -- C entry into the reference's own KMeansTopologyEngine (topology_alternate_engines.cpp), compiled
// with it by oracle/topology_kmeans.mk into oracle/_ref/libref_topology_kmeans.so.  Test infrastructure only.
//
// buildArtifacts names its clusters by anchor hashes, so the shim returns the partition: label[i] = the rank of document i's
// cluster in order of first appearance (document order).  Documents get hashes "d%010zu", so hash order is document order.
#include <cstdint>
#include <cstdio>
#include <string>
#include <unordered_map>
#include <vector>

#include <yams/topology/topology_alternate_engines.h>

extern "C" int ref_topology_kmeans_partition(const float* rows, const uint32_t* dims, uint64_t n, uint32_t stride, uint64_t k,
                                             uint64_t max_iterations, int64_t* out_label) {
    using namespace yams::topology;
    std::vector<TopologyDocumentInput> docs(n);
    for (uint64_t i = 0; i < n; ++i) {
        char hash[32];
        std::snprintf(hash, sizeof hash, "d%010llu", (unsigned long long)i);
        docs[i].documentHash = hash;
        docs[i].embedding.assign(rows + i * stride, rows + i * stride + dims[i]);
    }
    TopologyBuildConfig cfg;
    cfg.kmeansK = k;
    cfg.kmeansMaxIterations = max_iterations;
    KMeansTopologyEngine engine;
    auto r = engine.buildArtifacts(docs, cfg);
    if (!r) return 1;
    std::unordered_map<std::string, uint64_t> index;
    for (uint64_t i = 0; i < n; ++i) index[docs[i].documentHash] = i;
    std::vector<std::string> cluster_of(n);
    for (const auto& m : r.value().memberships) cluster_of[index.at(m.documentHash)] = m.clusterId;
    std::unordered_map<std::string, int64_t> rank;
    for (uint64_t i = 0; i < n; ++i) {
        if (cluster_of[i].empty()) return 2;   // every document is a member of one cluster
        out_label[i] = rank.emplace(cluster_of[i], (int64_t)rank.size()).first->second;
    }
    return 0;
}
