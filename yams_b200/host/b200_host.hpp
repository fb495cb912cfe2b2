// b200_host.hpp -- C++ host-side mirror of the reference's operator interfaces for the hot path, written
// ONLY against the C ABI (include/yams_b200.h).  A YAMS maintainer would derive these from the real
// IChunker / IContentHasher / IVectorStore (INTEGRATION.md); here they are self-contained so they build without
// the YAMS tree, keeping the reference's member names, argument meaning and error behaviour:
//   IChunker         /root/reference/include/yams/chunking/chunker.h:65-92   (Chunk: :18-31, ChunkingConfig: :44-51)
//   IContentHasher   /root/reference/include/yams/crypto/hasher.h:14-46      (hex: src/crypto/sha256_hasher.cpp:19-30)
//   IVectorStore     /root/reference/include/yams/vector/vector_store.h:44-53, :121-138
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <fstream>
#include <filesystem>
#include <span>
#include <stdexcept>
#include <algorithm>
#include <cmath>
#include <limits>
#include <map>
#include <memory>
#include <optional>
#include <string>
#include <string_view>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "../../include/yams_b200.h"

namespace yams_b200::host {

using Hash = std::string;  // core/types.h:17

struct Chunk {  // chunker.h:18-31
    std::vector<std::byte> data;
    Hash hash;
    size_t offset = 0;
    size_t size = 0;
};

struct ChunkingConfig {  // chunker.h:44-51 (defaults: core/types.h:280-285)
    size_t windowSize = 48;
    size_t minChunkSize = 16 * 1024;
    size_t targetChunkSize = 256 * 1024;
    size_t maxChunkSize = 1024 * 1024;
    uint64_t polynomial = 0x3DA3358B4DC173ULL;
    uint64_t chunkMask = 0x1FFF;
};

inline std::string bytesToHex(const uint8_t* d, size_t n) {  // sha256_hasher.cpp:19-30
    static constexpr char kHex[] = "0123456789abcdef";
    std::string out(n * 2, '\0');
    for (size_t i = 0; i < n; ++i) {
        out[2 * i] = kHex[(d[i] >> 4) & 0xF];
        out[2 * i + 1] = kHex[d[i] & 0xF];
    }
    return out;
}

inline void throw_status(const char* what, yams_status_t st) {
    throw std::runtime_error(std::string(what) + " failed (status " + std::to_string(st) + "): " + yams_b200_last_error());
}

// IChunker over the GPU.  variant: YAMS_CDC_STREAMING mirrors StreamingChunker (what ContentStore uses,
// src/api/content_store_builder.cpp:152-165), YAMS_CDC_RABIN mirrors RabinChunker.
class B200Chunker {
public:
    explicit B200Chunker(ChunkingConfig config = {}, int variant = YAMS_CDC_STREAMING) : config_(config), variant_(variant) {}
    const ChunkingConfig& getConfig() const { return config_; }

    std::vector<Chunk> chunkData(std::span<const std::byte> data) { return run(data, false); }
    std::vector<Chunk> chunkDataLazy(std::span<const std::byte> data) { return run(data, true); }

    // Many buffers in one device pass (`yams add -r`): result[i] == chunkDataLazy(buffers[i]).
    std::vector<std::vector<Chunk>> chunkManyLazy(const std::vector<std::span<const std::byte>>& buffers) {
        std::vector<const uint8_t*> ptrs(buffers.size());
        std::vector<size_t> lens(buffers.size());
        for (size_t i = 0; i < buffers.size(); ++i) {
            ptrs[i] = reinterpret_cast<const uint8_t*>(buffers[i].data());
            lens[i] = buffers[i].size();
        }
        std::vector<uint64_t> first(buffers.size() + 1, 0);
        yams_cdc_config c = cfg();
        yams_chunk_desc* d = nullptr;
        size_t n = 0;
        yams_status_t st = yams_b200_chunk_and_hash_batch(nullptr, ptrs.data(), lens.data(), buffers.size(), &c, &d, &n, first.data());
        if (st != YAMS_OK) throw_status("chunk_and_hash_batch", st);
        std::vector<std::vector<Chunk>> out(buffers.size());
        static const std::vector<std::byte> none;
        for (size_t i = 0; i < buffers.size(); ++i) append(out[i], d + first[i], (size_t)(first[i + 1] - first[i]), none, true);
        yams_b200_free_chunks(nullptr, d, n);
        return out;
    }

    // streaming_chunker.cpp:71-90 / streaming_chunker.h:78-121: 64 KiB reads fed to a session
    std::vector<Chunk> chunkFile(const std::filesystem::path& path) {
        std::ifstream file(path, std::ios::binary);
        if (!file) throw std::runtime_error("Failed to open file: " + path.string());  // rabin_chunker.cpp:156-158
        yams_cdc_config c = cfg();
        yams_b200_ingest* s = nullptr;
        yams_status_t st = yams_b200_ingest_open(nullptr, &c, &s);
        if (st != YAMS_OK) throw_status("ingest_open", st);
        std::vector<Chunk> chunks;
        std::vector<std::byte> whole;  // Chunk::data is filled from the bytes read (non-lazy contract of chunkFile)
        std::vector<char> buf(1 << 22);
        try {
            for (;;) {
                file.clear();
                file.read(buf.data(), (std::streamsize)buf.size());
                std::streamsize got = file.gcount();
                if (got <= 0) break;
                whole.insert(whole.end(), reinterpret_cast<std::byte*>(buf.data()), reinterpret_cast<std::byte*>(buf.data()) + got);
                yams_chunk_desc* d = nullptr;
                size_t n = 0;
                st = yams_b200_ingest_feed(s, reinterpret_cast<const uint8_t*>(buf.data()), (size_t)got, &d, &n);
                if (st != YAMS_OK) throw_status("ingest_feed", st);
                append(chunks, d, n, whole, false);
                yams_b200_free_chunks(nullptr, d, n);
            }
            yams_chunk_desc* d = nullptr;
            size_t n = 0;
            st = yams_b200_ingest_finish(s, &d, &n);
            if (st != YAMS_OK) throw_status("ingest_finish", st);
            append(chunks, d, n, whole, false);
            yams_b200_free_chunks(nullptr, d, n);
        } catch (...) {
            yams_b200_ingest_close(s);
            throw;
        }
        yams_b200_ingest_close(s);
        return chunks;
    }

private:
    yams_cdc_config cfg() const {
        yams_cdc_config c{};
        c.window_size = config_.windowSize;
        c.min_chunk = config_.minChunkSize;
        c.max_chunk = config_.maxChunkSize;
        c.polynomial = config_.polynomial;
        c.mask = config_.chunkMask;
        c.variant = variant_;
        return c;
    }
    static void append(std::vector<Chunk>& out, const yams_chunk_desc* d, size_t n, const std::vector<std::byte>& bytes, bool lazy) {
        for (size_t i = 0; i < n; ++i) {
            Chunk ch;
            ch.offset = (size_t)d[i].offset;
            ch.size = (size_t)d[i].size;
            ch.hash = bytesToHex(d[i].digest, 32);
            if (!lazy) ch.data.assign(bytes.begin() + (ptrdiff_t)ch.offset, bytes.begin() + (ptrdiff_t)(ch.offset + ch.size));
            out.push_back(std::move(ch));
        }
    }
    std::vector<Chunk> run(std::span<const std::byte> data, bool lazy) {
        yams_cdc_config c = cfg();
        yams_chunk_desc* d = nullptr;
        size_t n = 0;
        yams_status_t st = yams_b200_chunk_and_hash(nullptr, reinterpret_cast<const uint8_t*>(data.data()), data.size(), &c, &d, &n);
        if (st != YAMS_OK) throw_status("chunk_and_hash", st);
        std::vector<Chunk> out;
        out.reserve(n);
        for (size_t i = 0; i < n; ++i) {
            Chunk ch;
            ch.offset = (size_t)d[i].offset;
            ch.size = (size_t)d[i].size;
            ch.hash = bytesToHex(d[i].digest, 32);
            if (!lazy) ch.data.assign(data.begin() + (ptrdiff_t)ch.offset, data.begin() + (ptrdiff_t)(ch.offset + ch.size));
            out.push_back(std::move(ch));
        }
        yams_b200_free_chunks(nullptr, d, n);
        return out;
    }
    ChunkingConfig config_;
    int variant_;
};

// DeduplicationStats / calculateDeduplication (chunker.h:204-218, rabin_chunker.cpp:224-239)
struct DeduplicationStats {
    size_t totalSize = 0, uniqueSize = 0, chunkCount = 0, uniqueChunks = 0;
    double getRatio() const { return totalSize == 0 ? 0.0 : 1.0 - static_cast<double>(uniqueSize) / static_cast<double>(totalSize); }
};
inline DeduplicationStats calculateDeduplication(const std::vector<Chunk>& chunks) {
    std::vector<yams_chunk_desc> d(chunks.size());
    for (size_t i = 0; i < chunks.size(); ++i) {
        d[i].offset = chunks[i].offset;
        d[i].size = chunks[i].size;
        for (int b = 0; b < 32; ++b) d[i].digest[b] = (uint8_t)std::stoi(chunks[i].hash.substr(2 * b, 2), nullptr, 16);
    }
    yams_dedup_stats st{};
    yams_status_t rc = yams_b200_dedup_stats(nullptr, d.data(), d.size(), &st);
    if (rc != YAMS_OK) throw_status("dedup_stats", rc);
    return DeduplicationStats{(size_t)st.total_size, (size_t)st.unique_size, (size_t)st.chunk_count, (size_t)st.unique_chunks};
}

// IContentHasher: init / update / finalize accumulate on the host side (the digest of ONE message is a serial
// chain; the GPU earns its keep when many messages are hashed at once -> hashMany).
class B200ContentHasher {
public:
    void init() { buf_.clear(); }
    void update(std::span<const std::byte> data) { buf_.insert(buf_.end(), data.begin(), data.end()); }
    std::string finalize() {
        std::string h = hash(std::span<const std::byte>(buf_.data(), buf_.size()));
        buf_.clear();  // sha256_hasher.cpp:104: finalize re-initialises
        return h;
    }
    static std::string hash(std::span<const std::byte> data) {  // sha256_hasher.cpp:167-195
        uint64_t off = 0, sz = data.size();
        uint8_t dg[32];
        yams_status_t st = yams_b200_sha256_batch(nullptr, reinterpret_cast<const uint8_t*>(data.data()), data.size(), &off, &sz, 1, dg);
        if (st != YAMS_OK) throw_status("sha256_batch", st);
        return bytesToHex(dg, 32);
    }
    static std::vector<std::string> hashMany(std::span<const std::byte> base, const std::vector<uint64_t>& offsets,
                                             const std::vector<uint64_t>& sizes) {
        std::vector<uint8_t> dg(offsets.size() * 32);
        yams_status_t st = yams_b200_sha256_batch(nullptr, reinterpret_cast<const uint8_t*>(base.data()), base.size(), offsets.data(),
                                                  sizes.data(), offsets.size(), dg.data());
        if (st != YAMS_OK) throw_status("sha256_batch", st);
        std::vector<std::string> out(offsets.size());
        for (size_t i = 0; i < offsets.size(); ++i) out[i] = bytesToHex(dg.data() + 32 * i, 32);
        return out;
    }

    // separately held spans (no common base buffer): one device pass
    static std::vector<std::string> hashSpans(const std::vector<std::span<const std::byte>>& spans) {
        std::vector<const uint8_t*> ptrs(spans.size());
        std::vector<size_t> lens(spans.size());
        for (size_t i = 0; i < spans.size(); ++i) {
            ptrs[i] = reinterpret_cast<const uint8_t*>(spans[i].data());
            lens[i] = spans[i].size();
        }
        std::vector<uint8_t> dg(spans.size() * 32);
        yams_status_t st = yams_b200_sha256_many(nullptr, ptrs.data(), lens.data(), spans.size(), dg.data());
        if (st != YAMS_OK) throw_status("sha256_many", st);
        std::vector<std::string> out(spans.size());
        for (size_t i = 0; i < spans.size(); ++i) out[i] = bytesToHex(dg.data() + 32 * i, 32);
        return out;
    }

    // IContentHasher::hashFile (src/crypto/sha256_hasher.cpp:111-150): same error behaviour (std::runtime_error when the file cannot be
    // opened).  One file is one SHA-256 lane on the device (~80 MB/s): use hashFiles for more than a handful, it hashes all of
    // them in one pass.
    static std::string hashFile(const std::filesystem::path& path) { return hashFiles({path}).front(); }
    static std::vector<std::string> hashFiles(const std::vector<std::filesystem::path>& paths) {
        std::vector<std::vector<std::byte>> bufs(paths.size());
        std::vector<std::span<const std::byte>> spans(paths.size());
        for (size_t i = 0; i < paths.size(); ++i) {
            std::ifstream f(paths[i], std::ios::binary);
            if (!f) throw std::runtime_error("Failed to open file: " + paths[i].string());
            f.seekg(0, std::ios::end);
            const std::streamoff n = f.tellg();
            f.seekg(0, std::ios::beg);
            bufs[i].resize(n > 0 ? (size_t)n : 0);
            if (n > 0) f.read(reinterpret_cast<char*>(bufs[i].data()), n);
            spans[i] = std::span<const std::byte>(bufs[i].data(), bufs[i].size());
        }
        return hashSpans(spans);
    }

private:
    std::vector<std::byte> buf_;
};

// ChunkValidator::validateChunks (src/integrity/chunk_validator.cpp:173-213): every chunk is re-hashed and compared
// with the hash it is stored under.  One device pass instead of maxParallelValidations worker threads.
struct ChunkValidationResult {   // include/yams/integrity/chunk_validator.h (fields used by callers)
    std::string chunkHash;
    bool isValid = false;
    std::string errorMessage;
    size_t chunkSize = 0;
};
inline std::vector<ChunkValidationResult> validateChunks(const std::vector<std::pair<std::span<const std::byte>, std::string>>& chunks) {
    std::vector<std::span<const std::byte>> spans;
    spans.reserve(chunks.size());
    for (const auto& c : chunks) spans.push_back(c.first);
    auto actual = B200ContentHasher::hashSpans(spans);
    std::vector<ChunkValidationResult> out(chunks.size());
    for (size_t i = 0; i < chunks.size(); ++i) {
        out[i].chunkHash = chunks[i].second;
        out[i].chunkSize = chunks[i].first.size();
        out[i].isValid = actual[i] == chunks[i].second;
        if (!out[i].isValid) out[i].errorMessage = "Hash mismatch: expected " + chunks[i].second + ", got " + actual[i];
    }
    return out;
}

// The part of IVectorStore the hot path covers.  Records live in SQLite in the real backend; here a record is
// (rowid, chunk_id, document_hash, metadata) and `relevance_score` -- enough to express the WHERE clause of
// bruteForceSearchUnlocked (sqlite_vec_backend.cpp:4138-4175), its metadata filter (:4349-4360) and the tie-break
// contract of :4218-4223 (similarity desc, then chunk_id asc).
struct VectorHit {
    int64_t rowid = -1;
    std::string chunk_id;
    std::string document_hash;
    float relevance_score = 0.f;
};

// The fields of VectorSearchDiagnostics (include/yams/vector/vector_types.h:180-203) the exact scan fills
// (sqlite_vec_backend.cpp:4131-4135, 4336-4338, 4368-4370, 4404-4406)
struct VectorSearchDiagnostics {
    bool usedExactScan = false;
    bool rowsVisitedObserved = false;
    bool exactDistanceEvaluationsObserved = false;
    size_t rowsVisited = 0;
    size_t exactDistanceEvaluations = 0;
    size_t returnedRows = 0;
    size_t resolvedExhaustively = 0;   // extension: queries the device certificate sent to the exhaustive levels
};

class B200VectorStore {
public:
    static constexpr size_t kMaxDeviceK = 3072;   // yams_b200_search limit (include/yams_b200.h)

    B200VectorStore(uint32_t dim, int dtype = YAMS_B200_F32, int metric = YAMS_B200_COSINE) : dim_(dim), dtype_(dtype) {
        yams_status_t st = yams_b200_corpus_create(nullptr, dim, dtype, metric, 0, &c_);
        if (st != YAMS_OK) throw_status("corpus_create", st);
    }
    ~B200VectorStore() { yams_b200_corpus_destroy(c_); }
    B200VectorStore(const B200VectorStore&) = delete;
    B200VectorStore& operator=(const B200VectorStore&) = delete;

    // insertVectorsBatch: rows are fp32 (the reference BLOB layout, sqlite_vec_backend.cpp:343-363); rowids ascending.
    // An fp16 store converts on the device with the reference's truncating float16_t::from_float.
    void insertVectorsBatch(const std::vector<float>& rows, const std::vector<int64_t>& rowids, const std::vector<std::string>& chunk_ids,
                            const std::vector<std::string>& document_hashes = {},
                            const std::vector<std::map<std::string, std::string>>& metadata = {}) {
        if (rows.size() != rowids.size() * dim_ || chunk_ids.size() != rowids.size()) throw std::invalid_argument("insertVectorsBatch: shape mismatch");
        yams_status_t st = dtype_ == YAMS_B200_F16 ? yams_b200_corpus_append_f32_as_f16(c_, rows.data(), rowids.size(), rowids.data())
                                                   : yams_b200_corpus_append(c_, rows.data(), rowids.size(), rowids.data());
        if (st != YAMS_OK) throw_status("corpus_append", st);
        for (size_t i = 0; i < rowids.size(); ++i) {
            chunk_of_[rowids[i]] = chunk_ids[i];
            if (i < document_hashes.size()) {
                doc_of_[rowids[i]] = document_hashes[i];
                rows_of_doc_[document_hashes[i]].push_back(rowids[i]);
            }
            if (i < metadata.size() && !metadata[i].empty()) meta_of_[rowids[i]] = metadata[i];
            // rows the scan skips (isZeroNormEmbedding / isFiniteEmbedding, sqlite_vec_backend.cpp:204-235): only needed
            // to report exactDistanceEvaluations the way the reference counts it
            const float* r = rows.data() + i * dim_;
            double ss = 0.0;
            bool finite = true;
            for (uint32_t c = 0; c < dim_; ++c) {
                finite = finite && std::isfinite(r[c]);
                ss += (double)r[c] * (double)r[c];
            }
            if (!finite || ss <= 1e-12) skipped_.insert(rowids[i]);
        }
        all_rowids_.insert(all_rowids_.end(), rowids.begin(), rowids.end());
    }

    // deleteVector(chunk_id) / deleteVectorsByDocument(document_hash) (vector_store.h:39-40): the device mirror drops
    // the rows; the remaining rows keep their rowid order
    void deleteVector(const std::string& chunk_id) {
        std::vector<int64_t> gone;
        for (const auto& [rid, cid] : chunk_of_)
            if (cid == chunk_id) gone.push_back(rid);
        removeRows(gone);
    }
    void deleteVectorsByDocument(const std::string& document_hash) {
        auto it = rows_of_doc_.find(document_hash);
        if (it == rows_of_doc_.end()) return;
        std::vector<int64_t> gone = it->second;
        removeRows(gone);
    }

    // lookupCandidateRowidsUnlocked (sqlite_vec_backend.cpp:4412-4448): document hashes -> ascending rowids
    std::vector<int64_t> lookupCandidateRowids(const std::unordered_set<std::string>& candidate_hashes) const {
        std::vector<int64_t> out;
        for (const auto& h : candidate_hashes) {
            auto it = rows_of_doc_.find(h);
            if (it != rows_of_doc_.end()) out.insert(out.end(), it->second.begin(), it->second.end());
        }
        std::sort(out.begin(), out.end());
        out.erase(std::unique(out.begin(), out.end()), out.end());
        return out;
    }

    // searchSimilar (vector_store.h:44-49) with every argument of the reference: `document_hash`, `candidate_hashes`
    // and `metadata_filters` become ONE allowed-rowid set (the WHERE clause of :4138-4175 intersected with the metadata
    // predicate of :4349-4360) that the device scan honours.  InvalidArgument (std::invalid_argument here) for a
    // non-finite or zero-norm query; k == 0 -> empty.
    std::vector<VectorHit> searchSimilar(const std::vector<float>& query, size_t k, float similarity_threshold = 0.0f,
                                         const std::optional<std::string>& document_hash = std::nullopt,
                                         const std::unordered_set<std::string>& candidate_hashes = {},
                                         const std::map<std::string, std::string>& metadata_filters = {},
                                         VectorSearchDiagnostics* diagnostics = nullptr) {
        if (query.size() != dim_) throw std::invalid_argument("query dimension mismatch");
        if (k == 0) return {};
        std::optional<std::vector<int64_t>> allowed = allowedRows(document_hash, candidate_hashes, metadata_filters, diagnostics);
        auto all = searchImpl(query.data(), 1, k, similarity_threshold, allowed ? &*allowed : nullptr, diagnostics);
        return all.empty() ? std::vector<VectorHit>{} : std::move(all[0]);
    }

    // searchExactCandidatesWithDiagnostics (vector_store.h:121-129): exact top-k within the candidate documents
    std::vector<VectorHit> searchExactCandidates(const std::vector<float>& query, size_t k, float similarity_threshold,
                                                 const std::unordered_set<std::string>& candidate_hashes,
                                                 VectorSearchDiagnostics* diagnostics = nullptr) {
        if (query.size() != dim_) throw std::invalid_argument("query dimension mismatch");
        if (k == 0) return {};
        std::optional<std::vector<int64_t>> allowed = allowedRows(std::nullopt, candidate_hashes, {}, diagnostics);
        if (!allowed) allowed.emplace();   // an empty candidate set selects nothing here (the seam is candidate-only)
        auto all = searchImpl(query.data(), 1, k, similarity_threshold, &*allowed, diagnostics);
        return all.empty() ? std::vector<VectorHit>{} : std::move(all[0]);
    }

    // searchAllExactCandidateRowsWithDiagnostics (vector_store.h:131-138): every passing row of the candidate documents
    std::vector<VectorHit> searchAllExactCandidateRows(const std::vector<float>& query, float similarity_threshold,
                                                       const std::unordered_set<std::string>& candidate_hashes,
                                                       VectorSearchDiagnostics* diagnostics = nullptr) {
        if (query.size() != dim_) throw std::invalid_argument("query dimension mismatch");
        std::optional<std::vector<int64_t>> allowed = allowedRows(std::nullopt, candidate_hashes, {}, diagnostics);
        if (!allowed || allowed->empty()) return {};
        auto hits = allMatching(query.data(), similarity_threshold, *allowed);
        if (diagnostics) diagnostics->returnedRows = hits.size();
        return hits;
    }

    // IDocumentCandidateVectorStore::searchDocumentCandidatesWithDiagnostics (vector_store.h:109-116), what
    // CandidateFilterMode::DocumentTopK reaches (vector_database.cpp:553-569): the k best candidate DOCUMENTS, each represented
    // by its best chunk (retainBestRecordPerDocument, sqlite_vec_backend.cpp:86-125).  The documents go to the device sorted by
    // document_hash and their rows by chunk_id, so its position tie-breaks are the reference's.  pq: the PQ engine's branch
    // (rows in the index, its rerank arithmetic); nullptr: the exact fallback.  std::invalid_argument on an empty candidate set
    // (vector_database.cpp:554-557), a non-finite or zero query (exact mode) or a stale index (PQ mode).
    std::vector<VectorHit> searchDocumentCandidates(const std::vector<float>& query, size_t k, float similarity_threshold,
                                                    const std::unordered_set<std::string>& candidate_hashes, yams_b200_pq* pq = nullptr,
                                                    VectorSearchDiagnostics* diagnostics = nullptr) {
        if (query.size() != dim_) throw std::invalid_argument("query dimension mismatch");
        if (candidate_hashes.empty()) throw std::invalid_argument("Document candidate search requires candidate hashes");
        if (k > 4096) throw std::invalid_argument("k exceeds the device limit of 4096 documents per query");
        std::vector<std::string> docs;
        for (const auto& h : candidate_hashes)
            if (rows_of_doc_.count(h)) docs.push_back(h);
        std::sort(docs.begin(), docs.end());
        std::vector<int64_t> rids;
        std::vector<uint64_t> doffs{0};
        for (const auto& h : docs) {
            std::vector<int64_t> rs = rows_of_doc_.at(h);
            std::sort(rs.begin(), rs.end(), [&](int64_t a, int64_t b) {
                const std::string &ca = chunk_of_.at(a), &cb = chunk_of_.at(b);
                return ca != cb ? ca < cb : a < b;
            });
            rids.insert(rids.end(), rs.begin(), rs.end());
            doffs.push_back(rids.size());
        }
        if (diagnostics) {
            noteScan(diagnostics);
            diagnostics->rowsVisited += rids.size();
        }
        const uint64_t qdocs[2] = {0, docs.size()};
        const size_t kk = std::max<size_t>(k, 1);
        std::vector<int64_t> out_docs(kk), out_rid(kk);
        std::vector<float> out_sc(kk);
        uint32_t cnt = 0;
        int64_t none = 0;
        yams_status_t st = yams_b200_search_documents(c_, pq, query.data(), 1, (uint32_t)k, similarity_threshold, rids.empty() ? &none : rids.data(),
                                                      doffs.data(), qdocs, out_docs.data(), out_rid.data(), out_sc.data(), &cnt);
        if (st == YAMS_ERR_INVALID_ARG) throw std::invalid_argument(yams_b200_last_error());
        if (st != YAMS_OK) throw_status("search_documents", st);
        std::vector<VectorHit> hits(cnt);
        for (uint32_t i = 0; i < cnt; ++i) {
            hits[i].rowid = out_rid[i];
            hits[i].relevance_score = out_sc[i];
            hits[i].chunk_id = chunk_of_.at(out_rid[i]);
            hits[i].document_hash = docs[(size_t)out_docs[i]];
        }
        if (diagnostics) diagnostics->returnedRows += hits.size();
        return hits;
    }

    // searchSimilarBatch (vector_store.h:51-53; the reference loops over the queries, :4531-4546): one device call
    std::vector<std::vector<VectorHit>> searchSimilarBatch(const std::vector<std::vector<float>>& queries, size_t k,
                                                           float similarity_threshold = 0.0f, VectorSearchDiagnostics* diagnostics = nullptr) {
        std::vector<std::vector<VectorHit>> out(queries.size());
        if (queries.empty() || k == 0) return out;
        std::vector<float> flat;
        flat.reserve(queries.size() * dim_);
        for (const auto& q : queries) {
            if (q.size() != dim_) throw std::invalid_argument("All query embeddings must have the same dimension");  // :1620-1627
            flat.insert(flat.end(), q.begin(), q.end());
        }
        if (diagnostics) {
            noteScan(diagnostics);
            diagnostics->rowsVisited += all_rowids_.size() * queries.size();
            diagnostics->exactDistanceEvaluations += (all_rowids_.size() - skipped_.size()) * queries.size();
        }
        return searchImpl(flat.data(), queries.size(), k, similarity_threshold, nullptr, diagnostics);
    }

    size_t size() const {
        uint64_t n = 0;
        yams_b200_corpus_size(c_, &n);
        return (size_t)n;
    }

private:
    static void noteScan(VectorSearchDiagnostics* d) {
        d->usedExactScan = true;
        d->rowsVisitedObserved = true;
        d->exactDistanceEvaluationsObserved = true;
    }
    // The rows `SELECT ... WHERE [document_hash = ?] [AND document_hash IN (...)]` visits, minus those failing the
    // metadata predicate; nullopt = no restriction at all.  Fills rowsVisited / exactDistanceEvaluations like the reference
    // counts them (visited = rows the statement yields; evaluated = rows that reach the similarity computation).
    std::optional<std::vector<int64_t>> allowedRows(const std::optional<std::string>& document_hash,
                                                    const std::unordered_set<std::string>& candidate_hashes,
                                                    const std::map<std::string, std::string>& metadata_filters,
                                                    VectorSearchDiagnostics* d) const {
        const bool restricted = document_hash.has_value() || !candidate_hashes.empty();
        std::vector<int64_t> rows;
        if (restricted) {
            if (document_hash && (candidate_hashes.empty() || candidate_hashes.count(*document_hash))) {
                auto it = rows_of_doc_.find(*document_hash);
                if (it != rows_of_doc_.end()) rows = it->second;
                std::sort(rows.begin(), rows.end());
            } else if (!document_hash) {
                rows = lookupCandidateRowids(candidate_hashes);
            }
        } else if (!metadata_filters.empty()) {
            rows = all_rowids_;
        }
        const size_t visited = (restricted || !metadata_filters.empty()) ? rows.size() : all_rowids_.size();
        if (!metadata_filters.empty()) {
            std::vector<int64_t> kept;
            for (int64_t r : rows) {
                auto m = meta_of_.find(r);
                bool match = true;
                for (const auto& [key, value] : metadata_filters) {
                    if (m == meta_of_.end()) { match = false; break; }
                    auto f = m->second.find(key);
                    if (f == m->second.end() || f->second != value) { match = false; break; }
                }
                if (match) kept.push_back(r);
            }
            rows.swap(kept);
        }
        if (d) {
            noteScan(d);
            d->rowsVisited += visited;
            size_t evaluated = (restricted || !metadata_filters.empty()) ? rows.size() : all_rowids_.size();
            if (restricted || !metadata_filters.empty()) {
                for (int64_t r : rows) evaluated -= skipped_.count(r);
            } else {
                evaluated -= skipped_.size();
            }
            d->exactDistanceEvaluations += evaluated;
        }
        if (!restricted && metadata_filters.empty()) return std::nullopt;
        return rows;
    }

    std::vector<VectorHit> allMatching(const float* query, float threshold, const std::vector<int64_t>& allowed) {
        std::vector<int64_t> rid(allowed.size());
        std::vector<float> sc(allowed.size());
        uint64_t cnt = 0;
        yams_status_t st = yams_b200_search_all_matching(c_, query, threshold, allowed.data(), allowed.size(), rid.data(), sc.data(), &cnt);
        if (st == YAMS_ERR_INVALID_ARG) throw std::invalid_argument("Exact vector search requires a finite, non-zero query embedding");
        if (st != YAMS_OK) throw_status("search_all_matching", st);
        return materialise(rid.data(), sc.data(), (uint32_t)cnt, (size_t)cnt);
    }

    // One device call for nq queries (optionally all restricted to the same allowed-rowid set).  The device breaks equal
    // scores by rowid and raises TIE_AT_K when an equal-score run straddles the requested count; the reference breaks by
    // chunk_id (:4218-4223), so the request carries slack and is widened until the run fits (at most kMaxDeviceK rows;
    // beyond that the whole candidate set is fetched with the AllMatching selection and cut here).
    std::vector<std::vector<VectorHit>> searchImpl(const float* flat, size_t nq, size_t k, float threshold, const std::vector<int64_t>* allowed,
                                                   VectorSearchDiagnostics* d) {
        if (k > kMaxDeviceK)
            throw std::invalid_argument("k exceeds the device top-k limit of 3072 rows per query; page the request or use the all-matching selection");
        std::vector<std::vector<VectorHit>> out(nq);
        std::vector<uint64_t> offs;
        int64_t none = 0;
        if (allowed) {
            offs.resize(nq + 1);
            for (size_t q = 0; q <= nq; ++q) offs[q] = q * allowed->size();
        }
        std::vector<int64_t> allowed_rep;
        if (allowed && nq > 1) {
            allowed_rep.reserve(allowed->size() * nq);
            for (size_t q = 0; q < nq; ++q) allowed_rep.insert(allowed_rep.end(), allowed->begin(), allowed->end());
        }
        const int64_t* al = !allowed ? nullptr : (allowed->empty() ? &none : (nq > 1 ? allowed_rep.data() : allowed->data()));
        size_t kk = std::min(kMaxDeviceK, k + 8);
        for (;;) {
            std::vector<int64_t> rid(nq * kk);
            std::vector<float> sc(nq * kk);
            std::vector<uint32_t> cnt(nq);
            std::vector<uint64_t> flg(nq);
            yams_status_t st = yams_b200_search(c_, flat, (uint32_t)nq, (uint32_t)kk, threshold, al, allowed ? offs.data() : nullptr, rid.data(),
                                                sc.data(), cnt.data(), flg.data());
            if (st == YAMS_ERR_INVALID_ARG) throw std::invalid_argument("Exact vector search requires a finite, non-zero query embedding");
            if (st != YAMS_OK) throw_status("search", st);
            bool widen = false;
            for (size_t q = 0; q < nq; ++q)
                if ((flg[q] & YAMS_B200_FLAG_TIE_AT_K) && cnt[q] == kk && kk < kMaxDeviceK) widen = true;
            if (widen) { kk = std::min(kMaxDeviceK, kk * 2); continue; }
            for (size_t q = 0; q < nq; ++q) {
                if ((flg[q] & YAMS_B200_FLAG_TIE_AT_K) && cnt[q] == kk) {
                    // an equal-score run longer than the device can return: take every matching row and cut here
                    std::vector<int64_t> everything = allowed ? *allowed : all_rowids_;
                    std::sort(everything.begin(), everything.end());
                    out[q] = allMatching(flat + q * dim_, threshold, everything);
                    if (out[q].size() > k) out[q].resize(k);
                } else {
                    out[q] = materialise(rid.data() + q * kk, sc.data() + q * kk, cnt[q], k);
                }
                if (d) {
                    d->returnedRows += out[q].size();
                    if (flg[q] & YAMS_B200_FLAG_FALLBACK_PATH) ++d->resolvedExhaustively;
                }
            }
            return out;
        }
    }

    // records for the winners + the chunk_id tie-break of sqlite_vec_backend.cpp:4218-4223
    std::vector<VectorHit> materialise(const int64_t* rid, const float* sc, uint32_t cnt, size_t k) const {
        std::vector<VectorHit> hits(cnt);
        for (uint32_t i = 0; i < cnt; ++i) {
            hits[i].rowid = rid[i];
            hits[i].relevance_score = sc[i];
            auto it = chunk_of_.find(rid[i]);
            hits[i].chunk_id = it == chunk_of_.end() ? std::string() : it->second;
            auto dh = doc_of_.find(rid[i]);
            if (dh != doc_of_.end()) hits[i].document_hash = dh->second;
        }
        std::stable_sort(hits.begin(), hits.end(), [](const VectorHit& a, const VectorHit& b) {
            if (a.relevance_score != b.relevance_score) return a.relevance_score > b.relevance_score;
            return a.chunk_id < b.chunk_id;
        });
        if (hits.size() > k) hits.resize(k);
        return hits;
    }
    void removeRows(const std::vector<int64_t>& gone) {
        if (gone.empty()) return;
        yams_status_t st = yams_b200_corpus_remove(c_, gone.data(), gone.size(), nullptr);
        if (st != YAMS_OK) throw_status("corpus_remove", st);
        std::unordered_set<int64_t> g(gone.begin(), gone.end());
        all_rowids_.erase(std::remove_if(all_rowids_.begin(), all_rowids_.end(), [&](int64_t r) { return g.count(r) != 0; }), all_rowids_.end());
        for (int64_t r : gone) {
            chunk_of_.erase(r);
            meta_of_.erase(r);
            skipped_.erase(r);
            auto d = doc_of_.find(r);
            if (d != doc_of_.end()) {
                auto& v = rows_of_doc_[d->second];
                v.erase(std::remove(v.begin(), v.end(), r), v.end());
                if (v.empty()) rows_of_doc_.erase(d->second);
                doc_of_.erase(d);
            }
        }
    }
    yams_b200_corpus* c_ = nullptr;
    uint32_t dim_;
    int dtype_;
    std::vector<int64_t> all_rowids_;   // ascending (append order)
    std::unordered_set<int64_t> skipped_;
    std::unordered_map<int64_t, std::string> chunk_of_;
    std::unordered_map<int64_t, std::string> doc_of_;
    std::unordered_map<int64_t, std::map<std::string, std::string>> meta_of_;
    std::unordered_map<std::string, std::vector<int64_t>> rows_of_doc_;
};

// IEmbeddingBackend-shaped adapter over the device encoder (src/embedding_simeon/simeon_embedding_backend.cpp:183-215): the default
// Simeon profile only -- any other recipe stays on the reference's CPU encoder.
class B200SimeonBackend {
public:
    // EmbeddingConfig::SimeonEncoderProfile (include/yams/vector/embedding_generator.h:29-37): Configurable is the default
    enum class Profile { Configurable, FixedHash384 };
    explicit B200SimeonBackend(const yams_simeon_config* cfg = nullptr) {
        yams_simeon_config c;
        if (cfg) c = *cfg; else yams_b200_simeon_default_config(&c);
        init(c);
    }
    // resolveEncoder (simeon_embedding_backend.cpp:118-135) for an unconfigured [embeddings.simeon]: FixedHash384 -> simeon_v1_384_config,
    // Configurable -> CharAndWord + Fwht with output_dim = embedding_dim
    B200SimeonBackend(Profile profile, uint32_t embedding_dim) {
        yams_simeon_config c;
        if (profile == Profile::FixedHash384) yams_b200_simeon_default_config(&c);
        else yams_b200_simeon_yams_config(&c, embedding_dim);
        init(c);
    }
    std::string getEmbeddingSpaceIdentity() const { return identity_; }
    ~B200SimeonBackend() { yams_b200_simeon_destroy(e_); }
    B200SimeonBackend(const B200SimeonBackend&) = delete;
    B200SimeonBackend& operator=(const B200SimeonBackend&) = delete;
    std::vector<float> generateEmbedding(const std::string& text) const {
        auto all = generateEmbeddings(std::span<const std::string>(&text, 1));
        return std::move(all[0]);
    }
    std::vector<std::vector<float>> generateEmbeddings(std::span<const std::string> texts) const {
        std::vector<const char*> ptrs(texts.size());
        std::vector<size_t> lens(texts.size());
        for (size_t i = 0; i < texts.size(); ++i) { ptrs[i] = texts[i].data(); lens[i] = texts[i].size(); }
        std::vector<float> flat(texts.size() * dim_);
        yams_status_t st = yams_b200_simeon_encode(e_, ptrs.data(), lens.data(), texts.size(), flat.data());
        if (st != YAMS_OK) throw_status("simeon_encode", st);
        std::vector<std::vector<float>> out(texts.size());
        for (size_t i = 0; i < texts.size(); ++i) out[i].assign(flat.begin() + i * dim_, flat.begin() + (i + 1) * dim_);
        return out;
    }
    size_t getEmbeddingDimension() const { return dim_; }
    std::string getBackendName() const { return "Simeon"; }

private:
    void init(const yams_simeon_config& c) {
        dim_ = c.output_dim;
        const bool word = (c.flags & YAMS_SIMEON_WORD_TOKENS) != 0, fwht = (c.flags & YAMS_SIMEON_PROJECTION_FWHT) != 0;
        if (!word && !fwht && c.ngram_min == 3 && c.ngram_max == 5 && c.sketch_dim == 4096 && c.output_dim == 384 && c.l2_normalize) {
            identity_ = "simeon-v1-384";                                       // simeon.hpp:151
        } else {                                                               // configurableSpaceIdentity, simeon_embedding_backend.cpp:100-116
            identity_ = std::string("simeon-config-v1:") + (word ? "char_and_word" : "char") + ":" + std::to_string(c.ngram_min) + "-" +
                        std::to_string(c.ngram_max) + ":sketch=" + std::to_string(c.sketch_dim) + ":output=" + std::to_string(c.output_dim) +
                        ":projection=" + (fwht ? "fwht" : "achlioptas_sparse") + ":l2=" + (c.l2_normalize ? "1" : "0");
        }
        yams_status_t st = yams_b200_simeon_create(nullptr, &c, &e_);
        if (st != YAMS_OK) throw_status("simeon_create", st);
    }
    yams_b200_encoder* e_ = nullptr;
    size_t dim_ = 0;
    std::string identity_;
};

// ManifestManager::createManifest (src/manifest/manifest_manager.cpp:411-436) over a chunk table: ChunkRefs + checksum in one device call
struct ManifestChunkRef {   // include/yams/manifest/manifest_manager.h:48-61
    std::string hash;
    uint64_t offset = 0;
    uint32_t size = 0;
    uint32_t flags = 0;
};
struct ManifestCore {
    std::string fileHash;
    uint64_t fileSize = 0;
    std::vector<ManifestChunkRef> chunks;
    uint32_t checksum = 0;
    bool valid = false;   // Manifest::isValid && the offset / size rules of validateManifest
};
inline ManifestCore createManifest(const std::string& fileHashHex, uint64_t fileSize, const std::vector<Chunk>& chunks) {
    if (fileHashHex.size() != 64) throw std::invalid_argument("file hash must be 64 hex characters");
    auto nib = [](char c) -> int { return c >= '0' && c <= '9' ? c - '0' : c >= 'a' && c <= 'f' ? c - 'a' + 10 : c >= 'A' && c <= 'F' ? c - 'A' + 10 : -1; };
    auto unhex = [&](const std::string& h, uint8_t* out) {
        for (int i = 0; i < 32; ++i) {
            int hi = nib(h[2 * i]), lo = nib(h[2 * i + 1]);
            if (hi < 0 || lo < 0) throw std::invalid_argument("hash is not hex");
            out[i] = (uint8_t)(hi * 16 + lo);
        }
    };
    uint8_t fd[32];
    unhex(fileHashHex, fd);
    std::vector<yams_chunk_desc> table(chunks.size());
    for (size_t i = 0; i < chunks.size(); ++i) {
        if (chunks[i].hash.size() != 64) throw std::invalid_argument("chunk hash must be 64 hex characters");
        table[i].offset = chunks[i].offset;
        table[i].size = chunks[i].size;
        unhex(chunks[i].hash, table[i].digest);
    }
    std::vector<yams_chunk_ref> refs(chunks.size());
    yams_manifest_summary sum{};
    yams_status_t st = yams_b200_manifest_build(nullptr, table.data(), table.size(), fd, fileSize, refs.data(), &sum);
    if (st != YAMS_OK) throw_status("manifest_build", st);
    ManifestCore m;
    m.fileHash = fileHashHex;
    m.fileSize = fileSize;
    m.checksum = sum.checksum;
    m.valid = sum.valid != 0;
    m.chunks.resize(chunks.size());
    for (size_t i = 0; i < chunks.size(); ++i) m.chunks[i] = {std::string(refs[i].hash, 64), refs[i].offset, refs[i].size, refs[i].flags};
    return m;
}

// VectorDatabase::computeCosineSimilarity (vector_database.cpp:1786-1810)
inline double computeCosineSimilarity(const std::vector<float>& a, const std::vector<float>& b) {
    double out = 0.0;
    yams_status_t st = yams_b200_compute_cosine_similarity(nullptr, a.data(), a.size(), b.data(), b.size(), &out);
    if (st != YAMS_OK) throw_status("compute_cosine_similarity", st);
    return out;
}

// The exists / store loop of ContentStore::store (content_store_impl.cpp:245-288) over one file's chunk table.
class B200ChunkIndex {
public:
    B200ChunkIndex() {
        yams_status_t st = yams_b200_digest_set_create(nullptr, 0, &s_);
        if (st != YAMS_OK) throw_status("digest_set_create", st);
    }
    ~B200ChunkIndex() { yams_b200_digest_set_destroy(s_); }
    B200ChunkIndex(const B200ChunkIndex&) = delete;
    B200ChunkIndex& operator=(const B200ChunkIndex&) = delete;
    struct StoreAccounting {
        uint64_t bytesStored = 0, bytesDeduped = 0;   // StoreResult fields, content_store_impl.cpp:255,277
        std::vector<bool> existed;
    };
    // hashes are the 64-char lowercase hex strings of Chunk::hash
    StoreAccounting addChunks(const std::vector<Chunk>& chunks) {
        std::vector<uint8_t> dg(chunks.size() * 32);
        for (size_t i = 0; i < chunks.size(); ++i) hexToBytes(chunks[i].hash, dg.data() + 32 * i);
        std::vector<uint8_t> ex(chunks.size());
        yams_status_t st = yams_b200_digest_set_insert(s_, dg.data(), 32, chunks.size(), ex.data(), nullptr);
        if (st != YAMS_OK) throw_status("digest_set_insert", st);
        StoreAccounting a;
        a.existed.resize(chunks.size());
        for (size_t i = 0; i < chunks.size(); ++i) {
            a.existed[i] = ex[i] != 0;
            (ex[i] ? a.bytesDeduped : a.bytesStored) += chunks[i].size;
        }
        return a;
    }
    size_t size() const {
        uint64_t n = 0;
        yams_b200_digest_set_size(s_, &n);
        return (size_t)n;
    }

private:
    static void hexToBytes(const std::string& hex, uint8_t* out) {
        if (hex.size() != 64) throw std::invalid_argument("chunk hash must be 64 hex characters");
        auto nib = [](char c) -> int { return c >= '0' && c <= '9' ? c - '0' : c >= 'a' && c <= 'f' ? c - 'a' + 10 : c >= 'A' && c <= 'F' ? c - 'A' + 10 : -1; };
        for (int i = 0; i < 32; ++i) {
            int hi = nib(hex[2 * i]), lo = nib(hex[2 * i + 1]);
            if (hi < 0 || lo < 0) throw std::invalid_argument("chunk hash is not hex");
            out[i] = (uint8_t)(hi * 16 + lo);
        }
    }
    yams_b200_digest_set* s_ = nullptr;
};

// One document-level vector as forEachDocumentLevelVector streams it (sqlite_vec_backend.cpp:1818-1862): the fields the
// semantic graph reads.
struct SemanticDoc {
    std::string hash;               // document_hash
    std::vector<float> embedding;
};

// The pair loop of EmbeddingService::updateSemanticNeighborGraphUnlocked (EmbeddingService.cpp:856-1030) and of
// rebuildSemanticNeighborGraphForCorpus (:1119-1156) on the device: every source document's top-k neighbour documents.  The
// daemon keeps the edge weights, ranks and KG writes (:1038-1075).
class B200SemanticGraph {
public:
    using Neighbors = std::vector<std::pair<std::string, float>>;   // (document_hash, similarity) in rank order
    // docs: the streamed records (empty hashes and embeddings skipped, the first record per hash kept, :864-882); sources: the
    // requested hashes (empty = every document, the rebuild).  out: one entry per source document that has an embedding with
    // a positive norm, in hash order, with its neighbours (none above the threshold: an empty list).  explicitThreshold is
    // YAMS_GRAPH_SEMANTIC_THRESHOLD (clamped to [0, 1] here, :395-403); nullopt is the adaptive mode (sim > 0).
    // YAMS_ERR_UNSUPPORTED when the embeddings have more than one dimension: the reference scores those pairs 0, and the
    // caller keeps its own loop.  Unlike the reference's streaming branch above 250 000 pairs (:555-610, HNSW), the answer is
    // always exact.
    static yams_status_t neighbors(const std::vector<SemanticDoc>& docs, const std::vector<std::string>& sources, size_t topK,
                                   std::optional<float> explicitThreshold, std::vector<std::pair<std::string, Neighbors>>* out) {
        out->clear();
        std::unordered_set<std::string> seen;
        std::vector<const SemanticDoc*> corpus;
        for (const auto& d : docs)
            if (!d.hash.empty() && !d.embedding.empty() && seen.insert(d.hash).second) corpus.push_back(&d);
        if (corpus.empty() || topK == 0) return YAMS_OK;
        const size_t dim = corpus[0]->embedding.size();
        for (const auto* d : corpus)
            if (d->embedding.size() != dim) return YAMS_ERR_UNSUPPORTED;
        if (topK > 3072) return YAMS_ERR_INVALID_ARG;
        std::sort(corpus.begin(), corpus.end(), [](const SemanticDoc* a, const SemanticDoc* b) { return a->hash < b->hash; });
        // the daemon's own float values: an fp32 corpus (the tf32 tensor-core engine), rowid = position in hash order
        std::vector<float> rows(corpus.size() * dim);
        std::vector<int64_t> rowids(corpus.size());
        for (size_t i = 0; i < corpus.size(); ++i) {
            std::memcpy(rows.data() + i * dim, corpus[i]->embedding.data(), dim * sizeof(float));
            rowids[i] = (int64_t)i;
        }
        std::vector<int64_t> src;
        if (!sources.empty()) {
            std::unordered_set<std::string> want(sources.begin(), sources.end());
            for (size_t i = 0; i < corpus.size(); ++i)
                if (want.count(corpus[i]->hash)) src.push_back((int64_t)i);
            if (src.empty()) return YAMS_OK;
        }
        const float threshold = explicitThreshold ? std::clamp(*explicitThreshold, 0.0f, 1.0f) : std::numeric_limits<float>::denorm_min();
        yams_b200_corpus* c = nullptr;
        yams_status_t st = yams_b200_corpus_create(nullptr, (uint32_t)dim, YAMS_B200_F32, YAMS_B200_COSINE, corpus.size(), &c);
        if (st != YAMS_OK) return st;
        const size_t ns = sources.empty() ? corpus.size() : src.size();
        std::vector<int64_t> nb(ns * topK);
        std::vector<float> sims(ns * topK);
        std::vector<uint32_t> counts(ns);
        std::vector<uint64_t> flags(ns);
        st = yams_b200_corpus_append(c, rows.data(), corpus.size(), rowids.data());
        if (st == YAMS_OK)
            st = yams_b200_semantic_neighbors(c, sources.empty() ? nullptr : src.data(), ns, (uint32_t)topK, threshold, nb.data(),
                                              sims.data(), counts.data(), flags.data());
        yams_b200_corpus_destroy(c);
        if (st != YAMS_OK) return st;
        for (size_t i = 0; i < ns; ++i) {
            const size_t row = sources.empty() ? i : (size_t)src[i];
            if (flags[i] & YAMS_B200_FLAG_NOT_A_SOURCE) continue;   // zero-norm or non-finite document (:904, 916)
            Neighbors list;
            for (uint32_t j = 0; j < counts[i]; ++j) list.emplace_back(corpus[(size_t)nb[i * topK + j]]->hash, sims[i * topK + j]);
            out->emplace_back(corpus[row]->hash, std::move(list));
        }
        return YAMS_OK;
    }
};

// The k-means topology engine's clustering (KMeansTopologyEngine::buildArtifacts -> runKMeans,
// src/topology/topology_alternate_engines.cpp:341-478): the per-document assignment runKMeans returns.  embeddings: each
// document's embedding in span order (empty: none).  A usable document has a non-empty embedding of the first non-empty one's
// size (:349-361); fewer than 2 usable -> every document is its own cluster (iota); the usable ones are clustered on the
// device (yams_b200_topology_kmeans, an fp32 corpus of the daemon's own values), the others become singletons numbered k,
// k + 1, ... in document order (:471-476).
class B200TopologyKMeans {
public:
    static yams_status_t assign(const std::vector<std::span<const float>>& embeddings, size_t requestedK, size_t maxIterations,
                                std::vector<int64_t>* out) {
        const size_t n = embeddings.size();
        out->assign(n, -1);
        std::vector<size_t> usable;
        size_t dim = 0;
        for (size_t i = 0; i < n; ++i) {
            if (embeddings[i].empty()) continue;
            if (dim == 0) dim = embeddings[i].size();
            if (embeddings[i].size() == dim) usable.push_back(i);
        }
        if (usable.size() < 2) {
            for (size_t i = 0; i < n; ++i) (*out)[i] = (int64_t)i;
            return YAMS_OK;
        }
        if (usable.size() >= 0xFFFFFFFFull || requestedK > 0xFFFFFFFFull || maxIterations > 0xFFFFFFFFull) return YAMS_ERR_INVALID_ARG;
        std::vector<float> rows(usable.size() * dim);
        for (size_t u = 0; u < usable.size(); ++u) std::memcpy(rows.data() + u * dim, embeddings[usable[u]].data(), dim * sizeof(float));
        yams_b200_corpus* c = nullptr;
        yams_status_t st = yams_b200_corpus_create(nullptr, (uint32_t)dim, YAMS_B200_F32, YAMS_B200_COSINE, usable.size(), &c);
        if (st != YAMS_OK) return st;
        std::vector<uint32_t> membership(usable.size());
        uint32_t k = 0, iterations = 0;
        st = yams_b200_corpus_append(c, rows.data(), usable.size(), nullptr);
        if (st == YAMS_OK)
            st = yams_b200_topology_kmeans(c, (uint32_t)requestedK, (uint32_t)maxIterations, membership.data(), nullptr, &k, &iterations);
        yams_b200_corpus_destroy(c);
        if (st != YAMS_OK) return st;
        for (size_t u = 0; u < usable.size(); ++u) (*out)[usable[u]] = membership[u];
        int64_t singleton = k;
        for (size_t i = 0; i < n; ++i)
            if ((*out)[i] < 0) (*out)[i] = singleton++;
        return YAMS_OK;
    }
};

// simeon::Bm25Index (third_party/simeon/include/simeon/bm25.hpp) as SimeonLexicalBackend uses it
// (src/search/simeon_lexical_backend.cpp: buildAsync adds every document then finalizes; score fills a vector of all document
// scores): add_doc buffers the text, finalize() makes one device build (yams_b200_bm25_build), score() runs on the device.
// Errors the reference reports by throwing (add_doc after finalize, score before it or into a span of the wrong size) throw
// std::runtime_error here too, as does a failed device call.  Atire and SubwordAwareBackoff only (yams_bm25_config).
class B200ConceptIndex;

class B200Bm25Index {
public:
    // lead_tokens > 0: every document also gets extract_lead_tokens(text, lead_tokens) as its aux field, as the lexical backend's
    // add_doc(text, lead) does with the strategy router on (64); finalize builds both fields in one device build
    explicit B200Bm25Index(const yams_bm25_config* cfg = nullptr, uint32_t lead_tokens = 0) : lead_(lead_tokens) {
        if (cfg) cfg_ = *cfg; else yams_b200_bm25_default_config(&cfg_);
    }
    ~B200Bm25Index() { yams_b200_bm25_destroy(idx_); }
    B200Bm25Index(const B200Bm25Index&) = delete;
    B200Bm25Index& operator=(const B200Bm25Index&) = delete;

    void add_doc(std::string_view text) {
        if (idx_) throw std::runtime_error("Bm25Index::add_doc after finalize()");
        texts_.emplace_back(text);
    }
    void finalize() {
        if (idx_) return;
        std::vector<const char*> ptrs;
        std::vector<size_t> lens;
        for (const auto& t : texts_) { ptrs.push_back(t.data()); lens.push_back(t.size()); }
        check(yams_b200_bm25_build_lead(nullptr, &cfg_, ptrs.data(), lens.data(), texts_.size(), lead_, &idx_), "build");
        n_ = texts_.size();
        texts_.clear();
        texts_.shrink_to_fit();
        check(yams_b200_bm25_stats(idx_, &stats_), "stats");
        doc_lengths_.resize(n_);
        check(yams_b200_bm25_doc_lengths(idx_, 0, doc_lengths_.data()), "doc_lengths");
    }
    void score(std::string_view query, std::span<float> out_scores) const {
        if (!idx_) throw std::runtime_error("Bm25Index::score before finalize()");
        if (out_scores.size() != n_) throw std::runtime_error("Bm25Index::score out_scores size mismatch");
        const char* q = query.data();
        const size_t len = query.size();
        check(yams_b200_bm25_score(idx_, &q, &len, 1, out_scores.data(), 0, nullptr, nullptr, nullptr), "score");
    }
    // SimeonLexicalBackend::score with its concept index: the BM25 scores, then concepts->blend_into(query, scores, weight), fused
    // on the device (a null or empty concept index, or one of another document count, adds nothing)
    void score(std::string_view query, std::span<float> out_scores, const B200ConceptIndex* concepts, float weight) const;
    // The strategy router's pool (YAMS_BM25_STRATEGY_BM25 / KEYPHRASE / LEAD_FIELD: Bm25Strategy, KeyphraseStrategy and the
    // "keyphrase" arm, LeadFieldStrategy and the "lead_field" arm) or its routed choice (YAMS_BM25_STRATEGY_ROUTED:
    // SimeonLexicalBackend::scoreStrategyRouted), then concepts->blend_into(query, scores, weight), in one device call.  Returns the
    // pool that scored.
    uint32_t score_strategy(uint32_t strategy, std::string_view query, std::span<float> out_scores,
                            const B200ConceptIndex* concepts = nullptr, float weight = 0.0f) const;
    uint32_t score_strategy_routed(std::string_view query, std::span<float> out_scores, const B200ConceptIndex* concepts = nullptr,
                                   float weight = 0.0f) const {
        return score_strategy(YAMS_BM25_STRATEGY_ROUTED, query, out_scores, concepts, weight);
    }
    // SimeonLexicalBackend::scoreRouted with router_enabled, in one device call: QueryRouter::features and choose over this index
    // (router: NULL = the backend's preset), the recipe's scores -- Bm25Atire as this index's Atire view, so no second index and
    // no QueryRouter are needed -- then concepts->blend_into(query, scores, weight).  Returns the recipe (YAMS_BM25_RECIPE_*).
    uint32_t score_routed(std::string_view query, std::span<float> out_scores, const B200ConceptIndex* concepts = nullptr,
                          float weight = 0.0f, const yams_bm25_router_config* router = nullptr) const;
    // The same, projected onto the backend's candidate pool (its RescoreDecision scores): out[i] = the finite score of document
    // index candidates[i], else 0, 0 for NOT_INDEXED; gathered on the device, so only the pool crosses PCIe.
    static constexpr uint32_t NOT_INDEXED = 0xFFFFFFFFu;
    uint32_t score_routed(std::string_view query, std::span<const uint32_t> candidates, std::span<float> out,
                          const B200ConceptIndex* concepts = nullptr, float weight = 0.0f,
                          const yams_bm25_router_config* router = nullptr) const;
    // QueryRouter::features(query) over this index (no scoring)
    yams_bm25_query_features router_features(std::string_view query, const yams_bm25_router_config* router = nullptr) const;
    // The Atire index SimeonLexicalBackend builds beside a SubwordAwareBackoff primary for RRF (and its router), served from this
    // index's word field without a second build (yams_b200_bm25_atire_view).  The view and this index may go in either order.
    std::unique_ptr<B200Bm25Index> atire_view() const {
        if (!idx_) throw std::runtime_error("Bm25Index::atire_view before finalize()");
        std::unique_ptr<B200Bm25Index> v(new B200Bm25Index(&cfg_, lead_));
        v->cfg_.variant = YAMS_BM25_ATIRE;
        check(yams_b200_bm25_atire_view(idx_, &v->idx_), "atire_view");
        v->n_ = n_;
        check(yams_b200_bm25_stats(v->idx_, &v->stats_), "stats");
        v->doc_lengths_ = doc_lengths_;
        return v;
    }
    uint32_t doc_count() const noexcept { return (uint32_t)(idx_ ? n_ : texts_.size()); }
    float avg_dl() const noexcept { return idx_ ? stats_.avg_dl : 0.0f; }
    yams_b200_bm25* handle() const noexcept { return idx_; }
    uint32_t doc_length(uint32_t doc_id) const noexcept { return doc_id < doc_lengths_.size() ? doc_lengths_[doc_id] : 0u; }
    uint64_t total_tokens() const noexcept { return idx_ ? stats_.total_tokens : 0; }
    // Bm25Index::df / idf / total_tf: the raw term's hash (no tokenising, no case folding), 0 when unknown or not finalized
    uint32_t df(std::string_view term) const { return lookup(term).df; }
    float idf(std::string_view term) const { return lookup(term).idf; }
    uint64_t total_tf(std::string_view term) const { return lookup(term).total_tf; }
    uint64_t hash_term(std::string_view term) const noexcept {
        // splitmix64_hash (simeon src/hasher.cpp:33-47)
        auto mix = [](uint64_t z) {
            z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
            z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
            return z ^ (z >> 31);
        };
        uint64_t h = mix(cfg_.hash_seed ^ 0x9E3779B97F4A7C15ULL);
        const size_t n = term.size();
        size_t i = 0;
        for (; i + 8 <= n; i += 8) {
            uint64_t chunk = 0;
            for (int b = 0; b < 8; ++b) chunk |= (uint64_t)(uint8_t)term[i + b] << (8 * b);
            h = mix(h ^ chunk);
        }
        if (i < n) {
            uint64_t tail = 0;
            for (size_t j = 0; i + j < n; ++j) tail |= (uint64_t)(uint8_t)term[i + j] << (8 * j);
            h = mix(h ^ (tail ^ ((uint64_t)(n - i) << 56)));
        }
        return mix(h ^ (uint64_t)n);
    }

private:
    struct Term {
        uint32_t df = 0;
        float idf = 0.0f;
        uint64_t total_tf = 0;
    };
    Term lookup(std::string_view term) const {
        Term t;
        if (!idx_ || term.empty()) return t;
        check(yams_b200_bm25_postings(idx_, 0, hash_term(term), &t.df, &t.idf, &t.total_tf, nullptr, nullptr, 0), "postings");
        return t;
    }
    static void check(yams_status_t st, const char* what) {
        if (st != YAMS_OK) throw std::runtime_error(std::string("yams_b200_bm25 ") + what + ": " + yams_b200_last_error());
    }
    yams_bm25_config cfg_{};
    uint32_t lead_ = 0;
    std::vector<std::string> texts_;
    yams_b200_bm25* idx_ = nullptr;
    uint64_t n_ = 0;
    yams_bm25_stats stats_{};
    std::vector<uint32_t> doc_lengths_;
};

// simeon::ConceptEntry / ConceptIndex (include/simeon/concept_mining.hpp) mined on the device: size, doc_count, avg_dl, find,
// score and blend_into as the lexical backend calls them.  It owns its device state and may outlive the index it was mined
// against.
struct B200ConceptEntry {
    float pmi = 0.0f;
    float idf = 0.0f;
    uint64_t total_tf = 0;
    uint64_t a_hash = 0;
    uint64_t b_hash = 0;
    std::vector<std::pair<uint32_t, uint32_t>> docs;
};

class B200ConceptIndex {
public:
    B200ConceptIndex() = default;
    ~B200ConceptIndex() { yams_b200_concepts_destroy(c_); }
    B200ConceptIndex(B200ConceptIndex&& o) noexcept : c_(o.c_), stats_(o.stats_) { o.c_ = nullptr; o.stats_ = {}; }
    B200ConceptIndex& operator=(B200ConceptIndex&& o) noexcept {
        if (this != &o) {
            yams_b200_concepts_destroy(c_);
            c_ = o.c_;
            stats_ = o.stats_;
            o.c_ = nullptr;
            o.stats_ = {};
        }
        return *this;
    }
    B200ConceptIndex(const B200ConceptIndex&) = delete;
    B200ConceptIndex& operator=(const B200ConceptIndex&) = delete;

    uint32_t size() const noexcept { return (uint32_t)stats_.size; }
    uint32_t doc_count() const noexcept { return (uint32_t)stats_.doc_count; }
    float avg_dl() const noexcept { return stats_.avg_bigram_dl; }
    // ConceptIndex::find: nullopt when the hash is not a kept concept
    std::optional<B200ConceptEntry> find(uint64_t concept_hash) const {
        if (!c_) return std::nullopt;
        uint32_t found = 0, df = 0;
        B200ConceptEntry e;
        check(yams_b200_concepts_find(c_, concept_hash, &found, &e.pmi, &e.idf, &e.total_tf, &e.a_hash, &e.b_hash, &df, nullptr, nullptr, 0),
              "find");
        if (!found) return std::nullopt;
        std::vector<uint32_t> docs(df), tfs(df);
        check(yams_b200_concepts_find(c_, concept_hash, &found, &e.pmi, &e.idf, &e.total_tf, &e.a_hash, &e.b_hash, &df, docs.data(),
                                      tfs.data(), df),
              "find");
        for (uint32_t i = 0; i < df; ++i) e.docs.emplace_back(docs[i], tfs[i]);
        return e;
    }
    void score(std::string_view query, std::span<float> out_scores) const { blend_into(query, out_scores, 1.0f); }
    void blend_into(std::string_view query, std::span<float> out_scores, float weight) const {
        if (!c_) return;
        check(yams_b200_concepts_blend(c_, query.data(), query.size(), weight, out_scores.data(), out_scores.size()), "blend");
    }
    const yams_b200_concepts* handle() const noexcept { return c_; }

private:
    friend B200ConceptIndex mine_concepts(const B200Bm25Index&, std::span<const std::string_view>, const yams_concept_config&);
    static void check(yams_status_t st, const char* what) {
        if (st != YAMS_OK) throw std::runtime_error(std::string("yams_b200_concepts ") + what + ": " + yams_b200_last_error());
    }
    yams_b200_concepts* c_ = nullptr;
    yams_concepts_stats stats_{};
};

// simeon::mine_concepts(idx, docs, cfg) on the device.  The backend mines only corpora of 100 documents or more
// (simeon_lexical_backend.cpp:507); that rule stays the caller's, as in INTEGRATION §11.
inline B200ConceptIndex mine_concepts(const B200Bm25Index& idx, std::span<const std::string_view> docs, const yams_concept_config& cfg) {
    if (!idx.handle()) throw std::runtime_error("mine_concepts before finalize()");
    std::vector<const char*> ptrs;
    std::vector<size_t> lens;
    for (const auto& d : docs) { ptrs.push_back(d.data()); lens.push_back(d.size()); }
    B200ConceptIndex out;
    B200ConceptIndex::check(yams_b200_concepts_mine(idx.handle(), &cfg, ptrs.data(), lens.data(), docs.size(), &out.c_), "mine");
    B200ConceptIndex::check(yams_b200_concepts_stats(out.c_, &out.stats_), "stats");
    return out;
}

inline uint32_t B200Bm25Index::score_strategy(uint32_t strategy, std::string_view query, std::span<float> out_scores,
                                              const B200ConceptIndex* concepts, float weight) const {
    if (!idx_) throw std::runtime_error("Bm25Index::score before finalize()");
    if (out_scores.size() != n_) throw std::runtime_error("Bm25Index::score out_scores size mismatch");
    const char* q = query.data();
    const size_t len = query.size();
    uint32_t chosen = 0;
    check(yams_b200_bm25_score_strategy(idx_, strategy, concepts ? concepts->handle() : nullptr, weight, &q, &len, 1, out_scores.data(), 0,
                                        nullptr, nullptr, nullptr, &chosen),
          "score_strategy");
    return chosen;
}

inline uint32_t B200Bm25Index::score_routed(std::string_view query, std::span<float> out_scores, const B200ConceptIndex* concepts,
                                            float weight, const yams_bm25_router_config* router) const {
    if (!idx_) throw std::runtime_error("Bm25Index::score before finalize()");
    if (out_scores.size() != n_) throw std::runtime_error("Bm25Index::score out_scores size mismatch");
    const char* q = query.data();
    const size_t len = query.size();
    uint32_t recipe = 0;
    check(yams_b200_bm25_score_routed(idx_, router, concepts ? concepts->handle() : nullptr, weight, &q, &len, 1, out_scores.data(), 0,
                                      nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, &recipe, nullptr),
          "score_routed");
    return recipe;
}

inline uint32_t B200Bm25Index::score_routed(std::string_view query, std::span<const uint32_t> candidates, std::span<float> out,
                                            const B200ConceptIndex* concepts, float weight, const yams_bm25_router_config* router) const {
    if (!idx_) throw std::runtime_error("Bm25Index::score before finalize()");
    if (out.size() != candidates.size()) throw std::runtime_error("Bm25Index::score_routed out size mismatch");
    const char* q = query.data();
    const size_t len = query.size();
    const uint64_t off[2] = {0, candidates.size()};
    uint32_t recipe = 0;
    check(yams_b200_bm25_score_routed(idx_, router, concepts ? concepts->handle() : nullptr, weight, &q, &len, 1, nullptr, 0, nullptr,
                                      nullptr, nullptr, off, candidates.data(), out.data(), &recipe, nullptr),
          "score_routed");
    return recipe;
}

inline yams_bm25_query_features B200Bm25Index::router_features(std::string_view query, const yams_bm25_router_config* router) const {
    if (!idx_) throw std::runtime_error("Bm25Index::router_features before finalize()");
    const char* q = query.data();
    const size_t len = query.size();
    yams_bm25_query_features f{};
    check(yams_b200_bm25_score_routed(idx_, router, nullptr, 0.0f, &q, &len, 1, nullptr, 0, nullptr, nullptr, nullptr, nullptr, nullptr,
                                      nullptr, nullptr, &f),
          "router_features");
    return f;
}

inline void B200Bm25Index::score(std::string_view query, std::span<float> out_scores, const B200ConceptIndex* concepts, float weight) const {
    if (!idx_) throw std::runtime_error("Bm25Index::score before finalize()");
    if (out_scores.size() != n_) throw std::runtime_error("Bm25Index::score out_scores size mismatch");
    const char* q = query.data();
    const size_t len = query.size();
    check(yams_b200_bm25_score_blended(idx_, concepts ? concepts->handle() : nullptr, weight, &q, &len, 1, out_scores.data(), 0, nullptr,
                                       nullptr, nullptr),
          "score_blended");
}

// simeon::score_bm25_variants_rrf(variants, query, out_scores, k_rrf) (fusion.hpp) on the device, and SimeonLexicalBackend::score
// with bm25_variants_rrf: the fusion, then concepts->blend_into(query, out_scores, weight), in one call
// (yams_b200_bm25_score_rrf).  out_scores must have the variants' document count; a variant not finalized, variants of
// different document counts or k_rrf < 0 throw std::runtime_error.  No variants: zeros (then the blend), as the reference.
inline void score_bm25_variants_rrf(std::span<const B200Bm25Index* const> variants, std::string_view query, std::span<float> out_scores,
                                    const B200ConceptIndex* concepts, float weight, float k_rrf = 60.0f) {
    std::fill(out_scores.begin(), out_scores.end(), 0.0f);
    if (variants.empty()) {
        if (concepts) concepts->blend_into(query, out_scores, weight);
        return;
    }
    std::vector<const yams_b200_bm25*> hs;
    for (const B200Bm25Index* v : variants) {
        if (!v || !v->handle()) throw std::runtime_error("score_bm25_variants_rrf: a variant is not finalized");
        hs.push_back(v->handle());
    }
    if (out_scores.size() != variants[0]->doc_count()) throw std::runtime_error("score_bm25_variants_rrf: out_scores size mismatch");
    const char* q = query.data();
    const size_t len = query.size();
    const yams_status_t st = yams_b200_bm25_score_rrf(hs.data(), (uint32_t)hs.size(), k_rrf, concepts ? concepts->handle() : nullptr, weight,
                                                      &q, &len, 1, out_scores.data(), 0, nullptr, nullptr, nullptr);
    if (st != YAMS_OK) throw std::runtime_error(std::string("yams_b200_bm25 score_rrf: ") + yams_b200_last_error());
}
inline void score_bm25_variants_rrf(std::span<const B200Bm25Index* const> variants, std::string_view query, std::span<float> out_scores,
                                    float k_rrf = 60.0f) {
    score_bm25_variants_rrf(variants, query, out_scores, nullptr, 0.0f, k_rrf);
}

}  // namespace yams_b200::host
