/*
 * yams_b200.h -- C ABI of libyams_b200.so: the H100-native drop-in for YAMS's data-parallel hot
 * path (brute-force vector scan behind src/vector + the sqlite-vec-cpp operator surface, and the
 * CDC + SHA-256 ingest path behind src/chunking + src/crypto).
 *
 * Conventions follow the reference's plugin ABI (all path:line relative to the reference source tree):
 *   - envelope: include/yams/plugins/abi.h:17-33 (8 symbols, YAMS_PLUGIN_* return codes);
 *   - vtables:  include/yams/plugins/model_provider_v1.h:44-130 -- struct starts with
 *     {uint32_t abi_version; void* self;}, every fn takes self first and returns yams_status_t,
 *     plugin-allocated buffers are released by a paired free_* fn (host never calls free()),
 *     contiguous row-major [batch, dim] float buffers;
 *   - status codes: model_provider_v1.h:17-25.
 * No exceptions cross this boundary; CUDA failures map to YAMS_ERR_INTERNAL and the text is
 * available through yams_plugin_get_health_json().
 *
 * There is NO CPU fallback: every compute entry point returns YAMS_ERR_INTERNAL (and says why in the
 * health JSON) when no sm_90 device (H100) is usable.
 *
 * Threading (model_provider_v1.h:45 "all functions must be thread-safe unless documented"): every entry point may
 * be called from any host thread.  Calls on one corpus or one digest set are serialised by a per-handle mutex; the
 * handle-less ingest entries (chunk_and_hash*, sha256_*) draw a private device workspace from a pool, so concurrent
 * callers run on separate CUDA streams; an ingest SESSION (ingest_open..ingest_close) belongs to one thread at a time.
 * Input pointers are borrowed for the duration of the call only.
 */
#ifndef YAMS_B200_H
#define YAMS_B200_H

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__) || defined(__clang__)
#define YAMS_B200_API __attribute__((visibility("default")))
#else
#define YAMS_B200_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

/* ---- status codes (model_provider_v1.h:17-25) --------------------------------------------- */
#ifndef YAMS_PLUGINS_MODEL_PROVIDER_V1_H
enum yams_status_e {
    YAMS_OK = 0,
    YAMS_ERR_INVALID_ARG = 1,
    YAMS_ERR_NOT_FOUND = 2,
    YAMS_ERR_IO = 3,
    YAMS_ERR_INTERNAL = 4,
    YAMS_ERR_UNSUPPORTED = 5
};
typedef int yams_status_t;
#endif

/* ---- plugin envelope (abi.h:17-33) ----------------------------------------------------------
 * Loader: src/daemon/resource/abi_plugin_loader.cpp:303-341 (dlopen RTLD_LAZY|RTLD_LOCAL, dlsym of
 * each symbol), manifest regex-parsed :54-79, interface fetched by id+version :657-680. */
#define YAMS_PLUGIN_ABI_VERSION 1
#define YAMS_PLUGIN_OK 0
#define YAMS_PLUGIN_ERR_INCOMPATIBLE -1
#define YAMS_PLUGIN_ERR_NOT_FOUND -2
#define YAMS_PLUGIN_ERR_INIT_FAILED -3
#define YAMS_PLUGIN_ERR_INVALID -4

YAMS_B200_API int yams_plugin_get_abi_version(void);
YAMS_B200_API const char* yams_plugin_get_name(void);
YAMS_B200_API const char* yams_plugin_get_version(void);
YAMS_B200_API const char* yams_plugin_get_manifest_json(void);
/* config_json keys (all optional): "device": int (default: LOCAL_RANK env or 0) */
YAMS_B200_API int yams_plugin_init(const char* config_json, const void* host_context);
YAMS_B200_API void yams_plugin_shutdown(void);
YAMS_B200_API int yams_plugin_get_interface(const char* iface_id, uint32_t version, void** out_iface);
/* *out_json is malloc'd (strdup), as s3_plugin.cpp does; release with free().  "device_buffer_bytes" and
 * "pinned_buffer_bytes" are the bytes the library's device and pinned host buffers hold in this process now. */
YAMS_B200_API int yams_plugin_get_health_json(char** out_json);

#define YAMS_IFACE_VECTOR_SCAN_V1 "vector_scan_v1"
#define YAMS_IFACE_VECTOR_SCAN_V1_VERSION 1u
#define YAMS_IFACE_CONTENT_INGEST_V1 "content_ingest_v1"
#define YAMS_IFACE_CONTENT_INGEST_V1_VERSION 1u

/* =============================================================================================
 * content_ingest_v1 -- replaces IChunker (include/yams/chunking/chunker.h:65-92) +
 * IContentHasher (include/yams/crypto/hasher.h:14-46) as injected at
 * src/api/content_store_builder.cpp:152-170.
 * ============================================================================================= */

enum yams_cdc_variant_e {
    YAMS_CDC_STREAMING = 0, /* StreamingChunker (streaming_chunker.h:146-181) -- what `yams add` uses */
    YAMS_CDC_RABIN = 1      /* RabinChunker (rabin_chunker.cpp:63-152) -- bench/test class          */
};

/* ChunkingConfig (chunker.h:44-51) + which reference class to mirror */
typedef struct yams_cdc_config {
    uint64_t window_size; /* 1..48 (the reference ring is a fixed 48-byte array, chunker.h:151) */
    uint64_t min_chunk;
    uint64_t max_chunk;
    uint64_t polynomial;  /* 0 -> default 0x3DA3358B4DC173 (rabin_chunker.cpp:30-36)             */
    uint64_t mask;
    int32_t variant;      /* yams_cdc_variant_e */
    int32_t reserved;
} yams_cdc_config;

/* One chunk: Chunk{hash,offset,size} (chunker.h:18-23) with the raw 32-byte digest; the host
 * adapter hex-encodes (sha256_hasher.cpp:19-30) */
typedef struct yams_chunk_desc {
    uint64_t offset;
    uint64_t size;
    uint8_t digest[32];
} yams_chunk_desc;

typedef struct yams_b200_ingest yams_b200_ingest; /* opaque streaming session */

YAMS_B200_API void yams_b200_cdc_default_config(yams_cdc_config* cfg);

/* IChunker::chunkData / chunkDataLazy (rabin_chunker.cpp:112-152, streaming_chunker.cpp:92-137):
 * boundaries + per-chunk SHA-256 of a HOST buffer. *out is plugin-allocated; free with
 * yams_b200_free_chunks. len == 0 -> *out_n = 0. */
YAMS_B200_API yams_status_t yams_b200_chunk_and_hash(void* self, const uint8_t* data, size_t len,
                                                     const yams_cdc_config* cfg,
                                                     yams_chunk_desc** out, size_t* out_n);
/* Many files per call -- the shape of `yams add -r` (one StreamingChunker run per file; the reference spreads files
 * over ingest workers, src/app/services/indexing_service.cpp, src/api/content_store_impl.cpp:199-220).  Every file is
 * an independent stream (rolling hash and cut positions restart at its first byte), but the whole batch shares ONE
 * candidate scan, ONE cut-selection pass and ONE SHA-256 launch, so small files reach the throughput of one large
 * stream.  files[i] / lens[i]: HOST buffers.  out: plugin-allocated table (free_chunks) with offsets relative to the
 * owning file; chunks of file i are out[out_first[i] .. out_first[i+1]); out_first holds n_files + 1 entries. */
YAMS_B200_API yams_status_t yams_b200_chunk_and_hash_batch(void* self, const uint8_t* const* files,
                                                           const size_t* lens, size_t n_files,
                                                           const yams_cdc_config* cfg, yams_chunk_desc** out,
                                                           size_t* out_n, uint64_t* out_first);

YAMS_B200_API void yams_b200_free_chunks(void* self, yams_chunk_desc* chunks, size_t n);

/* Same with the input already resident in HBM (device pointer). Results come back on the host. */
YAMS_B200_API yams_status_t yams_b200_chunk_and_hash_device(void* self, const uint8_t* d_data,
                                                            size_t len, const yams_cdc_config* cfg,
                                                            yams_chunk_desc** out, size_t* out_n);

/* Streaming form: StreamingChunker::processStream/processBuffer (streaming_chunker.h:78-181).
 * Fragmentation is invisible (tests/unit/chunking/chunking_test.cpp:481-523): feeding any split of
 * a stream yields the same chunks as one call.  Each feed returns the chunks completed so far;
 * finish returns the trailing partial chunk (streaming_chunker.h:115-118). Offsets are stream
 * offsets. */
YAMS_B200_API yams_status_t yams_b200_ingest_open(void* self, const yams_cdc_config* cfg,
                                                  yams_b200_ingest** out);
YAMS_B200_API yams_status_t yams_b200_ingest_feed(yams_b200_ingest* s, const uint8_t* data,
                                                  size_t len, yams_chunk_desc** out, size_t* out_n);
YAMS_B200_API yams_status_t yams_b200_ingest_finish(yams_b200_ingest* s, yams_chunk_desc** out,
                                                    size_t* out_n);
YAMS_B200_API void yams_b200_ingest_close(yams_b200_ingest* s);

/* SHA256Hasher::hash over many spans of one HOST buffer (sha256_hasher.cpp:167-195);
 * digests: n x 32 bytes, caller-owned. */
YAMS_B200_API yams_status_t yams_b200_sha256_batch(void* self, const uint8_t* base, size_t base_len,
                                                   const uint64_t* offsets, const uint64_t* sizes,
                                                   size_t n, uint8_t* digests);
/* base is a device pointer; offsets/sizes/digests are host arrays */
YAMS_B200_API yams_status_t yams_b200_sha256_batch_device(void* self, const uint8_t* d_base,
                                                          size_t base_len, const uint64_t* offsets,
                                                          const uint64_t* sizes, size_t n,
                                                          uint8_t* digests);

/* Only the CDC boundaries (no digests): (offset,size) pairs, digest field zero. */
YAMS_B200_API yams_status_t yams_b200_chunk_boundaries(void* self, const uint8_t* data, size_t len,
                                                       const yams_cdc_config* cfg,
                                                       yams_chunk_desc** out, size_t* out_n);

/* SHA-256 of n SEPARATE host messages in one device pass (IContentHasher::hash per span, hasher.h:14-46;
 * ChunkValidator::validateChunks hashes chunks fetched one by one, src/integrity/chunk_validator.cpp:173-213).
 * digests: n x 32 bytes. */
YAMS_B200_API yams_status_t yams_b200_sha256_many(void* self, const uint8_t* const* msgs, const size_t* lens,
                                                  size_t n, uint8_t* digests);

/* calculateDeduplication (src/chunking/rabin_chunker.cpp:224-239): unique-hash accounting over a chunk table.
 * A chunk is "unique" the first time its digest appears.  chunks: HOST array (as returned by chunk_and_hash). */
typedef struct yams_dedup_stats {
    uint64_t total_size;     /* DeduplicationStats::totalSize   (chunker.h:204-209) */
    uint64_t unique_size;    /* uniqueSize   */
    uint64_t chunk_count;    /* chunkCount   */
    uint64_t unique_chunks;  /* uniqueChunks */
} yams_dedup_stats;
YAMS_B200_API yams_status_t yams_b200_dedup_stats(void* self, const yams_chunk_desc* chunks, size_t n,
                                                  yams_dedup_stats* out);

/* ---- device-resident digest set (SURVEY.md §8f N1) --------------------------------------------------------
 * Batched form of the per-chunk `storage_->exists(hash)` / `storage_->store(hash, data)` loop that follows
 * chunking (src/api/content_store_impl.cpp:245-288, src/storage/storage_engine.cpp:281-305): one call answers
 * the existence question for every chunk of a file. digests are HOST pointers, `stride` bytes apart (32 for a
 * packed array; sizeof(yams_chunk_desc) with digests = chunks[0].digest for a chunk table). */
typedef struct yams_b200_digest_set yams_b200_digest_set;
YAMS_B200_API yams_status_t yams_b200_digest_set_create(void* self, uint64_t capacity_hint,
                                                        yams_b200_digest_set** out);
/* exists-then-store: out_existed[i] = 1 iff digest i was in the set before the call or equals an EARLIER
 * digest of this batch (exactly what the sequential loop observes); afterwards every digest is in the set.
 * out_existed and out_new (number of digests that were new) are nullable. */
YAMS_B200_API yams_status_t yams_b200_digest_set_insert(yams_b200_digest_set* s, const uint8_t* digests,
                                                        size_t stride, size_t n, uint8_t* out_existed,
                                                        uint64_t* out_new);
/* read-only membership (storage_->exists) */
YAMS_B200_API yams_status_t yams_b200_digest_set_contains(yams_b200_digest_set* s, const uint8_t* digests,
                                                          size_t stride, size_t n, uint8_t* out_exists);
YAMS_B200_API yams_status_t yams_b200_digest_set_size(yams_b200_digest_set* s, uint64_t* out);
/* device time (ms) of the kernels of the last insert/contains call */
YAMS_B200_API yams_status_t yams_b200_digest_set_last_ms(yams_b200_digest_set* s, float* out_ms);
YAMS_B200_API void yams_b200_digest_set_destroy(yams_b200_digest_set* s);

/* ---- manifest of one file (SURVEY.md §8f N2) ---------------------------------------------------------------
 * The consumer of the chunk table: ManifestManager::createManifest (src/manifest/manifest_manager.cpp:411-436) turns it
 * into ChunkRef{hash (64 lowercase hex chars), offset, u32 size, flags} (include/yams/manifest/manifest_manager.h:48-61)
 * and seals it with calculateChecksum (:705-730): a bit-serial CRC-32 over fileHash || to_string(fileSize) || for each
 * chunk hash || to_string(offset) || to_string(size) -- ~80 text bytes per chunk on one dependent chain.  Here the hex
 * rendering, the per-record CRCs and their GF(2) combination run on the device; the checksum is bit-identical. */
typedef struct yams_chunk_ref {
    char hash[64];      /* lowercase hex, NOT NUL-terminated (HASH_STRING_SIZE, core/types.h:279) */
    uint64_t offset;
    uint32_t size;      /* static_cast<uint32_t>(chunk.size), manifest_manager.h:209 */
    uint32_t flags;
} yams_chunk_ref;
typedef struct yams_manifest_summary {
    uint32_t checksum;             /* Manifest::checksum */
    uint32_t valid;                /* Manifest::isValid (manifest_manager.h:98-104) && the offset / size rules of validateManifest (:452-468) */
    uint32_t offsets_sequential;   /* every chunk.offset == running sum of the sizes */
    uint32_t sizes_valid;          /* every size > 0 and representable in 32 bits */
    uint64_t chunk_count;
    uint64_t total_size;           /* Manifest::calculateTotalSize */
    uint64_t checksum_text_bytes;  /* length of the text the CRC ran over */
} yams_manifest_summary;
/* chunks: HOST table as returned by chunk_and_hash (n may be 0); file_digest: SHA-256 of the whole file (FileInfo::hash,
 * raw 32 bytes); out_refs: nullable HOST array of n entries. */
YAMS_B200_API yams_status_t yams_b200_manifest_build(void* self, const yams_chunk_desc* chunks, size_t n,
                                                     const uint8_t file_digest[32], uint64_t file_size,
                                                     yams_chunk_ref* out_refs, yams_manifest_summary* out);

/* Per-stage timings (ms) of the last chunk_and_hash* / chunk_boundaries call on this thread:
 * device time of [0] candidate scan, [1] cut selection, [2] sha256, [3] the whole call;
 * host wall-clock time of [4] the wait after the candidate scan, [5] the wait after the chunk-count scan,
 * [6] descriptor-table growth, [7] cut processing as a whole.
 * chunk_and_hash_batch sums [0..3] over its file groups and sets [4..7] to 0. */
YAMS_B200_API yams_status_t yams_b200_ingest_last_timings(void* self, float out_ms[8]);

typedef struct yams_content_ingest_v1 {
    uint32_t abi_version; /* YAMS_IFACE_CONTENT_INGEST_V1_VERSION */
    void* self;
    yams_status_t (*chunk_and_hash)(void* self, const uint8_t* data, size_t len,
                                    const yams_cdc_config* cfg, yams_chunk_desc** out,
                                    size_t* out_n);
    void (*free_chunks)(void* self, yams_chunk_desc* chunks, size_t n);
    yams_status_t (*ingest_open)(void* self, const yams_cdc_config* cfg, yams_b200_ingest** out);
    yams_status_t (*ingest_feed)(yams_b200_ingest* s, const uint8_t* data, size_t len,
                                 yams_chunk_desc** out, size_t* out_n);
    yams_status_t (*ingest_finish)(yams_b200_ingest* s, yams_chunk_desc** out, size_t* out_n);
    void (*ingest_close)(yams_b200_ingest* s);
    yams_status_t (*sha256_batch)(void* self, const uint8_t* base, size_t base_len,
                                  const uint64_t* offsets, const uint64_t* sizes, size_t n,
                                  uint8_t* digests);
    yams_status_t (*dedup_stats)(void* self, const yams_chunk_desc* chunks, size_t n,
                                 yams_dedup_stats* out);
    yams_status_t (*chunk_and_hash_batch)(void* self, const uint8_t* const* files, const size_t* lens,
                                          size_t n_files, const yams_cdc_config* cfg, yams_chunk_desc** out,
                                          size_t* out_n, uint64_t* out_first);
    yams_status_t (*sha256_many)(void* self, const uint8_t* const* msgs, const size_t* lens, size_t n,
                                 uint8_t* digests);
    yams_status_t (*digest_set_create)(void* self, uint64_t capacity_hint, yams_b200_digest_set** out);
    yams_status_t (*digest_set_insert)(yams_b200_digest_set* s, const uint8_t* digests, size_t stride,
                                       size_t n, uint8_t* out_existed, uint64_t* out_new);
    yams_status_t (*digest_set_contains)(yams_b200_digest_set* s, const uint8_t* digests, size_t stride,
                                         size_t n, uint8_t* out_exists);
    yams_status_t (*digest_set_size)(yams_b200_digest_set* s, uint64_t* out);
    void (*digest_set_destroy)(yams_b200_digest_set* s);
    yams_status_t (*manifest_build)(void* self, const yams_chunk_desc* chunks, size_t n, const uint8_t file_digest[32],
                                    uint64_t file_size, yams_chunk_ref* out_refs, yams_manifest_summary* out);
} yams_content_ingest_v1;

/* =============================================================================================
 * vector_scan_v1 -- replaces the exact scan behind IVectorStore::searchSimilar /
 * searchSimilarBatch (include/yams/vector/vector_store.h:44-53) and the exact-candidate seams
 * (:121-138), i.e. SqliteVecBackend::Impl::bruteForceSearchUnlocked
 * (src/vector/sqlite_vec_backend.cpp:4115-4410), and vec0_run_exact_query
 * (third_party/sqlite-vec-cpp/include/sqlite-vec-cpp/sqlite/vec0_module.hpp:376-430).
 * ============================================================================================= */

enum yams_b200_dtype_e { YAMS_B200_F32 = 0, YAMS_B200_F16 = 1 };
enum yams_b200_metric_e { YAMS_B200_COSINE = 0, YAMS_B200_L2 = 1 };

typedef struct yams_b200_corpus yams_b200_corpus; /* opaque device-resident mirror of `vectors` */

/* rows are stored row-major [n, dim] in HBM in `dtype` (fp32 = the reference's BLOB layout,
 * sqlite_vec_backend.cpp:343-363; fp16 = IEEE half bit patterns, utils/float16.hpp). */
YAMS_B200_API yams_status_t yams_b200_corpus_create(void* self, uint32_t dim, int dtype, int metric,
                                                    uint64_t capacity_hint, yams_b200_corpus** out);
/* rows: HOST pointer, n x dim elements of the corpus dtype; rowids nullable (then consecutive,
 * continuing from the current size). Rowids must be non-negative (-1 marks an unused result slot) and appended in
 * strictly ascending order (the reference scans ORDER BY rowid, sqlite_vec_backend.cpp:4175). A rejected batch leaves
 * the corpus unchanged. */
YAMS_B200_API yams_status_t yams_b200_corpus_append(yams_b200_corpus* c, const void* rows, uint64_t n,
                                                    const int64_t* rowids);
/* fp32 HOST rows converted with the reference's TRUNCATING float16_t::from_float
 * (utils/float16.hpp:20-40) into an fp16 corpus */
YAMS_B200_API yams_status_t yams_b200_corpus_append_f32_as_f16(yams_b200_corpus* c, const float* rows,
                                                               uint64_t n, const int64_t* rowids);
/* Synthetic rows generated on the device (SURVEY.md §8d generator; bit-identical to
 * oracle yo_gen_rows_f32 [+ truncating fp16]); rowid = first_row + i */
YAMS_B200_API yams_status_t yams_b200_corpus_append_synthetic(yams_b200_corpus* c, uint64_t seed,
                                                              uint64_t first_row, uint64_t n);
/* Remove rows by rowid (IVectorStore::deleteVector / deleteVectorsByDocument after the SQLite delete,
 * vector_store.h; the scan then no longer sees them, exactly as `SELECT ... FROM vectors` would not).
 * Unknown rowids are ignored; the remaining rows keep their order (ORDER BY rowid). Stable on-device compaction.
 * out_removed (nullable) receives the number of rows actually removed. */
YAMS_B200_API yams_status_t yams_b200_corpus_remove(yams_b200_corpus* c, const int64_t* rowids, uint64_t n,
                                                    uint64_t* out_removed);
YAMS_B200_API yams_status_t yams_b200_corpus_clear(yams_b200_corpus* c);
YAMS_B200_API yams_status_t yams_b200_corpus_size(const yams_b200_corpus* c, uint64_t* out_n);
YAMS_B200_API void yams_b200_corpus_destroy(yams_b200_corpus* c);

#define YAMS_B200_FLAG_TIE_AT_K 1ull       /* equal scores straddle the k boundary: the host   */
                                           /* adapter must re-break by chunk_id (:4218-4223)   */
#define YAMS_B200_FLAG_FALLBACK_PATH 2ull  /* the fast path could not PROVE its answer exact;   */
                                           /* the query was answered by an exhaustive level     */
#define YAMS_B200_FLAG_NOT_A_SOURCE 4ull   /* yams_b200_semantic_neighbors: the rowid is unknown */
                                           /* or its row is not in the graph (count 0)          */

/* Exact top-k of every query against the corpus (bruteForceSearchUnlocked fast path semantics,
 * sqlite_vec_backend.cpp:4203-4331):
 *   cosine: sim = float(dot / (|row| * |q|)) accumulated in double; rows with a non-finite element
 *   or |row|^2 <= 1e-12 are skipped; sim < threshold dropped; order (sim desc, rowid asc).
 *   l2 (vec0 surface, vec0_module.hpp:376-430): dist = sqrtf(sum (q-r)^2) in float, evaluated as the reference build does
 *   (AVX lane order when dim % 16 == 0, simd/avx.hpp:20-66); order (dist asc, rowid asc); threshold ignored.
 * How "exact" is guaranteed: a tensor-core pass ranks all rows by an approximate score with a known error bound eps, the
 * best K' = k + max(16, k/4) rows are re-scored exactly, and a device-side certificate checks that no other row can
 * reach the k-th exact score (bound + eps < k-th score).  A query that fails the check (near-duplicate rows, an
 * overflowing or short candidate list) is re-run exhaustively inside the same call -- CUDA-core scores of all rows +
 * exact re-scoring of the best 4096, then, if even that cannot be certified, the exact score of every row -- and carries
 * YAMS_B200_FLAG_FALLBACK_PATH.  The returned ids/scores are the reference's in every case.
 * queries: HOST, Q x dim fp32 row-major.  A query that is non-finite or has |q|^2 < 1e-10 makes
 * the whole call return YAMS_ERR_INVALID_ARG (:4127-4130).  k == 0 -> all counts 0 (:4123-4126).
 * allowed_rowids: nullable; when given, query i may only match rowids in
 * allowed_rowids[allowed_offsets[i] .. allowed_offsets[i+1]) (ascending) -- CandidateFilterMode::
 * Exact (src/vector/vector_database.cpp:570-597). allowed_offsets has Q+1 entries.
 * Outputs (caller-owned HOST): out_rowids/out_scores Q x k (unused slots: rowid -1, score 0),
 * out_counts Q, out_flags Q (nullable). * k <= 3072. */
YAMS_B200_API yams_status_t yams_b200_search(yams_b200_corpus* c, const float* queries, uint32_t nq,
                                             uint32_t k, float threshold,
                                             const int64_t* allowed_rowids,
                                             const uint64_t* allowed_offsets, int64_t* out_rowids,
                                             float* out_scores, uint32_t* out_counts,
                                             uint64_t* out_flags);

/* ExactRowSelection::AllMatching (sqlite_vec_backend.cpp:4283-4288,4315-4316; IAllExactCandidateVectorStore,
 * vector_store.h:131-138): EVERY row of the candidate set that passes the skip rules and the threshold, ordered
 * (sim desc, rowid asc), scored exactly (double accumulation). One query. out arrays hold n_allowed entries.
 * allowed_rowids == NULL means the whole corpus (out arrays then hold corpus_size entries). */
YAMS_B200_API yams_status_t yams_b200_search_all_matching(yams_b200_corpus* c, const float* query, float threshold,
                                                          const int64_t* allowed_rowids, uint64_t n_allowed,
                                                          int64_t* out_rowids, float* out_scores,
                                                          uint64_t* out_count);

/* The semantic-neighbour graph over document-level embeddings (EmbeddingService::updateSemanticNeighborGraphUnlocked,
 * src/daemon/components/EmbeddingService.cpp:405-431, 856-1030): the exact top-k neighbour DOCUMENTS of every source document.
 * c is a cosine corpus (fp32 or fp16; L2 -> YAMS_ERR_INVALID_ARG) of one document per row, appended in document_hash order,
 * so that rowid ascending is the reference's hash ascending.
 *   row taken  every element finite and inv = float(1 / sqrt(sum (double)r^2)) > 0 (:405-415, :875-877).  Unlike
 *              yams_b200_search, rows with 0 < |r|^2 <= 1e-12 ARE neighbours, and so are rows whose inv overflows to +inf
 *              (|r|^2 < 2^-256; their similarities are +-inf, and every source then goes to the exhaustive levels).
 *   NaN        the one case without a reference answer: a NaN similarity (a row with a NaN element, whose inv is NaN, or
 *              0 * inf from a row with an infinite inv) enters the reference's candidate lists, where its replace-worst
 *              and sort have no defined result.  Here it is never a neighbour; a row with a NaN element is not a source.
 *   score      sim = float((dot * (double)inv_s) * (double)inv_n), dot the sequential double sum of s[i] * n[i], s the source
 *              (cosineSimilarity, :417-431).  The source's own row is never its neighbour.  sim < threshold is dropped.
 *              The reference's adaptive mode (no explicit threshold: sim > 0) is threshold = FLT_TRUE_MIN; its explicit
 *              YAMS_GRAPH_SEMANTIC_THRESHOLD is that value clamped to [0, 1].
 *   order      (sim desc, rowid asc), -0.0 and +0.0 one score; the best k kept (:949-1017).
 * source_rowids: NULL = every row is a source (n_sources must equal the corpus size), else strictly ascending rowids; an unknown
 * rowid or a row that is not taken gets count 0 and YAMS_B200_FLAG_NOT_A_SOURCE.  k == 0 -> all counts and flags 0;
 * k <= 3072.
 * Outputs (caller-owned HOST) n_sources x k: out_rowids (unused slots -1), out_sims (unused slots 0), out_counts, out_flags
 * (nullable; YAMS_B200_FLAG_TIE_AT_K and YAMS_B200_FLAG_FALLBACK_PATH as for yams_b200_search, NOT_A_SOURCE above).  The sources run in batches of
 * 1024 through the exact scan of yams_b200_search, with the same certificate and exhaustive levels. */
YAMS_B200_API yams_status_t yams_b200_semantic_neighbors(yams_b200_corpus* c, const int64_t* source_rowids, uint64_t n_sources,
                                                         uint32_t k, float threshold, int64_t* out_rowids, float* out_sims,
                                                         uint32_t* out_counts, uint64_t* out_flags);
/* diagnostics: dense stage-1 scores of the graph (the graph's own 1/|r| scales) of every corpus row against the n_sources
 * (<= 1024, all taken) sources with the chosen engine (0 cuda-core, 1 wgmma) -> out_scores[s * corpus_size + row] (HOST), and
 * the certificate's per-source error bound (stage 1 plus the score's float cast) -> out_eps[s] */
YAMS_B200_API yams_status_t yams_b200_debug_semantic_stage1(yams_b200_corpus* c, const int64_t* source_rowids, uint32_t n_sources,
                                                            int engine, float* out_scores, float* out_eps);

/* The k-means topology engine's clustering (KMeansTopologyEngine, src/topology/topology_alternate_engines.cpp:341-478 runKMeans):
 * a deterministic spherical k-means over document-level embeddings, bit-identical to the reference.  c is a cosine corpus
 * (fp32 or fp16, defined on the stored values; L2 -> YAMS_ERR_INVALID_ARG) of one row per USABLE document, appended in document
 * order (documents without an embedding of the first embedding's size are the caller's singletons, see B200TopologyKMeans).
 *   k          k_requested, or round(sqrt(rows)) when 0, clamped to [2, rows]
 *   distance   cosineDistance: dot, |a|^2, |b|^2 as sequential double sums; 2.0 when a norm is <= 0, else
 *              1 - clamp(dot / (sqrt(|a|^2) * sqrt(|b|^2)), -1, 1), a NaN kept
 *   init       farthest-first: centroid 0 = normalized(row 0), then k - 1 picks of the first unselected row with the largest
 *              distance to its nearest centroid so far
 *   iterate    max_iterations (0 means 10) rounds of: assignment to the first centroid with the strictly smallest distance (0
 *              when all are NaN); centroid = normalized(float mean of the members in row order) for every non-empty cluster;
 *              empty clusters repaired in order by the row farthest from its centroid among clusters of more than one member;
 *              stop when nothing changed
 * Outputs (HOST): out_assignment[rows] = the cluster of every row, numbered as runKMeans numbers them; out_centroids
 * (nullable) [k][dim] the final centroids; *out_k = k; *out_iterations = the rounds run.  Fewer than 2 rows: out_assignment[i] =
 * i, *out_k = *out_iterations = 0.  Every distance is computed exactly in fp64 on the device (DESIGN.md §4.10). */
YAMS_B200_API yams_status_t yams_b200_topology_kmeans(yams_b200_corpus* c, uint32_t k_requested, uint32_t max_iterations,
                                                      uint32_t* out_assignment, float* out_centroids, uint32_t* out_k,
                                                      uint32_t* out_iterations);
/* the last yams_b200_topology_kmeans call on c: out_ms[0..2] device ms of the init, the assignments and the centroid updates
 * (repairs included), out_ms[3] the call's host wall time */
YAMS_B200_API yams_status_t yams_b200_topology_kmeans_last_timings(yams_b200_corpus* c, float out_ms[4]);

/* Device-pointer form for multi-GPU sharding: queries and outputs are DEVICE pointers, the whole pipeline is enqueued on
 * the corpus stream and the call returns WITHOUT synchronising (query validity, list overflow and the exactness
 * certificate are evaluated on the device and parked in a status block).  Outputs are the rank-local partial top-k in
 * the padded Q x k layout (unused: score -inf / +inf(l2), rowid -1).  k <= 768.
 * yams_b200_search_device_finish waits for the stream, returns YAMS_ERR_INVALID_ARG if a query was non-finite / zero,
 * and re-runs the queries the certificate rejected through the exhaustive levels, patching the device outputs in place
 * (*out_resolved = how many; 0 for ordinary data).  A caller that pipelines batches calls it before it consumes the
 * outputs of that batch.  A pending search is finished against the corpus it was enqueued on before any other call on that
 * corpus runs (an append, remove or clear, a search of any form, the graph, k-means, document search, a diagnostic): that
 * call first waits for the stream and runs the exhaustive levels, and search_device_finish later returns what they returned
 * and resolved.  The output buffers must therefore stay valid until search_device_finish or until the next call on the
 * corpus.  Only a later search_device supersedes a pending search, without waiting for it: its finish then reports
 * nothing for the superseded batch, whose rejected queries are never re-run. */
YAMS_B200_API yams_status_t yams_b200_search_device(yams_b200_corpus* c, const float* d_queries,
                                                    uint32_t nq, uint32_t k, float threshold,
                                                    int64_t* d_out_rowids, float* d_out_scores);
YAMS_B200_API yams_status_t yams_b200_search_device_finish(yams_b200_corpus* c, uint32_t* out_resolved);
/* The exhaustive reference inside the library: exact score of EVERY row (the reference's loop, row-parallel) + a global
 * sort, no tensor-core stage, no thresholds.  Same outputs as yams_b200_search.  This is what the fast path is checked
 * against at corpus sizes a CPU oracle cannot reach (bench.py parity_full, tests); ~3 ms per query per 10 M rows. */
YAMS_B200_API yams_status_t yams_b200_search_exhaustive(yams_b200_corpus* c, const float* queries, uint32_t nq,
                                                        uint32_t k, float threshold, int64_t* out_rowids,
                                                        float* out_scores, uint32_t* out_counts,
                                                        uint64_t* out_flags);
/* Merge R partial results laid out [R][Q][k] (as produced by an all-gather of search_device
 * outputs) into the global top-k, same order. All DEVICE pointers. */
YAMS_B200_API yams_status_t yams_b200_merge_partials_device(yams_b200_corpus* c,
                                                            const int64_t* d_rowids,
                                                            const float* d_scores, uint32_t nranks,
                                                            uint32_t nq, uint32_t k,
                                                            int64_t* d_out_rowids,
                                                            float* d_out_scores,
                                                            uint32_t* d_out_counts);
/* Same merge over the PACKED record an all-gather of one buffer produces: rank r's record is
 * [nq*k int64 rowids][nq*k float scores] (12*nq*k bytes, SURVEY.md §8e), records back to back.  search_device writes
 * such a record when d_out_scores = (float*)(d_out_rowids + nq*k).  stream: cudaStream_t to launch on (NULL = the
 * corpus stream) so that gather + merge of batch i can overlap the scan of batch i+1. */
YAMS_B200_API yams_status_t yams_b200_merge_packed_device(yams_b200_corpus* c, const void* d_packed,
                                                          uint32_t nranks, uint32_t nq, uint32_t k,
                                                          int64_t* d_out_rowids, float* d_out_scores,
                                                          uint32_t* d_out_counts, void* stream);
YAMS_B200_API yams_status_t yams_b200_corpus_sync(yams_b200_corpus* c);
/* raw cudaStream_t of the corpus (for event timing by the bench) */
YAMS_B200_API void* yams_b200_corpus_stream(yams_b200_corpus* c);

/* vec0_run_exact_query (vec0_module.hpp:376-430): L2 + sqrt in float over fp32 HOST rows, ascending
 * by distance (ties rowid asc), truncated to k when k > 0 (k == 0: all rows); optional inclusive
 * rowid range. out arrays hold min(n, k?k:n) entries. */
YAMS_B200_API yams_status_t yams_b200_vec0_exact(void* self, const float* query, uint32_t dim,
                                                 const float* rows, const int64_t* rowids,
                                                 uint64_t n, uint64_t k, int use_range,
                                                 int64_t rowid_lo, int64_t rowid_hi,
                                                 int64_t* out_rowids, float* out_dist,
                                                 uint64_t* out_count);

/* sqlite-vec-cpp batch surface (distances/batch.hpp:24-146): ONE query against n contiguous fp32 rows, float accumulation
 * in the operation ORDER of the reference build (AVX lane order, simd/avx.hpp; see csrc/ref_order.cuh), so distances are
 * bit-identical to distances::{cosine,l2}_distance<float> (cosine DISTANCE = 1 - cos, 1.0 when the norm product < 1e-8).
 *   mode ALL      batch_distance / batch_distance_contiguous / batch_distance_parallel: out_dist[n] in row order
 *   mode TOP_K    batch_top_k: indices of the k smallest distances, ascending (ties by index -- a legal refinement
 *                 of the reference's unstable partial_sort); out_idx[min(k,n)], out_dist optional
 *   mode FILTERED batch_distance_filtered: every (index, dist) with dist < threshold, ascending; out arrays hold n
 * database is a HOST pointer (n x dim, row-major). */
#define YAMS_B200_BATCH_ALL 0
#define YAMS_B200_BATCH_TOP_K 1
#define YAMS_B200_BATCH_FILTERED 2
YAMS_B200_API yams_status_t yams_b200_batch_distance(void* self, int metric, const float* query, uint32_t dim,
                                                     const float* database, uint64_t n, int mode, uint64_t k,
                                                     float threshold, uint64_t* out_idx, float* out_dist,
                                                     uint64_t* out_count);

/* VectorDatabase::computeCosineSimilarity (vector_database.cpp:1786-1810): double dot / (sqrt(na) * sqrt(nb)),
 * 0 on a size mismatch, an empty vector or a zero norm. Sequential double accumulation -> bit-identical. */
YAMS_B200_API yams_status_t yams_b200_compute_cosine_similarity(void* self, const float* a, size_t na,
                                                                const float* b, size_t nb, double* out);
/* The rerank loops that call computeCosineSimilarity once per candidate (sqlite_vec_backend.cpp:4025,4374,4507) as ONE
 * device pass: n pairs (a_i, b_i), row-major a[n][dim] and b[n][dim] HOST arrays -> out[n]. Same arithmetic per pair. */
YAMS_B200_API yams_status_t yams_b200_compute_cosine_similarity_many(void* self, const float* a, const float* b,
                                                                     size_t n, size_t dim, double* out);

/* ---- SimeonPqAdc engine (SURVEY.md §8f N3) -----------------------------------------------------------------
 * The reference's default engine (src/vector/sqlite_vec_backend.cpp:3868-4056): a product-quantised index over the
 * L2-normalised embeddings (third_party/simeon/include/simeon/pq.hpp:20-136: m sub-quantisers x k <= 256 centroids,
 * one byte per subspace), scanned with an asymmetric-distance lookup table per query, the best
 * max(k, k * rerank_factor) rows re-scored exactly.  Here the index lives beside a corpus: codes [rows][m] bytes in HBM
 * (32 B per row at the defaults, 1/48 of the fp16 corpus), the exact rerank reads the corpus rows.
 *   pq_build   rebuildSimeonPqIndex (:3540-3690) minus the training: rows with |row|^2 <= 1e-20 are left out, every other
 *              row is normalised like normalizeEmbeddingInPlace (:213-226) and encoded like ProductQuantizer::encode
 *              (simeon/src/pq.cpp:218-235) with the given codebooks [m][k][dim/m] (ProductQuantizer::import_codebooks; the
 *              k-means training of <= 4096 samples stays where it is).  tie_break_keys: nullable, one per corpus row (the
 *              FNV-1a of chunk_id the reference orders equal approximate scores by); NULL = row order.
 *   pq_search  simeonPqSearchUnlocked: normalised query, lookup table (simd::dot order of the x86 build), ADC scores as
 *              sequential float sums, best approxK by (score desc, tie key asc), exact double cosine of the ORIGINAL query
 *              against the stored row (computeCosineSimilarity), threshold, order (similarity desc, rowid asc; TIE_AT_K
 *              flag for the host's chunk_id re-break), k results.  Approximate scores, survivors and final scores are
 *              bit-identical to the reference engine.  A query that cannot be normalised returns nothing.
 * The index is invalidated by any corpus mutation (the reference marks it dirty): pq_search then returns INVALID_ARG. */
typedef struct yams_b200_pq yams_b200_pq;
YAMS_B200_API yams_status_t yams_b200_pq_build(yams_b200_corpus* c, uint32_t m, uint32_t k, const float* codebooks,
                                               const uint64_t* tie_break_keys, yams_b200_pq** out);
YAMS_B200_API yams_status_t yams_b200_pq_search(yams_b200_pq* pq, const float* queries, uint32_t nq, uint32_t k,
                                                uint32_t rerank_factor, float threshold, int64_t* out_rowids,
                                                float* out_scores, uint32_t* out_counts, uint64_t* out_flags);
/* simeonPqSearchUnlocked with candidateHashes, VectorTopK (sqlite_vec_backend.cpp:3910-4051): query i only scores the indexed
 * rows of allowed_rowids[allowed_offsets[i] .. allowed_offsets[i+1]) (the format of yams_b200_search, any order; a rowid listed
 * twice counts once; rowids unknown to the corpus or left out of the index are ignored).  candidateCount = the distinct indexed
 * candidates (0: no results), approxK = min(candidateCount, max(k, k * rerank_factor)) <= 1024.  After the ADC scores the chain
 * is pq_search's; with every indexed row in every list the results and flags are bit-identical to pq_search. */
YAMS_B200_API yams_status_t yams_b200_pq_search_candidates(yams_b200_pq* pq, const float* queries, uint32_t nq, uint32_t k,
                                                           uint32_t rerank_factor, float threshold,
                                                           const int64_t* allowed_rowids, const uint64_t* allowed_offsets,
                                                           int64_t* out_rowids, float* out_scores, uint32_t* out_counts,
                                                           uint64_t* out_flags);
/* CandidateFilterMode::DocumentTopK (vector_database.cpp:553-569): the k best DOCUMENTS of every query, each represented by its
 * best row (retainBestRecordPerDocument, sqlite_vec_backend.cpp:86-125).  Document d is the rows
 * doc_rowids[doc_offsets[d] .. doc_offsets[d+1]) in the caller's chunk order; query q considers documents
 * query_docs[q] .. query_docs[q+1] (nq + 1 entries) in the caller's document order.  Callers pass documents sorted by
 * document_hash and rows by chunk_id: the position tie-breaks below then are the reference's.
 *   pq == NULL  the exact fallback (:1508-1518, :3882-3893): every candidate row scored like yams_b200_search_all_matching
 *               (skip rules, threshold); a non-finite / zero query makes the call return YAMS_ERR_INVALID_ARG.
 *   pq != NULL  the PQ engine's DocumentTopK branch (:3957-3958, :4022-4048): every candidate row IN THE INDEX re-scored like
 *               pq_search's rerank (NaN and sim < threshold dropped); a query that cannot be normalised gets count 0.  The
 *               index must be current and belong to c.
 * A document's best row: (sim desc, position in the document asc); documents without a surviving row are absent; documents
 * ordered (best sim desc, document index asc), k <= 4096 returned per query.  Outputs Q x k: out_docs = document index,
 * out_rowids / out_scores = its best row and score; unused slots -1 / -1 / 0.  k == 0: all counts 0.  Unknown rowids are
 * ignored.  YAMS_ERR_INVALID_ARG before any device work for non-monotone offsets, a document of 2^32 - 1 rows or more, or a
 * rowid that appears twice among one query's documents. */
YAMS_B200_API yams_status_t yams_b200_search_documents(yams_b200_corpus* c, yams_b200_pq* pq, const float* queries, uint32_t nq,
                                                       uint32_t k, float threshold, const int64_t* doc_rowids,
                                                       const uint64_t* doc_offsets, const uint64_t* query_docs,
                                                       int64_t* out_docs, int64_t* out_rowids, float* out_scores,
                                                       uint32_t* out_counts);
/* the index content, for parity checks: out_codes [n_indexed][m], out_rowids [n_indexed] (both nullable), *out_n */
YAMS_B200_API yams_status_t yams_b200_pq_codes(yams_b200_pq* pq, uint8_t* out_codes, int64_t* out_rowids,
                                               uint64_t* out_n);
YAMS_B200_API void yams_b200_pq_destroy(yams_b200_pq* pq);

/* ---- Simeon text encoder, default profile (SURVEY.md §8f N4) ---------------------------------------------------
 * third_party/simeon Encoder::encode (src/simeon.cpp:190-262) for the profile YAMS runs (`simeon-v1-384`, src/simeon.cpp:75-93;
 * src/embedding_simeon/simeon_embedding_backend.cpp:118-135): byte n-grams of length ngram_min..ngram_max over the raw text,
 * SplitMix64 hashing, integer count sketch (+-2 per gram), Achlioptas sparse projection (int64 sums, one float scale),
 * L2 normalisation in the AVX2 tier's lane order.  Bit-identical to the reference encoder.  flags select the other recipe YAMS
 * runs: word tokens (CharAndWord) and the Fwht projection.  Other encoder modes (sub-word tokens, ASCII lowering, word-bounded
 * n-grams, IDF / PMI / sqrt-TF weighting, Gaussian / sparse-JL projections, matryoshka) are not served here. */
typedef struct yams_simeon_config {
    uint32_t ngram_min, ngram_max;     /* 3, 5 */
    uint32_t sketch_dim, output_dim;   /* 4096, 384 */
    uint64_t hash_seed;                /* 0xA5A5A5A5A5A5A5A5 */
    uint64_t projection_seed;          /* 0xDEADBEEFCAFEBABE */
    int32_t l2_normalize;              /* 1 */
    int32_t flags;                     /* YAMS_SIMEON_* below; 0 = the simeon-v1-384 recipe */
} yams_simeon_config;
/* NGramMode::CharAndWord (third_party/simeon/src/tokenizer.cpp:40-52): besides the byte n-grams, every maximal [A-Za-z0-9_]+
 * run is one feature of weight 0.5 (+-1 in the integer sketch) */
#define YAMS_SIMEON_WORD_TOKENS 1
/* ProjectionMode::Fwht (third_party/simeon/src/projection.cpp:149-186,359-374): sign diagonal, Walsh-Hadamard transform of the
 * zero-padded sketch, output_dim sampled coordinates scaled by 1/sqrt(output_dim); requires output_dim <= next_pow2(sketch_dim).
 * Without this flag the projection is AchlioptasSparse. */
#define YAMS_SIMEON_PROJECTION_FWHT 2
typedef struct yams_b200_encoder yams_b200_encoder;
/* simeon_v1_384_config (third_party/simeon/src/simeon.cpp:75-93): EmbeddingConfig::SimeonEncoderProfile::FixedHash384 */
YAMS_B200_API void yams_b200_simeon_default_config(yams_simeon_config* cfg);
/* the encoder YAMS builds when [embeddings.simeon] is left unconfigured (SimeonEncoderProfile::Configurable, the default;
 * /root/reference/src/embedding_simeon/simeon_embedding_backend.cpp:18-47,118-135): CharAndWord, n-grams 3..5, sketch 4096,
 * Fwht, output_dim = embedding_dim (0 -> 1024, EmbeddingConfig's default), L2-normalised */
YAMS_B200_API void yams_b200_simeon_yams_config(yams_simeon_config* cfg, uint32_t embedding_dim);
YAMS_B200_API yams_status_t yams_b200_simeon_create(void* self, const yams_simeon_config* cfg /* NULL = default */,
                                                    yams_b200_encoder** out);
/* IEmbeddingBackend::generateEmbeddings (simeon_embedding_backend.cpp:194-209): n HOST texts (bytes, not NUL-terminated)
 * -> out[n][output_dim] HOST floats, one device pass */
YAMS_B200_API yams_status_t yams_b200_simeon_encode(yams_b200_encoder* e, const char* const* texts, const size_t* lens,
                                                    size_t n, float* out);
YAMS_B200_API void yams_b200_simeon_destroy(yams_b200_encoder* e);

/* ---- Simeon BM25 lexical index (DESIGN.md §4.11) ----------------------------------------------------------------
 * third_party/simeon Bm25Index (src/bm25.cpp), as the lexical backend builds and scores it (SimeonLexicalBackend:
 * src/search/simeon_lexical_backend.cpp), for the two variants that backend selects: Atire and SubwordAwareBackoff.
 *   build  add_doc(text) for each document in order, then finalize(): words are the maximal runs of [A-Za-z0-9_] (bytes >= 0x80
 *          separate words), ASCII-lowercased and hashed with SplitMix64; dl = words of the document; SubwordAwareBackoff also
 *          indexes every n-gram (k = ngram_min..ngram_max, every position) of every lowercased word, ngram_dl = their count,
 *          and drops n-grams whose df exceeds size_t(double(prune_ratio) * n) (prune_ratio 0: none).  Posting lists are in
 *          document order; idf = logf((n - df + 0.5f) / (df + 0.5f) + 1.0f), avg_dl = float(double(sum dl) / n).
 *   score  for each query word in order (duplicates kept), Atire adds score_atire to every document of its posting list;
 *          SubwordAwareBackoff adds alpha * bm25plus over the word's list (alpha = df / (df + gamma), 0 when df = 0) when
 *          alpha > 0, and (1 - alpha) * bm25plus over the list of each distinct n-gram of the word still in the index when
 *          alpha < 1.  Every float operation is the reference's, in its order, without fused multiply-adds.
 * Scores are bit-identical to the reference.  The concept blend (ConceptIndex::blend_into) is the concepts block below.  The lead-text
 * aux field and the strategy router are yams_b200_bm25_build_lead and yams_b200_bm25_score_strategy; the query router is
 * yams_b200_bm25_score_routed.  Out of scope (the caller's, as today): fragment geometry, SDM / word bigrams, PRF, and the caller's document windowing (buildEnhancementText).  RRF over variants is
 * yams_b200_bm25_score_rrf. */
#define YAMS_BM25_ATIRE 0                    /* simeon::Bm25Variant::Atire */
#define YAMS_BM25_SUBWORD_AWARE_BACKOFF 7    /* simeon::Bm25Variant::SubwordAwareBackoff */
typedef struct yams_bm25_config {
    float k1, b, delta;           /* 1.2, 0.75, 1.0 */
    float subword_gamma;          /* 5 (the lexical backend's); alpha = df / (df + gamma) */
    uint32_t variant;             /* YAMS_BM25_*; any other value -> YAMS_ERR_UNSUPPORTED */
    uint32_t ngram_min, ngram_max;   /* 3, 4 */
    float ngram_df_prune_ratio;   /* 0.5 */
    uint64_t hash_seed;           /* 0xB252B252B252B252 */
} yams_bm25_config;
typedef struct yams_b200_bm25 yams_b200_bm25;
/* the lexical backend's configuration: SubwordAwareBackoff, gamma 5, Bm25Config's defaults otherwise */
YAMS_B200_API void yams_b200_bm25_default_config(yams_bm25_config* cfg);
/* builds and finalizes an index of n_docs HOST texts (bytes, not NUL-terminated; a NULL text of length 0 is an empty document;
 * n_docs = 0 is an empty index).  Corpora larger than one device pass are built in document slices; beyond device memory the
 * call fails with YAMS_ERR_INTERNAL and says so.  n_docs < 2^32 - 1. */
YAMS_B200_API yams_status_t yams_b200_bm25_build(void* self, const yams_bm25_config* cfg /* NULL = default */,
                                                 const char* const* texts, const size_t* lens, uint64_t n_docs,
                                                 yams_b200_bm25** out);
/* Bm25Index::score for nq HOST queries.  out_scores (nullable): [nq][n_docs] HOST floats, the full score vectors.  k > 0
 * (<= 4096): the documents of score > 0, best first (score descending, then document ascending), k of them at most ->
 * out_docs[nq][k] (padded with 0xFFFFFFFF), out_topk_scores[nq][k] (padded with 0), out_counts[nq]. */
YAMS_B200_API yams_status_t yams_b200_bm25_score(yams_b200_bm25* idx, const char* const* queries, const size_t* qlens, uint32_t nq,
                                                 float* out_scores, uint32_t k, uint32_t* out_docs, float* out_topk_scores,
                                                 uint32_t* out_counts);
typedef struct yams_bm25_stats {
    uint64_t n_docs;
    float avg_dl, ngram_avg_dl;   /* ngram_avg_dl: 0 for Atire */
    uint64_t total_tokens;        /* sum of dl */
    uint64_t terms[2];            /* distinct hashes of field 0 (words) and 1 (n-grams, after pruning) */
    uint64_t postings[2];         /* (term, document) entries per field */
    uint64_t pruned;              /* n-grams dropped by the df rule */
} yams_bm25_stats;
YAMS_B200_API yams_status_t yams_b200_bm25_stats(yams_b200_bm25* idx, yams_bm25_stats* out);
/* the posting list of term_hash in field 0 (words), 1 (n-grams), 2 (lead words) or 3 (lead n-grams): *out_df (0 when absent), *out_idf, *out_total_tf, and the
 * first min(df, cap) (document, tf) entries in document order (out_docs / out_tfs nullable when cap = 0).  Bm25Index::df /
 * idf / total_tf of a term are these of field 0 for the term's hash. */
YAMS_B200_API yams_status_t yams_b200_bm25_postings(yams_b200_bm25* idx, uint32_t field, uint64_t term_hash, uint32_t* out_df,
                                                    float* out_idf, uint64_t* out_total_tf, uint32_t* out_docs, uint32_t* out_tfs,
                                                    uint64_t cap);
/* dl (field 0), ngram_dl (field 1, zeros for Atire) or the lead field's (2, 3; zeros without an active lead field) of every
 * document -> out[n_docs] (HOST) */
YAMS_B200_API yams_status_t yams_b200_bm25_doc_lengths(yams_b200_bm25* idx, uint32_t field, uint32_t* out);
/* out_ms[0..3]: the last build's device ms of the upload, the tokenising (per-document counts, words, n-gram pairs), the sorts,
 * the posting lists (runs, pruning, dictionary), [4] its host wall ms, [5] its document slices; [6] the last score call's
 * device ms, [7] its host wall ms */
YAMS_B200_API yams_status_t yams_b200_bm25_last_timings(yams_b200_bm25* idx, float out_ms[8]);
YAMS_B200_API void yams_b200_bm25_destroy(yams_b200_bm25* idx);
/* An Atire view of idx -> *out: a handle that answers every yams_b200_bm25_* call and yams_b200_concepts_mine exactly as an
 * Atire index built from the same texts with idx's k1, b and hash_seed would (SimeonLexicalBackend's second index for RRF, built
 * with Bm25Config's defaults otherwise).  Such an index's word field and idf table are idx's, whatever idx's variant: n-grams
 * and their pruning never touch words.  The view reads them in place, with no copy and no build; its n-gram field is empty
 * (stats: ngram_avg_dl, terms[1], postings[1] and pruned 0; field 1 postings and doc lengths empty and zero).  A view of an
 * Atire index is equivalent to the index.  The view has its own stream, lock and score workspace, so it may be scored
 * concurrently with idx, and the two may be destroyed in either order. */
YAMS_B200_API yams_status_t yams_b200_bm25_atire_view(yams_b200_bm25* idx, yams_b200_bm25** out);

/* ---- the lead-text field (DESIGN.md §4.14) ----------------------------------------------------------------------
 * yams_b200_bm25_build with Bm25Index::add_doc(text, extract_lead_tokens(text, lead_tokens)) for each document, as the lexical
 * backend builds with strategy_router_enabled (lead_tokens 64).  The lead text is the text up to the whitespace byte (C-locale
 * isspace) that ends its lead_tokens-th whitespace-delimited token (all of it when it has fewer), whitespace turned into ' ',
 * trailing spaces trimmed.  It is indexed as an aux word field (field 2) and, for SubwordAwareBackoff, an aux n-gram field
 * (field 3), with their own lengths, averages and n-gram pruning.  The aux field is active from the first document whose lead
 * text is non-empty, earlier documents counting length 0, so it exists for all documents or for none (every lead text empty).
 * lead_tokens = 0 is yams_b200_bm25_build.  An Atire view (yams_b200_bm25_atire_view) shares the aux word field. */
YAMS_B200_API yams_status_t yams_b200_bm25_build_lead(void* self, const yams_bm25_config* cfg /* NULL = default */,
                                                      const char* const* texts, const size_t* lens, uint64_t n_docs,
                                                      uint32_t lead_tokens, yams_b200_bm25** out);
/* the aux fields' yams_bm25_stats: n_docs (n_docs when the aux field is active, else 0), avg_dl / ngram_avg_dl, total_tokens,
 * terms / postings of fields 2 and 3, and the aux n-grams the df rule dropped */
YAMS_B200_API yams_status_t yams_b200_bm25_aux_stats(yams_b200_bm25* idx, yams_bm25_stats* out);

/* ---- Simeon word-bigram concepts (DESIGN.md §4.12) ---------------------------------------------------------------
 * third_party/simeon ConceptIndex (src/concept_mining.cpp) mined against a BM25 index, and its blend into BM25 scores, as the
 * lexical backend configures them (concept mining on, concept_weight 0.5).
 *   mine   words as in the index but hashed WITHOUT case folding; a document of w >= 2 words has the w - 1 ordered bigrams
 *          hash_bigram(a, b) and bigram_dl = w - 1 (else 0); avg = float(double(sum bigram_dl) / n).  Nothing is kept when the
 *          index has no tokens or no document has a bigram.  A bigram is kept when total_tf >= min_ttf, both words of its first
 *          occurrence are in the index (their index total_tf: an uppercase word never is), and pmi = log((ttf / sum_bdl) /
 *          ((tf_a / T) * (tf_b / T))) is finite and >= pmi_floor (T = the index's total_tokens); over max_concepts, the highest
 *          float pmi are kept, and a tie across the cut is settled as the reference settles it (std::nth_element over its map's
 *          order).  idf = logf((n - df + 0.5f) / (df + 0.5f) + 1.0f).
 *   blend  for queries of >= 2 (unfolded) words, each distinct adjacent bigram that is a concept, in the reference's order, adds
 *          weight * pmi * score_atire(tf, bigram_dl, idf, k1, b, avg) to each document of its posting list.
 * Everything is bit-identical to the reference.  One device pass: beyond device memory the call fails with YAMS_ERR_INTERNAL
 * (about 16 bytes per word pair plus the sort's double buffer and the postings). */
typedef struct yams_concept_config {
    uint32_t min_ttf;             /* 5 */
    float pmi_floor;              /* 2.0 */
    uint32_t max_concepts;        /* 200 000 */
    float k1, b;                  /* 1.2, 0.75 */
} yams_concept_config;
typedef struct yams_b200_concepts yams_b200_concepts;
YAMS_B200_API void yams_b200_concepts_default_config(yams_concept_config* cfg);
/* mine_concepts(idx, texts, cfg) over n_docs HOST texts (they may differ from the index's, as the backend's raw texts do; NULL
 * text of length 0 = empty).  The handle owns what it needs (hash seed included) and may outlive idx.  n_docs < 2^32 - 1. */
YAMS_B200_API yams_status_t yams_b200_concepts_mine(yams_b200_bm25* idx, const yams_concept_config* cfg /* NULL = default */,
                                                    const char* const* texts, const size_t* lens, uint64_t n_docs,
                                                    yams_b200_concepts** out);
/* yams_b200_bm25_score, then ConceptIndex::blend_into(query, scores, weight) of each query before the top-k: the same outputs
 * and limits.  concepts NULL, empty, or of another document count than idx: no blend (the reference's size test). */
YAMS_B200_API yams_status_t yams_b200_bm25_score_blended(yams_b200_bm25* idx, const yams_b200_concepts* concepts, float weight,
                                                         const char* const* queries, const size_t* qlens, uint32_t nq,
                                                         float* out_scores, uint32_t k, uint32_t* out_docs, float* out_topk_scores,
                                                         uint32_t* out_counts);
/* ConceptIndex::blend_into(query, inout_scores[n], weight) on a HOST vector: a no-op unless n == doc_count */
YAMS_B200_API yams_status_t yams_b200_concepts_blend(yams_b200_concepts* concepts, const char* query, size_t qlen, float weight,
                                                     float* inout_scores, uint64_t n);
typedef struct yams_concepts_stats {
    uint64_t size;                /* kept concepts */
    uint64_t doc_count;
    float avg_bigram_dl;
    uint32_t replayed;            /* 1: a pmi tie crossed max_concepts and the reference's selection order was replayed */
    uint64_t sum_bigram_dl;
    uint64_t distinct;            /* distinct bigram hashes */
    uint64_t passed_min_ttf;      /* of these, total_tf >= min_ttf */
    uint64_t accepted;            /* accepted before the cap */
} yams_concepts_stats;
YAMS_B200_API yams_status_t yams_b200_concepts_stats(yams_b200_concepts* concepts, yams_concepts_stats* out);
/* ConceptIndex::find(hash): *found 0/1; pmi, idf, total_tf, a_hash, b_hash, df and the first min(df, cap) (document, tf)
 * postings in document order (out_docs / out_tfs nullable when cap = 0) */
YAMS_B200_API yams_status_t yams_b200_concepts_find(yams_b200_concepts* concepts, uint64_t hash, uint32_t* found, float* pmi, float* idf,
                                                    uint64_t* total_tf, uint64_t* a_hash, uint64_t* b_hash, uint32_t* df,
                                                    uint32_t* out_docs, uint32_t* out_tfs, uint64_t cap);
/* the kept concepts' hashes, ascending -> out[size] (HOST) */
YAMS_B200_API yams_status_t yams_b200_concepts_hashes(yams_b200_concepts* concepts, uint64_t* out);
/* bigram_dl of every document -> out[doc_count] (HOST) */
YAMS_B200_API yams_status_t yams_b200_concepts_bigram_lengths(yams_b200_concepts* concepts, uint32_t* out);
/* out_ms: the mining's device ms of [0] the upload, [1] the tokenising (words, pairs), [2] the sort, [3] the runs and the filter,
 * [4] the gather of the kept postings; [5] its host ms of the log, the floor and the cap, [6] of the replay alone (0 when it did
 * not run), [7] its host wall ms */
YAMS_B200_API yams_status_t yams_b200_concepts_last_timings(yams_b200_concepts* concepts, float out_ms[8]);
YAMS_B200_API void yams_b200_concepts_destroy(yams_b200_concepts* concepts);

/* ---- reciprocal-rank fusion of BM25 variants (DESIGN.md §4.13) ---------------------------------------------------
 * score_bm25_variants_rrf(variants, query, scores, k_rrf) of each of nq HOST queries (fusion.cpp), then, with concepts,
 * ConceptIndex::blend_into(query, scores, weight): SimeonLexicalBackend::score with bm25_variants_rrf on.  Each variant, in the
 * given order, ranks the documents of finite score > 0 by score descending, then document ascending; rank r (1, 2, ...) adds
 * 1.0f / (k_rrf + (float)r) to its document, the variants' additions in their order from 0.0f (an unranked document stays 0).
 * The blend adds onto the fused scores.  Outputs and limits are yams_b200_bm25_score's.  Bit-identical to the reference; ranks
 * above 2^24, where (float)r rounds, need more than 16.7 M documents and are not tested.
 *   - The same index may appear more than once (its ranks then count twice).  Every distinct index is locked for the call, in
 *     an order that cannot deadlock; the work runs on the first variant's stream and workspace, whose last_timings [6] and [7]
 *     record it.  Queries are batched so that the score rows, ranked keys and the sort's double buffer stay within 1 GiB.
 *   - YAMS_ERR_INVALID_ARG: a null index, indexes of different document counts, k_rrf not finite or < 0 (the backend passes
 *     60), k > 4096, nv * n_docs >= 2^32.  YAMS_ERR_UNSUPPORTED: indexes on different devices.
 *   - nv = 0: nothing is ranked and there is no document count: no score row is written, every count is 0.
 *   - concepts NULL, empty or of another document count: no blend (as yams_b200_bm25_score_blended). */
YAMS_B200_API yams_status_t yams_b200_bm25_score_rrf(const yams_b200_bm25* const* variants, uint32_t nv, float k_rrf,
                                                     const yams_b200_concepts* concepts, float weight, const char* const* queries,
                                                     const size_t* qlens, uint32_t nq, float* out_scores, uint32_t k,
                                                     uint32_t* out_docs, float* out_topk_scores, uint32_t* out_counts);

/* ---- the strategy router (DESIGN.md §4.14) ----------------------------------------------------------------------
 * The strategy router's pools over an index built with the lead field and its route, as the lexical backend constructs them (simeon_lexical_backend.cpp:563-580):
 *   YAMS_BM25_STRATEGY_BM25        pool 0, Bm25Strategy: score_bm25f(q, lead(q, 64), 0.85, 0.15), or Bm25Index::score(q) when
 *                                  the query's lead text is empty;
 *   YAMS_BM25_STRATEGY_LEAD_FIELD  pool 2, LeadFieldStrategy (the "lead_field" bandit arm): score_bm25f(q, q, 0.85, 0.15).
 * score_bm25f(body, aux, wb, wa): the body score, times wb, then the aux legs -- SubwordAwareBackoff adds (wa * alpha) *
 * bm25plus over the aux query's words in field 2 and (wa * (1 - alpha)) * bm25plus over their n-grams in field 3, alpha from the
 * field-2 df; Atire adds wa * score_atire over field 2.  An index built without the lead field has empty aux fields: wb * body.
 *   YAMS_BM25_STRATEGY_KEYPHRASE   pool 1, KeyphraseStrategy(0.25, 0.30) (the "keyphrase" bandit arm): the plain score; the
 *                                  normalised softmax entropy (double) of simeon::top_k(scores, 10), which keeps zero scores;
 *                                  below 0.30f, or without keyphrases (alphabetic runs of >= 2 bytes, lowercased, stopwords
 *                                  dropped), the plain score; else the z-score (two sequential double sums over the n scores)
 *                                  plus (lam * 0.25f) * (matches / keyphrases), lam = 1 / (1 + expf(-(entropy - 0.48f) * 8)), a
 *                                  document matching a keyphrase when its single-term score is > 0.  Scores may be negative.
 *   YAMS_BM25_STRATEGY_ROUTED      SimeonLexicalBackend::scoreStrategyRouted: bm25_entropy = float(sum over the documents of
 *                                  plain score s > 0, in document order, of sn * -log(sn), sn = (double)(s / max), over their
 *                                  count); < 0.05f -> pool 0, > 0.50f -> pool 2, else pool 1.  The device's profile comes with a
 *                                  bound on its distance from the reference's; a row whose route the bound cannot settle is
 *                                  copied back and the backend's loop replayed with std::log.  YAMS_B200_BM25_ROUTE_MARGIN = w > 0,
 *                                  read at every call, widens the entropy's interval by w (1 replays every row with a positive score).
 * score_bm25f(body, aux, wb, wa): the body score, times wb, then the aux legs -- SubwordAwareBackoff adds (wa * alpha) *
 * bm25plus over the aux query's words in field 2 and (wa * (1 - alpha)) * bm25plus over their n-grams in field 3, alpha from the
 * field-2 df; Atire adds wa * score_atire over field 2.  An index built without the lead field has empty aux fields: wb * body. */
#define YAMS_BM25_STRATEGY_BM25 0
#define YAMS_BM25_STRATEGY_KEYPHRASE 1
#define YAMS_BM25_STRATEGY_LEAD_FIELD 2
#define YAMS_BM25_STRATEGY_ROUTED 3
/* The strategy's scores of nq HOST queries, then, with concepts, ConceptIndex::blend_into(query, scores, weight): the outputs,
 * limits and locking of yams_b200_bm25_score_blended, bit-identical to the reference.  out_chosen (nullable): [nq] the pool
 * each query took.  KEYPHRASE and ROUTED batch queries so that their score rows and match rows stay within 1 GiB; all pools
 * of a batch run together, each row getting its own pool's legs.  strategy > 3: YAMS_ERR_INVALID_ARG. */
YAMS_B200_API yams_status_t yams_b200_bm25_score_strategy(yams_b200_bm25* idx, uint32_t strategy, const yams_b200_concepts* concepts,
                                                          float weight, const char* const* queries, const size_t* qlens, uint32_t nq,
                                                          float* out_scores, uint32_t k, uint32_t* out_docs, float* out_topk_scores,
                                                          uint32_t* out_counts, uint32_t* out_chosen);
typedef struct yams_bm25_strategy_stats {   /* of the index's last yams_b200_bm25_score_strategy call */
    uint32_t queries[3];          /* queries scored by pool 0, 1, 2 */
    uint32_t replayed;            /* ROUTED rows whose route was replayed on the host */
    uint32_t keyphrase_boosted;   /* pool-1 rows past the gate (z-scored and boosted) */
    float zscore_ms;              /* device ms of the z-score kernel */
    float device_ms, wall_ms;     /* the call's device and host wall ms */
} yams_bm25_strategy_stats;
YAMS_B200_API yams_status_t yams_b200_bm25_strategy_stats(yams_b200_bm25* idx, yams_bm25_strategy_stats* out);

/* ---- the query router (DESIGN.md §4.15) -------------------------------------------------------------------------
 * SimeonLexicalBackend::scoreRouted with router_enabled (fragment geometry and RRF off): simeon::QueryRouter::features(query) and
 * choose(features) over the index's field 0 (query_router.cpp:29-117, 222-238), the chosen index's scores -- Atire for
 * Bm25Atire (an Atire view of idx, yams_b200_bm25_atire_view), idx for Bm25SabSmooth and CascadeLinearAlpha; every recipe scores
 * Atire when idx is Atire -- then, with concepts, ConceptIndex::blend_into(query, scores, weight), then the projection onto the
 * caller's candidate pool.
 *   features  the query's words (maximal runs of [A-Za-z0-9_]) hashed WITHOUT case folding: a word with an uppercase letter is
 *             out of vocabulary for the router (df 0) although scoring folds it.  n_terms and avg_term_chars count every
 *             occurrence; scq_sum adds (1 + log(total_tf)) * idf per present occurrence; simplified_clarity sums, over the distinct
 *             present hashes in first-occurrence order, p_q * log(p_q / p_c), p_q = occurrences / n_terms (OOV words counted in
 *             n_terms), p_c = total_tf / total_tokens; idf_stddev is computed only with more than one present occurrence.  Every
 *             operation is the reference's, in its order, in double with glibc log, and so is the route.
 *   choose    the pool-based signals keep features()'s no-signal defaults (pool_overlap_jaccard 1, score_decay_rate 0) and are
 *             compared with atire_max_pool_jaccard and atire_min_score_decay as the reference compares them. */
#define YAMS_BM25_RECIPE_ATIRE 0              /* simeon::Recipe::Bm25Atire */
#define YAMS_BM25_RECIPE_SAB_SMOOTH 1         /* simeon::Recipe::Bm25SabSmooth */
#define YAMS_BM25_RECIPE_CASCADE 2            /* simeon::Recipe::CascadeLinearAlpha */
typedef struct yams_bm25_router_config {      /* simeon::RouterConfig's routing fields */
    float oov_threshold, high_idf_threshold;  /* 0, 3 */
    uint32_t atire_min_terms;                 /* 0 */
    float atire_min_idf_floor, atire_max_pool_jaccard, atire_min_score_decay, atire_min_scq, atire_max_clarity;   /* 0, 1, 0, 0, 3 */
    uint32_t cascade_min_terms;               /* 4 */
    float cascade_max_idf;                    /* 5 */
} yams_bm25_router_config;
typedef struct yams_bm25_query_features {     /* the fields simeon::QueryRouter::features fills */
    float oov_rate, avg_idf, max_idf, min_idf, idf_stddev;
    uint32_t n_terms;
    float avg_term_chars, scq_sum, simplified_clarity;
} yams_bm25_query_features;
/* the lexical backend's RouterPreset (passE: atire_max_clarity 3) over RouterConfig's defaults */
YAMS_B200_API void yams_b200_bm25_default_router_config(yams_bm25_router_config* cfg);
/* The routed scores of nq HOST queries: the outputs, top-k rule, limits, locking and 1 GiB batching of
 * yams_b200_bm25_score_blended; rows of different recipes share a batch.  out_recipe (nullable): [nq] YAMS_BM25_RECIPE_*;
 * out_features (nullable): [nq].
 * Candidate pools (cand_offsets nullable: none): query q's pool is cand_docs[cand_offsets[q] .. cand_offsets[q + 1]) (document
 * indices; 0xFFFFFFFF = a candidate the index does not hold), cand_offsets[0] = 0, non-decreasing; out_cand_scores[j] =
 * isfinite(row[d]) ? row[d] : 0, 0 for 0xFFFFFFFF -- gathered on the device, so with out_scores NULL and k = 0 only the pools
 * cross to the host.  A pool may repeat a document and be longer than n_docs.  A candidate index >= n_docs other than
 * 0xFFFFFFFF: YAMS_ERR_INVALID_ARG. */
YAMS_B200_API yams_status_t yams_b200_bm25_score_routed(yams_b200_bm25* idx, const yams_bm25_router_config* rcfg /* NULL = default */,
                                                        const yams_b200_concepts* concepts, float weight, const char* const* queries,
                                                        const size_t* qlens, uint32_t nq, float* out_scores, uint32_t k, uint32_t* out_docs,
                                                        float* out_topk_scores, uint32_t* out_counts, const uint64_t* cand_offsets,
                                                        const uint32_t* cand_docs, float* out_cand_scores, uint32_t* out_recipe,
                                                        yams_bm25_query_features* out_features);

/* [0] stage-1 scan ms, [1] rescoring+select ms, [2] total device ms of the last yams_b200_search or
 * yams_b200_search_device on this corpus (the latter's once its work is done); [3] unused (0);
 * [4] = which stage-1 kernel ran (0 cuda-core, 1 wgmma);
 * [5] = duration of the full-corpus filtered scan launch alone (the dominant kernel);
 * [6] = queries of that call the certificate sent to the exhaustive levels, [7] = of those, the queries level 1 could not
 * certify either, answered by the full exact pass ([6] and [7] of a search_device: set by yams_b200_search_device_finish) */
YAMS_B200_API yams_status_t yams_b200_search_last_timings(yams_b200_corpus* c, float out_ms[8]);

typedef struct yams_vector_scan_v1 {
    uint32_t abi_version; /* YAMS_IFACE_VECTOR_SCAN_V1_VERSION */
    void* self;
    yams_status_t (*corpus_create)(void* self, uint32_t dim, int dtype, int metric,
                                   uint64_t capacity_hint, yams_b200_corpus** out);
    yams_status_t (*corpus_append)(yams_b200_corpus* c, const void* rows, uint64_t n,
                                   const int64_t* rowids);
    yams_status_t (*corpus_clear)(yams_b200_corpus* c);
    yams_status_t (*corpus_size)(const yams_b200_corpus* c, uint64_t* out_n);
    void (*corpus_destroy)(yams_b200_corpus* c);
    yams_status_t (*search)(yams_b200_corpus* c, const float* queries, uint32_t nq, uint32_t k,
                            float threshold, const int64_t* allowed_rowids,
                            const uint64_t* allowed_offsets, int64_t* out_rowids, float* out_scores,
                            uint32_t* out_counts, uint64_t* out_flags);
    yams_status_t (*vec0_exact)(void* self, const float* query, uint32_t dim, const float* rows,
                                const int64_t* rowids, uint64_t n, uint64_t k, int use_range,
                                int64_t rowid_lo, int64_t rowid_hi, int64_t* out_rowids,
                                float* out_dist, uint64_t* out_count);
    yams_status_t (*corpus_remove)(yams_b200_corpus* c, const int64_t* rowids, uint64_t n,
                                   uint64_t* out_removed);
    yams_status_t (*search_all_matching)(yams_b200_corpus* c, const float* query, float threshold,
                                         const int64_t* allowed_rowids, uint64_t n_allowed,
                                         int64_t* out_rowids, float* out_scores, uint64_t* out_count);
    yams_status_t (*batch_distance)(void* self, int metric, const float* query, uint32_t dim,
                                    const float* database, uint64_t n, int mode, uint64_t k,
                                    float threshold, uint64_t* out_idx, float* out_dist,
                                    uint64_t* out_count);
    yams_status_t (*compute_cosine_similarity)(void* self, const float* a, size_t na, const float* b,
                                               size_t nb, double* out);
    yams_status_t (*compute_cosine_similarity_many)(void* self, const float* a, const float* b, size_t n,
                                                    size_t dim, double* out);
    yams_status_t (*search_exhaustive)(yams_b200_corpus* c, const float* queries, uint32_t nq, uint32_t k,
                                       float threshold, int64_t* out_rowids, float* out_scores,
                                       uint32_t* out_counts, uint64_t* out_flags);
    yams_status_t (*pq_build)(yams_b200_corpus* c, uint32_t m, uint32_t k, const float* codebooks,
                              const uint64_t* tie_break_keys, yams_b200_pq** out);
    yams_status_t (*pq_search)(yams_b200_pq* pq, const float* queries, uint32_t nq, uint32_t k,
                               uint32_t rerank_factor, float threshold, int64_t* out_rowids, float* out_scores,
                               uint32_t* out_counts, uint64_t* out_flags);
    void (*pq_destroy)(yams_b200_pq* pq);
    yams_status_t (*pq_search_candidates)(yams_b200_pq* pq, const float* queries, uint32_t nq, uint32_t k,
                                          uint32_t rerank_factor, float threshold, const int64_t* allowed_rowids,
                                          const uint64_t* allowed_offsets, int64_t* out_rowids, float* out_scores,
                                          uint32_t* out_counts, uint64_t* out_flags);
    yams_status_t (*search_documents)(yams_b200_corpus* c, yams_b200_pq* pq, const float* queries, uint32_t nq,
                                      uint32_t k, float threshold, const int64_t* doc_rowids, const uint64_t* doc_offsets,
                                      const uint64_t* query_docs, int64_t* out_docs, int64_t* out_rowids,
                                      float* out_scores, uint32_t* out_counts);
    yams_status_t (*semantic_neighbors)(yams_b200_corpus* c, const int64_t* source_rowids, uint64_t n_sources, uint32_t k,
                                        float threshold, int64_t* out_rowids, float* out_sims, uint32_t* out_counts,
                                        uint64_t* out_flags);
} yams_vector_scan_v1;

/* ---- sqlite-vec-cpp C API kept bit-for-bit in signature and error behaviour ------------------
 * third_party/sqlite-vec-cpp/src/sqlite_vec_c_api.cpp:57-105 (declared sqlite_vec.hpp:34-50):
 * sizes in BYTES, returns SQLITE_OK(0) / SQLITE_ERROR(1) on null pointer or dimension mismatch.
 * The library has no CPU arithmetic at all: a pair is evaluated by one device thread in the operation order of the
 * reference build (csrc/ref_order.cuh), through a pooled workspace (pinned staging + stream; no allocation per call).
 * One pair costs a launch round trip (~20 us) -- callers with many pairs should use yams_b200_batch_distance /
 * yams_b200_compute_cosine_similarity_many.  The SQL registration (sqlite3_vec_init, vec_distance_l2/cosine/l1 scalar
 * functions) is csrc/sqlite_glue.cpp, compiled only where sqlite3.h exists (INTEGRATION.md §4). */
YAMS_B200_API int sqlite3_vec_distance_l2(const void* vec1, size_t size1, const void* vec2,
                                          size_t size2, float* result);
YAMS_B200_API int sqlite3_vec_distance_cosine(const void* vec1, size_t size1, const void* vec2,
                                              size_t size2, float* result);
/* same contract for the L1 metric of the SQL scalar vec_distance_l1 (sqlite/functions.hpp:144-208, distances/l1.hpp:62-92);
 * the reference C API has no such symbol -- the SQL glue (csrc/sqlite_glue.cpp) needs it */
YAMS_B200_API int yams_b200_vec_distance_l1(const void* vec1, size_t size1, const void* vec2, size_t size2,
                                            float* result);

/* ---- bench / test utilities (SURVEY.md §8d synthetic inputs, generated straight into HBM) ------ */
/* byte[i] = (splitmix64(seed ^ (i>>3)) >> (8*(i&7))) & 0xFF for stream positions [start, start+n) */
YAMS_B200_API yams_status_t yams_b200_synth_bytes_device(uint64_t seed, uint64_t start, uint64_t n,
                                                         uint8_t* d_out);

/* rows [first_row, first_row + n) of the synthetic vector generator (x = (splitmix64(seed ^ (row*dim + c)) >> 40) * 2^-23 - 1,
 * L2-normalised in fp32; bit-identical to oracle yo_gen_rows_f32) as fp32 into a DEVICE buffer of n x dim floats */
YAMS_B200_API yams_status_t yams_b200_synth_rows_device(uint64_t seed, uint64_t first_row, uint64_t n, uint32_t dim,
                                                        float* d_out);

/* diagnostics: dense stage-1 (approximate) scores of rows row_start + i*row_stride, i < nrows, with the
 * chosen engine (0 = CUDA-core, 1 = wgmma); out[q * nrows + i] on the HOST. YAMS_ERR_UNSUPPORTED when the
 * engine cannot take the shape. */
YAMS_B200_API yams_status_t yams_b200_debug_stage1_scores(yams_b200_corpus* c, const float* queries, uint32_t nq,
                                                          int engine, uint64_t row_start, uint64_t row_stride,
                                                          uint64_t nrows, float* out);

/* diagnostics: the same rows and engines in FILTER mode, the candidate lists of the search's corpus pass.  Row i is
 * listed for query q when its stage-1 score is > tau[q] (and, with allowed lists in the format of yams_b200_search, the row
 * is in query q's set).  out_counts[q] = rows that passed (NOT capped at cap); out_cands[q * cap + j], j < min(count, cap),
 * = (float score, uint32 row index) pairs, 8 bytes each, in no particular order (HOST). YAMS_ERR_UNSUPPORTED when the
 * engine cannot take the shape.  engine = 2 is the gather engine of small ascending candidate sets: it scores every entry of
 * the allowed lists (each at most cap long) and ignores tau and the row range; out_counts[q] = list length, out_cands[q * cap
 * + j] = list entry j, (-inf, 0xFFFFFFFF) for a rowid that is unknown or repeats the previous entry. */
YAMS_B200_API yams_status_t yams_b200_debug_stage1_candidates(yams_b200_corpus* c, const float* queries, uint32_t nq,
                                                              int engine, uint64_t row_start, uint64_t row_stride,
                                                              uint64_t nrows, const float* tau, uint32_t cap,
                                                              const int64_t* allowed_rowids,
                                                              const uint64_t* allowed_offsets, uint32_t* out_counts,
                                                              void* out_cands);

/* diagnostics: one pass of the wgmma scan's profiling instantiation in filter mode over every row, as the search's corpus
 * pass runs it (thresholds tau[q], lists of cap entries).  out_cycles[4 * b + i] for CTA b < out_info[1] (<= max_ctas):
 * i = 0 cycles the first consumer warp waited for data (full barriers), 1 cycles the producer waited for a free stage
 * (empty barriers), 2 the first consumer warp's epilogue cycles, 3 its total cycles.  out_info[0] = query-tile columns,
 * out_info[1] = CTAs launched; out_ms = device time of the profiled launch (the counters slow it slightly). */
YAMS_B200_API yams_status_t yams_b200_debug_stage1_profile(yams_b200_corpus* c, const float* queries, uint32_t nq,
                                                           const float* tau, uint32_t cap, uint32_t max_ctas,
                                                           uint64_t* out_cycles, uint32_t* out_info, float* out_ms);

/* diagnostics: the search's top-K selection on caller-supplied scores (HOST in and out).  Input per query q, either
 *   dense (dense != NULL): dense[q * ld + i], i < len, row index row_start + i * row_stride; the device copy starts
 *                          dense_shift (0..3) floats past a 16-byte boundary, or
 *   lists: cands[q * cap + j] (float score, uint32 row) pairs, j < min(counts[q], cap), counts[q] may exceed cap; tau
 *          (nullable) bounds the scores of rows that never reached a list.
 * tau_only = 0: out_sel[q * K + j] = the K best (score desc, row asc) pairs, out_n[q] their number, out_bound[q] = an upper
 *               bound of every unselected score (K-th score when the input is longer than K, else tau[q] or -inf; +inf when
 *               counts[q] > cap); K <= 4096.
 * tau_only = 1: out_bound[q] = the K-th best score - tau_margin (-inf when fewer than K); fast_tau as in the threshold
 *               calibration of the corpus pass (K <= 16, len >= 4096: the K-th of the 256 per-thread maxima). */
YAMS_B200_API yams_status_t yams_b200_debug_select(yams_b200_corpus* c, uint32_t nq, const float* dense, uint64_t ld,
                                                   uint64_t len, uint64_t row_start, uint64_t row_stride, uint32_t dense_shift,
                                                   const void* cands, const uint32_t* counts, uint32_t cap, const float* tau,
                                                   uint32_t K, int tau_only, float tau_margin, int fast_tau, void* out_sel,
                                                   uint32_t* out_n, float* out_bound);

/* diagnostics: the search's final ordering and exactness certificate on caller-supplied exact scores (HOST in and out).
 * exact[q * Kp + i], i < (ex_n ? ex_n[q] : Kp): (float sim, uint32 row) pairs, NaN sim = no entry, row indexes this corpus's
 * rowid table; bound[q], eps[q], qnorm[q] (double, L2) are the certificate inputs; level 0 or 1 as in the exhaustive chain
 * (level 1 always flags the fallback).  Out: the k best by (sim desc, row asc) as rowids / scores (L2: negated sims = distances),
 * padded with -1 and -inf (L2: +inf), counts, flags, and the queries the certificate queued (out_queued[nq], in queue order). */
YAMS_B200_API yams_status_t yams_b200_debug_final(yams_b200_corpus* c, uint32_t nq, uint32_t Kp, uint32_t k, const void* exact,
                                                  const uint32_t* ex_n, const float* bound, const float* eps,
                                                  const double* qnorm, float threshold, int metric, int level,
                                                  int64_t* out_rowids, float* out_scores, uint32_t* out_counts,
                                                  uint64_t* out_flags, uint32_t* out_queued, uint32_t* out_n_queued);

/* diagnostics: the per-query stage-1 error bound eps[q] of the last search / debug_stage1_scores call (HOST out) */
YAMS_B200_API yams_status_t yams_b200_debug_last_eps(yams_b200_corpus* c, uint32_t nq, float* out);

/* diagnostics: the PQ lookup tables of pq_search (normalised query, LUT[mi][ki] = dot(q_sub, centroid)) of nq queries (HOST
 * in and out): out_lut[q * m * k + mi * k + ki], out_valid[q] = 0 when the query cannot be normalised (its table is then
 * not used by a search). */
YAMS_B200_API yams_status_t yams_b200_debug_pq_lut(yams_b200_pq* pq, const float* queries, uint32_t nq, float* out_lut,
                                                   uint32_t* out_valid);
/* diagnostics: the ADC pass the last yams_b200_pq_search batch took (the last slice of a call of more than 512 queries):
 * out[0] = 1 for the filtered pass (sampled threshold, one pass over every row), 0 for the per-tile sorting pass;
 * out[1] = queries per CTA of the filtered pass (1, 2 or 4); out[2] = the sampled tiles; out[3] = 1 when a filtered list
 * overflowed and the selection was redone unfiltered.  All 0 after a call that did no device work. */
YAMS_B200_API yams_status_t yams_b200_debug_pq_last_path(yams_b200_pq* pq, uint32_t* out);

/* ---- misc ------------------------------------------------------------------------------------ */
YAMS_B200_API int yams_b200_device_count(void);
/* last error text of the calling thread (static storage) */
YAMS_B200_API const char* yams_b200_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* YAMS_B200_H */
