"""yams_b200 -- H100-native drop-in for YAMS's data-parallel hot path (vector scan + CDC/SHA-256).

The product is ``libyams_b200.so`` (hand-written CUDA for sm_90a behind the C ABI declared in
``include/yams_b200.h``).  This package is only a thin ctypes mirror of that ABI, shaped like the
reference's C++ seams (IChunker / IContentHasher / IVectorStore), for tests and benchmarks.

There is no CPU fallback: importing works without a GPU (so the ABI can be inspected), but every
compute call raises ``YamsB200Error`` unless an sm_90 device (H100) is present, and importing fails
loudly if the shared library has not been built (``python -c "import __graft_entry__ as g; g.build()"``).
"""
from ._lib import (  # noqa: F401
    BATCH_ALL, BATCH_FILTERED, BATCH_TOP_K, BM25_ATIRE, BM25_NOT_INDEXED, BM25_RECIPE_ATIRE, BM25_RECIPE_CASCADE, BM25_RECIPE_SAB_SMOOTH, BM25_STRATEGY_BM25, BM25_STRATEGY_KEYPHRASE, BM25_STRATEGY_LEAD_FIELD, BM25_STRATEGY_ROUTED, BM25_SUBWORD_AWARE_BACKOFF, COSINE, F16, F32, FLAG_FALLBACK_PATH, FLAG_NOT_A_SOURCE, FLAG_TIE_AT_K, FLT_TRUE_MIN, L2, RABIN, STREAMING, Bm25Config, Bm25Index, CdcConfig, ConceptConfig, ConceptIndex, ChunkDesc, Corpus, DigestSet, IngestSession, PqIndex, QUERY_FEATURES_DTYPE, QueryFeatures, RouterConfig, SimeonEncoder, SIMEON_PROJECTION_FWHT, SIMEON_WORD_TOKENS, YamsB200Error,
    batch_distance, bm25_score_rrf, chunk_and_hash, chunk_and_hash_batch, chunk_and_hash_device, chunk_boundaries, compute_cosine_similarity, compute_cosine_similarity_many, dedup_stats, default_config, device_count,
    health, ingest_last_timings, lib, lib_chunk_dtype, lib_path, manifest_build, plugin_init, sha256_batch, sha256_batch_device, sha256_many,
    synth_bytes_device, synth_rows_device, vec0_exact, vec_distance_cosine, vec_distance_l1, vec_distance_l2,
)
