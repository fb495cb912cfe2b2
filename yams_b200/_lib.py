"""ctypes binding of include/yams_b200.h (every exported symbol is bound here; tests check that)."""
from __future__ import annotations

import ctypes as C
import json
import os
from typing import Optional

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(HERE, "libyams_b200.so")

STREAMING, RABIN = 0, 1
F32, F16 = 0, 1
COSINE, L2 = 0, 1
FLAG_TIE_AT_K, FLAG_FALLBACK_PATH, FLAG_NOT_A_SOURCE = 1, 2, 4
FLT_TRUE_MIN = float(np.float32(1.4e-45))   # the smallest positive float: semantic_neighbors' adaptive mode (sim > 0)

u8p = C.POINTER(C.c_uint8)
u32p = C.POINTER(C.c_uint32)
u64p = C.POINTER(C.c_uint64)
i64p = C.POINTER(C.c_int64)
f32p = C.POINTER(C.c_float)


class YamsB200Error(RuntimeError):
    def __init__(self, status: int, where: str, text: str):
        super().__init__(f"{where}: status {status}: {text}")
        self.status = status


class CdcConfig(C.Structure):
    """yams_cdc_config == ChunkingConfig (/root/reference/include/yams/chunking/chunker.h:44-51)."""
    _fields_ = [("window_size", C.c_uint64), ("min_chunk", C.c_uint64), ("max_chunk", C.c_uint64),
                ("polynomial", C.c_uint64), ("mask", C.c_uint64), ("variant", C.c_int32),
                ("reserved", C.c_int32)]


class ChunkDesc(C.Structure):
    _fields_ = [("offset", C.c_uint64), ("size", C.c_uint64), ("digest", C.c_uint8 * 32)]


class ManifestSummary(C.Structure):
    _fields_ = [("checksum", C.c_uint32), ("valid", C.c_uint32), ("offsets_sequential", C.c_uint32), ("sizes_valid", C.c_uint32),
                ("chunk_count", C.c_uint64), ("total_size", C.c_uint64), ("checksum_text_bytes", C.c_uint64)]


class SimeonConfig(C.Structure):
    _fields_ = [("ngram_min", C.c_uint32), ("ngram_max", C.c_uint32), ("sketch_dim", C.c_uint32), ("output_dim", C.c_uint32),
                ("hash_seed", C.c_uint64), ("projection_seed", C.c_uint64), ("l2_normalize", C.c_int32), ("flags", C.c_int32)]


class Bm25Config(C.Structure):
    _fields_ = [("k1", C.c_float), ("b", C.c_float), ("delta", C.c_float), ("subword_gamma", C.c_float), ("variant", C.c_uint32),
                ("ngram_min", C.c_uint32), ("ngram_max", C.c_uint32), ("ngram_df_prune_ratio", C.c_float), ("hash_seed", C.c_uint64)]


class Bm25Stats(C.Structure):
    _fields_ = [("n_docs", C.c_uint64), ("avg_dl", C.c_float), ("ngram_avg_dl", C.c_float), ("total_tokens", C.c_uint64),
                ("terms", C.c_uint64 * 2), ("postings", C.c_uint64 * 2), ("pruned", C.c_uint64)]


class Bm25StrategyStats(C.Structure):
    _fields_ = [("queries", C.c_uint32 * 3), ("replayed", C.c_uint32), ("keyphrase_boosted", C.c_uint32), ("zscore_ms", C.c_float),
                ("device_ms", C.c_float), ("wall_ms", C.c_float)]


class RouterConfig(C.Structure):
    """yams_bm25_router_config: simeon::RouterConfig's routing fields.  RouterConfig.default(**overrides) starts from the lexical
    backend's preset (yams_b200_bm25_default_router_config)."""
    _fields_ = [("oov_threshold", C.c_float), ("high_idf_threshold", C.c_float), ("atire_min_terms", C.c_uint32),
                ("atire_min_idf_floor", C.c_float), ("atire_max_pool_jaccard", C.c_float), ("atire_min_score_decay", C.c_float),
                ("atire_min_scq", C.c_float), ("atire_max_clarity", C.c_float), ("cascade_min_terms", C.c_uint32),
                ("cascade_max_idf", C.c_float)]

    @classmethod
    def default(cls, **overrides) -> "RouterConfig":
        cfg = cls()
        lib().yams_b200_bm25_default_router_config(C.byref(cfg))
        for k, v in overrides.items():
            setattr(cfg, k, v)
        return cfg


class QueryFeatures(C.Structure):
    """yams_bm25_query_features: the fields simeon::QueryRouter::features fills"""
    _fields_ = [("oov_rate", C.c_float), ("avg_idf", C.c_float), ("max_idf", C.c_float), ("min_idf", C.c_float), ("idf_stddev", C.c_float),
                ("n_terms", C.c_uint32), ("avg_term_chars", C.c_float), ("scq_sum", C.c_float), ("simplified_clarity", C.c_float)]


class ConceptConfig(C.Structure):
    _fields_ = [("min_ttf", C.c_uint32), ("pmi_floor", C.c_float), ("max_concepts", C.c_uint32), ("k1", C.c_float), ("b", C.c_float)]


class ConceptStats(C.Structure):
    _fields_ = [("size", C.c_uint64), ("doc_count", C.c_uint64), ("avg_bigram_dl", C.c_float), ("replayed", C.c_uint32),
                ("sum_bigram_dl", C.c_uint64), ("distinct", C.c_uint64), ("passed_min_ttf", C.c_uint64), ("accepted", C.c_uint64)]


BM25_ATIRE, BM25_SUBWORD_AWARE_BACKOFF = 0, 7   # simeon::Bm25Variant numbering
BM25_STRATEGY_BM25, BM25_STRATEGY_KEYPHRASE, BM25_STRATEGY_LEAD_FIELD = 0, 1, 2   # the strategy router's pool numbers
BM25_STRATEGY_ROUTED = 3
BM25_RECIPE_ATIRE, BM25_RECIPE_SAB_SMOOTH, BM25_RECIPE_CASCADE = 0, 1, 2   # simeon::Recipe numbering
BM25_NOT_INDEXED = 0xFFFFFFFF   # a candidate the index does not hold
QUERY_FEATURES_DTYPE = np.dtype([(n, "<u4" if t is C.c_uint32 else "<f4") for n, t in QueryFeatures._fields_])

SIMEON_WORD_TOKENS = 1        # NGramMode::CharAndWord
SIMEON_PROJECTION_FWHT = 2    # ProjectionMode::Fwht (default projection: AchlioptasSparse)

CHUNK_REF_DTYPE = np.dtype([("hash", "S64"), ("offset", "<u8"), ("size", "<u4"), ("flags", "<u4")])
assert CHUNK_REF_DTYPE.itemsize == 80
CHUNK_DTYPE = np.dtype([("offset", "<u8"), ("size", "<u8"), ("digest", "u1", (32,))])
assert CHUNK_DTYPE.itemsize == C.sizeof(ChunkDesc) == 48
CAND_DTYPE = np.dtype([("score", "<f4"), ("row", "<u4")])   # one stage-1 candidate list entry
EXACT_DTYPE = np.dtype([("sim", "<f4"), ("row", "<u4")])    # one exactly re-scored survivor (NaN sim: none)

# every symbol include/yams_b200.h declares: name -> (restype, argtypes)
_descpp = C.POINTER(C.POINTER(ChunkDesc))
_szp = C.POINTER(C.c_size_t)
SYMBOLS = {
    "yams_plugin_get_abi_version": (C.c_int, []),
    "yams_plugin_get_name": (C.c_char_p, []),
    "yams_plugin_get_version": (C.c_char_p, []),
    "yams_plugin_get_manifest_json": (C.c_char_p, []),
    "yams_plugin_init": (C.c_int, [C.c_char_p, C.c_void_p]),
    "yams_plugin_shutdown": (None, []),
    "yams_plugin_get_interface": (C.c_int, [C.c_char_p, C.c_uint32, C.POINTER(C.c_void_p)]),
    "yams_plugin_get_health_json": (C.c_int, [C.POINTER(C.c_void_p)]),
    "yams_b200_cdc_default_config": (None, [C.POINTER(CdcConfig)]),
    "yams_b200_chunk_and_hash": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(CdcConfig), _descpp, _szp]),
    "yams_b200_free_chunks": (None, [C.c_void_p, C.POINTER(ChunkDesc), C.c_size_t]),
    "yams_b200_chunk_and_hash_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(CdcConfig), _descpp, _szp]),
    "yams_b200_ingest_open": (C.c_int, [C.c_void_p, C.POINTER(CdcConfig), C.POINTER(C.c_void_p)]),
    "yams_b200_ingest_feed": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, _descpp, _szp]),
    "yams_b200_ingest_finish": (C.c_int, [C.c_void_p, _descpp, _szp]),
    "yams_b200_ingest_close": (None, [C.c_void_p]),
    "yams_b200_sha256_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, u64p, u64p, C.c_size_t, u8p]),
    "yams_b200_sha256_batch_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, u64p, u64p, C.c_size_t, u8p]),
    "yams_b200_chunk_boundaries": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(CdcConfig), _descpp, _szp]),
    "yams_b200_chunk_and_hash_batch": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_size_t,
                                                 C.POINTER(CdcConfig), C.POINTER(C.POINTER(ChunkDesc)), C.POINTER(C.c_size_t), u64p]),
    "yams_b200_sha256_many": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_size_t, C.c_void_p]),
    "yams_b200_digest_set_create": (C.c_int, [C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p)]),
    "yams_b200_digest_set_insert": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, u64p]),
    "yams_b200_digest_set_contains": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p]),
    "yams_b200_digest_set_size": (C.c_int, [C.c_void_p, u64p]),
    "yams_b200_digest_set_last_ms": (C.c_int, [C.c_void_p, f32p]),
    "yams_b200_digest_set_destroy": (None, [C.c_void_p]),
    "yams_b200_manifest_build": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint64, C.c_void_p, C.POINTER(ManifestSummary)]),
    "yams_b200_ingest_last_timings": (C.c_int, [C.c_void_p, f32p]),
    "yams_b200_dedup_stats": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]),
    "yams_b200_corpus_create": (C.c_int, [C.c_void_p, C.c_uint32, C.c_int, C.c_int, C.c_uint64, C.POINTER(C.c_void_p)]),
    "yams_b200_corpus_append": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, i64p]),
    "yams_b200_corpus_append_f32_as_f16": (C.c_int, [C.c_void_p, f32p, C.c_uint64, i64p]),
    "yams_b200_corpus_append_synthetic": (C.c_int, [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64]),
    "yams_b200_corpus_remove": (C.c_int, [C.c_void_p, i64p, C.c_uint64, u64p]),
    "yams_b200_corpus_clear": (C.c_int, [C.c_void_p]),
    "yams_b200_batch_distance": (C.c_int, [C.c_void_p, C.c_int, f32p, C.c_uint32, f32p, C.c_uint64, C.c_int, C.c_uint64,
                                           C.c_float, u64p, f32p, u64p]),
    "yams_b200_compute_cosine_similarity": (C.c_int, [C.c_void_p, f32p, C.c_size_t, f32p, C.c_size_t,
                                                      C.POINTER(C.c_double)]),
    "yams_b200_compute_cosine_similarity_many": (C.c_int, [C.c_void_p, f32p, f32p, C.c_size_t, C.c_size_t, C.POINTER(C.c_double)]),
    "yams_b200_corpus_size": (C.c_int, [C.c_void_p, u64p]),
    "yams_b200_corpus_destroy": (None, [C.c_void_p]),
    "yams_b200_search": (C.c_int, [C.c_void_p, f32p, C.c_uint32, C.c_uint32, C.c_float, i64p, u64p, i64p, f32p, u32p, u64p]),
    "yams_b200_search_all_matching": (C.c_int, [C.c_void_p, f32p, C.c_float, i64p, C.c_uint64, i64p, f32p, u64p]),
    "yams_b200_semantic_neighbors": (C.c_int, [C.c_void_p, i64p, C.c_uint64, C.c_uint32, C.c_float, i64p, f32p, u32p, u64p]),
    "yams_b200_debug_semantic_stage1": (C.c_int, [C.c_void_p, i64p, C.c_uint32, C.c_int, f32p, f32p]),
    "yams_b200_topology_kmeans": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, u32p, f32p, u32p, u32p]),
    "yams_b200_topology_kmeans_last_timings": (C.c_int, [C.c_void_p, f32p]),
    "yams_b200_search_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_float, C.c_void_p, C.c_void_p]),
    "yams_b200_search_device_finish": (C.c_int, [C.c_void_p, u32p]),
    "yams_b200_search_exhaustive": (C.c_int, [C.c_void_p, f32p, C.c_uint32, C.c_uint32, C.c_float, i64p, f32p, u32p, u64p]),
    "yams_b200_merge_packed_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p,
                                                C.c_void_p, C.c_void_p]),
    "yams_b200_merge_partials_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32,
                                                  C.c_void_p, C.c_void_p, C.c_void_p]),
    "yams_b200_corpus_sync": (C.c_int, [C.c_void_p]),
    "yams_b200_corpus_stream": (C.c_void_p, [C.c_void_p]),
    "yams_b200_vec0_exact": (C.c_int, [C.c_void_p, f32p, C.c_uint32, f32p, i64p, C.c_uint64, C.c_uint64, C.c_int,
                                       C.c_int64, C.c_int64, i64p, f32p, u64p]),
    "yams_b200_search_last_timings": (C.c_int, [C.c_void_p, f32p]),
    "sqlite3_vec_distance_l2": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, f32p]),
    "sqlite3_vec_distance_cosine": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, f32p]),
    "yams_b200_vec_distance_l1": (C.c_int, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, f32p]),
    "yams_b200_synth_bytes_device": (C.c_int, [C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p]),
    "yams_b200_debug_stage1_scores": (C.c_int, [C.c_void_p, f32p, C.c_uint32, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, f32p]),
    "yams_b200_debug_stage1_candidates": (C.c_int, [C.c_void_p, f32p, C.c_uint32, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, f32p,
                                                    C.c_uint32, i64p, u64p, u32p, C.c_void_p]),
    "yams_b200_synth_rows_device": (C.c_int, [C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint32, C.c_void_p]),
    "yams_b200_simeon_default_config": (None, [C.POINTER(SimeonConfig)]),
    "yams_b200_simeon_yams_config": (None, [C.POINTER(SimeonConfig), C.c_uint32]),
    "yams_b200_simeon_create": (C.c_int, [C.c_void_p, C.POINTER(SimeonConfig), C.POINTER(C.c_void_p)]),
    "yams_b200_simeon_encode": (C.c_int, [C.c_void_p, C.POINTER(C.c_char_p), C.POINTER(C.c_size_t), C.c_size_t, f32p]),
    "yams_b200_simeon_destroy": (None, [C.c_void_p]),
    "yams_b200_bm25_default_config": (None, [C.POINTER(Bm25Config)]),
    "yams_b200_bm25_build": (C.c_int, [C.c_void_p, C.POINTER(Bm25Config), C.POINTER(C.c_char_p), C.POINTER(C.c_size_t), C.c_uint64,
                                       C.POINTER(C.c_void_p)]),
    "yams_b200_bm25_score": (C.c_int, [C.c_void_p, C.POINTER(C.c_char_p), C.POINTER(C.c_size_t), C.c_uint32, f32p, C.c_uint32, u32p, f32p,
                                       u32p]),
    "yams_b200_bm25_stats": (C.c_int, [C.c_void_p, C.POINTER(Bm25Stats)]),
    "yams_b200_bm25_postings": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint64, u32p, f32p, u64p, u32p, u32p, C.c_uint64]),
    "yams_b200_bm25_doc_lengths": (C.c_int, [C.c_void_p, C.c_uint32, u32p]),
    "yams_b200_bm25_last_timings": (C.c_int, [C.c_void_p, f32p]),
    "yams_b200_bm25_destroy": (None, [C.c_void_p]),
    "yams_b200_concepts_default_config": (None, [C.POINTER(ConceptConfig)]),
    "yams_b200_concepts_mine": (C.c_int, [C.c_void_p, C.POINTER(ConceptConfig), C.POINTER(C.c_char_p), C.POINTER(C.c_size_t), C.c_uint64,
                                          C.POINTER(C.c_void_p)]),
    "yams_b200_bm25_score_blended": (C.c_int, [C.c_void_p, C.c_void_p, C.c_float, C.POINTER(C.c_char_p), C.POINTER(C.c_size_t), C.c_uint32,
                                               f32p, C.c_uint32, u32p, f32p, u32p]),
    "yams_b200_concepts_blend": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t, C.c_float, f32p, C.c_uint64]),
    "yams_b200_concepts_stats": (C.c_int, [C.c_void_p, C.POINTER(ConceptStats)]),
    "yams_b200_concepts_find": (C.c_int, [C.c_void_p, C.c_uint64, u32p, f32p, f32p, u64p, u64p, u64p, u32p, u32p, u32p, C.c_uint64]),
    "yams_b200_concepts_hashes": (C.c_int, [C.c_void_p, u64p]),
    "yams_b200_concepts_bigram_lengths": (C.c_int, [C.c_void_p, u32p]),
    "yams_b200_concepts_last_timings": (C.c_int, [C.c_void_p, f32p]),
    "yams_b200_concepts_destroy": (None, [C.c_void_p]),
    "yams_b200_bm25_atire_view": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p)]),
    "yams_b200_bm25_score_rrf": (C.c_int, [C.POINTER(C.c_void_p), C.c_uint32, C.c_float, C.c_void_p, C.c_float, C.POINTER(C.c_char_p),
                                           C.POINTER(C.c_size_t), C.c_uint32, f32p, C.c_uint32, u32p, f32p, u32p]),
    "yams_b200_bm25_build_lead": (C.c_int, [C.c_void_p, C.POINTER(Bm25Config), C.POINTER(C.c_char_p), C.POINTER(C.c_size_t), C.c_uint64,
                                            C.c_uint32, C.POINTER(C.c_void_p)]),
    "yams_b200_bm25_aux_stats": (C.c_int, [C.c_void_p, C.POINTER(Bm25Stats)]),
    "yams_b200_bm25_strategy_stats": (C.c_int, [C.c_void_p, C.POINTER(Bm25StrategyStats)]),
    "yams_b200_bm25_score_strategy": (C.c_int, [C.c_void_p, C.c_uint32, C.c_void_p, C.c_float, C.POINTER(C.c_char_p), C.POINTER(C.c_size_t),
                                                C.c_uint32, f32p, C.c_uint32, u32p, f32p, u32p, u32p]),
    "yams_b200_bm25_default_router_config": (None, [C.POINTER(RouterConfig)]),
    "yams_b200_bm25_score_routed": (C.c_int, [C.c_void_p, C.POINTER(RouterConfig), C.c_void_p, C.c_float, C.POINTER(C.c_char_p),
                                              C.POINTER(C.c_size_t), C.c_uint32, f32p, C.c_uint32, u32p, f32p, u32p, u64p, u32p, f32p, u32p,
                                              C.c_void_p]),
    "yams_b200_pq_build": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, f32p, u64p, C.POINTER(C.c_void_p)]),
    "yams_b200_pq_search": (C.c_int, [C.c_void_p, f32p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_float, i64p, f32p, u32p, u64p]),
    "yams_b200_pq_search_candidates": (C.c_int, [C.c_void_p, f32p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_float, i64p, u64p, i64p, f32p,
                                                 u32p, u64p]),
    "yams_b200_search_documents": (C.c_int, [C.c_void_p, C.c_void_p, f32p, C.c_uint32, C.c_uint32, C.c_float, i64p, u64p, u64p, i64p, i64p,
                                             f32p, u32p]),
    "yams_b200_pq_codes": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, u64p]),
    "yams_b200_pq_destroy": (None, [C.c_void_p]),
    "yams_b200_debug_last_eps": (C.c_int, [C.c_void_p, C.c_uint32, f32p]),
    "yams_b200_debug_stage1_profile": (C.c_int, [C.c_void_p, f32p, C.c_uint32, f32p, C.c_uint32, C.c_uint32, u64p, u32p, f32p]),
    "yams_b200_debug_pq_lut": (C.c_int, [C.c_void_p, f32p, C.c_uint32, f32p, u32p]),
    "yams_b200_debug_pq_last_path": (C.c_int, [C.c_void_p, u32p]),
    "yams_b200_debug_select": (C.c_int, [C.c_void_p, C.c_uint32, f32p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint32,
                                         C.c_void_p, u32p, C.c_uint32, f32p, C.c_uint32, C.c_int, C.c_float, C.c_int, C.c_void_p,
                                         u32p, f32p]),
    "yams_b200_debug_final": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, u32p, f32p, f32p,
                                        C.POINTER(C.c_double), C.c_float, C.c_int, C.c_int, i64p, f32p, u32p, u64p, u32p, u32p]),
    "yams_b200_device_count": (C.c_int, []),
    "yams_b200_last_error": (C.c_char_p, []),
}

_lib = None


def lib_path() -> str:
    return _SO


def lib():
    """The loaded shared library. Fails loudly when it has not been built -- there is no fallback."""
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            raise ImportError(
                f"{_SO} is missing: build it with `python -c \"import __graft_entry__ as g; g.build()\"` "
                "(nvcc, sm_90a). yams_b200 has no CPU or PyTorch fallback.")
        L = C.CDLL(_SO)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def _check(rc: int, where: str):
    if rc != 0:
        raise YamsB200Error(rc, where, (lib().yams_b200_last_error() or b"").decode(errors="replace"))


def device_count() -> int:
    return lib().yams_b200_device_count()


def plugin_init(config: Optional[dict] = None) -> int:
    return lib().yams_plugin_init(json.dumps(config or {}).encode(), None)


def health() -> dict:
    p = C.c_void_p()
    lib().yams_plugin_get_health_json(C.byref(p))
    s = C.cast(p, C.c_char_p).value.decode()
    C.CDLL(None).free(p)
    return json.loads(s)


def default_config(variant: int = STREAMING, **kw) -> CdcConfig:
    cfg = CdcConfig()
    lib().yams_b200_cdc_default_config(C.byref(cfg))
    cfg.variant = variant
    for k, v in kw.items():
        if k not in {f[0] for f in CdcConfig._fields_}:
            raise TypeError(f"unknown CdcConfig field {k!r}")
        setattr(cfg, k, v)
    return cfg


def lib_chunk_dtype():
    """numpy dtype of yams_chunk_desc (offset, size, digest[32])."""
    return CHUNK_DTYPE


def _as_u8(data) -> np.ndarray:
    if isinstance(data, np.ndarray):
        return np.ascontiguousarray(data, dtype=np.uint8)
    return np.frombuffer(bytes(data), dtype=np.uint8)


def _take(out_p, out_n) -> np.ndarray:
    n = out_n.value
    if n == 0:
        return np.zeros(0, dtype=CHUNK_DTYPE)
    buf = (ChunkDesc * n).from_address(C.addressof(out_p.contents))
    arr = np.frombuffer(buf, dtype=CHUNK_DTYPE).copy()
    lib().yams_b200_free_chunks(None, out_p, n)
    return arr


def _chunks(fn_name: str, ptr, length: int, cfg: CdcConfig) -> np.ndarray:
    out_p = C.POINTER(ChunkDesc)()
    out_n = C.c_size_t(0)
    rc = getattr(lib(), fn_name)(None, ptr, length, C.byref(cfg), C.byref(out_p), C.byref(out_n))
    _check(rc, fn_name)
    return _take(out_p, out_n)


def chunk_and_hash(data, cfg: Optional[CdcConfig] = None) -> np.ndarray:
    """IChunker::chunkDataLazy over a host buffer -> structured array (offset, size, digest[32])."""
    a = _as_u8(data)
    return _chunks("yams_b200_chunk_and_hash", a.ctypes.data if a.size else None, a.size, cfg or default_config())


def chunk_and_hash_batch(files, cfg: Optional[CdcConfig] = None):
    """Many files in one call (`yams add -r`): -> list of per-file chunk tables (offsets relative to each file)."""
    arrs = [_as_u8(f) for f in files]
    n = len(arrs)
    ptrs = (C.c_void_p * max(n, 1))(*[a.ctypes.data if a.size else None for a in arrs])
    lens = (C.c_size_t * max(n, 1))(*[a.size for a in arrs])
    first = np.zeros(n + 1, dtype=np.uint64)
    out_p = C.POINTER(ChunkDesc)()
    out_n = C.c_size_t(0)
    c = cfg or default_config()
    rc = lib().yams_b200_chunk_and_hash_batch(None, ptrs, lens, n, C.byref(c), C.byref(out_p), C.byref(out_n),
                                              first.ctypes.data_as(u64p))
    _check(rc, "chunk_and_hash_batch")
    table = _take(out_p, out_n)
    return [table[int(first[i]):int(first[i + 1])] for i in range(n)]


def sha256_many(messages) -> np.ndarray:
    """SHA-256 of separate host buffers in one device pass -> uint8[n, 32]."""
    arrs = [_as_u8(m) for m in messages]
    n = len(arrs)
    out = np.zeros((n, 32), dtype=np.uint8)
    if n:
        ptrs = (C.c_void_p * n)(*[a.ctypes.data if a.size else None for a in arrs])
        lens = (C.c_size_t * n)(*[a.size for a in arrs])
        _check(lib().yams_b200_sha256_many(None, ptrs, lens, n, out.ctypes.data), "sha256_many")
    return out


def chunk_boundaries(data, cfg: Optional[CdcConfig] = None) -> np.ndarray:
    a = _as_u8(data)
    return _chunks("yams_b200_chunk_boundaries", a.ctypes.data if a.size else None, a.size, cfg or default_config())


def chunk_and_hash_device(dev_ptr: int, length: int, cfg: Optional[CdcConfig] = None) -> np.ndarray:
    """Input already resident in HBM (e.g. ``tensor.data_ptr()``)."""
    return _chunks("yams_b200_chunk_and_hash_device", dev_ptr, length, cfg or default_config())


def dedup_stats(chunks: np.ndarray) -> dict:
    """calculateDeduplication over a chunk table (structured array from chunk_and_hash)."""
    arr = np.ascontiguousarray(chunks, dtype=CHUNK_DTYPE)
    out = (C.c_uint64 * 4)()
    _check(lib().yams_b200_dedup_stats(None, arr.ctypes.data if len(arr) else None, len(arr), out), "dedup_stats")
    total, unique, count, ucount = (int(x) for x in out)
    return {"totalSize": total, "uniqueSize": unique, "chunkCount": count, "uniqueChunks": ucount,
            "ratio": (1.0 - unique / total) if total else 0.0}


def manifest_build(chunks: np.ndarray, file_digest, file_size: int, want_refs: bool = True):
    """ManifestManager::createManifest over a chunk table: -> (ChunkRef table or None, summary dict incl. the CRC checksum)."""
    arr = np.ascontiguousarray(chunks, dtype=CHUNK_DTYPE)
    dg = np.ascontiguousarray(np.frombuffer(bytes(file_digest), dtype=np.uint8))
    assert dg.size == 32
    refs = np.zeros(max(len(arr), 1), dtype=CHUNK_REF_DTYPE) if want_refs else None
    out = ManifestSummary()
    _check(lib().yams_b200_manifest_build(None, arr.ctypes.data if len(arr) else None, len(arr), dg.ctypes.data, file_size,
                                          refs.ctypes.data if want_refs else None, C.byref(out)), "manifest_build")
    summary = {f[0]: int(getattr(out, f[0])) for f in ManifestSummary._fields_}
    return (refs[:len(arr)] if want_refs else None), summary


def ingest_last_timings() -> dict:
    ms = (C.c_float * 8)()
    lib().yams_b200_ingest_last_timings(None, ms)
    return {"scan_ms": ms[0], "select_ms": ms[1], "sha256_ms": ms[2], "total_ms": ms[3],
            "host_sync1_ms": ms[4], "host_sync2_ms": ms[5], "host_alloc_ms": ms[6], "host_process_ms": ms[7]}


class IngestSession:
    """StreamingChunker::processStream shaped session (open / feed... / finish)."""

    def __init__(self, cfg: Optional[CdcConfig] = None):
        self._h = C.c_void_p()
        self._cfg = cfg or default_config()
        _check(lib().yams_b200_ingest_open(None, C.byref(self._cfg), C.byref(self._h)), "ingest_open")

    def feed(self, data) -> np.ndarray:
        a = _as_u8(data)
        out_p = C.POINTER(ChunkDesc)()
        out_n = C.c_size_t(0)
        _check(lib().yams_b200_ingest_feed(self._h, a.ctypes.data if a.size else None, a.size, C.byref(out_p),
                                           C.byref(out_n)), "ingest_feed")
        return _take(out_p, out_n)

    def finish(self) -> np.ndarray:
        out_p = C.POINTER(ChunkDesc)()
        out_n = C.c_size_t(0)
        _check(lib().yams_b200_ingest_finish(self._h, C.byref(out_p), C.byref(out_n)), "ingest_finish")
        return _take(out_p, out_n)

    def close(self):
        if self._h:
            lib().yams_b200_ingest_close(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def sha256_batch(base, offsets, sizes) -> np.ndarray:
    a = _as_u8(base)
    offs = np.ascontiguousarray(offsets, dtype=np.uint64)
    szs = np.ascontiguousarray(sizes, dtype=np.uint64)
    out = np.zeros((len(offs), 32), dtype=np.uint8)
    _check(lib().yams_b200_sha256_batch(None, a.ctypes.data if a.size else None, a.size, offs.ctypes.data_as(u64p),
                                        szs.ctypes.data_as(u64p), len(offs), out.ctypes.data_as(u8p)), "sha256_batch")
    return out


def sha256_batch_device(dev_ptr: int, base_len: int, offsets, sizes) -> np.ndarray:
    offs = np.ascontiguousarray(offsets, dtype=np.uint64)
    szs = np.ascontiguousarray(sizes, dtype=np.uint64)
    out = np.zeros((len(offs), 32), dtype=np.uint8)
    _check(lib().yams_b200_sha256_batch_device(None, dev_ptr, base_len, offs.ctypes.data_as(u64p), szs.ctypes.data_as(u64p),
                                               len(offs), out.ctypes.data_as(u8p)), "sha256_batch_device")
    return out


def synth_bytes_device(seed: int, start: int, n: int, dev_ptr: int):
    _check(lib().yams_b200_synth_bytes_device(seed, start, n, dev_ptr), "synth_bytes_device")


def synth_rows_device(seed: int, first_row: int, n: int, dim: int, dev_ptr: int):
    """n x dim fp32 rows of the synthetic vector generator into a device buffer."""
    _check(lib().yams_b200_synth_rows_device(seed, first_row, n, dim, dev_ptr), "synth_rows_device")


class Corpus:
    """Device-resident mirror of the `vectors` table (row-major [n, dim], fp32 or fp16)."""

    def __init__(self, dim: int, dtype: int = F16, metric: int = COSINE, capacity_hint: int = 0):
        self._h = C.c_void_p()
        self.dim, self.dtype, self.metric = dim, dtype, metric
        _check(lib().yams_b200_corpus_create(None, dim, dtype, metric, capacity_hint, C.byref(self._h)), "corpus_create")

    @property
    def handle(self):
        return self._h

    def append(self, rows: np.ndarray, rowids=None):
        rows = np.ascontiguousarray(rows)
        n = rows.shape[0]
        rid = np.ascontiguousarray(rowids, dtype=np.int64) if rowids is not None else None
        ridp = rid.ctypes.data_as(i64p) if rid is not None else None
        if self.dtype == F16 and rows.dtype == np.float32:
            _check(lib().yams_b200_corpus_append_f32_as_f16(self._h, rows.ctypes.data_as(f32p), n, ridp), "corpus_append_f32_as_f16")
        else:
            want = np.uint16 if self.dtype == F16 else np.float32
            if self.dtype == F16 and rows.dtype == np.float16:
                rows = rows.view(np.uint16)
            assert rows.dtype == want, (rows.dtype, want)
            _check(lib().yams_b200_corpus_append(self._h, rows.ctypes.data, n, ridp), "corpus_append")

    def append_synthetic(self, seed: int, first_row: int, n: int):
        _check(lib().yams_b200_corpus_append_synthetic(self._h, seed, first_row, n), "corpus_append_synthetic")

    def clear(self):
        _check(lib().yams_b200_corpus_clear(self._h), "corpus_clear")

    def remove(self, rowids) -> int:
        """deleteVector / deleteVectorsByDocument mirror: drop rows by rowid, keep the rest in rowid order."""
        r = np.ascontiguousarray(rowids, dtype=np.int64).reshape(-1)
        out = C.c_uint64(0)
        _check(lib().yams_b200_corpus_remove(self._h, r.ctypes.data_as(i64p) if len(r) else None, len(r), C.byref(out)),
               "corpus_remove")
        return out.value

    def __len__(self):
        n = C.c_uint64(0)
        _check(lib().yams_b200_corpus_size(self._h, C.byref(n)), "corpus_size")
        return n.value

    def search(self, queries: np.ndarray, k: int, threshold: float = -1.0, allowed=None):
        """-> (rowids i64[Q,k], scores f32[Q,k], counts u32[Q], flags u64[Q]).
        allowed: optional list (len Q) of ascending rowid arrays (CandidateFilterMode::Exact)."""
        q = np.ascontiguousarray(queries, dtype=np.float32)
        if q.ndim == 1:
            q = q[None, :]
        nq = q.shape[0]
        out_r = np.full((nq, max(k, 1)), -1, dtype=np.int64)
        out_s = np.zeros((nq, max(k, 1)), dtype=np.float32)
        out_c = np.zeros(nq, dtype=np.uint32)
        out_f = np.zeros(nq, dtype=np.uint64)
        al_p = of_p = None
        if allowed is not None:
            offs = np.zeros(nq + 1, dtype=np.uint64)
            offs[1:] = np.cumsum([len(a) for a in allowed])
            al = np.ascontiguousarray(np.concatenate([np.asarray(a, dtype=np.int64) for a in allowed])
                                      if nq and int(offs[-1]) else np.zeros(1, dtype=np.int64), dtype=np.int64)
            al_p, of_p = al.ctypes.data_as(i64p), offs.ctypes.data_as(u64p)
        rc = lib().yams_b200_search(self._h, q.ctypes.data_as(f32p), nq, k, threshold, al_p, of_p,
                                    out_r.ctypes.data_as(i64p), out_s.ctypes.data_as(f32p), out_c.ctypes.data_as(u32p),
                                    out_f.ctypes.data_as(u64p))
        _check(rc, "search")
        return out_r[:, :k], out_s[:, :k], out_c, out_f

    def search_all_matching(self, query, threshold: float = -1.0, allowed=None):
        """ExactRowSelection::AllMatching: every passing row of the candidate set, sorted (sim desc, rowid asc)."""
        q = np.ascontiguousarray(query, dtype=np.float32).reshape(-1)
        al = np.ascontiguousarray(allowed, dtype=np.int64) if allowed is not None else None
        m = len(al) if al is not None else len(self)
        out_r = np.empty(max(m, 1), dtype=np.int64)
        out_s = np.empty(max(m, 1), dtype=np.float32)
        cnt = C.c_uint64(0)
        rc = lib().yams_b200_search_all_matching(self._h, q.ctypes.data_as(f32p), threshold,
                                                 al.ctypes.data_as(i64p) if al is not None and len(al) else None,
                                                 len(al) if al is not None else 0, out_r.ctypes.data_as(i64p),
                                                 out_s.ctypes.data_as(f32p), C.byref(cnt))
        _check(rc, "search_all_matching")
        return out_r[:cnt.value].copy(), out_s[:cnt.value].copy()

    def semantic_neighbors(self, k: int, threshold: float = FLT_TRUE_MIN, sources=None):
        """The semantic-neighbour graph (EmbeddingService's semantic_neighbor edges): the k best other rows of every source row by
        float((dot inv_s) inv_n), ordered (sim desc, rowid asc), sim >= threshold (FLT_TRUE_MIN: the reference's adaptive
        mode).  sources: None = every row, else strictly ascending rowids.
        -> (rowids i64[S,k] (-1 unused), sims f32[S,k] (0 unused), counts u32[S], flags u64[S])."""
        src = None if sources is None else np.ascontiguousarray(sources, dtype=np.int64).reshape(-1)
        ns = len(self) if src is None else len(src)
        out_r = np.full((max(ns, 1), max(k, 1)), -1, dtype=np.int64)
        out_s = np.zeros((max(ns, 1), max(k, 1)), dtype=np.float32)
        out_c = np.zeros(max(ns, 1), dtype=np.uint32)
        out_f = np.zeros(max(ns, 1), dtype=np.uint64)
        rc = lib().yams_b200_semantic_neighbors(self._h, src.ctypes.data_as(i64p) if src is not None else None, ns, k, threshold,
                                                out_r.ctypes.data_as(i64p), out_s.ctypes.data_as(f32p), out_c.ctypes.data_as(u32p),
                                                out_f.ctypes.data_as(u64p))
        _check(rc, "semantic_neighbors")
        return out_r[:ns, :k], out_s[:ns, :k], out_c[:ns], out_f[:ns]

    def debug_semantic_stage1(self, sources, engine: int):
        """-> (stage-1 scores f32[S, n] of the graph's scales, certificate error bound f32[S]) of the sources (rowids)"""
        src = np.ascontiguousarray(sources, dtype=np.int64).reshape(-1)
        out = np.empty((len(src), len(self)), dtype=np.float32)
        eps = np.empty(len(src), dtype=np.float32)
        _check(lib().yams_b200_debug_semantic_stage1(self._h, src.ctypes.data_as(i64p), len(src), engine, out.ctypes.data_as(f32p),
                                                     eps.ctypes.data_as(f32p)), "debug_semantic_stage1")
        return out, eps

    def topology_kmeans(self, k: int = 0, max_iterations: int = 0):
        """The k-means topology engine's spherical k-means (runKMeans) over the rows, one usable document each in document order:
        k = 0 is round(sqrt(rows)), max_iterations = 0 is 10.  -> (assignment u32[rows], centroids f32[k, dim], k, iterations)"""
        n = len(self)
        kk = 0 if n < 2 else min(max(k if k else int(np.floor(np.sqrt(n) + 0.5)), 2), n)
        asg = np.empty(max(n, 1), dtype=np.uint32)
        cent = np.empty((max(kk, 1), self.dim), dtype=np.float32)
        k_out, it_out = C.c_uint32(), C.c_uint32()
        _check(lib().yams_b200_topology_kmeans(self._h, k, max_iterations, asg.ctypes.data_as(u32p), cent.ctypes.data_as(f32p),
                                               C.byref(k_out), C.byref(it_out)), "topology_kmeans")
        assert k_out.value == kk
        return asg[:n], cent[:kk], k_out.value, it_out.value

    def topology_kmeans_last_timings(self) -> dict:
        ms = (C.c_float * 4)()
        _check(lib().yams_b200_topology_kmeans_last_timings(self._h, ms), "topology_kmeans_last_timings")
        return {"init_ms": ms[0], "assign_ms": ms[1], "update_ms": ms[2], "total_ms": ms[3]}

    def search_device(self, d_queries: int, nq: int, k: int, threshold: float, d_out_rowids: int, d_out_scores: int):
        _check(lib().yams_b200_search_device(self._h, d_queries, nq, k, threshold, d_out_rowids, d_out_scores), "search_device")

    def search_device_finish(self) -> int:
        """Blocks until the last search_device is done; raises on invalid queries; -> queries resolved exhaustively."""
        n = C.c_uint32(0)
        _check(lib().yams_b200_search_device_finish(self._h, C.byref(n)), "search_device_finish")
        return n.value

    def search_documents(self, queries, k: int, docs, threshold: float = -1.0, pq: Optional["PqIndex"] = None):
        """CandidateFilterMode::DocumentTopK: docs[q] is query q's list of documents, each an array of rowids in chunk order
        (pass documents sorted by document hash: ties between documents go to the earlier one, ties inside a document to the
        earlier row).  pq=None scores every row exactly (the exact fallback); with a PqIndex, the rows in the index are
        re-scored like its rerank.  -> (doc i64[Q,k] = position in docs[q], rowids i64[Q,k] = the document's best row,
        scores f32[Q,k], counts u32[Q]); unused slots -1 / -1 / 0."""
        nq = len(docs)
        qdocs = np.zeros(nq + 1, dtype=np.uint64)
        qdocs[1:] = np.cumsum([len(ds) for ds in docs])
        flat = [np.asarray(r, dtype=np.int64).reshape(-1) for ds in docs for r in ds]
        doffs = np.zeros(len(flat) + 1, dtype=np.uint64)
        doffs[1:] = np.cumsum([len(r) for r in flat])
        rid = np.concatenate(flat) if int(doffs[-1]) else np.zeros(0, dtype=np.int64)
        d, r, s, cnt = self.search_documents_csr(queries, k, rid, doffs, qdocs, threshold, pq)
        local = np.where(d >= 0, d - qdocs[:-1, None].astype(np.int64), -1)
        return local, r, s, cnt

    def search_documents_csr(self, queries, k: int, doc_rowids, doc_offsets, query_docs, threshold: float = -1.0,
                             pq: Optional["PqIndex"] = None):
        """search_documents on the C ABI's layout: document d = doc_rowids[doc_offsets[d] .. doc_offsets[d+1]), query q's documents
        query_docs[q] .. query_docs[q+1].  -> (global document index i64[Q,k], rowids, scores, counts)"""
        q = np.ascontiguousarray(queries, dtype=np.float32)
        if q.ndim == 1:
            q = q[None, :]
        nq = q.shape[0]
        qdocs = np.ascontiguousarray(query_docs, dtype=np.uint64)
        doffs = np.ascontiguousarray(doc_offsets, dtype=np.uint64)
        assert len(qdocs) == nq + 1
        rid = np.ascontiguousarray(doc_rowids, dtype=np.int64)
        if rid.size == 0:
            rid = np.zeros(1, dtype=np.int64)
        kk = max(k, 1)
        out_d = np.full((nq, kk), -1, dtype=np.int64)
        out_r = np.full((nq, kk), -1, dtype=np.int64)
        out_s = np.zeros((nq, kk), dtype=np.float32)
        out_c = np.zeros(nq, dtype=np.uint32)
        _check(lib().yams_b200_search_documents(self._h, pq.handle if pq is not None else None, q.ctypes.data_as(f32p), nq, k, threshold,
                                                rid.ctypes.data_as(i64p), doffs.ctypes.data_as(u64p), qdocs.ctypes.data_as(u64p),
                                                out_d.ctypes.data_as(i64p), out_r.ctypes.data_as(i64p), out_s.ctypes.data_as(f32p),
                                                out_c.ctypes.data_as(u32p)), "search_documents")
        return out_d[:, :k], out_r[:, :k], out_s[:, :k], out_c

    def search_exhaustive(self, queries: np.ndarray, k: int, threshold: float = -1.0):
        """The library's own exhaustive reference (exact score of every row + global sort); same outputs as search."""
        q = np.ascontiguousarray(queries, dtype=np.float32)
        if q.ndim == 1:
            q = q[None, :]
        nq = q.shape[0]
        out_r = np.full((nq, k), -1, dtype=np.int64)
        out_s = np.zeros((nq, k), dtype=np.float32)
        out_c = np.zeros(nq, dtype=np.uint32)
        out_f = np.zeros(nq, dtype=np.uint64)
        _check(lib().yams_b200_search_exhaustive(self._h, q.ctypes.data_as(f32p), nq, k, threshold, out_r.ctypes.data_as(i64p),
                                                 out_s.ctypes.data_as(f32p), out_c.ctypes.data_as(u32p), out_f.ctypes.data_as(u64p)),
               "search_exhaustive")
        return out_r, out_s, out_c, out_f

    def merge_packed_device(self, d_packed: int, nranks: int, nq: int, k: int, d_out_rowids: int, d_out_scores: int,
                            d_out_counts: int = 0, stream: int = 0):
        _check(lib().yams_b200_merge_packed_device(self._h, d_packed, nranks, nq, k, d_out_rowids, d_out_scores,
                                                   d_out_counts or None, stream or None), "merge_packed_device")

    def merge_partials_device(self, d_rowids: int, d_scores: int, nranks: int, nq: int, k: int, d_out_rowids: int,
                              d_out_scores: int, d_out_counts: int = 0):
        _check(lib().yams_b200_merge_partials_device(self._h, d_rowids, d_scores, nranks, nq, k, d_out_rowids, d_out_scores,
                                                     d_out_counts or None), "merge_partials_device")

    def debug_stage1_scores(self, queries, engine: int, row_start: int = 0, row_stride: int = 1, nrows: int = 0):
        q = np.ascontiguousarray(queries, dtype=np.float32)
        nrows = nrows or len(self)
        out = np.empty((q.shape[0], nrows), dtype=np.float32)
        _check(lib().yams_b200_debug_stage1_scores(self._h, q.ctypes.data_as(f32p), q.shape[0], engine, row_start, row_stride,
                                                   nrows, out.ctypes.data_as(f32p)), "debug_stage1_scores")
        return out

    def debug_stage1_candidates(self, queries, engine: int, tau, cap: int, row_start: int = 0, row_stride: int = 1, nrows: int = 0,
                                allowed=None):
        """Stage 1 in filter mode -> (counts u32[Q] (not capped), lists CAND_DTYPE[Q, cap]); entry j < min(counts[q], cap) of
        lists[q] is a row whose stage-1 score exceeded tau[q] (and is in allowed[q], a list of rowids, when given)."""
        q = np.ascontiguousarray(queries, dtype=np.float32)
        nq = q.shape[0]
        t = np.ascontiguousarray(tau, dtype=np.float32).reshape(nq)
        nrows = nrows or len(self)
        counts = np.zeros(nq, dtype=np.uint32)
        lists = np.empty((nq, max(cap, 1)), dtype=CAND_DTYPE)
        al_p = of_p = None
        if allowed is not None:
            offs = np.zeros(nq + 1, dtype=np.uint64)
            offs[1:] = np.cumsum([len(a) for a in allowed])
            al = np.ascontiguousarray(np.concatenate([np.asarray(a, dtype=np.int64) for a in allowed]) if int(offs[-1])
                                      else np.zeros(1, dtype=np.int64), dtype=np.int64)
            al_p, of_p = al.ctypes.data_as(i64p), offs.ctypes.data_as(u64p)
        _check(lib().yams_b200_debug_stage1_candidates(self._h, q.ctypes.data_as(f32p), nq, engine, row_start, row_stride, nrows,
                                                       t.ctypes.data_as(f32p), cap, al_p, of_p, counts.ctypes.data_as(u32p),
                                                       lists.ctypes.data), "debug_stage1_candidates")
        return counts, lists[:, :cap]

    def debug_select(self, K: int, dense=None, row_start: int = 0, row_stride: int = 1, dense_shift: int = 0, cands=None,
                     counts=None, tau=None, tau_only: bool = False, tau_margin: float = 0.0, fast_tau: bool = False):
        """The scan's top-K selection on given scores: dense f32[Q, L] (row index row_start + i * row_stride, device copy
        dense_shift floats past a 16-byte boundary) or lists CAND_DTYPE[Q, cap] with counts u32[Q] (may exceed cap) and an
        optional tau f32[Q].  -> (sel CAND_DTYPE[Q, K], n u32[Q], bound f32[Q]), or with tau_only the thresholds f32[Q]."""
        if dense is not None:
            d = np.ascontiguousarray(dense, dtype=np.float32)
            nq, L = d.shape
            dp, ld = d.ctypes.data_as(f32p), L
            cp = cntp = None
            cap = 0
        else:
            cl = np.ascontiguousarray(cands, dtype=CAND_DTYPE)
            nq, cap = cl.shape
            cnt = np.ascontiguousarray(counts, dtype=np.uint32).reshape(nq)
            dp, ld, L = None, 0, 0
            cp, cntp = cl.ctypes.data, cnt.ctypes.data_as(u32p)
        t = np.ascontiguousarray(tau, dtype=np.float32).reshape(nq) if tau is not None else None
        sel = np.empty((nq, max(K, 1)), dtype=CAND_DTYPE)
        n = np.zeros(nq, dtype=np.uint32)
        bound = np.empty(nq, dtype=np.float32)
        _check(lib().yams_b200_debug_select(self._h, nq, dp, ld, L, row_start, row_stride, dense_shift, cp, cntp, cap,
                                            t.ctypes.data_as(f32p) if t is not None else None, K, int(tau_only), tau_margin,
                                            int(fast_tau), sel.ctypes.data, n.ctypes.data_as(u32p), bound.ctypes.data_as(f32p)),
               "debug_select")
        return bound if tau_only else (sel[:, :K], n, bound)

    def debug_final(self, exact, k: int, bound, eps, qnorm=None, threshold: float = -1.0, metric: Optional[int] = None,
                    level: int = 0, ex_n=None):
        """The scan's final ordering + exactness certificate on given survivors exact EXACT_DTYPE[Q, Kp] (rows index this
        corpus) -> (rowids i64[Q, k], scores f32[Q, k], counts u32[Q], flags u64[Q], queued queries u32[m])."""
        ex = np.ascontiguousarray(exact, dtype=EXACT_DTYPE)
        nq, Kp = ex.shape
        b = np.ascontiguousarray(bound, dtype=np.float32).reshape(nq)
        e = np.ascontiguousarray(eps, dtype=np.float32).reshape(nq)
        qn = np.ascontiguousarray(qnorm if qnorm is not None else np.ones(nq), dtype=np.float64).reshape(nq)
        en = np.ascontiguousarray(ex_n, dtype=np.uint32).reshape(nq) if ex_n is not None else None
        out_r = np.empty((nq, k), dtype=np.int64)
        out_s = np.empty((nq, k), dtype=np.float32)
        out_c = np.empty(nq, dtype=np.uint32)
        out_f = np.empty(nq, dtype=np.uint64)
        queued = np.empty(nq, dtype=np.uint32)
        nqd = C.c_uint32(0)
        _check(lib().yams_b200_debug_final(self._h, nq, Kp, k, ex.ctypes.data, en.ctypes.data_as(u32p) if en is not None else None,
                                           b.ctypes.data_as(f32p), e.ctypes.data_as(f32p), qn.ctypes.data_as(C.POINTER(C.c_double)),
                                           threshold, self.metric if metric is None else metric, level, out_r.ctypes.data_as(i64p),
                                           out_s.ctypes.data_as(f32p), out_c.ctypes.data_as(u32p), out_f.ctypes.data_as(u64p),
                                           queued.ctypes.data_as(u32p), C.byref(nqd)), "debug_final")
        return out_r, out_s, out_c, out_f, queued[:nqd.value].copy()

    def debug_stage1_profile(self, queries, tau, cap: int, max_ctas: int = 1024):
        """One profiled wgmma pass in filter mode over every row -> (cycles u64[CTAs, 4] = consumer full-barrier wait,
        producer empty-barrier wait, epilogue, total; the launch layout {n_tile, ctas}; device ms)."""
        q = np.ascontiguousarray(queries, dtype=np.float32)
        nq = q.shape[0]
        t = np.ascontiguousarray(tau, dtype=np.float32).reshape(nq)
        cyc = np.zeros((max_ctas, 4), dtype=np.uint64)
        info = np.zeros(2, dtype=np.uint32)
        ms = C.c_float(0.0)
        _check(lib().yams_b200_debug_stage1_profile(self._h, q.ctypes.data_as(f32p), nq, t.ctypes.data_as(f32p), cap, max_ctas,
                                                    cyc.ctypes.data_as(u64p), info.ctypes.data_as(u32p), C.byref(ms)),
               "debug_stage1_profile")
        layout = {"n_tile": int(info[0]), "ctas": int(info[1])}
        return cyc[:layout["ctas"]].copy(), layout, float(ms.value)

    def debug_last_eps(self, nq: int) -> np.ndarray:
        out = np.empty(nq, dtype=np.float32)
        _check(lib().yams_b200_debug_last_eps(self._h, nq, out.ctypes.data_as(f32p)), "debug_last_eps")
        return out

    def sync(self):
        _check(lib().yams_b200_corpus_sync(self._h), "corpus_sync")

    @property
    def stream(self) -> int:
        return lib().yams_b200_corpus_stream(self._h) or 0

    def last_timings(self) -> dict:
        ms = (C.c_float * 8)()
        lib().yams_b200_search_last_timings(self._h, ms)
        return {"stage1_ms": ms[0], "stage2_ms": ms[1], "total_ms": ms[2], "scan_kernel_ms": ms[5],
                "engine": "wgmma" if ms[4] else "cuda-core", "resolved_exhaustively": int(ms[6]), "resolved_full_pass": int(ms[7])}

    def close(self):
        if self._h:
            lib().yams_b200_corpus_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class SimeonEncoder:
    """The Simeon text encoder: `profile="simeon-v1-384"` (byte n-grams -> count sketch -> Achlioptas projection -> L2) or
    `profile="yams-default"` (what an unconfigured YAMS runs: byte n-grams + word tokens -> count sketch -> FWHT -> L2,
    output_dim = embedding_dim)."""

    def __init__(self, profile: str = "simeon-v1-384", embedding_dim: int = 0, **overrides):
        cfg = SimeonConfig()
        if profile == "yams-default":
            lib().yams_b200_simeon_yams_config(C.byref(cfg), embedding_dim)
        else:
            assert profile == "simeon-v1-384", profile
            lib().yams_b200_simeon_default_config(C.byref(cfg))
        for k, v in overrides.items():
            setattr(cfg, k, v)
        self.cfg = cfg
        self._h = C.c_void_p()
        _check(lib().yams_b200_simeon_create(None, C.byref(cfg), C.byref(self._h)), "simeon_create")

    def encode(self, texts) -> np.ndarray:
        raw = [t.encode("utf-8") if isinstance(t, str) else bytes(t) for t in texts]
        n = len(raw)
        out = np.zeros((n, self.cfg.output_dim), dtype=np.float32)
        if n:
            ptrs = (C.c_char_p * n)(*raw)
            lens = (C.c_size_t * n)(*[len(r) for r in raw])
            _check(lib().yams_b200_simeon_encode(self._h, ptrs, lens, n, out.ctypes.data_as(f32p)), "simeon_encode")
        return out

    def close(self):
        if getattr(self, "_h", None):
            lib().yams_b200_simeon_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _texts(texts):
    raw = [t.encode("utf-8") if isinstance(t, str) else bytes(t) for t in texts]
    n = len(raw)
    return raw, (C.c_char_p * max(n, 1))(*raw), (C.c_size_t * max(n, 1))(*[len(r) for r in raw])


def _score_call(call, n, queries, k, full):
    """the outputs of one score call over `queries`: call(ptrs, lens, nq, scores, k, docs, topk_scores, counts)"""
    raw, ptrs, lens = _texts(queries)
    nq = len(raw)
    out = {}
    scores = np.zeros((nq, n), np.float32) if full else None
    docs = np.zeros((nq, max(k, 1)), np.uint32)
    tops = np.zeros((nq, max(k, 1)), np.float32)
    counts = np.zeros(max(nq, 1), np.uint32)
    call(ptrs, lens, nq, scores.ctypes.data_as(f32p) if full else None, k, docs.ctypes.data_as(u32p), tops.ctypes.data_as(f32p),
         counts.ctypes.data_as(u32p))
    if full:
        out["scores"] = scores
    if k:
        out.update(docs=docs, topk_scores=tops, counts=counts[:nq])
    return out


class Bm25Index:
    """simeon's Bm25Index built on the device over `texts` (add_doc for each, then finalize), as the lexical backend configures it
    unless overridden: SubwordAwareBackoff, gamma 5.  `variant` is BM25_ATIRE or BM25_SUBWORD_AWARE_BACKOFF.  With lead_tokens > 0
    each document also gets its lead text (extract_lead_tokens(text, lead_tokens)) as the aux field, as the backend builds with
    the strategy router on (64)."""

    def __init__(self, texts, lead_tokens: int = 0, **overrides):
        cfg = Bm25Config()
        lib().yams_b200_bm25_default_config(C.byref(cfg))
        for k, v in overrides.items():
            setattr(cfg, k, v)
        self.cfg = cfg
        raw, ptrs, lens = _texts(texts)
        self.n = len(raw)
        self.lead_tokens = lead_tokens
        self._h = C.c_void_p()
        _check(lib().yams_b200_bm25_build_lead(None, C.byref(cfg), ptrs, lens, self.n, lead_tokens, C.byref(self._h)), "bm25_build_lead")

    def score(self, queries, k: int = 0, full: bool = True, concepts: Optional["ConceptIndex"] = None, weight: float = 0.5):
        """Bm25Index::score of every query: {"scores": [nq][n_docs] (full=True)}, and for k > 0 the best k documents of score > 0
        ("docs", "topk_scores" padded with 0xFFFFFFFF / 0, "counts").  With `concepts`, each query's scores are then blended
        with ConceptIndex::blend_into(query, scores, weight) before the top-k, as the lexical backend scores."""
        if concepts is None:
            return _score_call(lambda *args: _check(lib().yams_b200_bm25_score(self._h, *args), "bm25_score"), self.n, queries, k, full)
        return _score_call(lambda *args: _check(lib().yams_b200_bm25_score_blended(self._h, concepts._h, weight, *args), "bm25_score_blended"),
                           self.n, queries, k, full)

    def score_strategy(self, queries, strategy: int, k: int = 0, full: bool = True, concepts: Optional["ConceptIndex"] = None,
                       weight: float = 0.5):
        """The strategy router's pool `strategy` (BM25_STRATEGY_BM25: Bm25Strategy, BM25_STRATEGY_KEYPHRASE: KeyphraseStrategy,
        BM25_STRATEGY_LEAD_FIELD: LeadFieldStrategy) or its routed choice (BM25_STRATEGY_ROUTED) for every query, then with
        `concepts` blend_into(query, scores, weight): the outputs of score, and "chosen" [nq], the pool each query took."""
        nq = len(queries)
        chosen = np.zeros(max(nq, 1), np.uint32)
        out = _score_call(lambda *args: _check(lib().yams_b200_bm25_score_strategy(self._h, strategy, concepts._h if concepts is not None
                                                                                    else None, weight, *args, chosen.ctypes.data_as(u32p)),
                                               "bm25_score_strategy"), self.n, queries, k, full)
        out["chosen"] = chosen[:nq]
        return out

    def score_routed(self, queries, k: int = 0, full: bool = True, concepts: Optional["ConceptIndex"] = None, weight: float = 0.5,
                     router: Optional[RouterConfig] = None, candidates=None):
        """The lexical backend's scoreRouted with router_enabled (yams_b200_bm25_score_routed): QueryRouter's features and recipe of
        each query over this index, the recipe's scores (Bm25Atire: as this index's Atire view), then with `concepts`
        blend_into(query, scores, weight).  The outputs of score, and "recipe" [nq] (BM25_RECIPE_*), "features" [nq]
        (QUERY_FEATURES_DTYPE); with `candidates` (one sequence of document indices per query, BM25_NOT_INDEXED for a candidate the
        index does not hold), "candidates": per query the finite score of each candidate, else 0, gathered on the device."""
        nq = len(queries)
        recipe = np.zeros(max(nq, 1), np.uint32)
        feats = np.zeros(max(nq, 1), QUERY_FEATURES_DTYPE)
        off = flat = proj = None
        if candidates is not None:
            assert len(candidates) == nq
            pools = [np.asarray(c, np.uint32).ravel() for c in candidates]
            off = np.zeros(nq + 1, np.uint64)
            off[1:] = np.cumsum([len(c) for c in pools], dtype=np.uint64)
            flat = np.concatenate(pools + [np.zeros(1, np.uint32)]) if pools else np.zeros(1, np.uint32)
            proj = np.zeros(max(int(off[-1]), 1), np.float32)
        rcfg = router if router is not None else RouterConfig.default()
        out = _score_call(lambda *args: _check(lib().yams_b200_bm25_score_routed(
            self._h, C.byref(rcfg), concepts._h if concepts is not None else None, weight, *args,
            off.ctypes.data_as(u64p) if off is not None else None, flat.ctypes.data_as(u32p) if flat is not None else None,
            proj.ctypes.data_as(f32p) if proj is not None else None, recipe.ctypes.data_as(u32p), feats.ctypes.data), "bm25_score_routed"),
            self.n, queries, k, full)
        out["recipe"] = recipe[:nq]
        out["features"] = feats[:nq]
        if candidates is not None:
            out["candidates"] = [proj[int(off[i]):int(off[i + 1])] for i in range(nq)]
        return out

    def strategy_stats(self) -> dict:
        """the last score_strategy call's pools, replayed routes, boosted keyphrase rows and times"""
        s = Bm25StrategyStats()
        _check(lib().yams_b200_bm25_strategy_stats(self._h, C.byref(s)), "bm25_strategy_stats")
        return {"queries": tuple(s.queries), "replayed": s.replayed, "keyphrase_boosted": s.keyphrase_boosted, "zscore_ms": s.zscore_ms,
                "device_ms": s.device_ms, "wall_ms": s.wall_ms}

    def aux_stats(self) -> dict:
        """stats() of the lead-text fields (2 and 3); n_docs 0 when no document has a lead text"""
        s = Bm25Stats()
        _check(lib().yams_b200_bm25_aux_stats(self._h, C.byref(s)), "bm25_aux_stats")
        return {"n_docs": s.n_docs, "avg_dl": np.float32(s.avg_dl), "ngram_avg_dl": np.float32(s.ngram_avg_dl),
                "total_tokens": s.total_tokens, "terms": tuple(s.terms), "postings": tuple(s.postings), "pruned": s.pruned}

    def atire_view(self) -> "Bm25Index":
        """The Atire index of the same texts with this index's k1, b and hash seed, served from this index's word field in place
        (yams_b200_bm25_atire_view): no copy, no build.  Either may be closed first."""
        v = object.__new__(Bm25Index)
        v.cfg = Bm25Config.from_buffer_copy(self.cfg)
        v.cfg.variant = BM25_ATIRE
        v.n = self.n
        v.lead_tokens = self.lead_tokens
        v._h = C.c_void_p()
        _check(lib().yams_b200_bm25_atire_view(self._h, C.byref(v._h)), "bm25_atire_view")
        return v

    def mine_concepts(self, texts, **overrides) -> "ConceptIndex":
        """mine_concepts(this index, texts, ConceptConfig) on the device; overrides: min_ttf, pmi_floor, max_concepts, k1, b."""
        return ConceptIndex(self, texts, **overrides)

    def stats(self) -> dict:
        s = Bm25Stats()
        _check(lib().yams_b200_bm25_stats(self._h, C.byref(s)), "bm25_stats")
        return {"n_docs": s.n_docs, "avg_dl": np.float32(s.avg_dl), "ngram_avg_dl": np.float32(s.ngram_avg_dl),
                "total_tokens": s.total_tokens, "terms": tuple(s.terms), "postings": tuple(s.postings), "pruned": s.pruned}

    def postings(self, field: int, term_hash: int):
        """(docs, tfs, idf, total_tf) of a hash in field 0 (words), 1 (n-grams), 2 (lead words) or 3 (lead n-grams); empty lists
        and 0 when absent."""
        df, idf, ttf = C.c_uint32(), C.c_float(), C.c_uint64()
        _check(lib().yams_b200_bm25_postings(self._h, field, term_hash, C.byref(df), C.byref(idf), C.byref(ttf), None, None, 0), "bm25_postings")
        docs = np.zeros(max(df.value, 1), np.uint32)
        tfs = np.zeros(max(df.value, 1), np.uint32)
        _check(lib().yams_b200_bm25_postings(self._h, field, term_hash, C.byref(df), C.byref(idf), C.byref(ttf), docs.ctypes.data_as(u32p),
                                             tfs.ctypes.data_as(u32p), df.value), "bm25_postings")
        return docs[:df.value], tfs[:df.value], np.float32(idf.value), ttf.value

    def doc_lengths(self, field: int = 0) -> np.ndarray:
        out = np.zeros(max(self.n, 1), np.uint32)
        _check(lib().yams_b200_bm25_doc_lengths(self._h, field, out.ctypes.data_as(u32p)), "bm25_doc_lengths")
        return out[:self.n]

    def last_timings(self) -> dict:
        ms = (C.c_float * 8)()
        _check(lib().yams_b200_bm25_last_timings(self._h, ms), "bm25_last_timings")
        return {"build_upload_ms": ms[0], "build_tokenise_ms": ms[1], "build_sort_ms": ms[2], "build_postings_ms": ms[3],
                "build_wall_ms": ms[4], "build_slices": int(ms[5]), "score_device_ms": ms[6], "score_wall_ms": ms[7]}

    def close(self):
        if getattr(self, "_h", None):
            lib().yams_b200_bm25_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class PqIndex:
    """SimeonPqAdc index over a Corpus (codes in HBM beside the rows); search = ADC scan + exact rerank."""

    def __init__(self, corpus: Corpus, m: int, k: int, codebooks: np.ndarray, tie_break_keys=None):
        cb = np.ascontiguousarray(codebooks, dtype=np.float32)
        assert cb.size == m * k * (corpus.dim // m)
        tk = np.ascontiguousarray(tie_break_keys, dtype=np.uint64) if tie_break_keys is not None else None
        self._h = C.c_void_p()
        self.m, self.k, self._corpus = m, k, corpus
        _check(lib().yams_b200_pq_build(corpus.handle, m, k, cb.ctypes.data_as(f32p), tk.ctypes.data_as(u64p) if tk is not None else None,
                                        C.byref(self._h)), "pq_build")

    def codes(self):
        n = C.c_uint64(0)
        _check(lib().yams_b200_pq_codes(self._h, None, None, C.byref(n)), "pq_codes")
        codes = np.zeros((max(n.value, 1), self.m), dtype=np.uint8)
        rowids = np.zeros(max(n.value, 1), dtype=np.int64)
        _check(lib().yams_b200_pq_codes(self._h, codes.ctypes.data, rowids.ctypes.data, C.byref(n)), "pq_codes")
        return codes[:n.value], rowids[:n.value]

    @property
    def handle(self):
        return self._h

    def search(self, queries, k: int, rerank_factor: int = 2, threshold: float = 0.0, allowed=None):
        """-> (rowids i64[Q,k], scores f32[Q,k], counts u32[Q], flags u64[Q]).  allowed: optional list (len Q) of rowid arrays
        (any order): query i only scores the indexed rows of allowed[i] (simeonPqSearchUnlocked with candidate documents)."""
        q = np.ascontiguousarray(queries, dtype=np.float32)
        if q.ndim == 1:
            q = q[None, :]
        nq = q.shape[0]
        out_r = np.full((nq, max(k, 1)), -1, dtype=np.int64)
        out_s = np.zeros((nq, max(k, 1)), dtype=np.float32)
        out_c = np.zeros(nq, dtype=np.uint32)
        out_f = np.zeros(nq, dtype=np.uint64)
        if allowed is None:
            _check(lib().yams_b200_pq_search(self._h, q.ctypes.data_as(f32p), nq, k, rerank_factor, threshold, out_r.ctypes.data_as(i64p),
                                             out_s.ctypes.data_as(f32p), out_c.ctypes.data_as(u32p), out_f.ctypes.data_as(u64p)), "pq_search")
        else:
            assert len(allowed) == nq
            offs = np.zeros(nq + 1, dtype=np.uint64)
            offs[1:] = np.cumsum([len(a) for a in allowed])
            al = np.ascontiguousarray(np.concatenate([np.asarray(a, dtype=np.int64).reshape(-1) for a in allowed])
                                      if nq and int(offs[-1]) else np.zeros(1, dtype=np.int64), dtype=np.int64)
            _check(lib().yams_b200_pq_search_candidates(self._h, q.ctypes.data_as(f32p), nq, k, rerank_factor, threshold,
                                                        al.ctypes.data_as(i64p), offs.ctypes.data_as(u64p), out_r.ctypes.data_as(i64p),
                                                        out_s.ctypes.data_as(f32p), out_c.ctypes.data_as(u32p), out_f.ctypes.data_as(u64p)),
                   "pq_search_candidates")
        return out_r[:, :k], out_s[:, :k], out_c, out_f

    def debug_lut(self, queries):
        """-> (lookup tables f32[Q, m, k], valid u32[Q]) as pq_search computes them"""
        q = np.ascontiguousarray(queries, dtype=np.float32).reshape(-1, self._corpus.dim)
        nq = q.shape[0]
        out = np.zeros((nq, self.m, self.k), dtype=np.float32)
        valid = np.zeros(nq, dtype=np.uint32)
        _check(lib().yams_b200_debug_pq_lut(self._h, q.ctypes.data_as(f32p), nq, out.ctypes.data_as(f32p), valid.ctypes.data_as(u32p)),
               "debug_pq_lut")
        return out, valid

    def last_path(self) -> dict:
        """the ADC pass the last search (without candidate lists) took: filtered, queries per CTA (qg), sampled tiles, rerun"""
        out = (C.c_uint32 * 4)()
        _check(lib().yams_b200_debug_pq_last_path(self._h, out), "debug_pq_last_path")
        return {"filtered": bool(out[0]), "qg": int(out[1]), "sample_tiles": int(out[2]), "rerun": bool(out[3])}

    def close(self):
        if getattr(self, "_h", None):
            lib().yams_b200_pq_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def vec0_exact(query, rows, k: int = 0, rowids=None, rowid_range=None):
    """vec0_run_exact_query: (rowids, distances) ascending by L2 distance."""
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    q = np.ascontiguousarray(query, dtype=np.float32)
    n, d = rows.shape if rows.ndim == 2 else (0, q.size)
    out_r = np.zeros(max(n, 1), dtype=np.int64)
    out_d = np.zeros(max(n, 1), dtype=np.float32)
    cnt = C.c_uint64(0)
    rid = np.ascontiguousarray(rowids, dtype=np.int64) if rowids is not None else None
    lo, hi = rowid_range if rowid_range is not None else (0, 0)
    rc = lib().yams_b200_vec0_exact(None, q.ctypes.data_as(f32p), d, rows.ctypes.data_as(f32p),
                                    rid.ctypes.data_as(i64p) if rid is not None else None, n, k,
                                    int(rowid_range is not None), lo, hi, out_r.ctypes.data_as(i64p),
                                    out_d.ctypes.data_as(f32p), C.byref(cnt))
    _check(rc, "vec0_exact")
    return out_r[:cnt.value].copy(), out_d[:cnt.value].copy()


class DigestSet:
    """Device-resident set of chunk digests: the batched `storage_->exists` / `store` loop
    (content_store_impl.cpp:245-288)."""

    def __init__(self, capacity_hint: int = 0):
        h = C.c_void_p()
        _check(lib().yams_b200_digest_set_create(None, capacity_hint, C.byref(h)), "digest_set_create")
        self._h = h

    @staticmethod
    def _digests(x):
        """chunk table (structured, field 'digest') or [n,32] uint8 -> (base pointer, stride, n, keepalive)"""
        a = np.asarray(x)
        if a.dtype.names and "digest" in a.dtype.names:
            a = np.ascontiguousarray(a)
            off = a.dtype.fields["digest"][1]
            return a.ctypes.data + off, a.dtype.itemsize, len(a), a
        a = np.ascontiguousarray(a, dtype=np.uint8).reshape(-1, 32)
        return a.ctypes.data, 32, len(a), a

    def insert(self, digests):
        """-> (existed uint8[n], n_new)"""
        ptr, stride, n, keep = self._digests(digests)
        existed = np.zeros(max(n, 1), dtype=np.uint8)
        new = C.c_uint64(0)
        _check(lib().yams_b200_digest_set_insert(self._h, ptr if n else None, stride, n, existed.ctypes.data, C.byref(new)),
               "digest_set_insert")
        return existed[:n], new.value

    def contains(self, digests) -> np.ndarray:
        ptr, stride, n, keep = self._digests(digests)
        out = np.zeros(max(n, 1), dtype=np.uint8)
        _check(lib().yams_b200_digest_set_contains(self._h, ptr if n else None, stride, n, out.ctypes.data), "digest_set_contains")
        return out[:n]

    def __len__(self):
        n = C.c_uint64(0)
        _check(lib().yams_b200_digest_set_size(self._h, C.byref(n)), "digest_set_size")
        return n.value

    def last_ms(self) -> float:
        v = C.c_float(0)
        _check(lib().yams_b200_digest_set_last_ms(self._h, C.byref(v)), "digest_set_last_ms")
        return v.value

    def close(self):
        if getattr(self, "_h", None):
            lib().yams_b200_digest_set_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


BATCH_ALL, BATCH_TOP_K, BATCH_FILTERED = 0, 1, 2


def batch_distance(query, database, metric: int = COSINE, mode: int = BATCH_ALL, k: int = 0, threshold: float = 0.0):
    """distances/batch.hpp: ALL -> dist[n]; TOP_K -> (idx[k], dist[k]); FILTERED -> (idx[m], dist[m])."""
    q = np.ascontiguousarray(query, dtype=np.float32).reshape(-1)
    db = np.ascontiguousarray(database, dtype=np.float32)
    n = db.shape[0] if db.ndim == 2 else 0
    out_i = np.zeros(max(n, 1), dtype=np.uint64)
    out_d = np.zeros(max(n, 1), dtype=np.float32)
    cnt = C.c_uint64(0)
    rc = lib().yams_b200_batch_distance(None, metric, q.ctypes.data_as(f32p), q.size, db.ctypes.data_as(f32p) if n else None,
                                        n, mode, k, threshold, out_i.ctypes.data_as(u64p), out_d.ctypes.data_as(f32p),
                                        C.byref(cnt))
    _check(rc, "batch_distance")
    if mode == BATCH_ALL:
        return out_d[:cnt.value].copy()
    return out_i[:cnt.value].copy(), out_d[:cnt.value].copy()


def compute_cosine_similarity(a, b) -> float:
    """VectorDatabase::computeCosineSimilarity (double)."""
    a = np.ascontiguousarray(a, dtype=np.float32).reshape(-1)
    b = np.ascontiguousarray(b, dtype=np.float32).reshape(-1)
    out = C.c_double(0)
    _check(lib().yams_b200_compute_cosine_similarity(None, a.ctypes.data_as(f32p), a.size, b.ctypes.data_as(f32p), b.size,
                                                     C.byref(out)), "compute_cosine_similarity")
    return out.value


def compute_cosine_similarity_many(a, b) -> np.ndarray:
    """n pairs in one device pass: a[n, d], b[n, d] -> float64[n]."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    b = np.ascontiguousarray(b, dtype=np.float32)
    assert a.shape == b.shape and a.ndim == 2
    out = np.zeros(a.shape[0], dtype=np.float64)
    _check(lib().yams_b200_compute_cosine_similarity_many(None, a.ctypes.data_as(f32p), b.ctypes.data_as(f32p), a.shape[0], a.shape[1],
                                                          out.ctypes.data_as(C.POINTER(C.c_double))), "compute_cosine_similarity_many")
    return out


def _pair(fn, a, b):
    a = np.ascontiguousarray(a, dtype=np.float32)
    b = np.ascontiguousarray(b, dtype=np.float32)
    out = C.c_float(0)
    rc = fn(a.ctypes.data, a.nbytes, b.ctypes.data, b.nbytes, C.byref(out))
    return rc, out.value


def vec_distance_l2(a, b):
    return _pair(lib().sqlite3_vec_distance_l2, a, b)


def vec_distance_cosine(a, b):
    return _pair(lib().sqlite3_vec_distance_cosine, a, b)


def vec_distance_l1(a, b):
    return _pair(lib().yams_b200_vec_distance_l1, a, b)


class ConceptIndex:
    """simeon's ConceptIndex mined on the device against a Bm25Index (Bm25Index.mine_concepts).  It holds what it scores with and
    may outlive the index."""

    def __init__(self, index: Bm25Index, texts, **overrides):
        cfg = ConceptConfig()
        lib().yams_b200_concepts_default_config(C.byref(cfg))
        for k, v in overrides.items():
            setattr(cfg, k, v)
        self.cfg = cfg
        raw, ptrs, lens = _texts(texts)
        self.n = len(raw)
        self._h = C.c_void_p()
        _check(lib().yams_b200_concepts_mine(index._h, C.byref(cfg), ptrs, lens, self.n, C.byref(self._h)), "concepts_mine")

    def stats(self) -> dict:
        s = ConceptStats()
        _check(lib().yams_b200_concepts_stats(self._h, C.byref(s)), "concepts_stats")
        return {"size": s.size, "doc_count": s.doc_count, "avg_bigram_dl": np.float32(s.avg_bigram_dl), "replayed": bool(s.replayed),
                "sum_bigram_dl": s.sum_bigram_dl, "distinct": s.distinct, "passed_min_ttf": s.passed_min_ttf, "accepted": s.accepted}

    def find(self, concept_hash: int):
        """ConceptIndex::find: None when absent, else {"pmi", "idf", "total_tf", "a_hash", "b_hash", "docs", "tfs"}."""
        found, df = C.c_uint32(), C.c_uint32()
        pmi, idf = C.c_float(), C.c_float()
        ttf, a, b = C.c_uint64(), C.c_uint64(), C.c_uint64()
        refs = [C.byref(v) for v in (found, pmi, idf, ttf, a, b, df)]
        _check(lib().yams_b200_concepts_find(self._h, concept_hash, *refs, None, None, 0), "concepts_find")
        if not found.value:
            return None
        docs = np.zeros(max(df.value, 1), np.uint32)
        tfs = np.zeros(max(df.value, 1), np.uint32)
        _check(lib().yams_b200_concepts_find(self._h, concept_hash, *refs, docs.ctypes.data_as(u32p), tfs.ctypes.data_as(u32p), df.value),
               "concepts_find")
        return {"pmi": np.float32(pmi.value), "idf": np.float32(idf.value), "total_tf": ttf.value, "a_hash": a.value, "b_hash": b.value,
                "docs": docs[:df.value], "tfs": tfs[:df.value]}

    def hashes(self) -> np.ndarray:
        """the kept concepts' hashes, ascending"""
        size = self.stats()["size"]
        out = np.zeros(max(size, 1), np.uint64)
        _check(lib().yams_b200_concepts_hashes(self._h, out.ctypes.data_as(u64p)), "concepts_hashes")
        return out[:size]

    def bigram_lengths(self) -> np.ndarray:
        out = np.zeros(max(self.n, 1), np.uint32)
        _check(lib().yams_b200_concepts_bigram_lengths(self._h, out.ctypes.data_as(u32p)), "concepts_bigram_lengths")
        return out[:self.n]

    def blend(self, query, scores: np.ndarray, weight: float = 0.5) -> np.ndarray:
        """ConceptIndex::blend_into(query, scores, weight) on a copy of the float32 vector `scores`, which is returned."""
        q = query.encode("utf-8") if isinstance(query, str) else bytes(query)
        out = np.array(scores, dtype=np.float32, copy=True).reshape(-1)
        _check(lib().yams_b200_concepts_blend(self._h, q, len(q), weight, out.ctypes.data_as(f32p), out.size), "concepts_blend")
        return out

    def last_timings(self) -> dict:
        ms = (C.c_float * 8)()
        _check(lib().yams_b200_concepts_last_timings(self._h, ms), "concepts_last_timings")
        return {"upload_ms": ms[0], "tokenise_ms": ms[1], "sort_ms": ms[2], "runs_filter_ms": ms[3], "gather_ms": ms[4],
                "host_ms": ms[5], "replay_ms": ms[6], "wall_ms": ms[7]}

    def close(self):
        if getattr(self, "_h", None):
            lib().yams_b200_concepts_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def bm25_score_rrf(indexes, queries, k: int = 0, full: bool = True, k_rrf: float = 60.0, concepts: Optional[ConceptIndex] = None,
                   weight: float = 0.5):
    """score_bm25_variants_rrf(indexes, query, scores, k_rrf) of every query, then with `concepts` ConceptIndex::blend_into(query,
    scores, weight): the lexical backend's score with bm25_variants_rrf on (yams_b200_bm25_score_rrf).  The outputs of
    Bm25Index.score; the score rows have the indexes' document count (0 without indexes)."""
    nv = len(indexes)
    hs = (C.c_void_p * max(nv, 1))(*[i._h for i in indexes])
    n = indexes[0].n if nv else 0
    return _score_call(lambda *args: _check(lib().yams_b200_bm25_score_rrf(hs, nv, k_rrf, concepts._h if concepts is not None else None,
                                                                            weight, *args), "bm25_score_rrf"), n, queries, k, full)
