"""simeon's reciprocal-rank fusion of BM25 variants (score_bm25_variants_rrf, third_party/simeon/src/fusion.cpp:24-63)
restated in float32 numpy over the restated indexes (tests/bm25_restated.py) and concept index (tests/concepts_restated.py).

Each variant, in the given order, ranks the documents of finite score > 0 by score descending, then document ascending; rank
r = 1, 2, ... adds 1.0f / (k + float(r)) to its document (two roundings), the variants' additions accumulating in their order
from 0.0f.  With a concept index the lexical backend then blends onto the fused scores (ConceptIndex::blend_into).

RefRrf below drives the reference's own fusion through oracle/_ref/libref_rrf.so (oracle/rrf.mk)."""
import ctypes as C
import functools
import os

import numpy as np

from tests import bm25_restated as B
from tests import concepts_restated as R

f32 = np.float32
_REF_SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libref_rrf.so")


def ranking(scores: np.ndarray, ties_descending: bool = False) -> np.ndarray:
    """the ranked documents of one variant's scores (fusion.cpp:14-20); ties_descending reverses the document tie order"""
    s = np.asarray(scores, np.float32)
    pos = np.flatnonzero(np.isfinite(s) & (s > 0))
    return pos[np.lexsort((-pos if ties_descending else pos, -s[pos].astype(np.float64)))]


def contributions(m: int, k_rrf: float) -> np.ndarray:
    """1.0f / (k + float(r)) for r = 1..m"""
    return f32(1.0) / (f32(k_rrf) + np.arange(1, m + 1, dtype=np.uint64).astype(np.float32))


def fuse(rows, n: int, k_rrf: float, ties_descending: bool = False) -> np.ndarray:
    """rrf_fuse of the variants' score rows, in their order, written into a zeroed vector of n"""
    out = np.zeros(n, np.float32)
    for s in rows:
        d = ranking(s, ties_descending)
        out[d] = out[d] + contributions(len(d), k_rrf)
    return out


def score(indexes, query: bytes, k_rrf: float = 60.0, concepts=None, weight: float = 0.5, n: int = None,
          ties_descending: bool = False) -> np.ndarray:
    """SimeonLexicalBackend::score with bm25_variants_rrf: the fusion of the restated indexes' scores, then the blend"""
    n = indexes[0].n if indexes else (0 if n is None else n)
    with np.errstate(all="ignore"):
        out = fuse([X.score(query) for X in indexes], n, k_rrf, ties_descending)
        if concepts is not None:
            out = concepts.blend(query, out, weight)
    return out


# ---- the reference's own fusion (oracle/_ref/libref_rrf.so) ----
def have_ref() -> bool:
    return os.path.exists(_REF_SO)


@functools.lru_cache(maxsize=None)
def _refl():
    L = C.CDLL(_REF_SO)
    p = C.c_void_p
    L.ref_rrf_index.restype = p
    L.ref_rrf_index.argtypes = [p, p, p, C.c_size_t]
    L.ref_rrf_index_destroy.argtypes = [p]
    L.ref_rrf_concepts.restype = p
    L.ref_rrf_concepts.argtypes = [p, p, p, p, C.c_size_t]
    L.ref_rrf_concepts_destroy.argtypes = [p]
    L.ref_rrf_score.argtypes = [p, C.c_size_t, C.c_char_p, C.c_size_t, C.c_float, p, C.c_float, p, C.c_size_t]
    return L


class RefIndex:
    """simeon::Bm25Index over texts, as the fusion reads it"""

    def __init__(self, cfg: B.Config, texts):
        c = B._Cfg(cfg.k1, cfg.b, cfg.delta, cfg.gamma, cfg.variant, cfg.ngram_min, cfg.ngram_max, cfg.prune_ratio, cfg.hash_seed)
        self._keep = R._arr(texts)
        _, ptrs, lens, self.n = self._keep
        self._h = _refl().ref_rrf_index(C.byref(c), ptrs, lens, self.n)

    def __del__(self):
        try:
            _refl().ref_rrf_index_destroy(self._h)
        except Exception:
            pass


class RefConcepts:
    """simeon::mine_concepts(index, texts, cfg)"""

    def __init__(self, index: RefIndex, texts, cfg: R.CCfg = R.CCfg()):
        cc = R._RefCCfg(cfg.min_ttf, cfg.pmi_floor, cfg.max_concepts, cfg.k1, cfg.b)
        self._keep = (index, R._arr(texts))
        _, ptrs, lens, n = self._keep[1]
        self._h = _refl().ref_rrf_concepts(index._h, C.byref(cc), ptrs, lens, n)

    def __del__(self):
        try:
            _refl().ref_rrf_concepts_destroy(self._h)
        except Exception:
            pass


def ref_score(indexes, query: bytes, k_rrf: float = 60.0, concepts: RefConcepts = None, weight: float = 0.5, n: int = None):
    """the reference: score_bm25_variants_rrf(indexes, query, out[n], k_rrf), then blend_into with concepts"""
    n = indexes[0].n if indexes else (0 if n is None else n)
    hs = (C.c_void_p * max(len(indexes), 1))(*[i._h for i in indexes])
    out = np.full(n, -1.0, np.float32)   # the reference fills it
    _refl().ref_rrf_score(hs, len(indexes), bytes(query), len(query), k_rrf, concepts._h if concepts else None, weight,
                          out.ctypes.data, n)
    return out


# ---- the cases the stored answers, the CPU pin and the device tests share ----
SAB = B.Config()
ATIRE = B.Config(variant=B.ATIRE)
OTHER = B.Config(k1=1.6, b=0.5, delta=0.5, gamma=1.0, ngram_min=2, ngram_max=5, prune_ratio=0.3)   # a third config


def tie_corpus(seed: int, n: int):
    """a concept corpus in which every document appears several times: heavy score ties within every ranking"""
    docs, voc, ph = R.gen_concept_corpus(seed, max(1, n // 4), 20, 600, 20, 2)
    rng = np.random.default_rng(seed)
    return [docs[int(i)] for i in rng.integers(0, len(docs), n)], voc, ph


def ngram_queries(voc, nq: int, seed: int):
    """queries of word fragments: the n-gram field ranks documents the word field does not"""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(nq):
        ws = [w for w in (voc[int(i)] for i in rng.integers(0, min(len(voc), 200), 3)) if len(w) >= 4]
        out.append(b" ".join(w[1:-1] if rng.random() < 0.6 else w for w in ws))
    return out


def case_inputs(case):
    """(docs, queries, variant configs) of a stored case"""
    if case["corpus"] == "ties":
        docs, voc, ph = tie_corpus(case["seed"], case["n"])
    elif case["corpus"] == "catch2":
        docs, voc, ph = [b"alpha beta", b"gamma delta"], [], []
    else:
        docs, voc, ph = R.gen_concept_corpus(case["seed"], case["n"], 30, 1500, 40, 0)
    if case["corpus"] == "catch2":
        queries = [b"absent"]
    elif case["queries"] == "ngram":
        queries = ngram_queries(voc, case["nq"], case["seed"] + 2)
    else:
        queries = R.gen_concept_queries(case["seed"] + 1, voc, ph, case["nq"]) + [b"", b"qqqqzz xxyyy"]
    cfgs = [{"sab": SAB, "atire": ATIRE, "other": OTHER}[v] for v in case["variants"]]
    return docs, queries, cfgs


# the CPU pin's and the device tests' grid: document count, variants, k_rrf, blend weight (None: plain)
GRID = [
    (1, ["sab", "atire"], 60.0, None),
    (37, ["sab", "atire"], 60.0, 0.5),
    (300, ["sab", "atire"], 0.0, 0.5),
    (300, ["atire", "sab"], 1.5, None),
    (600, ["sab", "atire", "other"], 60.0, 0.5),
    (600, ["other", "sab", "atire"], 1e6, None),
    (600, ["sab", "sab", "atire"], 60.0, 1.0),
    (1000, ["other"], 60.0, -0.5),
    (2000, ["sab", "atire"], 60.0, 0.5),
]


def grid_case(n, variants, seed=None):
    """(docs, queries, configs) of a grid point"""
    seed = seed if seed is not None else 300 + n
    docs, voc, ph = R.gen_concept_corpus(seed, n, 25, 900, 30, 0)
    queries = R.gen_concept_queries(seed + 1, voc, ph, 20) + ngram_queries(voc, 6, seed + 2) + [b"", b"zzqx"]
    return docs, queries, [{"sab": SAB, "atire": ATIRE, "other": OTHER}[v] for v in variants]
