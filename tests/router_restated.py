"""simeon's QueryRouter (third_party/simeon/src/query_router.cpp) and the lexical backend's routed dispatch
(SimeonLexicalBackend::scoreRouted with router_enabled, simeon_lexical_backend.cpp:836-934) restated over the restated indexes
(tests/bm25_restated.py) and concept index (tests/concepts_restated.py).

features(query) reads df, idf and total_tf of the index's word field for each query word WITHOUT case folding (the index folds,
so a word with an uppercase letter is out of vocabulary for the router), in double with glibc log (Python's math.log); choose
picks the recipe; Bm25Atire rows score with the Atire index of the same texts, the others with the primary; the concept blend
follows, then the projection onto the candidate pool.

RefIndex / ref_score below drive the reference's own router through oracle/_ref/libref_router.so (oracle/router.mk)."""
import ctypes as C
import functools
import math
import os
from dataclasses import dataclass, fields

import numpy as np

from tests import bm25_restated as B
from tests import concepts_restated as R

f32 = np.float32
_REF_SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libref_router.so")
ATIRE, SAB_SMOOTH, CASCADE = 0, 1, 2   # simeon::Recipe
NOT_INDEXED = 0xFFFFFFFF
FEATURES = ("oov_rate", "avg_idf", "max_idf", "min_idf", "idf_stddev", "n_terms", "avg_term_chars", "scq_sum", "simplified_clarity")


@dataclass
class RCfg:
    """simeon::RouterConfig's routing fields at the lexical backend's RouterPreset (passE: atire_max_clarity 3)"""
    oov_threshold: float = 0.0
    high_idf_threshold: float = 3.0
    atire_min_terms: int = 0
    atire_min_idf_floor: float = 0.0
    atire_max_pool_jaccard: float = 1.0
    atire_min_score_decay: float = 0.0
    atire_min_scq: float = 0.0
    atire_max_clarity: float = 3.0
    cascade_min_terms: int = 4
    cascade_max_idf: float = 5.0

    def kw(self):
        return {f.name: getattr(self, f.name) for f in fields(self)}


class _RCfg(C.Structure):   # yams_bm25_router_config
    _fields_ = [("oov_threshold", C.c_float), ("high_idf_threshold", C.c_float), ("atire_min_terms", C.c_uint32),
                ("atire_min_idf_floor", C.c_float), ("atire_max_pool_jaccard", C.c_float), ("atire_min_score_decay", C.c_float),
                ("atire_min_scq", C.c_float), ("atire_max_clarity", C.c_float), ("cascade_min_terms", C.c_uint32),
                ("cascade_max_idf", C.c_float)]


class _Feats(C.Structure):   # yams_bm25_query_features
    _fields_ = [(n, C.c_uint32 if n == "n_terms" else C.c_float) for n in FEATURES]


def router_words(query: bytes, fold: bool = False):
    """emit_word_tokens (tokenizer.cpp:40-52): the word runs of the query, in order, NOT lowercased (fold: lowercased)"""
    return [m.group(0).lower() if fold else m.group(0) for m in B._WORD.finditer(bytes(query))]


def features(X: B.Index, query: bytes, fold: bool = False, distinct_terms: bool = False) -> dict:
    """QueryRouter::features over X's word field.  fold lowercases the router's words, distinct_terms counts each distinct word
    once in n_terms: both are wrong, and the teeth tests show they change stored answers."""
    ws = router_words(query, fold)
    if distinct_terms:
        ws = list(dict.fromkeys(ws))
    f = {k: f32(0) for k in FEATURES}
    f["n_terms"] = len(ws)
    if not ws:
        return f
    oov = present = char_sum = 0
    idf_sum = idf_sq = scq = 0.0
    min_seen = f32(np.inf)
    q_count = {}
    stats = []
    for w in ws:
        char_sum += len(w)
        h = B.hash64(w, X.cfg.hash_seed)
        p = X.words.postings.get(h)
        stats.append((h, p))
        if p is None:
            oov += 1
            continue
        i, ttf = p[2], p[3]
        idf_sum += float(i)
        idf_sq += float(i) * float(i)
        if i > f["max_idf"]:
            f["max_idf"] = i
        if i < min_seen:
            min_seen = i
        present += 1
        if ttf > 0:
            scq += (1.0 + math.log(float(ttf))) * float(i)
        q_count[h] = q_count.get(h, 0) + 1
    f["oov_rate"] = f32(oov) / f32(len(ws))
    if present:
        f["avg_idf"] = f32(idf_sum / present)
        f["min_idf"] = min_seen
        if present > 1:
            mean = idf_sum / present
            var = idf_sq / present - mean * mean
            f["idf_stddev"] = f32(math.sqrt(var) if var > 0.0 else 0.0)
    f["avg_term_chars"] = f32(float(char_sum) / float(len(ws)))
    f["scq_sum"] = f32(scq)
    if q_count and X.total_tokens > 0:
        acc, seen = 0.0, set()
        for h, p in stats:   # distinct hashes in first-occurrence order
            if h in seen:
                continue
            seen.add(h)
            if p is None or p[3] == 0:
                continue
            p_q, p_c = q_count[h] / float(len(ws)), float(p[3]) / float(X.total_tokens)
            acc += p_q * math.log(p_q / p_c)
        f["simplified_clarity"] = f32(acc)
    return f


def choose(f: dict, cfg: RCfg = RCfg()) -> int:
    """QueryRouter::choose; the pool signals stay at features()'s no-signal defaults (jaccard 1, decay 0)"""
    c = {k: (v if isinstance(v, int) else f32(v)) for k, v in cfg.kw().items()}
    if f["n_terms"] == 0 or f["oov_rate"] > c["oov_threshold"]:
        return SAB_SMOOTH
    if (f["avg_idf"] > c["high_idf_threshold"] and f["n_terms"] >= c["atire_min_terms"] and f["min_idf"] >= c["atire_min_idf_floor"]
            and f32(1.0) <= c["atire_max_pool_jaccard"] and f32(0.0) >= c["atire_min_score_decay"] and f["scq_sum"] >= c["atire_min_scq"]
            and f["simplified_clarity"] <= c["atire_max_clarity"]):
        return ATIRE
    if f["n_terms"] >= c["cascade_min_terms"] and f["avg_idf"] <= c["cascade_max_idf"]:
        return CASCADE
    return SAB_SMOOTH


def project(row: np.ndarray, cands) -> np.ndarray:
    """scoreRouted's projection: the row's finite score of each candidate, 0 for a non-finite score or NOT_INDEXED"""
    c = np.asarray(cands, np.uint32)
    out = np.zeros(len(c), np.float32)
    ok = c != NOT_INDEXED
    v = row[c[ok].astype(np.int64)]
    out[ok] = np.where(np.isfinite(v), v, f32(0))
    return out


def score(X: B.Index, A: B.Index, query: bytes, cfg: RCfg = RCfg(), K: R.Concepts = None, weight: float = 0.5, **kw):
    """scoreRouted over primary X and its Atire index A (None when X is Atire): (recipe, features, scores)"""
    f = features(A if A is not None else X, query, **kw)
    r = choose(f, cfg)
    row = (A if r == ATIRE and A is not None else X).score(query)
    if K is not None:
        with np.errstate(all="ignore"):
            row = K.blend(query, row, weight)
    return r, f, row


def atire_of(cfg: B.Config):
    """the backend's second index beside a SubwordAwareBackoff primary: Atire with Bm25Config's defaults (None for Atire)"""
    return None if cfg.variant == B.ATIRE else B.Config(variant=B.ATIRE)


# ---- the reference's own router (oracle/_ref/libref_router.so) ----
def have_ref() -> bool:
    return os.path.exists(_REF_SO)


@functools.lru_cache(maxsize=None)
def _refl():
    L = C.CDLL(_REF_SO)
    p = C.c_void_p
    L.ref_router_index.restype = p
    L.ref_router_index.argtypes = [p, p, p, C.c_size_t]
    L.ref_router_index_destroy.argtypes = [p]
    L.ref_router_concepts.restype = p
    L.ref_router_concepts.argtypes = [p, p, p, p, C.c_size_t]
    L.ref_router_concepts_destroy.argtypes = [p]
    L.ref_router_score.argtypes = [p, p, p, C.c_char_p, C.c_size_t, p, C.c_float, p, C.c_size_t, p, C.c_size_t, p, p, p]
    return L


class RefIndex:
    """simeon::Bm25Index over texts"""

    def __init__(self, cfg: B.Config, texts):
        c = B._Cfg(cfg.k1, cfg.b, cfg.delta, cfg.gamma, cfg.variant, cfg.ngram_min, cfg.ngram_max, cfg.prune_ratio, cfg.hash_seed)
        self._keep = R._arr(texts)
        _, ptrs, lens, self.n = self._keep
        self._h = _refl().ref_router_index(C.byref(c), ptrs, lens, self.n)

    def __del__(self):
        try:
            _refl().ref_router_index_destroy(self._h)
        except Exception:
            pass


class RefConcepts:
    """simeon::mine_concepts(index, texts, cfg)"""

    def __init__(self, index: RefIndex, texts, cfg: R.CCfg = R.CCfg()):
        cc = R._RefCCfg(cfg.min_ttf, cfg.pmi_floor, cfg.max_concepts, cfg.k1, cfg.b)
        self._keep = (index, R._arr(texts))
        _, ptrs, lens, n = self._keep[1]
        self._h = _refl().ref_router_concepts(index._h, C.byref(cc), ptrs, lens, n)

    def __del__(self):
        try:
            _refl().ref_router_concepts_destroy(self._h)
        except Exception:
            pass


def ref_score(X: RefIndex, A: RefIndex, query: bytes, cfg: RCfg = RCfg(), K: RefConcepts = None, weight: float = 0.5, cands=()):
    """the reference's scoreRouted: (recipe, features, scores, projection of cands)"""
    rc = _RCfg(**cfg.kw())
    out = np.full(X.n, -1.0, np.float32)
    cand = np.ascontiguousarray(cands, np.uint32)
    proj = np.full(max(len(cand), 1), -1.0, np.float32)
    recipe = C.c_uint32()
    fe = _Feats()
    _refl().ref_router_score(X._h, A._h if A is not None else None, C.byref(rc), bytes(query), len(query), K._h if K is not None else None,
                             weight, out.ctypes.data, X.n, cand.ctypes.data, len(cand), proj.ctypes.data, C.byref(recipe), C.byref(fe))
    f = {k: (int(getattr(fe, k)) if k == "n_terms" else f32(getattr(fe, k))) for k in FEATURES}
    return recipe.value, f, out, proj[:len(cand)]


# ---- corpora and queries that reach every recipe and both sides of every threshold ----
def gen_router_corpus(seed: int, n: int):
    """B.gen_corpus documents (mixed case, bytes >= 0x80, empty documents) with planted phrases, plus bursty words: each in a few
    documents many times (high idf and high total_tf, hence low clarity).  -> (docs, vocabulary, phrases, bursty words)"""
    docs, voc, ph = R.gen_concept_corpus(seed, n, 30, 1500, 40, 0)
    rng = np.random.default_rng(seed + 11)
    burst = [b"burst%d" % i for i in range(40)]
    docs = list(docs)
    for i, w in enumerate(burst):
        for d in rng.choice(n, size=min(n, 1 + i % 12), replace=False) if n else []:
            docs[int(d)] += b" " + b" ".join([w] * int(rng.integers(20, 300)))
    return docs, voc, ph, burst


def gen_router_queries(seed: int, voc, ph, burst, nq: int):
    """random queries mixing common, rare, bursty, phrase and out-of-vocabulary words, 1..9 words, some duplicated, some
    upper case, some with bytes >= 0x80; then the fixed edge queries"""
    rng = np.random.default_rng(seed)
    low = [w for w in voc if w == w.lower()]
    out = []
    for _ in range(nq):
        m = int(rng.integers(1, 10))
        ws = []
        for _ in range(m):
            r = rng.random()
            if r < 0.3:
                ws.append(low[min(int(rng.zipf(1.3)) - 1, len(low) - 1)])
            elif r < 0.55:
                ws.append(burst[int(rng.integers(0, len(burst)))])
            elif r < 0.75:
                ws.append(low[int(rng.integers(0, len(low)))])
            elif r < 0.85 and ph:
                ws.extend(ph[int(rng.integers(0, len(ph)))])
            elif r < 0.93:
                ws.append(bytes(rng.integers(97, 123, int(rng.integers(3, 9))).astype(np.uint8)))
            else:
                ws.append(voc[int(rng.integers(0, len(voc)))])
        if rng.random() < 0.2:
            ws.append(ws[0])
        out.append(b" ".join(ws))
    return out


def edge_queries(voc, burst):
    """all-OOV, uppercase, duplicate, non-ASCII and empty queries"""
    low = [w for w in voc if w == w.lower() and len(w) > 2]
    return [b"", b"  ,;!", b"qqzzxv wwkkyy", b"\xc3\xa9\xc3\xa8 \xff\xfe", burst[0].upper(), burst[1] + b" " + burst[1].upper(),
            burst[2] + b" " + burst[2] + b" " + burst[2], low[0] + b" " + low[0] + b" " + low[1] + b" " + low[0],
            low[3] + b"\xc3\xa9" + low[4] + b"\xff" + burst[3], burst[4] + b"_" + burst[5], b"burst7 Burst7 BURST7 burst7"]


def bucket_queries(X: B.Index, A: B.Index, pool, per: int = 3):
    """from a pool of queries, `per` of each: recipe Atire / SabSmooth / Cascade; avg_idf just below and above 3 among present-only
    queries; clarity just below and above 3 with avg_idf > 3; n_terms 3 and 4 with avg_idf in (4, 5] and just above 5"""
    R_ = A if A is not None else X
    fs = [(q, features(R_, q)) for q in pool]
    clean = [(q, f) for q, f in fs if f["n_terms"] and f["oov_rate"] == 0]
    picks = {
        "atire": [q for q, f in fs if choose(f) == ATIRE],
        "sab": [q for q, f in fs if choose(f) == SAB_SMOOTH and f["n_terms"]],
        "cascade": [q for q, f in fs if choose(f) == CASCADE],
        "idf_below_3": [q for q, f in clean if 2.5 <= f["avg_idf"] <= 3.0],
        "idf_above_3": [q for q, f in clean if 3.0 < f["avg_idf"] <= 3.5],
        "clarity_below_3": [q for q, f in clean if f["avg_idf"] > 3 and 2.5 <= f["simplified_clarity"] <= 3.0],
        "clarity_above_3": [q for q, f in clean if f["avg_idf"] > 3 and 3.0 < f["simplified_clarity"] <= 3.5],
        "terms3_idf5": [q for q, f in clean if f["n_terms"] == 3 and 4.0 < f["avg_idf"] <= 5.0],
        "terms4_idf5": [q for q, f in clean if f["n_terms"] == 4 and 4.0 < f["avg_idf"] <= 5.0],
        "terms4_idf_above5": [q for q, f in clean if f["n_terms"] == 4 and 5.0 < f["avg_idf"] <= 6.0],
    }
    out = []
    for k, qs in picks.items():
        out.extend(q for q in qs[:per] if q not in out)
    return out, {k: len(v) for k, v in picks.items()}


def pool(seed: int, n: int, i: int) -> np.ndarray:
    """query i's candidate pool: empty, or 1 .. n + 40 candidates -- documents (repeats included) and NOT_INDEXED ids"""
    rng = np.random.default_rng(seed * 7919 + i)
    if i % 7 == 3:
        return np.zeros(0, np.uint32)
    m = n + int(rng.integers(1, 41)) if i % 7 == 5 else int(rng.integers(1, n + 41))
    c = rng.integers(0, max(n, 1), m).astype(np.uint32) if n else np.full(m, NOT_INDEXED, np.uint32)
    c[rng.random(m) < 0.1] = NOT_INDEXED
    return c


# the stored answers' cases: name, seed, n, primary variant, router config overrides
CASES = [
    ("sab_default", 7, 600, B.SAB, {}),
    ("atire_primary", 7, 600, B.ATIRE, {}),
    ("sab_forced_atire", 9, 300, B.SAB, {"high_idf_threshold": -1.0, "atire_max_clarity": float("inf")}),
    ("sab_forced_cascade", 9, 300, B.SAB, {"high_idf_threshold": 1e30, "cascade_min_terms": 0, "cascade_max_idf": 1e30}),
    ("sab_strict_gates", 11, 400, B.SAB, {"oov_threshold": 0.5, "atire_min_terms": 3, "atire_min_idf_floor": 2.0,
                                          "atire_min_scq": 20.0, "atire_max_pool_jaccard": 0.5}),
]


def case_inputs(name, seed, n, variant, overrides):
    """(docs, queries, primary config, router config) of a stored case"""
    docs, voc, ph, burst = gen_router_corpus(seed, n)
    cfg = B.Config(variant=variant)
    X = B.Index(cfg, docs)
    A = B.Index(atire_of(cfg), docs) if atire_of(cfg) else None
    qs, _ = bucket_queries(X, A, gen_router_queries(seed + 1, voc, ph, burst, 3000))
    queries = qs + edge_queries(voc, burst) + gen_router_queries(seed + 2, voc, ph, burst, 8)
    return docs, queries, cfg, RCfg(**overrides)
