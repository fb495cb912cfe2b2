"""The word-bigram concept index (simeon's ConceptIndex) restated: concepts_restated.cpp, compiled on first use into a temporary
directory, drives the mining and the blend; the BM25 part of a blended score comes from tests/bm25_restated.py.  RefConcepts
drives the reference's own ConceptIndex through oracle/_ref/libref_concepts.so (oracle/concepts.mk), and gen_concept_corpus
makes the corpora with planted collocations that the stored answers, the CPU pin and the device tests share."""
import atexit
import ctypes as C
import functools
import os
import shutil
import subprocess
import tempfile

import numpy as np

from tests import bm25_restated as B

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
_REF_SO = os.path.join(ROOT, "oracle", "_ref", "libref_concepts.so")
p = C.c_void_p


class CCfg:
    """ConceptConfig: the lexical backend's (the defaults)"""

    def __init__(self, min_ttf=5, pmi_floor=2.0, max_concepts=200_000, k1=1.2, b=0.75):
        self.min_ttf, self.pmi_floor, self.max_concepts, self.k1, self.b = min_ttf, pmi_floor, max_concepts, k1, b

    def kw(self):
        return dict(min_ttf=self.min_ttf, pmi_floor=self.pmi_floor, max_concepts=self.max_concepts, k1=self.k1, b=self.b)


def _arr(texts):
    raw = [bytes(t) for t in texts]
    n = len(raw)
    return raw, (C.c_char_p * max(n, 1))(*raw), (C.c_size_t * max(n, 1))(*[len(r) for r in raw]), n


@functools.lru_cache(maxsize=None)
def _lib():
    tmp = tempfile.mkdtemp(prefix="concepts_restated_")
    atexit.register(shutil.rmtree, tmp, True)
    out = os.path.join(tmp, "libconcepts_restated.so")
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-Wall", "-Wextra",
                           os.path.join(HERE, "concepts_restated.cpp"), "-o", out])
    L = C.CDLL(out)
    L.cr_mine.restype = p
    L.cr_mine.argtypes = [C.c_uint64, p, p, C.c_size_t, C.c_uint32, C.c_float, C.c_uint32, C.c_float, C.c_float, p, p, C.c_size_t, C.c_int]
    L.cr_stats.argtypes = [p, p, p]
    L.cr_bigram_lengths.argtypes = [p, p]
    L.cr_accepted_pmi.argtypes = [p, p]
    L.cr_hashes.argtypes = [p, p]
    L.cr_find.restype = C.c_int64
    L.cr_find.argtypes = [p, C.c_uint64, p, p, p, p, p, C.c_size_t]
    L.cr_blend.argtypes = [p, C.c_char_p, C.c_size_t, C.c_float, p, C.c_size_t, C.c_int]
    L.cr_destroy.argtypes = [p]
    return L


class _Common:
    def hashes(self) -> np.ndarray:
        out = np.zeros(max(self.stats()["size"], 1), np.uint64)
        self._f("hashes")(self._h, out.ctypes.data)
        return out[:self.stats()["size"]]

    def bigram_lengths(self) -> np.ndarray:
        out = np.zeros(max(self.n, 1), np.uint32)
        self._f("bigram_lengths")(self._h, out.ctypes.data)
        return out[:self.n]

    def find(self, h: int):
        pmi, idf = C.c_float(), C.c_float()
        u = np.zeros(3, np.uint64)
        df = self._f("find")(self._h, h, C.byref(pmi), C.byref(idf), u.ctypes.data, None, None, 0)
        if df < 0:
            return None
        docs = np.zeros(max(df, 1), np.uint32)
        tfs = np.zeros(max(df, 1), np.uint32)
        self._f("find")(self._h, h, C.byref(pmi), C.byref(idf), u.ctypes.data, docs.ctypes.data, tfs.ctypes.data, df)
        return {"pmi": np.float32(pmi.value), "idf": np.float32(idf.value), "total_tf": int(u[0]), "a_hash": int(u[1]),
                "b_hash": int(u[2]), "docs": docs[:df], "tfs": tfs[:df]}


class Concepts(_Common):
    """The restated mining of `texts` against an index over `index_texts`; cap_mode 1 selects another tied subset at the cap."""

    def __init__(self, index_texts, texts, cfg: CCfg = CCfg(), seed: int = B.SEED, cap_mode: int = 0):
        L = _lib()
        self._keep = (_arr(index_texts), _arr(texts))
        (_, ip, il, ni), (_, cp, cl, n) = self._keep
        self.n = n
        self._h = L.cr_mine(seed, ip, il, ni, cfg.min_ttf, cfg.pmi_floor, cfg.max_concepts, cfg.k1, cfg.b, cp, cl, n, cap_mode)

    def _f(self, name):
        return getattr(_lib(), "cr_" + name)

    def stats(self) -> dict:
        f = C.c_float()
        u = np.zeros(7, np.uint64)
        _lib().cr_stats(self._h, C.byref(f), u.ctypes.data)
        return {"size": int(u[0]), "doc_count": int(u[1]), "avg_bigram_dl": np.float32(f.value), "sum_bigram_dl": int(u[2]),
                "distinct": int(u[3]), "passed_min_ttf": int(u[4]), "accepted": int(u[5]), "replayed": bool(u[6])}

    def accepted_pmi(self) -> np.ndarray:
        """the accepted PMIs before the cap, descending"""
        out = np.zeros(max(self.stats()["accepted"], 1), np.float32)
        _lib().cr_accepted_pmi(self._h, out.ctypes.data)
        return out[:self.stats()["accepted"]]

    def blend(self, query: bytes, scores, weight: float, sorted_order: bool = False) -> np.ndarray:
        out = np.array(scores, np.float32, copy=True)
        _lib().cr_blend(self._h, bytes(query), len(query), weight, out.ctypes.data, out.size, 1 if sorted_order else 0)
        return out

    def __del__(self):
        try:
            _lib().cr_destroy(self._h)
        except Exception:
            pass


def blended(X: B.Index, K: Concepts, query: bytes, weight: float) -> np.ndarray:
    """SimeonLexicalBackend's lexical score: Bm25Index::score, then ConceptIndex::blend_into"""
    return K.blend(query, X.score(query), weight)


# ---- the reference's own ConceptIndex (oracle/_ref/libref_concepts.so) ----
def have_ref() -> bool:
    return os.path.exists(_REF_SO)


@functools.lru_cache(maxsize=None)
def _refl():
    R = C.CDLL(_REF_SO)
    R.ref_concepts_build.restype = p
    R.ref_concepts_build.argtypes = [p, p, p, C.c_size_t, p, p, p, C.c_size_t]
    R.ref_concepts_stats.argtypes = [p, p, p]
    R.ref_concepts_bigram_lengths.argtypes = [p, p]
    R.ref_concepts_hashes.argtypes = [p, p]
    R.ref_concepts_find.restype = C.c_int64
    R.ref_concepts_find.argtypes = [p, C.c_uint64, p, p, p, p, p, C.c_size_t]
    R.ref_concepts_blend.argtypes = [p, C.c_char_p, C.c_size_t, C.c_float, p, C.c_size_t]
    R.ref_concepts_score_blended.argtypes = [p, C.c_char_p, C.c_size_t, C.c_float, p]
    R.ref_concepts_mine_ms.restype = C.c_double
    R.ref_concepts_mine_ms.argtypes = [p]
    R.ref_concepts_destroy.argtypes = [p]
    return R


class _RefCCfg(C.Structure):
    _fields_ = [("min_ttf", C.c_uint32), ("pmi_floor", C.c_float), ("max_concepts", C.c_uint32), ("k1", C.c_float), ("b", C.c_float)]


class RefConcepts(_Common):
    """simeon's Bm25Index over index_texts and mine_concepts(index, texts, cfg)"""

    def __init__(self, bcfg: B.Config, index_texts, texts, cfg: CCfg = CCfg()):
        R = _refl()
        c = B._Cfg(bcfg.k1, bcfg.b, bcfg.delta, bcfg.gamma, bcfg.variant, bcfg.ngram_min, bcfg.ngram_max, bcfg.prune_ratio, bcfg.hash_seed)
        cc = _RefCCfg(cfg.min_ttf, cfg.pmi_floor, cfg.max_concepts, cfg.k1, cfg.b)
        self._keep = (_arr(index_texts), _arr(texts))
        (_, ip, il, ni), (_, cp, cl, n) = self._keep
        self.n = n
        self.n_index = ni
        self._h = R.ref_concepts_build(C.byref(c), ip, il, ni, C.byref(cc), cp, cl, n)

    def _f(self, name):
        return getattr(_refl(), "ref_concepts_" + name)

    def stats(self) -> dict:
        f = np.zeros(1, np.float32)
        u = np.zeros(3, np.uint64)
        _refl().ref_concepts_stats(self._h, f.ctypes.data, u.ctypes.data)
        return {"size": int(u[0]), "doc_count": int(u[1]), "avg_bigram_dl": f[0], "sum_bigram_dl": int(u[2])}

    def blend(self, query: bytes, scores, weight: float) -> np.ndarray:
        out = np.array(scores, np.float32, copy=True)
        _refl().ref_concepts_blend(self._h, bytes(query), len(query), weight, out.ctypes.data, out.size)
        return out

    def mine_ms(self) -> float:
        """the wall time of mine_concepts alone"""
        return _refl().ref_concepts_mine_ms(self._h)

    def score_blended(self, query: bytes, weight: float) -> np.ndarray:
        out = np.zeros(self.n_index, np.float32)
        _refl().ref_concepts_score_blended(self._h, bytes(query), len(query), weight, out.ctypes.data)
        return out

    def __del__(self):
        try:
            _refl().ref_concepts_destroy(self._h)
        except Exception:
            pass


# ---- corpora with planted collocations ----
def gen_concept_corpus(seed: int, n: int, mean_words: int = 30, vocab: int = 1500, phrases: int = 40, tie_groups: int = 0):
    """B.gen_corpus documents with planted two-word phrases of lowercase vocabulary words (about half the documents get one or
    more), some planted in upper case; tie_groups > 0 also plants that many pairs of words of their own, each pair in exactly 6
    documents, so that their PMIs are equal.  -> (docs, vocabulary, phrases)"""
    docs, voc = B.gen_corpus(seed, n, mean_words, vocab)
    rng = np.random.default_rng(seed + 7)
    low = [w for w in voc if w == w.lower() and w[:1].isalpha()]
    ph = [(low[int(rng.integers(0, len(low)))], low[int(rng.integers(0, len(low)))]) for _ in range(phrases)] if low and n else []
    out = []
    for d in docs:
        parts = [d]
        while ph and rng.random() < 0.5:
            a, b = ph[min(int(rng.zipf(1.5)) - 1, len(ph) - 1)]
            t = a + b" " + b
            parts.append(b" " + (t.upper() if rng.random() < 0.05 else t) + b" ")
        out.append(b"".join(parts))
    for g in range(tie_groups if n >= 6 else 0):
        a, b = b"tiea%d" % g, b"tieb%d" % g
        for j in rng.choice(n, 6, replace=False):
            out[int(j)] += b" " + a + b" " + b
    return out, voc, ph


def gen_concept_queries(seed: int, voc, ph, nq: int):
    """Queries of B.gen_queries, planted phrases (alone, repeated, within other words, upper case), and one-word queries"""
    rng = np.random.default_rng(seed)
    out = B.gen_queries(seed, voc, nq // 2)
    for _ in range(nq - len(out)):
        if not ph:
            out.append(b"x y")
            continue
        a, b = ph[int(rng.integers(0, len(ph)))]
        c, d = ph[int(rng.integers(0, len(ph)))]
        r = rng.random()
        if r < 0.3:
            out.append(a + b" " + b + b" " + c + b" " + d)
        elif r < 0.5:
            out.append(a + b" " + b + b" " + a + b" " + b + b" " + a)
        elif r < 0.6:
            out.append((a + b" " + b).upper())
        elif r < 0.7:
            out.append(a)
        else:
            out.append(voc[int(rng.integers(0, len(voc)))] + b" " + a + b" " + b + b", " + c + b" " + d + b" tiea0 tieb0")
    return out


# ---- the configuration grid the CPU pin and the device tests share ----
FLOORS = (-1e30, 0.0, 2.0, 1e30)
CAPS = ("0", "1", "tie", "loose")
WEIGHTS = (0.0, 0.5, 1.0, -0.5)
GRID = [(n, B.SAB if i % 2 == 0 else B.ATIRE, (1, 5)[i % 2 == (n % 2)], FLOORS[i % 4], CAPS[(i + n) % 4], WEIGHTS[(i // 2 + n) % 4])
        for n in (0, 1, 2, 99, 100, 1000) for i in range(10)]


def tie_cap(pmis) -> int:
    """a max_concepts at which equal PMIs straddle the cut (0 when none exists)"""
    for c in range(1, len(pmis)):
        if pmis[c - 1] == pmis[c]:
            return c
    return 0


def grid_case(n, variant, min_ttf, floor, cap):
    """(docs, queries, CCfg) of one grid point; the corpus is mixed case with planted phrases and tied pairs"""
    docs, voc, ph = gen_concept_corpus(500 + n, n, 25, 1200, 30, 8)
    queries = gen_concept_queries(600 + n, voc, ph, 16) + [b"", b"one", b"tiea0 tieb0 tiea0 tieb0", b"TIEA0 tieb0"]
    cfg = CCfg(min_ttf=min_ttf, pmi_floor=floor)
    if cap in ("0", "1"):
        cfg.max_concepts = int(cap)
    else:
        pm = Concepts(docs, docs, cfg).accepted_pmi()
        cfg.max_concepts = (tie_cap(pm) or max(len(pm) // 2, 1)) if cap == "tie" else len(pm) + 10
    return docs, queries, cfg
