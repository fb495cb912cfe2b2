"""A restatement of the lead-text field and the two BM25F strategies of simeon's lexical backend's strategy router, over
bm25_restated.py and concepts_restated.py:

- lead(text, L): extract_lead_tokens (third_party/simeon/src/corpus_adapter.cpp:16-39), the bytes up to the whitespace byte
  (C-locale isspace) that ends the L-th whitespace-delimited token, whitespace turned into ' ', trailing spaces trimmed.
- Index(cfg, texts, L): Bm25Index with add_doc(text, lead(text, L)) (bm25.cpp:563-656).  The aux field is active from the first
  non-empty lead text on, earlier documents back-filled with length 0, so it exists for every document or for none; its words
  and n-grams are those of the lead texts, with their own lengths, averages and pruning, and the idf of the same document count.
- bm25f(body_query, aux_query, wb, wa) (Bm25Index::score_bm25f, bm25.cpp:978-1144): the body score; times wb when wb != 1; then
  the aux legs: SubwordAwareBackoff adds fl(wa * alpha) * bm25plus over aux words and fl(wa * (1 - alpha)) * bm25plus over their
  aux n-grams, alpha from the AUX df; Atire adds wa * score_atire.
- score(pool, query): pool 0, Bm25Strategy with the query's lead text as evidence (bm25f(q, lead(q, 64), 0.85, 0.15), plain
  score when that lead text is empty); pool 1, KeyphraseStrategy(0.25, 0.30) (retrieval_strategy.cpp:192-252); pool 2,
  LeadFieldStrategy (bm25f(q, q, 0.85, 0.15)); ROUTED, the backend's entropy profile (simeon_lexical_backend.cpp:998-1048)
  and EntropyRouter::route over the three.
- keyphrase: the plain score; the normalised softmax entropy of simeon::top_k(scores, 10), which keeps zero scores (the
  positives by score descending, then the lowest-index zeros); below 0.30 or without keyphrases the plain score, else the
  z-score (two sequential double sums: np.cumsum over float64 is sequential, np.sum is pairwise) plus
  fl(lam * 0.25) * (matches / keyphrases), a document matching a keyphrase when its single-term score is > 0.

RefStrategy drives the reference's own build and strategies through oracle/_ref/libref_strategy.so (oracle/strategy.mk)."""
from __future__ import annotations

import ctypes as C
import math
import os
import re

import numpy as np

from tests import bm25_restated as B
from tests import concepts_restated as R

f32 = np.float32
LEAD = 64                       # the backend's lead length (TextAdapter, extract_lead_tokens(text, 64))
WB, WA = f32(0.85), f32(0.15)   # the backend's body and aux weights for both strategies
POOL_BM25, POOL_KEYPHRASE, POOL_LEAD_FIELD, ROUTED = 0, 1, 2, 3
STOPWORDS = set(b"a an the and or but in on at to for of with by from is are was were be been being have has had do does did will would "
                b"could should may might can shall this that these those it its they them we us he she his her their our my your not no "
                b"nor so as if than then also very just about into over after before between under during without".split())
_libm = C.CDLL("libm.so.6")
_libm.expf.restype = C.c_float
_libm.expf.argtypes = [C.c_float]
_libm.log.restype = C.c_double
_libm.log.argtypes = [C.c_double]
_libm.exp.restype = C.c_double
_libm.exp.argtypes = [C.c_double]
SPACE = b" \t\n\v\f\r"          # isspace in the C locale


def lead_cut(text: bytes, L: int) -> int:
    """The end of the lead prefix: the index of the whitespace byte that ends the L-th token, else len(text)."""
    tokens, in_token = 0, False
    for i, c in enumerate(text):
        if c in SPACE:
            if in_token:
                tokens += 1
                in_token = False
            if tokens >= L:
                return i
        else:
            in_token = True
    return len(text)


def lead(text: bytes, L: int) -> bytes:
    return bytes(32 if c in SPACE else c for c in text[:lead_cut(text, L)]).rstrip(b" ")


class Index(B.Index):
    def __init__(self, cfg: B.Config, texts, L: int = LEAD):
        super().__init__(cfg, texts)
        leads = [lead(bytes(t), L) if L else b"" for t in texts]
        self.aux_active = any(leads)
        A = B.Index(cfg, leads)   # the same n: the same idf table and df limit; lengths 0 before activation are the same
        self.aux_words = A.words
        self.aux_ngrams = A.ngrams
        if not self.aux_active:   # no aux field: no lengths, averages 0
            self.aux_words = B.Field(np.zeros(0, np.uint32))
            self.aux_ngrams = B.Field(np.zeros(0, np.uint32))

    def field(self, f: int) -> B.Field:
        return (self.words, self.ngrams, self.aux_words, self.aux_ngrams)[f]

    def doc_lengths(self, f: int) -> np.ndarray:
        out = np.zeros(self.n, np.uint32)
        L = self.field(f).lengths
        out[:len(L)] = L
        return out

    def bm25f(self, body_query: bytes, aux_query: bytes, wb=WB, wa=WA, scale_after_aux: bool = False) -> np.ndarray:
        """score_bm25f; scale_after_aux moves the body scale after the aux legs (a deliberate mistake the tests must catch)"""
        wb, wa = f32(wb), f32(wa)
        if wb == 1 and wa == 0:
            return self.score(body_query)
        out = self.score(body_query) if wb != 0 else np.zeros(self.n, np.float32)
        if wb != 1 and not scale_after_aux:
            out = out * wb
        if wa != 0 and (self.aux_words.postings or (self.cfg.variant == B.SAB and self.aux_ngrams.postings)):
            with np.errstate(all="ignore"):
                for fld, w, h in self._aux_legs(aux_query):
                    F = self.aux_words if fld == 0 else self.aux_ngrams
                    docs, tfs, idf, _ = F.postings[h]
                    avg = F.avg if F.avg > 0 else f32(1.0)
                    tf = tfs.astype(np.float32)
                    dl = F.lengths[docs].astype(np.float32)
                    if w is None:
                        out[docs] = out[docs] + wa * self._atire(tf, dl, idf, avg)
                    else:
                        out[docs] = out[docs] + (wa * w) * self._bm25_plus(tf, dl, idf, avg)
        if wb != 1 and scale_after_aux:
            out = out * wb
        return out

    def _aux_legs(self, query: bytes):
        """Index.legs over the aux fields: alpha from the aux df"""
        saved = self.words, self.ngrams
        self.words, self.ngrams = self.aux_words, self.aux_ngrams
        try:
            return self.legs(query)
        finally:
            self.words, self.ngrams = saved

    def presence(self, word: bytes) -> np.ndarray:
        """score_weighted_hashes({hash_term(word), 1}) > 0 per document"""
        out = np.zeros(self.n, bool)
        p = self.words.postings.get(self.h(word))
        if p is not None:
            docs, tfs, idf, _ = p
            avg = self.words.avg if self.words.avg > 0 else f32(1.0)
            tf, dl = tfs.astype(np.float32), self.words.lengths[docs].astype(np.float32)
            with np.errstate(all="ignore"):
                v = self._bm25_plus(tf, dl, idf, avg) if self.cfg.variant == B.SAB else self._atire(tf, dl, idf, avg)
            out[docs] = (f32(1.0) * v) > 0
        return out

    def keyphrase(self, query: bytes, pad: bool = True, pairwise: bool = False) -> np.ndarray:
        """KeyphraseStrategy(0.25, 0.30); pad=False drops top_k's zeros and pairwise=True sums with np.sum (deliberate mistakes
        the tests must catch)"""
        s = self.score(query)
        ent = keyphrase_entropy(s, pad)
        kps = keyphrases(query)
        if ent < f32(0.30) or not kps:
            return s
        count = np.zeros(self.n, np.uint32)
        for kp in kps:
            count += self.presence(kp)
        x = s.astype(np.float64)
        mean, var = zscore_sums(s, pairwise)
        sd = f32(math.sqrt(var / float(self.n)) + 1e-12)
        z = ((x - mean) / float(sd)).astype(np.float32)
        lam = f32(1.0) / (f32(1.0) + f32(_libm.expf(C.c_float(float(-(ent - f32(0.48)) * f32(8.0))))))
        with np.errstate(all="ignore"):
            return z + (lam * f32(0.25)) * (count.astype(np.float32) / f32(len(kps)))

    def strategy(self, pool: int, query: bytes, **kw) -> np.ndarray:
        if pool == ROUTED:
            return self.strategy(route(self.score(query)), query, **kw)
        if pool == POOL_KEYPHRASE:
            return self.keyphrase(query, **kw)
        if pool == POOL_BM25:
            aux = lead(bytes(query), LEAD)
            return self.bm25f(query, aux, **kw) if aux else self.score(query)
        if pool == POOL_LEAD_FIELD:
            return self.bm25f(query, query, **kw)
        raise ValueError(pool)


def keyphrases(query: bytes):
    """extract_keyphrases: alphabetic runs (C locale) of length >= 2, lowercased, stopwords dropped, sorted, de-duplicated"""
    ws = [m.group(0).lower() for m in re.finditer(rb"[A-Za-z]+", bytes(query))]
    return sorted({w for w in ws if len(w) >= 2 and w not in STOPWORDS})


def zscore_sums(s: np.ndarray, pairwise: bool = False):
    """zscore_inplace's mean and sum of squared deviations: two sequential double sums in document order (np.cumsum); pairwise
    sums them as np.sum does"""
    x = s.astype(np.float64)
    total = (lambda v: np.sum(v)) if pairwise else (lambda v: np.cumsum(v)[-1])
    mean = total(x) / float(len(x))
    return mean, total((x - mean) * (x - mean))


def keyphrase_entropy(s: np.ndarray, pad: bool = True) -> np.float32:
    """the normalised softmax entropy of simeon::top_k(s, 10), in its order, in double"""
    k = min(10, len(s))
    _, vals = B.topk(s, k)
    vals = [float(v) for v in vals] + ([0.0] * (k - len(vals)) if pad else [])
    ent = 0.0
    if len(vals) >= 2:
        sum_exp = 0.0
        for v in vals:
            sum_exp += _libm.exp(v)
        for v in vals:
            p = _libm.exp(v) / sum_exp
            if p > 1e-12:
                ent -= p * _libm.log(p)
        ent /= _libm.log(float(len(vals)))
    return f32(ent)


def route_entropy(s: np.ndarray) -> np.float32:
    """the backend's profile: mean over positive scores, in document order, of sn * -log(sn), sn = float(s / max)"""
    top = s.max() if len(s) else f32(0)
    if not top > 0:
        return f32(0)
    pos = s[s > 0]
    sn = (pos / top).astype(np.float32).astype(np.float64)
    terms = np.array([v * -_libm.log(v) if v > 0 else 0.0 for v in sn])
    return f32(np.cumsum(terms)[-1] / float(len(pos)))


def route(s: np.ndarray) -> int:
    e = route_entropy(s)
    return POOL_BM25 if e < f32(0.05) else POOL_LEAD_FIELD if e > f32(0.50) else POOL_KEYPHRASE


def score(X: Index, pool: int, query: bytes, K: R.Concepts | None = None, weight: float = 0.5, **kw) -> np.ndarray:
    """the backend's strategy score, then blend_into(query, scores, weight) with a concept index"""
    s = X.strategy(pool, query, **kw)
    return K.blend(query, s, weight) if K is not None else s


# ---- the reference's own build and strategies (oracle/_ref/libref_strategy.so) ----
_REF_SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libref_strategy.so")
_ref = None


def have_ref() -> bool:
    return os.path.exists(_REF_SO)


def _refl():
    global _ref
    if _ref is None:
        L = C.CDLL(_REF_SO)
        L.ref_strategy_lead.restype = C.c_size_t
        L.ref_strategy_lead.argtypes = [C.c_char_p, C.c_size_t, C.c_uint32, C.c_char_p]
        L.ref_strategy_build.restype = C.c_void_p
        L.ref_strategy_build.argtypes = [C.POINTER(B._Cfg), C.POINTER(C.c_char_p), C.POINTER(C.c_size_t), C.c_size_t, C.c_uint32]
        L.ref_strategy_destroy.argtypes = [C.c_void_p]
        L.ref_strategy_concepts.restype = C.c_void_p
        L.ref_strategy_concepts.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_char_p), C.POINTER(C.c_size_t), C.c_size_t]
        L.ref_strategy_concepts_destroy.argtypes = [C.c_void_p]
        L.ref_strategy_score.restype = C.c_int
        L.ref_strategy_score.argtypes = [C.c_void_p, C.c_int, C.c_char_p, C.c_size_t, C.c_void_p, C.c_float, C.c_void_p]
        L.ref_strategy_field_stats.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        L.ref_strategy_postings.restype = C.c_uint32
        L.ref_strategy_postings.argtypes = [C.c_void_p, C.c_int, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
        L.ref_strategy_doc_lengths.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        _ref = L
    return _ref


def ref_lead(text: bytes, L: int) -> bytes:
    buf = C.create_string_buffer(max(len(text), 1))
    m = _refl().ref_strategy_lead(bytes(text), len(text), L, buf)
    return buf.raw[:m]


class RefStrategy:
    """simeon's Bm25Index built with lead-text aux fields, its Bm25Strategy and LeadFieldStrategy, and optionally its
    ConceptIndex mined against it (min_ttf etc. from `ccfg`) over the same texts."""

    def __init__(self, cfg: B.Config, texts, L: int = LEAD, ccfg: R.CCfg | None = None):
        raw = [bytes(t) for t in texts]
        self._keep = raw
        self.n = len(raw)
        ptrs = (C.c_char_p * max(self.n, 1))(*raw)
        lens = (C.c_size_t * max(self.n, 1))(*[len(r) for r in raw])
        c = B._Cfg(cfg.k1, cfg.b, cfg.delta, cfg.gamma, cfg.variant, cfg.ngram_min, cfg.ngram_max, cfg.prune_ratio, cfg.hash_seed)
        self._h = _refl().ref_strategy_build(C.byref(c), ptrs, lens, self.n, L)
        self._c = None
        if ccfg is not None:
            cc = R._RefCCfg(ccfg.min_ttf, ccfg.pmi_floor, ccfg.max_concepts, ccfg.k1, ccfg.b)
            self._c = _refl().ref_strategy_concepts(self._h, C.byref(cc), ptrs, lens, self.n)

    def score(self, pool: int, query: bytes, weight: float | None = None, chosen: bool = False):
        out = np.zeros(self.n, np.float32)
        c = _refl().ref_strategy_score(self._h, pool, bytes(query), len(query), self._c if weight is not None else None,
                                       0.0 if weight is None else weight, out.ctypes.data)
        return (out, c) if chosen else out

    def field_stats(self, f: int) -> dict:
        a = np.zeros(1, np.float32)
        u = np.zeros(4, np.uint64)
        _refl().ref_strategy_field_stats(self._h, f, a.ctypes.data, u.ctypes.data)
        return {"docs": int(u[0]), "avg": a[0], "sum": int(u[1]), "terms": int(u[2]), "postings": int(u[3])}

    def postings(self, f: int, h: int):
        idf, ttf = C.c_float(), C.c_uint64()
        df = _refl().ref_strategy_postings(self._h, f, h, C.byref(idf), C.byref(ttf), None, None, 0)
        docs, tfs = np.zeros(df, np.uint32), np.zeros(df, np.uint32)
        if df:
            _refl().ref_strategy_postings(self._h, f, h, C.byref(idf), C.byref(ttf), docs.ctypes.data, tfs.ctypes.data, df)
        return docs, tfs, f32(idf.value), int(ttf.value)

    def doc_lengths(self, f: int) -> np.ndarray:
        out = np.zeros(self.n, np.uint32)
        _refl().ref_strategy_doc_lengths(self._h, f, out.ctypes.data)
        return out

    def close(self):
        if self._c:
            _refl().ref_strategy_concepts_destroy(self._c)
            self._c = None
        if self._h:
            _refl().ref_strategy_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ---- generated corpora and queries ----
WS = [b" ", b"\t", b"\n", b"\v", b"\f", b"\r", b"  ", b" \n\t"]


def gen_lead_corpus(seed: int, n: int, vocab: int = 800):
    """Documents of 0..150 tokens (shorter and longer than 64), separated by every isspace byte and by runs of them, with
    punctuation-only tokens, bytes >= 0x80, leading and trailing whitespace, empty and whitespace-only documents."""
    rng = np.random.default_rng(seed)
    voc = B.zipf_vocab(rng, vocab) + [b"--", b"\xc3\xa9t\xc3\xa9", b"a.b", b"x\x00y", b"!!"]
    docs = []
    for _ in range(n):
        r = rng.random()
        if r < 0.03:
            docs.append(b"")
            continue
        if r < 0.06:
            docs.append(b"".join(WS[int(i)] for i in rng.integers(0, len(WS), int(rng.integers(1, 5)))))
            continue
        m = int(rng.integers(1, 40)) if rng.random() < 0.5 else int(rng.integers(55, 150))
        ids = np.minimum(rng.zipf(1.3, m) - 1, len(voc) - 1)
        parts = [WS[int(rng.integers(0, len(WS)))]] if rng.random() < 0.2 else []
        for i in ids:
            parts.append(voc[i])
            parts.append(WS[int(rng.integers(0, len(WS)))] if rng.random() < 0.9 else b" ,")
        docs.append(b"".join(parts))
    return docs, voc


def gen_lead_queries(seed: int, voc, nq: int):
    """Queries of 0..8 words, plus one longer than 64 tokens (its lead text differs from the query) and whitespace-only ones."""
    rng = np.random.default_rng(seed)
    out = B.gen_queries(seed, voc, max(nq - 3, 0))
    out.append(b"\t".join(voc[min(int(rng.zipf(1.3)) - 1, len(voc) - 1)] for _ in range(80)))
    out.append(b" \n ")
    out.append(voc[0] + b"\v" + voc[1] + b"\r\n")
    return out[:nq] if nq < 3 else out
