"""A restatement of simeon's Bm25Index (third_party/simeon/src/bm25.cpp) for the two variants the lexical backend selects:
Atire (0) and SubwordAwareBackoff (7).  Build = add_doc for each document, then finalize(); score = Bm25Index::score.

Every float is float32 and every operation is the reference's, in its order and without fused multiply-adds (bm25.cpp is
built without -mfma).  IDF is logf of a float expression, taken from the C library like std::log(float).  The tests pin this
restatement to the stored answers of the reference build (tests/golden/ref_bm25.json) and, where oracle/_ref exists, to
that build itself; the device is then checked against it at any configuration.

RefIndex below drives the reference's own index through oracle/_ref/libref_bm25.so (oracle/bm25.mk)."""
from __future__ import annotations

import ctypes as C
import os
import re
from dataclasses import dataclass, field

import numpy as np

ATIRE, SAB = 0, 7
SEED = 0xB252B252B252B252
M64 = (1 << 64) - 1
f32 = np.float32

_libm = C.CDLL("libm.so.6")
_libm.logf.restype = C.c_float
_libm.logf.argtypes = [C.c_float]


def logf(x) -> np.float32:
    return f32(_libm.logf(C.c_float(float(x))))


@dataclass
class Config:
    k1: float = 1.2
    b: float = 0.75
    delta: float = 1.0
    gamma: float = 5.0
    variant: int = SAB
    ngram_min: int = 3
    ngram_max: int = 4
    prune_ratio: float = 0.5
    hash_seed: int = SEED


def _mix(z: int) -> int:
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def hash64(s: bytes, seed: int = SEED) -> int:
    """splitmix64_hash (simeon src/hasher.cpp:33-47)."""
    h = _mix(seed ^ 0x9E3779B97F4A7C15)
    n = len(s)
    i = 0
    while i + 8 <= n:
        h = _mix(h ^ int.from_bytes(s[i:i + 8], "little"))
        i += 8
    if i < n:
        h = _mix(h ^ int.from_bytes(s[i:], "little") ^ ((n - i) << 56))
    return _mix(h ^ n)


_WORD = re.compile(rb"[A-Za-z0-9_]+")   # isalnum || '_' in the C locale: bytes >= 0x80 separate words


def words(text: bytes):
    """The lowercased words of text in order (collect_field_term_stats / emit_word_tokens + ascii_fold)."""
    return [m.group(0).lower() for m in _WORD.finditer(text)]


def ngrams(word: bytes, kmin: int, kmax: int):
    """Every n-gram of the word: k ascending, then position ascending (bm25.cpp:136-147, tokenizer.cpp:25-38)."""
    out = []
    n = len(word)
    k = kmin
    while k <= kmax and n >= k:
        out.extend(word[p:p + k] for p in range(n - k + 1))
        k += 1
    return out


@dataclass
class Field:
    lengths: np.ndarray = None                       # uint32 per document
    avg: np.float32 = f32(0)
    postings: dict = field(default_factory=dict)     # hash -> (docs uint32, tfs uint32, idf float32, total_tf int)
    pruned: int = 0


class Index:
    def __init__(self, cfg: Config, texts):
        self.cfg = cfg
        self._hash = {}
        self._grams = {}
        sab = cfg.variant == SAB
        n = len(texts)
        self.n = n
        wl = np.zeros(n, np.uint32)
        gl = np.zeros(n, np.uint32)
        wpost, gpost = {}, {}
        for d, t in enumerate(texts):
            tf, gtf = {}, {}
            ws = words(bytes(t))
            wl[d] = len(ws)
            for w in ws:
                h = self.h(w)
                tf[h] = tf.get(h, 0) + 1
                if sab:
                    gs = self.gram_hashes(w)
                    gl[d] += len(gs)
                    for g in gs:
                        gtf[g] = gtf.get(g, 0) + 1
            for h, c in tf.items():
                wpost.setdefault(h, []).append((d, c))
            for h, c in gtf.items():
                gpost.setdefault(h, []).append((d, c))
        self.words = self._finalize(wl, wpost, prune=False)
        self.ngrams = self._finalize(gl, gpost, prune=True) if sab else Field(np.zeros(0, np.uint32))
        self.total_tokens = int(wl.astype(np.uint64).sum())

    def h(self, w: bytes) -> int:
        v = self._hash.get(w)
        if v is None:
            v = self._hash[w] = hash64(w, self.cfg.hash_seed)
        return v

    def gram_hashes(self, w: bytes):
        v = self._grams.get(w)
        if v is None:
            v = self._grams[w] = [hash64(g, self.cfg.hash_seed) for g in ngrams(w, self.cfg.ngram_min, self.cfg.ngram_max)]
        return v

    def idf(self, df: int) -> np.float32:
        nf, dff = f32(self.n), f32(df)
        return logf((nf - dff + f32(0.5)) / (dff + f32(0.5)) + f32(1.0))

    def _finalize(self, lengths, post, prune):
        n = self.n
        F = Field(lengths)
        F.avg = f32(0) if n == 0 else f32(float(int(lengths.astype(np.uint64).sum())) / float(n))
        if prune and float(f32(self.cfg.prune_ratio)) > 0 and n > 0:
            df_max = int(float(f32(self.cfg.prune_ratio)) * float(n))
            keep = {h: v for h, v in post.items() if len(v) <= df_max}
            F.pruned = len(post) - len(keep)
            post = keep
        for h, v in post.items():
            a = np.array(v, dtype=np.uint32).reshape(-1, 2)
            F.postings[h] = (a[:, 0].copy(), a[:, 1].copy(), self.idf(len(v)), int(a[:, 1].astype(np.uint64).sum()))
        return F

    # per-(term, doc) contributions (bm25.cpp:163-188), vectorised over a posting list in float32
    def _bm25_plus(self, tf, dl, idf, avg):
        c = self.cfg
        k1, b, delta = f32(c.k1), f32(c.b), f32(c.delta)
        denom = tf + k1 * ((f32(1.0) - b) + (b * dl) / avg)
        return idf * ((tf * (k1 + f32(1.0))) / denom + delta)

    def _atire(self, tf, dl, idf, avg):
        c = self.cfg
        k1, b = f32(c.k1), f32(c.b)
        denom = tf + k1 * ((f32(1.0) - b) + (b * dl) / avg)
        return ((idf * tf) * (k1 + f32(1.0))) / denom

    def legs(self, query: bytes):
        """The query's ordered additions: (field, weight, posting hash), weight None for Atire."""
        out = []
        terms = words(bytes(query))
        if self.cfg.variant != SAB:
            return [(0, None, self.h(t)) for t in terms if self.h(t) in self.words.postings]
        gamma = f32(self.cfg.gamma)
        for t in terms:
            h = self.h(t)
            p = self.words.postings.get(h)
            df = 0 if p is None else len(p[0])
            alpha = f32(df) / (f32(df) + gamma) if df > 0 else f32(0)
            if alpha > 0:
                out.append((0, alpha, h))
            if alpha < 1:
                seen = list(dict.fromkeys(self.gram_hashes(t)))   # first occurrence of each hash, in emission order
                w = f32(1.0) - alpha
                out.extend((1, w, g) for g in seen if g in self.ngrams.postings)
        return out

    def score(self, query: bytes) -> np.ndarray:
        with np.errstate(all="ignore"):
            out = np.zeros(self.n, np.float32)
            for fld, w, h in self.legs(query):
                F = self.words if fld == 0 else self.ngrams
                docs, tfs, idf, _ = F.postings[h]
                avg = F.avg if F.avg > 0 else f32(1.0)
                tf = tfs.astype(np.float32)
                dl = F.lengths[docs].astype(np.float32)
                if w is None:
                    out[docs] = out[docs] + self._atire(tf, dl, idf, avg)
                else:
                    out[docs] = out[docs] + w * self._bm25_plus(tf, dl, idf, avg)
            return out

    def stats(self) -> dict:
        return {"n_docs": self.n, "avg_dl": self.words.avg, "ngram_avg_dl": self.ngrams.avg, "total_tokens": self.total_tokens,
                "terms": (len(self.words.postings), len(self.ngrams.postings)),
                "postings": tuple(sum(len(v[0]) for v in F.postings.values()) for F in (self.words, self.ngrams)),
                "pruned": self.ngrams.pruned}


def topk(scores: np.ndarray, k: int):
    """The fused top-k: documents of score > 0, by score descending, then document ascending."""
    pos = np.flatnonzero(scores > 0)
    order = np.lexsort((pos, -scores[pos].astype(np.float64)))
    sel = pos[order][:k]
    return sel.astype(np.uint32), scores[sel]


# ---- the reference's own index (oracle/_ref/libref_bm25.so) ----
_REF_SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libref_bm25.so")


class _Cfg(C.Structure):
    _fields_ = [("k1", C.c_float), ("b", C.c_float), ("delta", C.c_float), ("gamma", C.c_float), ("variant", C.c_uint32),
                ("ngram_min", C.c_uint32), ("ngram_max", C.c_uint32), ("prune_ratio", C.c_float), ("hash_seed", C.c_uint64)]


_ref = None


def have_ref() -> bool:
    return os.path.exists(_REF_SO)


def _refl():
    global _ref
    if _ref is None:
        R = C.CDLL(_REF_SO)
        R.ref_bm25_build.restype = C.c_void_p
        R.ref_bm25_build.argtypes = [C.POINTER(_Cfg), C.POINTER(C.c_char_p), C.POINTER(C.c_size_t), C.c_size_t]
        R.ref_bm25_score.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.c_void_p]
        R.ref_bm25_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        R.ref_bm25_postings.restype = C.c_uint32
        R.ref_bm25_postings.argtypes = [C.c_void_p, C.c_int, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
        R.ref_bm25_doc_lengths.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        R.ref_bm25_term.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
        R.ref_bm25_hash.restype = C.c_uint64
        R.ref_bm25_hash.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
        R.ref_bm25_destroy.argtypes = [C.c_void_p]
        _ref = R
    return _ref


class RefIndex:
    """simeon::Bm25Index itself, built and finalized over texts."""

    def __init__(self, cfg: Config, texts):
        R = _refl()
        c = _Cfg(cfg.k1, cfg.b, cfg.delta, cfg.gamma, cfg.variant, cfg.ngram_min, cfg.ngram_max, cfg.prune_ratio, cfg.hash_seed)
        raw = [bytes(t) for t in texts]
        n = len(raw)
        self._keep = raw
        self.n = n
        ptrs = (C.c_char_p * max(n, 1))(*raw)
        lens = (C.c_size_t * max(n, 1))(*[len(r) for r in raw])
        self._h = R.ref_bm25_build(C.byref(c), ptrs, lens, n)

    def score(self, query: bytes) -> np.ndarray:
        out = np.zeros(self.n, np.float32)
        _refl().ref_bm25_score(self._h, bytes(query), len(query), out.ctypes.data)
        return out

    def stats(self) -> dict:
        f = np.zeros(2, np.float32)
        u = np.zeros(6, np.uint64)
        _refl().ref_bm25_stats(self._h, f.ctypes.data, u.ctypes.data)
        return {"n_docs": int(u[0]), "avg_dl": f[0], "ngram_avg_dl": f[1], "total_tokens": int(u[1]),
                "terms": (int(u[2]), int(u[3])), "postings": (int(u[4]), int(u[5]))}

    def postings(self, fld: int, h: int):
        idf = C.c_float()
        ttf = C.c_uint64()
        df = _refl().ref_bm25_postings(self._h, fld, h, C.byref(idf), C.byref(ttf), None, None, 0)
        docs = np.zeros(df, np.uint32)
        tfs = np.zeros(df, np.uint32)
        if df:
            _refl().ref_bm25_postings(self._h, fld, h, C.byref(idf), C.byref(ttf), docs.ctypes.data, tfs.ctypes.data, df)
        return docs, tfs, f32(idf.value), int(ttf.value)

    def doc_lengths(self, fld: int) -> np.ndarray:
        out = np.zeros(self.n, np.uint32)
        _refl().ref_bm25_doc_lengths(self._h, fld, out.ctypes.data)
        return out

    def term(self, t: bytes):
        df = C.c_uint32()
        idf = C.c_float()
        ttf = C.c_uint64()
        _refl().ref_bm25_term(self._h, t, len(t), C.byref(df), C.byref(idf), C.byref(ttf))
        return int(df.value), f32(idf.value), int(ttf.value)

    def hash(self, t: bytes) -> int:
        """Bm25Index::hash_term"""
        return int(_refl().ref_bm25_hash(self._h, t, len(t)))

    def close(self):
        if self._h:
            _refl().ref_bm25_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ---- generated corpora and queries (shared by the stored answers, the CPU pin and the device tests) ----
def zipf_vocab(rng, size: int):
    """Mixed-case words of 1..12 letters/digits/underscores."""
    alpha = np.frombuffer(b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789_", np.uint8)
    out = []
    for _ in range(size):
        L = int(rng.integers(1, 13))
        out.append(bytes(alpha[rng.integers(0, 26 if rng.random() < 0.8 else len(alpha), L)]))
    return out


def gen_corpus(seed: int, n: int, mean_words: int = 40, vocab: int = 2000):
    """n documents of Zipf-distributed words with punctuation, bytes >= 0x80, empty and word-free documents."""
    rng = np.random.default_rng(seed)
    voc = zipf_vocab(rng, vocab)
    seps = [b" ", b"  ", b", ", b".\n", b"-", b"\xc3\xa9", b"\xff", b"\t"]
    docs = []
    for _ in range(n):
        r = rng.random()
        if r < 0.03:
            docs.append(b"")
            continue
        if r < 0.05:
            docs.append(b" .,;\xe2\x80\x94 !"[: int(rng.integers(1, 9))])
            continue
        m = int(rng.poisson(mean_words)) + 1
        ids = np.minimum(rng.zipf(1.3, m) - 1, vocab - 1)
        parts = []
        for i in ids:
            parts.append(voc[i])
            parts.append(seps[int(rng.integers(0, len(seps)))])
        docs.append(b"".join(parts))
    return docs, voc


def gen_queries(seed: int, voc, nq: int):
    """Queries of 0..6 words drawn from the vocabulary, unknown words and case variants; some repeat a word."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(nq):
        m = int(rng.integers(0, 7))
        ws = []
        for _ in range(m):
            r = rng.random()
            if r < 0.6:
                ws.append(voc[min(int(rng.zipf(1.3)) - 1, len(voc) - 1)])
            elif r < 0.8:
                ws.append(bytes(rng.integers(97, 123, int(rng.integers(1, 10))).astype(np.uint8)))   # mostly out of vocabulary
            else:
                ws.append(voc[int(rng.integers(0, len(voc)))].upper())
        if ws and rng.random() < 0.2:
            ws.append(ws[0])
        out.append(b" ".join(ws) + (b"?" if rng.random() < 0.3 else b""))
    return out
