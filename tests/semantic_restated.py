"""The semantic-neighbour graph's oracle (semantic_graph_restated.c, compiled on first use into a temporary directory) and a
direct Python transcription of the reference loop that the oracle is checked against."""
import atexit
import ctypes as C
import functools
import os
import shutil
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
FLT_TRUE_MIN = float(np.float32(1.4e-45))


@functools.lru_cache(maxsize=None)
def _lib():
    tmp = tempfile.mkdtemp(prefix="semantic_restated_")
    atexit.register(shutil.rmtree, tmp, True)
    out = os.path.join(tmp, "libsemantic_restated.so")
    subprocess.check_call(["/usr/bin/gcc", "-O2", "-fopenmp", "-fPIC", "-shared", "-Wall", "-Wextra",
                           os.path.join(HERE, "semantic_graph_restated.c"), "-o", out, "-lm"])
    lib = C.CDLL(out)
    p = C.c_void_p
    lib.sg_semantic_neighbors.restype = C.c_int
    lib.sg_semantic_neighbors.argtypes = [p, C.c_uint64, C.c_uint32, p, C.c_uint64, C.c_uint32, C.c_int, C.c_float, p, p, p, p]
    return lib


def semantic_neighbors(rows, k, threshold=None, sources=None):
    """rows [n, d] (fp16 rows are widened to fp32 exactly); threshold None = the adaptive mode (sim > 0); sources: None = every
    row, else row indices (>= n: unknown).  -> (rows i64[S,k] (-1 unused), sims f32[S,k] (0 unused), counts u32[S], inv f32[n])"""
    x = np.ascontiguousarray(rows, dtype=np.float32)
    n, d = x.shape if x.ndim == 2 else (0, 0)
    src = None if sources is None else np.ascontiguousarray(sources, dtype=np.int64).reshape(-1)
    ns = n if src is None else len(src)
    out_r = np.empty((max(ns, 1), max(k, 1)), dtype=np.int64)
    out_s = np.empty((max(ns, 1), max(k, 1)), dtype=np.float32)
    out_c = np.empty(max(ns, 1), dtype=np.uint32)
    inv = np.empty(max(n, 1), dtype=np.float32)
    rc = _lib().sg_semantic_neighbors(x.ctypes.data if n else None, n, d, src.ctypes.data if src is not None and ns else None, ns, k,
                                      1 if threshold is None else 0, 0.0 if threshold is None else threshold, out_r.ctypes.data,
                                      out_s.ctypes.data, out_c.ctypes.data, inv.ctypes.data)
    assert rc == 0
    return out_r[:ns, :k], out_s[:ns, :k], out_c[:ns], inv[:n]


def transcribed(rows, k, threshold=None, sources=None):
    """EmbeddingService.cpp:405-431, 856-1017 line by line in Python (float32 / float64 scalars), for small inputs: the
    reference's corpus filter, source list, pair loop, replace-worst top-k and final sort.  -> list of [(row, sim)] per source."""
    x = np.asarray(rows, dtype=np.float32)
    n = x.shape[0]

    def inverse_norm(v):
        norm = 0.0
        for f in v:
            norm += float(f) * float(f)
        return np.float32(0.0) if norm <= 0.0 else np.float32(1.0 / np.sqrt(norm))

    def cosine(a, ia, b, ib):
        dot = 0.0
        for u, v in zip(a, b):
            dot += float(u) * float(v)
        return np.float32(dot * float(ia) * float(ib))

    def better(l, r):
        return l[1] > r[1] if l[1] != r[1] else l[0] < r[0]

    with np.errstate(all="ignore"):
        inv = [inverse_norm(x[r]) for r in range(n)]
    corpus = [r for r in range(n) if inv[r] > 0]
    wanted = range(n) if sources is None else sources
    out = []
    for s in wanted:
        if s not in corpus:
            out.append([])
            continue
        top = []
        for r in corpus:
            if r == s:
                continue
            with np.errstate(all="ignore"):
                sim = cosine(x[s], inv[s], x[r], inv[r])
            if sim != sim:              # NaN: no reference answer, never a neighbour
                continue
            if threshold is not None:
                if sim < np.float32(threshold):
                    continue
            elif sim <= 0:
                continue
            cand = (r, sim)
            if len(top) < k:
                top.append(cand)
                continue
            worst = 0
            for j in range(1, len(top)):
                if better(top[worst], top[j]):
                    worst = j
            if better(cand, top[worst]):
                top[worst] = cand
        top = sorted(top, key=functools.cmp_to_key(lambda a, b: -1 if better(a, b) else (1 if better(b, a) else 0)))
        out.append(top)
    return out
