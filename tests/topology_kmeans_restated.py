"""The k-means topology engine's oracle (topology_kmeans_restated.c, compiled on first use into a temporary directory) and a
line-by-line Python transcription of the reference's runKMeans that the oracle is checked against."""
import atexit
import ctypes as C
import functools
import math
import os
import shutil
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


@functools.lru_cache(maxsize=None)
def _lib():
    tmp = tempfile.mkdtemp(prefix="topology_kmeans_restated_")
    atexit.register(shutil.rmtree, tmp, True)
    out = os.path.join(tmp, "libtopology_kmeans_restated.so")
    subprocess.check_call(["/usr/bin/gcc", "-O2", "-fopenmp", "-fPIC", "-shared", "-Wall", "-Wextra",
                           os.path.join(HERE, "topology_kmeans_restated.c"), "-o", out, "-lm"])
    lib = C.CDLL(out)
    p = C.c_void_p
    lib.tk_kmeans.restype = C.c_int
    lib.tk_kmeans.argtypes = [p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, p, p, p, p]
    return lib


def effective_k(n, k_requested):
    """runKMeans's k for n usable documents (0 below 2 documents)"""
    if n < 2:
        return 0
    k = k_requested if k_requested else int(math.floor(math.sqrt(n) + 0.5))   # std::round of a non-negative value
    return min(max(k, 2), n)


def kmeans(rows, k_requested=0, max_iterations=0):
    """rows [n, d] of usable documents (fp16 rows are widened to fp32 exactly).
    -> (assignment u32[n], centroids f32[k, d], k, iterations)"""
    x = np.ascontiguousarray(rows, dtype=np.float32)
    n, d = x.shape
    kk = effective_k(n, k_requested)
    asg = np.empty(max(n, 1), dtype=np.uint32)
    cent = np.empty((max(kk, 1), d), dtype=np.float32)
    k_out, it_out = C.c_uint32(), C.c_uint32()
    rc = _lib().tk_kmeans(x.ctypes.data if n else None, n, d, k_requested, max_iterations, asg.ctypes.data, cent.ctypes.data,
                          C.addressof(k_out), C.addressof(it_out))
    assert rc == 0 and k_out.value == kk
    return asg[:n], cent[:kk], k_out.value, it_out.value


def transcribed(rows, k_requested=0, max_iterations=0):
    """runKMeans (topology_alternate_engines.cpp:288-478) line by line with Python floats (double) and float32 scalars, over the
    usable documents only, for small inputs.  -> (assignment list, centroids list of float32 arrays, k, iterations)"""
    docs = [np.asarray(r, dtype=np.float32) for r in np.asarray(rows, dtype=np.float32)]
    n = len(docs)
    if n < 2:
        return list(range(n)), [], 0, 0

    def cosine_distance(a, b):
        dot = na = nb = 0.0
        for x, y in zip(a, b):
            dot += float(x) * float(y)
            na += float(x) * float(x)
            nb += float(y) * float(y)
        if na <= 0.0 or nb <= 0.0:
            return 2.0
        cs = dot / (math.sqrt(na) * math.sqrt(nb))
        cs = -1.0 if cs < -1.0 else (1.0 if 1.0 < cs else cs)
        return 1.0 - cs

    def normalized(v):
        norm = 0.0
        for x in v:
            norm += float(x) * float(x)
        v = v.copy()
        if norm > 0.0:
            inv = np.float32(1.0 / math.sqrt(norm))
            for i in range(len(v)):
                v[i] = np.float32(v[i] * inv)
        return v

    def mean_embedding(members):
        c = np.zeros(len(docs[0]), dtype=np.float32)
        for m in members:
            for i in range(len(c)):
                c[i] = np.float32(c[i] + docs[m][i])
        for i in range(len(c)):
            c[i] = np.float32(c[i] / np.float32(len(members)))
        return c

    k = effective_k(n, k_requested)
    centroids = [normalized(docs[0])]
    selected = [False] * n
    selected[0] = True
    min_dist = [float(np.finfo(np.float64).max)] * n
    while len(centroids) < k:
        farthest, farthest_dist = n, -1.0
        for u in range(n):
            if selected[u]:
                continue
            dd = cosine_distance(docs[u], centroids[-1])
            if dd < min_dist[u]:
                min_dist[u] = dd
            if min_dist[u] > farthest_dist:
                farthest_dist, farthest = min_dist[u], u
        if farthest == n:
            break
        selected[farthest] = True
        centroids.append(normalized(docs[farthest]))
    k = len(centroids)

    membership = [0] * n
    iterations = max_iterations if max_iterations else 10
    it = 0
    for _ in range(iterations):
        it += 1
        changed = False
        for u in range(n):
            best, best_dist = 0, float(np.finfo(np.float64).max)
            for c in range(k):
                dd = cosine_distance(docs[u], centroids[c])
                if dd < best_dist:
                    best_dist, best = dd, c
            if best != membership[u]:
                membership[u] = best
                changed = True
        members = [[] for _ in range(k)]
        for u in range(n):
            members[membership[u]].append(u)
        for c in range(k):
            if members[c]:
                centroids[c] = normalized(mean_embedding(members[c]))
        for c in range(k):
            if members[c]:
                continue
            worst, donor, worst_dist = n, k, -1.0
            for u in range(n):
                mc = membership[u]
                if len(members[mc]) <= 1:
                    continue
                dd = cosine_distance(docs[u], centroids[mc])
                if dd > worst_dist:
                    worst_dist, worst, donor = dd, u, mc
            if worst == n:
                continue
            members[donor].remove(worst)
            membership[worst] = c
            members[c].append(worst)
            centroids[c] = normalized(docs[worst])
            centroids[donor] = normalized(mean_embedding(members[donor]))
            changed = True
        if not changed:
            break
    return membership, centroids, k, it


def edge_rows(seed, n, d, dtype=np.float32):
    """A clustered corpus with the k-means edge rows: exact duplicates (empty clusters and chained repairs), a zero row, a NaN
    row, tiny norms (1e-20 in fp32, subnormal in fp16) and a row equidistant to two others."""
    rng = np.random.default_rng(seed)
    centers = rng.standard_normal((max(2, n // 16), d)).astype(np.float32)
    x = centers[rng.integers(0, len(centers), n)] + np.float32(0.3) * rng.standard_normal((n, d)).astype(np.float32)
    if n >= 12:
        x[1:5] = x[0]                     # duplicates of the first centroid
        x[6] = 0.0
        x[7] = np.nan
        x[8] = x[9] * np.float32(1e-20) if dtype == np.float32 else np.float32(1e-7)
        x[10] = 0.0
        x[10, 0] = 1.0
        x[11] = 0.0
        x[11, 0] = 1.0
        x[11, min(1, d - 1)] += 1.0       # equidistant from e0 and e1 directions when d > 1
    return x.astype(dtype).astype(np.float32)


def run_kmeans(embeddings, k_requested=0, max_iterations=0, cluster=None):
    """runKMeans over whole documents (embeddings: a list of 1-d arrays, empty = no embedding): the usable-document rule, iota
    below 2 usable documents, singletons numbered k, k + 1, ... in document order.  cluster(rows, k, iters) -> (assignment, k)
    clusters the usable rows (default: the restatement).  -> int64[n], the vector runKMeans returns."""
    n = len(embeddings)
    dim = next((len(e) for e in embeddings if len(e)), 0)
    usable = [i for i, e in enumerate(embeddings) if len(e) and len(e) == dim]
    if len(usable) < 2:
        return np.arange(n, dtype=np.int64)
    rows = np.stack([np.asarray(embeddings[i], dtype=np.float32) for i in usable])
    if cluster is None:
        asg, _, k, _ = kmeans(rows, k_requested, max_iterations)
    else:
        asg, k = cluster(rows, k_requested, max_iterations)
    out = np.full(n, -1, dtype=np.int64)
    out[usable] = asg
    rest = np.flatnonzero(out < 0)
    out[rest] = k + np.arange(len(rest))
    return out


def partition(labels):
    """cluster labels -> the rank of each document's cluster in order of first appearance (a partition's canonical form)"""
    rank = {}
    return [rank.setdefault(int(v), len(rank)) for v in labels]


REF_SO = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "libref_topology_kmeans.so")


@functools.lru_cache(maxsize=None)
def _ref():
    if not os.path.exists(REF_SO):
        return None
    lib = C.CDLL(REF_SO)
    p = C.c_void_p
    lib.ref_topology_kmeans_partition.restype = C.c_int
    lib.ref_topology_kmeans_partition.argtypes = [p, p, C.c_uint64, C.c_uint32, C.c_uint64, C.c_uint64, p]
    return lib


def have_ref():
    return _ref() is not None


def ref_partition(embeddings, k_requested=0, max_iterations=0):
    """The reference's own KMeansTopologyEngine::buildArtifacts (oracle/_ref) over the documents: its partition, canonical"""
    n = len(embeddings)
    stride = max([len(e) for e in embeddings] + [1])
    rows = np.zeros((n, stride), dtype=np.float32)
    dims = np.array([len(e) for e in embeddings], dtype=np.uint32)
    for i, e in enumerate(embeddings):
        rows[i, :len(e)] = e
    out = np.empty(max(n, 1), dtype=np.int64)
    assert _ref().ref_topology_kmeans_partition(rows.ctypes.data, dims.ctypes.data, n, stride, k_requested, max_iterations,
                                                out.ctypes.data) == 0
    return out[:n].tolist()


def golden_documents(case):
    """The documents of a stored reference case (tests/golden/ref_topology_kmeans.json): edge_rows of the case's seed and shape
    in its dtype's values, with the listed documents made unusable (empty, or one element short)."""
    dtype = np.float16 if case["dtype"] == "f16" else np.float32
    x = edge_rows(case["seed"], case["n"], case["d"], dtype)
    docs = [x[i] for i in range(case["n"])]
    for i in case.get("empty", []):
        docs[i] = np.zeros(0, dtype=np.float32)
    for i in case.get("short", []):
        docs[i] = docs[i][:-1]
    return docs
