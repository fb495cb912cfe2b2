"""A plain numpy restatement of the Simeon text encoder (yams_b200/csrc/simeon_encode.cu), bit for bit.

Written from the semantics of simeon's Encoder (splitmix64_hash, sketch_bucket, SketchSink, emit_char_ngrams,
emit_word_tokens, the AchlioptasSparse and Fwht projections, simd::l2_normalize of the AVX2 tier), not from the kernel.
Everything up to the projection is integer arithmetic and exact; every float operation is float32 and correctly rounded,
as numpy float32 arithmetic is, and nothing here mixes dtypes in one float operation.  tests/test_simeon_restated.py anchors
it to the reference's stored digests (and to simeon's own encoder where that is built); tests/test_gpu_simeon_restated.py
judges the device against it at configurations and texts no stored digest covers."""
import functools
import re

import numpy as np

from tests.pq_restated import fma32

F32 = np.float32
F64 = np.float64
U64 = np.uint64
M64 = (1 << 64) - 1

WORD_TOKENS = 1                      # NGramMode::CharAndWord
PROJECTION_FWHT = 2                  # ProjectionMode::Fwht (otherwise AchlioptasSparse)
DEFAULT_HASH_SEED = 0xA5A5A5A5A5A5A5A5
DEFAULT_PROJECTION_SEED = 0xDEADBEEFCAFEBABE
GAMMA = 0x9E3779B97F4A7C15           # splitmix64's increment: seeds the hash and the Fwht sign chain
SAMPLE_SALT = 0xBF58476D1CE4E5B9     # seeds the Fwht row sample
ACH_LOW = U64(0x2AAAAAAAAAAAAAAB)    # h < LOW: -1 (p = 1/6)
ACH_HIGH = U64(0xD555555555555555)   # h >= HIGH: +1 (p = 1/6)
WORD_RUN = re.compile(rb"[A-Za-z0-9_]+")   # std::isalnum in the "C" locale, or '_'
EXACT_F64 = 2 ** 53


def config(profile: str = "simeon-v1-384", embedding_dim: int = 0, **overrides) -> dict:
    """encode()'s keyword arguments for a SimeonEncoder(profile, embedding_dim, **overrides): simeon_v1_384_config, or the
    encoder an unconfigured YAMS builds (CharAndWord + Fwht, output_dim = embedding_dim or 1024)"""
    cfg = dict(ngram_min=3, ngram_max=5, sketch_dim=4096, output_dim=384, hash_seed=DEFAULT_HASH_SEED,
               projection_seed=DEFAULT_PROJECTION_SEED, l2_normalize=1, flags=0)
    if profile == "yams-default":
        cfg.update(output_dim=embedding_dim or 1024, flags=WORD_TOKENS | PROJECTION_FWHT)
    else:
        assert profile == "simeon-v1-384", profile
    cfg.update(overrides)
    return cfg


# ---- splitmix64 ----------------------------------------------------------------------------------------------------------

def mix_int(z: int) -> int:
    z &= M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def mix(z) -> np.ndarray:
    """splitmix64_mix elementwise on uint64 (products wrap mod 2^64)"""
    z = np.asarray(z, dtype=U64)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> U64(30))) * U64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> U64(27))) * U64(0x94D049BB133111EB)
    return z ^ (z >> U64(31))


def le_words(buf: np.ndarray) -> np.ndarray:
    """the little-endian uint64 starting at every byte of buf (which must end in at least 7 padding bytes)"""
    w = np.lib.stride_tricks.sliding_window_view(buf, 8)
    return np.ascontiguousarray(w).view("<u8").reshape(-1).astype(U64)


def tail_word(le, at, r) -> np.ndarray:
    """splitmix64_hash's tail of r = 1..7 bytes at `at`: the bytes little-endian, tagged with r << 56"""
    r = np.asarray(r, dtype=U64)
    return (le[at] & ((U64(1) << (U64(8) * r)) - U64(1))) ^ (r << U64(56))


def hash_runs(le, starts, lens, h0: int) -> np.ndarray:
    """splitmix64_hash of the byte runs (starts[i], lens[i]) of the buffer behind `le`: h0, one mix per full 8-byte word,
    one per tagged tail, a last one with the length.  lens must be sorted by full-word count, largest first, so that the
    runs still in the word loop are a prefix."""
    starts = np.asarray(starts, dtype=np.int64)
    lens = np.asarray(lens, dtype=np.int64)
    nw = lens // 8
    neg = -nw
    assert np.all(np.diff(neg) >= 0)
    h = np.full(len(starts), h0, dtype=U64)
    q, qmax = 0, int(nw[0]) if len(nw) else 0
    while q < qmax:
        a = int(np.searchsorted(neg, -q, side="left"))        # runs with more than q full words
        if a <= 4:
            break
        h[:a] = mix(h[:a] ^ le[starts[:a] + 8 * q])
        q += 1
    for i in range(int(np.searchsorted(neg, -q, side="left"))):   # the last few long runs: word by word, Python integers
        x = int(h[i])
        for w in le[starts[i] + 8 * np.arange(q, nw[i])].tolist():
            x = mix_int(x ^ w)
        h[i] = x
    r = lens % 8
    t = r > 0
    h[t] = mix(h[t] ^ tail_word(le, starts[t] + 8 * nw[t], r[t]))
    return mix(h ^ lens.astype(U64))


def bucket_of(h, dim: int) -> np.ndarray:
    """sketch_bucket: the low 32 bits, masked for a power-of-two dim, else modulo"""
    low = np.asarray(h, dtype=U64).astype(np.uint32)
    b = low & np.uint32(dim - 1) if dim & (dim - 1) == 0 else low % np.uint32(dim)
    return b.astype(np.int64)


# ---- count sketch --------------------------------------------------------------------------------------------------------

def sketches(texts, ngram_min: int, ngram_max: int, sketch_dim: int, hash_seed: int, word_tokens: bool) -> np.ndarray:
    """SketchSink over emit_char_ngrams (+-2 per byte n-gram of every length ngram_min..ngram_max, a text stops at the first
    length longer than itself) and, with word_tokens, emit_word_tokens (+-1 per maximal [A-Za-z0-9_]+ run).  The sign is the
    hash's top bit.  -> int64 [len(texts), sketch_dim]; the reference's int32 sketch equals it while nothing wraps."""
    texts = [bytes(t) for t in texts]
    T = len(texts)
    lens = np.array([len(t) for t in texts], dtype=np.int64)
    offs = np.concatenate([[0], np.cumsum(lens)])
    n = int(offs[-1])
    buf = np.frombuffer(b"".join(texts) + bytes(16), dtype=np.uint8)
    le = le_words(buf)
    h0 = mix_int(hash_seed ^ GAMMA)
    acc = np.zeros(T * sketch_dim, dtype=np.int64)

    def add(tids, h, weight):
        keys = (tids * sketch_dim + bucket_of(h, sketch_dim)) * 2 + (h >> U64(63)).astype(np.int64)
        counts = np.bincount(keys, minlength=2 * T * sketch_dim).reshape(-1, 2)
        acc[:] += weight * (counts[:, 0] - counts[:, 1])

    # char n-grams: the positions with at least k bytes left in their text.  Sorted by that room, largest first, the
    # positions of every k are a prefix, and the prefix hash over full words is shared by all k.
    room = np.repeat(offs[1:], lens) - np.arange(n, dtype=np.int64)
    pos = np.argsort(-room, kind="stable")
    tid = np.repeat(np.arange(T, dtype=np.int64), lens)[pos]
    neg_room = -room[pos]
    h = np.full(n, h0, dtype=U64)
    words_done = 0
    for k in range(ngram_min, ngram_max + 1):
        c = int(np.searchsorted(neg_room, -k, side="right"))
        if c == 0:
            break
        while words_done < k // 8:
            h[:c] = mix(h[:c] ^ le[pos[:c] + 8 * words_done])
            words_done += 1
        r = k % 8
        hk = h[:c] if r == 0 else mix(h[:c] ^ tail_word(le, pos[:c] + 8 * words_done, r))
        add(tid[:c], mix(hk ^ U64(k)), 2)

    if word_tokens:
        starts, rlen, rtid = [], [], []
        for i, t in enumerate(texts):
            for m in WORD_RUN.finditer(t):
                starts.append(int(offs[i]) + m.start())
                rlen.append(m.end() - m.start())
                rtid.append(i)
        if starts:
            starts, rlen, rtid = (np.array(a, dtype=np.int64) for a in (starts, rlen, rtid))
            o = np.argsort(-(rlen // 8), kind="stable")
            add(rtid[o], hash_runs(le, starts[o], rlen[o], h0), 1)
    return acc.reshape(T, sketch_dim)


# ---- projections ---------------------------------------------------------------------------------------------------------

@functools.lru_cache(maxsize=4)
def achlioptas_signs(sketch_dim: int, output_dim: int, seed: int) -> np.ndarray:
    """achlioptas_entry's sign of every (row, col) as int8 [sketch_dim, output_dim]: h = mix(((row << 32) ^ col) ^ seed)"""
    out = np.empty((sketch_dim, output_dim), dtype=np.int8)
    rows = np.arange(output_dim, dtype=U64) << U64(32)
    step = max(1, (1 << 22) // output_dim)
    for c0 in range(0, sketch_dim, step):
        cols = np.arange(c0, min(c0 + step, sketch_dim), dtype=U64)
        h = mix((rows[None, :] ^ cols[:, None]) ^ U64(seed))
        out[c0:c0 + len(cols)] = np.where(h < ACH_LOW, -1, np.where(h >= ACH_HIGH, 1, 0))
    return out


def achlioptas(sk: np.ndarray, output_dim: int, seed: int) -> np.ndarray:
    """(sum of the sketch under +) - (sum under -) in int64, converted to float once and multiplied once by
    float(sqrt(3f) * (1f / sqrt(float(output_dim)))).  The sums are taken as float64 products over the non-zero columns:
    every partial sum is an integer of magnitude at most sum |sketch| < 2^53, so they are exact in any order."""
    T, dim = sk.shape
    signs = achlioptas_signs(dim, output_dim, seed)
    assert np.all(np.abs(sk).sum(axis=1) < EXACT_F64)
    cols = np.nonzero(np.any(sk != 0, axis=0))[0]
    acc = np.zeros((T, output_dim), dtype=F64)
    for c0 in range(0, len(cols), 1024):
        c = cols[c0:c0 + 1024]
        acc += sk[:, c].astype(F64) @ signs[c].astype(F64)
    scale = np.sqrt(F32(3.0)) * (F32(1.0) / np.sqrt(F32(output_dim)))
    return acc.astype(F32) * scale                  # an exact integer rounded once to float32, then one float multiply


def next_pow2(n: int) -> int:
    p = 1
    while p < n:
        p <<= 1
    return p


@functools.lru_cache(maxsize=8)
def fwht_plan(sketch_dim: int, output_dim: int, seed: int):
    """-> (float32 +-1 signs [pad_n], sampled rows int64 [output_dim]): the sign of i is bit 0 of the chain
    rng = mix(rng + i) from mix(seed ^ GAMMA); the rows are a partial Fisher-Yates over [0, pad_n) driven by the chain
    srng = mix(srng + i) from mix(seed ^ SAMPLE_SALT)"""
    pad_n = next_pow2(sketch_dim)
    assert output_dim <= pad_n
    signs = np.empty(pad_n, dtype=F32)
    rng = mix_int(seed ^ GAMMA)
    for i in range(pad_n):
        rng = mix_int(rng + i)
        signs[i] = -1.0 if rng & 1 else 1.0
    idx = list(range(pad_n))
    srng = mix_int(seed ^ SAMPLE_SALT)
    for i in range(output_dim):
        srng = mix_int(srng + i)
        pick = i + srng % (pad_n - i)
        idx[i], idx[pick] = idx[pick], idx[i]
    return signs, np.array(idx[:output_dim], dtype=np.int64)


def fwht(sk: np.ndarray, output_dim: int, seed: int) -> np.ndarray:
    """float(sketch) * sign, zero-padded to pad_n; the in-place butterflies stage by stage (h = 1, 2, 4, ...: x + y into
    the first half of each 2h block, x - y into the second); the sampled rows times float(1f / sqrt(float(output_dim)))"""
    T, dim = sk.shape
    signs, sample = fwht_plan(dim, output_dim, seed)
    pad_n = len(signs)
    x = np.zeros((T, pad_n), dtype=F32)
    x[:, :dim] = sk.astype(F64).astype(F32) * signs[:dim]
    h = 1
    while h < pad_n:
        v = x.reshape(T, -1, 2, h)
        a, b = v[:, :, 0, :], v[:, :, 1, :]
        x = np.stack([a + b, a - b], axis=2).reshape(T, pad_n)
        h <<= 1
    return x[:, sample] * (F32(1.0) / np.sqrt(F32(output_dim)))


# ---- normalisation -------------------------------------------------------------------------------------------------------

def l2_normalized(v: np.ndarray) -> np.ndarray:
    """simd::l2_normalize, AVX2 tier, per row: two 8-lane FMA accumulators over 16-element blocks, acc0 + acc1, the 8 lanes
    summed left to right, an FMA over the tail; a sum <= 0 leaves the row as it is (a NaN sum does not), otherwise every
    element times inv = 1 / sqrt(sum)"""
    v = np.asarray(v, dtype=F32)
    T, n = v.shape
    n16 = n & ~15
    acc0 = np.zeros((T, 8), dtype=F32)
    acc1 = np.zeros((T, 8), dtype=F32)
    for i in range(0, n16, 16):
        acc0 = fma32(v[:, i:i + 8], v[:, i:i + 8], acc0)
        acc1 = fma32(v[:, i + 8:i + 16], v[:, i + 8:i + 16], acc1)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        lanes = acc0 + acc1
        s = lanes[:, 0]
        for lane in range(1, 8):
            s = s + lanes[:, lane]
        for i in range(n16, n):
            s = fma32(v[:, i], v[:, i], s)
        inv = F32(1.0) / np.sqrt(s)
        return np.where((s <= 0)[:, None], v, v * inv[:, None])


# ---- the encoder ---------------------------------------------------------------------------------------------------------

def encode(texts, ngram_min=3, ngram_max=5, sketch_dim=4096, output_dim=384, hash_seed=DEFAULT_HASH_SEED,
           projection_seed=DEFAULT_PROJECTION_SEED, l2_normalize=1, flags=0) -> np.ndarray:
    """Encoder::encode of byte strings -> float32 [len(texts), output_dim] (texts are taken in groups to bound memory)"""
    raw = [t.encode("utf-8") if isinstance(t, str) else bytes(t) for t in texts]
    out = np.zeros((len(raw), output_dim), dtype=F32)
    width = max(sketch_dim, next_pow2(sketch_dim), output_dim)
    group = max(1, (1 << 22) // width)
    for g0 in range(0, len(raw), group):
        sk = sketches(raw[g0:g0 + group], ngram_min, ngram_max, sketch_dim, hash_seed, bool(flags & WORD_TOKENS))
        if flags & PROJECTION_FWHT:
            v = fwht(sk, output_dim, projection_seed)
        else:
            v = achlioptas(sk, output_dim, projection_seed)
        out[g0:g0 + len(sk)] = l2_normalized(v) if l2_normalize else v
    return out
