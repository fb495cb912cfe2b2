"""The Simeon text encoder on the device against the numpy restatement (tests/simeon_restated.py), bit for bit, where the
stored digests of tests/test_gpu_simeon.py do not reach:

* a grid of configurations over both projections, word tokens, L2, n-gram ranges up to 64 bytes, sketch widths 1..16384,
  output widths 1..4096 and seeds, each encoding texts at the edges of the hashing, the projections and the normaliser;
* CTAs that encode three and four texts in one call (a long text, then a short one, then an empty one), and grids of
  just below, at and just above one text per CTA;
* encoders of different shared-memory sizes, and two threads on one encoder, encoding at the same time;
* the argument limits of yams_b200_simeon_create and yams_b200_simeon_encode.

tests/test_simeon_restated.py anchors the restatement to the reference (its stored digests everywhere, simeon's own encoder
on this grid where that is built)."""
import ctypes as C
import functools
import threading

import numpy as np
import pytest

from tests import simeon_restated as R

pytestmark = pytest.mark.gpu

DEF = None                        # the profile's default seed
SEED_NAMES = {0: "0", 1: "1", 2 ** 64 - 1: "max", DEF: "def"}


def point(proj, words, l2, ngram, sketch, out, hseed=DEF, pseed=DEF) -> dict:
    """one grid point as SimeonEncoder overrides (also encode()'s keyword arguments)"""
    return dict(ngram_min=ngram[0], ngram_max=ngram[1], sketch_dim=sketch, output_dim=out,
                hash_seed=R.DEFAULT_HASH_SEED if hseed is DEF else hseed,
                projection_seed=R.DEFAULT_PROJECTION_SEED if pseed is DEF else pseed, l2_normalize=l2,
                flags=(R.WORD_TOKENS if words else 0) | (R.PROJECTION_FWHT if proj == "fwht" else 0),
                id=f"{proj}-{'words' if words else 'chars'}-{'l2' if l2 else 'raw'}-n{ngram[0]}_{ngram[1]}-s{sketch}-o{out}"
                   f"-h{SEED_NAMES[hseed]}-p{SEED_NAMES[pseed]}")


M = 2 ** 64 - 1
# Every n-gram range, sketch width, output width and seed of the grid appears at least once under each projection where it
# is allowed (Fwht: output_dim <= next_pow2(sketch_dim)); 16384 x 4096 is the largest layout the ABI accepts.
GRID = [
    point("ach", 0, 1, (1, 1), 1, 1),
    point("ach", 0, 1, (1, 8), 1, 384, hseed=0),
    point("ach", 1, 1, (3, 5), 1, 17),
    point("ach", 1, 1, (3, 5), 2, 7, pseed=0),
    point("ach", 0, 0, (8, 8), 2, 33, hseed=1),
    point("ach", 0, 1, (1, 64), 2, 1),
    point("ach", 0, 1, (9, 16), 3, 15, pseed=1),
    point("ach", 1, 0, (16, 16), 3, 16, hseed=M),
    point("ach", 0, 1, (17, 24), 16, 17, pseed=M),
    point("ach", 1, 1, (60, 64), 16, 31, hseed=0, pseed=0),
    point("ach", 0, 1, (1, 64), 4095, 1000, hseed=1, pseed=1),
    point("ach", 0, 0, (16, 16), 4095, 384),
    point("ach", 1, 1, (3, 5), 4096, 4096),
    point("ach", 0, 1, (8, 8), 4096, 7),
    point("ach", 1, 1, (3, 5), 4096, 384),
    point("ach", 0, 1, (3, 5), 5000, 384, hseed=M, pseed=M),
    point("ach", 1, 1, (17, 24), 5000, 1000, pseed=0),
    point("ach", 1, 0, (1, 8), 16383, 33),
    point("ach", 1, 1, (60, 64), 16383, 16, hseed=1),
    point("ach", 0, 1, (9, 16), 16384, 4096),
    point("ach", 1, 1, (1, 1), 16384, 1, hseed=0),
    point("fwht", 0, 1, (1, 1), 1, 1),
    point("fwht", 1, 1, (60, 64), 1, 1, pseed=0),
    point("fwht", 1, 1, (1, 8), 2, 1, hseed=0),
    point("fwht", 1, 1, (3, 5), 3, 1, pseed=1),
    point("fwht", 0, 1, (17, 24), 3, 1, hseed=1, pseed=1),
    point("fwht", 0, 1, (8, 8), 16, 16),
    point("fwht", 1, 0, (9, 16), 16, 7, hseed=M),
    point("fwht", 0, 1, (16, 16), 16, 15, pseed=M),
    point("fwht", 0, 1, (1, 64), 16, 1),
    point("fwht", 1, 1, (17, 24), 4095, 4096),
    point("fwht", 1, 1, (16, 16), 4095, 384, hseed=0, pseed=M),
    point("fwht", 0, 1, (60, 64), 4096, 384, hseed=1, pseed=0),
    point("fwht", 1, 0, (1, 1), 4096, 1000, pseed=1),
    point("fwht", 1, 1, (1, 64), 5000, 1000),
    point("fwht", 0, 0, (3, 5), 5000, 17, hseed=0),
    point("fwht", 1, 1, (1, 8), 16383, 31),
    point("fwht", 1, 1, (8, 8), 16383, 16),
    point("fwht", 1, 1, (3, 5), 16384, 4096),
    point("fwht", 0, 1, (9, 16), 16384, 33, hseed=M, pseed=M),
]
GRID_IDS = [p.pop("id") for p in GRID]


# ---- texts ----------------------------------------------------------------------------------------------------------------

WORD_BYTES = np.frombuffer(b"ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789_", dtype=np.uint8)


@functools.lru_cache(maxsize=None)
def fixed_texts():
    """(name, text) pairs every grid point encodes"""
    rng = np.random.default_rng(2024)
    mixed = np.frombuffer(b"abcdefgh _-.,XYZ019\x00\xff", dtype=np.uint8)
    texts = [("empty", b"")]
    texts += [(f"len{n}", bytes(rng.choice(mixed, n))) for n in (7, 8, 9, 15, 16, 17, 63, 64, 65)]   # around the 8-byte words
    texts += [
        ("bytes-00-ff", bytes(range(256))),
        ("every-byte-glued-to-words", b" ".join(b"ab" + bytes([c]) + b"Z9" for c in range(256))),
        ("high-bytes-in-a-word", "Größe_42 naïve日本語_x".encode()),
        ("words-at-both-ends", b"Start_1 (middle) -- end_2"),
        ("word-run-100KB", bytes(rng.choice(WORD_BYTES, 100_000))),
        ("random-1MB", rng.integers(0, 256, 1 << 20, dtype=np.uint8).tobytes()),
        ("one-byte-200KB", b"z" * 200_000),      # every gram of a length lands in one bucket: sketch values in the 10^5..10^7
    ]
    return texts


def cancelling_texts(cfg) -> list:
    """Non-empty texts whose whole sketch cancels to zero at cfg (one per alphabet that has one among 2048 candidates of
    ngram_min + 1 .. ngram_min + 4 bytes); only a sketch of one or two buckets makes them easy to find"""
    rng = np.random.default_rng(99)
    k = cfg["ngram_min"]
    found = []
    for alphabet in (b"!-.,;:/()[]{}<>?", b"ab_ .xyZ9-"):
        a = np.frombuffer(alphabet, dtype=np.uint8)
        cands = [bytes(rng.choice(a, k + 1 + i % 4)) for i in range(2048)]
        sk = R.sketches(cands, k, cfg["ngram_max"], cfg["sketch_dim"], cfg["hash_seed"], bool(cfg["flags"] & R.WORD_TOKENS))
        hits = np.nonzero(~np.any(sk != 0, axis=1))[0]
        if len(hits):
            found.append(cands[hits[0]])
    assert found, cfg
    return found


def edge_texts(cfg) -> list:
    """(name, text) pairs of one grid point: the fixed set, a text one byte shorter than ngram_min and one exactly that
    long, and at a sketch of one or two buckets texts whose sketch cancels to zero"""
    k = cfg["ngram_min"]
    rng = np.random.default_rng(k)
    texts = [("ngram_min-1", bytes(rng.choice(WORD_BYTES, k - 1))), ("ngram_min", bytes(rng.choice(WORD_BYTES, k)))]
    texts += fixed_texts()
    if cfg["sketch_dim"] <= 2:
        texts += [(f"cancels-{i}", t) for i, t in enumerate(cancelling_texts(cfg))]
    return texts


def assert_same_bits(got, want, names):
    assert got.shape == want.shape
    bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
    if len(bad):
        i, j = bad[0]
        pytest.fail(f"{len(bad)} coordinates differ; the first in text {i} ({names[i]}), coordinate {j}: "
                    f"device {got[i, j]!r} ({got[i, j:j + 1].view(np.uint32)[0]:#010x}), "
                    f"restatement {want[i, j]!r} ({want[i, j:j + 1].view(np.uint32)[0]:#010x})")


# ---- device -------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def Y():
    import yams_b200
    assert yams_b200.device_count() > 0
    assert yams_b200.plugin_init() == 0, yams_b200.health()
    return yams_b200


def encode_once(Y, cfg, texts):
    enc = Y.SimeonEncoder(**cfg)
    try:
        return enc.encode(texts)
    finally:
        enc.close()


@pytest.mark.parametrize("cfg", GRID, ids=GRID_IDS)
def test_encoder_matches_the_restatement_on_the_grid(Y, cfg):
    named = edge_texts(cfg)
    names = [n for n, _ in named]
    texts = [t for _, t in named]
    got = encode_once(Y, cfg, texts)
    want = R.encode(texts, **cfg)
    assert_same_bits(got, want, names)
    no_features = ["empty"] + ["ngram_min-1"] * (cfg["ngram_min"] == 1 or not cfg["flags"] & R.WORD_TOKENS)
    for i, name in enumerate(names):
        if name.startswith("cancels") or name in no_features:
            assert not np.any(want[i]), name          # a zero vector: the normaliser's sum <= 0 branch


def multi_text_batch(G: int, n: int) -> list:
    """n texts for a grid of G CTAs (CTA b encodes b, b + G, b + 2G, ...): the first round long, the second short, the third
    empty, the rest of mixed length -- what a CTA keeps of its previous text would show in the next"""
    rng = np.random.default_rng(n)
    pool = np.frombuffer(b"the quick brown fox_42 JUMPS over lazy dogs, \x00\x80\xff.", dtype=np.uint8)
    out = []
    for t in range(n):
        rnd = t // G
        if rnd == 0:
            size = int(rng.integers(1500, 4000))
        elif rnd == 1:
            size = int(rng.integers(3, 40))
        elif rnd == 2:
            size = 0
        else:
            size = int(rng.integers(0, 3000))
        out.append(bytes(rng.choice(pool, size)))
    return out


@pytest.mark.parametrize("profile", ["simeon-v1-384", "yams-default"])
def test_ctas_that_encode_several_texts(Y, profile):
    import torch
    G = torch.cuda.get_device_properties(0).multi_processor_count * 8
    cfg = R.config(profile)
    n = 3 * G + 5
    texts = multi_text_batch(G, n)
    enc = Y.SimeonEncoder(profile)
    got = enc.encode(texts)
    want = R.encode(texts, **cfg)
    assert_same_bits(got, want, [f"round {t // G} of CTA {t % G}, {len(texts[t])} bytes" for t in range(n)])
    assert not np.any(want[2 * G:3 * G]) and np.all(np.any(want[:2 * G] != 0, axis=1))
    for t in (G, G + 1, 2 * G - 1, 2 * G, 3 * G - 1, 3 * G, n - 1):   # texts a CTA encoded after another
        assert np.array_equal(enc.encode([texts[t]])[0].view(np.uint32), got[t].view(np.uint32)), t
    enc.close()


@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_one_text_per_cta_and_one_more(Y, delta):
    import torch
    G = torch.cuda.get_device_properties(0).multi_processor_count * 8
    rng = np.random.default_rng(40 + delta)
    texts = [bytes(rng.integers(0, 256, int(rng.integers(0, 600)), dtype=np.uint8)) for _ in range(G + delta)]
    texts[-1] = b"a last text that the first CTA encodes twice when there is one text more than CTAs"
    for profile in ("simeon-v1-384", "yams-default"):
        got = encode_once(Y, R.config(profile), texts)
        assert_same_bits(got, R.encode(texts, **R.config(profile)), [f"text {t}" for t in range(len(texts))])


def test_concurrent_encoders(Y):
    """Two encoders of different shared-memory size (34 KB and 147 KB) and two threads on one encoder, all encoding at the
    same time: every call succeeds and equals the restatement.  A bounded run: 50 calls per thread."""
    small = R.config()
    big = R.config("yams-default", 4096, sketch_dim=16384)
    rng = np.random.default_rng(5)
    batches = [[bytes(rng.integers(0, 256, int(rng.integers(0, 2500)), dtype=np.uint8)) for _ in range(6)] for _ in range(4)]
    enc_small, enc_big = Y.SimeonEncoder(**small), Y.SimeonEncoder(**big)
    jobs = [(enc_small, small, batches[0]), (enc_big, big, batches[1]), (enc_big, big, batches[2]), (enc_small, small, batches[3])]
    wants = [R.encode(b, **c) for _, c, b in jobs]
    failures = []
    start = threading.Barrier(len(jobs))

    def run(j):
        enc, _, batch = jobs[j]
        start.wait()
        for call in range(50):
            try:
                got = enc.encode(batch)
            except Exception as e:                      # noqa: BLE001 -- reported below
                failures.append((j, call, repr(e)))
                return
            if not np.array_equal(got.view(np.uint32), wants[j].view(np.uint32)):
                failures.append((j, call, "differs from the restatement"))
                return

    threads = [threading.Thread(target=run, args=(j,)) for j in range(len(jobs))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    enc_small.close()
    enc_big.close()
    assert not failures, failures


def test_accepted_argument_limits(Y):
    texts = [b"", b"x", b"an edge of the argument range", bytes(range(256)) * 3]
    for cfg in (R.config(ngram_min=1, ngram_max=64), R.config(ngram_min=64, ngram_max=64),
                R.config(sketch_dim=16384, output_dim=4096),
                R.config(sketch_dim=3, output_dim=4, flags=R.PROJECTION_FWHT),          # output_dim == pad_n
                R.config("yams-default", 1, sketch_dim=1)):                           # pad_n = 1
        assert_same_bits(encode_once(Y, cfg, texts), R.encode(texts, **cfg), [repr(t[:8]) for t in texts])
    from yams_b200._lib import f32p, lib
    enc = Y.SimeonEncoder()
    # a null text of length 0 is the empty text
    out = np.full((2, 384), np.nan, dtype=np.float32)
    ptrs = (C.c_char_p * 2)(None, b"abcdef")
    lens = (C.c_size_t * 2)(0, 6)
    assert lib().yams_b200_simeon_encode(enc._h, ptrs, lens, 2, out.ctypes.data_as(f32p)) == 0
    assert_same_bits(out, R.encode([b"", b"abcdef"]), ["null", "abcdef"])
    # no texts: nothing is read or written
    assert lib().yams_b200_simeon_encode(enc._h, None, None, 0, None) == 0
    assert enc.encode([]).shape == (0, 384)
    enc.close()


@pytest.mark.parametrize("bad", [
    dict(ngram_max=65), dict(ngram_min=0), dict(ngram_min=6, ngram_max=5), dict(sketch_dim=0), dict(sketch_dim=16385),
    dict(output_dim=0), dict(output_dim=4097), dict(flags=4), dict(flags=-1),
    dict(flags=R.PROJECTION_FWHT, sketch_dim=3, output_dim=5),                       # Fwht: output_dim > next_pow2(sketch_dim)
    dict(flags=R.PROJECTION_FWHT, sketch_dim=1, output_dim=2),
], ids=lambda d: "-".join(f"{k}={v}" for k, v in d.items()))
def test_rejected_arguments(Y, bad):
    with pytest.raises(Y.YamsB200Error) as e:
        Y.SimeonEncoder(**bad)
    assert e.value.status == 1
