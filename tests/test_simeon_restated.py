"""The numpy restatement of the Simeon text encoder (tests/simeon_restated.py) anchored to the reference, without a GPU:

* its vectorised hashing and count sketch against a literal per-gram loop of splitmix64_hash on short texts;
* on the inputs of the encoder parity tests (tests/test_gpu_simeon.py) it reproduces every stored digest of simeon's own
  encoder (tests/golden/ref_checks.json) and the committed golden embeddings (simeon_golden.json), which makes it a stand-in
  for the reference where no reference is built;
* where the reference build exists (oracle/_ref), it equals simeon's own encoder on the configuration grid and the edge
  texts of tests/test_gpu_simeon_restated.py, under the "C" locale YAMS runs in."""
import contextlib
import json
import locale
import os

import numpy as np
import pytest

from tests import ref_checks
from tests import simeon_restated as R
from tests import test_gpu_simeon as TS
from tests import test_gpu_simeon_restated as TG


# ---- the vectorised hashing against a literal loop ------------------------------------------------------------------------

def splitmix64_hash(s: bytes, seed: int) -> int:
    h = R.mix_int(seed ^ R.GAMMA)
    i = 0
    while i + 8 <= len(s):
        h = R.mix_int(h ^ int.from_bytes(s[i:i + 8], "little"))
        i += 8
    if i < len(s):
        h = R.mix_int(h ^ int.from_bytes(s[i:], "little") ^ ((len(s) - i) << 56))
    return R.mix_int(h ^ len(s))


def sketch_by_loop(text: bytes, kmin, kmax, dim, seed, words) -> np.ndarray:
    sk = np.zeros(dim, dtype=np.int64)
    feats = [(text[i:i + k], 2) for k in range(kmin, kmax + 1) if k <= len(text) for i in range(len(text) - k + 1)]
    if words:
        feats += [(m.group(), 1) for m in R.WORD_RUN.finditer(text)]
    for f, w in feats:
        h = splitmix64_hash(f, seed)
        low = h & 0xFFFFFFFF
        sk[low & (dim - 1) if dim & (dim - 1) == 0 else low % dim] += -w if h >> 63 else w
    return sk


def test_sketch_matches_a_literal_loop():
    rng = np.random.default_rng(3)
    texts = [b"", b"a", b"__", b"ab cd_ef", bytes(range(256))] + [
        bytes(rng.choice(np.frombuffer(b"ab_ 9.\x00\xff", dtype=np.uint8), int(n))) for n in rng.integers(0, 90, 20)]
    for kmin, kmax in ((1, 1), (1, 9), (7, 17), (15, 24), (60, 64), (1, 64)):
        for dim, seed, words in ((1, 0, True), (3, R.DEFAULT_HASH_SEED, False), (4096, 2 ** 64 - 1, True), (5000, 1, True)):
            got = R.sketches(texts, kmin, kmax, dim, seed, words)
            for t, row in zip(texts, got):
                assert np.array_equal(row, sketch_by_loop(t, kmin, kmax, dim, seed, words)), (t[:16], kmin, kmax, dim)


def test_hash_of_long_runs_matches_a_literal_loop():
    rng = np.random.default_rng(4)
    text = bytes(rng.integers(0, 256, 3000, dtype=np.uint8))
    runs = [(0, 3000), (5, 2999 - 5), (100, 64), (7, 65), (1, 8), (2, 1), (9, 0)]
    runs.sort(key=lambda r: -(r[1] // 8))
    le = R.le_words(np.frombuffer(text + bytes(8), dtype=np.uint8))
    got = R.hash_runs(le, [s for s, _ in runs], [n for _, n in runs], R.mix_int(7 ^ R.GAMMA))
    assert [int(h) for h in got] == [splitmix64_hash(text[s:s + n], 7) for s, n in runs]


# ---- the stored reference answers -----------------------------------------------------------------------------------------

@pytest.mark.parametrize("cfg", TS.SIMEON_CFGS)
def test_restatement_reproduces_the_reference_encoder_digests(cfg):
    want = ref_checks.load()["simeon_encoder"][ref_checks.key(cfg)]
    got = R.encode(TS.simeon_texts(cfg), **R.config(**cfg))
    assert list(got.shape) == want["shape"]
    assert ref_checks.digest(got.view(np.uint32)) == want["sha256"]


@pytest.mark.parametrize("cfg", TS.YAMS_PROFILE_CFGS)
def test_restatement_reproduces_the_reference_yams_profile_digests(cfg):
    want = ref_checks.load()["simeon_yams_profile"][ref_checks.key(cfg)]
    got = R.encode(TS.yams_profile_texts(), **R.config(**cfg))
    assert list(got.shape) == want["shape"]
    assert ref_checks.digest(got.view(np.uint32)) == want["sha256"]


def test_restatement_reproduces_the_golden_embeddings():
    with open(os.path.join(ref_checks.GOLDEN, "simeon_golden.json")) as f:
        g = json.load(f)
    for key, kw in TS.GOLDEN_PROFILES:
        got = R.encode([t.encode("utf-8") for t in g["texts"]], **R.config(**kw))
        assert np.array_equal(got.view(np.uint32), np.array(g[key], dtype=np.uint32)), key


# ---- simeon's own encoder, where it is built ------------------------------------------------------------------------------

@contextlib.contextmanager
def c_locale():
    """std::isalnum follows the process locale; YAMS never calls setlocale, so it classifies bytes as "C" does"""
    old = locale.setlocale(locale.LC_CTYPE)
    locale.setlocale(locale.LC_CTYPE, "C")
    try:
        yield
    finally:
        locale.setlocale(locale.LC_CTYPE, old)


def reference_encode(O, texts, cfg):
    kw = {k: v for k, v in cfg.items() if k != "flags"}
    with c_locale():
        if cfg["flags"] == 0:
            return O.simeon_encode_ref(texts, **kw)
        return O.simeon_encode_modes_ref(texts, "CharAndWord" if cfg["flags"] & R.WORD_TOKENS else "CharOnly",
                                         "Fwht" if cfg["flags"] & R.PROJECTION_FWHT else "AchlioptasSparse", **kw)


@pytest.mark.parametrize("cfg", TG.GRID, ids=TG.GRID_IDS)
def test_restatement_matches_simeon_on_the_grid(oracle, cfg):
    O = oracle
    if not O.ref_available():
        pytest.skip("the reference build (oracle/_ref) is not present")
    named = TG.edge_texts(cfg)
    texts = [t for _, t in named]
    TG.assert_same_bits(R.encode(texts, **cfg), reference_encode(O, texts, cfg), [n for n, _ in named])
