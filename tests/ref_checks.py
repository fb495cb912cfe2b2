"""Stored results of the reference build (tests/golden/ref_checks.json): what the reference's own sources, compiled by
`make -C oracle ref`, return for the inputs the tests construct (same seeds, same case lists).

Large reference outputs are kept as (128-bit truncated) SHA-256 digests of their bytes: a test compares the digest of what it
computed with the stored one, which is as strict as comparing the arrays."""
import base64
import functools
import hashlib
import json
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@functools.lru_cache(maxsize=None)
def load() -> dict:
    with open(os.path.join(GOLDEN, "ref_checks.json")) as f:
        return json.load(f)


def digest(*arrays) -> str:
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()[:32]


def key(obj) -> str:
    """Stable key of a test parameter (dict or tuple)."""
    return json.dumps(obj, sort_keys=True)


def f32_from_bits(bits) -> np.ndarray:
    return np.asarray(bits, dtype=np.uint32).view(np.float32)


def unpack_f32(text) -> np.ndarray:
    return np.frombuffer(base64.b64decode(text), dtype="<f4")


def pack_f32(a) -> str:
    return base64.b64encode(np.ascontiguousarray(a, dtype="<f4").tobytes()).decode()


def l2_near_tie_case(O, dtype: str):
    """The L2 near-tie corpus (key "l2_near_tie"): 5000 unit rows of the oracle's generator, 300 of them replaced by an
    adversarial query plus offsets on a 2^-14 grid (squared distances within ~1e-5 of each other), 7 ordinary queries and
    the adversarial one last.  Built from the generator and integer draws only -- no reductions, no libm -- so every machine
    rebuilds the same bits.  -> (rows to append, the float32 values the corpus holds, queries)"""
    n, d = 5000, 128
    rng = np.random.default_rng(12)
    rows = O.gen_rows_f32(42, 0, n, d)
    q_adv = O.gen_rows_f32(77, 0, 1, d)[0]
    pos = np.sort(rng.choice(n, size=300, replace=False))
    rows[pos] = q_adv[None, :] + (rng.integers(-4, 5, size=(300, d)) * 2.0 ** -14).astype(np.float32)
    queries = np.concatenate([O.gen_rows_f32(43, 0, 7, d), q_adv[None, :]])
    if dtype == "f16":
        bits = O.f16_from_float(rows).reshape(n, d)
        return bits.view(np.float16), O.f16_to_float(bits).reshape(n, d), queries
    return rows, rows, queries
