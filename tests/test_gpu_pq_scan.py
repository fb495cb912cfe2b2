"""The full-scan PQ search (yams_b200_pq_search -> pq_search_batch) against the numpy restatement of the engine
(tests/pq_restated.py, anchored to the reference's stored answers by tests/test_pq_restated.py), bit for bit: rowids, scores,
counts and flags of every query, codes (on a sample of rows for the large indexes), lookup tables (PqIndex.debug_lut).  Every
case asserts through PqIndex.last_path() the branch it is there for: the filtered pass (its 16-byte code branch at m % 16 == 0
and the scalar one), 4, 2 and 1 lookup tables per CTA, sample doubling, the 63/64-tile switch, the overflow re-run, and the
per-tile sorting pass (YAMS_B200_PQ_UNFILTERED=1, which must give the same bytes).  Large batches repeat <= 40 distinct queries
in a scrambled order, so the restatement runs once per distinct query."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import pq_restated as R
from tests import test_gpu_pq as TP
from tests.test_pq_restated import GRID_DSUB, GRID_K, grid_case, same_bits

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TILE = 4096


@pytest.fixture(scope="module")
def Y():
    import yams_b200
    assert yams_b200.device_count() > 0
    assert yams_b200.plugin_init() == 0, yams_b200.health()
    return yams_b200


def scrambled(n_distinct: int, nq: int, seed: int) -> np.ndarray:
    """nq indexes into n_distinct queries, neighbours always different"""
    idx = np.random.default_rng(seed).integers(0, n_distinct, nq)
    for i in range(1, nq):
        if n_distinct > 1 and idx[i] == idx[i - 1]:
            idx[i] = (idx[i] + 1) % n_distinct
    return idx


class Case:
    """a corpus + PQ index on the device and its restatement (device codes, checked on a sample of rows)"""

    def __init__(self, Y, O, d, dtype, m, kc, codebooks, tie_keys=None, rows=None, synth=None, rowids=None, sample=2000, seed=0):
        self.O, self.d = O, d
        self.c = Y.Corpus(d, dtype, Y.COSINE)
        if synth is not None:                                    # rows generated on the device: (seed, n)
            s, n = synth
            self.c.append_synthetic(s, 0, n)
            f16 = dtype == Y.F16

            def held(r):
                g = np.concatenate([O.gen_rows_f32(s, int(x), 1, d) for x in np.atleast_1d(r)]) if np.size(r) else np.zeros((0, d), np.float32)
                return O.f16_to_float(O.f16_from_float(g)).reshape(-1, d) if f16 else g
            self.held = held
            rowids = np.arange(n, dtype=np.int64)
            idx_rows = np.arange(n)
        else:
            n = len(rows)
            if dtype == Y.F16:
                bits = O.f16_from_float(rows).reshape(n, d)
                self.c.append(bits.view(np.float16), rowids=rowids)
                rows = O.f16_to_float(bits).reshape(n, d)
            else:
                self.c.append(rows, rowids=rowids)
            self.held = rows
            rowids = np.arange(n, dtype=np.int64) if rowids is None else rowids
            idx_rows = np.nonzero(R.normalise(rows)[1])[0]
        self.pq = Y.PqIndex(self.c, m, kc, codebooks, tie_break_keys=tie_keys)
        codes, code_rowids = self.pq.codes()
        assert np.array_equal(code_rowids, rowids[idx_rows])
        self.index = R.Index(self.held, rowids, m, kc, codebooks, tie_keys, codes=codes, idx_rows=idx_rows)
        rng = np.random.default_rng(seed)
        pick = np.unique(np.concatenate([[0, len(idx_rows) - 1], rng.choice(len(idx_rows), min(sample, len(idx_rows)), replace=False)]))
        want = R.encode(R.normalise(self.index.rows_of(idx_rows[pick]))[0], codebooks, m, kc)
        assert np.array_equal(codes[pick], want)

    @functools.lru_cache(maxsize=None)
    def answer(self, qbytes, k, rf, thr):
        return self.index.search(np.frombuffer(qbytes, dtype=np.float32), k, rf, thr)

    def check(self, queries, k, rf, thr):
        """search the batch on the device; every query's answer equals the restatement's"""
        got = self.pq.search(queries, k, rerank_factor=rf, threshold=thr)
        for qi, q in enumerate(queries):
            r, s, cnt, fl = self.answer(np.ascontiguousarray(q, dtype=np.float32).tobytes(), k, rf, thr)
            assert got[2][qi] == cnt, (qi, k, rf)
            assert np.array_equal(got[0][qi], r), (qi, k, rf)
            assert np.array_equal(got[1][qi].view(np.uint32), s.view(np.uint32)), (qi, k, rf)
            assert got[3][qi] == fl, (qi, k, rf)
        return got

    def check_luts(self, queries):
        table, valid = self.pq.debug_lut(queries)
        for qi, q in enumerate(queries):
            t, ok = self.index.query_table(q)
            assert valid[qi] == ok, qi
            if ok:
                assert np.all(same_bits(table[qi], t)), qi

    def close(self):
        self.pq.close()
        self.c.close()


def path(filtered, qg=0, sample_tiles=0, rerun=False):
    return {"filtered": filtered, "qg": qg, "sample_tiles": sample_tiles, "rerun": rerun}


def qg_of(nq, lut_bytes):
    g = 4 if nq >= 4 else (2 if nq >= 2 else 1)
    while g > 1 and g * lut_bytes > 200 * 1024:
        g //= 2
    return g


# ---- the cases (each builder is also run unfiltered in a subprocess) -------------------------------------------------------

BENCH_N = 64 * TILE + 123
BENCH_CFGS = ((10, 1), (10, 2), (64, 16), (1024, 1))


def bench_case(Y, O):
    """the shape bench.py times, scaled: fp16, d = 768, m = 32, k = 256 (the 16-byte code branch), 65 tiles"""
    d, m, kc = 768, 32, 256
    rng = np.random.default_rng(7)
    cb = (rng.normal(size=(m, kc, d // m)) / np.sqrt(d)).astype(np.float32).reshape(-1)
    tk = rng.integers(0, 1 << 64, size=BENCH_N, dtype=np.uint64)
    cs = Case(Y, O, d, Y.F16, m, kc, cb, tie_keys=tk, synth=(42, BENCH_N))
    queries = O.gen_rows_f32(43, 0, 40, d) * np.float32(1.7)
    queries[5] = cs.held(1234)[0]                                 # a corpus row: its own best match
    return cs, queries


def test_bench_shape(Y, oracle):
    cs, queries = bench_case(Y, oracle)
    cs.check_luts(queries)
    for nq in (1, 2, 3, 4, 5, 16, 256, 600):
        batch = queries[scrambled(len(queries), nq, nq)]
        for k, rf in BENCH_CFGS:
            cs.check(batch, k, rf, -1.0)
            last = nq - (nq - 1) // 512 * 512                      # queries of the last slice
            assert cs.pq.last_path() == path(True, qg_of(last, 32 * 256 * 4), 16), (nq, k, rf)
    cs.check(queries[:7], 10, 2, 0.05)
    cs.close()


def group_width_case(Y, O, m, d):
    kc = 256
    rng = np.random.default_rng(m)
    cb = (rng.normal(size=(m, kc, d // m)) / np.sqrt(d)).astype(np.float32).reshape(-1)
    cs = Case(Y, O, d, Y.F16, m, kc, cb, tie_keys=rng.permutation(64 * TILE + 5).astype(np.uint64), synth=(44, 64 * TILE + 5), sample=600)
    return cs, O.gen_rows_f32(45, 0, 5, d)


@pytest.mark.parametrize("m,d,qg", [(96, 768, 2), (160, 640, 1)])
def test_lut_size_group_widths(Y, oracle, m, d, qg):
    """a 96 KiB table leaves room for 2 tables per CTA, a 160 KiB one for 1 (and the largest per-tile pass shared memory)"""
    cs, queries = group_width_case(Y, oracle, m, d)
    cs.check_luts(queries)
    for k, rf in ((10, 2), (64, 16)):
        cs.check(queries, k, rf, -1.0)
        assert cs.pq.last_path() == path(True, qg, 16)
    cs.close()


def scalar_code_case(Y, O):
    """m = 24 (no 16-byte code rows), k = 100 centroids, dsub = 17 (the FMA tail of the table)"""
    m, kc, d = 24, 100, 24 * 17
    rng = np.random.default_rng(24)
    cb = (rng.normal(size=(m, kc, d // m)) / np.sqrt(d)).astype(np.float32).reshape(-1)
    cs = Case(Y, O, d, Y.F32, m, kc, cb, synth=(46, 64 * TILE + 7), sample=1000)
    return cs, O.gen_rows_f32(47, 0, 5, d)


def test_scalar_code_branch(Y, oracle):
    cs, queries = scalar_code_case(Y, oracle)
    cs.check_luts(queries)
    for k, rf in ((10, 2), (64, 16)):
        cs.check(queries, k, rf, -1.0)
        assert cs.pq.last_path() == path(True, 4, 16)
    cs.close()


def tie_storm_case(Y, O, keyed: bool):
    """~2000 copies of one row in every tile (sampled or not) and 50 in the partial last tile; tie keys shuffled, with
    duplicates and values >= 2^63, or absent (row order)"""
    n, d, m, kc = 70 * TILE + 100, 64, 8, 16
    rng = np.random.default_rng(99)
    rows = O.gen_rows_f32(42, 0, n, d)
    tiles = (n + TILE - 1) // TILE
    copies = np.concatenate([t * TILE + rng.choice(min(TILE, n - t * TILE), 2000 if t < tiles - 1 else 50, replace=False) for t in range(tiles)])
    rows[copies] = rows[777]
    tk = None
    if keyed:
        tk = rng.permutation(n).astype(np.uint64)
        tk[::3] |= np.uint64(1 << 63)
        tk[1::7] = tk[0::7][:len(tk[1::7])]
    cb = (rng.normal(size=(m, kc, d // m)) / np.sqrt(d)).astype(np.float32).reshape(-1)
    cs = Case(Y, O, d, Y.F32, m, kc, cb, tie_keys=tk, rows=rows, sample=3000)
    queries = O.gen_rows_f32(48, 0, 5, d)
    queries[0] = rows[777] * np.float32(0.5)
    queries[3] = rows[777] * np.float32(3.0)
    return cs, queries


@pytest.mark.parametrize("keyed", [True, False])
def test_tie_storms(Y, oracle, keyed):
    """equal ADC scores across every tile: the threshold test at equality, tile-local truncation, rank -> row.  The approx
    cut falls inside the run of copies."""
    cs, queries = tie_storm_case(Y, oracle, keyed)
    for k, rf in ((10, 1), (50, 20), (1024, 1)):
        cs.check(queries, k, rf, -1.0)
        assert cs.pq.last_path() == path(True, 4, 16)
    cs.check(queries[:1], 1, 1, -1.0)
    assert cs.pq.last_path() == path(True, 1, 16)
    cs.close()


def sample_doubling_case(Y, O):
    d, m, kc = 32, 8, 16
    rng = np.random.default_rng(129)
    cb = (rng.normal(size=(m, kc, d // m)) / np.sqrt(d)).astype(np.float32).reshape(-1)
    cs = Case(Y, O, d, Y.F32, m, kc, cb, tie_keys=rng.permutation(129 * TILE + 17).astype(np.uint64), synth=(49, 129 * TILE + 17))
    return cs, O.gen_rows_f32(50, 0, 3, d)


def test_sample_doubling(Y, oracle):
    """130 tiles with approx = 1024: 32 sampled tiles"""
    cs, queries = sample_doubling_case(Y, oracle)
    for k, rf in ((64, 16), (1024, 1)):
        cs.check(queries, k, rf, -1.0)
        assert cs.pq.last_path() == path(True, 2, 32)
    cs.check(queries, 10, 2, -1.0)
    assert cs.pq.last_path() == path(True, 2, 16)
    cs.close()


def boundary_case(Y, O, n_idx):
    """64 tiles of corpus rows, zero rows (left out of the index) leaving n_idx indexed"""
    n, d, m, kc = 64 * TILE + 10, 32, 8, 16
    rng = np.random.default_rng(63)
    rows = O.gen_rows_f32(51, 0, n, d)
    rows[np.sort(rng.choice(n, n - n_idx, replace=False))] = 0
    cb = (rng.normal(size=(m, kc, d // m)) / np.sqrt(d)).astype(np.float32).reshape(-1)
    cs = Case(Y, O, d, Y.F32, m, kc, cb, tie_keys=rng.permutation(n).astype(np.uint64), rows=rows)
    assert len(cs.index.idx_rows) == n_idx
    return cs, O.gen_rows_f32(52, 0, 2, d)


@pytest.mark.parametrize("n_idx,filtered", [(63 * TILE, False), (63 * TILE + 1, True)])
def test_filter_switch_is_on_indexed_rows(Y, oracle, n_idx, filtered):
    cs, queries = boundary_case(Y, oracle, n_idx)
    cs.check(queries, 10, 2, -1.0)
    assert cs.pq.last_path() == (path(True, 2, 16) if filtered else path(False))
    cs.close()


def overflow_case(Y, O):
    """the adversarial corpus of test_pq_filtered_scan_overflow_falls_back, its query third of five"""
    cs0 = TP.pq_overflow_case(O)
    cs = Case(Y, O, 64, Y.F32, cs0["m"], cs0["kc"], cs0["codebooks"], tie_keys=cs0["tie_keys"], rows=cs0["rows"], rowids=cs0["rowids"])
    queries = O.gen_rows_f32(53, 0, 5, 64)
    queries[2] = cs0["query"][0]
    return cs, queries


def test_overflow_rerun_with_many_queries(Y, oracle):
    cs, queries = overflow_case(Y, oracle)
    cs.check(queries, 10, 2, -1.0)
    assert cs.pq.last_path() == path(True, 4, 16, rerun=True)
    cs.close()


# ---- filtered == unfiltered ----------------------------------------------------------------------------------------------

UNFILTERED_RUNS = {
    "bench": (bench_case, ((5, 10, 2), (600, 64, 16))),
    "scalar": (scalar_code_case, ((5, 64, 16),)),
    "ties": (functools.partial(tie_storm_case, keyed=True), ((5, 50, 20), (5, 1024, 1))),
    "overflow": (overflow_case, ((5, 10, 2),)),
}


def unfiltered_outputs(Y, O):
    """name -> (bytes of every search's outputs, whether every search took the filtered pass)"""
    out = {}
    for name, (build, searches) in UNFILTERED_RUNS.items():
        cs, queries = build(Y, O)
        blobs, filt = [], []
        for nq, k, rf in searches:
            got = cs.pq.search(queries[scrambled(len(queries), nq, nq)], k, rerank_factor=rf, threshold=-1.0)
            blobs.append(b"".join(np.ascontiguousarray(a).tobytes() for a in got))
            filt.append(cs.pq.last_path()["filtered"])
        cs.close()
        out[name] = (b"".join(blobs), all(filt))
    return out


def test_filtered_and_unfiltered_passes_give_the_same_bytes(Y, oracle, tmp_path):
    here = unfiltered_outputs(Y, oracle)
    assert all(f for _, f in here.values())
    code = (
        "import sys, pickle; sys.path.insert(0, %r)\n"
        "import yams_b200 as Y\n"
        "from oracle import oracle as O\n"
        "from tests.test_gpu_pq_scan import unfiltered_outputs\n"
        "assert Y.plugin_init() == 0\n"
        "pickle.dump(unfiltered_outputs(Y, O), open(%r, 'wb'))\n"
        "print('UNFILTERED OK')\n" % (ROOT, str(tmp_path / "out.pkl")))
    env = dict(os.environ, YAMS_B200_PQ_UNFILTERED="1")
    run = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1200)
    assert "UNFILTERED OK" in run.stdout, run.stdout[-2000:] + run.stderr[-2000:]
    import pickle
    with open(tmp_path / "out.pkl", "rb") as f:
        there = pickle.load(f)
    for name in UNFILTERED_RUNS:
        assert not there[name][1], name
        assert there[name][0] == here[name][0], name


# ---- encoder and lookup-table grid, contract edges ------------------------------------------------------------------------

@pytest.mark.parametrize("k", GRID_K)
def test_encoder_and_lut_grid(Y, oracle, k):
    """duplicate centroids, centroids at +-1e20, NaN entries, an all-NaN subspace; rows at |r|^2 just above / at most 1e-20,
    zero, inf and NaN rows; fp16 subnormal rows; queries whose |q|^2 overflows float"""
    O = oracle
    for dsub in GRID_DSUB:
        g = grid_case(O, k, dsub)
        rows, cb, m = g["rows"], g["codebooks"], g["m"]
        d = rows.shape[1]
        for dtype in ((Y.F32, Y.F16) if dsub in (16, 17) else (Y.F32,)):
            r = rows.copy()
            if dtype == Y.F16:
                r[40:50] *= np.float32(1e-4)                        # fp16 subnormals (|x| < 6.1e-5)
            cs = Case(Y, O, d, dtype, m, k, cb, rows=r, sample=len(r))
            assert np.array_equal(cs.pq.codes()[0], R.encode(R.normalise(cs.held[cs.index.idx_rows])[0], cb, m, k)), (k, dsub)
            if dtype == Y.F16:
                assert np.any((cs.held[40:50] != 0) & (np.abs(cs.held[40:50]) < 6.1e-5))
            cs.check_luts(g["queries"])
            cs.check(g["queries"], 5, 2, -1.0)
            cs.close()


def test_overflowing_query_norm_gives_a_zero_table(Y, oracle):
    g = grid_case(oracle, 33, 17)
    c = Y.Corpus(g["rows"].shape[1], Y.F32, Y.COSINE)
    c.append(g["rows"])
    pq = Y.PqIndex(c, g["m"], 33, g["codebooks"])
    q = np.full((1, g["rows"].shape[1]), 1e30, dtype=np.float32)
    table, valid = pq.debug_lut(q)
    finite = ~np.isnan(g["codebooks"].reshape(g["m"], 33, -1)).any(axis=2)
    assert valid[0] == 1 and np.all(table[0][finite] == 0)
    pq.close()
    c.close()


def test_contract_edges(Y, oracle):
    O = oracle
    n, d, m, kc = 3000, 32, 4, 16
    rng = np.random.default_rng(5)
    rows = O.gen_rows_f32(54, 0, n, d)
    rows[100:140] = rows[99]
    cb = (rng.normal(size=(m, kc, d // m)) / np.sqrt(d)).astype(np.float32).reshape(-1)
    tk = rng.integers(0, 1 << 64, size=n, dtype=np.uint64)
    cs = Case(Y, O, d, Y.F32, m, kc, cb, tie_keys=tk, rows=rows, rowids=np.arange(n, dtype=np.int64) * 3 + 2)
    queries = O.gen_rows_f32(55, 0, 9, d)
    queries[1] = 0                                               # cannot be normalised: nothing
    queries[3, 4] = np.inf                                       # |q|^2 = inf: valid, NaN table entries
    queries[5, 7] = np.nan                                       # NaN norm: valid (not <= 1e-20), NaN table
    queries[7] = np.float32(3e30)                                # |q|^2 overflows float: valid, a table of zeros
    queries[8] = rows[99] * np.float32(2.0)
    cs.check_luts(queries)
    for k, rf in ((10, 0), (10, 1), (5, 4), (64, 16), (1, 1)):
        cs.check(queries, k, rf, -1.0)
        assert cs.pq.last_path() == path(False)
    # a threshold equal to a returned similarity keeps that row
    got = cs.check(queries, 10, 2, -1.0)
    thr = float(got[1][8, 4])
    got2 = cs.check(queries, 10, 2, thr)
    assert got2[2][8] >= 5 and got2[1][8, got2[2][8] - 1] == np.float32(thr)
    # k * rerank_factor: 1024 is served, 1025 is refused (status 1); k = 0 returns nothing
    cs.check(queries[:2], 64, 16, -1.0)
    with pytest.raises(Y.YamsB200Error) as e:
        cs.pq.search(queries[:2], 25, rerank_factor=41, threshold=-1.0)
    assert e.value.status == 1
    assert list(cs.pq.search(queries, 0)[2]) == [0] * len(queries)
    assert cs.pq.last_path() == path(False)
    cs.close()
    # an index smaller than k, and one of a single row
    for n_small in (7, 1):
        cs = Case(Y, O, d, Y.F32, m, kc, cb, rows=rows[:n_small].copy())
        cs.check(queries, 10, 2, -1.0)
        cs.check(queries, 10, 200, -1.0)                          # approx = n_idx: k * rerank_factor > 1024 is fine
        cs.close()
