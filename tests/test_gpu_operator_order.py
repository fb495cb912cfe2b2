"""Exact result order of the sqlite-vec operator surface (batch_distance TOP_K / FILTERED, vec0_exact).

BATCH_ALL is bit-identical to the reference build, so every ordered mode is pinned against the device sort key built from
that output: (fkey(-dist) << 32) | (0xFFFFFFFF - i), descending.  Equal distances therefore come back by ascending row
index, and a NaN distance (fkey 0) ranks after every finite one in TOP_K mode and drops out of FILTERED mode."""
import numpy as np
import pytest

from tests.pq_restated import fkey

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def Y():
    import yams_b200
    assert yams_b200.device_count() > 0
    assert yams_b200.plugin_init() == 0, yams_b200.health()
    return yams_b200


def make_rows(n, d, seed):
    rng = np.random.default_rng(seed)
    rows = rng.normal(size=(n, d)).astype(np.float32)
    rows[11] = rows[3]           # exact duplicates: equal distances
    rows[n - 1] = rows[3]
    rows[20] = 0                 # zero row
    rows[29, d // 2] = np.nan    # NaN distance under both metrics
    return rows, rng.normal(size=d).astype(np.float32)


def expected_order(dist):
    """row indices in the device's descending key order"""
    i = np.arange(len(dist), dtype=np.uint64)
    keys = (fkey(-np.asarray(dist, dtype=np.float32)) << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - i)
    return np.argsort(keys)[::-1]


def check(got_ids, got_dist, want_ids, all_dist):
    """ids equal; finite distances bit for bit; a NaN distance only where it falls (its bits come back through the key)"""
    assert np.array_equal(got_ids, want_ids)
    want = all_dist[want_ids]
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got_dist), nan)
    assert np.array_equal(got_dist[~nan].view(np.uint32), want[~nan].view(np.uint32))


@pytest.mark.parametrize("n", [1000, 1024])
@pytest.mark.parametrize("d", [33, 64])
def test_batch_distance_order(Y, n, d):
    rows, q = make_rows(n, d, seed=n + d)
    for metric in (Y.COSINE, Y.L2):
        dist = Y.batch_distance(q, rows, metric=metric, mode=Y.BATCH_ALL)
        assert dist.shape == (n,) and np.isnan(dist[29])
        order = expected_order(dist)
        for k in (1, 10, 257, n, n + 5):
            idx, got = Y.batch_distance(q, rows, metric=metric, mode=Y.BATCH_TOP_K, k=k)
            check(idx.astype(np.int64), got, order[:min(k, n)], dist)
        finite = np.sort(dist[~np.isnan(dist)])
        for thr in (float(finite[n // 3]), float(finite[-1]), float("inf")):
            idx, got = Y.batch_distance(q, rows, metric=metric, mode=Y.BATCH_FILTERED, threshold=thr)
            with np.errstate(invalid="ignore"):
                want = order[dist[order] < np.float32(thr)]
            check(idx.astype(np.int64), got, want, dist)


@pytest.mark.parametrize("n", [1000, 1024])
def test_vec0_exact_order(Y, n):
    d = 48
    rows, q = make_rows(n, d, seed=n)
    dist = Y.batch_distance(q, rows, metric=Y.L2, mode=Y.BATCH_ALL)   # vec0_exact ranks by the same L2 distances
    rowids = np.arange(n, dtype=np.int64) * 3 + 100
    for rid in (None, rowids):
        table = np.arange(n, dtype=np.int64) if rid is None else rid
        lo, hi = int(table[n // 5]), int(table[n - n // 4])
        for rng_ in (None, (lo, hi)):
            keep = np.arange(n) if rng_ is None else np.nonzero((table >= lo) & (table <= hi))[0]
            sub = dist[keep]
            order = expected_order(sub)
            for k in (0, 1, 10, 257, len(keep), len(keep) + 5):
                got_rid, got = Y.vec0_exact(q, rows, k=k, rowids=rid, rowid_range=rng_)
                m = len(keep) if k == 0 else min(k, len(keep))
                assert np.array_equal(got_rid, table[keep[order[:m]]]), (rid is None, rng_, k)
                check(np.arange(len(got)), got, np.arange(m), sub[order[:m]])
