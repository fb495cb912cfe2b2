"""The k-means topology engine's oracle (topology_kmeans_restated.c) against a line-by-line Python transcription of the
reference's runKMeans, and hand-worked answers."""
import numpy as np
import pytest

from tests import topology_kmeans_restated as T


def _same(got, want):
    asg, cent, k, it = got
    wa, wc, wk, wi = want
    assert (k, it) == (wk, wi)
    assert asg.tolist() == list(wa)
    assert cent.view(np.uint32).tolist() == np.array(wc, dtype=np.float32).reshape(cent.shape).view(np.uint32).tolist()


@pytest.mark.parametrize("d", [1, 3, 8])
@pytest.mark.parametrize("k,iters", [(0, 0), (2, 1), (5, 10), (40, 3)])
def test_oracle_matches_transcription(d, k, iters):
    for seed, dtype in ((1, np.float32), (2, np.float16)):
        x = T.edge_rows(seed, 30, d, dtype)
        _same(T.kmeans(x, k, iters), T.transcribed(x, k, iters))


def test_duplicates_force_chained_repairs():
    # 9 copies of one row and 3 of another: farthest-first picks the second row, then duplicates of the first
    x = np.array([[1, 0]] * 9 + [[0, 1]] * 3, dtype=np.float32)
    got = T.kmeans(x, 5, 10)
    _same(got, T.transcribed(x, 5, 10))
    asg = got[0]
    assert sorted(set(asg.tolist())) == [0, 1, 2, 3, 4]   # every cluster was repaired by a copy of the big cluster


def test_equidistant_ties_take_the_lowest_centroid():
    x = np.array([[1, 0], [0, 1], [1, 1]], dtype=np.float32)
    asg, _, k, _ = T.kmeans(x, 2, 1)
    assert k == 2 and asg.tolist() == [0, 1, 0]


def test_nan_and_zero_rows():
    x = np.array([[1, 0], [np.nan, 0], [0, 0], [0.5, 0.5], [0, 1]], dtype=np.float32)
    for k in (0, 2, 3, 5):
        _same(T.kmeans(x, k, 10), T.transcribed(x, k, 10))


def test_fewer_than_two_rows_are_singletons():
    asg, cent, k, it = T.kmeans(np.ones((1, 4), dtype=np.float32), 3, 10)
    assert asg.tolist() == [0] and k == 0 and it == 0


def test_k_rule():
    assert [T.effective_k(n, 0) for n in (2, 3, 6, 7, 12, 13, 100_000)] == [2, 2, 2, 3, 3, 4, 316]
    assert T.effective_k(5, 1) == 2 and T.effective_k(5, 9) == 5
