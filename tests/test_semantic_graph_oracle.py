"""The semantic-neighbour graph's oracle (semantic_graph_restated.c) against a direct Python transcription of the reference loop,
hand-worked answers, and the graph entry point without a GPU."""
import numpy as np
import pytest

from tests import semantic_restated as S


def _as_lists(rows, sims, counts):
    return [[(int(rows[i, j]), float(sims[i, j])) for j in range(int(counts[i]))] for i in range(len(counts))]


def _same(got, want):
    """(row, sim bits) lists"""
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert [r for r, _ in g] == [r for r, _ in w]
        assert [np.float32(s).view(np.uint32) for _, s in g] == [np.float32(s).view(np.uint32) for _, s in w]


def _corpus(seed, n, d):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, d)).astype(np.float32)
    x[3] = x[1]                       # duplicate embeddings
    x[4] = x[1]
    x[5] = 0.0                        # zero row: not in the corpus
    x[6, 2] = np.inf                  # inf element: inverseNorm 0
    x[7] = x[7] * np.float32(1e-8)    # tiny norm (|r|^2 <= 1e-12): in the graph
    x[8] = -x[2]
    x[9, :] = 0.0
    x[9, 0] = 1.0
    x[10] = np.float32(1e-45)         # sum of squares below 2^-256: inverseNorm overflows to +inf, similarities +-inf or NaN
    return x


@pytest.mark.parametrize("threshold", [None, 0.0, 0.3, 1.0])
@pytest.mark.parametrize("k", [1, 3, 8, 40])
def test_oracle_matches_transcription(threshold, k):
    x = _corpus(7, 24, 5)
    for sources in (None, [0, 1, 5, 6, 7, 9, 23, 30]):
        r, s, c, _ = S.semantic_neighbors(x, k, threshold, sources)
        _same(_as_lists(r, s, c), S.transcribed(x, k, threshold, sources))
        assert (r[np.arange(k)[None, :] >= c[:, None]] == -1).all()
        assert (s[np.arange(k)[None, :] >= c[:, None]] == 0).all()


def test_oracle_inverse_norm_rules():
    x = _corpus(11, 12, 4)
    x[11, 1] = np.nan
    r, s, c, inv = S.semantic_neighbors(x, 4)
    assert inv[5] == 0 and inv[6] == 0 and np.isinf(inv[10]) and inv[7] > 1e6 and np.isnan(inv[11])
    assert c[5] == 0 and c[6] == 0 and c[11] == 0 and c[7] > 0
    assert c[10] > 0 and np.isposinf(s[10, 0])           # an infinite scale is taken, with infinite similarities
    assert not (r == 11).any()                           # NaN similarities are never neighbours


def test_self_skipped_and_ties_by_position():
    x = np.array([[1, 0], [1, 0], [1, 0], [0, 1]], dtype=np.float32)
    r, s, c, _ = S.semantic_neighbors(x, 2)
    assert c.tolist() == [2, 2, 2, 0]          # row 3 is orthogonal to all others: sim 0 is dropped in adaptive mode
    assert r[0].tolist() == [1, 2] and r[1].tolist() == [0, 2] and r[2].tolist() == [0, 1]
    assert (s[:3] == 1).all()


def test_negative_zero_only_at_threshold_zero():
    # s = (1, 0) against n = (-2^-149, 4): dot = -2^-149, inv_n = 1/4 -> sim rounds to -0.0
    x = np.array([[1, 0], [-1.4e-45, 4], [0, 1]], dtype=np.float32)
    for thr in (None, S.FLT_TRUE_MIN, 0.3):
        assert S.semantic_neighbors(x, 2, thr, [0])[2][0] == 0, thr
    r, s, c, _ = S.semantic_neighbors(x, 2, 0.0, [0])
    assert c[0] == 2 and r[0].tolist() == [1, 2]   # -0.0 and +0.0 are one score: row order
    assert np.float32(s[0, 0]).view(np.uint32) == 0x80000000 and np.float32(s[0, 1]).view(np.uint32) == 0


def test_adaptive_is_smallest_positive_threshold():
    x = _corpus(5, 20, 6)
    a = S.semantic_neighbors(x, 6)
    b = S.semantic_neighbors(x, 6, S.FLT_TRUE_MIN)
    for u, v in zip(a[:3], b[:3]):
        assert np.array_equal(u.view(np.uint8), v.view(np.uint8))


def test_semantic_neighbors_fails_without_gpu():
    import yams_b200 as Y
    if Y.device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(Y.YamsB200Error):
        Y.Corpus(8).semantic_neighbors(8)
    out_c = np.zeros(1, dtype=np.uint32)
    assert Y.lib().yams_b200_semantic_neighbors(None, None, 0, 8, Y.FLT_TRUE_MIN, None, None,
                                                out_c.ctypes.data_as(Y._lib.u32p), None) != 0
