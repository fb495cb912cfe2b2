"""The wgmma scan's filter epilogue (csrc/knn_umma.cu): the per-(group, row) bounds are taken while the first K block's
MMAs run, then a one-branch common path sends a thread to the cold per-column test only when some group of its rows passes.
The filter must still list exactly the rows whose stage-1 score is > tau[q] (and that are allowed), with the dense pass's
score, at the shapes where bounds could be taken from the wrong tile or row: one or two K blocks per tile (the bounds are
computed in the only / the first K block), a single row tile, row-tile counts that do not divide among the CTAs, 16 query
tiles, a partial last query tile, candidate sets (the mask test in the cold path), and ties that send every warp into the
cold path."""
import numpy as np
import pytest

from tests.test_gpu_stage1 import WGMMA_MAX_NQ, check_lists, make_corpus

pytestmark = pytest.mark.gpu

ENGINE = 1   # wgmma
COMBOS = [("f16", "cosine"), ("f16", "l2"), ("f32", "cosine"), ("f32", "l2")]


@pytest.fixture(scope="module")
def Y():
    import yams_b200
    assert yams_b200.device_count() > 0
    assert yams_b200.plugin_init() == 0, yams_b200.health()
    return yams_b200


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def below(x):
    return np.nextafter(np.asarray(x, dtype=np.float32), np.float32(-np.inf), dtype=np.float32)


def gen_rows(rng, n, d, dtype):
    r = (rng.standard_normal((n, d)) * np.exp(rng.uniform(-1.0, 1.0, size=(n, 1)))).astype(np.float32)
    return r.astype(np.float16) if dtype == "f16" else r


def mixed_tau(dense, rng):
    """per query: just below its 1st / 5th / 40th best score, +inf or -inf -- neighbouring columns of one threshold group
    with very different thresholds"""
    srt = np.sort(dense, axis=1)
    nq = dense.shape[0]
    k = min(40, dense.shape[1])
    pick = [below(srt[:, -1]), below(srt[:, -min(5, k)]), below(srt[:, -k]), np.full(nq, np.inf), np.full(nq, -np.inf)]
    which = rng.integers(0, len(pick), size=nq)
    return np.array([pick[w][i] for i, w in enumerate(which)], dtype=np.float32)


def check_filter(Y, rows, metric, q, tau_of, allowed=None, cap=None):
    c = make_corpus(Y, rows, metric)
    dense = c.debug_stage1_scores(q, ENGINE)
    tau = tau_of(dense)
    valid = np.isfinite(dense).any(axis=0)
    cap = cap or rows.shape[0]
    counts, lists = c.debug_stage1_candidates(q, ENGINE, tau, cap, allowed=allowed)
    check_lists(dense, counts, lists, tau, cap, 0, 1, valid, allowed)
    c.close()
    return counts


def f16_or_f32_dims(dtype):
    # one K block and two K blocks per tile
    return (64, 72) if dtype == "f16" else (32, 36)


@pytest.mark.parametrize("dtype,metric", COMBOS)
@pytest.mark.parametrize("dim_index", [0, 1])
def test_one_or_two_k_blocks(Y, sms, dtype, metric, dim_index):
    """1 or 2 K blocks per tile, 2 query tiles (the second partial), 235 row tiles: more than the CTAs, not a multiple"""
    d = f16_or_f32_dims(dtype)[dim_index]
    rng = np.random.default_rng(100 + d)
    n = 235 * 128 - 77
    assert (-(-n // 128)) % sms != 0
    rows = gen_rows(rng, n, d, dtype)
    q = (rng.standard_normal((300, d)) * 2.0).astype(np.float32)
    counts = check_filter(Y, rows, metric, q, lambda dense: mixed_tau(dense, rng))
    assert counts.any()


@pytest.mark.parametrize("dtype,metric", COMBOS)
def test_one_row_tile(Y, dtype, metric):
    rng = np.random.default_rng(7)
    d = 200 if dtype == "f16" else 100
    rows = gen_rows(rng, 100, d, dtype)
    q = (rng.standard_normal((520, d)) * 2.0).astype(np.float32)   # 3 query tiles, the last partial
    check_filter(Y, rows, metric, q, lambda dense: mixed_tau(dense, rng))


@pytest.mark.parametrize("dtype,metric", COMBOS)
def test_row_tiles_not_a_multiple_of_the_grid(Y, sms, dtype, metric):
    """2 1/2 row tiles per CTA: some CTAs run one more (row tile, query tile) pair than others"""
    rng = np.random.default_rng(9)
    d = 768 if dtype == "f16" else 100
    n = (2 * sms + sms // 2) * 128 + 5
    rows = gen_rows(rng, n, d, dtype)
    q = (rng.standard_normal((257, d)) * 2.0).astype(np.float32)
    check_filter(Y, rows, metric, q, lambda dense: mixed_tau(dense, rng))


@pytest.mark.parametrize("dtype,metric", COMBOS)
def test_sixteen_query_tiles(Y, dtype, metric):
    rng = np.random.default_rng(16)
    d = 72 if dtype == "f16" else 36
    rows = gen_rows(rng, 3000, d, dtype)
    q = (rng.standard_normal((WGMMA_MAX_NQ, d)) * 2.0).astype(np.float32)
    check_filter(Y, rows, metric, q, lambda dense: mixed_tau(dense, rng))


@pytest.mark.parametrize("dtype", ["f16", "f32"])
def test_candidate_sets(Y, dtype):
    """allowed lists: the rare path's mask test decides, with tau = -inf (every allowed row) and a per-query median"""
    rng = np.random.default_rng(21)
    d = 72 if dtype == "f16" else 36
    n, nq = 20_000, 300
    rows = gen_rows(rng, n, d, dtype)
    q = (rng.standard_normal((nq, d)) * 2.0).astype(np.float32)
    allowed = []
    for i in range(nq):
        kind = i % 4
        if kind == 0:
            allowed.append(np.zeros(0, np.int64))
        elif kind == 1:
            allowed.append(np.sort(rng.choice(n, n // 2, replace=False)).astype(np.int64))
        elif kind == 2:
            allowed.append(np.sort(rng.choice(n, 37, replace=False)).astype(np.int64))
        else:
            allowed.append(np.arange(0, n, 129, dtype=np.int64))
    check_filter(Y, rows, "cosine", q, lambda dense: np.full(nq, -np.inf, np.float32), allowed=allowed)
    check_filter(Y, rows, "cosine", q, lambda dense: np.median(dense, axis=1).astype(np.float32), allowed=allowed)


@pytest.mark.parametrize("dtype,metric", COMBOS)
@pytest.mark.parametrize("at_tau", [False, True])
def test_tie_storm(Y, dtype, metric, at_tau):
    """one row repeated, so a query scores every row the same and every group of every warp passes its bound and takes the
    rare path; tau either just below that score (every row listed) or equal to it (none listed)"""
    rng = np.random.default_rng(33)
    d = 200 if dtype == "f16" else 100
    n, nq = 40 * 128 + 9, 300
    rows = np.repeat(gen_rows(rng, 1, d, dtype), n, axis=0)
    q = (rng.standard_normal((nq, d)) * 2.0).astype(np.float32)

    def tau_of(dense):
        assert (dense == dense[:, :1]).all()
        return (dense[:, 0] if at_tau else below(dense[:, 0])).astype(np.float32)
    counts = check_filter(Y, rows, metric, q, tau_of, cap=n)
    if at_tau:
        assert not counts.any()
    else:
        assert (counts == n).all()

