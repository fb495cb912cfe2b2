"""The profiling instantiation of the wgmma scan (yams_b200_debug_stage1_profile, tools/prof_stage1.py): it runs the search's
filter pass over every row and returns, per CTA, the cycles the first consumer warp waited for data, the cycles the producer
waited for a free ring stage, the epilogue cycles and the total.  Checked here: the launch layout it reports, that every
CTA reports, and that the parts fit inside the total.  Also the filter epilogue's pre-filter, which bounds each row per group
of 32 query columns."""
import numpy as np
import pytest

from tests.test_gpu_stage1 import WGMMA_MAX_NQ, make_corpus

pytestmark = pytest.mark.gpu

UNSUPPORTED = 5


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


@pytest.mark.parametrize("dtype,d,n,nq", [("f16", 72, 40_000, 64), ("f16", 768, 40_000, 300), ("f16", 200, 1000, 1024),
                                          ("f32", 100, 30_000, 257)])
def test_profile_reports_every_cta(Y, sms, dtype, d, n, nq):
    rng = np.random.default_rng(d + nq)
    r = rng.standard_normal((n, d)).astype(np.float32)
    rows = r.astype(np.float16) if dtype == "f16" else r
    c = make_corpus(Y, rows, "cosine")
    q = rng.standard_normal((nq, d)).astype(np.float32)
    dense = c.debug_stage1_scores(q, 1, nrows=min(n, 4096))
    tau = np.sort(dense, axis=1)[:, -4].astype(np.float32)
    cyc, layout, ms = c.debug_stage1_profile(q, tau, cap=4096)
    nrt = -(-n // 128)
    assert layout == {"n_tile": 64 if nq <= 64 else 256, "ctas": min(nrt, sms)}, layout
    assert cyc.shape == (layout["ctas"], 4) and ms > 0
    total = cyc[:, 3].astype(np.int64)
    assert (total > 0).all()
    for i in range(3):
        assert (cyc[:, i].astype(np.int64) <= total).all(), i
    assert (cyc[:, 2] > 0).all()                       # every CTA ran at least one epilogue
    c.close()


def test_profile_declines_what_the_engine_declines(Y):
    d = 64
    rows = np.random.default_rng(1).standard_normal((1000, d)).astype(np.float16)
    c = make_corpus(Y, rows, "cosine")
    q = np.random.default_rng(2).standard_normal((WGMMA_MAX_NQ + 1, d)).astype(np.float32)
    with pytest.raises(Y.YamsB200Error) as e:
        c.debug_stage1_profile(q, np.zeros(len(q), np.float32), cap=16)
    assert e.value.status == UNSUPPORTED
    c.close()


@pytest.mark.parametrize("dtype,metric", [("f16", "cosine"), ("f16", "l2"), ("f32", "cosine")])
def test_filter_bound_per_group_of_32_columns(Y, dtype, metric):
    """The filter epilogue bounds each row per group of 32 query columns by the group's smallest threshold.  Every query but
    a few probes has tau = +inf, so each probe alone sets its group's bound; the probes sit at group edges in both query
    tiles of a 400-query batch (the second one partial).  Each probe must list exactly the rows above its tau: a bound
    taken from another group, or from the wrong query tile, drops them."""
    from tests.test_gpu_stage1 import check_lists
    n, d = 20_000, 72
    rng = np.random.default_rng(11)
    r = (rng.standard_normal((n, d)) * np.exp(rng.uniform(-1.0, 1.0, size=(n, 1)))).astype(np.float32)
    rows = r.astype(np.float16) if dtype == "f16" else r
    c = make_corpus(Y, rows, metric)
    nq = 400
    q = (rng.standard_normal((nq, d)) * 2.0).astype(np.float32)
    dense = c.debug_stage1_scores(q, 1)
    probes = [0, 31, 32, 63, 200, 352, 383, 384, 399]
    tau = np.full(nq, np.inf, dtype=np.float32)
    for i, p in enumerate(probes):
        kth = np.sort(dense[p])[-(3 + 5 * i)]
        tau[p] = np.nextafter(np.float32(kth), np.float32(-np.inf), dtype=np.float32)
    valid = np.isfinite(dense).any(axis=0)
    counts, lists = c.debug_stage1_candidates(q, 1, tau, 256)
    check_lists(dense, counts, lists, tau, 256, 0, 1, valid)
    assert all(counts[p] >= 3 for p in probes) and counts.sum() == sum(int(counts[p]) for p in probes)
    c.close()
