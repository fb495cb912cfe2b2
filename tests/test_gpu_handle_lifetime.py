"""Every handle frees what it reserved.  The health JSON counts the bytes the library's device and pinned buffers hold in this
process; a create ... destroy cycle must leave both counts exactly where they were, and each destroy must drop them by at
least the handle's own buffers.  The pooled workspaces (the operator pool, the ingest pool) are warmed by a first run, so
later runs of the same shapes reserve nothing new in them."""
import gc

import numpy as np
import pytest

REPEATS = 20


def counters(Y):
    gc.collect()   # a handle of an earlier test that only the cycle collector reaches must not be freed mid-measurement
    h = Y.health()
    return h["device_buffer_bytes"], h["pinned_buffer_bytes"]


def destroy(Y, handle, device_bytes, pinned_bytes=0):
    """close the handle; the counters must fall by at least the bytes it is known to hold"""
    before = counters(Y)
    handle.close()
    after = counters(Y)
    assert before[0] - after[0] >= device_bytes, (before, after, device_bytes)
    assert before[1] - after[1] >= pinned_bytes, (before, after, pinned_bytes)


def cycles(Y, run):
    run()   # warms the pools
    base = counters(Y)
    for i in range(REPEATS):
        run()
        assert counters(Y) == base, i


@pytest.fixture(scope="module")
def Y():
    import yams_b200
    assert yams_b200.device_count() > 0, "these tests need an H100"
    assert yams_b200.plugin_init() == 0, yams_b200.health()
    return yams_b200


def test_buffer_counters_are_zero_without_gpu():
    import yams_b200 as Y
    if Y.device_count() > 0:
        pytest.skip("a GPU is present")
    h = Y.health()
    assert h["device_buffer_bytes"] == 0 and h["pinned_buffer_bytes"] == 0


@pytest.mark.gpu
def test_corpus_frees_everything(Y):
    import torch
    n, d, nq, k = 20_000, 128, 4, 10
    rng = np.random.default_rng(1)
    rows = rng.standard_normal((n, d)).astype(np.float16)
    q = rng.standard_normal((nq, d)).astype(np.float32)
    dq = torch.from_numpy(q).cuda()
    out_r = torch.empty((nq, k), dtype=torch.int64, device="cuda")
    out_s = torch.empty((nq, k), dtype=torch.float32, device="cuda")
    gone = np.arange(0, n, 3)

    def run():
        c = Y.Corpus(d, Y.F16, Y.COSINE, capacity_hint=n)
        c.append(rows)
        _, _, cnt, _ = c.search(q, k)
        assert (cnt == k).all()
        c.search_device(dq.data_ptr(), nq, k, -1.0, out_r.data_ptr(), out_s.data_ptr())
        c.search_device_finish()
        assert c.remove(gone) == len(gone)
        destroy(Y, c, n * d * 2 + n * 8 + n * 4)   # rows, rowids, inverse norms

    cycles(Y, run)


@pytest.mark.gpu
def test_pq_index_frees_everything(Y):
    n, d, m, kc, nq, k = 8192, 64, 8, 16, 4, 10
    rng = np.random.default_rng(2)
    c = Y.Corpus(d, Y.F32, Y.COSINE)
    c.append(rng.standard_normal((n, d)).astype(np.float32))
    codebooks = (rng.standard_normal((m, kc, d // m)) / np.sqrt(d)).astype(np.float32).reshape(-1)
    q = rng.standard_normal((nq, d)).astype(np.float32)

    def run():
        pq = Y.PqIndex(c, m, kc, codebooks)
        _, _, cnt, _ = pq.search(q, k, threshold=-1.0)
        assert (cnt == k).all()
        destroy(Y, pq, codebooks.nbytes + n * m + 3 * n * 4)   # codebooks, codes, index rows, tie ranks and their order

    try:
        cycles(Y, run)
    finally:
        c.close()


@pytest.mark.gpu
def test_digest_set_frees_everything(Y):
    n = 3000
    digests = np.random.default_rng(3).integers(0, 256, (n, 32), dtype=np.uint8)

    def run():
        s = Y.DigestSet(capacity_hint=1024)
        _, new = s.insert(digests)   # 3000 entries: the table grows past its 2048 initial slots
        assert new == n and len(s) == n
        destroy(Y, s, n * 32 + 2 * n * 4)   # the stored digests and a table of >= 2n slots

    cycles(Y, run)


@pytest.mark.gpu
@pytest.mark.parametrize("profile", ["simeon-v1-384", "yams-default"])
def test_simeon_encoder_frees_everything(Y, profile):
    texts = ["the quick brown fox", "jumps over the lazy dog", "", "x" * 5000]

    def run():
        enc = Y.SimeonEncoder(profile=profile)
        out = enc.encode(texts)
        cfg = enc.cfg
        assert out.shape == (len(texts), cfg.output_dim)
        if cfg.flags & Y.SIMEON_PROJECTION_FWHT:
            pad_n = 1 << (cfg.sketch_dim - 1).bit_length()
            held = pad_n * 4 + cfg.output_dim * 4                      # sign diagonal and row sample
        else:
            held = cfg.sketch_dim * ((cfg.output_dim + 15) // 16) * 4   # the packed projection table
        destroy(Y, enc, held)

    cycles(Y, run)


@pytest.mark.gpu
def test_ingest_session_returns_to_the_pool(Y):
    data = np.random.default_rng(4).integers(0, 256, 3 << 20, dtype=np.uint8)

    def run():
        with Y.IngestSession() as s:
            chunks = [s.feed(data[:1 << 20]), s.feed(data[1 << 20:]), s.finish()]
        assert sum(int(c["size"].sum()) for c in chunks) == data.size

    cycles(Y, run)


@pytest.mark.gpu
def test_operator_pool_holds_steady(Y):
    rng = np.random.default_rng(5)
    db = rng.standard_normal((5000, 64)).astype(np.float32)
    q = rng.standard_normal(64).astype(np.float32)

    def run():
        assert Y.batch_distance(q, db).shape == (5000,)
        rid, _ = Y.vec0_exact(q, db, k=10)
        assert len(rid) == 10

    cycles(Y, run)
