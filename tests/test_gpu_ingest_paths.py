"""The public ingest entries agree with each other: every chunking entry gives the same table for the same bytes, every
hashing entry gives the same digests for the same spans, the timing slots are filled after each entry, and a rejected
call leaves the pooled workspaces usable."""
import hashlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def Y():
    import yams_b200
    assert yams_b200.device_count() > 0, "these tests need an H100"
    assert yams_b200.plugin_init() == 0, yams_b200.health()
    return yams_b200


def _device_stream(Y, n, seed):
    import torch
    t = torch.empty(max(n, 1), dtype=torch.uint8, device="cuda")
    Y.synth_bytes_device(seed, 0, max(n, 1), t.data_ptr())
    return t


def _configs(Y):
    return [Y.default_config(Y.STREAMING), Y.default_config(Y.RABIN),
            Y.default_config(Y.STREAMING, min_chunk=512, max_chunk=8192, mask=0x3FF)]


def _session_pieces(n):
    """Uneven feed sizes: tiny, odd, just above the 4 MiB staging threshold, and more than one 256 MiB slice."""
    cycle = [7, 65537, (4 << 20) + 5, 1, (300 << 20) + 13, 4097]
    out, pos, i = [], 0, 0
    while pos < n:
        ln = min(cycle[i % len(cycle)], n - pos)
        out.append((pos, pos + ln))
        pos += ln
        i += 1
    return out


def _spot_check_digests(table, host):
    rng = np.random.default_rng(len(table))
    for i in set(rng.integers(0, len(table), 12).tolist()) | {0, len(table) - 1}:
        o, s = int(table["offset"][i]), int(table["size"][i])
        assert bytes(table["digest"][i]) == hashlib.sha256(host[o:o + s].tobytes()).digest(), i


@pytest.mark.parametrize("n", [5, (4 << 20) + 4099, (600 << 20) + 12345])
def test_every_chunking_entry_gives_the_same_table(Y, n):
    import torch
    t = _device_stream(Y, n, 20261 + n)
    pinned = torch.empty(n, dtype=torch.uint8).pin_memory()
    pinned.copy_(t[:n])
    host = pinned.numpy().copy()                       # ordinary pageable memory
    for cfg in _configs(Y):
        want = Y.chunk_and_hash(host, cfg)
        assert int(want["size"].sum()) == n and want["offset"][0] == 0
        _spot_check_digests(want, host)
        got = {"pinned": Y.chunk_and_hash(pinned.numpy(), cfg),
               "device": Y.chunk_and_hash_device(t.data_ptr(), n, cfg),
               "batch": Y.chunk_and_hash_batch([host], cfg)[0]}
        with Y.IngestSession(cfg) as s:
            parts = [s.feed(host[a:b]) for a, b in _session_pieces(n)]
            parts.append(s.finish())
        got["session"] = np.concatenate(parts)
        for name, table in got.items():
            assert np.array_equal(table, want), (name, n, cfg.variant, cfg.min_chunk)


@pytest.mark.parametrize("big", [False, True])
def test_every_hashing_entry_gives_the_same_digests(Y, big):
    n = (40 << 20) + 77 if big else (8 << 20) + 3
    cfg = Y.default_config(min_chunk=1024, max_chunk=16384, mask=0x3FF) if big else Y.default_config()
    t = _device_stream(Y, n, 777 + n)
    host = t.cpu().numpy()
    table = Y.chunk_and_hash(host, cfg)
    assert (len(table) > 4096) == big                  # the longest-first order runs only for >= 4096 spans
    offs, sizes = table["offset"], table["size"]
    want = np.ascontiguousarray(table["digest"])
    spans = [host[int(o):int(o + s)] for o, s in zip(offs, sizes)]
    assert np.array_equal(Y.sha256_many(spans), want)
    assert np.array_equal(Y.sha256_batch(host, offs, sizes), want)
    assert np.array_equal(Y.sha256_batch_device(t.data_ptr(), n, offs, sizes), want)
    # spans out of table order, overlapping and empty
    rng = np.random.default_rng(5)
    perm = rng.permutation(len(offs))
    o2 = np.concatenate([offs[perm], [0, 0, n]]).astype(np.uint64)
    s2 = np.concatenate([sizes[perm], [n, 0, 0]]).astype(np.uint64)
    d2 = Y.sha256_batch_device(t.data_ptr(), n, o2, s2)
    assert np.array_equal(d2[:len(perm)], want[perm])
    assert bytes(d2[-3]) == hashlib.sha256(host.tobytes()).digest()
    assert bytes(d2[-2]) == bytes(d2[-1]) == hashlib.sha256(b"").digest()
    assert np.array_equal(Y.sha256_batch(host, o2, s2), d2)


def _check_timings(t, batch):
    ms = [t[k] for k in ("scan_ms", "select_ms", "sha256_ms", "total_ms",
                         "host_sync1_ms", "host_sync2_ms", "host_alloc_ms", "host_process_ms")]
    assert all(x >= 0 for x in ms[:4]), ms
    assert ms[3] > 0 and ms[3] >= ms[2], ms
    if batch:
        assert ms[4:] == [0, 0, 0, 0], ms
    return ms


def test_last_timings_after_each_entry(Y):
    n = 16 << 20
    t = _device_stream(Y, n, 99)
    host = t.cpu().numpy()
    cfg = Y.default_config()
    Y.chunk_and_hash(host, cfg)
    ms = _check_timings(Y.ingest_last_timings(), False)
    assert ms[2] > 0
    Y.chunk_boundaries(host, cfg)
    _check_timings(Y.ingest_last_timings(), False)
    Y.chunk_and_hash_device(t.data_ptr(), n, cfg)
    ms = _check_timings(Y.ingest_last_timings(), False)
    assert ms[2] > 0
    Y.chunk_and_hash_batch([host[:3 << 20], host[5:70000], host[:0]], cfg)
    _check_timings(Y.ingest_last_timings(), True)
    Y.chunk_and_hash(host[:1000], cfg)                 # the host slots are written again after a batch
    _check_timings(Y.ingest_last_timings(), False)


def test_rejected_calls_leave_the_pool_usable(Y):
    n = (2 << 20) + 333
    t = _device_stream(Y, n, 4242)
    host = t.cpu().numpy()
    cfg = Y.default_config(min_chunk=2048, max_chunk=32768, mask=0x7FF)
    want = Y.chunk_and_hash(host, cfg)
    offs, sizes = want["offset"], want["size"]
    bad_cfg = Y.default_config(window_size=49)
    rejected = [lambda: Y.chunk_and_hash(host, bad_cfg),
                lambda: Y.chunk_and_hash_device(t.data_ptr(), n, bad_cfg),
                lambda: Y.chunk_and_hash_batch([host, host[:100]], bad_cfg),
                lambda: Y.IngestSession(bad_cfg),
                lambda: Y.sha256_batch(host, [0, n - 10], [5, 11]),            # span past the end of the base buffer
                lambda: Y.sha256_batch_device(t.data_ptr(), n, [n + 1], [0])]
    for rnd in range(40):                              # more rounds than the pool keeps workspaces
        with pytest.raises(Y.YamsB200Error) as e:
            rejected[rnd % len(rejected)]()
        assert e.value.status == 1, str(e.value)
        k = rnd % 5
        if k == 0:
            got = Y.chunk_and_hash(host, cfg)
        elif k == 1:
            got = Y.chunk_and_hash_device(t.data_ptr(), n, cfg)
        elif k == 2:
            got = Y.chunk_and_hash_batch([host], cfg)[0]
        elif k == 3:
            with Y.IngestSession(cfg) as s:
                got = np.concatenate([s.feed(host[:n // 3]), s.feed(host[n // 3:]), s.finish()])
        else:
            assert np.array_equal(Y.sha256_batch(host, offs, sizes), want["digest"])
            got = want
        assert np.array_equal(got, want), rnd
