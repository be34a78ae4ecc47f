"""BASELINE.json configs C3 / C4 / C5 at sizes the oracle finishes in seconds — bit-exact against the
oracle through the C ABI (the full-size runs of the same shapes are in bench_configs.py / bench.py)."""
import random

import numpy as np
import pytest

from gpu_world import World
from oracle import oracle as orc

pytestmark = pytest.mark.gpu


def test_c4_direct_many_keys(pcdn):
    """config 4 shape: 128-byte keys, uniform recipients, 512-byte payloads, 10 % unknown keys"""
    rng = random.Random(4)
    w = World(pcdn, max_conns=32768, max_keys=32768, max_batch_msgs=65536, max_batch_bytes=64 << 20,
              ring_bytes_per_conn=1 << 15, max_batch_deliveries=1 << 17)
    keys = [rng.getrandbits(1024).to_bytes(128, "little") for _ in range(30000)]
    for k in keys:
        w.add_user(k, [])
    payload = bytes(range(256)) * 2
    for j in range(40000):
        rc = rng.choice(keys) if rng.random() < 0.9 else rng.getrandbits(1024).to_bytes(128, "little")
        w.direct(rc, orc.direct_frame(rc, payload))
    n = w.check()
    assert 35000 < n < 37000
    assert w.e.last_result.n_direct_dropped == 40000 - n


def test_c3_zipf_mixed_sizes_extended_topics(pcdn):
    """config 3 shape: Zipf-0.99 subscriptions over MORE than 256 topics (engine topic ids are u16;
    the wire's List(UInt8) cannot carry them, the ABI takes topics separately), payloads 256 B-64 KiB"""
    rng = np.random.default_rng(3)
    T, n, M = 600, 3000, 48
    p = 1.0 / np.arange(1, T + 1) ** 0.99
    p /= p.sum()
    w = World(pcdn, max_conns=4096, max_topics=1024, ring_bytes_per_conn=4 << 20, max_batch_bytes=16 << 20,
              max_batch_deliveries=1 << 18)
    for i in range(n):
        w.add_user(i.to_bytes(8, "little") * 4, [int(t) for t in rng.choice(T, size=8, replace=False, p=p)])
    for j in range(M):
        t = int(rng.choice(T, p=p))
        k = int(rng.choice([256 << i for i in range(9)]))
        raw = orc.broadcast_frame([t & 0xFF], bytes(rng.integers(0, 256, size=k, dtype=np.uint8)))
        w.bcast([t], raw)
    assert w.check() > 5000


@pytest.mark.parametrize("dense", [True, False])
def test_c5_4k_broadcast(pcdn, dense):
    """config 5 shard shape: 4 KiB payloads (records > 4 KiB: message-major staged path), all
    subscribed / 4 of 64 topics"""
    rng = random.Random(5)
    w = World(pcdn, max_conns=8192, ring_bytes_per_conn=1 << 17, max_batch_deliveries=1 << 18)
    for i in range(6000):
        w.add_user(i.to_bytes(8, "little"), [0] if dense else rng.sample(range(64), 4))
    for m in range(8 if dense else 40):
        t = 0 if dense else rng.randrange(64)
        w.bcast([t], orc.broadcast_frame([t], bytes([m]) * 4096))
    n = w.check()
    assert n == 48000 if dense else n > 10000


@pytest.mark.parametrize("n_users,k", [(128, 1024), (2, 10000)])
def test_c1_reference_bench_shape(pcdn, n_users, k):
    """config 1 — the reference's own CPU bench shape (cdn-broker/benches/broadcast.rs:50-75) through the
    GPU engine: every subscriber including the sender gets the identical bytes, one message per batch"""
    w = World(pcdn, max_conns=256, ring_bytes_per_conn=1 << 16)
    for i in range(n_users):
        w.add_user(i.to_bytes(8, "little"), [0])
    raw = orc.broadcast_frame([0], bytes((i * 7 + 1) & 0xFF for i in range(k)))
    for _ in range(3):
        assert w.e.user_receive((0).to_bytes(8, "little"), raw) == 0
        assert w.o.user_receive((0).to_bytes(8, "little"), raw) == 0
        assert w.check() == n_users


@pytest.mark.parametrize("staged", [False, True])
def test_span_runs_compress_a_dense_batch(pcdn, staged):
    """PCDN_FLAG_SPAN_RUNS: a dense broadcast batch comes back as one run per 256 (staged: k_offsets
    CTA) or 1024 (fused small-engine kernel) consecutive connections; holes (a connection that is not
    subscribed, one that also got a direct message, a ring that wrapped) break runs exactly there; the
    expanded table equals the plain one and the streams equal the oracle's."""
    flags = pcdn.FLAG_SPAN_RUNS | (pcdn.FLAG_STAGED_SPANS if staged else 0)
    w = World(pcdn, max_conns=8192, ring_bytes_per_conn=1 << 14, flags=flags)
    keys = [i.to_bytes(8, "little") for i in range(6000)]
    for i, k in enumerate(keys):
        w.add_user(k, [] if i in (100, 3000) else [0])       # two holes
    for m in range(3):
        w.bcast([0], orc.broadcast_frame([0], bytes([m]) * 700))
    w.direct(keys[777], orc.direct_frame(keys[777], b"only for 777"))   # 777 has one record more than its neighbours
    b = w.e.flush()
    res = w.e.poll(b)
    assert not res.spans and res.n_runs > 0 and res.n_spans == 5998
    runs = [(res.runs[i].conn0, res.runs[i].n_conns) for i in range(res.n_runs)]
    assert sum(n for _, n in runs) == 5998
    assert res.n_runs <= 5998 // (256 if staged else 1024) + 12, res.n_runs
    starts = {c for c, _ in runs}
    cid = {k: c for c, k in zip(sorted(w.map), keys)}  # ids were handed out in order
    for i in (101, 3001, 777, 778):
        assert cid[keys[i]] in starts, i          # a run starts right after each hole / around the odd one
    got = w.e.collect_frames(res)
    w.e.release_batch(b)
    assert got == w.expect()
    # next batches wrap the 16 KiB rings: two spans for every connection, still exact
    for rnd in range(6):
        for m in range(4):
            w.bcast([0], orc.broadcast_frame([0], bytes([m + rnd]) * 900))
        assert w.check() == 4 * 5998
    w.e.close()


@pytest.mark.parametrize("staged", [False, True])
def test_output_pool_backpressure_and_wrap(pcdn, staged):
    """PCDN_FLAG_OUTPUT_POOL: batches take contiguous regions of one shared pool; a batch that does not
    fit is refused as a whole (status PCDN_EAGAIN, nothing delivered, nothing dropped) together with
    every batch launched after it, and goes through once older batches are released and it is retried
    — the Limiter's ingress back-pressure (cdn-proto/src/connection/limiter/mod.rs:56-68) instead of
    the fixed rings' per-connection overflow.  Regions wrap around the pool end; one hot connection can
    take what 1000 idle ones do not use."""
    flags = pcdn.FLAG_OUTPUT_POOL | (pcdn.FLAG_STAGED_SPANS if staged else 0)
    w = World(pcdn, max_conns=4096, flags=flags, pool_bytes=4 << 20, batch_slots=4, max_batch_bytes=8 << 20)
    keys = [i.to_bytes(8, "little") for i in range(1000)]
    for i, k in enumerate(keys):
        w.add_user(k, [0] if i < 500 else [1])
    hot = keys[7]
    # 1. one connection alone takes 3 MB in one batch (its fixed ring would have been 4 MB / 4096 = 1 KB)
    for j in range(30):
        w.direct(hot, orc.direct_frame(hot, bytes([j]) * 100_000))
    assert w.check() == 30
    # 2. three batches of 1.7 MB each: the third does not fit beside the first two -> refused, as is a fourth
    def big_batch(tag):
        for j in range(3):
            w.bcast([0], orc.broadcast_frame([0], bytes([tag, j]) * 550))   # 500 recipients x 3 x ~1.1 KB
        return w.e.flush()
    b1, b2, b3 = big_batch(1), big_batch(2), big_batch(3)
    w.direct(hot, orc.direct_frame(hot, b"small, but queued behind the refused batch"))
    b4 = w.e.flush()
    r1, r2, r3, r4 = (w.e.poll(b) for b in (b1, b2, b3, b4))
    assert (r1.status, r2.status, r3.status, r4.status) == (0, 0, 11, 11) and r3.n_deliveries == 0 == r4.n_deliveries
    assert r1.n_overflow == r2.n_overflow == r3.n_overflow == 0
    with pytest.raises(pcdn.PcdnError):
        w.e.retry_batch(b3)                      # not the oldest unreleased batch yet
    got = {}
    for b, r in ((b1, r1), (b2, r2)):
        for c, fr in w.e.collect_frames(r).items():
            got.setdefault(c, []).extend(fr)
        w.e.release_batch(b)
    for b in (b3, b4):                           # oldest first: retry, poll again, consume
        w.e.retry_batch(b)
        r = w.e.poll(b)
        assert r.status == 0 and r.n_deliveries > 0
        for c, fr in w.e.collect_frames(r).items():
            got.setdefault(c, []).extend(fr)
        w.e.release_batch(b)
    assert got == w.expect()
    # 3. many more batches: the regions wrap around the 4 MB pool again and again (drain() retries by itself)
    total = 0
    for rnd in range(12):
        for j in range(2):
            w.bcast([rnd % 2], orc.broadcast_frame([rnd % 2], bytes([rnd, j]) * 700))
        w.direct(hot, orc.direct_frame(hot, bytes([rnd]) * 5000))
        total += w.check()
    assert total == 12 * (2 * 500 + 1)
    # 4. a batch larger than the whole pool can never fit: E2BIG, not a retry loop
    for j in range(5):
        w.bcast([0], orc.broadcast_frame([0], bytes([j]) * 2000))       # 5 x 500 x 2 KB = 5 MB > 4 MB
    b = w.e.flush()
    assert w.e.poll(b).status == 12
    w.e.release_batch(b)
    w.o.clear()
    w.taken.clear()
    w.bcast([1], orc.broadcast_frame([1], b"still alive"))
    assert w.check() == 500
    w.e.close()


@pytest.mark.parametrize("pool,pack_variant", [(False, 0), (True, 0), (True, 6 << 8)], ids=["False", "True", "True-6ctas"])
def test_alternating_batch_classes_in_flight(pcdn, pool, pack_variant):
    """The engine moves the pack of short message-major-only batches to its pack stream (so the next
    batch's control kernels run beside it) and decides that from the last COMPLETED batch
    (engine.cu batch_begin, batch_pack).  Several batches are in flight here and their classes alternate
    — sparse 4 KiB broadcasts (message-major only), dense 1 KiB broadcasts (connection-major), direct
    only — so successive packs land on different streams in every order; per-connection order and bytes
    must still be the oracle's.  pack_variant 6 << 8: k_pack with 6 CTAs per SM instead of the 3 or 4
    the engine picks."""
    rng = random.Random(77)
    cfg = dict(max_conns=8192, ring_bytes_per_conn=1 << 18, max_batch_deliveries=1 << 18, batch_slots=4,
               max_batch_bytes=8 << 20, pack_variant=pack_variant)
    if pool:
        cfg.update(flags=pcdn.FLAG_OUTPUT_POOL, pool_bytes=1 << 30)
    w = World(pcdn, **cfg)
    keys = [i.to_bytes(8, "little") for i in range(6000)]
    for i, k in enumerate(keys):
        w.add_user(k, [0] + rng.sample(range(1, 64), 3))
    kinds = ["sparse", "sparse", "dense", "sparse", "direct", "sparse", "sparse", "dense", "dense", "sparse", "direct", "sparse"]
    got, total = {}, 0
    for rnd in range(3):
        ids = []
        for bi, kind in enumerate(kinds):
            tag = rnd * 16 + bi
            if kind == "sparse":
                for m in range(6):
                    t = rng.randrange(1, 64)
                    w.bcast([t], orc.broadcast_frame([t], bytes([tag, m]) * 2100))
            elif kind == "dense":
                for m in range(3):
                    w.bcast([0], orc.broadcast_frame([0], bytes([tag, m]) * 400))
            else:
                for m in range(3000):
                    k = rng.choice(keys)
                    w.direct(k, orc.direct_frame(k, bytes([tag, m & 0xFF]) * 40))
            ids.append(w.e.flush())
            if len(ids) == 4 or bi == len(kinds) - 1:      # four in flight, then consume them oldest first
                for b in ids:
                    r = w.e.poll(b)
                    assert r.status == 0 and r.n_overflow == 0
                    total += r.n_deliveries
                    for c, fr in w.e.collect_frames(r).items():
                        got.setdefault(c, []).extend(fr)
                    w.e.release_batch(b)
                ids = []
    assert got == w.expect()
    assert total > 3 * (3 * 6000 * 3 + 2 * 3000)
    w.e.close()
