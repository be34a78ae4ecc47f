"""GPU parity tests: the CUDA path, called through the C ABI, against the oracle on the same seeded
inputs.  Bit-exact: every connection must receive exactly the oracle's frames, in the oracle's
order (integer/byte work — no tolerance).  Run with `pytest -m gpu` on an H100.
"""
import random

import numpy as np

import pytest

import gpu_workloads as workloads
import scenarios
from gpu_world import PCDN_EAGAIN, World, payload
from harness import EngineBackend
from oracle import oracle as orc

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------ the reference's own scenarios
@pytest.mark.parametrize("scenario", scenarios.ALL, ids=lambda f: f.__name__)
def test_reference_scenario_on_gpu(pcdn, scenario):
    scenario(EngineBackend(pcdn))


@pytest.mark.parametrize("scenario", scenarios.ALL, ids=lambda f: f.__name__)
def test_reference_scenario_host_rings(pcdn, scenario):
    """egress hand-off mode (PCDN_FLAG_HOST_RINGS): the pack stores the framed records into mapped
    pinned host memory; the scenarios read them in place"""
    scenario(EngineBackend(pcdn, flags=pcdn.FLAG_HOST_RINGS))


@pytest.mark.parametrize("variant", workloads.MIXED_LAYOUTS)
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_mixed_batches(pcdn, seed, variant):
    """users + peer brokers, multi-topic broadcasts (fat and thin recipient sets), directs to local,
    remote and unknown keys, frame sizes from 0 B to 3 staging chunks, several batches.
    Small engines publish spans straight into mapped host memory; "staged" forces the span path of
    large engines (table in HBM, copied out while the pack runs) on the same workload.
    The 'shards-*' variants run the SAME workload on ONE engine whose connections are spread over
    several shards (pcdn_config.devices) and compare with the same single unsharded oracle; the
    '*-staged' ones force the regular control kernels there, so they run with conn_base != 0."""
    workloads.random_mixed_batches(pcdn, seed, variant)


def test_state_change_is_ordered_with_messages(pcdn):
    """R12: a subscribe/unsubscribe/remove between two messages affects only the later one, even
    when both travel through the engine back to back"""
    w = World(pcdn)
    a = w.add_user(b"a" * 8, [])
    w.add_user(b"b" * 8, [1])
    m1, m2, m3 = (orc.broadcast_frame([1], b"m%d" % i) for i in (1, 2, 3))
    w.bcast([1], m1)
    w.both("subscribe_user_to", b"a" * 8, [1])
    w.bcast([1], m2)
    w.both("remove_user", b"b" * 8)
    w.bcast([1], m3)
    got = w.e.drain()
    assert got[a] == [m2, m3]
    want = w.expect()
    assert got == want


def test_direct_hot_recipient_keeps_order(pcdn):
    """many directs to ONE key in one batch (votes to a leader): per-connection order = batch order
    (R9) — exercises the stable (connection, message) sort"""
    workloads.direct_hot_recipient_keeps_order(pcdn)


def test_ring_wrap_and_release(pcdn):
    """rings much smaller than the traffic: records never straddle the ring end, spans split at the
    wrap, released space is reused; delivered streams stay identical to the oracle's"""
    rng = random.Random(11)
    w = World(pcdn, ring_bytes_per_conn=8192, max_conns=256)
    for i in range(100):
        w.add_user(bytes([i]) * 8, [0] if i % 2 == 0 else [1])
    for rnd in range(60):
        for j in range(rng.randrange(1, 5)):
            t = rng.randrange(2)
            w.bcast([t], orc.broadcast_frame([t], payload(rng, rng.randrange(0, 1500))))
        w.direct(bytes([rnd % 100]) * 8, orc.direct_frame(bytes([rnd % 100]) * 8, payload(rng, rng.randrange(0, 900))))
        w.check()


@pytest.mark.parametrize("staged", [False, True])
def test_ring_overflow_reports_connection(pcdn, staged):
    """a slow consumer (nothing released) overflows its ring: deliveries stop at the overflow point,
    the connection is reported so the host can remove it (the R13 analogue); others are unaffected"""
    w = World(pcdn, ring_bytes_per_conn=4096, max_conns=64, flags=pcdn.FLAG_STAGED_SPANS if staged else 0)
    a = w.add_user(b"slow" * 2, [0])
    b = w.add_user(b"fast" * 2, [1])
    frames = [orc.broadcast_frame([0], bytes([i]) * 900) for i in range(8)]
    other = [orc.broadcast_frame([1], bytes([i]) * 10) for i in range(8)]
    for f, g in zip(frames, other):
        w.e.handle_broadcast_message([0], f)
        w.e.handle_broadcast_message([1], g)
    w.e.flush()
    bid = w.e.next_batch()
    res = w.e.poll(bid)
    got = w.e.collect_frames(res)
    assert res.n_overflow == 1 and res.overflow_conns[0] == a
    assert got[b] == other
    k = len(got[a])
    assert 0 < k < 8 and got[a] == frames[:k]      # a prefix, in order
    assert res.n_deliveries == k + 8
    w.e.release_batch(bid)


def test_explicit_submit_and_counters(pcdn):
    w = World(pcdn)
    for i in range(64):
        w.add_user(bytes([i]) * 8, [i % 4])
    msgs, raws = [], []
    for j in range(20):
        if j % 3:
            raw = orc.broadcast_frame([j % 4], b"x" * (j * 31))
            msgs.append(("b", [j % 4], raw, False))
            w.o.handle_broadcast_message([j % 4], raw)
        else:
            raw = orc.direct_frame(bytes([j]) * 8, b"y" * (j * 17))
            msgs.append(("d", bytes([j]) * 8, raw, False))
            w.o.handle_direct_message(bytes([j]) * 8, raw)
    bid = w.e.submit(msgs)
    res = w.e.poll(bid)
    assert res.n_msgs == 20 and res.status == 0
    assert res.n_deliveries == w.o.deliveries() and res.bytes_out == w.o.bytes_sent() + 4 * w.o.deliveries()
    got = w.e.collect_frames(res)
    w.e.release_batch(bid)
    assert got == w.expect()
    # metrics.rs analogues: BYTES_RECV, BYTES_SENT, LATENCY histogram (one observation per released batch)
    st = w.e.stats()
    assert st.bytes_in == sum(len(m[2]) for m in msgs)
    assert st.bytes_out == res.bytes_out and st.released_batches == 1
    assert sum(st.latency_hist_us) == 1 and st.latency_ms_sum > 0


def test_batch_capacity_rejected_not_truncated(pcdn):
    """more deliveries than max_batch_deliveries: the device rejects the whole batch (E2BIG),
    nothing is written and ring cursors are untouched"""
    w = World(pcdn, max_batch_deliveries=1000, max_conns=4096, batch_slots=1, ring_bytes_per_conn=4096)
    for i in range(2000):
        w.add_user(i.to_bytes(8, "little"), [1] if i < 900 else [0])
    # first a batch that fits (leaves this slot's per-connection unit counts non-zero) ...
    for _ in range(3):
        w.bcast([1], orc.broadcast_frame([1], b"fits" * 200))
        assert w.check() == 900
    w.both("subscribe_user_to", (1).to_bytes(8, "little"), [0])
    for i in range(900):
        w.both("subscribe_user_to", i.to_bytes(8, "little"), [0])
    raw = orc.broadcast_frame([0], b"big fan-out")
    # ... then, in the SAME slot, one that does not: releasing it must not hand back ring space twice
    w.e.handle_broadcast_message([0], raw)
    w.e.flush()
    bid = w.e.next_batch()
    res = w.e.poll(bid)
    assert res.status == 12 and res.n_deliveries == 0 and res.n_spans == 0
    w.e.release_batch(bid)
    for _ in range(6):  # ring accounting still exact: 4 KB rings wrap and never report overflow
        w.bcast([1], orc.broadcast_frame([1], b"fits" * 200))
        assert w.check() == 900
        assert w.e.last_result.n_overflow == 0
    # the engine keeps working afterwards
    w.both("unsubscribe_user_from", (5).to_bytes(8, "little"), [0])
    for i in range(1500):
        w.both("unsubscribe_user_from", (i + 100).to_bytes(8, "little"), [0])
    w.bcast([0], raw)
    assert w.check() == 499


def test_global_memory_pool_backpressure(pcdn):
    """Limiter analogue (cdn-proto/src/connection/limiter/mod.rs:56-68): inbound bytes are admitted
    against a global budget and given back when their batch is released"""
    w = World(pcdn, global_memory_pool_size=10_000, max_conns=64)
    a = w.add_user(b"a" * 8, [0])
    raw = orc.broadcast_frame([0], b"x" * 3000)       # L = 3056
    for _ in range(3):
        w.e.handle_broadcast_message([0], raw)
    with pytest.raises(pcdn.PcdnError) as ei:
        w.e.handle_broadcast_message([0], raw)         # 4 x 3056 > 10 000
    assert ei.value.code == PCDN_EAGAIN               # the reference would await the semaphore
    assert w.e.stats().inflight_bytes == 3 * len(raw)
    assert w.e.next_batch() != 0 and w.e.stats().batches == 1   # the refusal launched the open batch (no flush yet)
    got = w.e.drain()                                  # poll + release → permits returned
    assert got[a] == [raw] * 3
    st = w.e.stats()
    assert st.inflight_bytes == 0 and st.released_batches == 1 and st.latency_ms_sum > 0
    w.e.handle_broadcast_message([0], raw)             # admitted again
    assert w.e.drain()[a] == [raw]
    with pytest.raises(pcdn.PcdnError) as ei:
        w.e.handle_broadcast_message([0], orc.broadcast_frame([0], b"y" * 20000))
    assert ei.value.code == -1                         # can never fit


def test_edge_cases(pcdn):
    """empty topic list (legal on the wire, routes to nobody — SURVEY App. B), zero-length raw through
    the ABI, 200 topics in one message, a 1.5 MB frame (94 staging chunks), 1-byte and 128-byte keys,
    broadcast whose only subscriber is a peer broker, empty batch"""
    w = World(pcdn, max_conns=512, ring_bytes_per_conn=4 << 20, max_batch_bytes=64 << 20, max_batch_deliveries=1 << 16)
    for i in range(100):
        w.add_user(bytes([i + 1]) * (1 if i % 2 else 128), list(range(i % 7, 200, 7)))
    w.add_broker("only/broker", [201])
    assert w.e.flush() == 0                                            # empty batch: nothing launched
    w.bcast([], orc.broadcast_frame([], b"to nobody"))
    w.bcast([3], b"")                                                  # zero-length raw is still a frame: header only
    w.bcast(list(range(200)), orc.broadcast_frame(list(range(200)), b"everyone once"))
    big = orc.broadcast_frame([5], bytes(range(256)) * 6000)           # 1.5 MB, 2 capnp segments
    w.bcast([5], big)
    w.bcast([201], orc.broadcast_frame([201], b"for the mesh"))
    w.bcast([201], orc.broadcast_frame([201], b"not for brokers"), True)
    w.direct(bytes([2]), orc.direct_frame(bytes([2]), b"one-byte key"))
    w.direct(bytes([3]) * 128, orc.direct_frame(bytes([3]) * 128, big[:70000]))
    n = w.check()
    assert n > 100


def test_concurrent_ingest_and_egress_threads(pcdn):
    """one host thread feeds frames (pcdn_user_receive + flush), another polls / reads / releases
    batches at the same time (the engine locks internally; pcdn_poll waits outside the lock).
    Per-connection delivery order must still be the order in which the frames were handed over."""
    import threading
    import time

    rng = random.Random(21)
    w = World(pcdn, max_conns=1024, ring_bytes_per_conn=1 << 20, batch_slots=4, max_batch_msgs=256)
    keys = [i.to_bytes(8, "little") for i in range(600)]
    for k in keys:
        w.add_user(k, [x for x in range(6) if rng.random() < 0.3])
    frames = []
    for j in range(3000):
        if rng.random() < 0.5:
            raw = orc.broadcast_frame([rng.randrange(6)], j.to_bytes(4, "little") * rng.randrange(1, 40))
        else:
            raw = orc.direct_frame(rng.choice(keys), j.to_bytes(4, "little") * rng.randrange(1, 40))
        frames.append((rng.choice(keys), raw))
        w.o.user_receive(frames[-1][0], raw)
    got, done, errs = {}, threading.Event(), []

    def consumer():
        try:
            while True:
                b = w.e.next_batch()
                if not b:
                    if done.is_set() and not w.e.next_batch():
                        return
                    time.sleep(0.0005)
                    continue
                res = w.e.poll(b)
                for conn, fr in w.e.collect_frames(res).items():
                    got.setdefault(conn, []).extend(fr)
                w.e.release_batch(b)
        except Exception as ex:  # pragma: no cover
            errs.append(ex)

    t = threading.Thread(target=consumer)
    t.start()
    for i, (sender, raw) in enumerate(frames):
        while True:
            rc = w.e.user_receive(sender, raw)
            if rc != PCDN_EAGAIN:  # all batch slots in flight — the consumer will free one
                break
            time.sleep(0.0002)
        assert rc == 0
        if i % 97 == 0:
            w.e.flush()
    w.e.flush()
    done.set()
    t.join(60)
    assert not errs and not t.is_alive()
    want = w.expect()
    assert set(got) == set(want)
    for c in want:
        assert got[c] == want[c], c


def test_connection_id_quarantined_until_batches_released(pcdn):
    """spans name connections by id: an id freed by a disconnect / kick must not be handed to another
    user while a batch launched before the removal is still unreleased (its records belong to the old
    socket — protocols/mod.rs:287-306 soft_close drains them, nobody else may receive them)"""
    e = pcdn.Engine(max_conns=8192, max_topics=256, max_keys=64, ring_bytes_per_conn=1 << 16, batch_slots=4)
    A, Bk, Ck = b"A" * 8, b"B" * 8, b"C" * 8
    a = e.add_user(A, [0])
    raw1 = orc.broadcast_frame([0], b"for A only")
    e.handle_broadcast_message([0], raw1)
    b1 = e.flush()
    e.remove_user(A)                       # A disconnects; batch b1 (unreleased) still names id `a`
    b = e.add_user(Bk, [0])
    assert b != a
    a2 = e.add_user(A, [0])                # A reconnects: also a fresh id
    assert a2 not in (a, b)
    k = e.add_user(A, [0])                 # double connect: kicks a2, which is quarantined too
    assert k not in (a, b, a2)
    raw2 = orc.broadcast_frame([0], b"second")
    e.handle_broadcast_message([0], raw2)
    b2 = e.flush()
    r1 = e.poll(b1)
    assert e.collect_frames(r1) == {a: [raw1]}
    r2 = e.poll(b2)
    assert e.collect_frames(r2) == {b: [raw2], k: [raw2]}
    e.release_batch(b1)
    e.release_batch(b2)
    c = e.add_user(Ck, [0])                # everything released: freed ids circulate again
    assert c in (a, a2)
    e.close()

    # a full table: the kick would need a second id while the first is still named by a live batch
    e = pcdn.Engine(max_conns=2, max_topics=256, max_keys=64, ring_bytes_per_conn=1 << 16, batch_slots=4)
    e.add_user(A, [0]); e.add_user(Bk, [0])
    e.handle_broadcast_message([0], raw1)
    b1 = e.flush()
    with pytest.raises(pcdn.PcdnError) as ei:
        e.add_user(A, [0])
    assert ei.value.code == PCDN_EAGAIN
    assert e.num_users()[0] == 2           # refused before the kick: A is still connected
    e.poll(b1); e.release_batch(b1)
    e.add_user(A, [0])                     # now the kick + re-add goes through
    assert e.num_users()[0] == 2
    e.close()


POOL_FLAGS = {"pool": 16, "pool-runs": 16 | 8}   # FLAG_OUTPUT_POOL, | FLAG_SPAN_RUNS


@pytest.mark.parametrize("staged,max_conns", [(False, 8192), (True, 8192), (False, 20000), (False, 65536), (False, 65537)] +
                         [(p, n) for n in (20000, 65536, 65537) for p in POOL_FLAGS])
def test_small_engine_batch_sizes_across_the_fused_limit(pcdn, staged, max_conns):
    """engines with <= 65536 connection slots route batches of <= 256 messages through the fused
    control kernel (k_ctrl_small: 1, 3 and 8 passes of 8192 connections here) and larger ones through
    the regular pipeline; all must agree with the oracle at and around the limit (1, 2, 255, 256, 257,
    700 messages; broadcasts, directs incl. a hot recipient and unknown keys).  65537 slots is the
    first geometry that always takes the regular pipeline with the staged span table.
    staged = "pool" / "pool-runs": output-pool engines (plain / run-length span table), whose regular
    pipeline finishes the pool offsets in k_pool_finish with one CTA per 8192 slots: 3, 8 and 9 CTAs here."""
    rng = random.Random(11)
    kw = dict(flags=POOL_FLAGS[staged], pool_bytes=1 << 28) if isinstance(staged, str) else \
        dict(flags=pcdn.FLAG_STAGED_SPANS if staged else 0)
    w = World(pcdn, ring_bytes_per_conn=1 << 18, max_batch_msgs=1024, max_batch_bcast=1024, max_conns=max_conns,
              max_keys=max(16384, max_conns + 2048), **kw)
    # connection ids are handed out densely: with the bulk loader the later 8192-connection blocks of a
    # large engine get users too (topic 9 only, so they stay out of the checked traffic)
    if max_conns > 8192:
        n_fill = max_conns - 2000
        fill = np.zeros((n_fill, 8), dtype=np.uint8)
        fill[:, :4] = np.arange(n_fill, dtype=np.uint32).view(np.uint8).reshape(n_fill, 4)
        fill[:, 7] = 0xEE
        conns = w.e.add_users_bulk(fill, 8, np.full(n_fill, 9, dtype=np.uint16), np.arange(n_fill + 1, dtype=np.uint32))
        for i in range(0, n_fill, max(1, n_fill // 40)):   # ... except a sample, known to the oracle, that also takes topic 8
            k = fill[i].tobytes()
            w.e.subscribe_user_to(k, [8])
            w.map[int(conns[i])] = w.o.add_user(k, [9, 8])
    keys = [rng.getrandbits(64).to_bytes(8, "little") * 4 for _ in range(700)]
    for k in keys:
        w.add_user(k, [t for t in range(8) if rng.random() < (0.5 if t == 0 else 0.05)])
    w.add_broker("p/q", [0, 3])
    hot = keys[5]
    for n in (1, 2, 255, 256, 257, 700, 3):
        for j in range(n):
            r = rng.random()
            if r < 0.4:
                t = [rng.randrange(9)] + ([0] if rng.random() < 0.3 else [])
                w.bcast(t, orc.broadcast_frame(t, payload(rng, rng.choice([0, 5, 300, 1500]))), rng.random() < 0.2)
            else:
                rc = hot if r < 0.6 else rng.choice(keys) if r < 0.9 else b"nobody-home"
                w.direct(rc, orc.direct_frame(rc, j.to_bytes(4, "little") * rng.randrange(1, 40)))
        assert w.check() > 0
