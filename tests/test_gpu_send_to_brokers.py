"""pcdn_send_to_broker / pcdn_send_to_brokers on the GPU: the broker's own frames (the UserSync and TopicSync
messages of cdn-broker/src/tasks/broker/sync.rs) go to one peer broker or to every peer broker as one message
of the open batch, in order with the routed traffic of the same link.  Every connection's stream is compared
frame for frame with the oracle's, which sends them through try_send_to_broker(s) (tasks/broker/sender.rs:17-59,
restated in gpu_world.py and tested in test_send_to_brokers_host.py), on every span layout, both control paths, shards, device parse,
in-batch subscription events, shared payload, a by-reference threshold, the output pool's refusal and retry, and
the egress writer."""
import random

import pytest

from gpu_world import (BIG, PCDN_EAGAIN, PCDN_ENOSPC, STATUS_EAGAIN, PoolWorld, Reader, Sends, World, flush_until_done,
                       layout, payload, shard_cfg, sock_pair, user_sync, wire)
from kconst import K
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

# (layout, delivery) under this file's test ids
LAYOUTS = [pytest.param(n, "copy", id=n) for n in ("rings", "staged", "runs", "host", "pool", "shards-host", "shards-nccl")] + \
          [pytest.param("rings", "shared", id="shared"), pytest.param("rings", ("ref", 2048), id="ref")]


class SendWorld(Sends, World):
    pass


class SendPoolWorld(Sends, PoolWorld):
    pass


def topic_sync(tag, n=40):
    return orc.serialize(orc.KIND_TOPIC_SYNC, b"", bytes([tag % 256, 0xAB]) * n)


def populate(w, n_users=200, remote=8):
    """users on topics 0..3, `remote` users owned by peer broker B"""
    for i in range(n_users):
        w.add_user(b"user-%05d" % i, [i % 4])
    w.add_broker("b/b")
    w.add_broker("c/c", [2])
    w.both("apply_user_sync", "b/b", [(b"remote-%02d" % i, 1, "b/b") for i in range(remote)])


def connect_flow(w, rng, across, users_only, tag=0):
    """the reference's connect flow (tasks/broker/handler.rs:95-120): add_broker(B), a full topic sync and a
    full user sync to B, then routed broadcasts and directs that reach B (subscribed; owner of remote users)"""
    w.add_broker("n/n", [1])
    w.both("apply_user_sync", "n/n", [(b"far-%02d" % i, 1, "n/n") for i in range(4)])
    assert w.send("n/n", topic_sync(tag)) == 0
    if across:
        w.e.flush()
    if users_only:
        w.bcast([1], orc.broadcast_frame([1], payload(rng, 900)), True)
    assert w.send("n/n", user_sync(tag, 5000)) == 0
    for j in range(12):
        t = [j % 4]
        w.bcast(t, orc.broadcast_frame(t, payload(rng, rng.randint(1, 3000))), users_only and j % 3 == 0)
        if j % 4 == 1:
            w.direct(b"far-%02d" % (j % 4), orc.direct_frame(b"far-%02d" % (j % 4), payload(rng, 200)))
        if across and j % 5 == 4:
            w.e.flush()
    assert w.send(None, topic_sync(tag + 1, 3)) == 0     # the partial syncs of run_sync_task (sync.rs:129-143)
    assert w.send(None, user_sync(tag + 1, 64)) == 0


@pytest.mark.parametrize("flow", ["one-batch", "across", "users-only"])
@pytest.mark.parametrize("name,delivery", LAYOUTS)
def test_connect_flow(pcdn, request, name, delivery, flow):
    cfg = layout(pcdn, name)
    if name == "pool":
        cfg["pool_bytes"] = 256 << 20
    w = SendWorld(pcdn, max_conns=1024, delivery=delivery, **cfg)
    rng = random.Random(request.node.callspec.id)          # seeded by the test id, "<layout>-<flow>"
    populate(w)
    connect_flow(w, rng, flow == "across", flow == "users-only")
    assert w.check() > 0
    assert w.e.last_result.n_overflow == 0
    w.e.close()


@pytest.mark.parametrize("control", ["fused", "fused-full", "regular-conns", "regular-msgs"])
def test_control_paths(pcdn, control):
    """fused k_ctrl_small; the same with kSmallCtrlItems (broadcast, 8192-connection block) match items, one per
    warp of the kernel, and in-batch subscription events of users on both match blocks and of a broker between
    the sends; k_match on an engine with more than kSmallCtrlConns slots; k_match for a batch of more than
    kSmallCtrlMsgs messages"""
    block = K.kBlockWords * 32
    cfg = dict(max_conns=1024)
    if control == "regular-conns":
        cfg = dict(max_conns=K.kSmallCtrlConns * 2, ring_bytes_per_conn=1 << 14, max_keys=1 << 17)
    if control == "fused-full":
        cfg = dict(max_conns=2 * block, ring_bytes_per_conn=1 << 17, flags=pcdn.FLAG_INBATCH_SUBSCRIBE)
    w = SendWorld(pcdn, **cfg)
    rng = random.Random(3)
    n_users = block + 200 if control == "fused-full" else 200
    populate(w, n_users)
    n = K.kSmallCtrlMsgs + 20 if control == "regular-msgs" else 30
    if control == "fused-full":
        nblk = -(-w.e.shard_info(0).shard_stride // block)
        assert nblk == 2
        n = K.kSmallCtrlItems // nblk
    edges = [0, 31, 32, block - 1, block, block + 1, n_users - 1]
    b0 = w.e.stats().batches
    for j in range(n):
        if control == "fused-full" and j % 5 == 2:
            sub = j % 2
            w.both("subscribe_user_to" if sub else "unsubscribe_user_from", b"user-%05d" % edges[j % len(edges)], [(j + 1) % 4])
            w.both("subscribe_broker_to" if sub else "unsubscribe_broker_from", "b/b", [j % 4])
        if j % 7 == 3:
            assert w.send("b/b" if j % 2 else None, user_sync(j, rng.randint(1, 2000))) == 0
        else:
            w.bcast([j % 4], orc.broadcast_frame([j % 4], payload(rng, rng.randint(1, 600))))
    assert w.check() > 0
    if control == "fused-full":
        assert w.e.stats().batches == b0 + 1
    w.e.close()


def test_recipients_and_nothing_to_send_to(pcdn):
    """every connected broker, subscribed or not; no user, however subscribed; 1 and nothing appended when
    the identifier is unknown or no broker is connected"""
    w = SendWorld(pcdn, max_conns=1024)
    users = [w.add_user(b"all-%03d" % i, list(range(8))) for i in range(50)]
    assert w.send(None, user_sync(1)) == 1
    assert w.send("b/b", user_sync(1)) == 1
    assert w.e.flush() == 0 and w.e.stats().msgs == 0
    brokers = [w.add_broker("p%d/p" % i) for i in range(5)]
    assert w.send(None, user_sync(2)) == 0
    assert w.send("nobody/x", user_sync(3)) == 1
    msgs = w.e.stats().msgs
    w.check()
    got = w.e.last_result
    assert got.n_msgs == 1 and got.n_deliveries == len(brokers)
    assert w.e.stats().msgs == msgs + 1
    assert not any(w.o.frames(w.map[u]) for u in users)
    w.e.close()


def test_r12_add_remove_kick_after_the_send(pcdn):
    """the recipients are the brokers connected at the call: a broker added after it gets nothing, a removed
    one still gets it (and its id stays quarantined until the batch is released), a kicked one keeps it"""
    w = SendWorld(pcdn, max_conns=64)
    a = w.add_broker("a/a")
    r = w.add_broker("r/r")
    k = w.add_broker("k/k")
    assert w.send(None, user_sync(1)) == 0
    assert w.send("k/k", topic_sync(1)) == 0
    late = w.add_broker("late/x")
    w.both("remove_broker", "r/r")
    k2 = w.add_broker("k/k")
    assert k2 != k
    assert w.send("k/k", topic_sync(2)) == 0
    fresh = [w.add_user(b"fresh-%02d" % i, [0]) for i in range(3)]
    assert r not in fresh                                # quarantined while a batch naming it is in flight
    got = w.e.drain()
    want = w.expect()
    w.compare(w.e, got, want)
    assert want[r] == [user_sync(1)] and want[k] == [user_sync(1), topic_sync(1)] and want[k2] == [topic_sync(2)]
    assert late not in want and want[a] == [user_sync(1)]
    w.e.close()


@pytest.mark.parametrize("control", ["fused", "regular"])
def test_pool_retry_delivers_to_the_set_at_launch(pcdn, control):
    """a refused batch holding sends; between the refusal and the retry one broker is removed and another
    added: the retried batch delivers to the brokers connected when it was launched"""
    w = SendPoolWorld(pcdn, "one-shard", pcdn.FLAG_STAGED_SPANS if control == "regular" else 0)
    w.add_broker("r/s", [])
    b0 = w.fill_hot()
    assert w.send(None, user_sync(7, 20000)) == 0
    assert w.send("r/s", topic_sync(7)) == 0
    b1 = w.traffic(1, (w.keys[0],))
    assert w.e.poll(b0).status == 0 and w.e.poll(b1).status == STATUS_EAGAIN
    w.both("remove_broker", "p/q")
    w.add_broker("t/u", [0])
    got = {}
    w.consume(b0, got)
    w.consume(b1, got, retry=True)
    assert w.compare(w.e, got, w.expect()) > 0
    w.e.close()


def test_device_parse_and_inbatch_events(pcdn):
    """device-parse frames and sends in one batch; in-batch broker subscribe / unsubscribe events before and
    after a send change nothing for it: a broker that left all its topics in-batch still gets the frame"""
    w = SendWorld(pcdn, max_conns=1024, flags=pcdn.FLAG_DEVICE_PARSE | pcdn.FLAG_INBATCH_SUBSCRIBE, n_valid_topics=8)
    rng = random.Random(5)
    for i in range(100):
        w.add_user(b"user-%05d" % i, [i % 4])
    w.add_broker("b/b", [0, 1])
    w.add_broker("c/c")
    sender = b"user-00001"
    for j in range(40):
        if j == 10:
            w.both("unsubscribe_broker_from", "b/b", [0, 1])
        if j == 20:
            w.both("subscribe_broker_to", "c/c", [2])
        if j % 6 == 5:
            assert w.send(None if j % 12 == 5 else "b/b", user_sync(j, rng.randint(1, 3000))) == 0
        t = [j % 4]
        raw = orc.broadcast_frame(t, payload(rng, rng.randint(1, 1500)))
        assert w.e.user_receive(sender, raw) == 0 and w.o.user_receive(sender, raw) == 0
    w.check()
    assert w.e.stats().batches == 1
    w.e.close()


@pytest.mark.parametrize("n_brokers", [1, K.kFatMin - 1, K.kFatMin, K.kFatMin + 1, "dense"])
@pytest.mark.parametrize("raw_len", [100, K.kCmMaxBytes - 4, K.kCmMaxBytes - 3, 20000])
def test_broker_counts_and_lengths(pcdn, n_brokers, raw_len):
    """thin (< kFatMin recipients), message-major, and connection-major when brokers >= N/16 (records up to
    kCmMaxBytes); raw lengths on both sides of kCmMaxBytes"""
    n_conns = 512
    nb = 2 * (n_conns >> K.kCmDenseShift) if n_brokers == "dense" else n_brokers
    w = SendWorld(pcdn, max_conns=n_conns)
    for i in range(nb):
        w.add_broker("b%03d/x" % i, [i % 2])
    for i in range(20):
        w.add_user(b"u%03d" % i, [0])
    raw = user_sync(1, raw_len)[:raw_len]
    for j in range(3):
        w.bcast([j % 2], orc.broadcast_frame([j % 2], b"x" * (50 + j)))
        assert w.send(None, raw) == 0
    assert w.send("b000/x", raw[::-1]) == 0
    assert w.check() >= 3 * nb + 1
    w.e.close()


def test_overflow_in_copy_mode(pcdn):
    """a frame larger than one broker's free ring space: that broker is reported in overflow_conns, as for
    a routed message of that size"""
    e = pcdn.Engine(max_conns=64, ring_bytes_per_conn=1 << 16)
    b = e.add_broker("b/b")
    c = e.add_broker("c/c")
    e.subscribe_broker_to("c/c", [0])
    e.handle_broadcast_message([0], b"y" * 60000)     # c's ring is nearly full
    assert e.send_to_brokers(b"s" * 20000) == 0
    bid = e.flush()
    r = e.poll(bid)
    assert r.status == 0 and r.n_overflow == 1 and r.overflow_conns[0] == c
    assert e.collect_frames(r)[b] == [b"s" * 20000]
    e.release_batch(bid)
    e.close()


def test_by_reference_threshold(pcdn):
    """ref_min_bytes = T: a sync frame >= T and larger than a ring is delivered by reference without an
    overflow, one below T is framed"""
    w = SendWorld(pcdn, max_conns=64, ring_bytes_per_conn=1 << 16, delivery=("ref", 4096))
    w.add_broker("b/b")
    w.add_user(b"u", [0])
    assert w.send(None, user_sync(1, 200_000)) == 0
    assert w.send("b/b", topic_sync(1, 1000)) == 0
    w.bcast([0], orc.broadcast_frame([0], b"z" * 10))
    w.check()
    assert w.e.last_result.n_overflow == 0
    w.e.close()


def test_counters_and_memory_pool(pcdn):
    """msgs, deliveries and bytes_out count the sends; bytes_in and inflight_bytes do not; a send is accepted
    while a routed frame gets PCDN_EAGAIN from the memory pool"""
    w = SendWorld(pcdn, max_conns=64, global_memory_pool_size=10_000)
    w.add_broker("b/b")
    w.add_broker("c/c", [0])
    w.add_user(b"u", [0])
    routed = orc.broadcast_frame([0], b"r" * 9000)
    w.bcast([0], routed)
    with pytest.raises(pcdn.PcdnError) as ei:
        w.e.handle_broadcast_message([0], routed)
    assert ei.value.code == PCDN_EAGAIN
    s = w.send(None, user_sync(1, 30_000))            # larger than the whole pool: no permits taken
    assert s == 0
    st = w.e.stats()
    assert st.bytes_in == len(routed) and st.inflight_bytes == len(routed)
    w.check()
    st = w.e.stats()
    assert st.msgs == 2 and st.deliveries == 2 + 2
    assert st.bytes_out == 2 * (len(routed) + 4) + 2 * (len(user_sync(1, 30_000)) + 4)
    w.e.close()


def test_full_batch_and_too_large(pcdn):
    """a full max_batch_bcast: the send opens the next batch, order kept; raw_len > max_batch_bytes: PCDN_ENOSPC
    and nothing appended"""
    w = SendWorld(pcdn, max_conns=64, max_batch_bcast=4, max_batch_bytes=1 << 16)
    w.add_broker("b/b", [0])
    for j in range(4):
        w.bcast([0], orc.broadcast_frame([0], bytes([j]) * 100))
    assert w.send("b/b", topic_sync(1)) == 0
    assert w.e.stats().batches == 1
    with pytest.raises(pcdn.PcdnError) as ei:
        w.e.send_to_brokers(b"q" * (1 << 16))
    assert ei.value.code == PCDN_ENOSPC
    w.check()
    assert w.e.stats().msgs == 5 and w.e.stats().batches == 2
    w.e.close()


def test_launches_match_broadcasts(pcdn):
    """a batch with sends launches as many kernels as the same batch with each send replaced by a broadcast"""
    counts = []
    for sends in (True, False):
        e = pcdn.Engine(max_conns=1024)
        for i in range(40):
            e.add_broker("b%02d/x" % i)
            e.subscribe_broker_to("b%02d/x" % i, [0])
        for j in range(10):
            raw = user_sync(j, 500)
            if sends and j % 3 == 0:
                assert e.send_to_brokers(raw) == 0
            else:
                e.handle_broadcast_message([0], raw)
        k0 = e.stats().kernel_launches
        e.drain()
        counts.append(e.stats().kernel_launches - k0)
        e.close()
    assert counts[0] == counts[1]


@pytest.mark.parametrize("mode", ["rings", "shards-host"])
def test_egress_backlog_stalled_broker_and_soft_close(pcdn, mode):
    """egress to socketpairs attached to broker connections, one broker stalled behind a 4 KiB send buffer so
    it takes a backlog; after flush_backlog every stream equals the oracle's.  soft_close of a broker right
    after a send delivers it"""
    cfg = dict(max_conns=1024, ring_bytes_per_conn=1 << 20, max_batch_bytes=8 << 20, batch_slots=2)
    if mode == "shards-host":
        cfg.update(shard_cfg(pcdn, mode))
    w = SendWorld(pcdn, **cfg)
    eg = pcdn.Egress(w.e, n_threads=4, backlog_bytes_per_conn=BIG)
    rng = random.Random(9)
    names = ["s%d/x" % i for i in range(3)]
    conns = [w.add_broker(n, [0]) for n in names]
    pairs = [sock_pair(4096 if i == 0 else 1 << 20) for i in range(3)]
    for c, (s, _) in zip(conns, pairs):
        eg.attach(c, s.fileno())
    readers = [Reader(r.fileno(), started=i != 0) for i, (_, r) in enumerate(pairs)]
    want = {}
    for k in range(4):
        for j in range(6):
            w.bcast([0], orc.broadcast_frame([0], payload(rng, rng.randint(1, 30000))))
            if j % 2:
                assert w.send(None if j % 3 else names[k % 3], user_sync(k * 10 + j, rng.randint(1, 40000))) == 0
        b = w.e.flush()
        eg.write_batch(b)
        w.e.release_batch(b)
        for c, fr in w.expect().items():
            want.setdefault(c, bytearray()).extend(wire(fr))
    assert readers[1].wait_for(len(want[conns[1]]), eg) == bytes(want[conns[1]])
    readers[0].go()
    assert flush_until_done(eg) == 0
    assert readers[0].wait_for(len(want[conns[0]])) == bytes(want[conns[0]])
    # soft close right after a send (the frame is still in the open batch): it reaches the peer
    assert w.send(names[2], user_sync(99, 777)) == 0
    w.bcast([0], orc.broadcast_frame([0], b"after"))
    assert eg.soft_close(conns[2]) == pairs[2][0].fileno()
    for c, fr in w.expect().items():
        want[c].extend(wire(fr))
    assert eg.backlog() == ([], 0) and eg.failed() == []
    pairs[2][0].close()
    assert readers[2].finish() == bytes(want[conns[2]])
    assert readers[1].wait_for(len(want[conns[1]])) == bytes(want[conns[1]])
    assert readers[0].wait_for(len(want[conns[0]])) == bytes(want[conns[0]])
    for s, _ in pairs[:2]:
        s.close()
    for r in readers:
        r.finish()
    for _, r in pairs:
        r.close()
    eg.close()
    w.e.close()
