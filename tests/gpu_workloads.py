"""Workload bodies that more than one GPU test module runs (not a test module: nothing here is collected).  Each
takes the engine layout or mode its home test is parametrized over, `delivery` ("copy", "shared" or ("ref", T),
see gpu_world.engine) and, where the write-set guard runs it, `world` (the World class to build).  The tests that
run them are named in each docstring's first line.

Assertions here carry explicit messages: pytest rewrites `assert` only in test modules."""
import os
import random
import socket
import threading
import time

import pytest

from gpu_world import (PCDN_EAGAIN, STATUS_EAGAIN, IDLE_LIMIT, BIG, CM_DENSE, PoolWorld, Reader, World,
                       backlog_world, chunk_streams, cm_frame, cm_world, engine, flush_until_done, layout, payload,
                       shard_cfg, sock_pair, wire)
from kconst import K
from oracle import oracle as orc


# ------------------------------------------------------------------ test_gpu_parity.py
# the layouts of the randomized mixed workload, under the ids its tests have always had
MIXED_LAYOUTS = [pytest.param("rings", id="0"), "staged", "runs", "runs-staged", "pool", "pool-staged-runs", "pool-host",
                 pytest.param("pool-shards-host", id="pool-shards"), pytest.param("pool-runs-shards-nccl", id="pool-shards-nccl"),
                 pytest.param("pool-shards-host-staged", id="pool-shards-staged"), "host", "shards-host", "shards-host-staged",
                 "shards-nccl"]


def random_mixed_batches(pcdn, seed, name, delivery="copy", world=World):
    """test_random_mixed_batches on layout `name` → the world"""
    rng = random.Random(seed)
    kw = layout(pcdn, name)
    if name.startswith("pool"):
        # PCDN_FLAG_OUTPUT_POOL: one shared output pool (1 GiB; a batch here delivers a few hundred MB)
        # instead of per-connection rings
        kw["pool_bytes"] = 1 << 30
    else:
        kw["ring_bytes_per_conn"] = 1 << 20
    if "devices" in kw:
        kw["max_conns"] = 1024
    if name == "host":
        kw["max_conns"] = 2048
    w = world(pcdn, delivery=delivery, **kw)
    if name == "host":
        assert w.e.host_rings() != 0, "host rings are not in host memory"
    if "devices" in kw:
        assert w.e.num_shards()[0] >= 2, w.e.num_shards()
    keys = []
    for i in range(1500):
        k = rng.getrandbits(64).to_bytes(8, "little") * rng.choice([1, 4, 16])
        keys.append(k)
        # topic 0 is popular (fat path), topics 10+ are rare (thin path)
        t = [x for x in range(16) if rng.random() < (0.6 if x == 0 else 0.1 if x < 10 else 0.004)]
        w.add_user(k, t)
    for b in range(3):
        w.add_broker(f"b{b}/p{b}", [rng.randrange(16) for _ in range(3)])
    remote = [b"remote%d" % i for i in range(8)]
    w.both("apply_user_sync", "b1/p1", [(k, 1, "b1/p1") for k in remote])
    total = 0
    for batch in range(4):
        for j in range(rng.randrange(20, 120)):
            r = rng.random()
            size = rng.choice([0, 1, 11, 12, 13, 100, 1024, 4096, 16000, 16384, 20000, 40000]) if rng.random() < 0.5 \
                else rng.randrange(0, 3000)
            if r < 0.55:
                topics = [rng.randrange(16) for _ in range(rng.randrange(1, 4))]
                if rng.random() < 0.4:
                    topics.append(0)
                w.bcast(topics, orc.broadcast_frame([t for t in topics], payload(rng, size)), rng.random() < 0.3)
            else:
                rc = rng.choice(keys) if rng.random() < 0.7 else rng.choice(remote + [b"nobody", b""])
                w.direct(rc, orc.direct_frame(rc, payload(rng, size)), rng.random() < 0.3)
        if batch == 2:  # state change between batches
            for k in rng.sample(keys, 50):
                w.both("remove_user", k)
            for k in rng.sample(keys, 50):
                w.both("subscribe_user_to", k, [rng.randrange(16)])
        total += w.check()
    assert total > 1000, total
    return w


def direct_hot_recipient_keeps_order(pcdn, delivery="copy"):
    """test_direct_hot_recipient_keeps_order"""
    rng = random.Random(7)
    w = World(pcdn, max_conns=20480, max_keys=65536, max_batch_msgs=8192, ring_bytes_per_conn=1 << 20,
              max_batch_bytes=8 << 20, delivery=delivery)
    keys = [rng.getrandbits(128).to_bytes(16, "little") * 8 for _ in range(20000)]  # 128-byte keys
    for k in keys:
        w.add_user(k, [0] if rng.random() < 0.001 else [])
    leader = keys[123]
    for j in range(6000):
        r = rng.random()
        if r < 0.5:
            rc = leader
        elif r < 0.9:
            rc = rng.choice(keys)
        else:
            rc = rng.getrandbits(128).to_bytes(16, "little") * 8  # unknown: dropped
        w.direct(rc, orc.direct_frame(rc, j.to_bytes(4, "little") * rng.randrange(1, 30)))
        if j % 500 == 0:
            w.bcast([0], orc.broadcast_frame([0], b"tick%d" % j))
    n = w.check()
    assert n > 5000, n
    assert w.e.last_result.n_direct_dropped > 300, w.e.last_result.n_direct_dropped


# ------------------------------------------------------------------ test_gpu_device_parse.py
def _mutate(rng, raw):
    raw = bytearray(raw)
    for _ in range(rng.randrange(1, 3)):
        raw[rng.randrange(8, min(len(raw), 56))] = rng.randrange(256)
    return bytes(raw)


def frames_through_receive_loops(pcdn, seed, delivery="copy"):
    """test_frames_through_receive_loops"""
    rng = random.Random(seed)
    # seed 2 also forces the large-engine span path (span table staged in HBM, copied out during the pack)
    w = World(pcdn, n_valid_topics=12, flags=pcdn.FLAG_DEVICE_PARSE | (pcdn.FLAG_STAGED_SPANS if seed == 2 else 0),
              ring_bytes_per_conn=1 << 20, delivery=delivery)
    keys = []
    for i in range(1200):
        k = rng.getrandbits(64).to_bytes(8, "little") * rng.choice([1, 4, 16])
        keys.append(k)
        w.add_user(k, [x for x in range(12) if rng.random() < (0.5 if x == 0 else 0.08)])
    w.add_broker("b0/p0", [0, 3])
    w.both("apply_user_sync", "b0/p0", [(b"far-away", 1, "b0/p0")])
    total_err = 0
    for batch in range(3):
        frames, want_rc = [], []
        for j in range(rng.randrange(60, 160)):
            size = rng.choice([0, 5, 100, 1000, 9000, 20000]) if rng.random() < 0.4 else rng.randrange(0, 2000)
            pl = bytes([j & 0xFF]) * size
            r = rng.random()
            if r < 0.5:
                topics = [rng.randrange(16) for _ in range(rng.randrange(1, 5))]      # 12..15 are invalid
                if rng.random() < 0.3:
                    topics = [topics[0]] * 2 + topics                                    # consecutive duplicates
                raw = orc.broadcast_frame(topics, pl)
            elif r < 0.9:
                rc = rng.choice(keys) if rng.random() < 0.8 else rng.choice([b"far-away", b"nobody", b""])
                raw = orc.direct_frame(rc, pl)
            else:
                raw = orc.broadcast_frame([rng.randrange(12, 200)] * rng.randrange(1, 3), pl)  # only invalid topics
            if rng.random() < 0.15:
                raw = _mutate(rng, raw)
            origin = 1 if rng.random() < 0.25 else 0
            sender = rng.choice(keys)
            frames.append((sender, origin, raw))
            want_rc.append(w.o.broker_receive(raw) if origin else w.o.user_receive(sender, raw))
        # mutated frames may decode as Subscribe/Unsubscribe: those change state on both sides alike
        rcs = w.e.receive_frames(frames)
        got = w.e.drain()
        res = w.e.last_result
        # per-frame outcome: synchronous code, or (device-parsed kinds) the batch's msg_status
        deferred = [i for i, (rc, wrc) in enumerate(zip(rcs, want_rc)) if rc != wrc]
        n_err_want = sum(1 for i in deferred if want_rc[i] < 0)
        assert all(rcs[i] == 0 and want_rc[i] in (-7, -8) for i in deferred), [(rcs[i], want_rc[i]) for i in deferred][:5]
        assert res.n_msg_errors == n_err_want, (res.n_msg_errors, n_err_want)
        total_err += n_err_want
        want = w.expect()
        assert set(got) == set(want), sorted(set(got) ^ set(want))[:10]
        for c in want:
            assert got[c] == want[c], c
    assert total_err > 5, total_err


def msg_status_codes(pcdn, staged, delivery="copy"):
    """test_msg_status_codes"""
    w = World(pcdn, n_valid_topics=2, flags=pcdn.FLAG_DEVICE_PARSE | (pcdn.FLAG_STAGED_SPANS if staged else 0),
              delivery=delivery)
    a = w.add_user(b"a" * 8, [0, 1])
    good = orc.broadcast_frame([0], b"ok")
    bad_topics = orc.broadcast_frame([9, 9, 7], b"nope")
    broken = bytearray(orc.direct_frame(b"a" * 8, b"x" * 64)); broken[36:40] = (0xFFFFFFF).to_bytes(4, "little")  # recipient list beyond the segment
    rcs = w.e.receive_frames([(b"a" * 8, 0, good), (b"a" * 8, 0, bad_topics), (b"a" * 8, 0, bytes(broken)),
                              (b"a" * 8, 1, bad_topics)])
    assert rcs == [0, 0, 0, 0], rcs
    got = w.e.drain()
    res = w.e.last_result
    st = [res.msg_status[i] for i in range(res.n_msgs)]
    assert st == [0, -8, -7, 0], st        # broker-origin topics are not pruned (handler.rs:157): no error, no recipients
    assert res.n_msg_errors == 2 and got[a] == [good], (res.n_msg_errors, got.get(a))


# ------------------------------------------------------------------ test_gpu_pool_retry.py
def retry_routes_as_launched(pcdn, layout, control, runs, delivery="copy"):
    """test_retry_routes_as_launched (layout: "one-shard" or "shards-host")"""
    flags = (pcdn.FLAG_STAGED_SPANS if control == "regular" else 0) | (pcdn.FLAG_SPAN_RUNS if runs else 0)
    w = PoolWorld(pcdn, layout, flags, delivery=delivery)
    t0, t1 = w.on_shard(w.home, 0), w.on_shard(w.home, 1)
    unsub, removed, moved = t0[0], t0[1], t1[0]
    kicked, newcomer = t1[1], b"newcomer"
    directs = (unsub, removed, kicked, moved, newcomer)
    b0 = w.fill_hot()
    b1 = w.traffic(1, directs)
    assert w.e.poll(b0).status == 0, "the batch that fills the pool is refused"
    st1 = w.statuses(b1)
    assert st1[w.home] == STATUS_EAGAIN and w.e.poll(b1).status == STATUS_EAGAIN, st1
    w.add_user(newcomer, [0])
    w.both("unsubscribe_user_from", unsub, [0])
    w.both("remove_user", removed)
    w.add_user(kicked, [0])                                   # same key, new connection: the old one is kicked
    w.both("apply_user_sync", "p/q", [(moved, 1000, "p/q")])  # the peer now owns this user
    w.both("subscribe_broker_to", "p/q", [1])
    b2 = w.traffic(2, directs)
    assert w.statuses(b2)[w.home] == STATUS_EAGAIN, w.statuses(b2)   # queued behind the refused batch
    got = {}
    w.consume(b0, got)
    w.consume(b1, got, retry=True)
    w.consume(b2, got, retry=True)
    n = w.compare(w.e, got, w.expect())
    assert n > 2 * 3 * 290, n
    w.e.close()


def reconnect_onto(w, key, target, fillers):
    """reconnect `key` (the kick frees its old connection first) so that the new connection lands on
    shard `target`: ids go to the least-loaded shard, so idle filler users leave `target` until it is"""
    loads = [w.e.shard_info(i).n_conns for i in range(w.nl)]
    loads[w.shard_of(key)] -= 1
    while min(l for i, l in enumerate(loads) if i != target) <= loads[target]:
        w.both("remove_user", fillers[target].pop())
        loads[target] -= 1
    old = w.conn[key]
    new = w.add_user(key, [0])
    assert new // w.stride == target and old // w.stride != target, (old, new)


def partial_refusal_across_shards(pcdn, delivery="copy"):
    """test_partial_refusal_across_shards"""
    w = PoolWorld(pcdn, "shards-host", delivery=delivery)
    assert w.nl == 3, w.nl
    fillers = {s: [] for s in range(w.nl)}
    for i in range(30):
        k = b"filler-%02d" % i
        w.add_user(k, [])
        fillers[w.shard_of(k)].append(k)
    accept = (w.home + 1) % w.nl
    x, y = w.on_shard(accept)[0], w.on_shard(w.home)[0]      # x: accepting shard -> home; y: home -> accepting
    b0 = w.fill_hot()
    for j in range(3):
        w.direct(x, orc.direct_frame(x, b"to x, %d" % j))
        w.direct(y, orc.direct_frame(y, b"to y, %d" % j))
    b1 = w.traffic(1)
    assert w.e.poll(b0).status == 0, "the batch that fills the pool is refused"
    want_st = [STATUS_EAGAIN if s == w.home else 0 for s in range(w.nl)]
    assert w.statuses(b1) == want_st, (w.statuses(b1), want_st)
    assert w.e.poll(b1).status == STATUS_EAGAIN, w.e.poll(b1).status   # the combined result: "retry" wins
    reconnect_onto(w, x, w.home, fillers)
    reconnect_onto(w, y, accept, fillers)
    b2 = w.traffic(2, (x, y))                                 # the new connections, after the moves
    got = {}
    w.consume(b0, got)
    w.e.retry_batch(b1)
    assert w.statuses(b1) == [0] * w.nl, w.statuses(b1)
    w.consume(b1, got)
    w.consume(b2, got, retry=True)
    frames = [f for fr in got.values() for f in fr]
    copies = {(who, j): frames.count(orc.direct_frame(k, b"to %s, %d" % (who, j)))
              for who, k in ((b"x", x), (b"y", y)) for j in range(3)}
    assert copies == {wj: 1 for wj in copies}, copies
    w.compare(w.e, got, w.expect())
    w.e.close()


def _fd_bytes(fd):
    os.lseek(fd, 0, os.SEEK_SET)
    return os.read(fd, os.fstat(fd).st_size + 16)


def egress_refused_shard_is_written_once(pcdn, how, delivery="copy"):
    """test_egress_refused_shard_is_written_once (its "drain" sink walks framed records only)"""
    w = PoolWorld(pcdn, "shards-host", delivery=delivery)
    eg = pcdn.Egress(w.e, n_threads=4)
    fds = {}
    if how != "drain":
        for c in w.map:                                       # every user and the peer broker
            fds[c] = os.memfd_create("conn%d" % c)
            eg.attach(c, fds[c])
    b0 = w.fill_hot()
    b1 = w.traffic(1, w.keys[::37])
    assert w.statuses(b1) == [STATUS_EAGAIN if s == w.home else 0 for s in range(w.nl)], w.statuses(b1)
    if how == "drain":
        got = {}
        eg.drain(b0, lambda ch: chunk_streams(ch, got))
        calls = []
        with pytest.raises(pcdn.PcdnError) as ei:
            eg.drain(b1, lambda ch: calls.append(ch.n_spans))
        assert ei.value.code == PCDN_EAGAIN and calls == [], (ei.value.code, calls)
        w.e.release_batch(b0)
        w.e.retry_batch(b1)
        eg.drain(b1, lambda ch: chunk_streams(ch, got))
        w.e.release_batch(b1)
        streams = {c: bytes(v) for c, v in got.items()}
    else:
        if how == "write_batch":
            eg.write_batch(b0)
            before = {c: _fd_bytes(fd) for c, fd in fds.items()}
            with pytest.raises(pcdn.PcdnError) as ei:
                eg.write_batch(b1)
            assert ei.value.code == PCDN_EAGAIN, ei.value.code
            assert {c: _fd_bytes(fd) for c, fd in fds.items()} == before, "a refused batch reached a descriptor"
            w.e.release_batch(b0)
            w.e.retry_batch(b1)
            eg.write_batch(b1)
            w.e.release_batch(b1)
        else:
            eg.soft_close(w.conn[w.keys[3]])                  # writes and releases b0, then b1 (retried)
            assert w.e.next_batch() == 0, "soft_close left a batch unreleased"
        assert eg.failed() == [], eg.failed()
        streams = {c: _fd_bytes(fd) for c, fd in fds.items()}
        streams = {c: s for c, s in streams.items() if s}
        for fd in fds.values():
            os.close(fd)
    want = {c: wire(fr) for c, fr in w.expect().items()}
    assert streams.keys() == want.keys(), sorted(set(streams) ^ set(want))[:10]
    for c in want:
        assert streams[c] == want[c], c
    eg.close()
    w.e.close()


# ------------------------------------------------------------------ test_gpu_inbatch_subscribe.py
SUB, UNSUB = orc.KIND_SUBSCRIBE, orc.KIND_UNSUBSCRIBE
# (32 batch slots: the unflagged engine cuts a batch at every change and keeps them all until the drain)
BASE = dict(max_conns=8192, max_topics=256, max_keys=32768, ring_bytes_per_conn=1 << 17, max_batch_msgs=1024,
            max_batch_bcast=512, max_batch_bytes=4 << 20, max_batch_deliveries=1 << 20, batch_slots=32, identity="/")


def key(i):
    return b"user-%06d" % i


def sub_frame(kind, topics):
    return orc.serialize(kind, bytes(topics))


class Trio:
    """one call sequence on the flagged engine, the unflagged engine and the oracle; streams by name.  Both
    engines are built on layout `variant` (its pool: 64 MiB) and deliver as `delivery` says."""

    def __init__(self, pcdn, variant="rings", n_valid_topics=0, delivery="copy", **cfg):
        kw = dict(BASE, n_valid_topics=n_valid_topics, **layout(pcdn, variant))
        if variant.startswith("pool"):
            kw["pool_bytes"] = 64 << 20
        kw.update(cfg)
        flags = kw.pop("flags", 0)
        self.pcdn = pcdn
        self.on = engine(pcdn, delivery, flags=flags | pcdn.FLAG_INBATCH_SUBSCRIBE, **kw)
        self.off = engine(pcdn, delivery, flags=flags, **kw)
        self.o = orc.Oracle("/", n_valid_topics)
        self.via_frames = bool(flags & pcdn.FLAG_DEVICE_PARSE)   # broadcasts arrive as user frames (parsed on the device)
        self.conn = [{}, {}, {}]           # name → conn id on on / off / oracle
        self.got = [{}, {}]                # conn → frames delivered so far (engines)
        self.b0 = self.on.stats().batches

    def engines(self):
        return (self.on, self.off)

    def add_user(self, k, topics=()):
        for i, e in enumerate(self.engines()):
            self.conn[i][k] = e.add_user(k, list(topics))
        self.conn[2][k] = self.o.add_user(k, list(topics))

    def add_users(self, n, topics_of=lambda i: ()):
        for i in range(n):
            self.add_user(key(i), topics_of(i))

    def add_broker(self, ident, topics=()):
        for i, e in enumerate(self.engines()):
            self.conn[i][ident] = e.add_broker(ident)
        self.conn[2][ident] = self.o.add_broker(ident)
        if topics:
            self.call("subscribe_broker_to", ident, list(topics))

    def call(self, name, *a):
        """the same call on all three (state changes, handle_* messages)"""
        for e in self.engines():
            getattr(e, name)(*a)
        getattr(self.o, name)(*a)

    def recv(self, k, raw):
        rcs = [e.user_receive(k, raw) for e in self.engines()] + [self.o.user_receive(k, raw)]
        assert rcs[0] == rcs[1] and (rcs[0] == 0) == (rcs[2] == 0), rcs
        return rcs[0]

    def bcast(self, topics, payload, users_only=False):
        raw = orc.broadcast_frame(list(topics), payload)
        if self.via_frames and not users_only:
            self.recv(b"broadcaster", raw)
        else:
            self.call("handle_broadcast_message", list(topics), raw, users_only)

    def drain(self):
        for i, e in enumerate(self.engines()):
            for c, fr in e.drain().items():
                self.got[i].setdefault(c, []).extend(fr)

    def batches(self):
        return self.on.stats().batches - self.b0

    def check(self, batches=None):
        self.drain()
        n = 0
        for name, oc in self.conn[2].items():
            want = self.o.frames(oc)
            for i in range(2):
                got = self.got[i].get(self.conn[i][name], [])
                assert got == want, f"{'flag on' if i == 0 else 'flag off'}: stream of {name!r} differs from the oracle " \
                                    f"({len(got)} frames, oracle {len(want)})"
            n += len(want)
        if batches is not None:
            assert self.batches() == batches, (self.batches(), batches)
        return n

    def close(self):
        for e in self.engines():
            e.close()


# ---- call sequences: each takes a Trio, drives it and returns the batches the flagged engine launches
def case_sub_around_broadcast(t):
    """a subscribe before and after a broadcast to its topic, an unsubscribe mid-batch, sub / unsub / sub
    of one (connection, topic) with broadcasts between them: one batch"""
    t.add_users(40, lambda i: [i % 3])
    t.bcast([7], b"before")                      # nobody on 7 yet
    t.call("subscribe_user_to", key(1), [7])
    t.bcast([7], b"after sub 1")
    t.call("unsubscribe_user_from", key(2), [2])
    t.bcast([2], b"after unsub 2")
    for j, (name, tp) in enumerate([("subscribe_user_to", 9), ("unsubscribe_user_from", 9), ("subscribe_user_to", 9)]):
        t.bcast([9], b"toggle %d" % j)
        t.call(name, key(5), [tp])
    t.bcast([9], b"toggle end")
    return 1


def case_multi_topic_dedup(t):
    """a multi-topic broadcast where the recipient drops one of its matching topics and keeps another (R3)"""
    t.add_users(10, lambda i: [1, 2] if i < 5 else [3])
    t.bcast([1, 2], b"both")
    t.call("unsubscribe_user_from", key(0), [1])
    t.bcast([1, 2], b"dropped 1, keeps 2")
    t.call("unsubscribe_user_from", key(0), [2])
    t.bcast([1, 2], b"dropped both")
    t.call("subscribe_user_to", key(7), [1, 2])
    t.bcast([2, 1, 2], b"joined both")
    return 1


def case_idempotent(t):
    """a subscribe to a topic the connection already has, an unsubscribe of an absent topic"""
    t.add_users(8, lambda i: [4])
    t.bcast([4], b"a")
    t.call("subscribe_user_to", key(3), [4, 4])
    t.call("unsubscribe_user_from", key(3), [5, 200])
    t.call("unsubscribe_user_from", b"nobody-here", [4])
    t.bcast([4, 5], b"b")
    return 1


def case_own_echo(t):
    """a user's own Subscribe frame, then its own broadcast to that topic (R5: the sender receives it)"""
    t.add_users(6, lambda i: [0])
    t.recv(key(2), orc.broadcast_frame([6], b"not yet"))
    assert t.recv(key(2), sub_frame(SUB, [6])) == 0, "Subscribe frame refused"
    t.recv(key(2), orc.broadcast_frame([6], b"echo"))
    assert t.recv(key(2), sub_frame(UNSUB, [6, 0])) == 0, "Unsubscribe frame refused"
    t.recv(key(2), orc.broadcast_frame([6, 0], b"gone"))
    return 1


def case_broker_events(t):
    """broker subscribe / unsubscribe events, to_users_only on and off"""
    t.add_users(5, lambda i: [1])
    t.add_broker("a/a", [1])
    t.add_broker("b/b")
    for uo in (False, True):
        t.bcast([2], b"pre %d" % uo, uo)
        t.call("subscribe_broker_to", "b/b", [2])
        t.bcast([2], b"post %d" % uo, uo)
        t.call("unsubscribe_broker_from", "a/a", [1])
        t.bcast([1], b"a left %d" % uo, uo)
        t.call("subscribe_broker_to", "a/a", [1])
        t.call("unsubscribe_broker_from", "b/b", [2])
        t.bcast([1, 2], b"swap %d" % uo, uo)
    return 1


def case_shared_word(t):
    """connection 0 subscribes through a flushing call, connection 1 (same 32-bit word) subscribes
    in-batch after a broadcast: the broadcast reaches 0 and not 1"""
    t.add_user(key(0), [])
    t.add_user(key(1), [])
    t.bcast([3], b"nobody")
    t.add_user(key(2), [3])                      # flushing: launches "nobody", then dirties the word
    t.call("subscribe_user_to", key(0), [3])     # an event at position 0: the batch is empty
    t.bcast([3], b"to 0 and 2")
    t.call("subscribe_user_to", key(1), [3])
    t.bcast([3], b"to all three")
    # the same word once more, with the first change made between batches by a kick
    t.add_user(key(0), [3])
    t.bcast([3], b"after kick")
    t.call("unsubscribe_user_from", key(1), [3])
    t.bcast([3], b"1 left")
    return 3


def case_edges(t):
    """events of connections on lane (256), word (32) and match-block (8192) edges, and a broadcast to
    many topics at once"""
    edges = [0, 31, 32, 255, 256, 8191, 8192, 8193, 16383]
    t.add_users(16384, lambda i: [i % 5])
    for j, c in enumerate(edges):
        t.bcast([10, c % 5], b"edge %d" % j)
        t.call("subscribe_user_to", key(c), [10])
        t.call("unsubscribe_user_from", key(c), [c % 5])
    t.bcast([10], b"all edges")
    t.bcast(list(range(5)), b"the rest")
    return 1


def case_class_thresholds(t):
    """events that move a message's recipient count across kFatMin and the connection-major threshold"""
    n_cm = t.on.shard_info(0).shard_stride >> K.kCmDenseShift
    t.add_users(n_cm + 8, lambda i: ([11] if i < K.kFatMin - 1 else []) + ([12] if i < n_cm - 1 else []))
    t.bcast([11], b"thin")
    t.call("subscribe_user_to", key(K.kFatMin), [11])
    t.bcast([11], b"fat")
    t.call("unsubscribe_user_from", key(0), [11])
    t.bcast([11], b"thin again")
    t.bcast([12], b"message-major " * 10)
    t.call("subscribe_user_to", key(n_cm + 1), [12])
    t.bcast([12], b"connection-major " * 10)
    t.call("unsubscribe_user_from", key(3 * K.kFatMin), [12])
    t.bcast([12], b"message-major again " * 10)
    return 1


def case_events_only(t):
    """a batch that holds only events, and an event as the last call before pcdn_flush"""
    t.add_users(20, lambda i: [0])
    t.call("subscribe_user_to", key(1), [1])
    t.call("unsubscribe_user_from", key(2), [0])
    t.drain()                                   # no message: nothing launched
    t.bcast([0, 1], b"sees both events")
    t.call("subscribe_user_to", key(3), [1])    # the last call before the flush
    t.drain()
    t.bcast([1], b"next batch")
    return 2


def case_capacity_fallback(t):
    """more events than max_batch_msgs: the first that does not fit launches the batch"""
    t.add_users(30, lambda i: [0])
    t.bcast([1], b"first")
    for i in range(12):                         # max_batch_msgs = 8 in this case
        t.call("subscribe_user_to", key(i), [1])
        if i % 3 == 2:
            t.bcast([1], b"after %d" % i)
    t.bcast([1], b"last")
    return None                                 # (checked by its test)


def case_kick(t):
    """a kick (add_user with a known key) between events"""
    t.add_users(10, lambda i: [0])
    t.call("subscribe_user_to", key(4), [2])
    t.bcast([2], b"to 4")
    t.add_user(key(4), [0])                     # launches the batch; 4 is back on topic 0 only
    t.call("subscribe_user_to", key(5), [2])
    t.bcast([0, 2], b"after kick")
    return 2


def case_wide(t):
    """a 256-topic subscribe meeting a 256-topic broadcast"""
    t.add_users(64, lambda i: [i % 4])
    everything = list(range(256))
    t.bcast(everything, b"wide 0")
    t.call("unsubscribe_user_from", key(1), everything)
    t.bcast(everything[::-1], b"wide 1")
    t.call("subscribe_user_to", key(1), everything)
    t.call("subscribe_user_to", key(2), everything)
    t.bcast(everything, b"wide 2")
    t.call("unsubscribe_user_from", key(2), everything[1:])
    t.bcast(everything[1:], b"wide 3")
    return 1


def case_many_messages(t):
    """more than 256 messages in the batch (the regular plan kernels), events spread through it"""
    t.add_users(300, lambda i: [i % 7])
    for j in range(500):
        if j % 37 == 5:
            t.call("subscribe_user_to" if j % 2 else "unsubscribe_user_from", key(j % 300), [(j // 37) % 7])
        t.bcast([j % 7], b"m%d" % j)
    return 1


CASES = [case_sub_around_broadcast, case_multi_topic_dedup, case_idempotent, case_own_echo, case_broker_events,
         case_shared_word, case_edges, case_class_thresholds, case_events_only, case_kick, case_wide, case_many_messages]


def inbatch_subscribe(pcdn, case, variant, delivery="copy"):
    """test_inbatch_subscribe: one call sequence on a Trio of layout `variant`"""
    cfg = {}
    if case is case_edges and variant != "shards-host":   # (three shards hold 3 x 8192 ids already)
        cfg = dict(max_conns=16384, max_keys=65536)
    t = Trio(pcdn, variant, delivery=delivery, **cfg)
    try:
        expect = case(t)
        assert t.check(expect) > 0, "nothing delivered"
    finally:
        t.close()


# ------------------------------------------------------------------ test_gpu_egress.py
def traffic(w, rng, keys, n):
    for _ in range(n):
        size = rng.choice([0, 5, 100, 1000, 1024, 5000, 20000])
        if rng.random() < 0.6:
            t = [rng.randrange(4)]
            w.bcast(t, orc.broadcast_frame(t, payload(rng, size)))
        else:
            k = rng.choice(keys)
            w.direct(k, orc.direct_frame(k, payload(rng, size)))


def writer_to_file_descriptors(pcdn, mode, delivery="copy"):
    """test_writer_to_file_descriptors"""
    cfg = dict(max_conns=2048, ring_bytes_per_conn=3 << 18)   # 768 KiB: a batch never overflows a ring, several wrap it
    if mode == "host-rings":
        cfg["flags"] = pcdn.FLAG_HOST_RINGS
    if mode == "shards-host":
        cfg.update(shard_cfg(pcdn, mode), max_conns=1024)
    if mode == "pool-runs":
        cfg.update(flags=pcdn.FLAG_OUTPUT_POOL | pcdn.FLAG_SPAN_RUNS, pool_bytes=512 << 20)
    w = World(pcdn, delivery=delivery, **cfg)
    eg = pcdn.Egress(w.e, n_threads=8)
    rng = random.Random(8)
    keys = [rng.getrandbits(64).to_bytes(8, "little") * 2 for _ in range(1300)]
    fds = {}
    for i, k in enumerate(keys):
        c = w.add_user(k, [x for x in range(4) if rng.random() < 0.5])
        if i < 1100:
            fds[c] = os.memfd_create("conn%d" % c)
            eg.attach(c, fds[c])
    stream = {c: bytearray() for c in fds}
    nbytes = 0
    for rnd in range(6):
        traffic(w, rng, keys, 30)
        b = w.e.flush()
        st = eg.write_batch(b)
        assert w.e.poll(b).n_overflow == 0, "a ring overflowed"
        w.e.release_batch(b)
        exp = w.expect()
        for c, fr in exp.items():
            if c in stream:
                stream[c] += wire(fr)
        attached_bytes = sum(len(wire(fr)) for c, fr in exp.items() if c in fds)
        assert st.fd_bytes == attached_bytes, (st.fd_bytes, attached_bytes)
        assert st.unattached_spans >= sum(1 for c in exp if c not in fds), st.unattached_spans
        nbytes += st.fd_bytes
    assert eg.failed() == [], eg.failed()
    for c, fd in fds.items():
        os.lseek(fd, 0, os.SEEK_SET)
        got = os.read(fd, len(stream[c]) + 16)
        assert got == bytes(stream[c]), c
        os.close(fd)
    assert nbytes > 10_000_000, nbytes
    eg.close()
    w.e.close()


def sockets_backpressure_failure_and_soft_close(pcdn, delivery="copy"):
    """test_sockets_backpressure_failure_and_soft_close"""
    w = World(pcdn, max_conns=256, ring_bytes_per_conn=1 << 20, max_batch_bytes=8 << 20, delivery=delivery)
    eg = pcdn.Egress(w.e, n_threads=4)
    ka, kb, kc = b"alice-key", b"bob-key", b"carol-key"
    ca, cb_, cc = w.add_user(ka, [0]), w.add_user(kb, [0]), w.add_user(kc, [0])
    sa, ra = socket.socketpair()
    sa.setsockopt(socket.SOL_SOCKET, socket.SO_SNDBUF, 4096)
    sa.setblocking(False)
    sb, rb = socket.socketpair()
    rb.close()                      # bob is gone
    sc, rc_ = socket.socketpair()
    eg.attach(ca, sa.fileno()); eg.attach(cb_, sb.fileno()); eg.attach(cc, sc.fileno())
    got_a, got_c = bytearray(), bytearray()

    def reader(sock, buf):
        while True:
            d = sock.recv(3000)
            if not d:
                return
            buf.extend(d)

    ta = threading.Thread(target=reader, args=(ra, got_a)); ta.start()
    tc = threading.Thread(target=reader, args=(rc_, got_c)); tc.start()
    rng = random.Random(1)
    for _ in range(30):
        w.bcast([0], orc.broadcast_frame([0], payload(rng, 30000)))
    b = w.e.flush()
    st = eg.write_batch(b)
    w.e.release_batch(b)
    failed = [eg.failed(), eg.failed()]
    assert failed == [[cb_], []], failed       # reported once
    exp = w.expect()
    want_a, want_c = bytearray(wire(exp[ca])), bytearray(wire(exp[cc]))
    # the host removes the failed peer, exactly as the reference does
    w.both("remove_user", kb)
    # soft_close: these frames are only in the OPEN batch when the close is requested
    for i in range(5):
        w.direct(ka, orc.direct_frame(ka, b"last words %d" % i))
        w.bcast([0], orc.broadcast_frame([0], payload(rng, 2000)))
    fd = eg.soft_close(ca)
    assert fd == sa.fileno(), (fd, sa.fileno())
    exp = w.expect()
    want_a += wire(exp[ca]); want_c += wire(exp[cc])
    assert cb_ not in exp, "the removed peer still receives"
    sa.close(); sc.close()
    ta.join(20); tc.join(20)
    assert bytes(got_a) == bytes(want_a) and bytes(got_c) == bytes(want_c), \
        f"alice {len(got_a)} of {len(want_a)} bytes, carol {len(got_c)} of {len(want_c)}"
    ra.close(); rc_.close(); sb.close()
    eg.close()
    w.e.close()


# ------------------------------------------------------------------ test_gpu_egress_backlog.py
def send_batches(w, eg, rng, n_batches, topics=(0,), per_batch=8, lo=1, hi=40000, between=None):
    """n batches of broadcasts of lo..hi bytes, each written then released at once; returns the
    oracle's stream per connection"""
    want = {}
    for k in range(n_batches):
        for _ in range(per_batch):
            t = [rng.choice(topics)]
            w.bcast(t, orc.broadcast_frame(t, payload(rng, rng.randint(lo, hi))))
        b = w.e.flush()
        eg.write_batch(b)
        w.e.release_batch(b)
        for c, fr in w.expect().items():
            want.setdefault(c, bytearray()).extend(wire(fr))
        if between:
            between(k, want)
    return want


def stalled_peer_does_not_stall_the_others(pcdn, name, delivery="copy"):
    """test_stalled_peer_does_not_stall_the_others on layout `name`"""
    w = backlog_world(pcdn, name, delivery)
    eg = pcdn.Egress(w.e, n_threads=4, backlog_bytes_per_conn=BIG, backlog_bytes_total=4 * BIG)
    rng = random.Random(11)
    conns = [w.add_user(b"user-%03d" % i, [0]) for i in range(12)]   # three shards: spread A, B, C
    a, b, c = conns[0], conns[4], conns[8]
    sa, ra = sock_pair(4096)
    sb, rb = sock_pair()
    sc, rc_ = sock_pair()
    eg.attach(a, sa.fileno()); eg.attach(b, sb.fileno()); eg.attach(c, sc.fileno())
    reader_a = Reader(ra.fileno(), started=False)
    reader_b, reader_c = Reader(rb.fileno()), Reader(rc_.fileno())
    t0 = time.time()
    want = send_batches(w, eg, rng, 6)
    assert time.time() - t0 < IDLE_LIMIT / 2 and not reader_a.late, "the writer waited for the stalled peer"
    assert reader_b.wait_for(len(want[b]), eg) == bytes(want[b]), "B's stream"
    assert reader_c.wait_for(len(want[c]), eg) == bytes(want[c]), "C's stream"
    assert eg.failed() == [], eg.failed()
    pend, nbytes = eg.backlog()
    assert pend == [a] and 0 < nbytes < len(want[a]), (pend, nbytes, len(want[a]))
    assert len(reader_a.buf) == 0, len(reader_a.buf)
    reader_a.go()
    assert flush_until_done(eg) == 0, "backlog left after flush_backlog"
    assert eg.backlog() == ([], 0), eg.backlog()
    assert reader_a.wait_for(len(want[a])) == bytes(want[a]), "A's stream"
    assert eg.failed() == [], eg.failed()
    for s in (sa, sb, sc):
        s.close()
    for r in (reader_a, reader_b, reader_c):
        r.finish()
    for s in (ra, rb, rc_):
        s.close()
    eg.close()
    w.e.close()


# ------------------------------------------------------------------ test_gpu_shards.py
def sharded_device_resident_batch(pcdn, variant, delivery="copy"):
    """test_sharded_device_resident_batch"""
    import torch

    w = World(pcdn, max_conns=2048, ring_bytes_per_conn=1 << 16, max_batch_bytes=1 << 20, delivery=delivery,
              **shard_cfg(pcdn, variant))
    rng = random.Random(3)
    keys = [rng.getrandbits(64).to_bytes(8, "little") * 4 for _ in range(1000)]
    for i, k in enumerate(keys):
        w.add_user(k, [i % 3])
    M = 12
    frames, kinds, topics, aux_off, aux_len = [], [], [], [], []
    arena = bytearray()
    slot_off = []
    for m in range(M):
        if m % 4 == 3:
            rc = keys[m * 17]
            fr = orc.direct_frame(rc, payload(rng, 100 + m))
            w.o.handle_direct_message(rc, fr, False)
            kinds.append(3)
        else:
            t = [m % 3]
            fr = orc.broadcast_frame(t, payload(rng, 500 * m + 1))
            w.o.handle_broadcast_message(t, fr, False)
            kinds.append(4)
        slot_off.append(len(arena) // 16)
        arena += bytes(4) + fr + bytes((-(4 + len(fr))) % 16)
        if kinds[-1] == 3:
            aux_off.append(len(arena)); aux_len.append(len(rc))
            arena += rc + bytes((-len(rc)) % 16)
        else:
            aux_off.append(len(topics)); aux_len.append(1)
            topics.append(m % 3)
        frames.append(fr)
    dev = torch.device("cuda", w.e.shard_info(0).device)
    t8 = lambda a: torch.tensor(list(a), dtype=torch.uint8, device=dev)
    t32 = lambda a: torch.tensor(list(a), dtype=torch.int32, device=dev)
    d_arena = t8(arena + bytes(64))
    d_kind, d_flags = t8(kinds), t8([0] * M)
    d_slot, d_len, d_aoff, d_alen = t32(slot_off), t32([len(f) for f in frames]), t32(aux_off), t32(aux_len)
    d_topics = torch.tensor(topics, dtype=torch.int16, device=dev)
    bidx = [i for i in range(M) if kinds[i] == 4]
    d_bidx = t32(bidx)
    torch.cuda.synchronize(dev)
    db = pcdn.DeviceBatch(M, len(bidx), d_arena.data_ptr(), len(arena), d_kind.data_ptr(), d_flags.data_ptr(), d_slot.data_ptr(),
                          d_len.data_ptr(), d_aoff.data_ptr(), d_alen.data_ptr(), d_topics.data_ptr(), len(topics), d_bidx.data_ptr())
    for _ in range(3):   # slots are reused: the ingest regions must be rewritten correctly each time
        b = w.e.submit_device(db)
        res = w.e.poll(b)
        assert res.status == 0, res.status
        got = w.e.collect_frames(res)
        w.e.release_batch(b)
        want = w.expect()
        assert got == want, sorted(c for c in set(got) | set(want) if got.get(c) != want.get(c))[:10]
        for m in range(M):
            if kinds[m] == 3:
                w.o.handle_direct_message(keys[m * 17], frames[m], False)
            else:
                w.o.handle_broadcast_message([m % 3], frames[m], False)
    w.e.close()


# ------------------------------------------------------------------ test_gpu_cm_runs.py
def groups_that_are_not_one_run(pcdn, name, world=World):
    """test_groups_that_are_not_one_run on layout `name` → the world"""
    w = cm_world(pcdn, name, world)
    for i in range(CM_DENSE):
        w.add_user(b"dense%05d" % i, [0])
    x = b"inter-leaved"
    w.add_user(x, [0, 1, 2])                   # topic 1: thin (x alone), topic 2: message-major (x + 63 others)
    for i in range(63):
        w.add_user(b"fat%05d" % i, [2])
    w.add_user(b"partial", [3])                # receives group messages 0, 2 and 5 only
    w.add_user(b"second-group", [4])           # receives nothing of the first group, all of the second
    shards = max(1, w.e.num_shards()[0])
    assert 16 * (CM_DENSE // shards) >= w.e.shard_info(0).shard_stride, "topic 0 must be connection-major on every shard"
    tag = 0

    def bcast(topics, size=1000):
        nonlocal tag
        tag += 1
        w.bcast(topics, cm_frame(topics, tag, size))

    # a partial match: messages 0, 2 and 5 of a group
    for i in range(K.kCmGroup):
        bcast([0, 3] if i in (0, 2, 5) else [0])
    n = w.check()
    assert n == K.kCmGroup * (CM_DENSE + 1) + 3, n

    # a thin, a message-major and a direct record of x between connection-major messages of one group
    for i in range(K.kCmGroup):
        bcast([0])
        if i == 2:
            bcast([1], 300)
        if i == 4:
            bcast([2], 500)
        if i == 5:
            tag += 1
            w.direct(x, orc.direct_frame(x, bytes([tag]) * 200))
    assert w.check() > 0, "nothing delivered"

    # a last group of fewer than kCmGroup messages; a connection that matches nothing of the first group
    for i in range(K.kCmGroup + 3):
        bcast([0, 4] if i >= K.kCmGroup else [0])
    assert w.check() > 0, "nothing delivered"

    # rings of CM_RING bytes: the batches of 8 records wrap inside a group (the pool has no wrap)
    for _ in range(3):
        for i in range(K.kCmGroup):
            bcast([0])
        assert w.check() > 0, "nothing delivered"
    w.e.close()
    return w
