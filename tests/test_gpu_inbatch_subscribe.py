"""In-batch subscription changes (PCDN_FLAG_INBATCH_SUBSCRIBE): a Subscribe / Unsubscribe, from the C ABI
or a user's frame, becomes an event of the open batch instead of launching it.

Every case runs ONE call sequence on three backends: an engine with the flag, the same engine without
it, and the oracle (which applies every call at once).  Each connection's delivered byte stream must be
equal on all three, and the flagged engine must launch the batches the case expects (pcdn_stats.batches).
The cases run on the engine variants that change how a match is computed or consumed: the fused and the
regular control kernels, run-length spans, the output pool, shared payload, three shards on one GPU and
device parse."""
import ctypes as C

import pytest

from kconst import K
from oracle import oracle as orc
from test_gpu_parity import shard_cfg

pytestmark = pytest.mark.gpu

SUB, UNSUB = orc.KIND_SUBSCRIBE, orc.KIND_UNSUBSCRIBE
# (32 batch slots: the unflagged engine cuts a batch at every change and keeps them all until the drain)
BASE = dict(max_conns=8192, max_topics=256, max_keys=32768, ring_bytes_per_conn=1 << 17, max_batch_msgs=1024,
            max_batch_bcast=512, max_batch_bytes=4 << 20, max_batch_deliveries=1 << 20, batch_slots=32, identity="/")


def key(i):
    return b"user-%06d" % i


def sub_frame(kind, topics):
    return orc.serialize(kind, bytes(topics))


def variant_cfg(pcdn, variant):
    return {
        "fused": {},
        "staged": dict(flags=pcdn.FLAG_STAGED_SPANS),
        "runs": dict(flags=pcdn.FLAG_SPAN_RUNS | pcdn.FLAG_STAGED_SPANS),
        "pool": dict(flags=pcdn.FLAG_OUTPUT_POOL, pool_bytes=64 << 20),
        "shared": dict(flags=pcdn.FLAG_SHARED_PAYLOAD),
        "shards": shard_cfg(pcdn, "shards-host") if variant == "shards" else {},
        "devparse": dict(flags=pcdn.FLAG_DEVICE_PARSE),
    }[variant]


VARIANTS = ["fused", "staged", "runs", "pool", "shared", "shards", "devparse"]


class Trio:
    """one call sequence on the flagged engine, the unflagged engine and the oracle; streams by name"""

    def __init__(self, pcdn, variant="fused", n_valid_topics=0, **cfg):
        kw = dict(BASE, n_valid_topics=n_valid_topics)
        kw.update(variant_cfg(pcdn, variant))
        kw.update(cfg)
        flags = kw.pop("flags", 0)
        self.pcdn = pcdn
        self.on = pcdn.Engine(flags=flags | pcdn.FLAG_INBATCH_SUBSCRIBE, **kw)
        self.off = pcdn.Engine(flags=flags, **kw)
        self.o = orc.Oracle("/", n_valid_topics)
        self.via_frames = variant == "devparse"   # broadcasts arrive as user frames (parsed on the device)
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
            assert self.batches() == batches
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
    assert t.recv(key(2), sub_frame(SUB, [6])) == 0
    t.recv(key(2), orc.broadcast_frame([6], b"echo"))
    assert t.recv(key(2), sub_frame(UNSUB, [6, 0])) == 0
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
    return None                                 # (checked below)


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


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("case", CASES, ids=lambda f: f.__name__[5:])
def test_inbatch_subscribe(pcdn, case, variant):
    cfg = {}
    if case is case_edges and variant != "shards":   # (three shards hold 3 x 8192 ids already)
        cfg = dict(max_conns=16384, max_keys=65536)
    t = Trio(pcdn, variant, **cfg)
    try:
        expect = case(t)
        assert t.check(expect) > 0
    finally:
        t.close()


@pytest.mark.parametrize("variant", ["fused", "staged", "shards"])
def test_event_capacity_fallback(pcdn, variant):
    t = Trio(pcdn, variant, max_batch_msgs=8)
    try:
        case_capacity_fallback(t)
        t.check()
        # 12 events on 8-event batches: the 9th launches the first batch, which holds the 4 broadcasts
        # before it; the rest is the second batch
        assert t.batches() == 2
    finally:
        t.close()


@pytest.mark.parametrize("variant", ["fused", "staged", "shards"])
def test_hooked_subscribe(pcdn, variant):
    """a user hook rewrites the topics of a Subscribe frame: the event carries the rewritten topics"""
    t = Trio(pcdn, variant)
    try:
        t.add_users(12, lambda i: [0])

        def hook(m):
            if m.kind == SUB and m.n_topics >= 2:
                m.topics[0] = m.topics[m.n_topics - 1]   # [a, .., z] -> [z]
                m.n_topics = 1
            return pcdn.HOOK_PROCESS

        for e in t.engines():
            e.set_message_hook(0, hook)
        t.bcast([3], b"before")
        for e in t.engines():
            assert e.user_receive(key(1), sub_frame(SUB, [2, 3])) == 0
        assert t.o.user_receive(key(1), sub_frame(SUB, [3])) == 0
        t.bcast([2, 3], b"only 3 is subscribed")
        assert t.check(1) > 0
    finally:
        t.close()


@pytest.mark.parametrize("variant", ["fused", "staged", "pool", "shards"])
def test_pool_retry_keeps_events(pcdn, variant):
    """a batch with events refused by the output pool and retried: it is routed as it was launched"""
    cfg = dict(variant_cfg(pcdn, variant))
    cfg["flags"] = cfg.get("flags", 0) | pcdn.FLAG_OUTPUT_POOL
    cfg.update(pool_bytes=4 << 20, batch_slots=16, max_batch_bytes=8 << 20)   # (slots: the unflagged engine cuts 13 batches)
    t = Trio(pcdn, "fused", **cfg)
    try:
        hot = b"hot-connection"
        t.add_users(200, lambda i: [i % 2])
        t.add_user(hot, [])
        for e in t.engines():                    # 3.8 MB of a 4 MiB pool, held by an unreleased batch
            for j in range(38):
                e.handle_direct_message(hot, orc.direct_frame(hot, bytes([j]) * 100_000))
        for j in range(38):
            t.o.handle_direct_message(hot, orc.direct_frame(hot, bytes([j]) * 100_000))
        first = [e.flush() for e in t.engines()]
        # the next batch carries events and does not fit until the first is released
        for j in range(4):
            t.bcast([0], bytes([j]) * 2500)
            t.call("subscribe_user_to", key(2 * j + 1), [0])
            t.call("unsubscribe_user_from", key(2 * j), [0])
            t.call("subscribe_user_to", hot, [0])
        t.bcast([0, 1], b"end" * 800)
        e = t.on                                   # (the unflagged engine's batches are retried by its drain)
        b = e.flush()
        assert e.poll(b).status == 11              # refused: the pool is held by the first batch
        for c, fr in e.collect_frames(e.poll(first[0])).items():
            t.got[0].setdefault(c, []).extend(fr)
        e.release_batch(first[0])
        e.retry_batch(b)
        r = e.poll(b)
        assert r.status == 0
        for c, fr in e.collect_frames(r).items():
            t.got[0].setdefault(c, []).extend(fr)
        e.release_batch(b)
        assert t.check(2) > 0
    finally:
        t.close()


@pytest.mark.parametrize("variant", ["fused", "staged", "devparse", "shards"])
def test_threaded_receive(pcdn, variant):
    """one threaded pcdn_receive_frames call of 4096 frames with Subscribe / Unsubscribe frames spread
    through it: the flagged engine consumes every frame in one call and one batch; without the flag the
    call stops early (each change cuts the batch and the batch slots run out)"""
    t = Trio(pcdn, variant, n_valid_topics=16, max_batch_msgs=4096, max_batch_bcast=4096, batch_slots=4)
    try:
        t.add_users(512, lambda i: [i % 16])
        frames = []
        for j in range(4096):
            k = key((j * 7) % 512)
            if j % 97 == 13:
                raw = sub_frame(SUB if j % 2 else UNSUB, [(j // 97) % 16, (j // 5) % 16])
            elif j % 53 == 7:
                raw = sub_frame(SUB, [99])               # pruned away: PCDN_EPRUNE, no event
            else:
                raw = orc.broadcast_frame([j % 16], b"f%d" % j)
            frames.append((k, 0, raw))
        rc_on = t.on.receive_frames(frames)              # raises unless every frame is consumed in one call
        rc_off, got_off = t.off.receive_frames_all(frames)
        rc_o = [t.o.user_receive(k, raw) for k, _, raw in frames]
        assert rc_on == rc_off
        assert [r == 0 for r in rc_on] == [r == 0 for r in rc_o]
        assert t.off.stats().batches > 4
        assert t.batches() == 0                           # nothing launched before the flush: one open batch
        for c, fr in got_off.items():
            t.got[1].setdefault(c, []).extend(fr)
        assert t.check(1) > 0
    finally:
        t.close()


def test_unflagged_engine_is_unchanged(pcdn):
    """without the flag every subscription change still launches the open batch first"""
    e = pcdn.Engine(**BASE)
    try:
        e.add_user(key(0), [0])
        b0 = e.stats().batches
        for j in range(3):
            e.handle_broadcast_message([0], orc.broadcast_frame([0], b"x%d" % j))
            e.subscribe_user_to(key(0), [1 + j])
        assert e.stats().batches - b0 == 3
        e.drain()
    finally:
        e.close()
