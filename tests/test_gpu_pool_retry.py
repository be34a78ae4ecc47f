"""The output pool's back-pressure path (PCDN_FLAG_OUTPUT_POOL): a batch that does not fit is refused
(status PCDN_EAGAIN), the host releases older batches and calls pcdn_retry_batch.  The refused batch
must come out as if it had fit at launch: routed against the tables as they were when it was launched
(R12), on every shard of a sharded engine, with its device-parse outcomes unchanged, and written by
the egress consumer exactly once.  Every stream is compared bit for bit with the oracle, which
processes the refused batch's messages before any later state change.

The refusal is arranged the same way everywhere: 4 MiB pools, and one hot connection that takes
3.8 MB of its shard's pool in an earlier batch that stays unreleased.  The next batch's share on that
shard (about 0.8 MB) no longer fits there; on the other shards it does."""
import os

import pytest

from oracle import oracle as orc
from test_gpu_egress import chunk_streams, wire
from test_gpu_parity import World, shard_cfg

pytestmark = pytest.mark.gpu

EAGAIN = 11          # pcdn_batch_result.status of a batch refused for space
HOT = b"hot-connection"


class PoolWorld(World):
    """a World on a small output pool, with 300 users on topics 0 / 1, a hot user and a peer broker"""

    def __init__(self, pcdn, layout, flags=0, n_users=300, **cfg):
        kw = dict(max_conns=1024, flags=pcdn.FLAG_OUTPUT_POOL | flags, pool_bytes=4 << 20, batch_slots=4,
                  max_batch_bytes=8 << 20)
        if layout == "shards-host":
            kw.update(shard_cfg(pcdn, layout))
        kw.update(cfg)
        super().__init__(pcdn, **kw)
        self.conn = {}
        self.keys = [b"user-%04d" % i for i in range(n_users)]
        for i, k in enumerate(self.keys):
            self.add_user(k, [i % 2])
        self.add_user(HOT, [])
        self.add_broker("p/q", [0])
        self.nl = max(1, self.e.num_shards()[0])
        self.stride = self.e.shard_info(0).shard_stride
        self.home = self.shard_of(HOT)

    def add_user(self, key, topics):
        self.conn[key] = super().add_user(key, topics)
        return self.conn[key]

    def shard_of(self, key):
        return self.conn[key] // self.stride

    def on_shard(self, shard, topic=None):
        return [k for i, k in enumerate(self.keys) if self.shard_of(k) == shard and (topic is None or i % 2 == topic)]

    def fill_hot(self):
        """38 x 100 KB to the hot connection: 3.8 MB of its shard's 4 MiB pool"""
        for j in range(38):
            self.direct(HOT, orc.direct_frame(HOT, bytes([j]) * 100_000))
        return self.e.flush()

    def traffic(self, tag, directs=()):
        """three 2.5 KB broadcasts to each topic (7.7 KB per user) and a direct to each of `directs`"""
        for t in (0, 1):
            for j in range(3):
                self.bcast([t], orc.broadcast_frame([t], bytes([tag, t, j]) * 1250))
        for k in directs:
            self.direct(k, orc.direct_frame(k, b"batch %d to %s" % (tag, k)))
        return self.e.flush()

    def statuses(self, b):
        return [self.e.poll_shard(b, li).status for li in range(self.nl)]

    def consume(self, b, got, retry=False):
        """(retry,) poll, collect every connection's frames, release"""
        if retry:
            self.e.retry_batch(b)
        r = self.e.poll(b)
        assert r.status == 0 and r.n_overflow == 0
        self.e.last_result = r                                # (World.dump reports it on a mismatch)
        for c, fr in self.e.collect_frames(r).items():
            got.setdefault(c, []).extend(fr)
        self.e.release_batch(b)
        return r


@pytest.mark.parametrize("runs", [False, True], ids=["spans", "span-runs"])
@pytest.mark.parametrize("control", ["fused", "regular"])
@pytest.mark.parametrize("layout", ["one-shard", "shards-host"])
def test_retry_routes_as_launched(pcdn, layout, control, runs):
    """state changes between a refusal and its retry (subscribe a new user, unsubscribe, remove, the
    kick of a reconnect, a user moved to a peer broker, a broker subscription) reach only batches
    launched after them: the retried batch delivers what it would have delivered at launch, and a
    batch launched after the changes, while the pool is still blocked, sees the new tables.
    control = "regular": FLAG_STAGED_SPANS, so k_match / k_offsets / k_pool_finish run instead of the
    fused k_ctrl_small (with conn_base != 0 on the sharded engine)."""
    flags = (pcdn.FLAG_STAGED_SPANS if control == "regular" else 0) | (pcdn.FLAG_SPAN_RUNS if runs else 0)
    w = PoolWorld(pcdn, layout, flags)
    t0, t1 = w.on_shard(w.home, 0), w.on_shard(w.home, 1)
    unsub, removed, moved = t0[0], t0[1], t1[0]
    kicked, newcomer = t1[1], b"newcomer"
    directs = (unsub, removed, kicked, moved, newcomer)
    b0 = w.fill_hot()
    b1 = w.traffic(1, directs)
    assert w.e.poll(b0).status == 0
    st1 = w.statuses(b1)
    assert st1[w.home] == EAGAIN and w.e.poll(b1).status == EAGAIN, st1
    w.add_user(newcomer, [0])
    w.both("unsubscribe_user_from", unsub, [0])
    w.both("remove_user", removed)
    w.add_user(kicked, [0])                                   # same key, new connection: the old one is kicked
    w.both("apply_user_sync", "p/q", [(moved, 1000, "p/q")])  # the peer now owns this user
    w.both("subscribe_broker_to", "p/q", [1])
    b2 = w.traffic(2, directs)
    assert w.statuses(b2)[w.home] == EAGAIN                   # queued behind the refused batch
    got = {}
    w.consume(b0, got)
    w.consume(b1, got, retry=True)
    w.consume(b2, got, retry=True)
    assert w.compare(w.e, got, w.expect()) > 2 * 3 * 290
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


def test_partial_refusal_across_shards(pcdn):
    """one shard refuses its share, the others accept theirs; users reconnect across shards in both
    directions before the retry.  Each direct message arrives exactly once, at the connection its key
    named at launch, and every stream equals the oracle's."""
    w = PoolWorld(pcdn, "shards-host")
    assert w.nl == 3
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
    assert w.e.poll(b0).status == 0
    want_st = [EAGAIN if s == w.home else 0 for s in range(w.nl)]
    assert w.statuses(b1) == want_st
    assert w.e.poll(b1).status == EAGAIN                     # the combined result: "retry" wins
    reconnect_onto(w, x, w.home, fillers)
    reconnect_onto(w, y, accept, fillers)
    b2 = w.traffic(2, (x, y))                                 # the new connections, after the moves
    got = {}
    w.consume(b0, got)
    w.e.retry_batch(b1)
    assert w.statuses(b1) == [0] * w.nl
    w.consume(b1, got)
    w.consume(b2, got, retry=True)
    frames = [f for fr in got.values() for f in fr]
    copies = {(who, j): frames.count(orc.direct_frame(k, b"to %s, %d" % (who, j)))
              for who, k in ((b"x", x), (b"y", y)) for j in range(3)}
    assert copies == {wj: 1 for wj in copies}, copies
    w.compare(w.e, got, w.expect())
    w.e.close()


def _broken_direct(key):
    raw = bytearray(orc.direct_frame(key, b"x" * 64))
    raw[36:40] = (0xFFFFFFF).to_bytes(4, "little")            # recipient list beyond the segment
    return bytes(raw)


@pytest.mark.parametrize("layout", ["one-shard", "shards-host"])
def test_device_parse_retry_keeps_msg_status(pcdn, layout):
    """FLAG_DEVICE_PARSE: k_parse records each message's outcome and rewrites the descriptor of the
    ones it rejects.  After the retry msg_status and n_msg_errors, on every shard, are what the first
    poll said and what the oracle's receive loops return: a parse error stays -7, a prune error -8, a
    broker-origin broadcast with only invalid topics and a direct to a key longer than max_key_len stay
    0 (not routed, no error)."""
    w = PoolWorld(pcdn, layout, pcdn.FLAG_DEVICE_PARSE, n_valid_topics=4)
    sender = w.keys[0]
    frames = [(sender, 0, _broken_direct(w.keys[1])),
              (sender, 0, orc.broadcast_frame([9, 7], b"only invalid topics")),
              (sender, 1, orc.broadcast_frame([9, 7], b"only invalid topics, from a broker")),
              (sender, 0, orc.direct_frame(b"L" * 200, b"to a key longer than max_key_len"))]
    for t in (0, 1):
        for j in range(3):
            frames.append((sender, 0, orc.broadcast_frame([t], bytes([t, j]) * 1250)))
    for k in w.keys[2:8] + [HOT, b"nobody"]:
        frames.append((sender, 0, orc.direct_frame(k, b"direct to " + k)))
    b0 = w.fill_hot()
    want_rc = [w.o.broker_receive(raw) if origin else w.o.user_receive(s, raw) for s, origin, raw in frames]
    rcs = w.e.receive_frames(frames)
    b1 = w.e.flush()
    assert rcs == [0] * len(frames)
    assert want_rc[:4] == [-7, -8, 0, 0] and set(want_rc[4:]) == {0}
    results = lambda: [w.e.poll_shard(b1, li) for li in range(w.nl)] + [w.e.poll(b1)]
    first = [(r.status, [r.msg_status[i] for i in range(r.n_msgs)], r.n_msg_errors) for r in results()]
    assert first[-1][0] == EAGAIN and first[w.home][0] == EAGAIN
    for st, ms, ne in first:
        assert ms == want_rc and ne == 2
    got = {}
    w.consume(b0, got)
    w.e.retry_batch(b1)
    again = [(r.status, [r.msg_status[i] for i in range(r.n_msgs)], r.n_msg_errors) for r in results()]
    assert again == [(0, ms, ne) for _, ms, ne in first]
    w.consume(b1, got)
    w.compare(w.e, got, w.expect())
    w.e.close()


def _fd_bytes(fd):
    os.lseek(fd, 0, os.SEEK_SET)
    return os.read(fd, os.fstat(fd).st_size + 16)


@pytest.mark.parametrize("how", ["drain", "write_batch", "soft_close"])
def test_egress_refused_shard_is_written_once(pcdn, how):
    """the egress consumer on a batch one shard refused: nothing of it reaches the sink (PCDN_EAGAIN)
    until it is retried, then every shard's share is written exactly once — through a Python sink,
    through write_batch to memfds, and inside soft_close, which releases, retries and writes by itself."""
    w = PoolWorld(pcdn, "shards-host")
    eg = pcdn.Egress(w.e, n_threads=4)
    fds = {}
    if how != "drain":
        for c in w.map:                                       # every user and the peer broker
            fds[c] = os.memfd_create("conn%d" % c)
            eg.attach(c, fds[c])
    b0 = w.fill_hot()
    b1 = w.traffic(1, w.keys[::37])
    assert w.statuses(b1) == [EAGAIN if s == w.home else 0 for s in range(w.nl)]
    if how == "drain":
        got = {}
        eg.drain(b0, lambda ch: chunk_streams(ch, got))
        calls = []
        with pytest.raises(pcdn.PcdnError) as ei:
            eg.drain(b1, lambda ch: calls.append(ch.n_spans))
        assert ei.value.code == -EAGAIN and calls == []
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
            assert ei.value.code == -EAGAIN
            assert {c: _fd_bytes(fd) for c, fd in fds.items()} == before
            w.e.release_batch(b0)
            w.e.retry_batch(b1)
            eg.write_batch(b1)
            w.e.release_batch(b1)
        else:
            eg.soft_close(w.conn[w.keys[3]])                  # writes and releases b0, then b1 (retried)
            assert w.e.next_batch() == 0
        assert eg.failed() == []
        streams = {c: _fd_bytes(fd) for c, fd in fds.items()}
        streams = {c: s for c, s in streams.items() if s}
        for fd in fds.values():
            os.close(fd)
    want = {c: wire(fr) for c, fr in w.expect().items()}
    assert streams.keys() == want.keys()
    for c in want:
        assert streams[c] == want[c], c
    eg.close()
    w.e.close()
