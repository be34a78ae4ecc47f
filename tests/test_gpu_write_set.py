"""Where the pack stores, not only what: every local shard's whole output allocation (all rings, or the
output pool) is filled with a position- and epoch-dependent canary, and after each drained cycle every
32-byte unit that no span of an accepted batch covers must still hold it.  That catches a store outside
the spans — wrap padding, a neighbour's ring, free ring space, the pool's skip tail, another batch's
region — which the frame-by-frame comparison with the oracle never reads.  The same guard checks the
span table's shape, that spans of batches unreleased at the same time never overlap, and that a batch
refused by the device (output pool full, or E2BIG) wrote nothing.

It also pins the overflow contract in both directions: a drained ring takes any record that fits an
empty ring, wherever its tail stood, and a ring that is really full stops at an in-order prefix
without touching the unreleased batches before it."""
import ctypes
import random

import numpy as np
import pytest

import gpu_workloads as workloads
from gpu_world import (CM_DENSE, CM_IDS, CM_MODES, CM_RING, EDGE_SLOTS, PCDN_ENOENT, STATUS_E2BIG, STATUS_EAGAIN, World,
                       check, cm_frame, cm_world, edge_sizes, edge_world, layout, payload, raw, shard_cfg, span_table, units)
from kconst import K
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

CHUNK_WORDS = 1 << 24           # canary generated / compared 128 MiB at a time
M64 = (1 << 64) - 1


def _s64(x):
    x &= M64
    return x - (1 << 64) if x >> 63 else x


class _Cuda:
    """a raw device allocation as a 1-D int64 tensor (no copy)"""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i8", "data": (ptr, False), "version": 3}


class Guard:
    """the canary over every local shard's output memory, and the record of every batch polled since
    it was last filled (per shard: status, pool_base, expanded span table, placement / release time);
    `verified` counts the drained cycles whose write set it checked"""

    def __init__(self, pcdn, e):
        import torch

        self.torch = torch
        self.e = e
        sh = e.shards()
        self.pool = bool(e.cfg.flags & pcdn.FLAG_OUTPUT_POOL)
        self.stride = sh[0].shard_stride
        self.R = sh[0].ring_bytes                     # bytes per connection ring, or of the whole pool
        self.max_conns = e.cfg.max_conns
        nbytes = self.R if self.pool else self.max_conns * self.R
        assert nbytes % K.kUnit == 0
        self.units = nbytes // K.kUnit
        self.views, self.dev = [], []
        for d in sh:
            n = nbytes // 8
            if d.rings_host:
                arr = np.ctypeslib.as_array((ctypes.c_int64 * n).from_address(d.rings_host))
                self.views.append(torch.from_numpy(arr))
            else:
                self.views.append(torch.as_tensor(_Cuda(d.rings_dev, n), device=torch.device("cuda", d.device)))
            self.dev.append(torch.device("cuda", d.device))
        self.gindex = [d.global_index for d in sh]
        self.epoch = 0
        self.clock = 0
        self.batches = {}           # batch id -> Rec, since the last fill
        self.launched = {}          # batch id -> clock at launch (batches launched through launch())
        self.verified = 0
        self.fill()

    def tick(self):
        self.clock += 1
        return self.clock

    # ---- canary
    def pattern(self, li, a, b):
        t = self.torch
        x = t.arange(a, b, dtype=t.int64, device=self.dev[li]) * _s64(0x9E3779B97F4A7C15)
        x += _s64((self.gindex[li] * 0x10001 + self.epoch + 1) * 0xBF58476D1CE4E5B9)
        x ^= x >> 31
        x *= _s64(0x94D049BB133111EB)
        x ^= x >> 29
        return x

    def fill(self):
        assert self.e.next_batch() == 0, "the canary is laid only while no batch is unreleased"
        self.epoch += 1
        for li, v in enumerate(self.views):
            for a in range(0, v.numel(), CHUNK_WORDS):
                b = min(v.numel(), a + CHUNK_WORDS)
                v[a:b].copy_(self.pattern(li, a, b))
        self.torch.cuda.synchronize()
        self.batches = {}
        self.launched = {}

    # ---- coverage of a set of spans, in 32-byte units of one shard's allocation
    def ranges(self, li, rec):
        s = rec.shards[li]
        t = s.table
        if self.pool:
            start = s.pool_base + t[:, 1]
        else:
            start = (t[:, 0] % self.stride) * (self.R // K.kUnit) + t[:, 1] // K.kUnit
        return start, start + t[:, 2] // K.kUnit

    def coverage(self, li, recs):
        t = self.torch
        diff = t.zeros(self.units + 1, dtype=t.int32, device=self.dev[li])
        for r in recs:
            a, b = self.ranges(li, r)
            if len(a):
                one = t.ones(len(a), dtype=t.int32, device=self.dev[li])
                diff.index_add_(0, t.from_numpy(a).to(self.dev[li]), one)
                diff.index_add_(0, t.from_numpy(b).to(self.dev[li]), -one)
        return t.cumsum(diff[:-1], 0, dtype=t.int32)

    def untouched(self, li, cov, what):
        """every unit of shard li that cov does not cover still holds the canary"""
        v = self.views[li]
        for a in range(0, v.numel(), CHUNK_WORDS):
            b = min(v.numel(), a + CHUNK_WORDS)
            mem = v[a:b].to(self.dev[li]).view(-1, 4)
            bad = (mem != self.pattern(li, a, b).view(-1, 4)).any(1) & (cov[a // 4:b // 4] == 0)
            if bool(bad.any()):
                u = a // 4 + self.torch.nonzero(bad)[:5, 0].cpu().numpy()
                where = [("pool unit", int(x)) if self.pool else
                         ("conn", int(x) // (self.R // K.kUnit) + self.gindex[li] * self.stride, "byte", int(x) % (self.R // K.kUnit) * K.kUnit)
                         for x in u]
                raise AssertionError(f"{what}: {int(bad.sum())} units outside every span changed on shard {li}, first {where}")

    # ---- per-batch records
    def record(self, bid, t0):
        """the per-shard results of batch bid (already polled), with their span-table sanity checks"""
        rec = self.batches.get(bid)
        if rec is None:
            rec = self.batches[bid] = Rec(bid, self.launched.get(bid, t0), len(self.views))
        for li in range(len(self.views)):
            r = self.e.poll_shard(bid, li)
            s = rec.shards[li]
            s.status, s.pool_base = r.status, r.pool_base
            s.table = span_table(r) if r.status == 0 else np.zeros((0, 4), dtype=np.int64)
            if r.status:
                assert r.n_spans == 0 and r.n_deliveries == 0 and r.n_overflow == 0, (bid, li, r.status)
            else:
                self.sane(li, s)
        return rec

    def sane(self, li, s):
        t = s.table
        if not len(t):
            return
        conn, off, ln, nrec = t[:, 0], t[:, 1], t[:, 2], t[:, 3]
        assert (conn // self.stride == self.gindex[li]).all() and (conn % self.stride < self.max_conns).all()
        assert (ln > 0).all() and (ln % K.kUnit == 0).all() and (nrec >= 1).all()
        assert (nrec <= ln // K.kUnit).all()
        if self.pool:
            # one region per batch and shard: the spans tile [0, sum of len / 32) without gap or overlap
            assert len(np.unique(conn)) == len(conn), "one span per connection in the pool"
            o = np.argsort(off, kind="stable")
            u = ln[o] // K.kUnit
            assert off[o][0] == 0 and np.array_equal(off[o][1:], np.cumsum(u)[:-1]), "the spans do not tile the region"
            assert s.pool_base + int(u.sum()) <= self.units, "region beyond the pool end"
        else:
            assert (off % K.kUnit == 0).all() and (off + ln <= self.R).all(), "span crosses the ring end"
            c, k = np.unique(conn, return_counts=True)
            assert (k <= 2).all(), "more than two spans of one connection in one batch"
            for x in c[k == 2]:
                i = np.searchsorted(conn, x)            # (table sorted by connection, then offset)
                assert off[i] == 0 and ln[i] <= off[i + 1], ("the second span of a wrapped ring starts at 0", int(x))

    def refused(self, rec, t0):
        """a refusal wrote nothing: everything outside the spans of the batches accepted so far (and of the
        batches launched after it, polled here so that their packs are finished) is still canary"""
        b = rec.bid + 1
        while True:
            try:
                self.e.poll(b)
            except Exception as ex:
                if getattr(ex, "code", None) == PCDN_ENOENT:
                    break
                raise
            self.record(b, t0)
            b += 1
        for li in range(len(self.views)):
            ok = [r for r in self.batches.values() if r.shards[li].status == 0]
            self.untouched(li, self.coverage(li, ok), f"batch {rec.bid} refused with status {rec.shards[li].status}")

    def verify(self):
        """after a drain: the write set and the overlap of live batches, then a fresh canary"""
        assert self.e.next_batch() == 0
        recs = list(self.batches.values())
        for li in range(len(self.views)):
            ok = [r for r in recs if r.shards[li].status == 0]
            cov = self.coverage(li, ok)
            self.untouched(li, cov, "write set")
            for r in ok:     # every placement: the batches live at that moment own disjoint units
                p = r.shards[li].placed
                live = [q for q in ok if q.shards[li].placed <= p < q.released]
                if len(live) > 1:
                    m = int(self.coverage(li, live).max())
                    assert m <= 1, f"spans of batches {[q.bid for q in live]}, unreleased together, overlap on shard {li}"
        self.verified += 1
        self.fill()


class _ShardRec:
    def __init__(self, placed):
        self.placed, self.status, self.pool_base, self.table = placed, 0, 0, None


class Rec:
    def __init__(self, bid, placed, n_shards):
        self.bid = bid
        self.shards = [_ShardRec(placed) for _ in range(n_shards)]
        self.released = None
        self.overflow = []
        self.frames = {}


class GuardedWorld(World):
    """World whose check() drains under the guard: records every polled batch, checks refusals when they
    are polled, and verifies the write set once everything is released"""

    def __init__(self, pcdn, *a, **kw):
        super().__init__(pcdn, *a, **kw)
        self.guard = Guard(pcdn, self.e)
        self.refusals = 0

    def launch(self):
        b = self.e.flush()
        if b:
            self.guard.launched[b] = self.guard.tick()
        return b

    def step(self, b, t0):
        """poll batch b (the oldest), retry it if the pool refused it, collect its frames, release it"""
        g, e = self.guard, self.e
        res = e.poll(b)
        rec = g.record(b, t0)
        if res.status:
            g.refused(rec, t0)
        if res.status == STATUS_EAGAIN:
            self.refusals += 1
            e.retry_batch(b)
            t = g.tick()
            for s in rec.shards:
                if s.status == STATUS_EAGAIN:
                    s.placed = t
            res = e.poll(b)
            rec = g.record(b, t0)
            if res.status:
                g.refused(rec, t0)
        if res.status == 0:
            rec.frames = e.collect_frames(res)
            rec.overflow = [res.overflow_conns[i] for i in range(res.n_overflow)]
            e.last_result = res
        rec.status = res.status
        e.release_batch(b)
        rec.released = g.tick()
        return rec

    def drain(self, first=()):
        """flush, poll the batches in `first` (in that order), then step through every batch oldest first"""
        self.launch()
        t0 = self.guard.tick()
        for b in first:
            self.e.poll(b)
            self.guard.record(b, t0)
        out, self.drained = {}, []
        while True:
            b = self.e.next_batch()
            if not b:
                return out
            rec = self.step(b, t0)
            self.drained.append(rec)
            for c, fr in rec.frames.items():
                out.setdefault(c, []).extend(fr)

    def check(self, first=()):
        got = self.drain(first)
        want = self.expect()
        n = self.compare(self.e, got, want)
        self.guard.verify()
        return n

    def spans_of(self, rec, conn):
        li = conn // self.guard.stride - self.guard.gindex[0]
        t = rec.shards[li].table
        return t[t[:, 0] == conn][:, 1:].tolist()


# ------------------------------------------------------------------ the guard around existing workloads
# (layout, delivery) under this file's test ids
EDGE_MODES = [pytest.param("rings", "copy", id="rings-fused"), pytest.param("staged", "copy", id="rings-regular"),
              pytest.param("pool", "copy", id="pool-fused"), pytest.param("pool-staged", "copy", id="pool-regular"),
              pytest.param("runs", "copy", id="runs"), pytest.param("rings", "shared", id="shared-payload"),
              pytest.param("rings", ("ref", 12000), id="ref-min")]


@pytest.mark.parametrize("name,delivery", EDGE_MODES)
def test_size_and_recipient_classes_under_guard(pcdn, name, delivery):
    """every raw length of edge_sizes() to every recipient count of recipient_counts(): thin, message-major
    (tile edges), dense message-major and connection-major, then connection-major groups of kCmGroup - 1,
    kCmGroup and kCmGroup + 1; 64 KiB rings, so a batch carries as many of the topics as fit a ring with
    its wrap padding, and the rings wrap from batch to batch"""
    ring = 1 << 16
    cfg = layout(pcdn, name)
    if name.startswith("pool"):
        cfg["pool_bytes"] = 1 << 30
    w, keys, topic = edge_world(pcdn, GuardedWorld, ring_bytes_per_conn=ring, delivery=delivery, **cfg)
    tag = 0
    for s in edge_sizes():
        rec = units(s) * K.kUnit
        per = max(1, (ring - rec + K.kUnit) // rec)    # what fits a ring wherever it wraps (padding < one record)
        items = list(topic.items())
        for i in range(0, len(items), per):
            for d, t in items[i:i + per]:
                tag += 1
                w.bcast([t], raw(s, tag))
            assert check(w) == sum(d for d, _ in items[i:i + per])
    cm_len = K.kCmMaxBytes - 4
    dense = EDGE_SLOTS >> K.kCmDenseShift
    for g in (K.kCmGroup - 1, K.kCmGroup, K.kCmGroup + 1):
        for i in range(g):
            tag += 1
            w.bcast([topic[dense + i % 2]], raw(cm_len, tag))
        assert check(w) == sum(dense + i % 2 for i in range(g))
    w.e.close()
    assert w.guard.verified > 0


@pytest.mark.parametrize("name", CM_MODES, ids=CM_IDS)
def test_connection_major_groups_under_guard(pcdn, name):
    """test_gpu_cm_runs: partial groups, thin / message-major / direct records inside a group, groups that
    wrap their 16 KiB rings"""
    w = workloads.groups_that_are_not_one_run(pcdn, name, world=GuardedWorld)
    assert w.guard.verified > 0


@pytest.mark.parametrize("variant", ["pool", "pool-staged-runs", "pool-host", pytest.param("pool-shards-host", id="pool-shards"),
                                     "shards-host"])
def test_random_mixed_batches_under_guard(pcdn, variant):
    """test_gpu_parity's randomized mixed batches (sizes 0 B to 40 KB, fat and thin broadcasts, directs to
    local, remote and unknown keys, state changes between batches)"""
    w = workloads.random_mixed_batches(pcdn, 0, variant, world=GuardedWorld)
    assert w.guard.verified > 0


def test_direct_thresholds_under_guard(pcdn):
    """the direct batches of test_gpu_kernel_edges on 4096 connections (256 KiB rings: 1 GiB guarded):
    2 / kHotMin / kHotMin + 1 hits on one connection, kHotCtas + 8 hot connections (k_dsort_hot's grid), a
    batch of more than 8192 messages whose hot recipient has hits on both sides of message 8192 (~1300
    records in one ring), kThinSeparateMin - 1 / kThinSeparateMin directs with and without a broadcast,
    hits on the 1024-entry tile edges of k_dscan and the last connection"""
    n = 4096
    w = GuardedWorld(pcdn, max_conns=n, max_keys=n + 1024, max_batch_msgs=12288, ring_bytes_per_conn=1 << 18,
                     flags=pcdn.FLAG_STAGED_SPANS)
    keys = [c.to_bytes(4, "little") + b"edge" for c in range(n)]
    for c, k in enumerate(keys):
        assert w.add_user(k, [0] if c % 64 == 5 else []) == c      # topic 0: 64 users, message-major
    rng = random.Random(9)
    edges = [1023, 1024, 1025, n - 1]
    seq = [0]

    def send(targets):
        for c in targets:
            seq[0] += 1
            k = keys[c] if c is not None else b"nobody%d" % seq[0]
            w.direct(k, orc.direct_frame(k, seq[0].to_bytes(4, "little") * rng.randrange(1, 24)))

    def batch(hot, total=0):
        t = [c for c, h in hot.items() for _ in range(h)] + edges + [None] * 3
        t += [rng.randrange(n) for _ in range(total - len(t) if total else 50)]
        rng.shuffle(t)
        return t

    for hits in (2, K.kHotMin, K.kHotMin + 1):
        send(batch({777: hits, 1024: hits}))
        assert w.check() > 2 * hits
    hot = list(range(300, n, (n - 300) // (K.kHotCtas + 8)))[:K.kHotCtas + 8]
    assert len(hot) == K.kHotCtas + 8
    send(batch({c: K.kHotMin + 1 + c % 3 for c in hot}))
    assert w.check() > (K.kHotCtas + 8) * (K.kHotMin + 1)
    big = 8192 + 808
    t = [rng.randrange(n) for _ in range(big)]
    t[8191] = t[8192] = 2121
    for j in range(0, big, 7):
        t[j] = 2121
    send(t)
    assert w.check() > big - 10
    for total in (K.kThinSeparateMin - 1, K.kThinSeparateMin):
        for with_bcast in (False, True):
            t = batch({3000: K.kHotMin + 9}, total)
            assert len(t) == total
            send(t[:total // 2])
            if with_bcast:
                w.bcast([0], raw(300, total))
            send(t[total // 2:])
            assert w.check() > total - 10
    w.e.close()
    assert w.guard.verified > 0


@pytest.mark.parametrize("staged", [False, True])
def test_device_parse_errors_write_nothing(pcdn, staged):
    """malformed and all-invalid-topic frames among valid ones: a message whose msg_status is not 0 stores nothing"""
    rng = random.Random(5)
    w = GuardedWorld(pcdn, n_valid_topics=8, max_conns=512, ring_bytes_per_conn=1 << 15,
                     flags=pcdn.FLAG_DEVICE_PARSE | (pcdn.FLAG_STAGED_SPANS if staged else 0))
    keys = [b"dp-user-%03d" % i for i in range(300)]
    for i, k in enumerate(keys):
        w.add_user(k, [0] + ([1 + i % 7] if i % 3 else []))
    errs = 0
    for batch in range(4):
        frames = []
        for j in range(80):
            pl = bytes([j]) * rng.choice([0, 10, 300, 1000])
            r = rng.random()
            if r < 0.4:
                fr = orc.broadcast_frame([rng.randrange(8)], pl)
            elif r < 0.6:
                fr = orc.broadcast_frame([rng.randrange(8, 200)] * 2, pl)        # only invalid topics
            else:
                fr = orc.direct_frame(rng.choice(keys), pl)
            if rng.random() < 0.2:
                fr = bytearray(fr)
                fr[rng.randrange(8, min(len(fr), 48))] ^= 0xFF
                fr = bytes(fr)
            sender = rng.choice(keys)
            frames.append((sender, 0, fr))
            w.o.user_receive(sender, fr)
        w.e.receive_frames(frames)
        assert w.check() > 0
        errs += w.e.last_result.n_msg_errors
    assert errs > 0
    w.e.close()


def test_e2big_batch_writes_nothing(pcdn):
    """a batch over max_batch_deliveries is rejected whole on the device: no byte of any ring changes, and
    the rings go on where they were"""
    w = GuardedWorld(pcdn, max_batch_deliveries=1000, max_conns=2048, ring_bytes_per_conn=4096)
    for i in range(1200):
        w.add_user(i.to_bytes(8, "little"), [0] + ([1] if i < 500 else []))
    for rnd in range(3):
        w.bcast([1], orc.broadcast_frame([1], b"fits" * (100 + rnd * 200)))
        assert w.check() == 500
    w.e.handle_broadcast_message([0], orc.broadcast_frame([0], b"too many recipients"))   # the oracle never sees it
    w.check()
    assert [r.status for r in w.drained] == [STATUS_E2BIG]
    for rnd in range(3):
        w.bcast([1], orc.broadcast_frame([1], b"more" * 300))
        assert w.check() == 500 and w.e.last_result.n_overflow == 0
    w.e.close()


# ------------------------------------------------------------------ batches in flight together
INFLIGHT_RING = 1 << 15          # 1024 units
INFLIGHT_REC = 3600              # raw bytes: 113 units, a connection-major record (<= kCmMaxBytes)


def inflight_world(pcdn, mode):
    """every user of the world receives exactly two INFLIGHT_REC records per batch, through one pack class:
    a dense group (topic 0, connection-major), 64 users on topic 1 (message-major), 4 on topic 2 (thin)
    and 5 that get directs.  Four batches take 904 of a ring's 1024 units, and with the wrap padding of
    less than one record they fill it; successive rounds wrap every ring."""
    cfg = dict(max_conns=1024, ring_bytes_per_conn=INFLIGHT_RING, batch_slots=4)
    if mode == "rings-regular":
        cfg.update(flags=pcdn.FLAG_STAGED_SPANS)
    elif mode == "pool":
        cfg.update(flags=pcdn.FLAG_OUTPUT_POOL, pool_bytes=16 << 20)
    elif mode == "host":
        cfg.update(flags=pcdn.FLAG_HOST_RINGS)
    elif mode == "shards":
        cfg.update(shard_cfg(pcdn, "shards-host"), max_conns=2048)
    w = GuardedWorld(pcdn, delivery="shared" if mode == "shared-payload" else "copy", **cfg)
    n_dense = (3 if mode == "shards" else 1) * w.e.shard_info(0).shard_stride >> K.kCmDenseShift
    for i in range(n_dense + 8):
        w.add_user(b"dense%05d" % i, [0])
    for i in range(64):
        w.add_user(b"fat%03d" % i, [1])
    for i in range(4):
        w.add_user(b"thin%d" % i, [2])
    for i in range(5):
        w.add_user(b"direct%d" % i, [])
    return w


def inflight_batch(w, rng, tag, rounds=1):
    """`rounds` times: two records for every user (connection-major, message-major, thin, direct), in a
    shuffled order, and a direct to an unknown key"""
    ops = []
    for _ in range(rounds):
        ops += [("b", [t]) for t in (0, 1, 2) for _ in range(2)]
        ops += [("d", b"direct%d" % i) for i in range(5) for _ in range(2)] + [("d", b"nobody")]
    rng.shuffle(ops)
    for kind, to in ops:
        tag += 1
        if kind == "b":
            w.bcast(to, raw(INFLIGHT_REC, tag))
        else:
            w.direct(to, raw(INFLIGHT_REC, tag))
    return w.launch()


@pytest.mark.parametrize("mode", ["rings-fused", "rings-regular", "pool", "host", "shards", "shared-payload"])
def test_four_batches_in_flight(pcdn, mode):
    """four batches launched and none polled, the newest polled first (so every pack has finished), then all
    read oldest first: each batch's records are still the oracle's after the later packs, nothing lands
    outside the spans, and the spans of the four never overlap.  Rings: the four batches fill every 32 KiB
    ring up to less than one record, and every round wraps it (shared payload: one-unit reference records,
    the same placement with room to spare).  Pool (16 MiB): the fourth batch of a round does not fit
    behind the other three and is refused until they are released; then a batch launched after a partial
    release wraps around the pool end while the batch before it is still live."""
    rng = random.Random(3)
    w = inflight_world(pcdn, mode)
    tag = 0
    wrapped = 0
    for cycle in range(3):
        bids = []
        for _ in range(4):
            tag += 1000
            bids.append(inflight_batch(w, rng, tag))
        assert w.check(first=[bids[-1]]) > 0
        assert len(w.drained) == 4 and all(r.status == 0 and not r.overflow for r in w.drained)
        if cycle and not w.guard.pool:     # (the first round starts at offset 0 of fresh rings)
            c = int(w.drained[0].shards[0].table[0, 0])
            wrapped += any(sp[0] == 0 for r in w.drained for sp in w.spans_of(r, c))   # back to offset 0 while live
    if mode != "pool":
        assert mode == "shared-payload" or wrapped >= 2, "the rings must wrap while four batches are live"
        w.e.close()
        return
    assert w.refusals == 3
    # two rounds (8.6 MB) and one (4.3 MB) fill the pool up to its last 3.9 MB; after the first batch is
    # released, the next (4.3 MB) no longer fits behind the second and wraps to the pool start
    b1 = inflight_batch(w, rng, tag + 1000, rounds=2)
    b2 = inflight_batch(w, rng, tag + 2000)
    got = {}
    r1 = w.step(b1, w.guard.tick())
    b3 = inflight_batch(w, rng, tag + 3000)
    t = w.guard.tick()
    r2 = w.step(b2, t)
    r3 = w.step(b3, t)
    for r in (r1, r2, r3):
        assert r.status == 0
        for c, fr in r.frames.items():
            got.setdefault(c, []).extend(fr)
    assert w.refusals == 3 and r3.shards[0].pool_base == 0 < r2.shards[0].pool_base, "the third region must wrap"
    w.compare(w.e, got, w.expect())
    w.guard.verify()
    w.e.close()


# ------------------------------------------------------------------ the overflow contract
@pytest.mark.parametrize("out", ["rings", "host"])
@pytest.mark.parametrize("ctrl", ["fused", "regular"])
@pytest.mark.parametrize("cls", ["thin", "fat", "cm", "direct"])
def test_drained_ring_takes_any_record_that_fits_it(pcdn, cls, ctrl, out):
    """move every target connection's tail to p, release everything, then send a record of u units with
    p < u <= R and p + u > R: it does not fit before the ring end, but the ring is empty, so it goes to
    offset 0.  More records of the same class then fill the ring to exactly R units in the same batch:
    all are delivered, as one span [0, R), and nothing overflows.  cls: the pack path of the records —
    thin (4 recipients), message-major (64), connection-major (dense, records <= kCmMaxBytes, so 4 KiB
    rings) or direct."""
    R = 4096 if cls == "cm" else 8192
    Ru = R // K.kUnit
    flags = (pcdn.FLAG_STAGED_SPANS if ctrl == "regular" else 0) | (pcdn.FLAG_HOST_RINGS if out == "host" else 0)
    w = GuardedWorld(pcdn, max_conns=1024, ring_bytes_per_conn=R, flags=flags)
    dense = w.e.shard_info(0).shard_stride >> K.kCmDenseShift
    keys = [b"t%05d" % i for i in range({"thin": 4, "fat": 64, "cm": dense + 8, "direct": 5}[cls])]
    targets = [w.add_user(k, [0]) for k in keys]
    for i in range(40):
        w.add_user(b"other%03d" % i, [1])
    p, u = (40, 96) if cls == "cm" else (100, 200)     # cm: 96 units = 3072 B <= kCmMaxBytes
    assert p < u <= Ru and p + u > Ru
    tag = [0]

    def send(n_units):
        tag[0] += 1
        body = raw(n_units * K.kUnit - 4, tag[0])
        if cls == "direct":
            for k in keys:
                w.direct(k, body)
        else:
            w.bcast([0], body)
        w.bcast([1], raw(100, tag[0]))                 # other connections' traffic in the same batch

    send(p)
    assert w.check() > 0
    send(u)
    rest = Ru - u
    while rest:
        send(min(rest, u))
        rest -= min(rest, u)
    assert w.check() > 0
    last = w.drained[-1]
    assert len(last.overflow) == 0, f"a drained ring overflowed: n_overflow == {len(last.overflow)}"
    for c in targets:
        assert [sp[:2] for sp in w.spans_of(last, c)] == [[0, R]], (c, w.spans_of(last, c))
    w.e.close()


def test_ref_threshold_engine_never_overflows_when_drained(pcdn):
    """ref_min_bytes at the largest value an 8 KiB ring allows (its largest copied record is the whole
    ring): 300 seeded batches, drained between batches, each one copy-sized message (up to the whole ring)
    followed by up to three reference-sized ones (one unit each) — no connection overflows, every stream is
    the oracle's"""
    R = 8192
    T = R - 3                    # round_up(4 + T - 1, 32) == R
    rng = random.Random(17)
    w = GuardedWorld(pcdn, max_conns=64, ring_bytes_per_conn=R, delivery=("ref", T))
    for i in range(48):
        w.add_user(b"r%03d" % i, [i % 3, 3])
    for batch in range(300):
        size = rng.choice([rng.randrange(0, T), rng.randrange(T // 2, T), T - 1])
        w.bcast([3] if rng.random() < 0.7 else [rng.randrange(3)], payload(rng, size)[:size])
        for _ in range(min(rng.randrange(0, 4), R // K.kUnit - units(size))):   # the batch fits one ring
            size = rng.randrange(T, T + 5000)
            w.bcast([rng.randrange(4)], payload(rng, size)[:size])
        w.check()
        assert all(not r.overflow for r in w.drained), f"batch {batch}: n_overflow == {len(w.drained[-1].overflow)}"
    w.e.close()


def uncovered(w, conn, lo, hi):
    """units [lo, hi) of conn's ring are covered by no span of any batch polled since the canary was laid
    (so verify() compares them with it)"""
    g = w.guard
    li = conn // g.stride - g.gindex[0]
    at = conn % g.stride * (g.R // K.kUnit)
    return int(g.coverage(li, list(g.batches.values()))[at + lo:at + hi].abs().sum()) == 0


def test_full_ring_overflows_a_prefix_and_spares_older_batches(pcdn):
    """batches A and B stay unreleased and hold 192 of the 256 units of every target's 8 KiB ring; batch C
    then sends three 48-unit records: the first fits at [192, 240), the second would need the 16 units to
    the ring end as padding and overflows.  Thin, message-major, connection-major and direct targets are
    all reported, C delivers exactly that one record, A's and B's records read back as the oracle's after
    C has packed, and the 16 units after C's record — in no span — still hold the canary"""
    w = GuardedWorld(pcdn, max_conns=1024, ring_bytes_per_conn=8192)
    dense = w.e.shard_info(0).shard_stride >> K.kCmDenseShift
    fat = [w.add_user(b"fat%03d" % i, [0]) for i in range(64)]
    cm = [w.add_user(b"cm%04d" % i, [3]) for i in range(dense + 8)]
    thin = w.add_user(b"thin", [1])
    dk = b"direct-target"
    dc = w.add_user(dk, [])
    other = w.add_user(b"bystander", [2])
    targets = fat + cm + [thin, dc]

    def batch(n, n_units, tag):
        for j in range(n):
            fr = raw(n_units * K.kUnit - 4, tag * 10 + j)
            for t in (0, 1, 3):
                w.bcast([t], fr)
            w.direct(dk, fr)
            w.bcast([2], raw(10, tag * 10 + j))
        return w.launch()

    a, b, c = batch(2, 64, 1), batch(1, 64, 2), batch(3, 48, 3)
    got = w.drain(first=[c])
    want = w.expect()
    ra, rb, rc = w.drained
    assert [r.bid for r in w.drained] == [a, b, c]
    assert not ra.overflow and not rb.overflow
    assert sorted(rc.overflow) == sorted(targets)
    for x in targets:
        assert ra.frames[x] + rb.frames[x] == want[x][:3], x          # A and B intact after C packed
        assert rc.frames[x] == want[x][3:4], x                        # the one record that still fits
        assert w.spans_of(rc, x) == [[192 * K.kUnit, 48 * K.kUnit, 1]], x
        assert uncovered(w, x, 240, 256), x
    assert got[other] == want[other]
    w.guard.verify()
    w.e.close()


@pytest.mark.parametrize("name", CM_MODES[:4], ids=[i.removeprefix("rings-") for i in CM_IDS[:4]])
def test_overflow_inside_a_connection_major_group_under_guard(pcdn, name):
    """test_gpu_cm_runs' overflow inside a group, drained under the guard: 20 connection-major records of 34
    units into 512-unit rings; 15 fit, the 16th overflows in the second group of kCmGroup, so the group's
    run must stop there: the 2 units after the 15th record of every dense connection still hold the canary"""
    w = cm_world(pcdn, name, GuardedWorld)
    conns = [w.add_user(b"dense%05d" % i, [0]) for i in range(CM_DENSE)]
    frames = [cm_frame([0], t) for t in range(20)]
    for f in frames:
        w.e.handle_broadcast_message([0], f)                 # (engine only: the oracle would deliver all 20)
    u = units(len(frames[0]))
    k = CM_RING // K.kUnit // u
    assert K.kCmGroup < k < 2 * K.kCmGroup and k * u < CM_RING // K.kUnit
    got = w.drain()
    rec, = w.drained
    assert sorted(rec.overflow) == sorted(conns)
    for c in conns:
        assert got[c] == frames[:k], c
        assert uncovered(w, c, k * u, CM_RING // K.kUnit), c
    w.guard.verify()
    w.e.close()
    assert w.guard.verified > 0
