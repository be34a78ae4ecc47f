"""Support for the GPU tests (not a test module): the engine-plus-oracle World and the worlds built on it, the
engine layouts and delivery modes they run on, the record format of a span, and helpers that several test
modules use.  Importing it needs no GPU: the CPU tests take the error codes and the oracle's broker sends from here.

Assertions here carry explicit messages: pytest rewrites `assert` only in test modules."""
import ctypes as C
import os
import random
import socket
import struct
import threading
import time

import numpy as np
import pytest

from kconst import K
from oracle import oracle as orc

# pcdn_status return codes (negative, as the calls return or raise them) ...
PCDN_EINVAL, PCDN_ENODEV, PCDN_ENOSPC, PCDN_EPARSE, PCDN_EPRUNE, PCDN_ENOENT, PCDN_EAGAIN = -1, -3, -5, -7, -8, -10, -11
# ... and pcdn_batch_result.status of a refused batch (the same codes as positive numbers)
STATUS_EAGAIN, STATUS_E2BIG = 11, 12


# ------------------------------------------------------------------ engine layouts
# name -> (pcdn FLAG_* names, shards: None, "host" = three shards on GPU 0, "nccl" = one shard per GPU).  Sizes
# (pool_bytes, ring_bytes_per_conn, max_conns) are not part of a layout: each workload keeps its own.
LAYOUTS = {
    "rings": ((), None),
    "staged": (("STAGED_SPANS",), None),                  # the regular control kernels on a small engine
    "runs": (("SPAN_RUNS",), None),
    "runs-staged": (("SPAN_RUNS", "STAGED_SPANS"), None),
    "host": (("HOST_RINGS",), None),
    "devparse": (("DEVICE_PARSE",), None),
    "devparse-staged": (("DEVICE_PARSE", "STAGED_SPANS"), None),
    "pool": (("OUTPUT_POOL",), None),
    "pool-staged": (("OUTPUT_POOL", "STAGED_SPANS"), None),
    "pool-staged-runs": (("OUTPUT_POOL", "STAGED_SPANS", "SPAN_RUNS"), None),
    "pool-host": (("OUTPUT_POOL", "HOST_RINGS"), None),
    "shards-host": ((), "host"),
    "shards-host-staged": (("STAGED_SPANS",), "host"),
    "shards-nccl": ((), "nccl"),
    "pool-shards-host": (("OUTPUT_POOL",), "host"),
    "pool-shards-host-staged": (("OUTPUT_POOL", "STAGED_SPANS"), "host"),
    "pool-runs-shards-nccl": (("OUTPUT_POOL", "SPAN_RUNS"), "nccl"),
}


def layout(pcdn, name):
    """the engine keywords of a named layout: `flags` when it sets any, `devices` and `ingest` when it is sharded
    (skipped below two GPUs for the NCCL layouts)"""
    flag_names, shards = LAYOUTS[name]
    kw = {}
    flags = 0
    for f in flag_names:
        flags |= getattr(pcdn, "FLAG_" + f)
    if flags:
        kw["flags"] = flags
    if shards:
        kw.update(shard_cfg(pcdn, "shards-" + shards))
    return kw


def shard_cfg(pcdn, variant):
    """engine config of the sharded variants: 'shards-host' = three connection shards that share GPU 0
    (every shard copies the batch from pinned host memory: runs on a one-GPU box); 'shards-nccl' = one
    shard per GPU, the library moves every batch with ncclBroadcast (needs >= 2 GPUs)"""
    import torch

    if variant == "shards-host":
        return dict(devices=[0, 0, 0], ingest=pcdn.INGEST_HOST)
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    return dict(devices=list(range(min(n, 4))), ingest=pcdn.INGEST_NCCL)


# ------------------------------------------------------------------ delivery
def largest_threshold(cap):
    """the largest ref_min_bytes an engine whose ring (or pool) holds `cap` bytes admits: the largest copied
    record, round_up(4 + T - 1, 32), must fit it"""
    return cap - 3


def config_default(pcdn):
    cfg = pcdn.Config()
    pcdn.lib().pcdn_config_default(C.byref(cfg))
    return cfg


def engine(pcdn, delivery="copy", **kw):
    """pcdn.Engine(**kw) with the delivery mode applied to its final keywords: "copy" leaves them as they are,
    "shared" adds FLAG_SHARED_PAYLOAD (every delivery a reference record), ("ref", T) sets ref_min_bytes to T or
    to the largest threshold the engine's ring admits when that is smaller (output pool: the pool, or max_conns
    rings when pool_bytes is not set; pcdn_config_default fills what kw leaves out)"""
    if delivery == "shared":
        kw["flags"] = kw.get("flags", 0) | pcdn.FLAG_SHARED_PAYLOAD
    elif delivery != "copy":
        kind, threshold = delivery
        assert kind == "ref", f"unknown delivery {delivery!r}"
        d = config_default(pcdn)
        cap = kw.get("ring_bytes_per_conn", d.ring_bytes_per_conn)
        if kw.get("flags", 0) & pcdn.FLAG_OUTPUT_POOL:
            cap = kw.get("pool_bytes") or kw.get("max_conns", d.max_conns) * cap
        kw["ref_min_bytes"] = min(threshold, largest_threshold(cap))
    e = pcdn.Engine(**kw)
    by_ref = e.delivers_by_ref()
    if by_ref != (delivery != "copy"):
        e.close()
        raise AssertionError(f"delivery {delivery!r}: the engine delivers_by_ref() == {by_ref}")
    return e


# ------------------------------------------------------------------ the differential harness
class World:
    """drives engine and oracle with identical calls and compares delivered frames
    (record=True: also keeps the engine calls and the oracle's frames of every check(), so that
    replay() can run the same workload on engines of other configurations against this ONE oracle run)"""

    def __init__(self, pcdn, n_valid_topics=0, record=False, delivery="copy", **cfg):
        kw = dict(max_conns=8192, max_topics=256, max_keys=16384, ring_bytes_per_conn=1 << 18,
                  max_batch_msgs=4096, max_batch_bcast=512, max_batch_bytes=32 << 20,
                  max_batch_deliveries=1 << 20, identity="/", n_valid_topics=n_valid_topics)
        kw.update(cfg)
        self.pcdn = pcdn
        self.cfg = kw
        self.delivery = delivery
        self.e = engine(pcdn, delivery, **kw)
        self.o = orc.Oracle("/", n_valid_topics)
        self.map = {}
        self.taken = {}
        self.calls = [] if record else None

    def _engine(self, name, *a):
        r = getattr(self.e, name)(*a)
        if self.calls is not None:
            self.calls.append((name, a, r))
        return r

    def add_user(self, key, topics):
        c = self._engine("add_user", key, topics)
        self.map[c] = self.o.add_user(key, topics)
        return c

    def add_broker(self, ident, topics=()):
        c = self._engine("add_broker", ident)
        self.map[c] = self.o.add_broker(ident)
        if topics:
            self.both("subscribe_broker_to", ident, list(topics))
        return c

    def both(self, name, *a):
        self._engine(name, *a)
        getattr(self.o, name)(*a)

    def bcast(self, topics, raw, to_users_only=False):
        self.both("handle_broadcast_message", topics, raw, to_users_only)

    def direct(self, rcpt, raw, to_user_only=False):
        self.both("handle_direct_message", rcpt, raw, to_user_only)

    def expect(self):
        """oracle frames per ENGINE conn id since the last call"""
        out = {}
        for ec, oc in self.map.items():
            fr = self.o.frames(oc)
            k = self.taken.get(oc, 0)
            if len(fr) > k:
                out[ec] = fr[k:]
            self.taken[oc] = len(fr)
        return out

    def check(self):
        got = self.e.drain()
        want = self.expect()
        if self.calls is not None:
            self.calls.append(("check", (), want))
        return self.compare(self.e, got, want)

    def replay(self, **cfg):
        """the recorded engine calls on a fresh engine configured like this one updated by `cfg` (and delivering
        like it); every batch must deliver the oracle frames recorded for it"""
        e = engine(self.pcdn, self.delivery, **{**self.cfg, **cfg})
        try:
            for name, a, r in self.calls:
                if name == "check":
                    self.compare(e, e.drain(), r)
                else:
                    assert getattr(e, name)(*a) == r, name
        finally:
            e.close()

    def compare(self, e, got, want):
        bad = [c for c in sorted(set(got) | set(want)) if got.get(c, []) != want.get(c, [])]
        if bad:
            self.dump(e, bad, got, want)
        assert set(got) == set(want), (sorted(set(got) ^ set(want))[:10])
        for c in want:
            assert len(got[c]) == len(want[c]), (c, len(got[c]), len(want[c]))
            for i, (g, w) in enumerate(zip(got[c], want[c])):
                assert g == w, f"conn {c} frame {i}: {len(g)} vs {len(w)} bytes"
        return sum(len(v) for v in want.values())

    def dump(self, e, bad, got, want):
        """diagnostics for a failing comparison (pytest shows them with the failure)"""
        import sys
        f = sys.stdout
        f.write(f"==== {len(bad)} bad connections of {len(want)}; first: {bad[:20]}\n")
        r = e.last_result
        f.write(f"last batch: msgs={r.n_msgs} deliveries={r.n_deliveries} spans={r.n_spans} overflow={r.n_overflow} "
                f"dropped={r.n_direct_dropped} status={r.status}\n")
        for c in bad[:6]:
            g, w = got.get(c, []), want.get(c, [])
            f.write(f"conn {c}: got {len(g)} frames, want {len(w)}\n")
            sig = lambda fr: (len(fr), fr[:4].hex(), fr[-12:].hex())
            f.write("  got : " + " ".join(str(sig(x)) for x in g[:40]) + "\n")
            f.write("  want: " + " ".join(str(sig(x)) for x in w[:40]) + "\n")
            for i, (a, b) in enumerate(zip(g, w)):
                if a != b and len(a) == len(b):
                    d = next(k for k in range(len(a)) if a[k] != b[k])
                    f.write(f"  frame {i}: same length {len(a)}, first diff at byte {d}: {a[d:d+16].hex()} vs {b[d:d+16].hex()}\n")
                    break


def payload(rng, n):
    return bytes(rng.getrandbits(8) for _ in range(min(n, 64))) * (n // 64 + 1)


def wire(frames):
    """what the writer task sends for these raw frames"""
    return b"".join(len(f).to_bytes(4, "big") + f for f in frames)


# ------------------------------------------------------------------ records
def ref_record(raw_len, off, batch_id):
    """the model of a reference record (include/pcdn_fanout.h)"""
    return b"\xff\xff\xff\xff" + raw_len.to_bytes(4, "big") + struct.pack("<QQ", off, batch_id) + bytes(8)


def records(data, n_records, batch_id=None):
    """the n_records records of a span's bytes, each a copied frame (bytes) or a reference (raw length, offset in
    the batch's payload, batch id): a framed record is the u32 BE length and the frame padded to 32 bytes, a
    reference record 32 bytes that start with the 0xFFFFFFFF marker and end with 8 zero bytes.  The records must
    fill the span exactly; batch_id: every reference must name that batch"""
    out, p = [], 0
    for _ in range(n_records):
        L = int.from_bytes(data[p:p + 4], "big")
        if L == 0xFFFFFFFF:
            L = int.from_bytes(data[p + 4:p + 8], "big")
            off, bid = struct.unpack("<QQ", data[p + 8:p + 24])
            assert data[p + 24:p + 32] == bytes(8), f"reference record at byte {p}: non-zero tail"
            assert batch_id is None or bid == batch_id, f"reference record at byte {p}: batch id {bid}, not {batch_id}"
            out.append((L, off, bid))
            p += 32
        else:
            out.append(bytes(data[p + 4:p + 4 + L]))
            p += (4 + L + 31) // 32 * 32
    assert p == len(data), f"the records end at byte {p} of a {len(data)}-byte span"
    return out


def frames(recs, payload_base=None):
    """the frames a writer emits for records(): a reference resolved in the batch's payload at payload_base"""
    out = []
    for r in recs:
        if isinstance(r, tuple):
            assert payload_base is not None, "a reference record without the batch's payload"
            r = C.string_at(payload_base + r[1], r[0])
        out.append(r)
    return out


def chunk_streams(chunk, out, payload_base=None, batch_id=None):
    """walk an egress chunk (host memory) record by record and append each connection's wire bytes to
    out[conn]; references are resolved in the batch's payload (payload_base, batch_id)"""
    for i in range(chunk.n_spans):
        sp = chunk.spans[i]
        recs = records(C.string_at(chunk.data + chunk.data_off[i], sp.len), sp.n_records, batch_id)
        out.setdefault(sp.conn, bytearray()).extend(wire(frames(recs, payload_base)))


# ------------------------------------------------------------------ the broker's own frames
def relay_key(ident):
    """a DirectMap key owned by peer broker `ident` (no user key of these tests starts with 0xFF 0x00)"""
    return b"\xff\x00send-to:" + ident.encode()


def try_send_to_broker(o, ident, raw):
    """Inner::try_send_to_broker (cdn-broker/src/tasks/broker/sender.rs:17-45) on oracle `o`; 1 = no such broker
    (nothing sent).  The frame goes through the oracle's own send path: handle_direct_message
    (tasks/broker/handler.rs:197-237) of a key that `ident` owns ends in try_send_to_broker(ident) →
    send_message_raw on that broker's connection, so the frame takes its place in the broker's stream in call
    order with everything routed to it."""
    if o.broker_conn(ident) < 0:
        return 1                                       # if let Some(connection) = connection (sender.rs:29)
    key = relay_key(ident)
    o.apply_user_sync(ident, [(key, 1, ident)])        # (no local user has the key: nobody is removed)
    o.handle_direct_message(key, raw)
    return 0


def try_send_to_brokers(o, idents, raw):
    """Inner::try_send_to_brokers (sender.rs:49-59): try_send_to_broker for every connected broker.  `idents`: the
    identifiers ever added (the oracle does not list its brokers); 1 = none of them is connected."""
    live = [i for i in dict.fromkeys(idents) if o.broker_conn(i) >= 0]
    for i in live:
        try_send_to_broker(o, i, raw)
    return 0 if live else 1


class Sends:
    """a World (or one of its subclasses) that also sends the broker's own frames: the engine's
    pcdn_send_to_broker(s) against try_send_to_broker(s) on its oracle"""

    def add_broker(self, ident, topics=()):
        self.__dict__.setdefault("idents", []).append(ident)
        return super().add_broker(ident, topics)

    def send(self, ident, raw):
        """send_to_broker(ident, raw), or send_to_brokers(raw) with ident None, on both; the results must agree"""
        if ident is None:
            r, ro = self._engine("send_to_brokers", raw), try_send_to_brokers(self.o, self.__dict__.get("idents", []), raw)
        else:
            r, ro = self._engine("send_to_broker", ident, raw), try_send_to_broker(self.o, ident, raw)
        assert r == ro, (ident, r, ro)
        return r


def user_sync(tag, n=300):
    return orc.serialize(orc.KIND_USER_SYNC, b"", bytes([tag % 256]) * n)


# ------------------------------------------------------------------ a small output pool with a hot connection
HOT = b"hot-connection"


class PoolWorld(World):
    """a World on a small output pool, with 300 users on topics 0 / 1, a hot user and a peer broker
    (layout: "one-shard" or "shards-host")"""

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
        assert r.status == 0 and r.n_overflow == 0, (r.status, r.n_overflow)
        self.e.last_result = r                                # (World.dump reports it on a mismatch)
        for c, fr in self.e.collect_frames(r).items():
            got.setdefault(c, []).extend(fr)
        self.e.release_batch(b)
        return r


# ------------------------------------------------------------------ sockets of the egress writer
BIG = 64 << 20
IDLE_LIMIT = 60.0   # a stalled reader starts by itself after this long, so a writer that waits still ends


def backlog_world(pcdn, name, delivery="copy", **extra):
    """the egress backlog tests' World on layout `name`: 1 MiB rings (a 64 MiB pool), two batch slots"""
    cfg = dict(max_conns=1024, ring_bytes_per_conn=1 << 20, max_batch_bytes=8 << 20, batch_slots=2, **layout(pcdn, name))
    if name.startswith("pool"):
        cfg["pool_bytes"] = 64 << 20
    cfg.update(extra)
    return World(pcdn, delivery=delivery, **cfg)


class Reader:
    """the receiving end of a socketpair / pipe, read by a thread that starts when go() is called (or
    by itself after IDLE_LIMIT seconds: then `late` is set and the test fails)"""

    def __init__(self, fd, started=True):
        self.fd, self.buf, self.late = fd, bytearray(), False
        self.ev = threading.Event()
        if started:
            self.ev.set()
        self.th = threading.Thread(target=self._run, daemon=True)
        self.th.start()

    def _run(self):
        if not self.ev.wait(IDLE_LIMIT):
            self.late = True
        while True:
            try:
                d = os.read(self.fd, 65536)
            except OSError:
                return
            if not d:
                return
            self.buf.extend(d)

    def go(self):
        self.ev.set()

    def wait_for(self, n, eg=None, timeout=30.0):
        """the bytes read once n have arrived (eg: moving backlogs on meanwhile, as a host would)"""
        t = time.time() + timeout
        while len(self.buf) < n and time.time() < t:
            if eg is not None:
                eg.flush_backlog(0)
            time.sleep(0.005)
        return bytes(self.buf)

    def finish(self, timeout=30.0):
        self.th.join(timeout)
        assert not self.th.is_alive(), "the reader thread did not end"
        return bytes(self.buf)


def sock_pair(sndbuf=1 << 20):
    """4096: a stalled peer's buffer; the default asks for 1 MiB (the kernel caps it at its
    wmem_max, then doubles it), more than one batch's bytes for a peer read by a thread"""
    s, r = socket.socketpair()
    s.setsockopt(socket.SOL_SOCKET, socket.SO_SNDBUF, sndbuf)
    return s, r


def flush_until_done(eg, timeout=30.0):
    t = time.time() + timeout
    while eg.flush_backlog(100) and time.time() < t:
        pass
    return eg.flush_backlog(0)


# ------------------------------------------------------------------ a world whose every slot is a user
TILE_BYTES = K.kFatTileBytes   # bytes of stores a message-major tile aims at
EDGE_SLOTS = 2 * 32 * K.kBlockWords   # two match blocks


def vec_bytes(raw_len):
    return (4 + raw_len + 15) // 16 * 16


def units(raw_len):
    return (4 + raw_len + K.kUnit - 1) // K.kUnit


def tile_recipients(raw_len):
    return max(32, min(K.kTileRecipients, TILE_BYTES // min(vec_bytes(raw_len), K.kChunkBytes)))


def raw(n, tag):
    """n bytes that differ from vector to vector and from message to message"""
    return ((np.arange(n, dtype=np.int64) * 7 + tag * 13) % 251).astype(np.uint8).tobytes()


def edge_sizes():
    """raw lengths around every size threshold of the pack: b - 4, b - 1, b, b + 1, b + 4 (the 4-byte length
    prefix moves the 16-byte vector and 32-byte unit steps)"""
    out = set()
    for b in (K.kCmMaxBytes - 4,                   # largest record on the connection-major path
              K.kChunkBytes - 4,                   # one staging chunk
              2 * K.kChunkBytes - 4):              # two chunks
        out.update((b - 4, b - 1, b, b + 1, b + 4))
    return sorted(out)


def edge_conns(n):
    """k_offsets CTA (256), connection-major tile (32 * kCmTileWords), match block (32 * kBlockWords) edges"""
    tile, blk = 32 * K.kCmTileWords, 32 * K.kBlockWords
    return sorted({0, 255, 256, 257, tile - 1, tile, tile + 1, blk - 1, blk, blk + 1, n - 1})


def recipient_counts(n):
    dense = n >> K.kCmDenseShift
    out = {K.kFatMin - 1, K.kFatMin, K.kFatMin + 1, dense - 1, dense, dense + 1}
    for s in edge_sizes():
        out.update((tile_recipients(s), tile_recipients(s) + 1))
    return sorted(out)


def edge_world(pcdn, world=World, **cfg):
    """a `world` with EDGE_SLOTS users (connection c = user c); topic i reaches exactly recipient_counts()[i]
    users, every edge connection among them.  → (world, keys, {recipient count: topic})"""
    kw = dict(max_conns=EDGE_SLOTS, max_keys=EDGE_SLOTS + 1024, ring_bytes_per_conn=1 << 19)
    kw.update(cfg)
    w = world(pcdn, **kw)
    n = w.e.shard_info(0).shard_stride
    assert n == EDGE_SLOTS, (n, EDGE_SLOTS)
    rng = random.Random(1)
    edges = edge_conns(n)
    others = sorted(set(range(n)) - set(edges))
    subs = [[] for _ in range(n)]
    counts = recipient_counts(n)
    for t, d in enumerate(counts):
        for c in edges + rng.sample(others, d - len(edges)):
            subs[c].append(t)
    keys = [c.to_bytes(4, "little") + b"edge" for c in range(n)]
    kb = np.frombuffer(b"".join(keys), dtype=np.uint8).reshape(n, 8)
    offs = np.concatenate([[0], np.cumsum([len(s) for s in subs])]).astype(np.uint32)
    tp = np.array([t for s in subs for t in s], dtype=np.uint16)
    assert np.array_equal(w.e.add_users_bulk(kb, 8, tp, offs), np.arange(n)), "bulk-added users are not connections 0..n-1"
    for c in range(n):
        w.map[c] = w.o.add_user(keys[c], subs[c])
    return w, keys, {d: t for t, d in enumerate(counts)}


def check(w):
    """w.check(), after which the oracle forgets the frames it compared (it would copy its whole streams again
    at every later check)"""
    n = w.check()
    w.o.clear()
    w.taken.clear()
    return n


def span_table(res):
    """every span of a batch as int64 rows (conn, ring_off, len, n_records) sorted by connection and offset;
    the run-length form expanded (entry k of a run: conn0 + k at ring_off + k * off_stride)"""
    if res.n_spans == 0:
        return np.zeros((0, 4), dtype=np.int64)
    u32 = C.POINTER(C.c_uint32)
    if res.runs:
        r = np.ctypeslib.as_array(C.cast(res.runs, u32), shape=(res.n_runs, 6)).astype(np.int64)
        n = r[:, 1]
        k = np.arange(int(n.sum())) - np.repeat(np.cumsum(n) - n, n)
        t = np.stack([np.repeat(r[:, 0], n) + k, np.repeat(r[:, 2], n) + k * np.repeat(r[:, 5], n),
                      np.repeat(r[:, 3], n), np.repeat(r[:, 4], n)], axis=1)
    else:
        t = np.ctypeslib.as_array(C.cast(res.spans, u32), shape=(res.n_spans, 4)).astype(np.int64)
    assert len(t) == res.n_spans, (len(t), res.n_spans)
    return t[np.lexsort((t[:, 1], t[:, 0]))]


# ------------------------------------------------------------------ connection-major groups that are not one run
CM_DENSE = 2048    # users on topic 0: at least N/16 of every shard's 8192 slots, so topic 0 is connection-major
CM_RING = 1 << 14  # 15 records of a 1 KiB frame: the third batch of 8 wraps inside its group
# rings / pool x fused / regular control x one shard / three; the first four are the rings
CM_MODES = ["rings", "shards-host", "staged", "shards-host-staged",
            "pool", "pool-shards-host", "pool-staged", "pool-shards-host-staged"]
CM_IDS = ["%s-%s-%dshard" % (out, ctrl, shards) for out in ("rings", "pool") for ctrl in ("fused", "regular") for shards in (1, 3)]


def cm_frame(topics, tag, size=1000):
    return orc.broadcast_frame(topics, bytes((tag * 7 + i) & 0xFF for i in range(size)))


def cm_world(pcdn, name, world=World):
    kw = dict(flags=0, ring_bytes_per_conn=CM_RING, pool_bytes=1 << 28, max_conns=8192)
    kw.update(layout(pcdn, name))
    return world(pcdn, **kw)
