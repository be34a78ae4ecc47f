"""The kernels at the thresholds where they change code path, at launch geometries other than the
engine's defaults, and the output pool at the size it was built for — bit-exact through the C ABI
against the oracle, or against an exact numpy model where the oracle would be too slow.

Every threshold comes from kernels.cuh through kconst.K, so the cases stay on both sides of a limit
when it is retuned."""
import random

import numpy as np
import pytest

from gpu_world import EDGE_SLOTS, World, check, edge_sizes, edge_world, raw, records, span_table, units
from kconst import K
from oracle import oracle as orc

pytestmark = pytest.mark.gpu


PACK_MODES = [(out, ctrl) for out in ("rings", "pool") for ctrl in ("fused", "regular")]


@pytest.mark.parametrize("out,ctrl", PACK_MODES, ids=["-".join(m) for m in PACK_MODES])
def test_pack_size_and_recipient_boundaries(pcdn, out, ctrl):
    """every raw length of edge_sizes() to every recipient count of recipient_counts(): thin / fat / dense
    (connection-major) classes, message-major tile edges, the staging-chunk edges; then connection-major
    groups of 7, 8, 9 and 17 records of the largest connection-major size (8 of them fill the staging
    buffer exactly).  Recipients sit on the k_offsets CTA, connection-major tile and match-block edges.
    Small batches on a small engine take the fused control kernel; FLAG_STAGED_SPANS forces the regular
    pipeline (k_pool_finish on 2 CTAs for the pool)."""
    flags = (pcdn.FLAG_OUTPUT_POOL if out == "pool" else 0) | (pcdn.FLAG_STAGED_SPANS if ctrl == "regular" else 0)
    w, keys, topic = edge_world(pcdn, flags=flags, pool_bytes=1 << 30)
    n = EDGE_SLOTS
    dense = n >> K.kCmDenseShift
    tag = 0
    for s in edge_sizes():
        for d, t in topic.items():
            tag += 1
            w.bcast([t], raw(s, tag))
        assert check(w) == sum(topic)
    cm_len = K.kCmMaxBytes - 4
    for g in (K.kCmGroup - 1, K.kCmGroup, K.kCmGroup + 1, 2 * K.kCmGroup + 1):
        for i in range(g):
            tag += 1
            w.bcast([topic[dense + i % 2]], raw(cm_len, tag))
        assert check(w) == sum(dense + i % 2 for i in range(g))
    w.e.close()


def test_direct_thresholds(pcdn):
    """direct messages on the regular pipeline: 2, kHotMin and kHotMin + 1 hits on one connection (in-place
    insertion sort in k_offsets vs k_dsort_hot), kHotCtas + 8 hot connections (k_dsort_hot's grid-stride
    loop), a batch of more than 8192 messages (k_dsort_hot carries its count across 256-word passes of
    the bitmap) whose hot recipient has hits on both sides of message 8192, kThinSeparateMin - 1 and
    kThinSeparateMin directs (the separate k_pack_direct launch; alone, the batch moves to the pack
    stream) with and without one broadcast; every batch hits connections on the 1024-entry tile edges of
    k_dscan and the last slot.  Per-connection order is batch order (R9)."""
    w, keys, topic = edge_world(pcdn, flags=pcdn.FLAG_STAGED_SPANS, max_batch_msgs=12288, ring_bytes_per_conn=1 << 18)
    n = EDGE_SLOTS
    rng = random.Random(9)
    edges = [1023, 1024, 1025, n - 1]
    seq = [0]

    def send(targets):
        for c in targets:
            seq[0] += 1
            k = keys[c] if c is not None else b"nobody%d" % seq[0]
            w.direct(k, orc.direct_frame(k, seq[0].to_bytes(4, "little") * rng.randrange(1, 24)))

    def batch(hot, total=0):
        """hits on the hot connections, the edges and unknown keys, filled up to `total` (default: 50 more)"""
        t = [c for c, h in hot.items() for _ in range(h)] + edges + [None] * 3
        t += [rng.randrange(n) for _ in range(total - len(t) if total else 50)]
        rng.shuffle(t)
        return t

    for hits in (2, K.kHotMin, K.kHotMin + 1):
        send(batch({777: hits, 1024: hits}))
        assert check(w) > 2 * hits
    send(batch({c: K.kHotMin + 1 + c % 3 for c in range(300, n, (n - 300) // (K.kHotCtas + 8))[:K.kHotCtas + 8]}))
    assert check(w) > (K.kHotCtas + 8) * (K.kHotMin + 1)
    big = 8192 + 808
    t = [rng.randrange(n) for _ in range(big)]
    t[8191] = t[8192] = 4242
    for j in range(0, big, 7):
        t[j] = 4242
    send(t)
    assert check(w) > big - 10
    for total in (K.kThinSeparateMin - 1, K.kThinSeparateMin):
        for with_bcast in (False, True):
            t = batch({5000: K.kHotMin + 9}, total)
            assert len(t) == total
            send(t[:total // 2])
            if with_bcast:
                w.bcast([topic[K.kFatMin]], raw(300, total))
            send(t[total // 2:])
            assert check(w) > total - 10
    w.e.close()


# ------------------------------------------------------------------ launch geometry
# pack_variant (decoded by pcdn_create): bits 8-11 k_pack CTAs per SM, 12-15 k_pack_direct CTAs per SM
GEOMETRY = {
    "pack-1cta": 1 << 8, "pack-2cta": 2 << 8, "pack-3cta": 3 << 8, "pack-4cta": 4 << 8, "pack-6cta": 6 << 8,
    "pack-8cta": 8 << 8, "direct-1cta": 1 << 12, "direct-8cta": 8 << 12,
}


@pytest.mark.parametrize("out", ["rings", "pool"])
def test_cta_count_invariance(pcdn, out):
    """one workload that reaches every pack phase — connection-major, message-major over several chunks,
    dense message-major, thin, >= kThinSeparateMin directs with a hot recipient, unknown keys, three
    batches so that the rings wrap — checked against ONE oracle run on the default engine and on engines
    with other grid sizes: persistent-CTA phases must write the same bytes whatever the grid."""
    cfg = dict(ring_bytes_per_conn=1 << 18)
    if out == "pool":
        cfg.update(flags=pcdn.FLAG_OUTPUT_POOL, pool_bytes=1 << 28)
    w = World(pcdn, record=True, **cfg)
    rng = random.Random(31)
    keys = [i.to_bytes(8, "little") * 2 for i in range(3000)]
    for i, k in enumerate(keys):
        w.add_user(k, [0] + ([1] if i % 9 == 0 else []) + ([2 + i % 40] if i % 50 == 0 else []))
    hot = keys[17]
    tag = 0
    for b in range(3):
        ops = [("b", [0], rng.randrange(100, K.kCmMaxBytes - 4)) for _ in range(10)]       # connection-major
        ops += [("b", [1], s) for s in (K.kChunkBytes + 1, 2 * K.kChunkBytes + 3000, 20000)]   # message-major, 2-3 chunks
        ops += [("b", [0], K.kCmMaxBytes + 900)]                                         # dense message-major
        ops += [("b", [2 + rng.randrange(40)], rng.randrange(0, 3000)) for _ in range(20)]  # thin
        ops += [("d", hot if j % 7 == 0 else rng.choice(keys) if j % 20 else b"unknown%d" % j, rng.randrange(4, 200))
                for j in range(K.kThinSeparateMin + 50)]
        rng.shuffle(ops)
        for kind, to, size in ops:
            tag += 1
            if kind == "b":
                w.bcast(to, raw(size, tag))
            else:
                w.direct(to, orc.direct_frame(to, raw(size, tag)))
        assert w.check() > 30000
    for name, v in GEOMETRY.items():
        try:
            w.replay(pack_variant=v)
        except AssertionError as ex:
            raise AssertionError(f"pack_variant {name} ({v:#x}): {ex}") from ex
    w.e.close()


# ------------------------------------------------------------------ output pool at full size
FULL_SLOTS = (1 << 20) + 65536   # 136 x 8192: the k_pool_finish grid is min(SMs, slots / 8192) = every SM


def read_frames(e, res, t, conn, pool):
    """the frames a socket writer would send for `conn` (pcdn_read of its spans; a wrapped ring's piece
    that does not start at offset 0 comes first)"""
    lo, hi = np.searchsorted(t[:, 0], [conn, conn + 1])
    pieces = sorted(t[lo:hi, 1:].tolist(), key=lambda p: (p[0] == 0 and hi - lo > 1, p[0]))
    out = []
    for off, ln, nrec in pieces:
        out += records(e.read(conn, res.pool_base + off if pool else off, ln), nrec)
    return out


@pytest.mark.parametrize("out", ["pool", "pool-runs", "rings-runs"])
def test_full_size_output_pool(pcdn, out):
    """FULL_SLOTS connection slots, every one a user: traffic differs from k_offsets CTA to CTA (every 5th /
    11th / 97th connection on three topics, whole CTAs and whole 8192-blocks without subscribers) and a few
    directs.  Pool engines run k_pool_finish on one CTA per SM; the batch counters, the whole expanded span
    table (pool: a connection's region starts at the exclusive prefix of the units in connection order)
    and the region size (the next batch starts right after it) must equal the numpy model, the bytes of
    every k_offsets CTA's first and last connection must be the model's frames and those of a ~3000-user
    sample the oracle's.  The pool holds 2.5 batches: the third of three in flight is refused and retried,
    a later one wraps around the pool end.  rings-runs: per-connection 8 KiB rings (they wrap) with the
    run-length span table."""
    pool = out.startswith("pool")
    flags = (pcdn.FLAG_OUTPUT_POOL if pool else 0) | (pcdn.FLAG_SPAN_RUNS if out.endswith("runs") else 0)
    c = np.arange(FULL_SLOTS, dtype=np.int64)
    live = (c >> 8) % 13 != 6                                     # every 13th k_offsets CTA: nobody subscribed
    t1 = live & (c % 5 == 0) & ((c >> 8) % 7 != 3)
    t2 = live & np.isin(c % 11, (1, 2)) & ((c >> 13) % 3 != 1)    # whole match blocks without topic 2
    t3 = live & (c % 97 == 5)
    n_full = FULL_SLOTS
    # one batch: (kind, topics or target connection, raw length); the model's recipients of each message
    plan = [("b", [1], 300), ("d", n_full - 1, 100), ("b", [2], 500), ("d", 8192, 700), ("b", [1, 2], 60),
            ("d", 1 << 20, 40), ("b", [3], 3000), ("d", 37, 10), ("d", 37, 20)]
    masks = {1: t1, 2: t2, 3: t3}
    U = np.zeros(n_full, dtype=np.int64)
    R = np.zeros(n_full, dtype=np.int64)
    n_del = n_bytes = 0
    for kind, to, size in plan:
        m = np.zeros(n_full, dtype=bool)
        if kind == "b":
            for x in to:
                m |= masks[x]
        else:
            m[to] = True
        U += m * units(size)
        R += m
        n_del += int(m.sum())
        n_bytes += int(m.sum()) * (4 + size)
    total_units = int(U.sum())
    cfg = dict(max_conns=FULL_SLOTS, max_keys=FULL_SLOTS + 4096, max_batch_msgs=64, max_batch_bcast=16,
               max_batch_deliveries=1 << 21, batch_slots=3, flags=flags)
    if pool:
        cfg.update(pool_bytes=(total_units * 5 // 2) * K.kUnit)
    else:
        cfg.update(ring_bytes_per_conn=8192)
    w = World(pcdn, **cfg)
    e = w.e
    assert e.shard_info(0).shard_stride == FULL_SLOTS
    keys = np.zeros((n_full, 8), dtype=np.uint8)
    keys[:, :4] = c.astype(np.uint32).view(np.uint8).reshape(n_full, 4)
    keys[:, 7] = 0xEE
    sub = np.stack([t1, t2, t3], axis=1)
    topics = np.tile(np.array([1, 2, 3], dtype=np.uint16), n_full)[sub.ravel()]
    offs = np.concatenate([[0], np.cumsum(sub.sum(axis=1))]).astype(np.uint32)
    assert np.array_equal(e.add_users_bulk(keys, 8, topics, offs), c)
    sample = sorted({0, 255, 256, 8191, 8192, (1 << 20) - 1, 1 << 20, n_full - 1} | set(range(37, n_full, 353)))
    for x in sample:
        w.map[x] = w.o.add_user(keys[x].tobytes(), [i + 1 for i in range(3) if sub[x, i]])
    edges = sorted(set(range(0, n_full, 256)) | set(range(255, n_full, 256)))

    def model_frames(conn, msgs):
        return [r for r, kind, to in msgs if (conn in to if kind == "d" else any(masks[x][conn] for x in to))]

    tag = [0]

    def enqueue():
        """one batch of `plan`; → (batch id, its messages, the oracle's frames of the sample)"""
        msgs = []
        for kind, to, size in plan:
            tag[0] += 1
            r = raw(size, tag[0])
            if kind == "b":
                w.bcast(to, r)
                msgs.append((r, "b", to))
            else:
                k = keys[to].tobytes()
                w.direct(k, r)
                msgs.append((r, "d", (to,)))
        return e.flush(), msgs, w.expect()

    def check(res, msgs, want):
        assert res.status == 0 and res.n_overflow == 0
        assert (res.n_deliveries, res.bytes_out) == (n_del, n_bytes)
        t = span_table(res)
        has = np.nonzero(R)[0]
        if pool:
            assert res.n_spans == len(has)
            assert np.array_equal(t[:, 0], has)
            assert np.array_equal(t[:, 1], (np.cumsum(U) - U)[has]), "region offsets"
            assert np.array_equal(t[:, 2], U[has] * K.kUnit)
            assert np.array_equal(t[:, 3], R[has])
        else:
            assert np.array_equal(np.unique(t[:, 0]), has)
            assert np.array_equal(np.bincount(t[:, 0], weights=t[:, 2], minlength=n_full).astype(np.int64), U * K.kUnit)
            assert np.array_equal(np.bincount(t[:, 0], weights=t[:, 3], minlength=n_full).astype(np.int64), R)
        for x in edges:
            assert read_frames(e, res, t, x, pool) == model_frames(x, msgs), x
        for x in sample:
            assert read_frames(e, res, t, x, pool) == want.get(x, []), x

    if not pool:
        for _ in range(3):
            b, msgs, want = enqueue()
            check(e.poll(b), msgs, want)
            e.release_batch(b)
        e.close()
        return
    # three batches in flight: the pool holds two of them, the third is refused (and everything after it)
    (b1, m1, w1), (b2, m2, w2), (b3, m3, w3) = enqueue(), enqueue(), enqueue()
    r1, r2, r3 = e.poll(b1), e.poll(b2), e.poll(b3)
    assert (r1.status, r2.status, r3.status) == (0, 0, 11)
    check(r1, m1, w1)
    assert r2.pool_base == r1.pool_base + total_units          # region of batch 1 = its units, nothing more
    check(r2, m2, w2)
    e.release_batch(b1)
    e.release_batch(b2)
    e.retry_batch(b3)
    r3 = e.poll(b3)
    check(r3, m3, w3)
    b4, m4, w4 = enqueue()
    r4 = e.poll(b4)
    assert r4.status == 0 and r4.pool_base == r3.pool_base + total_units
    e.release_batch(b3)
    b5, m5, w5 = enqueue()                                     # does not fit behind batch 4: wraps to the pool start
    r5 = e.poll(b5)
    assert r5.status == 0 and r5.pool_base == 0 and r4.pool_base + 2 * total_units > cfg["pool_bytes"] // K.kUnit
    check(r5, m5, w5)
    check(r4, m4, w4)
    e.release_batch(b4)
    e.release_batch(b5)
    e.close()
