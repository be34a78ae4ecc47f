"""Delivery by reference above a size threshold (pcdn_config.ref_min_bytes): a routed message of at least
ref_min_bytes raw bytes is delivered as one 32-byte reference record per recipient, every shorter one as a
framed copy, in the same span and in batch order.  What a writer emits from either kind must be exactly the
oracle's stream; the records must be exactly the documented layouts; and a message far larger than a ring
must reach every recipient without an overflow.

Several tests run existing workloads (gpu_workloads) with delivery=("ref", T): their frames run from 0 B to
40 KB, so every batch mixes both kinds of record."""
import ctypes as C
import os
import random

import pytest

import gpu_workloads as workloads
from gpu_world import PCDN_EINVAL, STATUS_EAGAIN, World, chunk_streams, payload, records, shard_cfg, wire
from kconst import K
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

MIXED = ("ref", 2048)


def kinds(recs):
    return ["copy" if isinstance(r, bytes) else "ref" for r in recs]


def read_span(e, res, conn, off, ln, hb, ring_bytes, pool=False):
    """a span's bytes: read in place from host rings, else through pcdn_read"""
    if pool:   # unit offsets relative to the batch's region
        return e.read(conn, res.pool_base + off, ln)
    if hb:
        return C.string_at(hb + conn * ring_bytes + off, ln)
    return e.read(conn, off, ln)


# ------------------------------------------------------------------ 1. existing bodies on mixed engines
@pytest.mark.parametrize("variant", workloads.MIXED_LAYOUTS)
@pytest.mark.parametrize("seed", [0, 1])
def test_random_mixed_batches_mixed(pcdn, seed, variant):
    """the randomized workload (frames 0 B .. 40 KB, local / remote / unknown directs, state changes between
    batches) with messages of >= 2048 bytes delivered by reference, on every layout"""
    workloads.random_mixed_batches(pcdn, seed, variant, delivery=MIXED)


@pytest.mark.parametrize("seed", [0, 2])
def test_device_parse_mixed(pcdn, seed):
    """device parse (seed 2: regular control kernels): a frame with a non-zero msg_status writes no record"""
    workloads.frames_through_receive_loops(pcdn, seed, delivery=MIXED)


@pytest.mark.parametrize("staged", [False, True])
def test_device_parse_status_codes_mixed(pcdn, staged):
    workloads.msg_status_codes(pcdn, staged, delivery=MIXED)


# (these bodies arrange their refusal with 100 KB copies that fill a 4 MiB pool: there the threshold sits
#  above them, so a mixed engine runs them on batches without a by-reference message; the refusal and retry
#  of batches that hold references is test_pool_refusal_and_retry_with_references)
@pytest.mark.parametrize("runs", [False, True], ids=["spans", "span-runs"])
@pytest.mark.parametrize("control", ["fused", "regular"])
@pytest.mark.parametrize("layout", ["one-shard", "shards-host"])
def test_pool_retry_routes_as_launched_mixed(pcdn, layout, control, runs):
    workloads.retry_routes_as_launched(pcdn, layout, control, runs, delivery=("ref", 1 << 17))


def test_pool_partial_refusal_mixed(pcdn):
    workloads.partial_refusal_across_shards(pcdn, delivery=("ref", 1 << 17))


@pytest.mark.parametrize("how", ["write_batch", "soft_close"])   # (its "drain" sink walks framed records only)
def test_pool_egress_refused_shard_written_once_mixed(pcdn, how):
    workloads.egress_refused_shard_is_written_once(pcdn, how, delivery=("ref", 1 << 17))


@pytest.mark.parametrize("layout", ["one-shard", "shards-host"])
@pytest.mark.parametrize("control", ["fused", "regular"])
def test_pool_refusal_and_retry_with_references(pcdn, layout, control):
    """an 8 KiB pool (256 units) and threshold 16: an unreleased batch of 240 short copies to one hot
    connection, then a batch whose broadcast is a reference record to 120 users is refused, state changes
    follow, a later batch of a reference and a copy broadcast queues behind it.  After the releases the
    retried batches deliver what they would have delivered at launch, bit for bit against the oracle."""
    kw = dict(max_conns=1024, flags=pcdn.FLAG_OUTPUT_POOL | (pcdn.FLAG_STAGED_SPANS if control == "regular" else 0),
              pool_bytes=8192, batch_slots=4)
    if layout == "shards-host":
        kw.update(shard_cfg(pcdn, layout))
    w = World(pcdn, delivery=("ref", 16), **kw)
    keys = [b"user-%03d" % i for i in range(120)]
    conn = {k: w.add_user(k, [0]) for k in keys}
    hot = b"hot"
    conn[hot] = w.add_user(hot, [])
    stride = w.e.shard_info(0).shard_stride
    home = conn[hot] // stride
    on_home = [k for k in keys if conn[k] // stride == home]
    for j in range(240):                                        # < 16 bytes: one-unit copies
        w.direct(hot, b"f%d" % j)
    b0 = w.e.flush()
    w.bcast([0], b"refused first, by reference")
    for k in on_home[:3]:
        w.direct(k, b"short copy")
    b1 = w.e.flush()
    assert w.e.poll(b0).status == 0
    assert w.e.poll_shard(b1, home).status == STATUS_EAGAIN
    w.both("unsubscribe_user_from", on_home[0], [0])
    w.both("remove_user", on_home[1])
    w.add_user(b"newcomer", [0])
    w.bcast([0], b"after the changes, by reference")
    w.bcast([0], b"a copy")
    b2 = w.e.flush()
    assert w.e.poll_shard(b2, home).status == STATUS_EAGAIN
    got = {}
    for b, retry in ((b0, False), (b1, True), (b2, True)):
        if retry:
            w.e.retry_batch(b)
        r = w.e.poll(b)
        assert r.status == 0 and r.n_overflow == 0
        w.e.last_result = r
        for c, fr in w.e.collect_frames(r).items():
            got.setdefault(c, []).extend(fr)
        w.e.release_batch(b)
    assert w.compare(w.e, got, w.expect()) > 240 + 2 * 110


@pytest.mark.parametrize("variant", [pytest.param("rings", id="fused"), "staged", "pool", pytest.param("shards-host", id="shards")])
@pytest.mark.parametrize("case", [workloads.case_sub_around_broadcast, workloads.case_class_thresholds,
                                  workloads.case_many_messages, workloads.case_wide], ids=lambda f: f.__name__[5:])
def test_inbatch_subscribe_mixed(pcdn, case, variant):
    """in-batch subscription events on mixed engines (threshold 64: most broadcasts of these cases are references)"""
    workloads.inbatch_subscribe(pcdn, case, variant, delivery=("ref", 64))


# ------------------------------------------------------------------ 2. exact records at the threshold
@pytest.mark.parametrize("mode", ["rings", "host-rings", "pool"])
def test_records_at_the_threshold(pcdn, mode):
    """raw lengths T - 1, T and T + 1 in one batch, broadcast to a message-major set and a thin set and sent
    direct: the T - 1 message is a framed copy, the other two are exact reference records, at the unit
    offsets the model gives, in batch order inside each connection's span"""
    T, RB = 1000, 4096
    flags = {"rings": 0, "host-rings": pcdn.FLAG_HOST_RINGS, "pool": pcdn.FLAG_OUTPUT_POOL}[mode]
    e = pcdn.Engine(max_conns=256, max_topics=16, max_keys=256, ring_bytes_per_conn=RB, pool_bytes=1 << 20, flags=flags, ref_min_bytes=T)
    keys = [b"user%04d" % i for i in range(40)]
    conns = [e.add_user(k, [0] + ([1] if i < 10 else [])) for i, k in enumerate(keys)]   # topic 0: 40 (>= kFatMin), topic 1: 10
    hb = e.host_rings()
    assert bool(hb) == (mode == "host-rings")
    tail = {}
    for rnd in range(3):                     # new batch ids, ring tails move on
        msgs = [("b", [0], bytes([rnd, 1]) * ((T - 1) // 2) + b"x", False),   # T - 1
                ("b", [1], bytes([rnd, 2]) * (T // 2), False),                # T
                ("d", keys[3], bytes([rnd, 3]) * ((T + 1) // 2) + b"y", False),  # T + 1
                ("b", [0], bytes([rnd, 4]) * (T // 2) + b"zz", False),        # T + 2
                ("d", keys[3], bytes([rnd, 5]) * 10, False),                  # 20
                ("b", [1], bytes([rnd, 6]) * ((T + 1) // 2) + b"w", False)]   # T + 1
        offs, at = [], 0
        for m in msgs:                       # host-staged slots: 16-byte aligned, raw at +4, a direct's key staged behind
            offs.append(at + 4)
            at += (4 + len(m[2]) + 15) // 16 * 16 + ((len(m[1]) + 15) // 16 * 16 if m[0] == "d" else 0)
        b = e.submit(msgs)
        res = e.poll(b)
        assert res.status == 0 and res.n_overflow == 0
        base = e.batch_payload(b)
        spans = e.spans(res)
        assert len(spans) == len(conns)
        nrec_total = 0
        region = 0   # pool: the connections' regions follow each other in connection order
        for conn, off, ln, nrec in sorted(spans):
            i = conns.index(conn)
            mine = [m for m, x in enumerate(msgs)
                    if (x[0] == "b" and (x[1][0] == 0 or i < 10)) or (x[0] == "d" and x[1] == keys[i])]
            recs = records(read_span(e, res, conn, off, ln, hb, RB, mode == "pool"), nrec, b)
            assert len(recs) == len(mine) == nrec
            units = 0
            for m, r in zip(mine, recs):
                raw = msgs[m][2]
                if len(raw) < T:
                    assert r == raw, (conn, m)
                    units += (4 + len(raw) + 31) // 32
                else:
                    assert r == (len(raw), offs[m], b), (conn, m)
                    assert C.string_at(base + r[1], len(raw)) == raw
                    units += 1
            assert ln == units * 32
            if mode == "pool":
                assert off == region
                region += units
            else:            # (bytes) each ring continues where the previous batch ended: no wrap in three batches
                assert off == tail.get(conn, 0) * 32
                tail[conn] = off // 32 + units
            nrec_total += nrec
        assert res.n_deliveries == nrec_total
        assert res.bytes_out == sum(4 + len(msgs[m][2]) for i in range(40) for m, x in enumerate(msgs)
                                    if (x[0] == "b" and (x[1][0] == 0 or i < 10)) or (x[0] == "d" and x[1] == keys[i]))
        e.release_batch(b)
    e.close()


# ------------------------------------------------------------------ 3. messages larger than a ring
@pytest.mark.parametrize("mode", ["rings", "pool", "host-rings", "shards-host", "device"])
def test_message_larger_than_a_ring(pcdn, mode):
    """a 4 MiB broadcast to 4096 users on 64 KiB rings between 1 KiB broadcasts, plus 1 KiB directs and a
    100 KB direct, threshold 16 KiB: no connection overflows, the watched connections' memfds hold the
    oracle's streams, and the 1 KiB messages sit in the rings as framed copies.  device: the batch goes
    through pcdn_submit_device"""
    T, N = 16 << 10, 4096
    cfg = dict(max_conns=N, ring_bytes_per_conn=1 << 16, max_batch_bytes=24 << 20, max_batch_deliveries=1 << 16)
    if mode == "pool":
        cfg.update(flags=pcdn.FLAG_OUTPUT_POOL, pool_bytes=64 << 20)
    if mode == "host-rings":
        cfg.update(flags=pcdn.FLAG_HOST_RINGS)
    if mode == "shards-host":
        cfg.update(shard_cfg(pcdn, mode), max_conns=2048)
    w = World(pcdn, delivery=("ref", T), **cfg)
    keys = [b"user-%05d" % i for i in range(N)]
    conns = [w.add_user(k, [0]) for k in keys]
    eg = pcdn.Egress(w.e, n_threads=8)
    watched = conns[::64] + conns[1:9]
    fds = {}
    for c in watched:
        fds[c] = os.memfd_create("conn%d" % c)
        eg.attach(c, fds[c])
    stream = {c: bytearray() for c in fds}
    rng = random.Random(7)
    hb = w.e.host_rings()
    for rnd in range(2 if mode == "rings" else 1):   # (rings: a second batch on the released rings)
        msgs = [("b", orc.broadcast_frame([0], payload(rng, 1 << 10))),
                ("b", orc.broadcast_frame([0], payload(rng, 4 << 20))),
                ("b", orc.broadcast_frame([0], payload(rng, 1 << 10)))]
        msgs += [("d", keys[i], orc.direct_frame(keys[i], payload(rng, 1 << 10))) for i in range(1, 9)]
        msgs += [("d", keys[1], orc.direct_frame(keys[1], payload(rng, 100_000)))]
        if mode == "device":
            b, keep = submit_device(pcdn, w, msgs)
        else:
            for m in msgs:
                if m[0] == "b":
                    w.bcast([0], m[1])
                else:
                    w.direct(m[1], m[2])
            b = w.e.flush()
        res = w.e.poll(b)
        assert res.status == 0 and res.n_overflow == 0 and res.n_deliveries == 3 * N + 9
        # the ring of a watched connection: its 1 KiB messages are framed copies, the large ones references
        if mode in ("rings", "host-rings"):
            for conn, off, ln, nrec in w.e.spans(res):
                if conn == conns[1]:
                    got = kinds(records(read_span(w.e, res, conn, off, ln, hb, 1 << 16), nrec, b))
                    assert got == ["copy", "ref", "copy", "copy", "ref"], got
        st = eg.write_batch(b)
        w.e.release_batch(b)
        exp = w.expect()
        assert len(exp) == N
        for c in fds:
            stream[c] += wire(exp[c])
        assert st.fd_bytes == sum(len(wire(exp[c])) for c in fds)
    assert eg.failed() == []
    for c, fd in fds.items():
        os.lseek(fd, 0, os.SEEK_SET)
        got = bytearray()
        while True:
            d = os.read(fd, 1 << 24)
            if not d:
                break
            got += d
        assert bytes(got) == bytes(stream[c]), c
        os.close(fd)
    eg.close()
    w.e.close()


def submit_device(pcdn, w, msgs):
    """msgs as ('b', frame) / ('d', key, frame) through pcdn_submit_device (topic 0); the oracle gets them too"""
    import torch

    arena = bytearray()
    kinds, slot_off, lens, aux_off, aux_len, topics = [], [], [], [], [], []
    for m in msgs:
        fr = m[-1]
        slot_off.append(len(arena) // 16)
        arena += bytes(4) + fr + bytes((-(4 + len(fr))) % 16)
        lens.append(len(fr))
        if m[0] == "d":
            kinds.append(3)
            aux_off.append(len(arena)); aux_len.append(len(m[1]))
            arena += m[1] + bytes((-len(m[1])) % 16)
            w.o.handle_direct_message(m[1], fr, False)
        else:
            kinds.append(4)
            aux_off.append(len(topics)); aux_len.append(1)
            topics.append(0)
            w.o.handle_broadcast_message([0], fr, False)
    dev = torch.device("cuda", w.e.shard_info(0).device)
    t8 = lambda a: torch.tensor(list(a), dtype=torch.uint8, device=dev)
    t32 = lambda a: torch.tensor(list(a), dtype=torch.int32, device=dev)
    bidx = [i for i, k in enumerate(kinds) if k == 4]
    keep = [torch.frombuffer(bytearray(arena + bytes(64)), dtype=torch.uint8).to(dev), t8(kinds), t8([0] * len(msgs)), t32(slot_off),
            t32(lens), t32(aux_off), t32(aux_len), torch.tensor(topics, dtype=torch.int16, device=dev), t32(bidx)]
    torch.cuda.synchronize(dev)
    db = pcdn.DeviceBatch(len(msgs), len(bidx), keep[0].data_ptr(), len(arena), keep[1].data_ptr(), keep[2].data_ptr(),
                          keep[3].data_ptr(), keep[4].data_ptr(), keep[5].data_ptr(), keep[6].data_ptr(), keep[7].data_ptr(),
                          len(topics), keep[8].data_ptr())
    return w.e.submit_device(db), keep   # (the caller keeps the tensors alive until the batch has run)


# ------------------------------------------------------------------ 4. class and launch edges, T = 1024
@pytest.mark.parametrize("control", ["fused", "staged"])
def test_class_and_launch_edges_low_threshold(pcdn, control):
    """threshold 1024: a dense broadcast of 1020 B (connection-major copy) next to one of 1024 B (by
    reference, message-major entries, no tile) and 1023 B, to thin (< kFatMin), message-major and dense
    recipient sets; directs on both sides of T to local, remote and unknown keys; a batch of
    kThinSeparateMin directs (its own k_pack_direct launch) of both kinds — fused and regular control"""
    T = 1024
    w = World(pcdn, max_conns=8192, ring_bytes_per_conn=1 << 18, delivery=("ref", T),
              flags=pcdn.FLAG_STAGED_SPANS if control == "staged" else 0)
    rng = random.Random(9)
    N = 8192
    dense_min = N >> K.kCmDenseShift
    keys = [b"k%06d" % i for i in range(dense_min + 100)]
    for i, k in enumerate(keys):   # topic 0: dense; topic 1: 100 (message-major); topic 2: kFatMin - 1 (thin)
        t = [0] + ([1] if i < 100 else []) + ([2] if i < K.kFatMin - 1 else [])
        w.add_user(k, t)
    w.add_broker("b1/p1", [0, 1])
    remote = [b"remote%d" % i for i in range(4)]
    w.both("apply_user_sync", "b1/p1", [(k, 1, "b1/p1") for k in remote])

    def raw(n, tag):
        return bytes([tag]) * n

    for rnd in range(3):
        for t in (0, 1, 2):
            for n in (T - 4, T - 1, T, T + 1, 4096, 40000, 0, 12):
                w.bcast([t], raw(n, rnd * 16 + t), rng.random() < 0.2)
        for n in (T - 1, T, 20, 70000):
            w.direct(rng.choice(keys), raw(n, 0x40 + rnd))
            w.direct(rng.choice(remote), raw(n, 0x50 + rnd))
            w.direct(b"nobody", raw(n, 0x60 + rnd))
        assert w.check() > 0
    # kThinSeparateMin directs in one batch, on both sides of T
    for j in range(K.kThinSeparateMin):
        w.direct(keys[j % len(keys)], raw(T - 1 if j % 3 else T + j % 7, j & 0xFF))
    assert w.check() >= K.kThinSeparateMin
    # and with a broadcast of each kind in the same batch
    for j in range(K.kThinSeparateMin + 10):
        w.direct(keys[(7 * j) % len(keys)], raw(T + 1 if j % 2 else 100, j & 0xFF))
    w.bcast([0], raw(T - 4, 1))
    w.bcast([0], raw(T, 2))
    assert w.check() > 0
    w.e.close()


# ------------------------------------------------------------------ 5. launch count
@pytest.mark.parametrize("control", ["fused", "staged"])
def test_launch_count(pcdn, control):
    """a batch without a message >= T launches on a mixed engine exactly the kernels it launches on a copy
    engine; a batch with one launches exactly one more (k_pack_ref)"""
    T = 4096
    fl = pcdn.FLAG_STAGED_SPANS if control == "staged" else 0
    engines = {t: pcdn.Engine(max_conns=8192, ring_bytes_per_conn=1 << 18, flags=fl, ref_min_bytes=t) for t in (0, T)}
    keys = [b"user%05d" % i for i in range(3000)]
    for e in engines.values():
        for i, k in enumerate(keys):
            e.add_user(k, [i % 3])

    def launches(e, msgs):
        e.flush()
        b0 = e.submit([("b", [0], b"warm", False)])   # the journal of the state calls goes out with this batch
        e.poll(b0)
        e.release_batch(b0)
        n0 = e.stats().kernel_launches
        b = e.submit(msgs)
        assert e.poll(b).status == 0
        n = e.stats().kernel_launches - n0
        e.release_batch(b)
        return n

    small = [("b", [0], b"a" * 1000, False), ("b", [1], b"b" * (T - 1), False), ("d", keys[5], b"c" * 100, False)]
    big_b = small + [("b", [2], b"d" * T, False)]
    big_d = small + [("d", keys[6], b"e" * (T + 5), False)]
    directs = [("d", keys[i % len(keys)], b"f" * (100 + i % 50), False) for i in range(K.kThinSeparateMin)]
    for msgs, extra in ((small, 0), (big_b, 1), (big_d, 1), (directs, 0), (directs + [("d", keys[0], b"g" * T, False)], 1)):
        assert launches(engines[T], msgs) == launches(engines[0], msgs) + extra
    for e in engines.values():
        e.close()


# ------------------------------------------------------------------ 6. egress
@pytest.mark.parametrize("mode", ["hbm", "host-rings", "shards-host", "pool-runs"])
def test_writer_to_file_descriptors_mixed(pcdn, mode):
    """1100 memfds over six batches of 0 B .. 20 KB messages: each holds exactly the oracle's stream"""
    workloads.writer_to_file_descriptors(pcdn, mode, delivery=MIXED)


def test_sockets_backpressure_failure_and_soft_close_mixed(pcdn):
    workloads.sockets_backpressure_failure_and_soft_close(pcdn, delivery=MIXED)


@pytest.mark.parametrize("mode", ["hbm", "pool", "host-rings", "shards-host"])
def test_callback_sink_mixed(pcdn, mode):
    """a Python sink walks both kinds of record in the chunks (references resolved with batch_payload)"""
    cfg = dict(max_conns=2048, ring_bytes_per_conn=1 << 18)
    if mode == "host-rings":
        cfg["flags"] = pcdn.FLAG_HOST_RINGS
    if mode == "pool":
        cfg.update(flags=pcdn.FLAG_OUTPUT_POOL, pool_bytes=256 << 20)
    if mode == "shards-host":
        cfg.update(shard_cfg(pcdn, mode), max_conns=1024)
    w = World(pcdn, delivery=MIXED, **cfg)
    eg = pcdn.Egress(w.e)
    rng = random.Random(4)
    keys = [rng.getrandbits(64).to_bytes(8, "little") * 2 for _ in range(1200)]
    for k in keys:
        w.add_user(k, [x for x in range(4) if rng.random() < 0.4])
    for rnd in range(4):
        workloads.traffic(w, rng, keys, 60)
        b = w.e.flush()
        base = w.e.batch_payload(b)
        got = {}
        eg.drain(b, lambda ch: chunk_streams(ch, got, base, b))
        w.e.release_batch(b)
        assert {c: bytes(v) for c, v in got.items()} == {c: wire(fr) for c, fr in w.expect().items()}
    eg.close()
    w.e.close()


@pytest.mark.parametrize("mode", ["rings", "pool", "shards-host"])
def test_stalled_peer_gets_reference_payload_after_release(pcdn, mode):
    """a stalled peer's backlog holds the payload bytes of its reference records: the batches (and with
    batch_slots=2 their payload staging) are released and reused before the peer reads anything"""
    workloads.stalled_peer_does_not_stall_the_others(pcdn, mode, delivery=MIXED)


# ------------------------------------------------------------------ 7. configuration
# (the refused values: test_ref_threshold_config.py, on a host-only engine)
def test_old_config_size_is_a_copy_engine(pcdn):
    """a pcdn_config of the size before ref_min_bytes (struct_size = its offset) is a copy engine: the
    bytes behind that size are not read, so every record is a framed copy"""
    # (asked for threshold 64, which the old struct size hides from pcdn_create)
    w = World(pcdn, max_conns=1024, ring_bytes_per_conn=1 << 18, struct_size=pcdn.Config.ref_min_bytes.offset, delivery=("ref", 64))
    keys = [b"user%03d" % i for i in range(100)]
    for i, k in enumerate(keys):
        w.add_user(k, [i % 2])
    for n in (10, 64, 1000, 70000):
        w.bcast([0], bytes([n & 0xFF]) * n)
        w.direct(keys[1], bytes([n & 0x7F]) * n)
    b = w.e.flush()
    res = w.e.poll(b)
    assert res.status == 0 and res.n_overflow == 0
    for conn, off, ln, nrec in w.e.spans(res):
        assert kinds(records(w.e.read(conn, off, ln), nrec)) == ["copy"] * nrec, conn
    assert w.e.collect_frames(res) == w.expect()
    w.e.release_batch(b)
    w.e.close()
    with pytest.raises(pcdn.PcdnError) as ei:
        pcdn.Engine(max_conns=1024, struct_size=pcdn.Config.ref_min_bytes.offset - 8)
    assert ei.value.code == PCDN_EINVAL


@pytest.mark.parametrize("variant", [0, "pool", "shards-host"])
def test_threshold_zero_is_the_copy_engine(pcdn, variant):
    """ref_min_bytes = 0 and an engine that never sets it write byte-identical rings / pools on the same
    batches: one recorded workload replayed on both against one oracle run, and the records compared"""
    rng = random.Random(12)
    cfg = dict(max_conns=1024, ring_bytes_per_conn=1 << 18)
    if variant == "pool":
        cfg.update(flags=pcdn.FLAG_OUTPUT_POOL, pool_bytes=64 << 20)
    if variant == "shards-host":
        cfg.update(shard_cfg(pcdn, variant))
    a = pcdn.Engine(**cfg)
    z = pcdn.Engine(**cfg, ref_min_bytes=0)
    keys = [b"u%05d" % i for i in range(900)]
    for e in (a, z):
        for i, k in enumerate(keys):
            e.add_user(k, [i % 4, 4] if i % 5 == 0 else [i % 4])
    for rnd in range(3):
        msgs = []
        for _ in range(80):
            n = rng.choice([0, 5, 100, 1000, 1024, 4096, 20000])
            if rng.random() < 0.6:
                msgs.append(("b", [rng.randrange(5)], payload(rng, n), False))
            else:
                msgs.append(("d", rng.choice(keys), payload(rng, n), False))
        ra, rz = [], []
        for e, out in ((a, ra), (z, rz)):
            b = e.submit(msgs)
            res = e.poll(b)
            assert res.status == 0 and res.n_overflow == 0
            pool = bool(e.cfg.flags & pcdn.FLAG_OUTPUT_POOL)
            for conn, off, ln, nrec in sorted(e.spans(res)):
                recs = records(e.read(conn, res.pool_base + off if pool else off, ln), nrec)
                out.append((conn, off, ln, nrec, recs))
            out.append((res.n_deliveries, res.bytes_out, res.n_spans, res.pool_base))
            e.release_batch(b)
        assert ra == rz
    a.close()
    z.close()
