"""Shared-payload delivery (PCDN_FLAG_SHARED_PAYLOAD): every delivery is one 32-byte reference record
and the payload exists once per batch in pinned host memory (pcdn_batch_payload).  What a writer emits
from the records — p[4..8) then the L payload bytes — must be exactly the oracle's stream, on every
layout the copy mode supports, and the records themselves must be bit for bit the documented layout.

Several tests run the copy-mode workloads (gpu_workloads) with delivery="shared": the streams they compare are
the same, only the records in between differ."""
import ctypes as C
import os
import random
import struct

import numpy as np
import pytest

import gpu_workloads as workloads
from gpu_world import STATUS_EAGAIN, PCDN_ENOENT, PCDN_ENOSPC, World, frames, payload, records, ref_record, shard_cfg, wire
from oracle import oracle as orc

pytestmark = pytest.mark.gpu


def resolve(data, n_records, payload_base, batch_id):
    """the frames a writer emits for a span of reference records"""
    recs = records(data, n_records, batch_id)
    assert all(isinstance(r, tuple) for r in recs), "a shared-payload span holds a framed copy"
    return frames(recs, payload_base)


# ------------------------------------------------------------------ 1. randomized mixed workload
@pytest.mark.parametrize("variant", [pytest.param("rings", id="0"), "staged", "runs", "pool", "pool-staged-runs", "host", "pool-host",
                                     "shards-host-staged"])
@pytest.mark.parametrize("seed", [0, 1])
def test_random_mixed_batches_shared(pcdn, seed, variant):
    """the copy-mode randomized workload (frames 0 B .. 40 KB, local / remote / unknown directs, state
    changes between batches) with every delivery by reference: rings (0: the fused k_ctrl_small path of
    a small engine; staged: the regular control kernels), run-length spans, pool, pool + run-length spans,
    host rings, pool in host memory, three shards on GPU 0 with the regular control kernels"""
    workloads.random_mixed_batches(pcdn, seed, variant, delivery="shared")


@pytest.mark.parametrize("seed", [0, 2])
def test_device_parse_shared(pcdn, seed):
    """device parse (seed 2: with the regular control kernels): a frame with a non-zero msg_status
    writes no record; everything else is delivered by reference"""
    workloads.frames_through_receive_loops(pcdn, seed, delivery="shared")


@pytest.mark.parametrize("staged", [False, True])
def test_device_parse_status_codes_shared(pcdn, staged):
    workloads.msg_status_codes(pcdn, staged, delivery="shared")


# ------------------------------------------------------------------ 2. exact record bytes
@pytest.mark.parametrize("mode", ["rings", "host-rings", "pool"])
def test_reference_record_bytes(pcdn, mode):
    """every record of a small batch, read from the ring / pool, equals the model: marker, BE length,
    offset of the raw bytes in the batch's payload, batch id, zero tail; the payload holds the frame"""
    flags = {"rings": 0, "host-rings": pcdn.FLAG_HOST_RINGS, "pool": pcdn.FLAG_OUTPUT_POOL}[mode]
    e = pcdn.Engine(max_conns=256, max_topics=16, max_keys=256, ring_bytes_per_conn=4096, pool_bytes=1 << 16,
                    flags=flags | pcdn.FLAG_SHARED_PAYLOAD)
    conns = [e.add_user(b"user%04d" % i, [i % 3]) for i in range(40)]
    for rnd in range(3):                      # a second and third batch: new batch ids, ring tails move on
        sizes = [0, 1, 27, 28, 100, 5000, 70000, 12]
        frames = [orc.broadcast_frame([m % 3], bytes([rnd, m]) * (s // 2)) for m, s in enumerate(sizes)]
        offs, at = [], 0
        for fr in frames:                     # host-staged slots: 16-byte aligned, raw bytes at +4
            offs.append(at + 4)
            at += (4 + len(fr) + 15) // 16 * 16
        b = e.submit([("b", [m % 3], fr, False) for m, fr in enumerate(frames)])
        res = e.poll(b)
        assert res.status == 0 and res.n_overflow == 0
        base = e.batch_payload(b)
        for m, fr in enumerate(frames):
            assert C.string_at(base + offs[m], len(fr)) == fr
        hb = e.host_rings()
        assert bool(hb) == (mode == "host-rings")
        spans = e.spans(res)
        assert len(spans) == len(conns) and res.n_deliveries == sum(1 for c in range(40) for m in range(8) if m % 3 == c % 3)
        assert res.bytes_out == sum(4 + len(frames[m]) for c in range(40) for m in range(8) if m % 3 == c % 3)
        for conn, off, ln, nrec in spans:
            i = conns.index(conn)
            want = b"".join(ref_record(len(frames[m]), offs[m], b) for m in range(8) if m % 3 == i % 3)
            assert (ln, nrec) == (len(want), len(want) // 32)
            if mode == "pool":
                data = e.read(conn, res.pool_base + off, ln)
            elif hb:
                data = C.string_at(hb + conn * 4096 + off, ln)
            else:
                data = e.read(conn, off, ln)
            assert data == want, (conn, off)
        e.release_batch(b)
        with pytest.raises(pcdn.PcdnError) as ei:
            e.batch_payload(b)
        assert ei.value.code == PCDN_ENOENT              # released
    e.close()


# ------------------------------------------------------------------ 3. the capability itself
@pytest.mark.parametrize("out", ["rings", "pool"])
def test_large_messages_to_many_users(pcdn, out):
    """a 4 MiB broadcast and 1 MiB directs to 4096 users: with 64 KiB rings (or a 1 MiB output pool) no
    connection overflows, and every memfd the writer fills holds the oracle's stream"""
    cfg = dict(max_conns=4096, ring_bytes_per_conn=1 << 16, max_batch_bytes=24 << 20, max_batch_deliveries=1 << 16)
    if out == "pool":
        cfg.update(flags=pcdn.FLAG_OUTPUT_POOL, pool_bytes=1 << 20)
    w = World(pcdn, delivery="shared", **cfg)
    keys = [b"user-%05d" % i for i in range(4096)]
    conns = [w.add_user(k, [0]) for k in keys]
    eg = pcdn.Egress(w.e, n_threads=8)
    watched = conns[::64] + conns[1:9]               # 72 descriptors: the broadcast's recipients and the direct targets
    fds = {}
    for c in watched:
        fds[c] = os.memfd_create("conn%d" % c)
        eg.attach(c, fds[c])
    stream = {c: bytearray() for c in fds}
    rng = random.Random(5)
    for rnd in range(2):
        w.bcast([0], orc.broadcast_frame([0], payload(rng, 4 << 20)))
        for i in range(1, 9):
            w.direct(keys[i], orc.direct_frame(keys[i], payload(rng, 1 << 20)))
        b = w.e.flush()
        res = w.e.poll(b)
        assert res.status == 0 and res.n_overflow == 0 and res.n_deliveries == 4096 + 8
        st = eg.write_batch(b)
        w.e.release_batch(b)
        exp = w.expect()
        assert len(exp) == 4096
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


# ------------------------------------------------------------------ 4. egress
@pytest.mark.parametrize("mode", ["hbm", "host-rings", "shards-host", "pool-runs"])
def test_writer_to_file_descriptors_shared(pcdn, mode):
    """1100 memfds over six batches: each holds exactly the oracle's stream"""
    workloads.writer_to_file_descriptors(pcdn, mode, delivery="shared")


def test_sockets_backpressure_failure_and_soft_close_shared(pcdn):
    """a 4 KiB send buffer and a slow reader split writes between a record's 4 header bytes and its
    payload; a dead peer is reported once; soft_close still writes the open batch"""
    workloads.sockets_backpressure_failure_and_soft_close(pcdn, delivery="shared")


@pytest.mark.parametrize("mode", ["hbm-small-chunks", "pool", "host-rings", "shards-host"])
def test_callback_sink_resolves_through_batch_payload(pcdn, mode):
    """a Python sink walks the chunks' reference records and resolves them with batch_payload; small
    chunks force many chunks per batch"""
    cfg = dict(max_conns=2048, ring_bytes_per_conn=1 << 16)
    if mode == "host-rings":
        cfg["flags"] = pcdn.FLAG_HOST_RINGS
    if mode == "pool":
        cfg.update(flags=pcdn.FLAG_OUTPUT_POOL, pool_bytes=64 << 20)
    if mode == "shards-host":
        cfg.update(shard_cfg(pcdn, mode), max_conns=1024)
    w = World(pcdn, delivery="shared", **cfg)
    eg = pcdn.Egress(w.e, chunk_bytes=(1 << 17) if mode == "hbm-small-chunks" else 0)
    rng = random.Random(4)
    keys = [rng.getrandbits(64).to_bytes(8, "little") * 2 for _ in range(1200)]
    for k in keys:
        w.add_user(k, [x for x in range(4) if rng.random() < 0.4])
    for rnd in range(4):
        workloads.traffic(w, rng, keys, 60)
        b = w.e.flush()
        base = w.e.batch_payload(b)
        got = {}

        def sink(ch):
            for i in range(ch.n_spans):
                sp = ch.spans[i]
                data = C.string_at(ch.data + ch.data_off[i], sp.len)
                got.setdefault(sp.conn, bytearray()).extend(wire(resolve(data, sp.n_records, base, b)))

        st = eg.drain(b, sink)
        w.e.release_batch(b)
        assert {c: bytes(v) for c, v in got.items()} == {c: wire(fr) for c, fr in w.expect().items()}
        if mode == "hbm-small-chunks":
            assert st.chunks >= 2
    eg.close()
    w.e.close()


# ------------------------------------------------------------------ 5. pool refusal and retry
@pytest.mark.parametrize("layout", ["one-shard", "shards-host"])
@pytest.mark.parametrize("control", ["fused", "regular"])
def test_pool_refusal_and_retry_shared(pcdn, layout, control):
    """an 8 KiB pool (256 records): an unreleased batch holds 240 of them, the next batch does not fit
    and is refused, state changes follow, a later batch queues behind it.  After the release the retried
    batch writes the records it would have written at launch (its own batch id) and routes as launched."""
    kw = dict(max_conns=1024, flags=pcdn.FLAG_OUTPUT_POOL | (pcdn.FLAG_STAGED_SPANS if control == "regular" else 0),
              pool_bytes=8192, batch_slots=4)
    if layout == "shards-host":
        kw.update(shard_cfg(pcdn, layout))
    w = World(pcdn, delivery="shared", **kw)
    keys = [b"user-%03d" % i for i in range(120)]
    conn = {k: w.add_user(k, [0]) for k in keys}
    hot = b"hot"
    conn[hot] = w.add_user(hot, [])
    stride = w.e.shard_info(0).shard_stride
    home = conn[hot] // stride
    on_home = [k for k in keys if conn[k] // stride == home]
    for j in range(240):                                       # 240 records on the hot connection's shard
        w.direct(hot, orc.direct_frame(hot, b"fill %d" % j))
    b0 = w.e.flush()
    w.bcast([0], orc.broadcast_frame([0], b"refused first"))
    for k in on_home[:3]:
        w.direct(k, orc.direct_frame(k, b"direct in the refused batch"))
    b1 = w.e.flush()
    assert w.e.poll(b0).status == 0
    assert w.e.poll_shard(b1, home).status == STATUS_EAGAIN
    w.both("unsubscribe_user_from", on_home[0], [0])
    w.both("remove_user", on_home[1])
    w.add_user(b"newcomer", [0])
    w.bcast([0], orc.broadcast_frame([0], b"after the changes"))
    b2 = w.e.flush()
    assert w.e.poll_shard(b2, home).status == STATUS_EAGAIN
    got = {}

    def consume(b, retry):
        if retry:
            w.e.retry_batch(b)
        r = w.e.poll(b)
        assert r.status == 0 and r.n_overflow == 0
        w.e.last_result = r
        for c, fr in w.e.collect_frames(r).items():      # (collect_frames checks every record's batch id)
            got.setdefault(c, []).extend(fr)
        base = w.e.batch_payload(b)
        for c, off, ln, nrec in w.e.spans(r)[:50]:       # ... and here the whole record against the model
            data = w.e.read(c, r.pool_base + off, ln)
            for i, fr in enumerate(resolve(data, nrec, base, b)):
                o = struct.unpack("<Q", data[i * 32 + 8:i * 32 + 16])[0]
                assert data[i * 32:i * 32 + 32] == ref_record(len(fr), o, b)
        w.e.release_batch(b)

    consume(b0, False)
    consume(b1, True)
    consume(b2, True)
    assert w.compare(w.e, got, w.expect()) > 240 + 2 * 110
    w.e.close()


# ------------------------------------------------------------------ 6. direct paths
def test_direct_hot_recipient_keeps_order_shared(pcdn):
    """thousands of directs to one key in one batch (> kHotMin hits, >= kThinSeparateMin directs)"""
    workloads.direct_hot_recipient_keeps_order(pcdn, delivery="shared")


def test_sharded_device_resident_batch_shared(pcdn):
    """pcdn_submit_device on three shards of GPU 0: the payload comes from the first shard's ingest region"""
    workloads.sharded_device_resident_batch(pcdn, "shards-host", delivery="shared")


@pytest.mark.parametrize("ready", [False, True])
def test_device_resident_batch_payload(pcdn, ready):
    """pcdn_submit_device on one GPU: the frames are copied once into pinned staging, batch_payload
    returns them, and the streams match the oracle; an arena of max_batch_bytes + 64 bytes fits the
    staging, a larger one is ENOSPC"""
    import torch

    w = World(pcdn, max_conns=2048, max_batch_bytes=1 << 20, delivery="shared")
    rng = random.Random(6)
    keys = [b"k%07d" % i for i in range(600)]
    for i, k in enumerate(keys):
        w.add_user(k, [i % 3])
    M = 40
    frames, kinds, topics, aux_off, aux_len, slot_off = [], [], [], [], [], []
    arena = bytearray()
    for m in range(M):
        slot_off.append(len(arena) // 16)
        if m % 3 == 2:
            rc = keys[m * 7]
            fr = orc.direct_frame(rc, payload(rng, 50 + 37 * m))
            kinds.append(3)
        else:
            t = [m % 3]
            fr = orc.broadcast_frame(t, payload(rng, 300 * m + 1))
            kinds.append(4)
        arena += bytes(4) + fr + bytes((-(4 + len(fr))) % 16)
        if kinds[-1] == 3:
            aux_off.append(len(arena)); aux_len.append(len(rc))
            arena += rc + bytes((-len(rc)) % 16)
        else:
            aux_off.append(len(topics)); aux_len.append(1)
            topics.append(m % 3)
        frames.append(fr)
    dev = torch.device("cuda", 0)
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
    db.hints = pcdn.BATCH_READY if ready else 0

    def oracle_batch():
        for m in range(M):
            if kinds[m] == 3:
                w.o.handle_direct_message(keys[m * 7], frames[m], False)
            else:
                w.o.handle_broadcast_message([m % 3], frames[m], False)

    for rnd in range(3):       # slots are reused: the staging is rewritten each time
        oracle_batch()
        b = w.e.submit_device(db)
        res = w.e.poll(b)
        assert res.status == 0
        base = w.e.batch_payload(b)
        assert C.string_at(base, len(arena)) == bytes(arena)
        got = w.e.collect_frames(res)
        w.e.release_batch(b)
        assert got == w.expect()
    # the staging holds max_batch_bytes + 64 frame bytes: an arena of exactly that size is staged whole
    cap = (1 << 20) + 64
    d_full = torch.zeros(cap + 16, dtype=torch.uint8, device=dev)
    d_full[:len(arena)] = d_arena[:len(arena)]
    torch.cuda.synchronize(dev)

    def sized(ptr, arena_bytes):
        s = pcdn.DeviceBatch(M, len(bidx), ptr, arena_bytes, d_kind.data_ptr(), d_flags.data_ptr(), d_slot.data_ptr(),
                             d_len.data_ptr(), d_aoff.data_ptr(), d_alen.data_ptr(), d_topics.data_ptr(), len(topics), d_bidx.data_ptr())
        s.hints = db.hints
        return s

    oracle_batch()
    b = w.e.submit_device(sized(d_full.data_ptr(), cap))
    res = w.e.poll(b)
    assert res.status == 0
    assert C.string_at(w.e.batch_payload(b), cap) == bytes(arena) + bytes(cap - len(arena))
    got = w.e.collect_frames(res)
    w.e.release_batch(b)
    assert got == w.expect()
    for arena_bytes in (cap + 16, (1 << 20) + 4096):
        with pytest.raises(pcdn.PcdnError) as ei:
            w.e.submit_device(sized(d_full.data_ptr(), arena_bytes))
        assert ei.value.code == PCDN_ENOSPC             # nothing launched
        assert w.e.next_batch() == 0
    w.e.close()


# ------------------------------------------------------------------ 7. full size
def test_full_size_reference_records(pcdn):
    """2^20 connections x 8 x 1 KiB broadcasts into an output pool: every one of the 2^23 records checked
    on the device against the model (torch), then the batch drained to host memory and a sample of
    connections' expanded streams compared with the frames"""
    import torch

    N, M, L0 = 1 << 20, 8, 1024
    e = pcdn.Engine(max_conns=N, max_topics=256, max_keys=N + 4096, max_key_len=16, ring_bytes_per_conn=1 << 12,
                    max_batch_msgs=64, max_batch_bcast=16, max_batch_deliveries=M * N + 1024, batch_slots=2,
                    flags=pcdn.FLAG_OUTPUT_POOL | pcdn.FLAG_SPAN_RUNS | pcdn.FLAG_SHARED_PAYLOAD, pool_bytes=N * M * 32 + (1 << 20))
    keys = np.zeros((N, 8), dtype=np.uint8)
    keys[:, :4] = np.arange(N, dtype=np.uint32).view(np.uint8).reshape(N, 4)
    keys[:, 7] = 0xAB
    e.add_users_bulk(keys, 8, np.zeros(N, dtype=np.uint16), np.arange(N + 1, dtype=np.uint32))
    frames = [orc.broadcast_frame([0], bytes([m]) * L0) for m in range(M)]
    L = len(frames[0])
    slot = (4 + L + 15) // 16 * 16
    b = e.submit([("b", [0], fr, False) for fr in frames])
    res = e.poll(b)
    assert res.status == 0 and res.n_deliveries == M * N and res.bytes_out == M * N * (4 + L) and res.n_spans == N
    dev = torch.device("cuda", 0)
    base = e.shard_info(0).rings_dev + res.pool_base * 32

    class _Region:
        __cuda_array_interface__ = {"shape": (N * M * 8,), "typestr": "<i4", "data": (base, False), "version": 3}

    region = torch.as_tensor(_Region(), device=dev).view(N, M, 8)
    model = torch.tensor([list(struct.unpack("<8i", ref_record(L, m * slot + 4, b))) for m in range(M)], dtype=torch.int32, device=dev)
    assert bool((region == model.unsqueeze(0)).all().item()), "device records differ from the model"
    pb = e.batch_payload(b)
    for m, fr in enumerate(frames):
        assert C.string_at(pb + m * slot + 4, L) == fr
    sample = set(range(0, N, 4099)) | {N - 1}
    seen = {}
    eg = pcdn.Egress(e)

    def sink(ch):
        sp = np.ctypeslib.as_array(C.cast(ch.spans, C.POINTER(C.c_uint32)), shape=(ch.n_spans, 4))
        for i in np.nonzero(np.isin(sp[:, 0], list(sample)))[0]:
            data = C.string_at(ch.data + ch.data_off[int(i)], int(sp[i, 2]))
            seen[int(sp[i, 0])] = resolve(data, int(sp[i, 3]), pb, b)

    st = eg.drain(b, sink)
    assert st.spans == N and st.bytes == N * M * 32
    assert set(seen) == sample and all(v == frames for v in seen.values())
    eg.close()
    e.release_batch(b)
    e.close()
