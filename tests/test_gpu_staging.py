"""Host staging of a batch: the per-batch limits (messages, bytes, broadcasts, topic entries, memory
pool) as pcdn_submit, the one-frame-at-a-time receive calls and the threaded pcdn_receive_frames path
apply them, and where a direct message's recipient key is read from.  Outputs are compared with the
oracle, or between the two receive paths."""
import ctypes as C
import random

import pytest

from gpu_world import PCDN_EAGAIN, PCDN_ENOSPC, World
from oracle import oracle as orc

pytestmark = pytest.mark.gpu


def _staged(msgs, max_key_len):
    """bytes an explicit batch may stage: 16-byte frame slots plus, for direct messages, the key
    staged beside the frame (the worst case; a longer recipient as its first max_key_len + 1 bytes)"""
    n = 0
    for m in msgs:
        n += (4 + len(m[2]) + 15) // 16 * 16
        if m[0] == "d":
            n += (min(len(m[1]), max_key_len + 1) + 15) // 16 * 16
    return n


def _submit_both(w, msgs):
    for m in msgs:
        if m[0] == "b":
            w.o.handle_broadcast_message(m[1], m[2], m[3])
        else:
            w.o.handle_direct_message(m[1], m[2], m[3])
    return w.e.submit(msgs)


def _refused(pcdn, w, msgs, code):
    st = w.e.stats()
    before = (st.bytes_in, st.inflight_bytes)
    with pytest.raises(pcdn.PcdnError) as ei:
        w.e.submit(msgs)
    assert ei.value.code == code
    st = w.e.stats()
    assert (st.bytes_in, st.inflight_bytes) == before


def test_explicit_batch_refusals(pcdn):
    """pcdn_submit takes a batch whose staged size is exactly max_batch_bytes - 64 and refuses it 16
    bytes larger; also one broadcast over max_batch_bcast and one topic entry over the descriptor
    block's capacity (4 * max_batch_msgs + 4096).  A refused batch stages nothing: the counters stay,
    and the next batch delivers only its own messages."""
    B, M, MB, KL = 1 << 16, 256, 8, 64
    w = World(pcdn, max_conns=256, max_batch_msgs=M, max_batch_bcast=MB, max_batch_bytes=B, max_key_len=KL)
    keys = [bytes([i + 1]) * (8 if i % 3 else 40) for i in range(64)]
    for i, k in enumerate(keys):
        w.add_user(k, [i % 5, 7])
    rng = random.Random(5)
    base = []
    for j in range(12):
        if j % 3 == 0:
            t = [j % 5]
            base.append(("b", t, orc.broadcast_frame(t, bytes([j]) * rng.randrange(100, 3000)), j % 2 == 0))
        else:
            k = keys[rng.randrange(64)]
            base.append(("d", k, orc.direct_frame(k, bytes([j]) * rng.randrange(0, 3000)), False))

    def filled(extra):
        """base + one broadcast whose frame slot brings the staged size to B - 64 + extra"""
        left = B - 64 - _staged(base, KL) + extra
        assert left >= 32 and left % 16 == 0
        return base + [("b", [7], bytes([7]) * (left - 4), False)]

    _refused(pcdn, w, filled(16), PCDN_ENOSPC)
    assert _staged(filled(0), KL) == B - 64
    _submit_both(w, filled(0))
    assert w.check() > 12

    small = [("b", [t], orc.broadcast_frame([t], b"s%d" % t), False) for t in range(MB + 1)]
    _refused(pcdn, w, small, PCDN_ENOSPC)
    _submit_both(w, small[:MB])
    assert w.check() > 0

    cap = 4 * M + 4096
    many = [list(range(256)) * 10, list(range(256)) * 10]           # 2 x 2560 = cap entries
    assert sum(map(len, many)) == cap
    _refused(pcdn, w, [("b", many[0] + [1], b"t0", False), ("b", many[1], b"t1", False)], PCDN_ENOSPC)
    _submit_both(w, [("b", many[0], b"t0", False), ("b", many[1], b"t1", False)])
    assert w.check() > 0
    assert w.e.stats().inflight_bytes == 0

    p = World(pcdn, max_conns=64, global_memory_pool_size=10_000)
    p.add_user(b"a" * 8, [0])
    first = [("b", [0], b"x" * 5000, False)]
    bid = _submit_both(p, first)
    second = [("b", [0], b"y" * 3000, False), ("d", b"a" * 8, b"z" * 3000, False)]
    _refused(pcdn, p, second, PCDN_EAGAIN)
    assert p.e.stats().inflight_bytes == 5000
    res = p.e.poll(bid)
    assert p.e.collect_frames(res) == p.expect()
    p.e.release_batch(bid)
    _submit_both(p, second)
    assert p.check() == 2
    assert p.e.stats().inflight_bytes == 0 and p.e.stats().bytes_in == 11000


def _run_batches(e, sizes=None, out=None, flush=True):
    """flush (unless told not to), then poll every outstanding batch oldest first: (n_msgs of each
    batch, {conn: frames})"""
    if flush:
        e.flush()
    sizes, out = ([], {}) if sizes is None else (sizes, out)
    while True:
        b = e.next_batch()
        if not b:
            return sizes, out
        res = e.poll(b)
        assert res.status == 0 and res.n_overflow == 0
        sizes.append(res.n_msgs)
        for conn, fr in e.collect_frames(res).items():
            out.setdefault(conn, []).extend(fr)
        e.release_batch(b)


def _receive_all(pcdn, e, frames, batched):
    """Every frame in order: through pcdn_receive_frames calls (`batched`) or one user_receive /
    broker_receive call each.  Where the engine stops with PCDN_EAGAIN (memory pool exhausted), the
    batches it launched are drained WITHOUT a flush, and the frames resume where it stopped.  A stop must
    have launched the batch holding the permits: something is drained, and no message is left in an open
    batch.  Returns (codes, n_msgs of each batch, {conn: frames}, number of stops)."""
    n = len(frames)
    arr = (pcdn.Frame * n)(*[pcdn.Frame(s, len(s), o, raw, len(raw), 0) for s, o, raw in frames])
    rcs = (C.c_int32 * n)()
    sizes, out, pos, stops = [], {}, 0, 0
    while pos < n:
        if batched:
            done = e.L.pcdn_receive_frames(e.h, C.cast(C.byref(arr, pos * C.sizeof(pcdn.Frame)), C.POINTER(pcdn.Frame)), n - pos,
                                           C.cast(C.byref(rcs, pos * 4), C.POINTER(C.c_int32)))
        else:
            s, o, raw = frames[pos]
            rcs[pos] = e.broker_receive("b0/p0", raw) if o else e.user_receive(s, raw)
            done = PCDN_EAGAIN if rcs[pos] == PCDN_EAGAIN else 1
        assert done == PCDN_EAGAIN or done > 0
        pos += max(done, 0)
        if pos < n and (done == PCDN_EAGAIN or batched):
            stops += 1
            before = len(sizes)
            _run_batches(e, sizes, out, flush=False)
            assert len(sizes) > before and e.flush() == 0, "a pool refusal must launch the open batch"
    _run_batches(e, sizes, out)
    return list(rcs), sizes, out, stops


@pytest.mark.parametrize("flags,pool", [(0, 0), (1, 0), (0, 200_000), (1, 200_000)],
                         ids=["host-parse", "device-parse", "host-parse-pool", "device-parse-pool"])
def test_both_receive_paths_cut_the_same_batches(pcdn, flags, pool):
    """One pcdn_receive_frames call of >= 2048 frames (classified on several threads) and the same frames
    one at a time through user_receive / broker_receive must return the same codes, cut the same batches
    and deliver the same bytes.  The frames cut batches on the message, byte, broadcast and (host parse)
    topic-entry limits, with subscribe frames in between.  Enough batch slots that neither path has to
    drain during the call; with a global memory pool both stop with PCDN_EAGAIN where it is exhausted,
    after launching the open batch, and resume once their batches are drained."""
    cfg = dict(max_conns=512, max_topics=256, max_keys=2048, ring_bytes_per_conn=2 << 20, max_batch_msgs=1024,
               max_batch_bcast=300, max_batch_bytes=256 << 10, max_batch_deliveries=1 << 20, batch_slots=48,
               n_valid_topics=12, flags=flags, global_memory_pool_size=pool)
    engines = [pcdn.Engine(**cfg), pcdn.Engine(**cfg)]
    try:
        rng = random.Random(17)
        keys = [rng.getrandbits(64).to_bytes(8, "little") * 4 for _ in range(300)]
        subs = [[x for x in range(11) if rng.random() < 0.1] + ([11] if i < 2 else []) for i in range(len(keys))]
        for e in engines:
            for k, t in zip(keys, subs):
                e.add_user(k, t)
            e.add_broker("b0/p0")
        rng = random.Random(18)
        frames = []
        for j in range(2000):                                  # small frames: cut on max_batch_msgs
            r = rng.random()
            sender = rng.choice(keys)
            if j in (1100, 1500, 1800):
                frames.append((sender, 0, orc.serialize(orc.KIND_SUBSCRIBE, bytes([rng.randrange(11)]))))
            elif r < 0.2:                                      # few enough broadcasts that max_batch_bcast does not cut first
                frames.append((sender, int(rng.random() < 0.2), orc.broadcast_frame(
                    [rng.randrange(14) for _ in range(rng.randrange(1, 3))], bytes([j & 255]) * rng.randrange(0, 100))))
            elif r < 0.99:
                rc = rng.choice(keys) if rng.random() < 0.9 else b"nobody"
                frames.append((sender, 0, orc.direct_frame(rc, bytes([j & 255]) * rng.randrange(0, 100))))
            else:
                frames.append((sender, 0, orc.broadcast_frame([200], b"only invalid topics")))
        for j in range(60):                                    # 12 KB broadcasts: cut on max_batch_bytes
            frames.append((keys[0], j % 2, orc.broadcast_frame([11], bytes([j]) * 12000)))
        for j in range(400):                                   # cut on max_batch_bcast
            frames.append((rng.choice(keys), 0, orc.broadcast_frame([j % 11], b"c%d" % j)))
        for j in range(6):                                     # 3000 topic entries each: cut on the topic entries
            frames.append((keys[1], j % 2, orc.broadcast_frame([(t + j) % 12 for t in range(3000)], b"t%d" % j)))
        assert len(frames) >= 2048
        a, b = engines
        rc_a, sizes_a, got_a, stops_a = _receive_all(pcdn, a, frames, batched=True)
        rc_b, sizes_b, got_b, stops_b = _receive_all(pcdn, b, frames, batched=False)
        assert rc_a == rc_b
        assert sizes_a == sizes_b
        assert got_a == got_b
        assert stops_a == stops_b and (stops_a >= 3 if pool else stops_a == 0)
        assert 1024 in sizes_a and len(sizes_a) >= 8
        assert a.stats().bytes_in == b.stats().bytes_in and a.stats().inflight_bytes == b.stats().inflight_bytes == 0
    finally:
        for e in engines:
            e.close()


def test_direct_key_placement(pcdn):
    """pcdn_submit reads a recipient key in place when it lies inside the frame at a 4-byte aligned
    offset, and stages it beside the frame when it lies at an offset of 1 mod 4 or in its own buffer.
    A recipient longer than max_key_len is dropped and counted."""
    w = World(pcdn, max_conns=256, max_key_len=128)
    rng = random.Random(3)
    keys = [bytes([i + 1]) * ln for i, ln in enumerate([8, 13, 32, 128, 1, 40] * 6)]
    for k in keys:
        w.add_user(k, [])
    bufs, arr = [], (pcdn.Msg * 64)()
    n = 0
    for j in range(60):
        k = keys[j % len(keys)]
        mode = j % 3                          # 0: in place (offset 0 mod 4), 1: offset 1 mod 4, 2: separate buffer
        pad = 4 * rng.randrange(1, 5) + (1 if mode == 1 else 0)
        raw = bytes([j]) * pad + k + bytes([j ^ 0x5A]) * rng.randrange(0, 200)
        buf = C.create_string_buffer(raw, len(raw))
        bufs.append(buf)
        if mode == 2:
            rcpt = C.create_string_buffer(k, len(k))
            bufs.append(rcpt)
            rp = C.cast(rcpt, C.c_char_p)
        else:
            rp = C.cast(C.addressof(buf) + pad, C.c_char_p)
        arr[n] = pcdn.Msg(pcdn.KIND_DIRECT, 0, 0, None, rp, len(k), len(raw), C.cast(buf, C.c_char_p))
        w.o.handle_direct_message(k, raw)
        n += 1
    long_key = keys[3] + b"!"                 # one byte over max_key_len: no recipient
    raw = orc.direct_frame(long_key, b"dropped")
    arr[n] = pcdn.Msg(pcdn.KIND_DIRECT, 0, 0, None, long_key, len(long_key), len(raw), raw)
    w.o.handle_direct_message(long_key, raw)
    n += 1
    bid = C.c_uint64(0)
    w.e._chk(w.e.L.pcdn_submit(w.e.h, arr, n, C.byref(bid)))
    res = w.e.poll(bid.value)
    assert res.n_msgs == n and res.status == 0
    assert res.n_direct_dropped == 1 and res.n_deliveries == n - 1
    got = w.e.collect_frames(res)
    w.e.release_batch(bid.value)
    want = w.expect()
    assert got == want


def test_topic_overflow_frame_in_threaded_call(pcdn):
    """A user broadcast whose kept topic entries exceed what one batch holds (8192 > 4 * 512 + 4096)
    gets PCDN_ENOSPC inside a 3000-frame pcdn_receive_frames call, as it does through user_receive;
    the call consumes every frame and the others are delivered as the oracle delivers them."""
    w = World(pcdn, n_valid_topics=2, max_batch_msgs=512, batch_slots=16, max_conns=1024, ring_bytes_per_conn=1 << 20)
    rng = random.Random(23)
    keys = [rng.getrandbits(64).to_bytes(8, "little") * 2 for _ in range(400)]
    for k in keys:
        w.add_user(k, [t for t in range(2) if rng.random() < 0.3])
    big = orc.broadcast_frame([0, 1] * 4096, b"too many topic entries")
    frames, want_rc = [], []
    for j in range(3000):
        sender = rng.choice(keys)
        if j == 1500:
            frames.append((sender, 0, big))
            want_rc.append(PCDN_ENOSPC)
            continue
        if rng.random() < 0.5:
            raw = orc.broadcast_frame([rng.randrange(2)], bytes([j & 255]) * rng.randrange(0, 300))
        else:
            raw = orc.direct_frame(rng.choice(keys), bytes([j & 255]) * rng.randrange(0, 300))
        frames.append((sender, 0, raw))
        want_rc.append(w.o.user_receive(sender, raw))
    rcs = w.e.receive_frames(frames)
    assert rcs == want_rc
    got = w.e.drain()
    want = w.expect()
    assert set(got) == set(want)
    for c in want:
        assert got[c] == want[c], c
    assert w.e.user_receive(keys[0], big) == PCDN_ENOSPC
