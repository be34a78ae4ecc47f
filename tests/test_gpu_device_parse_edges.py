"""The device frame parser (PCDN_FLAG_DEVICE_PARSE: k_parse walks the Cap'n Proto message on the GPU,
k_match / the fused control kernel read the wire topic list in place and apply Topic::prune while
matching, the direct lookup reads the recipient in place) on every layout and topic-list edge a peer
can send, built by hand (capnp_frames.py) rather than by the oracle's one canonical encoder.

Every frame goes to a host-parse engine and a device-parse engine configured alike, each beside its
own oracle.  Per frame: the synchronous return code equals the oracle's receive loop, or — on the
device path, for a Direct / Broadcast the host only peeks — the code arrives in the batch's
`msg_status` (and `n_msg_errors`); every connection's bytes equal the oracle's; the two engines agree
frame for frame.  One difference is by design: the host path refuses with PCDN_ENOSPC a broadcast
whose topic entries (kept after prune for user origin, listed for broker origin) exceed what one
batch's descriptor block holds (4 × max_batch_msgs + 4096), while device parse routes it.

Paths: the fused control kernel (batches of at most kSmallCtrlMsgs messages), the regular pipeline
(staged spans; test_regular_pipeline_batches_over_one_plan_block also cuts batches of more than 256
messages, so k_plan_b / k_plan_c run), three connection shards on GPU 0, shared-payload engines, and
one threaded pcdn_receive_frames call against the same frames sent one at a time."""
import ctypes as C
import random

import numpy as np
import pytest

import capnp_frames as cf
from gpu_world import PCDN_ENOSPC, PCDN_EPARSE, PCDN_EPRUNE, World, shard_cfg
from kconst import K
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

MAX_KEY = 128                      # pcdn_config_default's max_key_len
BLOCK = K.kBlockWords * 32        # connections per match block (k_match: one warp per block)
MAX_CONNS = BLOCK + 256            # two match blocks, the second one eight words long
PLAN_CTA_MSGS = 256                # messages per k_plan_a CTA: a larger batch runs k_plan_b / k_plan_c (launch_plan)
N_VALID = 12
PATHS = ["fused", "regular", "shards", "shared"]
# topics the subscribers hold: valid ids, the ids around N_VALID, and ids only a broker-origin list routes
SUB_TOPICS = [0, 1, 2, 3, 4, 11, 12, 13, 200, 254, 255]
# connection ids of the subscribers: both sides of 32-connection words and of the first match block's end
EDGES = [0, 1, 30, 31, 32, 33, 63, 64, 255, 256, 257, BLOCK - 2, BLOCK - 1, BLOCK, BLOCK + 1, BLOCK + 31, BLOCK + 32]


def topics_cap(max_batch_msgs):
    """topic entries one batch's descriptor block holds (engine.cu: topics_cap)"""
    return 4 * max_batch_msgs + 4096


def engine_cfg(pcdn, path, ring=1 << 20):
    """World keyword arguments of an ingress path ("shared": the fused path delivering by reference)"""
    base = dict(max_conns=MAX_CONNS, max_keys=16384, ring_bytes_per_conn=ring, batch_slots=16)
    if path == "fused":
        return dict(base, max_batch_msgs=K.kSmallCtrlMsgs, max_batch_bcast=K.kSmallCtrlMsgs)
    if path == "regular":
        return dict(base, max_batch_msgs=1024, max_batch_bcast=1024, flags=pcdn.FLAG_STAGED_SPANS)
    if path == "shards":
        return dict(base, max_batch_msgs=1024, max_batch_bcast=1024, **shard_cfg(pcdn, "shards-host"))
    return dict(base, max_batch_msgs=K.kSmallCtrlMsgs, max_batch_bcast=K.kSmallCtrlMsgs, delivery="shared")


def calls_of(pcdn, path):
    """frames per pcdn_receive_frames call: a batch the fused control kernel takes (at most
    kSmallCtrlMsgs messages and kSmallCtrlItems (broadcast, 8192-connection block) items), or more
    than kSmallCtrlMsgs messages for the regular pipeline"""
    if engine_cfg(pcdn, path)["max_batch_msgs"] <= K.kSmallCtrlMsgs:
        return min(K.kSmallCtrlMsgs, K.kSmallCtrlItems // -(-MAX_CONNS // (K.kBlockWords * 32)))
    return 3 * K.kSmallCtrlMsgs // 2


def make_world(pcdn, path, device_parse, n_valid=N_VALID, ring=1 << 20):
    kw = engine_cfg(pcdn, path, ring)
    kw["flags"] = kw.get("flags", 0) | (pcdn.FLAG_DEVICE_PARSE if device_parse else 0)
    w = World(pcdn, n_valid_topics=n_valid, **kw)
    rng = random.Random(3)
    keys = [cf.key_of(n) for n in cf.field_sizes(MAX_KEY)[:-1]] + [b"edge-%d" % i for i in range(len(EDGES))]
    conn = 0
    for i, at in enumerate(EDGES):
        if at > conn:   # fillers without subscriptions: they must receive nothing
            n = at - conn
            fill = np.zeros((n, 8), dtype=np.uint8)
            fill[:, :4] = np.arange(conn, at, dtype=np.uint32).view(np.uint8).reshape(n, 4)
            fill[:, 7] = 0xF1
            w.e.add_users_bulk(fill, 8)
        c = w.add_user(keys[i], sorted({SUB_TOPICS[i % len(SUB_TOPICS)], rng.choice(SUB_TOPICS)}))
        if path != "shards":
            assert c == at
        conn = at + 1
    for k in keys[len(EDGES):]:
        w.add_user(k, [rng.choice(SUB_TOPICS)])
    w.add_broker("b0/p0", [0, 3, 255])
    w.both("apply_user_sync", "b0/p0", [(b"far-away", 1, "b0/p0")])
    return w


SENDER = cf.key_of(8)


def kept(topics, n_valid):
    return sum(1 for i, t in enumerate(topics) if not (i and t == topics[i - 1]) and not (n_valid and t >= n_valid))


def host_refuses(w, raw, origin):
    """the host path's PCDN_ENOSPC: a broadcast whose entries can never fit one batch"""
    d = orc.deserialize(raw)
    if d is None or d[0] != cf.BROADCAST:
        return False
    n = len(d[1]) if origin else kept(d[1], w.cfg["n_valid_topics"])
    return n > topics_cap(w.cfg["max_batch_msgs"])


def drain(e, out, status, sizes):
    """flush, then poll, collect and release every outstanding batch; the nonzero msg_status values go
    to `status` in message order, each batch's message count to `sizes`.  Returns the batches'
    n_msg_errors."""
    e.flush()
    n_err = 0
    while True:
        b = e.next_batch()
        if not b:
            return n_err
        res = e.poll(b)
        if res.status == 11:
            e.retry_batch(b)
            res = e.poll(b)
        e.last_result = res
        sizes.append(res.n_msgs)
        assert res.status == 0 and res.n_overflow == 0, (res.status, res.n_overflow)
        for c, fr in e.collect_frames(res).items():
            out.setdefault(c, []).extend(fr)
        if res.msg_status:
            status.extend(res.msg_status[i] for i in range(res.n_msgs) if res.msg_status[i])
        n_err += res.n_msg_errors
        e.release_batch(b)


def feed(pk, e, frames, chunk):
    """pcdn_receive_frames over `frames`, `chunk` frames per call, every batch drained after each call
    and whenever the engine stops early → (return codes, {conn: frames}, nonzero msg_status values in
    message order, sum of n_msg_errors, message count of every batch)"""
    n = len(frames)
    arr = (pk.Frame * max(1, n))()
    for i, (sender, origin, raw) in enumerate(frames):
        arr[i] = pk.Frame(sender, len(sender), origin, raw, len(raw), 0)
    rcs = (C.c_int32 * max(1, n))()
    out, status, sizes, n_err, pos = {}, [], [], 0, 0
    while pos < n:
        k = min(chunk, n - pos)
        done = e.L.pcdn_receive_frames(e.h, C.cast(C.byref(arr, pos * C.sizeof(pk.Frame)), C.POINTER(pk.Frame)), k,
                                       C.cast(C.byref(rcs, pos * 4), C.POINTER(C.c_int32)))
        assert done == -11 or done > 0, (done, e.L.pcdn_last_error())   # -11: every batch slot in flight
        pos += max(done, 0)
        n_err += drain(e, out, status, sizes)
    return list(rcs[:n]), out, status, n_err, sizes


def check(w, frames, device_parse, chunk=200):
    """send `frames` to w's engine and its oracle; returns the engine's codes (and keeps the message
    count of every batch in w.batch_msgs)"""
    want = []
    for s, o, raw in frames:
        if not device_parse and host_refuses(w, raw, o):
            want.append(PCDN_ENOSPC)        # by design: the oracle routes it, the host path refuses it
            continue
        want.append(w.o.broker_receive(raw) if o else w.o.user_receive(s, raw))
    rcs, got, status, n_err, w.batch_msgs = feed(w.pcdn, w.e, frames, chunk)
    if device_parse:
        bad = [(i, r, x) for i, (r, x) in enumerate(zip(rcs, want)) if r != x and not (r == 0 and x in (PCDN_EPARSE, PCDN_EPRUNE))]
        assert not bad, bad[:5]
        deferred = [(i, x) for i, (r, x) in enumerate(zip(rcs, want)) if r == 0 and x < 0]
        first = next((j for j, (s, d) in enumerate(zip(status, deferred)) if s != d[1]), min(len(status), len(deferred)))
        assert status == [x for _, x in deferred] and n_err == len(deferred), \
            (len(status), len(deferred), first, deferred[first:first + 1], frames[deferred[first][0]][2].hex() if first < len(deferred) else None)
    else:
        bad = [(i, r, x) for i, (r, x) in enumerate(zip(rcs, want)) if r != x]
        assert not bad, bad[:5]
        assert status == [] and n_err == 0
    exp = w.expect()
    assert w.compare(w.e, got, exp) >= 0
    return rcs


def both_paths(pcdn, path, frames, n_valid=N_VALID, chunk=None):
    """host parse and device parse on the same frames: each against its oracle, then frame for frame
    against each other; returns (host codes, device codes, (largest host batch, largest device batch))"""
    chunk = calls_of(pcdn, path) if chunk is None else chunk
    wh = make_world(pcdn, path, False, n_valid)
    wd = make_world(pcdn, path, True, n_valid)
    try:
        rh = check(wh, frames, False, chunk)
        rd = check(wd, frames, True, chunk)
        for i, (a, b) in enumerate(zip(rh, rd)):
            refused = host_refuses(wh, frames[i][2], frames[i][1])
            assert a == b or (b == 0 and a in (PCDN_EPARSE, PCDN_EPRUNE)) or (refused and a == PCDN_ENOSPC and b == 0), (i, a, b)
        return rh, rd, (max(wh.batch_msgs, default=0), max(wd.batch_msgs, default=0))
    finally:
        wh.e.close()
        wd.e.close()


def corpus_frames(specs):
    out = []
    for name, spec in specs:
        raw = cf.frame(spec)
        out.append((SENDER, 0, raw))
        out.append((b"", 1, raw))
    return out


# ------------------------------------------------------------------------------------- a. layouts
@pytest.mark.parametrize("path", PATHS)
def test_layout_corpus(pcdn, path):
    """every layout family (valid and malformed) × Direct, Broadcast, Subscribe, Unsubscribe, sync and
    auth kinds × field sizes 0, 1, 7, 8, 9, max_key_len − 1 / max_key_len / + 1, messages on both sides
    of the 1024-word first segment, from user and from broker origin"""
    frames = corpus_frames(cf.corpus(MAX_KEY))
    rh, rd, _ = both_paths(pcdn, path, frames)
    assert rh.count(PCDN_EPARSE) > 1000 and rd.count(0) > 1500


# ------------------------------------------------------------------------------------- b. mutation
@pytest.mark.parametrize("path", PATHS)
def test_structure_aware_mutation(pcdn, path):
    """the corpus with segment-table counts and sizes, pointer kind bits, offsets, far / double-far bits
    and target segments, list element sizes and counts and the union tag (8, 9, 0xFFFF) changed
    anywhere in the frame — 3000 frames per path, fixed seeds"""
    rng = random.Random(PATHS.index(path) + 100)
    specs = cf.corpus(MAX_KEY, kinds=(cf.DIRECT, cf.BROADCAST, cf.SUBSCRIBE))
    frames = []
    while len(frames) < 3000:
        name, spec = specs[rng.randrange(len(specs))]
        raw, lay = cf.build(spec)
        frames.append((SENDER, int(rng.random() < 0.3), cf.mutate(rng, raw, lay)))
    both_paths(pcdn, path, frames)


# ------------------------------------------------------------------------------------- c. topic lists
LENGTHS = [0, 1, 2, 31, 32, 33, 255, 256, 257, 8191, 8192, 8193, 20000]


def topic_shapes(n, n_valid):
    bad = 200 if n_valid else None         # an id Topic::prune drops (none when every id is valid)
    inv = bad if bad is not None else 255
    cyc = lambda vals: [vals[i % len(vals)] for i in range(n)]
    out = {
        "one-value": [0] * n,
        "alternating": cyc([0, 1]),
        "every-value": [i % 256 for i in range(n)],
        "dups-at-ends": ([3] * 3 + cyc([1, 2]) + [4] * 3)[:n] if n < 6 else [3] * 3 + cyc([1, 2])[:n - 6] + [4] * 3,
        "invalid-first": [inv] + cyc([2, 11])[: max(n - 1, 0)] if n else [],
        "invalid-last": cyc([2, 11])[: max(n - 1, 0)] + [inv] if n else [],
        "invalid-but-one": [inv] * (n // 2) + [13 if not n_valid else 1] + [inv] * (n - n // 2 - 1) if n else [],
        "around-n-valid": cyc([max(n_valid, 1) - 1, n_valid, 255]),
    }
    return {k: v[:n] for k, v in out.items()}


def topic_frames(n_valid, rng):
    frames = []
    for n in LENGTHS:
        for shape, topics in topic_shapes(n, n_valid).items():
            raw = cf.frame(cf.Spec(cf.BROADCAST, bytes(topics), bytes([n & 0xFF, len(shape)]) * rng.randrange(1, 40)))
            frames.append((SENDER, 0, raw))
            frames.append((b"", 1, raw))
    return frames


@pytest.mark.parametrize("n_valid", [0, N_VALID])
@pytest.mark.parametrize("path", PATHS)
def test_topic_lists_in_place(pcdn, path, n_valid):
    """wire topic lists of 0 … 20000 entries: one value, alternating, every value, consecutive
    duplicates at both ends, invalid ids first / last / everywhere but one, ids n_valid − 1, n_valid,
    255 — pruned for user origin, verbatim (users only) for broker origin; subscribers on the 32- and
    8192-connection edges.  A list whose entries exceed the descriptor block: PCDN_ENOSPC on the host
    path, routed by device parse"""
    frames = topic_frames(n_valid, random.Random(n_valid))
    rh, rd, _ = both_paths(pcdn, path, frames, n_valid)
    cap = topics_cap(engine_cfg(pcdn, path)["max_batch_msgs"])
    entries = [len(t) if o else kept(t, n_valid) for t, o in ((orc.deserialize(raw)[1], o) for s, o, raw in frames)]
    refused = [i for i, n in enumerate(entries) if n > cap]
    assert refused and [i for i, r in enumerate(rh) if r == PCDN_ENOSPC] == refused
    assert all(rd[i] == 0 for i in refused)


@pytest.mark.parametrize("path", ["regular", "shards"])
def test_regular_pipeline_batches_over_one_plan_block(pcdn, path):
    """Direct and Broadcast frames only — every valid and malformed layout family with small messages,
    and topic lists of up to 33 entries in every shape — in one pcdn_receive_frames call, so that no
    state change cuts the batch: both engines route batches of more than one k_plan_a CTA of messages,
    where launch_plan also runs k_plan_b and k_plan_c"""
    rng = random.Random(77)
    specs = [s for s in cf.corpus(MAX_KEY, kinds=(cf.DIRECT, cf.BROADCAST))
             if len(s[1].f1) < 100 and (s[1].kind == cf.DIRECT or len(s[1].f0) <= 9)]
    frames = corpus_frames(specs) + [f for f in topic_frames(N_VALID, rng) if len(orc.deserialize(f[2])[1]) <= 33]
    rng.shuffle(frames)
    assert len(frames) < engine_cfg(pcdn, path)["max_batch_msgs"]
    rh, rd, largest = both_paths(pcdn, path, frames, chunk=len(frames))
    assert min(largest) > PLAN_CTA_MSGS, largest
    assert rh.count(PCDN_EPARSE) > 50 and rd.count(0) > 2 * PLAN_CTA_MSGS


# ------------------------------------------------------------------------------------- d. threaded call
@pytest.mark.parametrize("device_parse", [False, True], ids=["host-parse", "device-parse"])
def test_threaded_call_matches_one_at_a_time(pcdn, device_parse):
    """one pcdn_receive_frames call of more than 2048 frames (the threaded parse / peek and copy) and the
    same frames one call per frame: identical codes and identical streams, both equal to the oracle"""
    rng = random.Random(41)
    # small messages only: every batch of the one call is in flight at once, within the rings
    specs = [s for s in cf.corpus(MAX_KEY, kinds=(cf.DIRECT, cf.BROADCAST, cf.SUBSCRIBE, 0)) if len(s[1].f1) < 100]
    frames = topic_frames(N_VALID, rng)
    for rep in range(3):
        for name, spec in specs:
            raw, lay = cf.build(spec)
            frames.append((SENDER, int(rng.random() < 0.3), raw if rep == 0 else cf.mutate(rng, raw, lay)))
    rng.shuffle(frames)
    assert len(frames) >= 2048
    codes = []
    for chunk in (len(frames), 1):
        w = make_world(pcdn, "regular", device_parse, ring=2 << 20)
        try:
            codes.append(check(w, frames, device_parse, chunk))
        finally:
            w.e.close()
    assert codes[0] == codes[1]


# ------------------------------------------------------------------------------------- long lists
@pytest.mark.parametrize("device_parse", [False, True], ids=["host-parse", "device-parse"])
def test_long_topic_list_broadcast(pcdn, device_parse):
    """a broadcast whose wire list has more than 8192 entries is routed as the reference routes it: from
    a user, [0] * 9000 prunes to topic 0; from a broker the 9000 entries are kept verbatim"""
    w = World(pcdn, n_valid_topics=N_VALID, flags=pcdn.FLAG_DEVICE_PARSE if device_parse else 0)
    a = w.add_user(b"a" * 8, [0])
    w.add_user(b"b" * 8, [1])
    w.add_broker("b0/p0", [0])
    for origin in (0, 1):
        for topics in ([0] * 9000, [0] * 8193, [1] + [0] * 9000 + [200] * 3):
            raw = orc.broadcast_frame(topics, b"long list %d" % origin)
            want = w.o.broker_receive(raw) if origin else w.o.user_receive(b"a" * 8, raw)
            got = w.e.receive_frames([(b"a" * 8, origin, raw)])
            assert got == [want] == [0], pcdn.lib().pcdn_last_error()
    got = w.e.drain()
    assert len(got[a]) == 6 and w.compare(w.e, got, w.expect()) == 6 + 2 + 3   # a: all six; b: the [1, ...] pair; broker: user origin
    w.e.close()
