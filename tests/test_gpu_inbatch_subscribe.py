"""In-batch subscription changes (PCDN_FLAG_INBATCH_SUBSCRIBE): a Subscribe / Unsubscribe, from the C ABI
or a user's frame, becomes an event of the open batch instead of launching it.

Every case runs ONE call sequence on three backends: an engine with the flag, the same engine without
it, and the oracle (which applies every call at once).  Each connection's delivered byte stream must be
equal on all three, and the flagged engine must launch the batches the case expects (pcdn_stats.batches).
The cases run on the engine variants that change how a match is computed or consumed: the fused and the
regular control kernels, run-length spans, the output pool, shared payload, three shards on one GPU and
device parse."""
import pytest

import gpu_workloads as workloads
from gpu_workloads import BASE, CASES, SUB, UNSUB, Trio, case_capacity_fallback, key, sub_frame
from gpu_world import STATUS_EAGAIN, layout
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

# (layout, delivery) under this file's test ids
FUSED = pytest.param("rings", "copy", id="fused")
STAGED = pytest.param("staged", "copy", id="staged")
POOL = pytest.param("pool", "copy", id="pool")
SHARDS = pytest.param("shards-host", "copy", id="shards")
DEVPARSE = pytest.param("devparse", "copy", id="devparse")
VARIANTS = [FUSED, STAGED, pytest.param("runs-staged", "copy", id="runs"), POOL,
            pytest.param("rings", "shared", id="shared"), SHARDS, DEVPARSE]


@pytest.mark.parametrize("variant,delivery", VARIANTS)
@pytest.mark.parametrize("case", CASES, ids=lambda f: f.__name__[5:])
def test_inbatch_subscribe(pcdn, case, variant, delivery):
    workloads.inbatch_subscribe(pcdn, case, variant, delivery)


@pytest.mark.parametrize("variant,delivery", [FUSED, STAGED, SHARDS])
def test_event_capacity_fallback(pcdn, variant, delivery):
    t = Trio(pcdn, variant, delivery=delivery, max_batch_msgs=8)
    try:
        case_capacity_fallback(t)
        t.check()
        # 12 events on 8-event batches: the 9th launches the first batch, which holds the 4 broadcasts
        # before it; the rest is the second batch
        assert t.batches() == 2
    finally:
        t.close()


@pytest.mark.parametrize("variant,delivery", [FUSED, STAGED, SHARDS])
def test_hooked_subscribe(pcdn, variant, delivery):
    """a user hook rewrites the topics of a Subscribe frame: the event carries the rewritten topics"""
    t = Trio(pcdn, variant, delivery=delivery)
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


@pytest.mark.parametrize("variant,delivery", [FUSED, STAGED, POOL, SHARDS])
def test_pool_retry_keeps_events(pcdn, variant, delivery):
    """a batch with events refused by the output pool and retried: it is routed as it was launched"""
    cfg = layout(pcdn, variant)
    cfg["flags"] = cfg.get("flags", 0) | pcdn.FLAG_OUTPUT_POOL
    cfg.update(pool_bytes=4 << 20, batch_slots=16, max_batch_bytes=8 << 20)   # (slots: the unflagged engine cuts 13 batches)
    t = Trio(pcdn, "rings", delivery=delivery, **cfg)
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
        assert e.poll(b).status == STATUS_EAGAIN   # refused: the pool is held by the first batch
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


@pytest.mark.parametrize("variant,delivery", [FUSED, STAGED, DEVPARSE, SHARDS])
def test_threaded_receive(pcdn, variant, delivery):
    """one threaded pcdn_receive_frames call of 4096 frames with Subscribe / Unsubscribe frames spread
    through it: the flagged engine consumes every frame in one call and one batch; without the flag the
    call stops early (each change cuts the batch and the batch slots run out)"""
    t = Trio(pcdn, variant, delivery=delivery, n_valid_topics=16, max_batch_msgs=4096, max_batch_bcast=4096, batch_slots=4)
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
