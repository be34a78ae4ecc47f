"""GPU tests of two boundary rows: the MessageHookDef seam on routed messages (SURVEY 8a10,
cdn-proto/src/def.rs:79-92) and inter-broker sync applied to a GPU-resident engine (SURVEY 8f-4,
cdn-broker/src/tasks/broker/{sync.rs,handler.rs:164-188}) — both against the oracle, through the C ABI."""
import ctypes as C
import random

import pytest

from gpu_world import World, payload, shard_cfg
from oracle import oracle as orc

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("devparse", [False, True])
def test_message_hook_on_routed_messages(pcdn, devparse):
    """Skip / Err / mutation of the routing fields before dispatch; the forwarded bytes stay the
    inbound frame.  With PCDN_FLAG_DEVICE_PARSE a hooked origin is parsed on the host (documented)."""
    w = World(pcdn, max_conns=256, flags=pcdn.FLAG_DEVICE_PARSE if devparse else 0, n_valid_topics=8)
    a, b, c = b"alice-key-000001", b"bob-key-00000002", b"carol-key-000003"
    w.add_user(a, [1]); w.add_user(b, [2]); w.add_user(c, [3])
    w.add_broker("p/p", [2])
    log = []

    def user_hook(m):
        raw = C.string_at(m.raw, m.raw_len)
        log.append((m.kind, raw))
        if m.kind == pcdn.KIND_DIRECT:
            rc = C.string_at(m.recipient, m.recipient_len)
            if rc == b"blocked-recipient":
                return pcdn.HOOK_SKIP
            if rc == b"poison":
                return -5
            if rc == a:                 # reroute alice's directs to carol (parsed message only)
                buf = C.create_string_buffer(c, len(c))
                user_hook.keep = buf
                m.recipient = C.cast(buf, C.c_void_p).value
                m.recipient_len = len(c)
        elif m.kind == pcdn.KIND_BROADCAST and m.n_topics == 2:
            m.topics[0] = 3             # [1, 2] -> [3]
            m.n_topics = 1
        return pcdn.HOOK_PROCESS

    w.e.set_message_hook(0, user_hook)
    sender = b
    f1 = orc.direct_frame(a, b"to alice, lands at carol")
    f2 = orc.direct_frame(b"blocked-recipient", b"never routed")
    f3 = orc.broadcast_frame([1, 2], b"rewritten to topic 3")
    f4 = orc.broadcast_frame([2], b"untouched")
    f5 = orc.direct_frame(b"poison", b"x")
    assert w.e.user_receive(sender, f1) == 0
    w.o.handle_direct_message(c, f1, False)            # what the mutated message routes to; bytes = f1
    assert w.e.user_receive(sender, f2) == 0           # skipped
    assert w.e.user_receive(sender, f3) == 0
    w.o.handle_broadcast_message([3], f3, False)
    assert w.e.user_receive(sender, f4) == 0
    w.o.handle_broadcast_message([2], f4, False)
    assert w.e.user_receive(sender, f5) == -13         # Err => the host disconnects the sender
    assert [k for k, _ in log] == [3, 3, 4, 4, 3] and log[0][1] == f1
    assert w.check() == 4                              # carol x2 (f1, f3), bob + broker p/p (f4)
    # broker-side hook: frames from a peer broker
    seen = []
    w.e.set_message_hook(1, lambda m: (seen.append(C.string_at(m.sender, m.sender_len)), pcdn.HOOK_SKIP if m.kind == 4 else 0)[1])
    f6, f7 = orc.broadcast_frame([1], b"skipped"), orc.direct_frame(a, b"kept")
    assert w.e.broker_receive("p/p", f6) == 0 and w.e.broker_receive("p/p", f7) == 0
    w.o.handle_direct_message(a, f7, True)
    assert seen == [b"p/p", b"p/p"]
    assert w.check() == 1
    w.e.close()


@pytest.mark.parametrize("variant", ["single", "shards-host"])
def test_inter_broker_sync_on_a_gpu_engine(pcdn, variant):
    """f-4 on the device: broker A (the GPU engine) and broker B (a second engine's tables) exchange
    user-sync and topic-sync maps exactly as tests/test_sync_maps.py does on CPU, with two oracle
    brokers exchanging the reference's maps beside them; after every exchange A's GPU must route
    directs (local / remote via B / unknown) and broadcasts exactly like oracle A."""
    cfg = shard_cfg(pcdn, variant) if variant != "single" else {}
    w = World(pcdn, max_conns=512, identity="a/a", **cfg)
    w.o = orc.Oracle("a/a")
    eb, ob = pcdn.Engine(device=-1, max_conns=512, max_keys=4096, identity="b/b"), orc.Oracle("b/b")
    rng = random.Random(13)
    ka = [b"a-user-%02d" % i for i in range(40)]
    kb = [b"b-user-%02d" % i for i in range(40)]
    for k in ka:
        w.add_user(k, [rng.randrange(4)])
    for k in kb:
        t = [rng.randrange(4)]
        eb.add_user(k, t); ob.add_user(k, t)
    w.add_broker("b/b")
    eb.add_broker("a/a"); ob.add_broker("a/a")

    def exchange(full):
        # B -> A and A -> B, user maps then topic maps (sync.rs:44-128; handler.rs:164-188)
        for (src_e, src_o, dst_e, dst_o, name) in ((eb, ob, w.e, w.o, "b/b"), (w.e, w.o, eb, ob, "a/a")):
            ents = src_e.get_user_sync(full)
            assert bool(ents) == src_o.user_sync_to(dst_o, full=full)
            if ents:
                dst_e.apply_user_sync(name, ents)
            ents = src_e.get_topic_sync(full)
            assert bool(ents) == src_o.topic_sync_to(dst_o, name, full=full)
            if ents:
                dst_e.apply_topic_sync(name, ents)

    delivered = 0
    for rnd in range(5):
        exchange(full=(rnd == 0))
        for j in range(60):
            if rng.random() < 0.5:
                k = rng.choice(ka + kb + [b"nobody"])
                w.direct(k, orc.direct_frame(k, payload(rng, 50 + j)), rng.random() < 0.3)
            else:
                t = [rng.randrange(4)]
                w.bcast(t, orc.broadcast_frame(t, payload(rng, 300)), rng.random() < 0.3)
        delivered += w.check()
        # churn: some of B's users reconnect to A, some of A's to B, some leave; B's interest moves
        for k in rng.sample(kb, 4):
            eb.remove_user(k); ob.remove_user(k)
            w.add_user(k, [rng.randrange(4)])
        for k in rng.sample(ka, 3):
            w.both("remove_user", k)
            t = [rng.randrange(4)]
            eb.add_user(k, t); ob.add_user(k, t)
        k, t = rng.choice(kb), [rng.randrange(4)]
        eb.subscribe_user_to(k, t); ob.subscribe_user_to(k, t)
    assert delivered > 300
    w.e.close()
