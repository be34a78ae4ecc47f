"""CPU tests of the product's host side through the C ABI with a host-only engine (device=-1):
the `Connections` mirror (bitmap / route table the GPU kernels read) against the oracle, the ingress
frame parser against the oracle's capnp restatement, and the ABI surface itself.  No compute calls.
"""
import ctypes as C
import os
import random
import re

import pytest

from oracle import oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol(pcdn):
    hdr = open(os.path.join(ROOT, "include", "pcdn_fanout.h")).read()
    declared = set(re.findall(r"\b(pcdn_[a-z_0-9]+)\s*\(", hdr))
    declared -= {"pcdn_engine"}
    assert len(declared) >= 30
    L = C.CDLL(pcdn.LIB_PATH)
    for name in sorted(declared):
        assert hasattr(L, name), f"{name} declared in pcdn_fanout.h but not exported"
    assert set(pcdn.ABI) == declared, (set(pcdn.ABI) ^ declared)


def test_no_cpu_data_path(pcdn):
    """the product must fail loudly without a device instead of falling back"""
    e = pcdn.Engine(device=-1, max_conns=64)
    e.add_user(b"k", [0])
    with pytest.raises(pcdn.PcdnError) as ei:
        e.handle_broadcast_message([0], b"12345678")
    assert ei.value.code == -3
    with pytest.raises(pcdn.PcdnError):
        e.handle_direct_message(b"k", b"12345678")
    assert e.user_receive(b"k", orc.broadcast_frame([0], b"x")) == -3


def test_product_does_not_import_oracle(pcdn):
    src = open(os.path.join(ROOT, "push-cdn_b200", "__init__.py")).read()
    assert "oracle" not in src.replace("oracle's", "")
    pk = os.path.join(ROOT, "push-cdn_b200")
    for d, _, files in os.walk(pk):
        for f in files:
            if f.endswith((".cu", ".cuh", ".cpp", ".h", ".py")):
                src = open(os.path.join(d, f)).read().lower().replace("oracle's", "")
                assert "import oracle" not in src and "from oracle" not in src and "oracle/" not in src, f


def _mk(pcdn, **kw):
    cfg = dict(device=-1, max_conns=512, max_topics=256, max_keys=2048, max_key_len=128, identity="me/me")
    cfg.update(kw)
    return pcdn.Engine(**cfg), orc.Oracle("me/me")


class Pair:
    """drives the product's host mirror and the oracle with the same calls; maps connection ids"""

    def __init__(self, pcdn, **kw):
        self.e, self.o = _mk(pcdn, **kw)
        self.map = {}  # engine conn -> oracle conn

    def add_user(self, k, t):
        self.map[self.e.add_user(k, t)] = self.o.add_user(k, t)

    def add_broker(self, b):
        self.map[self.e.add_broker(b)] = self.o.add_broker(b)

    def both(self, name, *a):
        getattr(self.e, name)(*a)
        getattr(self.o, name)(*a)

    def check(self, keys, rng):
        for _ in range(6):
            topics = [rng.randrange(8) for _ in range(rng.randrange(0, 4))]
            for flag in (False, True):
                got = sorted(self.map[c] for c in self.e.debug_interested(topics, flag))
                assert got == self.o.interested(topics, flag), (topics, flag)
        for k in keys:
            kind, conn = self.e.debug_route(k)
            okind, oconn = self.o.route(k)
            assert kind == okind, k
            assert (self.map[conn] if conn >= 0 else -1) == oconn, k
        assert self.e.num_users()[0] == self.o.num_users()


@pytest.mark.parametrize("seed", range(6))
def test_connections_mirror_matches_oracle(pcdn, seed):
    """random Connections::* call sequences (mod.rs:252-388 + apply_user_sync :154): the product's
    bitmap and route table resolve exactly like the reference's maps"""
    rng = random.Random(seed)
    p = Pair(pcdn)
    keys = [bytes([i]) * rng.choice([1, 8, 33, 128]) for i in range(24)]
    brokers = [f"b{i}/p{i}" for i in range(4)]
    for step in range(400):
        op = rng.randrange(10)
        k = rng.choice(keys)
        b = rng.choice(brokers)
        t = [rng.randrange(8) for _ in range(rng.randrange(0, 4))]
        if op == 0:
            p.add_user(k, t)
        elif op == 1:
            p.both("remove_user", k)
        elif op == 2:
            p.both("subscribe_user_to", k, t)
        elif op == 3:
            p.both("unsubscribe_user_from", k, t)
        elif op == 4:
            p.add_broker(b)
        elif op == 5:
            p.both("remove_broker", b)
        elif op == 6:
            p.both("subscribe_broker_to", b, t)
        elif op == 7:
            p.both("unsubscribe_broker_from", b, t)
        else:
            ents = [(rng.choice(keys), rng.randrange(1, 5), rng.choice(brokers + ["me/me", None]))
                    for _ in range(rng.randrange(1, 4))]
            # one entry per key (a remote map is a map)
            ents = list({e[0]: e for e in ents}.values())
            p.both("apply_user_sync", rng.choice(brokers), ents)
        if step % 20 == 0:
            p.check(keys, rng)
    p.check(keys, rng)


def test_add_user_kicks_same_key_and_reuses_ids(pcdn):
    e, _ = _mk(pcdn, max_conns=4)
    a = e.add_user(b"A", [1])
    b = e.add_user(b"A", [2])       # same key: old connection kicked (mod.rs:289-290)
    assert e.num_users() == (1, 0)
    assert e.debug_interested([1]) == [] and e.debug_interested([2]) == [b]
    for i in range(3):
        e.add_user(b"u%d" % i, [])
    with pytest.raises(pcdn.PcdnError) as ei:
        e.add_user(b"overflow", [])
    assert ei.value.code == -5       # PCDN_ENOSPC, state unchanged
    assert e.num_users() == (4, 0) and e.debug_route(b"overflow") == (0, -1)
    e.remove_user(b"u0")
    assert e.add_user(b"again", [7]) in (a, b, 0, 1, 2, 3)


def test_key_length_limit(pcdn):
    e, _ = _mk(pcdn, max_key_len=32)
    e.add_user(b"x" * 32, [])
    with pytest.raises(pcdn.PcdnError) as ei:
        e.add_user(b"x" * 33, [])
    assert ei.value.code == -6


def test_cuckoo_table_many_keys(pcdn):
    """fill the direct map to its configured capacity; every key resolves, erased keys do not"""
    n = 20000
    e = pcdn.Engine(device=-1, max_conns=n, max_keys=n, max_key_len=16)
    rng = random.Random(1)
    keys = [rng.getrandbits(128).to_bytes(16, "little") for _ in range(n)]
    conns = [e.add_user(k, []) for k in keys]
    for k, c in zip(keys[::97], conns[::97]):
        assert e.debug_route(k) == (1, c)
    for k in keys[:5000]:
        e.remove_user(k)
    for k in keys[:5000:53]:
        assert e.debug_route(k) == (0, -1)
    for k, c in zip(keys[5000::101], conns[5000::101]):
        assert e.debug_route(k) == (1, c)


def test_parse_frame_matches_oracle(pcdn):
    rng = random.Random(3)
    for _ in range(300):
        kind = rng.choice([3, 4, 5, 6, 7, 8])
        f0 = bytes(rng.randrange(256) for _ in range(rng.choice([0, 1, 2, 8, 9, 128])))
        pl = bytes(rng.randrange(256) for _ in range(rng.choice([0, 1, 7, 8, 100, 9000])))
        if kind in (5, 6):
            raw = orc.serialize(kind, f0)
        elif kind in (7, 8):
            raw = orc.serialize(kind, b"", pl)
        else:
            raw = orc.serialize(kind, f0, pl)
        k, topics, (off, ln) = pcdn.parse_frame(raw)
        ok, of0, opl = orc.deserialize(raw)
        assert k == ok == kind
        want = opl if kind in (7, 8) else of0
        assert raw[off:off + ln] == want
        if kind in (4, 5, 6):
            assert bytes(topics) == of0[:256]


def test_parse_frame_rejects_what_the_oracle_rejects(pcdn):
    rng = random.Random(4)
    good = [orc.broadcast_frame([0, 1], b"payload" * 3), orc.direct_frame(b"k" * 8, b"m" * 40),
            orc.broadcast_frame([1], bytes(9000))]
    n_bad = 0
    for _ in range(3000):
        raw = bytearray(rng.choice(good))
        for _ in range(rng.randrange(1, 4)):
            raw[rng.randrange(min(len(raw), 64))] = rng.randrange(256)
        if rng.random() < 0.2:
            raw = raw[: rng.randrange(len(raw))]
        raw = bytes(raw)
        want = orc.deserialize(raw)
        try:
            k, topics, (off, ln) = pcdn.parse_frame(raw)
        except pcdn.PcdnError as ex:
            assert ex.code == -7
            assert want is None, raw.hex()
            n_bad += 1
            continue
        assert want is not None, raw.hex()
        assert k == want[0]
        if k in (3, 4, 5, 6):
            assert raw[off:off + ln] == want[1]
    assert n_bad > 100


def test_prune_and_dispatch_errors(pcdn):
    """user_receive_loop error paths (user/handler.rs:133,142,153,160) need no device"""
    e = pcdn.Engine(device=-1, max_conns=16, n_valid_topics=2)
    e.add_user(b"u", [0])
    assert e.user_receive(b"u", b"\x01\x02") == -7                        # Error::Deserialize
    assert e.user_receive(b"u", orc.serialize(orc.KIND_SUBSCRIBE, bytes([9]))) == -8   # prune → Err
    assert e.user_receive(b"u", orc.serialize(orc.KIND_USER_SYNC, b"", b"x")) == -9    # invalid kind
    assert e.user_receive(b"u", orc.serialize(orc.KIND_SUBSCRIBE, bytes([1, 1, 9]))) == 0
    assert e.debug_interested([1]) == [0]
    assert e.user_receive(b"u", orc.serialize(orc.KIND_UNSUBSCRIBE, bytes([1]))) == 0
    assert e.debug_interested([1]) == []
    assert e.user_receive(b"u", orc.broadcast_frame([7], b"x")) == -8      # only invalid topics


@pytest.mark.parametrize("inbatch", [False, True], ids=["plain", "inbatch-subscribe"])
def test_receive_frames_call_on_a_host_only_engine(pcdn, inbatch):
    """One pcdn_receive_frames call of 3000 frames classifies them on several threads, also on a
    host-only engine.  The frames hold no routable message: Subscribe / Unsubscribe (from users, unknown
    senders and a peer broker), truncated frames, invalid kinds and topic lists with no valid topic.  The
    codes, the mirror and pcdn_last_error afterwards equal what the same frames leave one at a time."""
    flags = pcdn.FLAG_INBATCH_SUBSCRIBE if inbatch else 0
    rng = random.Random(31)
    keys = [b"user%03d" % i for i in range(200)]
    subs = [[rng.randrange(48) for _ in range(rng.randrange(3))] for _ in keys]
    engines = [pcdn.Engine(device=-1, max_conns=512, max_topics=64, max_keys=1024, n_valid_topics=48, flags=flags)
               for _ in range(2)]
    for e in engines:
        for k, t in zip(keys, subs):
            e.add_user(k, t)
        e.add_broker("p/p")
    frames = []
    for j in range(3000):
        sender = rng.choice(keys) if rng.random() < 0.95 else b"stranger%d" % j
        kind = orc.KIND_SUBSCRIBE if rng.random() < 0.6 else orc.KIND_UNSUBSCRIBE
        sub = orc.serialize(kind, bytes(rng.randrange(48) for _ in range(rng.randrange(1, 5))))
        r = rng.random()
        if r < 0.5:
            frames.append((sender, 0, sub))
        elif r < 0.6:                                             # no valid topic: PCDN_EPRUNE
            frames.append((sender, 0, orc.serialize(kind, bytes(rng.randrange(48, 256) for _ in range(rng.randrange(3))))))
        elif r < 0.7:                                             # truncated: PCDN_EPARSE
            frames.append((sender, 0, sub[:rng.randrange(len(sub))]))
        elif r < 0.8:                                             # PCDN_EKIND
            frames.append((sender, 0, orc.serialize(rng.choice([orc.KIND_USER_SYNC, orc.KIND_TOPIC_SYNC]), b"", b"x")))
        else:                                                     # broker origin: not routed here (1)
            frames.append((b"p/p", 1, sub))
    frames.append((keys[0], 0, orc.serialize(orc.KIND_USER_SYNC, b"", b"last")))
    a, b = engines
    want = [b.broker_receive(s.decode(), raw) if o else b.user_receive(s, raw) for s, o, raw in frames]
    want_err = pcdn.lib().pcdn_last_error().decode()
    assert want_err == "invalid message received" and {0, 1, -7, -8, -9} <= set(want)
    with pytest.raises(pcdn.PcdnError):
        a.add_user(b"k" * 300, [])                                # leaves another error text behind
    assert a.receive_frames(frames) == want
    assert pcdn.lib().pcdn_last_error().decode() == want_err

    def mirror(e):
        return ([sorted(e.debug_interested([t], to_users_only=uo)) for t in range(64) for uo in (False, True)],
                sorted(e.get_user_sync(full=True)), sorted(e.get_topic_sync(full=True)), e.num_users())

    assert mirror(a) == mirror(b)
    for e in engines:
        e.close()


def test_state_calls_from_many_threads(pcdn):
    """the engine serialises callers internally (one mutex = the reference's RwLock<Connections>):
    concurrent add/subscribe/remove from several host threads leave a consistent table"""
    import threading

    e = pcdn.Engine(device=-1, max_conns=8192, max_keys=16384, max_key_len=16)

    def work(t):
        for i in range(1500):
            k = bytes([t]) + i.to_bytes(4, "little")
            e.add_user(k, [t % 8])
            e.subscribe_user_to(k, [(t + 1) % 8])
            if i % 3 == 0:
                e.remove_user(k)

    th = [threading.Thread(target=work, args=(t,)) for t in range(4)]
    [x.start() for x in th]
    [x.join() for x in th]
    assert e.num_users() == (4 * 1000, 0)
    assert [len(e.debug_interested([t])) for t in range(5)] == [1000, 2000, 2000, 2000, 1000]
    for t in range(4):
        for i in (1, 2, 4, 1498):
            assert e.debug_route(bytes([t]) + i.to_bytes(4, "little"))[0] == 1
        assert e.debug_route(bytes([t]) + (3).to_bytes(4, "little")) == (0, -1)


def test_apply_user_sync_overlong_key_does_not_tear_the_merge(pcdn):
    """ADVICE r1: a peer's sync holding one key longer than max_key_len must not stop the merge half
    way.  VersionedMap::merge (versioned_map.rs:202-269) cannot fail and apply_user_sync always
    finishes with remove_user for every changed key (connections/mod.rs:157-161)."""
    e = pcdn.Engine(device=-1, max_conns=64, max_keys=256, max_key_len=16, identity="a/a")
    o = orc.Oracle("a/a")
    ec, oc = e.add_user(b"alice", [1, 2]), o.add_user(b"alice", [1, 2])
    long_key = b"L" * 40
    sync = [(b"alice", 5, "b/b"), (long_key, 3, "b/b"), (b"carol", 2, "b/b")]
    e.apply_user_sync("b/b", sync)   # no error: the over-long key simply has no device route
    o.apply_user_sync("b/b", sync)
    # alice moved to b/b: kicked locally (route REMOTE, no subscriptions, not a user any more)
    assert e.debug_route(b"alice")[0] == 2 and o.route(b"alice")[0] == 2
    assert e.debug_interested([1, 2]) == [] and o.interested([1, 2], False) == []
    assert e.num_users()[0] == 0 == o.num_users()
    assert e.debug_route(b"carol")[0] == 2
    # the CRDT map holds all three entries, exactly like the reference's
    got = sorted(e.get_user_sync(full=True))
    assert got == sorted([(b"alice", 5, "b/b"), (b"carol", 2, "b/b"), (long_key, 3, "b/b")])
    assert e.debug_route(long_key)[0] == 0   # never routable on the device (documented deviation 2)


def test_add_broker_reconnect_refused_before_anything_changes(pcdn):
    """ADVICE r1: add_broker with a full id space must refuse BEFORE dropping the existing broker."""
    e = pcdn.Engine(device=-1, max_conns=2, max_keys=64, identity="a/a")
    e.add_user(b"u0", [0])
    c = e.add_broker("b/b")
    e.subscribe_broker_to("b/b", [3])
    with pytest.raises(pcdn.PcdnError) as ei:
        e.add_broker("c/c")          # id space full: refused
    assert ei.value.code == -5
    assert e.debug_interested([3]) == [c] and e.num_users() == (1, 1)
    assert e.add_broker("b/b") == c  # a reconnect reuses its own id (no batch in flight)


def test_message_hook_seam_on_state_messages(pcdn):
    """MessageHookDef (cdn-proto/src/def.rs:79-92, called at cdn-broker/src/tasks/user/handler.rs:110-118):
    SkipMessage => the frame is ignored, Err => the receive loop ends, ProcessMessage => dispatch with
    whatever the hook changed in the parsed message.  Subscribe / Unsubscribe need no GPU."""
    import ctypes as C

    e = pcdn.Engine(device=-1, max_conns=64, max_keys=256, identity="a/a", n_valid_topics=8)
    c = e.add_user(b"alice", [])
    seen = []

    def hook(m):
        seen.append((m.kind, m.origin, C.string_at(m.sender, m.sender_len), [m.topics[i] for i in range(m.n_topics)]))
        if m.kind == pcdn.KIND_UNSUBSCRIBE:
            return pcdn.HOOK_SKIP
        if m.n_topics and m.topics[0] == 7:
            return -1                      # Err => disconnect
        if m.n_topics == 3:                # rewrite the parsed message: [1, 2, 3] -> [2, 5]
            m.topics[0], m.topics[1] = 2, 5
            m.n_topics = 2
        return pcdn.HOOK_PROCESS

    e.set_message_hook(0, hook)
    assert e.user_receive(b"alice", orc.serialize(pcdn.KIND_SUBSCRIBE, bytes([1, 2, 3]))) == 0
    assert e.debug_interested([2]) == [c] and e.debug_interested([5]) == [c] and e.debug_interested([1, 3]) == []
    assert e.user_receive(b"alice", orc.serialize(pcdn.KIND_UNSUBSCRIBE, bytes([2]))) == 0    # skipped
    assert e.debug_interested([2]) == [c]
    assert e.user_receive(b"alice", orc.serialize(pcdn.KIND_SUBSCRIBE, bytes([7]))) == -13    # PCDN_EHOOK
    assert e.debug_interested([7]) == []
    assert seen[0] == (pcdn.KIND_SUBSCRIBE, 0, b"alice", [1, 2, 3]) and len(seen) == 3
    e.set_message_hook(0, None)
    assert e.user_receive(b"alice", orc.serialize(pcdn.KIND_UNSUBSCRIBE, bytes([2]))) == 0    # hook removed: processed
    assert e.debug_interested([2]) == []


def test_config_validation_of_round2_fields(pcdn):
    """shard layout, ingest mode and output-pool size are checked before anything is allocated"""
    def bad(**kw):
        with pytest.raises(pcdn.PcdnError) as ei:
            pcdn.Engine(**dict(dict(device=-1, max_conns=64), **kw))
        assert ei.value.code == -1, kw

    bad(world_shards=2, first_shard=2)                       # first_shard + n_devices > world_shards
    bad(ingest=7)
    bad(flags=pcdn.FLAG_OUTPUT_POOL, pool_bytes=100)         # smaller than 4 KiB
    bad(flags=pcdn.FLAG_OUTPUT_POOL, pool_bytes=200 << 30)   # 2^32 units of 32 B = 128 GiB is the limit
    bad(max_conns=1 << 31, world_shards=4)                   # id space beyond 32 bits
    e = pcdn.Engine(device=-1, max_conns=64, flags=pcdn.FLAG_OUTPUT_POOL, world_shards=3, first_shard=1)
    assert e.num_shards() == (0, 3) and e.shard_info(0).conn_base == 8192
    with pytest.raises(pcdn.PcdnError) as ei:
        e.retry_batch(1)
    assert ei.value.code == -3                               # host-only engine: no data path


def test_pack_variant_takes_only_cta_counts(pcdn):
    """pack_variant holds the CTAs per SM of k_pack (bits 8-11) and k_pack_direct (bits 12-15); every other
    bit is refused with PCDN_EINVAL instead of being ignored"""
    for bit in [*range(8), *range(16, 32)]:
        with pytest.raises(pcdn.PcdnError) as ei:
            pcdn.Engine(device=-1, max_conns=64, pack_variant=1 << bit)
        assert ei.value.code == -1 and "CTA-count" in str(ei.value), bit
    for v in (0, 3 << 8, 8 << 12, 0xFF00):
        pcdn.Engine(device=-1, max_conns=64, pack_variant=v).close()
