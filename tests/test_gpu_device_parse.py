"""Device-side ingress parse (SURVEY 8f-1, PCDN_FLAG_DEVICE_PARSE): the host only peeks the union tag
and copies raw frames; k_parse walks the Cap'n Proto message, applies Topic::prune and extracts the
recipient on the GPU.  Outputs must equal the oracle's user_receive_loop / broker_receive_loop
(cdn-broker/src/tasks/user/handler.rs:104-161, tasks/broker/handler.rs:130-192) frame for frame;
malformed / all-invalid-topic frames are not routed and come back in msg_status."""
import random

import pytest

import scenarios
from harness import EngineBackend
from oracle import oracle as orc
from test_gpu_parity import World

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("scenario", scenarios.ALL, ids=lambda f: f.__name__)
def test_reference_scenario_device_parse(pcdn, scenario):
    scenario(EngineBackend(pcdn, flags=pcdn.FLAG_DEVICE_PARSE))


def _mutate(rng, raw):
    raw = bytearray(raw)
    for _ in range(rng.randrange(1, 3)):
        raw[rng.randrange(8, min(len(raw), 56))] = rng.randrange(256)
    return bytes(raw)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_frames_through_receive_loops(pcdn, seed):
    rng = random.Random(seed)
    # seed 2 also forces the large-engine span path (span table staged in HBM, copied out during the pack)
    w = World(pcdn, n_valid_topics=12, flags=pcdn.FLAG_DEVICE_PARSE | (pcdn.FLAG_STAGED_SPANS if seed == 2 else 0),
              ring_bytes_per_conn=1 << 20)
    keys = []
    for i in range(1200):
        k = rng.getrandbits(64).to_bytes(8, "little") * rng.choice([1, 4, 16])
        keys.append(k)
        w.add_user(k, [x for x in range(12) if rng.random() < (0.5 if x == 0 else 0.08)])
    w.add_broker("b0/p0", [0, 3])
    w.both("apply_user_sync", "b0/p0", [(b"far-away", 1, "b0/p0")])
    total_err = 0
    for batch in range(3):
        frames, want_rc = [], []
        for j in range(rng.randrange(60, 160)):
            size = rng.choice([0, 5, 100, 1000, 9000, 20000]) if rng.random() < 0.4 else rng.randrange(0, 2000)
            pl = bytes([j & 0xFF]) * size
            r = rng.random()
            if r < 0.5:
                topics = [rng.randrange(16) for _ in range(rng.randrange(1, 5))]      # 12..15 are invalid
                if rng.random() < 0.3:
                    topics = [topics[0]] * 2 + topics                                    # consecutive duplicates
                raw = orc.broadcast_frame(topics, pl)
            elif r < 0.9:
                rc = rng.choice(keys) if rng.random() < 0.8 else rng.choice([b"far-away", b"nobody", b""])
                raw = orc.direct_frame(rc, pl)
            else:
                raw = orc.broadcast_frame([rng.randrange(12, 200)] * rng.randrange(1, 3), pl)  # only invalid topics
            if rng.random() < 0.15:
                raw = _mutate(rng, raw)
            origin = 1 if rng.random() < 0.25 else 0
            sender = rng.choice(keys)
            frames.append((sender, origin, raw))
            want_rc.append(w.o.broker_receive(raw) if origin else w.o.user_receive(sender, raw))
        # mutated frames may decode as Subscribe/Unsubscribe: those change state on both sides alike
        rcs = w.e.receive_frames(frames)
        got = w.e.drain()
        res = w.e.last_result
        # per-frame outcome: synchronous code, or (device-parsed kinds) the batch's msg_status
        deferred = [i for i, (rc, wrc) in enumerate(zip(rcs, want_rc)) if rc != wrc]
        n_err_want = sum(1 for i in deferred if want_rc[i] < 0)
        assert all(rcs[i] == 0 and want_rc[i] in (-7, -8) for i in deferred), [(rcs[i], want_rc[i]) for i in deferred][:5]
        assert res.n_msg_errors == n_err_want
        total_err += n_err_want
        want = w.expect()
        assert set(got) == set(want)
        for c in want:
            assert got[c] == want[c], c
    assert total_err > 5


@pytest.mark.parametrize("staged", [False, True])
def test_msg_status_codes(pcdn, staged):
    w = World(pcdn, n_valid_topics=2, flags=pcdn.FLAG_DEVICE_PARSE | (pcdn.FLAG_STAGED_SPANS if staged else 0))
    a = w.add_user(b"a" * 8, [0, 1])
    good = orc.broadcast_frame([0], b"ok")
    bad_topics = orc.broadcast_frame([9, 9, 7], b"nope")
    broken = bytearray(orc.direct_frame(b"a" * 8, b"x" * 64)); broken[36:40] = (0xFFFFFFF).to_bytes(4, "little")  # recipient list beyond the segment
    rcs = w.e.receive_frames([(b"a" * 8, 0, good), (b"a" * 8, 0, bad_topics), (b"a" * 8, 0, bytes(broken)),
                              (b"a" * 8, 1, bad_topics)])
    assert rcs == [0, 0, 0, 0]
    got = w.e.drain()
    res = w.e.last_result
    st = [res.msg_status[i] for i in range(res.n_msgs)]
    assert st == [0, -8, -7, 0]            # broker-origin topics are not pruned (handler.rs:157): no error, no recipients
    assert res.n_msg_errors == 2 and got[a] == [good]


@pytest.mark.parametrize("flags", [0, 1], ids=["host-parse", "device-parse"])
def test_large_call_takes_the_threaded_path(pcdn, flags):
    """>= 2048 frames in one pcdn_receive_frames call: parallel parse/peek + parallel copy, with
    Subscribe/Unsubscribe frames (state changes that launch the open batch), malformed frames and batch
    capacity boundaries in the middle — order and outcomes must equal the one-at-a-time oracle"""
    rng = random.Random(99)
    w = World(pcdn, n_valid_topics=10, flags=flags, ring_bytes_per_conn=1 << 20, max_batch_msgs=1500, max_batch_bcast=512,
              batch_slots=8)
    keys = [rng.getrandbits(64).to_bytes(8, "little") * 4 for _ in range(800)]
    for k in keys:
        w.add_user(k, [x for x in range(10) if rng.random() < 0.15])
    frames, want_rc = [], []
    for j in range(7000):
        r = rng.random()
        sender = rng.choice(keys)
        origin = 0
        if r < 0.45:
            raw = orc.broadcast_frame([rng.randrange(12) for _ in range(rng.randrange(1, 3))], bytes([j & 255]) * rng.randrange(0, 300))
            origin = 1 if rng.random() < 0.2 else 0
        elif r < 0.9:
            raw = orc.direct_frame(rng.choice(keys), bytes([j & 255]) * rng.randrange(0, 300))
        elif r < 0.95:
            raw = orc.serialize(rng.choice([orc.KIND_SUBSCRIBE, orc.KIND_UNSUBSCRIBE]), bytes([rng.randrange(10)]))
        elif r < 0.975:
            raw = _mutate(rng, orc.direct_frame(rng.choice(keys), b"zzzz" * 20))
        else:
            raw = orc.broadcast_frame([77], b"only invalid topics")
        frames.append((sender, origin, raw))
        want_rc.append(w.o.broker_receive(raw) if origin else w.o.user_receive(sender, raw))
    rcs, got = w.e.receive_frames_all(frames)   # drains and resumes whenever all batch slots are in flight
    want = w.expect()
    assert set(got) == set(want)
    for c in want:
        assert got[c] == want[c], c
    if flags == 0:
        assert rcs == want_rc
    else:
        assert all(a == b or (a == 0 and b in (-7, -8)) for a, b in zip(rcs, want_rc))
