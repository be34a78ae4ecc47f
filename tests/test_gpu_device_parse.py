"""Device-side ingress parse (SURVEY 8f-1, PCDN_FLAG_DEVICE_PARSE): the host only peeks the union tag
and copies raw frames; k_parse walks the Cap'n Proto message, applies Topic::prune and extracts the
recipient on the GPU.  Outputs must equal the oracle's user_receive_loop / broker_receive_loop
(cdn-broker/src/tasks/user/handler.rs:104-161, tasks/broker/handler.rs:130-192) frame for frame;
malformed / all-invalid-topic frames are not routed and come back in msg_status."""
import random

import pytest

import gpu_workloads as workloads
import scenarios
from gpu_world import World
from harness import EngineBackend
from oracle import oracle as orc

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("scenario", scenarios.ALL, ids=lambda f: f.__name__)
def test_reference_scenario_device_parse(pcdn, scenario):
    scenario(EngineBackend(pcdn, flags=pcdn.FLAG_DEVICE_PARSE))


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_frames_through_receive_loops(pcdn, seed):
    workloads.frames_through_receive_loops(pcdn, seed)


@pytest.mark.parametrize("staged", [False, True])
def test_msg_status_codes(pcdn, staged):
    workloads.msg_status_codes(pcdn, staged)


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
            raw = workloads._mutate(rng, orc.direct_frame(rng.choice(keys), b"zzzz" * 20))
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
