"""Several connection shards behind ONE engine (pcdn_config.devices, SURVEY 8e), through the C ABI,
against ONE unsharded oracle, stream for stream.  'shards-host' puts the shards on GPU 0 (runs on a
one-GPU box); 'shards-nccl' uses one GPU per shard and the library's own ncclBroadcast ingest (needs
>= 2 GPUs).  The randomized mixed workload on sharded engines lives in
test_gpu_parity.py::test_random_mixed_batches[shards-*]."""
import random

import pytest

import gpu_workloads as workloads
import scenarios
from gpu_world import World, payload, shard_cfg
from harness import EngineBackend
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

VARIANTS = ["shards-host", "shards-nccl"]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("scenario", scenarios.ALL, ids=lambda f: f.__name__)
def test_reference_scenario_sharded(pcdn, scenario, variant):
    """the reference's own broker tests (cdn-broker/src/tests/{broadcast,direct}.rs) on a sharded engine"""
    scenario(EngineBackend(pcdn, **shard_cfg(pcdn, variant)))


@pytest.mark.parametrize("variant", VARIANTS)
def test_shards_balance_counters_and_per_shard_results(pcdn, variant):
    """connections go to the least-loaded shard; every span of a shard's result names a connection of
    that shard; the per-shard results add up to pcdn_poll's; an unroutable direct is counted once."""
    w = World(pcdn, max_conns=512, ring_bytes_per_conn=1 << 16, **shard_cfg(pcdn, variant))
    nl, nw = w.e.num_shards()
    assert nl == nw >= 2
    rng = random.Random(11)
    keys = [rng.getrandbits(64).to_bytes(8, "little") * 4 for _ in range(600)]
    for i, k in enumerate(keys):
        w.add_user(k, [0] if i % 2 == 0 else [1])
    w.add_broker("p/p", [0])
    w.both("apply_user_sync", "p/p", [(b"far-away", 1, "p/p")])
    descs = [w.e.shard_info(i) for i in range(nl)]
    loads = [d.n_conns for d in descs]
    assert sum(loads) == 601 and max(loads) - min(loads) <= 1, loads
    for d in descs[1:]:
        assert d.conn_base == d.global_index * d.shard_stride
    if variant == "shards-nccl":
        assert all(d.nccl_ranks == nw for d in descs), [d.nccl_ranks for d in descs]
        assert len({d.device for d in descs}) == nl
    msgs = [("b", [0], orc.broadcast_frame([0], payload(rng, 300)), False),
            ("d", keys[5], orc.direct_frame(keys[5], b"x" * 70), False),
            ("d", b"nobody", orc.direct_frame(b"nobody", b"y" * 10), False),
            ("d", b"far-away", orc.direct_frame(b"far-away", b"z" * 33), False),
            ("d", b"far-away", orc.direct_frame(b"far-away", b"z" * 33), True),     # to_user_only: not forwarded
            ("b", [1, 0], orc.broadcast_frame([1, 0], payload(rng, 2000)), True)]
    for m in msgs:
        if m[0] == "b":
            w.o.handle_broadcast_message(m[1], m[2], m[3])
        else:
            w.o.handle_direct_message(m[1], m[2], m[3])
    b = w.e.submit(msgs)
    tot = w.e.poll(b)
    per = [w.e.poll_shard(b, i) for i in range(nl)]
    assert tot.n_deliveries == sum(r.n_deliveries for r in per) == w.o.deliveries()
    assert tot.bytes_out == sum(r.bytes_out for r in per)
    assert tot.n_spans == sum(r.n_spans for r in per)
    assert tot.n_direct_dropped == 2 == sum(r.n_direct_dropped for r in per)  # "nobody" + the to_user_only remote
    for d, r in zip(descs, per):
        for i in range(r.n_spans):
            assert d.conn_base <= r.spans[i].conn < d.conn_base + d.shard_stride
    got = w.e.collect_frames(tot)
    w.e.release_batch(b)
    want = w.expect()
    assert got == want
    w.e.close()


@pytest.mark.parametrize("variant", VARIANTS)
def test_sharded_device_resident_batch(pcdn, variant):
    """pcdn_submit_device on a sharded engine: the batch lies on the root GPU (global shard 0) and the
    library replicates frames + descriptors to the other shards (NCCL broadcast / peer copies)."""
    workloads.sharded_device_resident_batch(pcdn, variant)


@pytest.mark.parametrize("variant", VARIANTS)
def test_sharded_user_moves_and_reconnects(pcdn, variant):
    """a user kicked by a same-key connect lands on another shard; a user-sync moves a local user to a
    peer broker; both keep exactly the oracle's streams (R12 ordering across the shards)."""
    w = World(pcdn, max_conns=256, ring_bytes_per_conn=1 << 16, **shard_cfg(pcdn, variant))
    rng = random.Random(9)
    keys = [b"user-%03d" % i for i in range(90)]
    for k in keys:
        w.add_user(k, [0, 1])
    w.add_broker("q/q", [1])
    for rnd in range(4):
        for j in range(30):
            k = rng.choice(keys)
            if rng.random() < 0.5:
                w.direct(k, orc.direct_frame(k, payload(rng, 64 + j)))
            else:
                w.bcast([rng.randrange(2)], orc.broadcast_frame([0], payload(rng, 200)))
        w.check()
        for k in rng.sample(keys, 10):      # reconnect: same key, new connection (maybe another shard)
            w.add_user(k, [1])
        moved = rng.sample(keys, 5)         # these users are now connected to q/q
        w.both("apply_user_sync", "q/q", [(k, 10 + rnd, "q/q") for k in moved])
    w.check()
    w.e.close()
