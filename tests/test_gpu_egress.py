"""The span consumer (pcdn_egress_*, SURVEY 8f-2) against the oracle: what lands in host memory /
on the file descriptors must be exactly the byte stream the reference's writer task would put on
each connection's socket (u32 BE length + raw bytes per message, in order:
cdn-proto/src/connection/protocols/mod.rs:156-186,354-394), including after soft_close (:287-306)."""
import random

import pytest

import gpu_workloads as workloads
from gpu_world import World, chunk_streams, shard_cfg, wire

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mode", ["hbm", "hbm-small-chunks", "host-rings", "shards-host", "pool", "pool-runs-host"])
def test_drain_to_host_memory_matches_oracle(pcdn, mode):
    cfg = dict(max_conns=2048, ring_bytes_per_conn=1 << 18)
    if mode == "host-rings":
        cfg["flags"] = pcdn.FLAG_HOST_RINGS
    if mode == "pool":        # shared output pool: spans are unit offsets relative to the batch's region
        cfg.update(flags=pcdn.FLAG_OUTPUT_POOL, pool_bytes=512 << 20)
    if mode == "pool-runs-host":
        cfg.update(flags=pcdn.FLAG_OUTPUT_POOL | pcdn.FLAG_SPAN_RUNS | pcdn.FLAG_HOST_RINGS, pool_bytes=512 << 20)
    if mode == "shards-host":
        cfg.update(shard_cfg(pcdn, mode), max_conns=1024)
    w = World(pcdn, **cfg)
    # small chunks force many chunks per batch (and the 3-buffer rotation): 2 x ring is the minimum
    eg = pcdn.Egress(w.e, chunk_bytes=(1 << 19) if mode == "hbm-small-chunks" else 0)
    rng = random.Random(4)
    keys = [rng.getrandbits(64).to_bytes(8, "little") * 2 for _ in range(1200)]
    for k in keys:
        w.add_user(k, [x for x in range(4) if rng.random() < 0.4])
    want_total = {}
    for rnd in range(5):   # enough rounds to wrap the rings (two spans per connection)
        workloads.traffic(w, rng, keys, 40)
        b = w.e.flush()
        got = {}
        st = eg.drain(b, lambda ch: chunk_streams(ch, got))
        assert w.e.poll(b).n_overflow == 0
        w.e.release_batch(b)
        want = {c: wire(fr) for c, fr in w.expect().items()}
        assert {c: bytes(v) for c, v in got.items()} == want
        assert st.spans >= len(want) and st.chunks >= 1
        if mode == "hbm-small-chunks":
            assert st.chunks > 4
    eg.close()
    w.e.close()


@pytest.mark.parametrize("mode", ["hbm", "host-rings", "shards-host", "pool-runs"])
def test_writer_to_file_descriptors(pcdn, mode):
    """>= 1 K sinks: every attached connection's memfd must hold exactly the oracle's stream for that
    connection over several batches; connections without a descriptor are counted, not written."""
    workloads.writer_to_file_descriptors(pcdn, mode)


def test_sockets_backpressure_failure_and_soft_close(pcdn):
    """real sockets: a non-blocking stream socket with a tiny send buffer and a slow reader (partial
    writes, EAGAIN), a peer that went away (write error => reported, like the reference removing the
    user), and soft_close: frames handed to the engine but not even launched yet still go out."""
    workloads.sockets_backpressure_failure_and_soft_close(pcdn)
