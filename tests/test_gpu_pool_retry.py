"""The output pool's back-pressure path (PCDN_FLAG_OUTPUT_POOL): a batch that does not fit is refused
(status PCDN_EAGAIN), the host releases older batches and calls pcdn_retry_batch.  The refused batch
must come out as if it had fit at launch: routed against the tables as they were when it was launched
(R12), on every shard of a sharded engine, with its device-parse outcomes unchanged, and written by
the egress consumer exactly once.  Every stream is compared bit for bit with the oracle, which
processes the refused batch's messages before any later state change.

The refusal is arranged the same way everywhere: 4 MiB pools, and one hot connection that takes
3.8 MB of its shard's pool in an earlier batch that stays unreleased.  The next batch's share on that
shard (about 0.8 MB) no longer fits there; on the other shards it does."""
import pytest

import gpu_workloads as workloads
from gpu_world import HOT, STATUS_EAGAIN, PoolWorld
from oracle import oracle as orc

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("runs", [False, True], ids=["spans", "span-runs"])
@pytest.mark.parametrize("control", ["fused", "regular"])
@pytest.mark.parametrize("layout", ["one-shard", "shards-host"])
def test_retry_routes_as_launched(pcdn, layout, control, runs):
    """state changes between a refusal and its retry (subscribe a new user, unsubscribe, remove, the
    kick of a reconnect, a user moved to a peer broker, a broker subscription) reach only batches
    launched after them: the retried batch delivers what it would have delivered at launch, and a
    batch launched after the changes, while the pool is still blocked, sees the new tables.
    control = "regular": FLAG_STAGED_SPANS, so k_match / k_offsets / k_pool_finish run instead of the
    fused k_ctrl_small (with conn_base != 0 on the sharded engine)."""
    workloads.retry_routes_as_launched(pcdn, layout, control, runs)


def test_partial_refusal_across_shards(pcdn):
    """one shard refuses its share, the others accept theirs; users reconnect across shards in both
    directions before the retry.  Each direct message arrives exactly once, at the connection its key
    named at launch, and every stream equals the oracle's."""
    workloads.partial_refusal_across_shards(pcdn)


def _broken_direct(key):
    raw = bytearray(orc.direct_frame(key, b"x" * 64))
    raw[36:40] = (0xFFFFFFF).to_bytes(4, "little")            # recipient list beyond the segment
    return bytes(raw)


@pytest.mark.parametrize("layout", ["one-shard", "shards-host"])
def test_device_parse_retry_keeps_msg_status(pcdn, layout):
    """FLAG_DEVICE_PARSE: k_parse records each message's outcome and rewrites the descriptor of the
    ones it rejects.  After the retry msg_status and n_msg_errors, on every shard, are what the first
    poll said and what the oracle's receive loops return: a parse error stays -7, a prune error -8, a
    broker-origin broadcast with only invalid topics and a direct to a key longer than max_key_len stay
    0 (not routed, no error)."""
    w = PoolWorld(pcdn, layout, pcdn.FLAG_DEVICE_PARSE, n_valid_topics=4)
    sender = w.keys[0]
    frames = [(sender, 0, _broken_direct(w.keys[1])),
              (sender, 0, orc.broadcast_frame([9, 7], b"only invalid topics")),
              (sender, 1, orc.broadcast_frame([9, 7], b"only invalid topics, from a broker")),
              (sender, 0, orc.direct_frame(b"L" * 200, b"to a key longer than max_key_len"))]
    for t in (0, 1):
        for j in range(3):
            frames.append((sender, 0, orc.broadcast_frame([t], bytes([t, j]) * 1250)))
    for k in w.keys[2:8] + [HOT, b"nobody"]:
        frames.append((sender, 0, orc.direct_frame(k, b"direct to " + k)))
    b0 = w.fill_hot()
    want_rc = [w.o.broker_receive(raw) if origin else w.o.user_receive(s, raw) for s, origin, raw in frames]
    rcs = w.e.receive_frames(frames)
    b1 = w.e.flush()
    assert rcs == [0] * len(frames)
    assert want_rc[:4] == [-7, -8, 0, 0] and set(want_rc[4:]) == {0}
    results = lambda: [w.e.poll_shard(b1, li) for li in range(w.nl)] + [w.e.poll(b1)]
    first = [(r.status, [r.msg_status[i] for i in range(r.n_msgs)], r.n_msg_errors) for r in results()]
    assert first[-1][0] == STATUS_EAGAIN and first[w.home][0] == STATUS_EAGAIN
    for st, ms, ne in first:
        assert ms == want_rc and ne == 2
    got = {}
    w.consume(b0, got)
    w.e.retry_batch(b1)
    again = [(r.status, [r.msg_status[i] for i in range(r.n_msgs)], r.n_msg_errors) for r in results()]
    assert again == [(0, ms, ne) for _, ms, ne in first]
    w.consume(b1, got)
    w.compare(w.e, got, w.expect())
    w.e.close()


@pytest.mark.parametrize("how", ["drain", "write_batch", "soft_close"])
def test_egress_refused_shard_is_written_once(pcdn, how):
    """the egress consumer on a batch one shard refused: nothing of it reaches the sink (PCDN_EAGAIN)
    until it is retried, then every shard's share is written exactly once — through a Python sink,
    through write_batch to memfds, and inside soft_close, which releases, retries and writes by itself."""
    workloads.egress_refused_shard_is_written_once(pcdn, how)
