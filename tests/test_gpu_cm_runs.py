"""The connection-major pack where a connection's records of one group of kCmGroup dense messages are NOT one
contiguous run: k_offsets then records where the run stops and writes scatter-list entries from there on, and
the pack follows the run start up to that position.  Every stream is compared with the oracle's, byte for
byte, on rings and the output pool, fused and regular control kernels, one shard and three."""
import pytest

from kconst import K
from oracle import oracle as orc
from test_gpu_parity import World, shard_cfg

pytestmark = pytest.mark.gpu

N_DENSE = 2048    # users on topic 0: at least N/16 of every shard's 8192 slots, so topic 0 is connection-major
RING = 1 << 14    # 15 records of a 1 KiB frame: the third batch of 8 wraps inside its group

MODES = [(out, ctrl, shards) for out in ("rings", "pool") for ctrl in ("fused", "regular") for shards in (1, 3)]
IDS = ["%s-%s-%dshard" % m for m in MODES]


def frame(topics, tag, size=1000):
    return orc.broadcast_frame(topics, bytes((tag * 7 + i) & 0xFF for i in range(size)))


def world(pcdn, out, ctrl, shards, **cfg):
    flags = (pcdn.FLAG_OUTPUT_POOL if out == "pool" else 0) | (pcdn.FLAG_STAGED_SPANS if ctrl == "regular" else 0)
    kw = dict(flags=flags, ring_bytes_per_conn=RING, pool_bytes=1 << 28, max_conns=8192)
    if shards > 1:
        kw.update(shard_cfg(pcdn, "shards-host"))
    kw.update(cfg)
    return World(pcdn, **kw)


@pytest.mark.parametrize("out,ctrl,shards", MODES, ids=IDS)
def test_groups_that_are_not_one_run(pcdn, out, ctrl, shards):
    w = world(pcdn, out, ctrl, shards)
    for i in range(N_DENSE):
        w.add_user(b"dense%05d" % i, [0])
    x = b"inter-leaved"
    w.add_user(x, [0, 1, 2])                   # topic 1: thin (x alone), topic 2: message-major (x + 63 others)
    for i in range(63):
        w.add_user(b"fat%05d" % i, [2])
    w.add_user(b"partial", [3])                # receives group messages 0, 2 and 5 only
    w.add_user(b"second-group", [4])           # receives nothing of the first group, all of the second
    assert 16 * (N_DENSE // shards) >= w.e.shard_info(0).shard_stride, "topic 0 must be connection-major on every shard"
    tag = 0

    def bcast(topics, size=1000):
        nonlocal tag
        tag += 1
        w.bcast(topics, frame(topics, tag, size))

    # a partial match: messages 0, 2 and 5 of a group
    for i in range(K.kCmGroup):
        bcast([0, 3] if i in (0, 2, 5) else [0])
    assert w.check() == K.kCmGroup * (N_DENSE + 1) + 3

    # a thin, a message-major and a direct record of x between connection-major messages of one group
    for i in range(K.kCmGroup):
        bcast([0])
        if i == 2:
            bcast([1], 300)
        if i == 4:
            bcast([2], 500)
        if i == 5:
            tag += 1
            w.direct(x, orc.direct_frame(x, bytes([tag]) * 200))
    assert w.check() > 0

    # a last group of fewer than kCmGroup messages; a connection that matches nothing of the first group
    for i in range(K.kCmGroup + 3):
        bcast([0, 4] if i >= K.kCmGroup else [0])
    assert w.check() > 0

    # rings of RING bytes: the batches of 8 records wrap inside a group (the pool has no wrap)
    for _ in range(3):
        for i in range(K.kCmGroup):
            bcast([0])
        assert w.check() > 0
    w.e.close()


@pytest.mark.parametrize("ctrl,shards", [(c, s) for c in ("fused", "regular") for s in (1, 3)],
                         ids=["%s-%dshard" % (c, s) for c in ("fused", "regular") for s in (1, 3)])
def test_overflow_inside_a_group(pcdn, ctrl, shards):
    """rings only (the pool refuses a batch as a whole instead): 20 records of 1 KiB into rings of 15 overflow in
    the second group; every connection gets a prefix of them, in order, and is reported"""
    w = world(pcdn, "rings", ctrl, shards)
    conns = [w.add_user(b"dense%05d" % i, [0]) for i in range(N_DENSE)]
    frames = [frame([0], t) for t in range(20)]
    for f in frames:
        w.e.handle_broadcast_message([0], f)
    w.e.flush()
    bid = w.e.next_batch()
    res = w.e.poll(bid)
    got = w.e.collect_frames(res)
    k = RING // ((4 + len(frames[0]) + K.kUnit - 1) // K.kUnit * K.kUnit)
    assert K.kCmGroup < k < 2 * K.kCmGroup
    assert res.n_overflow == N_DENSE and sorted(res.overflow_conns[i] for i in range(res.n_overflow)) == sorted(conns)
    for c in conns:
        assert got[c] == frames[:k]
    assert res.n_deliveries == k * N_DENSE
    w.e.release_batch(bid)
    w.e.close()
