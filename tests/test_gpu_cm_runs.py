"""The connection-major pack where a connection's records of one group of kCmGroup dense messages are NOT one
contiguous run: k_offsets then records where the run stops and writes scatter-list entries from there on, and
the pack follows the run start up to that position.  Every stream is compared with the oracle's, byte for
byte, on rings and the output pool, fused and regular control kernels, one shard and three."""
import pytest

import gpu_workloads as workloads
from gpu_world import CM_DENSE, CM_IDS, CM_MODES, CM_RING, cm_frame, cm_world
from kconst import K

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", CM_MODES, ids=CM_IDS)
def test_groups_that_are_not_one_run(pcdn, name):
    workloads.groups_that_are_not_one_run(pcdn, name)


@pytest.mark.parametrize("name", CM_MODES[:4], ids=[i.removeprefix("rings-") for i in CM_IDS[:4]])
def test_overflow_inside_a_group(pcdn, name):
    """rings only (the pool refuses a batch as a whole instead): 20 records of 1 KiB into rings of 15 overflow in
    the second group; every connection gets a prefix of them, in order, and is reported"""
    w = cm_world(pcdn, name)
    conns = [w.add_user(b"dense%05d" % i, [0]) for i in range(CM_DENSE)]
    frames = [cm_frame([0], t) for t in range(20)]
    for f in frames:
        w.e.handle_broadcast_message([0], f)
    w.e.flush()
    bid = w.e.next_batch()
    res = w.e.poll(bid)
    got = w.e.collect_frames(res)
    k = CM_RING // ((4 + len(frames[0]) + K.kUnit - 1) // K.kUnit * K.kUnit)
    assert K.kCmGroup < k < 2 * K.kCmGroup
    assert res.n_overflow == CM_DENSE and sorted(res.overflow_conns[i] for i in range(res.n_overflow)) == sorted(conns)
    for c in conns:
        assert got[c] == frames[:k]
    assert res.n_deliveries == k * CM_DENSE
    w.e.release_batch(bid)
    w.e.close()
