"""Per-connection backlogs of the egress writer (pcdn_egress_config.backlog_bytes_*): a peer that does
not read must not hold up the other connections or the release of the batch.  The reference gives
every connection its own writer task and unbounded queue (cdn-proto/src/connection/protocols/
mod.rs:150-186), so a slow peer only delays itself; here what a peer does not take is copied into its
backlog in host memory.  Every stream is compared byte for byte with the oracle's stream for that
connection (u32 BE length + raw bytes per message, in order), on rings, the output pool, host rings,
three shards and shared payload.  batch_slots=2 makes released slots (and their payload staging) get
reused while older bytes still wait in a backlog."""
import fcntl
import os
import random
import threading
import time

import pytest

import gpu_workloads as workloads
from gpu_world import BIG, PCDN_EINVAL, Reader, backlog_world, flush_until_done, payload, sock_pair, wire
from gpu_workloads import send_batches
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

# (layout, delivery) under this file's test ids
RINGS = pytest.param("rings", "copy", id="rings")
POOL = pytest.param("pool", "copy", id="pool")
HOST = pytest.param("host", "copy", id="host-rings")
SHARDS = pytest.param("shards-host", "copy", id="shards-host")
SHARED = pytest.param("rings", "shared", id="shared")
MODES = [RINGS, POOL, HOST, SHARDS, SHARED]


def shard_of(w, c):
    for li in range(w.e.num_shards()[0]):
        d = w.e.shard_info(li)
        if d.conn_base <= c < d.conn_base + d.shard_stride:
            return li
    raise AssertionError(c)


# ------------------------------------------------------------------ a stalled peer
@pytest.mark.parametrize("name,delivery", MODES)
def test_stalled_peer_does_not_stall_the_others(pcdn, name, delivery):
    """A (4 KiB send buffer, blocking socket) reads nothing; B and C are read by threads.  Six batches
    of 1 B - 40 KB broadcasts are written and released at once: every call returns, B and C hold
    their whole streams, A is not failed.  Then A's reader runs and flush_backlog completes A."""
    workloads.stalled_peer_does_not_stall_the_others(pcdn, name, delivery)


# ------------------------------------------------------------------ budgets
@pytest.mark.parametrize("name,delivery", [RINGS, POOL, SHARED])
def test_per_connection_budget(pcdn, name, delivery):
    """A's backlog would outgrow backlog_bytes_per_conn: A is reported exactly once and detached, it
    received a prefix of its stream, B and C are complete, the backlog total returns to 0"""
    w = backlog_world(pcdn, name, delivery)
    eg = pcdn.Egress(w.e, n_threads=4, backlog_bytes_per_conn=96 << 10)
    rng = random.Random(12)
    a, b, c = (w.add_user(k, [0]) for k in (b"alice", b"bob", b"carol"))
    sa, ra = sock_pair(4096)
    sb, rb = sock_pair()
    sc, rc_ = sock_pair()
    eg.attach(a, sa.fileno()); eg.attach(b, sb.fileno()); eg.attach(c, sc.fileno())
    reader_a = Reader(ra.fileno(), started=False)
    reader_b, reader_c = Reader(rb.fileno()), Reader(rc_.fileno())
    failed = []

    def between(_k, want):   # B and C catch up between batches: only A outgrows the budget
        failed.extend(eg.failed())
        reader_b.wait_for(len(want[b])); reader_c.wait_for(len(want[c]))

    want = send_batches(w, eg, rng, 6, between=between)
    assert failed == [a]
    assert eg.backlog() == ([], 0)
    assert reader_b.wait_for(len(want[b])) == bytes(want[b])
    assert reader_c.wait_for(len(want[c])) == bytes(want[c])
    reader_a.go()
    sa.close()
    got_a = reader_a.finish()
    assert len(got_a) < len(want[a]) and bytes(want[a]).startswith(got_a)
    assert eg.failed() == []
    sb.close(); sc.close()
    reader_b.finish(); reader_c.finish()
    ra.close(); rb.close(); rc_.close()
    eg.close()
    w.e.close()


@pytest.mark.parametrize("name,delivery", [RINGS, SHARDS])
def test_total_budget_two_stalled_peers(pcdn, name, delivery):
    """two stalled peers (on different shards with three shards) under backlog_bytes_total: first both
    backlog ~100 KB, then ~100 KB more for A1 alone — A1's own backlog stays under the budget, the two
    together cross it.  A1 is reported; A2 still receives its whole stream."""
    w = backlog_world(pcdn, name, delivery)
    budget = 260 << 10
    eg = pcdn.Egress(w.e, n_threads=4, backlog_bytes_total=budget)
    rng = random.Random(13)
    users = [w.add_user(b"user-%03d" % i, []) for i in range(12)]
    a1 = users[0]
    a2 = next(u for u in users[1:] if shard_of(w, u) != shard_of(w, a1)) if name == "shards-host" else users[1]
    w.both("subscribe_user_to", b"user-%03d" % users.index(a1), [0, 1])
    w.both("subscribe_user_to", b"user-%03d" % users.index(a2), [0])
    s1, r1 = sock_pair(4096)
    s2, r2 = sock_pair(4096)
    eg.attach(a1, s1.fileno()); eg.attach(a2, s2.fileno())
    reader1, reader2 = Reader(r1.fileno(), started=False), Reader(r2.fileno(), started=False)
    want = {}
    for topic in (0, 1):
        for _ in range(5):
            w.bcast([topic], orc.broadcast_frame([topic], payload(rng, 20000)))
        bid = w.e.flush()
        eg.write_batch(bid)
        w.e.release_batch(bid)
        for c, fr in w.expect().items():
            want.setdefault(c, bytearray()).extend(wire(fr))
        if topic == 0:
            pend, nbytes = eg.backlog()
            assert pend == sorted([a1, a2]) and 160 << 10 < nbytes < budget
            assert eg.failed() == []
    assert len(want[a1]) < budget
    assert eg.failed() == [a1] and eg.failed() == []
    assert eg.backlog()[0] == [a2]
    reader2.go()
    assert flush_until_done(eg) == 0
    assert reader2.wait_for(len(want[a2])) == bytes(want[a2])
    assert eg.backlog() == ([], 0)
    reader1.go()
    s1.close(); s2.close()
    got1 = reader1.finish()
    assert bytes(want[a1]).startswith(got1) and len(got1) < len(want[a1])
    reader2.finish()
    r1.close(); r2.close()
    eg.close()
    w.e.close()


# ------------------------------------------------------------------ order
@pytest.mark.parametrize("name,delivery", MODES)
def test_partly_drained_backlog_keeps_fifo(pcdn, name, delivery):
    """between batches the peer reads a little and flush_backlog(0) moves part of the backlog on; the
    next batch's records must still go behind what is left: one FIFO stream per connection"""
    w = backlog_world(pcdn, name, delivery)
    eg = pcdn.Egress(w.e, n_threads=4, backlog_bytes_per_conn=BIG)
    rng = random.Random(14)
    conns = [w.add_user(b"user-%03d" % i, [0]) for i in range(6)]
    a = conns[2]
    sa, ra = sock_pair(4096)
    eg.attach(a, sa.fileno())
    ra.setblocking(False)
    got = bytearray()
    partial = []

    def read_some(_k, _want):
        n = 0
        while n < 30000:                  # less than a batch: the backlog drains only partly
            try:
                d = ra.recv(4096)
                got.extend(d)
                n += len(d)
            except BlockingIOError:
                if not eg.backlog()[0]:
                    break
                eg.flush_backlog(0)       # the socket has room again: move part of the backlog on
        while True:                       # then leave the socket empty, the rest of the backlog waiting:
            try:                          # the next batch finds room, and its records must still queue
                got.extend(ra.recv(65536))
            except BlockingIOError:
                break
        partial.append(eg.backlog()[1])

    want = send_batches(w, eg, rng, 8, between=read_some)
    assert sum(1 for x in partial if x > 0) >= 6          # the backlog was still there when the next batch came
    ra.setblocking(True)
    reader = Reader(ra.fileno())
    assert flush_until_done(eg) == 0
    rest = reader.wait_for(len(want[a]) - len(got))
    assert bytes(got) + rest == bytes(want[a])
    assert eg.failed() == []
    sa.close()
    reader.finish()
    ra.close()
    eg.close()
    w.e.close()


# ------------------------------------------------------------------ lifecycle
@pytest.mark.parametrize("name,delivery", [RINGS, POOL, SHARED])
def test_soft_close_writes_the_backlog(pcdn, name, delivery):
    """a backlogged connection is soft-closed with its reader running: soft_close returns the fd once
    the whole stream (the backlog, then frames of the batch still open at the close) is written"""
    w = backlog_world(pcdn, name, delivery)
    eg = pcdn.Egress(w.e, n_threads=4, backlog_bytes_per_conn=BIG)
    rng = random.Random(15)
    ka = b"alice"
    a, b = w.add_user(ka, [0]), w.add_user(b"bob", [0])
    sa, ra = sock_pair(4096)
    sb, rb = sock_pair()
    eg.attach(a, sa.fileno()); eg.attach(b, sb.fileno())
    reader_a, reader_b = Reader(ra.fileno(), started=False), Reader(rb.fileno())
    want = send_batches(w, eg, rng, 4)
    assert eg.backlog()[0] == [a]
    for i in range(5):
        w.direct(ka, orc.direct_frame(ka, b"last words %d" % i))
        w.bcast([0], orc.broadcast_frame([0], payload(rng, 3000)))
    reader_a.go()
    assert eg.soft_close(a) == sa.fileno()
    for c, fr in w.expect().items():
        want[c].extend(wire(fr))
    assert eg.backlog() == ([], 0) and eg.failed() == []
    sa.close()
    assert reader_a.finish() == bytes(want[a])
    assert reader_b.wait_for(len(want[b])) == bytes(want[b])
    sb.close()
    reader_b.finish()
    ra.close(); rb.close()
    eg.close()
    w.e.close()


@pytest.mark.parametrize("name,delivery", [RINGS, SHARDS])
def test_detach_drops_the_backlog_and_a_reused_id_starts_clean(pcdn, name, delivery):
    """detach drops the connection's backlog at once (the total returns to 0, nothing is written to
    it later); after the id's quarantine a new user gets the same id on a new socket and receives
    only its own records"""
    w = backlog_world(pcdn, name, delivery)
    eg = pcdn.Egress(w.e, n_threads=4, backlog_bytes_per_conn=BIG)
    rng = random.Random(16)
    ka = b"alice"
    a, b = w.add_user(ka, [0]), w.add_user(b"bob", [0])
    sa, ra = sock_pair(4096)
    sb, rb = sock_pair()
    eg.attach(a, sa.fileno()); eg.attach(b, sb.fileno())
    reader_a, reader_b = Reader(ra.fileno(), started=False), Reader(rb.fileno())
    want = send_batches(w, eg, rng, 3)
    assert eg.backlog()[0] == [a]
    eg.detach(a)
    assert eg.backlog() == ([], 0)
    w.both("remove_user", ka)
    assert eg.flush_backlog(0) == 0 and eg.failed() == []
    reader_a.go()
    sa.close()
    old = reader_a.finish()
    assert bytes(want[a]).startswith(old) and len(old) < len(want[a])
    # every batch that named the old id is released: the id circulates again
    new = None
    for i in range(64):
        c = w.add_user(b"new-%02d" % i, [0])
        if c == a:
            new = b"new-%02d" % i
            break
    assert new is not None
    sn, rn = sock_pair(4096)
    eg.attach(a, sn.fileno())
    reader_n = Reader(rn.fileno())
    want2 = send_batches(w, eg, rng, 3)
    assert flush_until_done(eg) == 0
    assert reader_n.wait_for(len(want2[a])) == bytes(want2[a])
    want[b].extend(want2[b])
    assert reader_b.wait_for(len(want[b])) == bytes(want[b])
    assert eg.failed() == []
    sn.close(); sb.close()
    assert reader_n.finish() == bytes(want2[a])
    reader_b.finish()
    ra.close(); rb.close(); rn.close()
    eg.close()
    w.e.close()


# ------------------------------------------------------------------ other descriptors
@pytest.mark.parametrize("name,delivery", [RINGS, SHARED])
def test_non_blocking_pipe_takes_the_writev_path(pcdn, name, delivery):
    """a pipe is not a socket: the writer uses writev, and a non-blocking pipe of 4096 bytes answers
    EAGAIN; its backlog drains once the pipe is read"""
    w = backlog_world(pcdn, name, delivery)
    eg = pcdn.Egress(w.e, n_threads=4, backlog_bytes_per_conn=BIG)
    rng = random.Random(17)
    a, b = w.add_user(b"alice", [0]), w.add_user(b"bob", [0])
    pr, pw = os.pipe()
    fcntl.fcntl(pw, fcntl.F_SETPIPE_SZ, 4096)
    fcntl.fcntl(pw, fcntl.F_SETFL, fcntl.fcntl(pw, fcntl.F_GETFL) | os.O_NONBLOCK)
    eg.attach(a, pw)
    mb = os.memfd_create("bob")
    eg.attach(b, mb)
    reader = Reader(pr, started=False)
    want = send_batches(w, eg, rng, 4)
    pend, nbytes = eg.backlog()
    assert pend == [a] and nbytes >= len(want[a]) - 4096
    reader.go()
    assert flush_until_done(eg) == 0
    assert reader.wait_for(len(want[a])) == bytes(want[a])
    os.lseek(mb, 0, os.SEEK_SET)
    assert os.read(mb, len(want[b]) + 16) == bytes(want[b])
    assert eg.failed() == []
    os.close(pw)
    reader.finish()
    os.close(pr); os.close(mb)
    eg.close()
    w.e.close()


@pytest.mark.parametrize("name,delivery", [RINGS, SHARDS, SHARED])
def test_memfds_same_bytes_and_writes_with_and_without_backlog(pcdn, name, delivery):
    """a descriptor that always takes everything never backlogs: each batch written by an egress with
    a backlog and by one without gives the same fd_bytes, fd_writes and records, and the same files"""
    w = backlog_world(pcdn, name, delivery, batch_slots=4)
    plain = pcdn.Egress(w.e, n_threads=4)
    backlogged = pcdn.Egress(w.e, n_threads=4, backlog_bytes_per_conn=1 << 20, backlog_bytes_total=1 << 20)
    rng = random.Random(18)
    conns = [w.add_user(b"user-%03d" % i, [x for x in range(4) if rng.random() < 0.5]) for i in range(300)]
    fds = {}
    for eg in (plain, backlogged):
        fds[eg] = {c: os.memfd_create("c%d" % c) for c in conns[:250]}
        for c, fd in fds[eg].items():
            eg.attach(c, fd)
    for _ in range(4):
        for _ in range(20):
            t = [rng.randrange(4)]
            w.bcast(t, orc.broadcast_frame(t, payload(rng, rng.choice([0, 5, 1000, 20000]))))
        bid = w.e.flush()
        s1, s2 = plain.write_batch(bid), backlogged.write_batch(bid)
        w.e.release_batch(bid)
        assert (s1.fd_bytes, s1.fd_writes, s1.records) == (s2.fd_bytes, s2.fd_writes, s2.records)
        assert s1.fd_bytes > 0
        assert backlogged.backlog() == ([], 0)
    for c in conns[:250]:
        data = []
        for eg in (plain, backlogged):
            fd = fds[eg][c]
            os.lseek(fd, 0, os.SEEK_SET)
            data.append(os.read(fd, 1 << 24))
            os.close(fd)
        assert data[0] == data[1], c
    plain.close(); backlogged.close()
    w.e.close()


# ------------------------------------------------------------------ ABI
def test_old_config_size_means_no_backlog(pcdn):
    """an EgressConfig of the size before the backlog fields is accepted, and the writer behaves as
    it always did: it waits for the slow reader (nothing is backlogged even though the fields behind
    the old size are set), so write_batch returns with every byte in the socket; any other size is
    refused"""
    w = backlog_world(pcdn, "rings")
    eg = pcdn.Egress(w.e, n_threads=4, backlog_bytes_per_conn=1, backlog_bytes_total=1,
                     struct_size=pcdn.EGRESS_CONFIG_NO_BACKLOG_SIZE)
    rng = random.Random(19)
    a = w.add_user(b"alice", [0])
    sa, ra = sock_pair(4096)
    sa.setblocking(False)                  # EAGAIN: the writer polls and waits for the reader
    eg.attach(a, sa.fileno())
    got = bytearray()

    def slow_reader():
        while True:
            d = ra.recv(3000)
            if not d:
                return
            got.extend(d)
            time.sleep(0.0005)

    t = threading.Thread(target=slow_reader)
    t.start()
    want = send_batches(w, eg, rng, 3)
    assert eg.backlog() == ([], 0) and eg.flush_backlog(0) == 0 and eg.failed() == []
    sa.close()
    t.join(30)
    assert bytes(got) == bytes(want[a])
    ra.close()
    eg.close()
    with pytest.raises(pcdn.PcdnError) as ei:
        pcdn.Egress(w.e, struct_size=pcdn.EGRESS_CONFIG_NO_BACKLOG_SIZE + 8)
    assert ei.value.code == PCDN_EINVAL
    w.e.close()
