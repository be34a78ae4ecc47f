"""The kernels each class of batch launches, and the counters its result carries.

Per class, one batch is launched on a fresh engine whose table changes have already gone out with a warm-up
batch, and pcdn_stats.kernel_launches is read around it (the launch, or the retry, up to its poll; the release
is not counted).  The expected counts are the kernel sequences of engine.cu (batch_control, batch_pack):

  fused control ............ k_ctrl_small, k_pack (k_pack_ref on shared-payload engines; k_pack_ref after k_pack
                             when a message reaches ref_min_bytes)
  regular control .......... k_match, k_plan_a (+ k_plan_b, k_plan_c over 256 messages), k_offsets
                             (+ k_pool_finish on the output pool), k_pack
  device parse ............. k_parse ahead of either
  >= kThinSeparateMin directs  k_direct_lookup, k_dscan, k_dfill, k_dsort_hot, k_offsets, k_pack_direct
  pool retry ............... k_pool_retry_begin, then k_ctrl_small or k_offsets + k_pool_finish, then the pack

The memsets that zero the counters and the copies are not kernels.  Every batch's n_deliveries, bytes_out, n_spans,
n_overflow, n_direct_dropped and status must be what the oracle delivered for it, and every connection's frames
the oracle's."""
import pytest

from gpu_world import STATUS_EAGAIN, Sends, World, layout, user_sync
from kconst import K
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

N_USERS = 600
T_REF = 4096   # ref_min_bytes of the threshold classes

# per class: the kernel launches of one batch (the retry classes: its first launch, then the retry), and the
# engine's layout and delivery
LAUNCHES = {
    "fused-broadcast": (2, "rings", "copy"),
    "fused-direct": (2, "rings", "copy"),
    "regular-broadcast-one-block": (4, "staged", "copy"),
    "regular-broadcast-blocks": (6, "staged", "copy"),
    "device-parse-fused": (3, "devparse", "copy"),
    "device-parse-regular": (5, "devparse-staged", "copy"),
    "direct-only": (6, "rings", "copy"),
    "pool-fused": (2, "pool", "copy"),
    "pool-regular": (5, "pool-staged", "copy"),
    "pool-retry-fused": ((2, 3), "pool", "copy"),
    "pool-retry-regular": ((8, 4), "pool-staged", "copy"),
    "ref-below-threshold": (2, "rings", ("ref", T_REF)),
    "ref-at-threshold": (3, "rings", ("ref", T_REF)),
    "shared-payload": (2, "rings", "shared"),
    "targeted-fused": (2, "rings", "copy"),
    "targeted-regular": (4, "staged", "copy"),
}


class Seq(Sends, World):
    """users on topics 0 / 1 and one peer broker on topic 0; a warm-up batch takes the table changes to the device"""

    def __init__(self, pcdn, case):
        _, name, delivery = LAUNCHES[case]
        cfg = layout(pcdn, name)
        if case.startswith("pool-retry"):
            cfg.update(pool_bytes=4 << 20, batch_slots=4)
        elif name.startswith("pool"):
            cfg["pool_bytes"] = 64 << 20
        super().__init__(pcdn, max_conns=1024, delivery=delivery, **cfg)
        self.keys = [b"user-%04d" % i for i in range(N_USERS)]
        for i, k in enumerate(self.keys):
            self.add_user(k, [i % 2])
        self.add_broker("p/q", [0])
        self.bcast([0], b"warm-up")
        self.check()

    def launch(self):
        """flush the open batch, poll it: (its launches, its result, the oracle's frames for it)"""
        want = self.expect()
        n0 = self.e.stats().kernel_launches
        b = self.e.flush()
        res = self.e.poll(b)
        return self.e.stats().kernel_launches - n0, b, res, want

    def finish(self, b, res, want, drops=0):
        """the counters of a polled batch against the oracle's frames for it, then its frames; release it"""
        assert res.status == 0 and res.n_overflow == 0 and res.n_direct_dropped == drops
        assert res.n_deliveries == sum(len(f) for f in want.values())
        assert res.bytes_out == sum(4 + len(x) for f in want.values() for x in f)
        assert res.n_spans == len(want)   # one span per recipient: no ring wraps here
        self.e.last_result = res
        self.compare(self.e, self.e.collect_frames(res), want)
        self.e.release_batch(b)

    def batch(self, drops=0):
        n, b, res, want = self.launch()
        self.finish(b, res, want, drops)
        return n


def frame(j, n=300):
    return bytes([j & 0xFF]) * n


def broadcasts(w, n, size=300):
    for j in range(n):
        w.bcast([j % 2], frame(j, size))


def directs(w, n, size=200):
    for j in range(n):
        k = w.keys[(7 * j) % N_USERS]
        w.direct(k, frame(j, size))


@pytest.mark.parametrize("case", [c for c in LAUNCHES if not c.startswith("pool-retry")])
def test_launches_and_counters(pcdn, case):
    w = Seq(pcdn, case)
    drops = 0
    if case == "regular-broadcast-blocks":
        broadcasts(w, 300, 100)                      # 300 messages: three plan passes
    elif case.startswith("device-parse"):
        for j in range(12):
            raw = orc.broadcast_frame([j % 2], frame(j))
            assert w.e.user_receive(w.keys[j], raw) == 0 and w.o.user_receive(w.keys[j], raw) == 0
    elif case == "direct-only":
        directs(w, K.kThinSeparateMin)
    elif case.startswith("targeted"):
        broadcasts(w, 4)
        assert w.send(None, user_sync(1)) == 0
        assert w.send("p/q", user_sync(2)) == 0
    else:
        broadcasts(w, 12)
        if case in ("fused-direct", "shared-payload"):
            directs(w, 6)
            w.direct(b"nobody", b"dropped")
            drops = 1
        if case == "ref-below-threshold":
            w.bcast([1], frame(1, T_REF - 1))
        if case == "ref-at-threshold":
            w.bcast([1], frame(1, T_REF))
    assert w.batch(drops) == LAUNCHES[case][0], case
    w.e.close()


@pytest.mark.parametrize("control", ["fused", "regular"])
def test_pool_retry_launches_and_counters(pcdn, control):
    """a batch the output pool refuses launches its class's kernels; its retry launches k_pool_retry_begin and the
    passes that place and pack it, and then carries the counters of what it delivers"""
    case = "pool-retry-" + control
    w = Seq(pcdn, case)
    hot = w.keys[0]
    for j in range(38):                              # 3.8 MB of the 4 MiB pool, unreleased
        w.direct(hot, frame(j, 100_000))
    _, b0, r0, want0 = w.launch()
    broadcasts(w, 12)                                # 1.2 MB: fits the pool, not beside the first batch
    directs(w, 3)
    n1, b1, r1, want1 = w.launch()
    assert r1.status == STATUS_EAGAIN
    w.finish(b0, r0, want0)
    n0 = w.e.stats().kernel_launches
    w.e.retry_batch(b1)
    r1 = w.e.poll(b1)
    n_retry = w.e.stats().kernel_launches - n0
    w.finish(b1, r1, want1)
    assert (n1, n_retry) == LAUNCHES[case][0]
    w.e.close()
