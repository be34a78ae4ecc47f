#!/usr/bin/env python
"""Receive windows with the broker's partial syncs sent through pcdn_send_to_brokers, against the same
windows without them and against the way a host had to send them before (after draining the pipeline), on
GPU 0 in one process.

    python scripts/bench_send_to_brokers.py [--windows K] [--warmup W] [--out FILE]

2^16 users on 64 topics (1024 subscribers per topic) and 64 peer brokers (broker i subscribed to topic i).
A window is 4096 user broadcast frames of 64 B through pcdn_receive_frames; in the middle of it the host
sends one 64 KiB partial user sync and one 1 KiB partial topic sync to every broker (run_sync_task,
cdn-broker/src/tasks/broker/sync.rs:129-143).  Three engines, alternating window by window:
  plain    the frames only;
  sends    the two sync frames through pcdn_send_to_brokers at their place in the open batch;
  drained  the two sync frames written by the host itself after every batch launched so far was polled and
           released (pcdn_flush, poll, release), then the rest of the window: what a host without the call
           does so that its write cannot interleave with the egress writer's.
Per window: pcdn_flush, poll and release of what is left.  Reported per engine: batches per window, the
median and minimum wall time of a window (host clock around work that ends in a blocking poll) and the mean
k_match time per window (CUDA events of the engine's stage timing).  The card's name, power limit and SM
clock limit are read in the same run.  Prints one JSON object; with --out also writes it.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import __graft_entry__ as ge  # noqa: E402
from oracle import oracle as orc  # noqa: E402

N_USERS, N_TOPICS, N_BROKERS, WINDOW, PAYLOAD = 1 << 16, 64, 64, 4096, 64
USER_SYNC = orc.serialize(orc.KIND_USER_SYNC, b"", b"u" * (64 << 10))
TOPIC_SYNC = orc.serialize(orc.KIND_TOPIC_SYNC, b"", b"t" * (1 << 10))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=60)
    return q.stdout.strip()


def key(i):
    return b"u%07d" % i


class Leg:
    def __init__(self, pcdn, mode):
        self.pcdn, self.mode = pcdn, mode
        self.e = pcdn.Engine(device=0, max_conns=N_USERS + 2 * N_BROKERS, max_topics=256, max_keys=2 * N_USERS,
                             ring_bytes_per_conn=1 << 17, max_batch_msgs=WINDOW + 2, max_batch_bcast=WINDOW + 2,
                             max_batch_bytes=16 << 20, max_batch_deliveries=WINDOW * (N_USERS // N_TOPICS + 1) + (1 << 20))
        keys = b"".join(key(i) for i in range(N_USERS))
        kl = len(key(0))
        offs = (C.c_uint32 * (N_USERS + 1))(*range(N_USERS + 1))
        tops = (C.c_uint16 * N_USERS)(*[i % N_TOPICS for i in range(N_USERS)])
        out = (C.c_uint32 * N_USERS)()
        rc = self.e.L.pcdn_add_users_bulk(self.e.h, keys, kl, kl, N_USERS, tops, offs, out)
        assert rc == 0, rc
        for b in range(N_BROKERS):
            self.e.add_broker("b%02d/x" % b)
            self.e.subscribe_broker_to("b%02d/x" % b, [b % N_TOPICS])
        self.e.set_timing(True)
        self.written = {b: bytearray() for b in range(N_BROKERS)}   # the drained leg's own writes
        self.samples = []

    def release_all(self):
        while True:
            b = self.e.next_batch()
            if not b:
                return
            r = self.e.poll(b)
            assert r.status == 0 and r.n_overflow == 0, (r.status, r.n_overflow)
            self.e.release_batch(b)

    def receive(self, arr, lo, hi, rcs):
        L, e = self.e.L, self.e
        pos = lo
        while pos < hi:
            done = L.pcdn_receive_frames(e.h, C.cast(C.byref(arr, pos * C.sizeof(self.pcdn.Frame)), C.POINTER(self.pcdn.Frame)),
                                         hi - pos, C.cast(C.byref(rcs, pos * 4), C.POINTER(C.c_int32)))
            assert done >= 0 or done == -11, done
            pos += max(done, 0)
            if pos < hi:
                self.release_all()

    def run(self, arr, timed):
        e = self.e
        s0 = e.stats()
        rcs = (C.c_int32 * WINDOW)()
        t0 = time.perf_counter()
        self.receive(arr, 0, WINDOW // 2, rcs)
        if self.mode == "sends":
            assert e.send_to_brokers(USER_SYNC) == 0 and e.send_to_brokers(TOPIC_SYNC) == 0
        elif self.mode == "drained":
            e.flush()
            self.release_all()
            for b in range(N_BROKERS):
                for raw in (USER_SYNC, TOPIC_SYNC):
                    self.written[b] += len(raw).to_bytes(4, "big") + raw
                self.written[b].clear()
        self.receive(arr, WINDOW // 2, WINDOW, rcs)
        e.flush()
        self.release_all()
        dt = time.perf_counter() - t0
        s1 = e.stats()
        assert all(rcs[i] == 0 for i in range(WINDOW))
        if timed:
            self.samples.append((dt * 1e3, s1.batches - s0.batches, s1.ms_match - s0.ms_match, s1.deliveries - s0.deliveries))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--out")
    a = ap.parse_args()
    pcdn = ge.load_package()
    pcdn.build()
    names = ("plain", "sends", "drained")
    legs = {n: Leg(pcdn, n) for n in names}
    arr = (pcdn.Frame * WINDOW)()
    keep = []
    for j in range(WINDOW):
        k = key((j * 104729) % N_USERS)
        raw = orc.broadcast_frame([j % N_TOPICS], bytes([j & 255]) * PAYLOAD)
        keep.append((k, raw))
        arr[j] = pcdn.Frame(k, len(k), 0, raw, len(raw), 0)
    for w in range(a.warmup + a.windows):
        order = names[w % 3:] + names[:w % 3]
        for n in order:
            legs[n].run(arr, w >= a.warmup)
    res = {"card": card(), "users": N_USERS, "brokers": N_BROKERS, "window_frames": WINDOW,
           "sync_bytes": [len(USER_SYNC), len(TOPIC_SYNC)], "windows": a.windows}
    for n, leg in legs.items():
        s = leg.samples
        res[n] = {
            "batches_per_window": statistics.mean(x[1] for x in s),
            "window_ms_median": statistics.median(x[0] for x in s),
            "window_ms_min": min(x[0] for x in s),
            "match_ms_per_window": statistics.mean(x[2] for x in s),
            "deliveries_per_window": statistics.mean(x[3] for x in s),
        }
    assert res["sends"]["deliveries_per_window"] == res["plain"]["deliveries_per_window"] + 2 * N_BROKERS
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
