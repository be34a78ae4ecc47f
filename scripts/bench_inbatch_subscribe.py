#!/usr/bin/env python
"""Receive windows with Subscribe / Unsubscribe frames, without and with PCDN_FLAG_INBATCH_SUBSCRIBE, on
GPU 0 in one process.

    python scripts/bench_inbatch_subscribe.py [--windows K] [--warmup W] [--out FILE]

2^16 users on 64 topics (1024 subscribers per topic).  A window is 4096 user frames: broadcasts of 64 B to
one topic, and 1 % of them (every 100th) a Subscribe or Unsubscribe of its sender.  Per window and engine:
pcdn_receive_frames until every frame is consumed (when the call stops early because every batch slot is
in flight, the outstanding batches are polled and released first), then pcdn_flush, poll and release of
what is left.  The two engines alternate window by window.  Reported per engine: batches per window
(deterministic), the median wall time of a window (host clock around work that ends in a blocking poll)
and the mean k_match time per window (CUDA events of the engine's stage timing).  The card's name, power
limit and SM clock limit are read in the same run.  Prints one JSON object; with --out also writes it.
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

N_USERS, N_TOPICS, WINDOW, SUB_EVERY, PAYLOAD = 1 << 16, 64, 4096, 100, 64


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=60)
    return q.stdout.strip()


def key(i):
    return b"u%07d" % i


def window_frames(w):
    """window w: the Subscribe frames of even windows are Unsubscribe frames in odd ones, so the
    subscription state returns to where it was every two windows"""
    out = []
    for j in range(WINDOW):
        u = (w * 7919 + j * 104729) % N_USERS
        if j % SUB_EVERY == SUB_EVERY - 1:
            kind = orc.KIND_SUBSCRIBE if w % 2 == 0 else orc.KIND_UNSUBSCRIBE
            raw = orc.serialize(kind, bytes([(u + 1) % N_TOPICS]))
        else:
            raw = orc.broadcast_frame([j % N_TOPICS], bytes([w & 255, j & 255]) * (PAYLOAD // 2))
        out.append((key(u), raw))
    return out


class Leg:
    def __init__(self, pcdn, flags):
        self.pcdn = pcdn
        self.e = pcdn.Engine(device=0, max_conns=N_USERS, max_topics=256, max_keys=2 * N_USERS, ring_bytes_per_conn=1 << 16,
                             max_batch_msgs=WINDOW, max_batch_bcast=WINDOW, max_batch_bytes=16 << 20,
                             max_batch_deliveries=WINDOW * (N_USERS // N_TOPICS) + (1 << 20), flags=flags)
        keys = b"".join(key(i) for i in range(N_USERS))
        kl = len(key(0))
        offs = (C.c_uint32 * (N_USERS + 1))(*range(N_USERS + 1))
        tops = (C.c_uint16 * N_USERS)(*[i % N_TOPICS for i in range(N_USERS)])
        out = (C.c_uint32 * N_USERS)()
        rc = self.e.L.pcdn_add_users_bulk(self.e.h, keys, kl, kl, N_USERS, tops, offs, out)
        assert rc == 0, rc
        self.e.set_timing(True)
        self.samples = []

    def release_all(self):
        while True:
            b = self.e.next_batch()
            if not b:
                return
            r = self.e.poll(b)
            assert r.status == 0 and r.n_overflow == 0, (r.status, r.n_overflow)
            self.e.release_batch(b)

    def run(self, arr, n, timed):
        e, L = self.e, self.e.L
        s0 = e.stats()
        rcs = (C.c_int32 * n)()
        t0 = time.perf_counter()
        pos = 0
        while pos < n:
            done = L.pcdn_receive_frames(e.h, C.cast(C.byref(arr, pos * C.sizeof(self.pcdn.Frame)), C.POINTER(self.pcdn.Frame)),
                                         n - pos, C.cast(C.byref(rcs, pos * 4), C.POINTER(C.c_int32)))
            assert done >= 0 or done == -11, done
            pos += max(done, 0)
            if pos < n:
                self.release_all()
        e.flush()
        self.release_all()
        dt = time.perf_counter() - t0
        s1 = e.stats()
        assert all(rcs[i] == 0 for i in range(n))
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
    legs = {"off": Leg(pcdn, 0), "on": Leg(pcdn, pcdn.FLAG_INBATCH_SUBSCRIBE)}
    wins = []
    for w in range(2):   # two windows alternate (subscribe / unsubscribe), prebuilt
        fr = window_frames(w)
        arr = (pcdn.Frame * WINDOW)()
        keep = []
        for i, (k, raw) in enumerate(fr):
            keep.append((k, raw))
            arr[i] = pcdn.Frame(k, len(k), 0, raw, len(raw), 0)
        wins.append((arr, keep))
    for w in range(a.warmup + a.windows):
        for name in (("off", "on") if w % 2 == 0 else ("on", "off")):
            legs[name].run(wins[w % 2][0], WINDOW, w >= a.warmup)
    res = {"card": card(), "users": N_USERS, "window_frames": WINDOW, "sub_frames_per_window": WINDOW // SUB_EVERY,
           "windows": a.windows}
    for name, leg in legs.items():
        s = leg.samples
        res[name] = {
            "batches_per_window": statistics.mean(x[1] for x in s),
            "window_ms_median": statistics.median(x[0] for x in s),
            "window_ms_min": min(x[0] for x in s),
            "match_ms_per_window": statistics.mean(x[2] for x in s),
            "deliveries_per_window": statistics.mean(x[3] for x in s),
        }
    assert res["on"]["deliveries_per_window"] == res["off"]["deliveries_per_window"]
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
