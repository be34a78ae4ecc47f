#!/usr/bin/env python
"""The fd writer (pcdn_egress_write_batch) to 1000 socketpairs, without and with per-connection
backlogs (pcdn_egress_config.backlog_bytes_*), on GPU 0 in one process.

    python scripts/bench_egress_backlog.py [--steps K] [--stall-steps S] [--no-wait-leg] [--out FILE]

Two legs; the card's name and power limit are read in the same run and printed with the numbers.
  fast    every peer is read by reader threads (epoll): write_batch time per batch, alternating an
          egress without backlogs and one with them, batch by batch — the cost of the backlog on the
          path where no peer is slow.
  stalled the same, with one peer that never reads (4 KiB send buffer).  Without backlogs the writer
          waits the 30 s bound on that peer's non-blocking socket, then reports it (one batch, timed;
          --no-wait-leg skips it).  With backlogs: the time per batch and the backlog after each batch.
Each batch is 8 broadcasts of 1 KiB to all 1000 connections (8.3 MB on the sockets), host-submitted.
Prints one JSON object; with --out also writes it there.
"""
import argparse
import json
import os
import random
import resource
import selectors
import socket
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import __graft_entry__ as ge  # noqa: E402
from oracle import oracle as orc  # noqa: E402

N_CONNS, MSGS, PAYLOAD = 1000, 8, 1024


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=60)
    return q.stdout.strip()


class Readers:
    """reader threads that drain every socket handed to them (epoll) and count the bytes"""

    def __init__(self, socks, n_threads=8):
        self.stop = False
        self.bytes = [0] * n_threads
        self.th = []
        for t in range(n_threads):
            sel = selectors.EpollSelector()
            for s in socks[t::n_threads]:
                s.setblocking(False)
                sel.register(s, selectors.EVENT_READ)
            self.th.append(threading.Thread(target=self._run, args=(t, sel), daemon=True))
        for th in self.th:
            th.start()

    def _run(self, t, sel):
        while not self.stop:
            for key, _ in sel.select(0.05):
                try:
                    while True:
                        d = key.fileobj.recv(1 << 20)
                        if not d:
                            break
                        self.bytes[t] += len(d)
                except BlockingIOError:
                    pass
        sel.close()

    def total(self):
        return sum(self.bytes)

    def close(self):
        self.stop = True
        for th in self.th:
            th.join()


def batch(e, rng):
    for _ in range(MSGS):
        e.handle_broadcast_message([0], orc.broadcast_frame([0], bytes([rng.randrange(256)]) * PAYLOAD))
    return e.flush()


def timed_write(e, eg, rng):
    b = batch(e, rng)
    t0 = time.perf_counter()
    st = eg.write_batch(b)
    dt = time.perf_counter() - t0
    e.release_batch(b)
    return dt, st


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=40, help="timed batches per writer in the fast leg")
    ap.add_argument("--stall-steps", type=int, default=40)
    ap.add_argument("--no-wait-leg", action="store_true")
    ap.add_argument("--out")
    args = ap.parse_args()
    soft, hard = resource.getrlimit(resource.RLIMIT_NOFILE)
    if soft < 4 * N_CONNS + 256:   # this process's own descriptor limit: 2 per socketpair
        resource.setrlimit(resource.RLIMIT_NOFILE, (min(hard, 4 * N_CONNS + 256), hard))
    pkg = ge.load_package()
    e = pkg.Engine(device=0, max_conns=2048, max_topics=16, max_keys=4096, ring_bytes_per_conn=1 << 16,
                   max_batch_msgs=64, max_batch_bytes=1 << 20)
    conns = [e.add_user(b"user-%05d" % i, [0]) for i in range(N_CONNS)]
    pairs = [socket.socketpair() for _ in conns]
    plain = pkg.Egress(e)
    backlog = pkg.Egress(e, backlog_bytes_per_conn=64 << 20, backlog_bytes_total=1 << 30)
    for c, (s, _) in zip(conns, pairs):
        plain.attach(c, s.fileno())
        backlog.attach(c, s.fileno())
    rd = Readers([r for _, r in pairs])
    rng = random.Random(1)
    out = {"card": card(), "conns": N_CONNS, "batch": "%d x %d B broadcasts to every connection" % (MSGS, PAYLOAD)}

    # ---- fast: alternate the two writers batch by batch
    for _ in range(5):
        timed_write(e, plain, rng); timed_write(e, backlog, rng)
    times = {"off": [], "on": []}
    fd_bytes = 0
    for _ in range(args.steps):
        for name, eg in (("off", plain), ("on", backlog)):
            dt, st = timed_write(e, eg, rng)
            times[name].append(dt * 1e3)
            fd_bytes = st.fd_bytes
    out["fast"] = {k: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v)} for k, v in times.items()}
    out["fast"]["pending_after"] = backlog.flush_backlog(2000)   # a reader thread that fell behind by a batch
    assert plain.failed() == [] and backlog.failed() == []
    out["fast"]["fd_bytes_per_batch"] = fd_bytes
    out["fast"]["on_over_off"] = out["fast"]["on"]["median_ms"] / out["fast"]["off"]["median_ms"]

    # ---- stalled: one peer stops reading
    slow = socket.socketpair()
    slow[0].setsockopt(socket.SOL_SOCKET, socket.SO_SNDBUF, 4096)
    slow[0].setblocking(False)
    c_slow = conns[N_CONNS // 2]
    backlog.attach(c_slow, slow[0].fileno())
    st_times, sizes = [], []
    for _ in range(args.stall_steps):
        dt, st = timed_write(e, backlog, rng)
        st_times.append(dt * 1e3)
        sizes.append(backlog.backlog()[1])
    out["stalled_backlog_on"] = {"median_ms": statistics.median(st_times), "max_ms": max(st_times),
                                 "backlog_bytes_after_first": sizes[0], "backlog_bytes_after_last": sizes[-1],
                                 "batches": args.stall_steps, "failed": backlog.failed()}
    if not args.no_wait_leg:
        plain.attach(c_slow, slow[0].fileno())
        dt, st = timed_write(e, plain, rng)
        out["stalled_backlog_off"] = {"ms": dt * 1e3, "failed": plain.failed()}
    rd.close()
    plain.close(); backlog.close()
    e.close()
    slow[0].close(); slow[1].close()
    for s, r in pairs:
        s.close(); r.close()
    print(json.dumps(out))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
