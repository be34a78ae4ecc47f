#!/usr/bin/env python
"""Time of the fused small-engine control stage (k_ctrl_small: direct lookup and sort, match, plan and offsets in one
cluster launch) on GPU 0, per batch shape.

    python scripts/bench_ctrl_small.py [--batches K] [--warmup W] [--out FILE]

Engines of 8192 and 65536 connection slots (all but 8 of them users, 64 topics, each user on one; 8 peer brokers,
broker b on topic b).  Batch shapes, every message 256 B:
  one        1 broadcast;
  full       broadcasts filling the fused kernel's match: kSmallCtrlItems (broadcast, 8192-connection block) items,
             i.e. 256 broadcasts on 8192 slots and 32 on 65536;
  events     full, with 16 in-batch subscription events (PCDN_FLAG_INBATCH_SUBSCRIBE) spread over the batch: 8 users
             subscribe to a topic and then unsubscribe from it, so every batch starts from the same bitmap;
  send       full, with its middle broadcast replaced by a pcdn_send_to_broker to one peer broker;
  direct     full, with 64 direct messages to users interleaved; on 8192 slots the batch keeps 192 broadcasts, so
             that it stays within the fused kernel's kSmallCtrlMsgs = 256 messages.
Each batch is built through the handle_* calls, flushed, polled and released.  The stage time of a batch is the CUDA
event time the engine's stage timing (pcdn_set_timing) records around the fused kernel (pcdn_stats.ms_match); reported
per shape: its median and minimum over K batches after W warm-up batches, and the kernel launches per batch.  The card's
name, power limit and SM clock limit are read in the same run.  Prints one JSON object; with --out also writes it.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import __graft_entry__ as ge  # noqa: E402
from oracle import oracle as orc  # noqa: E402

N_TOPICS, N_BROKERS, PAYLOAD, ITEMS, MAX_MSGS, BLOCK = 64, 8, 256, 256, 256, 8192


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=60)
    return q.stdout.strip()


def key(i):
    return b"u%07d" % i


def engine(pcdn, n_slots):
    n_users = n_slots - N_BROKERS
    e = pcdn.Engine(device=0, max_conns=n_slots, max_topics=256, max_keys=2 * n_users, ring_bytes_per_conn=1 << 16,
                    max_batch_msgs=MAX_MSGS, max_batch_bcast=MAX_MSGS, max_batch_bytes=1 << 20,
                    max_batch_deliveries=1 << 20, batch_slots=2, flags=pcdn.FLAG_INBATCH_SUBSCRIBE)
    keys = np.frombuffer(b"".join(key(i) for i in range(n_users)), dtype=np.uint8).reshape(n_users, 8).copy()
    e.add_users_bulk(keys, 8, np.arange(n_users, dtype=np.uint16) % N_TOPICS, np.arange(n_users + 1, dtype=np.uint32))
    for b in range(N_BROKERS):
        e.add_broker("b%d/x" % b)
        e.subscribe_broker_to("b%d/x" % b, [b])
    e.set_timing(True)
    return e, n_users


def run_batch(e, n_users, shape, n_bcast):
    """one batch of `shape`; returns (stage ms, kernel launches)"""
    raw = orc.broadcast_frame([0], b"p" * PAYLOAD)
    draw = orc.direct_frame(key(0), b"d" * PAYLOAD)
    events = {n_bcast * k // 16: k for k in range(16)} if shape == "events" else {}
    st0 = e.stats()
    for j in range(n_bcast):
        if j in events:   # user u subscribes to topic t at event k, and leaves it again at event k + 8
            k = events[j]
            u, t = (k % 8) * (n_users // 8) + 1, (k % 8) + 9
            (e.subscribe_user_to if k < 8 else e.unsubscribe_user_from)(key(u), [t])
        if shape == "send" and j == n_bcast // 2:
            assert e.send_to_broker("b0/x", raw) == 0
        else:
            e.handle_broadcast_message([j % N_TOPICS], raw)
        for d in range(64 * j // n_bcast, 64 * (j + 1) // n_bcast) if shape == "direct" else ():
            e.handle_direct_message(key((d * 997) % n_users), draw)
    e.flush()
    while True:
        b = e.next_batch()
        if not b:
            break
        r = e.poll(b)
        assert r.status == 0 and r.n_overflow == 0, (r.status, r.n_overflow)
        e.release_batch(b)
    st1 = e.stats()
    assert st1.batches == st0.batches + 1 and st1.timed_batches == st0.timed_batches + 1
    return st1.ms_match - st0.ms_match, st1.kernel_launches - st0.kernel_launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out")
    args = ap.parse_args()
    pcdn = ge.load_package()
    out = {"card": card(), "metric": "fused control stage (k_ctrl_small) per batch, CUDA events, ms", "cases": []}
    for n_slots in (8192, 65536):
        e, n_users = engine(pcdn, n_slots)
        nblk = -(-n_slots // BLOCK)
        for shape in ("one", "full", "events", "send", "direct"):
            n_bcast = 1 if shape == "one" else ITEMS // nblk
            if shape == "direct":
                n_bcast = min(n_bcast, MAX_MSGS - 64)
            ms, launches = [], set()
            for i in range(args.warmup + args.batches):
                t, n = run_batch(e, n_users, shape, n_bcast)
                if i >= args.warmup:
                    ms.append(t)
                    launches.add(n)
            out["cases"].append({"slots": n_slots, "shape": shape, "broadcasts": n_bcast, "match_items": n_bcast * nblk,
                                 "median_ms": statistics.median(ms), "min_ms": min(ms), "launches": sorted(launches)})
        e.close()
    print(json.dumps(out), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
