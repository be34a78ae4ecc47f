#!/usr/bin/env python
"""Delivery by reference above a size threshold (pcdn_config.ref_min_bytes) on one GPU, in one process.

    python scripts/bench_ref_threshold.py [--steps K] [--reps R] [--out FILE]

The card's name, power limit and max SM clock are read in the same run and printed with the numbers.
Workload: 2^16 users on 64 KiB rings; one batch = 8 x 1 KiB broadcasts to all users, one 2 MiB broadcast
to all users and 1024 x 512 B direct messages.
  mixed      a mixed engine (ref_min_bytes = 16 KiB) against a shared-payload engine on that batch,
             alternated rep by rep: device step time of a device-resident batch (CUDA events), the
             engine's stage times, per-kernel times from torch.profiler (k_pack_ref alone, and the
             device-to-host copy of the frame arena), pcdn_submit -> pcdn_egress_drain, and
             pcdn_egress_write_batch into 1000 memfds
  copy       what a copy engine does with that batch: n_overflow
  no_large   the same batch without the 2 MiB broadcast on a copy engine and the mixed engine: device
             step time alternated, kernel launches per step, and the profiler's per-kernel times
Prints one JSON object; with --out also writes it there.
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import __graft_entry__ as ge  # noqa: E402
from bench import KEY_LEN, broadcast_frame  # noqa: E402
from bench_shared_payload import add_users, card, stage_times, time_steps  # noqa: E402

N = 1 << 16
RING = 1 << 16
T = 16 << 10
N_SMALL, SMALL, LARGE, N_DIRECT, DIRECT = 8, 1 << 10, 2 << 20, 1024, 512


def workload(with_large=True):
    """(kind, key or None, raw) in batch order: the small broadcasts, the large one after the fourth, the directs"""
    msgs = []
    for m in range(N_SMALL):
        msgs.append((4, None, broadcast_frame(0, bytes([(m * 37 + i) & 0xFF for i in range(SMALL)]))))
        if m == 3 and with_large:
            msgs.append((4, None, broadcast_frame(0, bytes([(i * 7) & 0xFF for i in range(256)]) * (LARGE // 256))))
    for d in range(N_DIRECT):
        key = np.zeros(KEY_LEN, dtype=np.uint8)
        key[:8] = np.array([d * 61 % N], dtype=np.uint64).view(np.uint8)
        msgs.append((3, key.tobytes(), bytes([d & 0xFF]) * DIRECT))
    return msgs


def device_batch(pkg, msgs, dev, stream):
    arena = bytearray()
    kinds, slot, lens, aoff, alen, bidx = [], [], [], [], [], []
    for i, (k, key, raw) in enumerate(msgs):
        slot.append(len(arena) // 16)
        arena += bytes(4) + raw + bytes((-(4 + len(raw))) % 16)
        kinds.append(k); lens.append(len(raw))
        if k == 3:
            aoff.append(len(arena)); alen.append(len(key))
            arena += key + bytes((-len(key)) % 16)
        else:
            aoff.append(len(bidx)); alen.append(1)
            bidx.append(i)
    M = len(msgs)
    with torch.cuda.stream(stream):
        t = dict(arena=torch.frombuffer(bytearray(arena + bytes(64)), dtype=torch.uint8).to(dev),
                 kind=torch.tensor(kinds, dtype=torch.uint8, device=dev), flags=torch.zeros(M, dtype=torch.uint8, device=dev),
                 slot=torch.tensor(slot, dtype=torch.int32, device=dev), len=torch.tensor(lens, dtype=torch.int32, device=dev),
                 aoff=torch.tensor(aoff, dtype=torch.int32, device=dev), alen=torch.tensor(alen, dtype=torch.int32, device=dev),
                 topics=torch.zeros(len(bidx), dtype=torch.int16, device=dev), bidx=torch.tensor(bidx, dtype=torch.int32, device=dev))
    torch.cuda.synchronize(dev)
    db = pkg.DeviceBatch(M, len(bidx), t["arena"].data_ptr(), len(arena), t["kind"].data_ptr(), t["flags"].data_ptr(),
                         t["slot"].data_ptr(), t["len"].data_ptr(), t["aoff"].data_ptr(), t["alen"].data_ptr(),
                         t["topics"].data_ptr(), len(bidx), t["bidx"].data_ptr())
    db.hints = pkg.BATCH_READY
    return db, t


def host_msgs(msgs):
    return [("b", [0], raw, False) if k == 4 else ("d", key, raw, False) for k, key, raw in msgs]


def engine(pkg, stream, **kw):
    e = pkg.Engine(device=0, stream=stream.cuda_stream, max_conns=N, max_topics=256, max_keys=N, max_key_len=KEY_LEN,
                   ring_bytes_per_conn=RING, max_batch_msgs=2048, max_batch_bcast=16, max_batch_bytes=4 << 20,
                   max_batch_deliveries=16 * N, batch_slots=4, **kw)
    add_users(e, N)
    return e


def kernel_times(eng, db, stream, steps):
    """ms per step of every kernel and copy in a torch.profiler run of its own (CUDA activities)"""
    from torch.profiler import ProfilerActivity, profile

    with torch.cuda.stream(stream):
        for _ in range(2):
            eng.release_batch(eng.submit_device(db))
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                eng.release_batch(eng.submit_device(db))
            torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            name = ev.key.split("(")[0].replace("void pcdn::", "").replace("pcdn::", "")
            out[name] = out.get(name, 0.0) + t / 1e3 / steps
    return dict(sorted(out.items(), key=lambda kv: -kv[1]))


def launches_per_step(eng, db, stream, steps):
    with torch.cuda.stream(stream):
        n0 = eng.stats().kernel_launches
        for _ in range(steps):
            eng.release_batch(eng.submit_device(db))
        torch.cuda.synchronize()
    return (eng.stats().kernel_launches - n0) / steps


def submit_drain_ms(pkg, eng, msgs, reps):
    """host clock around pcdn_submit + pcdn_egress_drain (into pinned host memory) + release"""
    eg = pkg.Egress(eng)
    eng.release_batch(_drained(eg, eng, msgs))
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        b = _drained(eg, eng, msgs)
        ts.append(time.perf_counter() - t0)
        eng.release_batch(b)
    eg.close()
    return 1e3 * statistics.median(ts), ts


def _drained(eg, eng, msgs):
    b = eng.submit(msgs)
    eg.drain(b)
    return b


def write_batch_ms(pkg, eng, msgs, reps, n_fds=1000):
    """pcdn_egress_write_batch into memfds of n_fds connections (host memory, not sockets), verified"""
    eg = pkg.Egress(eng, n_threads=8)
    conns = list(range(0, N, N // n_fds))[:n_fds]
    fds = [os.memfd_create("c%d" % c) for c in conns]
    for c, fd in zip(conns, fds):
        eg.attach(c, fd)
    ts = []
    for i in range(reps + 1):
        for fd in fds:
            os.ftruncate(fd, 0); os.lseek(fd, 0, os.SEEK_SET)
        b = eng.submit(msgs)
        eng.poll(b)
        t0 = time.perf_counter()
        st = eg.write_batch(b)
        t = time.perf_counter() - t0
        eng.release_batch(b)
        if i:
            ts.append(t)
    # (connection conns[1] receives every broadcast; the directs come after them in batch order)
    want = b"".join(len(m[2]).to_bytes(4, "big") + m[2] for m in msgs if m[0] == "b")
    os.lseek(fds[1], 0, os.SEEK_SET)
    verified = os.read(fds[1], len(want)) == want
    for fd in fds:
        os.close(fd)
    eg.close()
    return {"verified_broadcast_stream": verified, "write_batch_ms_median": 1e3 * statistics.median(ts), "fd_bytes": int(st.fd_bytes), "fd_writes": int(st.fd_writes),
            "gbs": st.fd_bytes / statistics.median(ts) / 1e9}


def alternate(engines, db, stream, steps, reps):
    for eng in engines.values():
        time_steps(eng, db, stream, 3)
    ms = {k: [] for k in engines}
    for _ in range(reps):
        for k, eng in engines.items():
            ms[k].append(time_steps(eng, db, stream, steps))
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    pkg = ge.load_package()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing is measured without a GPU")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    stream = torch.cuda.Stream(device=dev)
    res = {"card": card(), "workload": "2^16 users, 64 KiB rings; 8 x 1 KiB + 1 x 2 MiB broadcasts to all, 1024 x 512 B directs; T = 16 KiB"}
    msgs = workload(True)
    hm = host_msgs(msgs)
    db, keep = device_batch(pkg, msgs, dev, stream)

    # ---- mixed against shared payload
    engines = {"mixed": engine(pkg, stream, ref_min_bytes=T), "shared": engine(pkg, stream, flags=pkg.FLAG_SHARED_PAYLOAD)}
    for k, eng in engines.items():          # every delivery arrives, nothing overflows
        r = eng.poll(b := eng.submit(hm))
        assert r.status == 0 and r.n_overflow == 0 and r.n_deliveries == (N_SMALL + 1) * N + N_DIRECT, (k, r.n_deliveries, r.n_overflow)
        eng.release_batch(b)
    ms = alternate(engines, db, stream, args.steps, args.reps)
    out = {}
    for k, eng in engines.items():
        out[k] = {"device_ms_per_step_median": statistics.median(ms[k]), "device_ms_per_step_all": ms[k],
                  "stage_ms": stage_times(eng, db, stream, args.steps),
                  "kernel_ms_per_step": kernel_times(eng, db, stream, args.steps),
                  "launches_per_step": launches_per_step(eng, db, stream, args.steps)}
        d_ms, d_all = submit_drain_ms(pkg, eng, hm, max(3, args.reps))
        out[k]["submit_drain_ms_median"] = d_ms
        out[k]["submit_drain_ms_all"] = [1e3 * t for t in d_all]
        out[k]["writer"] = write_batch_ms(pkg, eng, hm, max(3, args.reps))
    for eng in engines.values():
        eng.close()
    res["mixed_vs_shared"] = out

    # ---- the copy engine on the same batch
    cp = engine(pkg, stream)
    r = cp.poll(b := cp.submit(hm))
    res["copy_full_batch"] = {"status": int(r.status), "n_overflow": int(r.n_overflow), "n_deliveries": int(r.n_deliveries)}
    cp.release_batch(b)
    cp.close()

    # ---- without the 2 MiB broadcast: copy engine against the mixed engine
    small = workload(False)
    db2, keep2 = device_batch(pkg, small, dev, stream)
    engines = {"copy": engine(pkg, stream), "mixed": engine(pkg, stream, ref_min_bytes=T)}
    ms = alternate(engines, db2, stream, args.steps, args.reps)
    out = {}
    for k, eng in engines.items():
        out[k] = {"device_ms_per_step_median": statistics.median(ms[k]), "device_ms_per_step_all": ms[k],
                  "stage_ms": stage_times(eng, db2, stream, args.steps),
                  "kernel_ms_per_step": kernel_times(eng, db2, stream, args.steps),
                  "launches_per_step": launches_per_step(eng, db2, stream, args.steps)}
        d_ms, d_all = submit_drain_ms(pkg, eng, host_msgs(small), max(3, args.reps))
        out[k]["submit_drain_ms_median"] = d_ms
    for eng in engines.values():
        eng.close()
    res["no_large"] = out
    res["card_after"] = card()
    s = json.dumps(res)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
