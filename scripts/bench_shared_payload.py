#!/usr/bin/env python
"""Copy mode against shared-payload mode (PCDN_FLAG_SHARED_PAYLOAD) on one GPU, in one process.

    python scripts/bench_shared_payload.py [--steps K] [--reps R] [--out FILE]

Three legs; the card's name and power limit are read in the same run and printed with the numbers.
  c2      the bench.py C2 shape (2^20 subscribers, 8 x 1 KiB broadcasts per batch, batch resident in HBM,
          run-length span table): device step time with CUDA events, alternating the two modes R times;
          the engine's stage times (match, plan + offsets, pack); the pack kernel's bytes/s over its
          algorithmic bytes against 3.35 TB/s; and pcdn_egress_drain of a host-submitted batch into pinned
          host memory, with every shared-mode record checked and a sample of streams expanded.
  large   16384 users x 4 broadcasts of 4 MiB per batch.  Shared mode only: copy mode would need
          16384 x 4 x 4 MiB = 256 GiB of rings or pool for one batch, so it cannot place it.
  writer  pcdn_egress_write_batch into memfds (host memory, not sockets) for a C2 subset of 1000
          connections, both modes.
Prints one JSON object; with --out also writes it there.
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

import __graft_entry__ as ge  # noqa: E402
from bench import KEY_LEN, MSGS_PER_STEP, N_CONNS, PAYLOAD, RING_RECORDS, broadcast_frame  # noqa: E402

HBM_PEAK = 3350.0   # GB/s, H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=60)
    return q.stdout.strip()


def add_users(eng, n, topic=0):
    keys = np.zeros((n, KEY_LEN), dtype=np.uint8)
    keys[:, :8] = np.arange(n, dtype=np.uint64).view(np.uint8).reshape(n, 8)
    eng.add_users_bulk(keys, KEY_LEN, np.full(n, topic, dtype=np.uint16), np.arange(n + 1, dtype=np.uint32))


def device_batch(pkg, frames, dev, stream):
    M, L = len(frames), len(frames[0])
    slot = (4 + L + 15) // 16 * 16
    arena = np.zeros(M * slot + 64, dtype=np.uint8)
    for m, fr in enumerate(frames):
        arena[m * slot + 4:m * slot + 4 + L] = np.frombuffer(fr, dtype=np.uint8)
    with torch.cuda.stream(stream):
        t = dict(arena=torch.from_numpy(arena).to(dev), kind=torch.full((M,), 4, dtype=torch.uint8, device=dev),
                 flags=torch.zeros(M, dtype=torch.uint8, device=dev),
                 slot=(torch.arange(M, device=dev) * (slot // 16)).to(torch.int32),
                 len=torch.full((M,), L, dtype=torch.int32, device=dev), aoff=torch.arange(M, dtype=torch.int32, device=dev),
                 alen=torch.ones(M, dtype=torch.int32, device=dev), topics=torch.zeros(M, dtype=torch.int16, device=dev),
                 bidx=torch.arange(M, dtype=torch.int32, device=dev))
    torch.cuda.synchronize(dev)
    db = pkg.DeviceBatch(M, M, t["arena"].data_ptr(), t["arena"].numel(), t["kind"].data_ptr(), t["flags"].data_ptr(),
                         t["slot"].data_ptr(), t["len"].data_ptr(), t["aoff"].data_ptr(), t["alen"].data_ptr(),
                         t["topics"].data_ptr(), M, t["bidx"].data_ptr())
    db.hints = pkg.BATCH_READY
    return db, t, slot


def time_steps(eng, db, stream, steps):
    """ms per step of submit_device + release (the bench.py loop), CUDA events on the engine's stream"""
    with torch.cuda.stream(stream):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(steps):
            eng.release_batch(eng.submit_device(db))
        e1.record(stream)
        e1.synchronize()
    return e0.elapsed_time(e1) / steps


def stage_times(eng, db, stream, steps):
    eng.set_timing(True)
    s0 = eng.stats()
    with torch.cuda.stream(stream):
        for _ in range(steps):
            b = eng.submit_device(db)
            eng.poll(b)
            eng.release_batch(b)
    s1 = eng.stats()
    eng.set_timing(False)
    n = max(1, s1.timed_batches - s0.timed_batches)
    return {"match": (s1.ms_match - s0.ms_match) / n, "plan_offsets": (s1.ms_plan - s0.ms_plan) / n,
            "direct": (s1.ms_direct - s0.ms_direct) / n, "pack": (s1.ms_pack - s0.ms_pack) / n}


def leg_c2(pkg, dev, stream, steps, reps):
    N, M = N_CONNS, MSGS_PER_STEP
    frames = [broadcast_frame(0, bytes(((i * 131 + m * 7 + 1) & 0xFF) for i in range(PAYLOAD))) for m in range(M)]
    L = len(frames[0]); F = 4 + L
    rec = (F + 31) // 32 * 32
    common = dict(device=0, stream=stream.cuda_stream, max_conns=N, max_topics=256, max_keys=N, max_key_len=KEY_LEN,
                  max_batch_msgs=64, max_batch_bcast=16, max_batch_bytes=1 << 20, max_batch_deliveries=M * N + 1024,
                  batch_slots=4)
    engines = {
        "copy": pkg.Engine(ring_bytes_per_conn=RING_RECORDS * rec, flags=pkg.FLAG_SPAN_RUNS, **common),
        "shared": pkg.Engine(ring_bytes_per_conn=RING_RECORDS * 32, flags=pkg.FLAG_SPAN_RUNS | pkg.FLAG_SHARED_PAYLOAD, **common),
    }
    for eng in engines.values():
        add_users(eng, N)
    db, keep, slot = device_batch(pkg, frames, dev, stream)
    for eng in engines.values():
        time_steps(eng, db, stream, 3)
    ms = {k: [] for k in engines}
    for _ in range(reps):                      # alternated in one process
        for k, eng in engines.items():
            ms[k].append(time_steps(eng, db, stream, steps))
    out = {}
    D = M * N
    for k, eng in engines.items():
        st = stage_times(eng, db, stream, steps)
        step = statistics.median(ms[k])
        if k == "copy":
            pack_bytes = M * (N * F + L)               # bench.py: D x F stores + L read per message
            note = "k_pack: D x F record stores + L frame bytes read per message"
        else:
            pack_bytes = D * (32 + 8) + M * 8          # D x 32 record stores + D x 8 scatter-list reads (+ per-message words)
            note = "k_pack_ref: D x 32 record stores + D x 8 B scatter-list entries read"
        out[k] = {"ms_per_step_median": step, "ms_per_step_all": ms[k], "stage_ms": st,
                  "ring_bytes_written_per_step": D * (rec if k == "copy" else 32),
                  "pack_algorithmic_bytes": pack_bytes, "pack_gbs": pack_bytes / (st["pack"] * 1e-3) / 1e9,
                  "pack_pct_of_3350": 100.0 * pack_bytes / (st["pack"] * 1e-3) / 1e9 / HBM_PEAK, "pack_bytes_note": note,
                  "wire_gbs": D * F / (step * 1e-3) / 1e9}
    # egress drain of a host-submitted batch into pinned host memory (PCIe-bound)
    host_msgs = [("b", [0], fr, False) for fr in frames]
    for k, eng in engines.items():
        eg = pkg.Egress(eng)
        b = eng.submit(host_msgs)
        eg.drain(b)
        eng.release_batch(b)
        ts = []
        for _ in range(max(3, min(steps, 6))):
            b = eng.submit(host_msgs)
            t0 = time.perf_counter()
            st = eg.drain(b)
            ts.append(time.perf_counter() - t0)
            eng.release_batch(b)
        out[k]["drain_ms_median"] = 1e3 * statistics.median(ts)
        out[k]["drain_bytes_per_step"] = int(st.bytes)
        out[k]["drain_chunks"] = int(st.chunks)
        if k == "shared":
            # every record made host-readable must be the model; a sample of connections expanded
            b = eng.submit(host_msgs)
            base = eng.batch_payload(b)
            model = np.frombuffer(b"".join(b"\xff\xff\xff\xff" + L.to_bytes(4, "big") + (m * slot + 4).to_bytes(8, "little") +
                                           b.to_bytes(8, "little") + bytes(8) for m in range(M)), dtype=np.uint8)
            seen = {"spans": 0, "bad": 0, "expanded": 0}

            def check(ch):
                n = ch.n_spans
                flat = np.ctypeslib.as_array(C.cast(ch.data, C.POINTER(C.c_uint8)), shape=(ch.bytes,))
                offs = np.ctypeslib.as_array(ch.data_off, shape=(n,)).astype(np.int64)
                # a staged chunk holds its spans back to back: one (n, M x 32) block
                ok = bool((offs == offs[0] + np.arange(n, dtype=np.int64) * M * 32).all()) and \
                    bool((flat[int(offs[0]):int(offs[0]) + n * M * 32].reshape(n, M * 32) == model[None, :]).all())
                seen["spans"] += ch.n_spans
                seen["bad"] += 0 if ok else 1
                for i in range(0, ch.n_spans, 9973):
                    p = ch.data + ch.data_off[i]
                    got = [C.string_at(base + int.from_bytes(C.string_at(p + 32 * r + 8, 8), "little"),
                                       int.from_bytes(C.string_at(p + 32 * r + 4, 4), "big")) for r in range(M)]
                    seen["bad"] += 0 if got == frames else 1
                    seen["expanded"] += 1

            eg.drain(b, check)
            eng.release_batch(b)
            assert seen["spans"] == N and seen["bad"] == 0, seen
            out[k]["drain_verify"] = "all %d x %d records bit-exact in host memory, %d connections' streams expanded" % (N, M, seen["expanded"])
        eg.close()
    for eng in engines.values():
        eng.close()
    out["step_speedup_device"] = out["copy"]["ms_per_step_median"] / out["shared"]["ms_per_step_median"]
    out["drain_speedup"] = out["copy"]["drain_ms_median"] / out["shared"]["drain_ms_median"]
    return out


def leg_large(pkg, dev, stream, steps):
    n_users, M, size = 16384, 4, 4 << 20
    eng = pkg.Engine(device=0, stream=stream.cuda_stream, max_conns=n_users, max_topics=256, max_keys=n_users, max_key_len=KEY_LEN,
                     ring_bytes_per_conn=1 << 16, max_batch_msgs=64, max_batch_bcast=16, max_batch_bytes=M * (size + 4096) + (1 << 20),
                     max_batch_deliveries=M * n_users + 1024, batch_slots=2, flags=pkg.FLAG_SHARED_PAYLOAD)
    add_users(eng, n_users)
    frames = [broadcast_frame(0, bytes([m + 1]) * size) for m in range(M)]
    db, keep, slot = device_batch(pkg, frames, dev, stream)
    time_steps(eng, db, stream, 2)
    dev_ms = time_steps(eng, db, stream, steps)
    eg = pkg.Egress(eng)
    msgs = [("b", [0], fr, False) for fr in frames]
    b = eng.submit(msgs)
    eg.drain(b)
    eng.release_batch(b)
    ts = []
    for _ in range(3):
        t0 = time.perf_counter()
        b = eng.submit(msgs)
        st = eg.drain(b)
        eng.release_batch(b)
        ts.append(time.perf_counter() - t0)
    res = None
    b = eng.submit(msgs)
    res = eng.poll(b)
    assert res.status == 0 and res.n_overflow == 0 and res.n_deliveries == M * n_users
    eng.release_batch(b)
    eg.close()
    eng.close()
    wire = M * n_users * (4 + len(frames[0]))
    return {"shape": "16384 users x 4 broadcasts of 4 MiB (64 KiB rings)", "device_ms_per_step": dev_ms,
            "host_submit_drain_ms_median": 1e3 * statistics.median(ts), "drain_bytes_per_step": int(st.bytes),
            "wire_bytes_per_step": wire, "wire_gbs_device": wire / (dev_ms * 1e-3) / 1e9,
            "wire_gbs_host_submit_drain": wire / statistics.median(ts) / 1e9,
            "copy_mode": "not measured: one batch would need 16384 x 4 x (4 MiB + 4) B = 256 GiB of rings or output pool"}


def leg_writer(pkg, stream, steps):
    n, M = 1000, MSGS_PER_STEP
    frames = [broadcast_frame(0, bytes(((i * 131 + m * 7 + 1) & 0xFF) for i in range(PAYLOAD))) for m in range(M)]
    msgs = [("b", [0], fr, False) for fr in frames]
    out = {}
    for k, fl in (("copy", pkg.FLAG_SPAN_RUNS), ("shared", pkg.FLAG_SPAN_RUNS | pkg.FLAG_SHARED_PAYLOAD)):
        eng = pkg.Engine(device=0, stream=stream.cuda_stream, max_conns=n, max_topics=256, max_keys=n, max_key_len=KEY_LEN,
                         ring_bytes_per_conn=1 << 16, flags=fl)
        add_users(eng, n)
        eg = pkg.Egress(eng)
        fds = [os.memfd_create("c%d" % c) for c in range(n)]
        for c, fd in enumerate(fds):
            eg.attach(c, fd)
        ts = []
        for i in range(steps + 2):
            for fd in fds:
                os.ftruncate(fd, 0); os.lseek(fd, 0, os.SEEK_SET)
            b = eng.submit(msgs)
            eng.poll(b)
            t0 = time.perf_counter()
            st = eg.write_batch(b)
            t = time.perf_counter() - t0
            eng.release_batch(b)
            if i >= 2:
                ts.append(t)
        want = b"".join(len(fr).to_bytes(4, "big") + fr for fr in frames)
        os.lseek(fds[n // 2], 0, os.SEEK_SET)
        assert os.read(fds[n // 2], len(want) + 1) == want
        for fd in fds:
            os.close(fd)
        out[k] = {"write_batch_ms_median": 1e3 * statistics.median(ts), "fd_bytes": int(st.fd_bytes), "fd_writes": int(st.fd_writes),
                  "gbs": st.fd_bytes / statistics.median(ts) / 1e9}
        eg.close()
        eng.close()
    out["note"] = "writev into memfds (host memory), not sockets; %d connections x %d x 1 KiB" % (n, M)
    return out


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
    res = {"card": card()}
    res["c2"] = leg_c2(pkg, dev, stream, args.steps, args.reps)
    res["large"] = leg_large(pkg, dev, stream, max(3, args.steps // 4))
    res["writer"] = leg_writer(pkg, stream, max(3, args.steps // 4))
    res["card_after"] = card()
    s = json.dumps(res)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
