#!/usr/bin/env python
"""bench_configs.py — the other BASELINE.json configs (C3, C4, C5) as secondary measurements.

`bench.py` is the driver-facing benchmark (config C2).  This script measures the remaining configs
of BASELINE.json on ONE GPU with the same rules (inputs resident in HBM, CUDA events on the engine's
stream, >= 3 warm-up steps, outputs far larger than L2) and prints one JSON line per workload:

    python bench_configs.py --workload C4        # direct path: 2^20 128-byte keys, 2^20 msgs/batch, 512 B
    python bench_configs.py --workload C3        # 64 K subs, 4 K topics Zipf-0.99, 256 B-64 KiB payloads
    python bench_configs.py --workload C5dense   # one shard of config 5: 2^20 subs, 4 KiB broadcast
    python bench_configs.py --workload C5sparse  # 1 K topics, 4 subscriptions per connection

Correctness of these paths is covered bit-exactly (against the oracle) by tests/test_gpu_parity.py and
tests/test_gpu_configs.py at sizes the oracle finishes in seconds; here only the engine's own counters
are cross-checked against the analytically expected delivery counts.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
import bench as B  # noqa: E402  (helpers only)


def direct_frame_template(key_len: int, payload_len: int):
    """single-segment Direct{recipient[key_len], message[payload_len]} (SURVEY Appendix B); returns
    (frame bytes with zero recipient/payload, recipient offset, payload offset)"""
    rw, pw = (key_len + 7) // 8, (payload_len + 7) // 8
    words = 5 + rw + pw
    out = bytearray()
    out += (0).to_bytes(4, "little") + words.to_bytes(4, "little")
    out += bytes.fromhex("0000000001000100")
    out += (3).to_bytes(8, "little")
    out += bytes.fromhex("0000000000000200")
    out += (5).to_bytes(4, "little") + (2 | (key_len << 3)).to_bytes(4, "little")
    out += ((rw << 2) | 1).to_bytes(4, "little") + (2 | (payload_len << 3)).to_bytes(4, "little")
    roff = len(out)
    out += bytes(rw * 8)
    poff = len(out)
    out += bytes(pw * 8)
    return bytes(out), roff, poff


def bcast_frame_n(topics_bytes: bytes, payload: bytes) -> bytes:
    n, k = len(topics_bytes), len(payload)
    tw = (n + 7) // 8
    words = 5 + tw + (k + 7) // 8
    out = bytearray()
    out += (0).to_bytes(4, "little") + words.to_bytes(4, "little")
    out += bytes.fromhex("0000000001000100") + (4).to_bytes(8, "little") + bytes.fromhex("0000000000000200")
    out += (5).to_bytes(4, "little") + (2 | (n << 3)).to_bytes(4, "little")
    out += ((tw << 2) | 1).to_bytes(4, "little") + (2 | (k << 3)).to_bytes(4, "little")
    out += topics_bytes + bytes((-n) % 8) + payload + bytes((-k) % 8)
    return bytes(out)


class DeviceBatch:
    """device-resident batch in the layout of pcdn_device_batch (slots 16-byte aligned, raw at +4)"""

    def __init__(self, pkg, torch, dev, arena_np, kind, flags, slot16, raw_len, aux_off, aux_len, topics, bidx):
        t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to(dev) if len(a) else torch.zeros(1, dtype=dt, device=dev)
        self.arena = t(arena_np, torch.uint8)
        self.kind = t(kind.astype(np.uint8), torch.uint8)
        self.flags = t(flags.astype(np.uint8), torch.uint8)
        self.slot = t(slot16.astype(np.int32), torch.int32)
        self.len = t(raw_len.astype(np.int32), torch.int32)
        self.aoff = t(aux_off.astype(np.int32), torch.int32)
        self.alen = t(aux_len.astype(np.int32), torch.int32)
        self.topics = t(topics.astype(np.int16), torch.int16)
        self.bidx = t(bidx.astype(np.int32), torch.int32)
        n, nb = len(kind), len(bidx)
        self.db = pkg.DeviceBatch(n, nb, self.arena.data_ptr(), self.arena.numel(), self.kind.data_ptr(), self.flags.data_ptr(),
                                  self.slot.data_ptr(), self.len.data_ptr(), self.aoff.data_ptr(), self.alen.data_ptr(),
                                  self.topics.data_ptr(), len(topics), self.bidx.data_ptr())
        self.db.hints = pkg.BATCH_READY   # complete in device memory before the first submit


def zipf_p(n, s=0.99):
    p = 1.0 / np.arange(1, n + 1) ** s
    return p / p.sum()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", required=True, choices=["C1", "C3", "C4", "C5dense", "C5sparse", "latency", "churn", "writer"])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--variant", type=int, default=0)
    ap.add_argument("--hit", type=float, default=1.0, help="C4: fraction of recipients that exist")
    ap.add_argument("--msgs", type=int, default=0, help="C3: messages per batch (default 128; SURVEY 8d asks for 1024, which needs --pool)")
    ap.add_argument("--pool", type=float, default=0.0, help="GB of shared output pool (PCDN_FLAG_OUTPUT_POOL) instead of per-connection rings")
    ap.add_argument("--ingest", choices=["host", "device"], default=None,
                    help="C4 only: measure end-to-end ingest of RAW FRAMES from host memory through pcdn_receive_frames with the host parser or the device parse kernel")
    args = ap.parse_args()
    import torch

    import __graft_entry__ as ge

    pkg = ge.load_package()
    wl = args.workload
    # config 5 proper: one process per GPU (torchrun), every rank owns a 2^20-connection shard, the
    # batch is generated on rank 0 and replicated with one NCCL broadcast per step (no other collective)
    rank, local, world = int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    if world > 1:
        import torch.distributed as dist
        assert wl in ("C5dense", "C5sparse"), "only config 5 is a multi-GPU workload"
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    dev = torch.device("cuda", local)
    torch.cuda.set_device(local)
    stream = torch.cuda.Stream(device=dev)
    t_setup = time.time()

    if wl == "latency":
        # one message at a time through the host-buffer API: submit → poll (counters + span table back)
        out = {"metric": "single-message fan-out latency, host buffers in, pcdn_submit → pcdn_poll complete (wall clock)", "unit": "us", "cases": []}
        for n, host_rings, runs in ((128, False, False), (128, True, False), (1 << 14, False, False), (1 << 20, False, False), (1 << 20, False, True)):
            rng = np.random.default_rng(9)
            keys = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
            keys[:, :8] = np.arange(n, dtype=np.uint64).view(np.uint8).reshape(n, 8)
            raw = B.broadcast_frame(0, bytes(1024))
            rec = (4 + len(raw) + 31) // 32 * 32
            eng = pkg.Engine(device=0, stream=stream.cuda_stream, max_conns=n, max_topics=16, max_keys=n, max_key_len=32,
                             ring_bytes_per_conn=16 * rec, max_batch_msgs=64, max_batch_bcast=16, max_batch_bytes=1 << 20,
                             max_batch_deliveries=n + 1024, batch_slots=2, pack_variant=args.variant,
                             flags=(pkg.FLAG_HOST_RINGS if host_rings else 0) | (pkg.FLAG_SPAN_RUNS if runs else 0))
            eng.add_users_bulk(keys, 32, np.zeros(n, dtype=np.uint16), np.arange(n + 1, dtype=np.uint32))
            rcpt = keys[n // 2].tobytes()
            tmpl, roff, poff = direct_frame_template(32, 512)
            draw = bytearray(tmpl); draw[roff:roff + 32] = rcpt; draw = bytes(draw)
            tag = " — rings in host memory (PCDN_FLAG_HOST_RINGS): framed bytes readable in place when poll returns" if host_rings else ""
            if runs:
                tag += " — run-length span table (PCDN_FLAG_SPAN_RUNS)"
            for name, msgs in (("broadcast 1 KiB to all %d subscribers%s" % (n, tag), [("b", [0], raw, False)]),
                               ("direct 512 B to one of %d users%s" % (n, tag), [("d", rcpt, draw, False)])):
                ts, tsub = [], []
                for it in range(220):
                    t0 = time.perf_counter()
                    b = eng.submit(msgs)
                    tm = time.perf_counter()
                    r = eng.poll(b)
                    t1 = time.perf_counter()
                    eng.release_batch(b)
                    if it >= 20:
                        ts.append((t1 - t0) * 1e6)
                        tsub.append((tm - t0) * 1e6)
                assert r.n_deliveries == (n if msgs[0][0] == "b" else 1)
                if host_rings:  # what the socket writers would send, read in place
                    b = eng.submit(msgs); r = eng.poll(b)
                    got = eng.collect_frames(r)
                    eng.release_batch(b)
                    assert len(got) == r.n_deliveries and all(f == [msgs[0][2]] for f in got.values())
                ts.sort(); tsub.sort()
                out["cases"].append({"case": name, "p50_us": ts[len(ts) // 2], "p99_us": ts[int(len(ts) * 0.99)], "min_us": ts[0],
                                     "submit_call_p50_us": tsub[len(tsub) // 2], "deliveries": int(r.n_deliveries)})
            eng.close()
        print(json.dumps(out), flush=True)
        return

    if wl == "writer":
        # f-2 egress writer: 8192 subscribers, each with its own memfd as "socket"; batches of 8 x 1 KiB broadcasts;
        # pcdn_egress_write_batch = poll + gather + DMA + one writev per connection and batch on the writer threads
        import resource
        soft, hard = resource.getrlimit(resource.RLIMIT_NOFILE)
        resource.setrlimit(resource.RLIMIT_NOFILE, (hard, hard))
        n, M = min(8192, hard - 256), 8
        rng = np.random.default_rng(12)
        keys = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
        keys[:, :8] = np.arange(n, dtype=np.uint64).view(np.uint8).reshape(n, 8)
        frames = [B.broadcast_frame(0, bytes(((i * 131 + m) & 0xFF) for i in range(1024))) for m in range(M)]
        L = len(frames[0]); rec = (4 + L + 31) // 32 * 32
        out = {"metric": "egress writer: pcdn_submit (host buffers) -> pcdn_egress_write_batch to one memfd per connection (wall clock)", "cases": []}
        for host_rings in (False, True):
            eng = pkg.Engine(device=0, stream=stream.cuda_stream, max_conns=n, max_topics=16, max_keys=n, max_key_len=32,
                             ring_bytes_per_conn=4 * M * rec, max_batch_msgs=64, max_batch_bcast=16, max_batch_bytes=1 << 20,
                             max_batch_deliveries=M * n + 1024, batch_slots=2, flags=pkg.FLAG_SPAN_RUNS | (pkg.FLAG_HOST_RINGS if host_rings else 0))
            conns = eng.add_users_bulk(keys, 32, np.zeros(n, dtype=np.uint16), np.arange(n + 1, dtype=np.uint32))
            eg = pkg.Egress(eng, n_threads=16)
            fds = [os.memfd_create("c%d" % c) for c in conns]
            for c, fd in zip(conns, fds):
                eg.attach(int(c), fd)
            msgs = [("b", [0], fr, False) for fr in frames]
            ts, nbytes = [], 0
            for it in range(8):
                t0 = time.perf_counter()
                b = eng.submit(msgs)
                st = eg.write_batch(b)
                eng.release_batch(b)
                t1 = time.perf_counter()
                assert st.fd_bytes == n * M * (4 + L) and st.unattached_spans == 0 and eg.failed() == []
                if it >= 2:
                    ts.append(t1 - t0); nbytes = st.fd_bytes
                if it == 7:   # what is in the "sockets" is the framed stream
                    want = b"".join(L.to_bytes(4, "big") + fr for fr in frames)
                    for fd in fds[:: max(1, n // 64)]:
                        sz = os.lseek(fd, 0, os.SEEK_END)
                        os.lseek(fd, sz - len(want), os.SEEK_SET)
                        assert os.read(fd, len(want)) == want
                for fd in fds:
                    os.ftruncate(fd, 0); os.lseek(fd, 0, os.SEEK_SET)
            ts.sort()
            p50 = ts[len(ts) // 2]
            out["cases"].append({"rings": "mapped pinned host memory (read in place)" if host_rings else "HBM (gather + DMA)", "connections": n,
                                 "bytes_per_batch": int(nbytes), "p50_ms_per_batch": p50 * 1e3, "GBps_to_file_descriptors": nbytes / p50 / 1e9,
                                 "writev_calls_per_batch": int(st.fd_writes), "writer_threads": 16})
            for fd in fds:
                os.close(fd)
            eg.close(); eng.close()
        print(json.dumps(out), flush=True)
        return

    if wl == "C1":
        # BASELINE config 1 (the reference's own bench shape, cdn-broker/benches/broadcast.rs): 128 users on
        # one topic, user 0 sends 1 KiB broadcasts, every user incl. the sender receives them.  Raw frames
        # in host memory → pcdn_receive_frames (host parse, R6 prune, staging) → flush → poll → release,
        # wall clock, for batches of 1 / 16 / 256 frames per receive call.
        import ctypes as C
        n, K = 128, 1024
        keys = [i.to_bytes(8, "little") for i in range(n)]                    # tests/mod.rs:111-115
        raw = bcast_frame_n(bytes([0]), bytes(((i * 7 + 1) & 0xFF) for i in range(K)))
        Lr = len(raw)
        eng = pkg.Engine(device=0, stream=stream.cuda_stream, max_conns=n, max_topics=256, max_keys=256, max_key_len=32,
                         ring_bytes_per_conn=1 << 20, max_batch_msgs=256, max_batch_bcast=256, max_batch_bytes=1 << 20,
                         max_batch_deliveries=256 * n + 1024, batch_slots=2, pack_variant=args.variant)
        for k in keys:
            eng.add_user(k, [0])
        out = {"metric": "config C1 through the engine: raw frames in host memory -> pcdn_receive_frames -> flush -> poll -> release (wall clock)",
               "config": {"workload": "C1: 128 subscribers, 1 topic, 1 KiB broadcast from user 0 (also a subscriber)", "frame_bytes": 4 + Lr},
               "cases": []}
        buf = (C.c_char * Lr).from_buffer_copy(raw)
        for M in (1, 16, 256):
            fa = (pkg.Frame * M)()
            for i in range(M):
                fa[i].sender = keys[0]; fa[i].sender_len = 8; fa[i].origin = 0
                fa[i].raw = C.cast(buf, C.c_char_p); fa[i].raw_len = Lr
            iters = 400 if M < 256 else 200
            ts = []
            for it in range(iters + 20):
                t0 = time.perf_counter()
                rc = eng.L.pcdn_receive_frames(eng.h, fa, M, None)
                assert rc == M, rc
                b = eng.flush()
                res = eng.poll(b)
                t1 = time.perf_counter()
                assert res.n_deliveries == M * n and res.status == 0 and res.n_overflow == 0
                eng.release_batch(b)
                if it >= 20:
                    ts.append(t1 - t0)
            ts.sort()
            p50 = ts[len(ts) // 2]
            out["cases"].append({"frames_per_call": M, "p50_us_per_batch": p50 * 1e6, "msgs_per_s": M / p50,
                                 "deliveries_per_s": M * n / p50, "egress_GBps": M * n * (4 + Lr) / p50 / 1e9})
        print(json.dumps(out), flush=True)
        eng.close()
        return

    if wl == "churn":
        # config C2 with connection / subscription churn between batches: every step 40 (un)subscribes and
        # 10 disconnect+connect pairs go through the state ABI (host mirror → journal → k_apply_* on the stream)
        n, M = 1 << 20, 8
        rng = np.random.default_rng(11)
        keys = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
        keys[:, :8] = np.arange(n, dtype=np.uint64).view(np.uint8).reshape(n, 8)
        frames = [B.broadcast_frame(0, bytes(((i * 131 + m) & 0xFF) for i in range(1024))) for m in range(M)]
        L = len(frames[0]); slot = (4 + L + 15) // 16 * 16; rec = (4 + L + 31) // 32 * 32
        eng = pkg.Engine(device=0, stream=stream.cuda_stream, max_conns=n, max_topics=256, max_keys=n + 4096, max_key_len=32,
                         ring_bytes_per_conn=16 * rec, max_batch_msgs=64, max_batch_bcast=16, max_batch_bytes=1 << 20,
                         max_batch_deliveries=M * n + 1024, batch_slots=4, pack_variant=args.variant)
        eng.add_users_bulk(keys, 32, np.zeros(n, dtype=np.uint16), np.arange(n + 1, dtype=np.uint32))
        arena = np.zeros(M * slot + 64, dtype=np.uint8)
        for m, fr in enumerate(frames):
            arena[m * slot + 4:m * slot + 4 + L] = np.frombuffer(fr, dtype=np.uint8)
        db = DeviceBatch(pkg, torch, dev, arena, np.full(M, 4), np.zeros(M), np.arange(M) * (slot // 16), np.full(M, L), np.arange(M),
                         np.ones(M), np.zeros(M), np.arange(M))
        kb = [keys[i].tobytes() for i in range(4096)]
        res = {}
        for churn in (False, True):
            it = 0
            def step():
                nonlocal it
                if churn:
                    base = (it * 50) % 4000
                    for q in range(40):
                        k = kb[base + q]
                        (eng.unsubscribe_user_from if it & 1 else eng.subscribe_user_to)(k, [0])
                    for q in range(40, 50):
                        k = kb[base + q]
                        eng.remove_user(k)
                        eng.add_user(k, [0])
                it += 1
                b = eng.submit_device(db.db)
                eng.release_batch(b)
            with torch.cuda.stream(stream):
                for _ in range(4):
                    step()
                torch.cuda.synchronize(dev)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0 = time.perf_counter()
                e0.record(stream)
                for _ in range(args.steps * 2):
                    step()
                e1.record(stream)
                torch.cuda.synchronize(dev)
                t1 = time.perf_counter()
            ms = e0.elapsed_time(e1) / (args.steps * 2)
            res["churn" if churn else "steady"] = {"ms_per_step": ms, "GBps": M * n * (4 + L) / ms / 1e6, "wall_ms_per_step": (t1 - t0) * 1e3 / (args.steps * 2)}
        print(json.dumps({"metric": "C2 with table churn between batches (40 (un)subscribes + 10 disconnect/connect per step)", **res}), flush=True)
        eng.close()
        return

    if wl == "C4":
        n, klen, K = 1 << 20, 128, 512
        rng = np.random.default_rng(6)
        keys = rng.integers(0, 256, size=(n, klen), dtype=np.uint8)
        keys[:, :8] = np.arange(n, dtype=np.uint64).view(np.uint8).reshape(n, 8)  # distinct
        tmpl, roff, poff = direct_frame_template(klen, K)
        L = len(tmpl); slot = (4 + L + 15) // 16 * 16
        M = n
        eng = pkg.Engine(device=0, stream=stream.cuda_stream, max_conns=n, max_topics=16, max_keys=n, max_key_len=klen,
                         ring_bytes_per_conn=16384, max_batch_msgs=M, max_batch_bcast=1, max_batch_bytes=M * slot + (1 << 16),
                         max_batch_deliveries=M + 1024, batch_slots=2, pack_variant=args.variant,
                         flags=pkg.FLAG_DEVICE_PARSE if args.ingest == "device" else 0)
        conns = eng.add_users_bulk(keys, klen)
        rcpt = rng.integers(0, n, size=M)
        arena = np.zeros((M, slot), dtype=np.uint8)
        arena[:, 4:4 + L] = np.frombuffer(tmpl, dtype=np.uint8)
        arena[:, 4 + roff:4 + roff + klen] = keys[rcpt]
        if args.hit < 1.0:
            miss = rng.random(M) >= args.hit
            arena[miss, 4 + roff + 8] ^= 0xFF  # unknown keys: must be dropped
        arena[:, 4 + poff:4 + poff + K] = rng.integers(0, 256, size=(1, K), dtype=np.uint8)
        idx = np.arange(M, dtype=np.int64)
        db = DeviceBatch(pkg, torch, dev, np.concatenate([arena.reshape(-1), np.zeros(64, np.uint8)]), np.full(M, 3), np.zeros(M),
                         idx * (slot // 16), np.full(M, L), idx * slot + 4 + roff, np.full(M, klen), np.zeros(1), np.zeros(0))
        expect_deliveries = None if args.hit < 1.0 else M
        alg_bytes = lambda d, bo: d * 0 + bo + M * L + M * (klen + 32)  # F per hit + L read + key compare + bucket sector
        desc = {"workload": "C4: direct path, 2^20 128-byte keys, uniform recipients, 512 B payloads, %d msgs per step" % M,
                "hit_rate": args.hit}
        F = 4 + L
    elif wl == "C3":
        n, T, M = 65536, 4096, (args.msgs or 128)
        rng = np.random.default_rng(3)
        p = zipf_p(T)
        keys = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
        keys[:, :8] = np.arange(n, dtype=np.uint64).view(np.uint8).reshape(n, 8)
        subs = np.stack([rng.choice(T, size=8, replace=False, p=p) for _ in range(n)]).astype(np.uint16)
        pool_kw = dict(flags=pkg.FLAG_OUTPUT_POOL, pool_bytes=int(args.pool * 1e9)) if args.pool else {}
        eng = pkg.Engine(device=0, stream=stream.cuda_stream, max_conns=n, max_topics=T, max_keys=n, max_key_len=32,
                         ring_bytes_per_conn=1 << 20, max_batch_msgs=M, max_batch_bcast=M, max_batch_bytes=max(16, M // 8) << 20,
                         max_batch_deliveries=min(M * n, 1 << 27), batch_slots=2, pack_variant=args.variant, **pool_kw)
        eng.add_users_bulk(keys, 32, subs.reshape(-1).copy(), (np.arange(n + 1) * 8).astype(np.uint32))
        rng4, rng5 = np.random.default_rng(4), np.random.default_rng(5)
        topics = rng4.choice(T, size=M, p=p)
        sizes = rng5.choice([256 << i for i in range(9)], size=M)
        frames = [bcast_frame_n(bytes([int(t) & 0xFF]), bytes(rng5.integers(0, 256, size=int(k), dtype=np.uint8))) for t, k in zip(topics, sizes)]
        offs, cur = [], 0
        for fr in frames:
            offs.append(cur); cur += (4 + len(fr) + 15) // 16 * 16
        arena = np.zeros(cur + 64, dtype=np.uint8)
        for o, fr in zip(offs, frames):
            arena[o + 4:o + 4 + len(fr)] = np.frombuffer(fr, dtype=np.uint8)
        lens = np.array([len(f) for f in frames])
        db = DeviceBatch(pkg, torch, dev, arena, np.full(M, 4), np.zeros(M), np.array(offs) // 16, lens, np.arange(M), np.ones(M),
                         topics.astype(np.int64), np.arange(M))
        per_topic = np.bincount(subs.reshape(-1), minlength=T)
        expect_deliveries = int(per_topic[topics].sum())
        alg_bytes = lambda d, bo: bo + int(lens.sum()) + M * (n // 8)
        desc = {"workload": "C3: 64 K subscribers, 4 K topics (extended ids) Zipf-0.99, 8 subscriptions each, payloads 256 B-64 KiB, %d msgs per step" % M,
                "output": ("shared output pool of %.0f GB (PCDN_FLAG_OUTPUT_POOL)" % args.pool) if args.pool else "per-connection rings of 1 MiB"}
        F = None
    else:
        n, K = 1 << 20, 4096
        dense = wl == "C5dense"
        M = 8 if dense else 64
        T = 1 if dense else 1024
        # N > 1: ONE sharded engine (pcdn_config.world_shards = N, this process drives shard `rank`);
        # every rank replays the same control plane over the whole population of N x 2^20 subscribers
        n_total = world * n
        rng = np.random.default_rng(7)
        keys = rng.integers(0, 256, size=(n_total, 32), dtype=np.uint8)
        keys[:, :8] = np.arange(n_total, dtype=np.uint64).view(np.uint8).reshape(n_total, 8)
        if dense:
            subs = np.zeros((n_total, 1), dtype=np.uint16)
        else:
            subs = np.stack([rng.permutation(T)[:4] for _ in range(1024)])[rng.integers(0, 1024, size=n_total)].astype(np.uint16)
        frames = [bcast_frame_n(bytes([m & 0xFF]), bytes(((i * 31 + m) & 0xFF) for i in range(K))) for m in range(M)]
        L = len(frames[0]); slot = (4 + L + 15) // 16 * 16; rec = (4 + L + 31) // 32 * 32
        shard_kw = {}
        if world > 1:
            uid = [pkg.nccl_unique_id() if rank == 0 else None]
            dist.broadcast_object_list(uid, src=0)
            shard_kw = dict(devices=[local], world_shards=world, first_shard=rank, nccl_unique_id=uid[0])
        eng = pkg.Engine(device=local, stream=stream.cuda_stream, max_conns=n, max_topics=max(T, 16), max_keys=n_total, max_key_len=32,
                         ring_bytes_per_conn=16 * rec, max_batch_msgs=M, max_batch_bcast=M, max_batch_bytes=4 << 20,
                         max_batch_deliveries=M * n if dense else 1 << 22, batch_slots=2, pack_variant=args.variant, **shard_kw)
        nsub = subs.shape[1]
        conn_ids = eng.add_users_bulk(keys, 32, subs.reshape(-1).copy(), (np.arange(n_total + 1) * nsub).astype(np.uint32))
        sd = eng.shard_info(0)
        mine = (conn_ids // sd.shard_stride) == rank          # the connections whose rings live on this GPU
        assert int(mine.sum()) == n == sd.n_conns and (world == 1 or sd.nccl_ranks == world)
        subs = subs[mine]
        topics = np.zeros(M, dtype=np.int64) if dense else np.random.default_rng(70).integers(0, T, size=M)  # same on all ranks
        arena = np.zeros(M * slot + 64, dtype=np.uint8)
        for m, fr in enumerate(frames):
            arena[m * slot + 4:m * slot + 4 + L] = np.frombuffer(fr, dtype=np.uint8)
        mk = lambda a: DeviceBatch(pkg, torch, dev, a, np.full(M, 4), np.zeros(M), np.arange(M) * (slot // 16), np.full(M, L),
                                   np.arange(M), np.ones(M), topics, np.arange(M))
        db = None
        # two ingest buffers alternate (the library's broadcast of step i+1 runs while step i's pack reads
        # the other one); ranks other than 0 hold zeros: what they fan out arrives over NVLink
        dbs = [mk(arena if rank == 0 else np.zeros_like(arena)) for _ in range(2)]
        per_topic = np.bincount(subs.reshape(-1), minlength=max(T, 1))
        expect_deliveries = int(per_topic[topics].sum())
        alg_bytes = lambda d, bo: bo + M * L + M * (n // 8)
        desc = {"workload": ("C5 shard, dense: 2^20 subscribers on 1 topic, 4 KiB broadcast, %d msgs per step" if dense else
                             "C5 shard, sparse: 2^20 subscribers, 1 K topics (extended ids), 4 uniform subscriptions each, 4 KiB broadcast, %d msgs per step") % M}
        F = 4 + L
    setup_s = time.time() - t_setup

    if args.ingest:
        # raw frames in pageable host memory → pcdn_receive_frames (tag peek or full parse + copy into
        # pinned staging) → flush (H2D + kernels) → poll (D2H) → release; wall clock per batch
        import ctypes as C
        assert wl == "C4"
        frames_np = np.ascontiguousarray(arena[:, 4:4 + L])
        fa = (pkg.Frame * M)()
        base = frames_np.ctypes.data
        sender = keys[0].tobytes()
        for i in range(M):
            fa[i].sender = sender; fa[i].sender_len = klen; fa[i].origin = 0
            fa[i].raw = C.cast(base + i * L, C.c_char_p); fa[i].raw_len = L
        times = []
        for it in range(2 + args.steps):
            t0 = time.perf_counter()
            rc = eng.L.pcdn_receive_frames(eng.h, fa, M, None)
            assert rc == M, rc
            t1 = time.perf_counter()
            b = eng.flush()
            res = eng.poll(b)
            assert res.n_deliveries == M and res.n_msg_errors == 0, (res.n_deliveries, res.n_msg_errors)
            eng.release_batch(b)
            torch.cuda.synchronize(dev)
            t2 = time.perf_counter()
            if it >= 2:
                times.append((t1 - t0, t2 - t0))
        rx = sum(t[0] for t in times) / len(times); tot = sum(t[1] for t in times) / len(times)
        print(json.dumps({"metric": "C4 ingest of raw frames from host memory (PCDN_INGEST_THREADS host threads)", "host_threads": int(os.environ.get("PCDN_INGEST_THREADS", min(16, os.cpu_count() or 1))), "ingest": args.ingest,
                          "msgs_per_s": M / tot, "egress_GBps": M * F / tot / 1e9, "host_receive_s_per_batch": rx,
                          "batch_s": tot, "msgs_per_batch": M, "host_ns_per_frame": rx / M * 1e9,
                          "h2d_bytes_per_step": M * slot, "d2h_bytes_per_step": 16 * M + M}), flush=True)
        eng.close()
        return

    prev = 0
    it = 0
    multi = wl in ("C5dense", "C5sparse")

    with torch.cuda.stream(stream):
        def step():
            nonlocal prev, it
            if prev and args.pool and wl == "C3" and M > 512:
                eng.release_batch(prev)          # the pool holds ONE such batch: its consumer must be done before the next fits
                prev = 0
            b = eng.submit_device((dbs[it & 1] if multi else db).db)   # N > 1: the library broadcasts it to every shard
            it += 1
            if prev:
                eng.release_batch(prev)
            prev = b

        def drain():
            nonlocal prev, it
            if prev:
                eng.release_batch(prev)
                prev = 0
            it = 0

        for _ in range(max(3, args.warmup)):
            step()
        drain()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize(dev)
        sampler = B.ClockSampler(local)
        sampler.start()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.steps):
            step()
        drain()
        e1.record(stream)
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize(dev)
        ms = e0.elapsed_time(e1)
        if world > 1:
            tm = torch.tensor([ms], dtype=torch.float64, device=dev)
            dist.all_reduce(tm, op=dist.ReduceOp.MAX)   # max over ranks
            ms = float(tm.item())
        # counters of one batch + per-stage device times
        eng.set_timing(True)
        s0 = eng.stats()
        res = None
        for _ in range(max(3, args.steps // 2)):
            b = eng.submit_device((dbs[0] if multi else db).db)
            res = eng.poll(b)
            d, bo, dropped, ovf, status = res.n_deliveries, res.bytes_out, res.n_direct_dropped, res.n_overflow, res.status
            eng.release_batch(b)
        s1 = eng.stats()
        clocks = sampler.stop()
    assert status == 0 and ovf == 0, (status, ovf)
    if expect_deliveries is not None:
        assert d == expect_deliveries, (d, expect_deliveries)
    nb = max(1, s1.timed_batches - s0.timed_batches)
    st = {k: (getattr(s1, k) - getattr(s0, k)) / nb for k in ("ms_direct", "ms_match", "ms_plan", "ms_pack")}
    peak, peak_src = B.measured_peak()
    step_s = ms * 1e-3 / args.steps
    ab = alg_bytes(d, bo)
    pack_bytes = bo + int((dbs[0] if multi else db).len.sum().item())
    bo_all, d_all = bo, d
    if world > 1:
        tot = torch.tensor([bo, d], dtype=torch.float64, device=dev)
        dist.all_reduce(tot, op=dist.ReduceOp.SUM)   # whole job = sum of the shards
        bo_all, d_all = float(tot[0].item()), float(tot[1].item())
        desc = dict(desc, parallelism="connection shards x%d (2^20 per GPU) behind one sharded engine; the library broadcasts each batch "
                                      "from rank 0's GPU with ncclBroadcast on its ingest stream (%d ranks)" % (world, sd.nccl_ranks))
        if rank != 0:
            eng.close()
            dist.barrier()
            dist.destroy_process_group()
            return
    line = {
        "metric": "fan-out egress GB/s; msgs/s and deliveries/s alongside (secondary config)", "value": bo_all / step_s / 1e9, "unit": "GB/s",
        "n_gpus": world, "scaling": "weak", "job_deliveries_per_s": d_all / step_s, "steps": args.steps, "warmup": max(3, args.warmup), "ms_per_step": ms / args.steps, "higher_is_better": True,
        "dtype": "u8", "data": "synthetic", "msgs_per_s": res.n_msgs / step_s, "deliveries_per_s": d / step_s,
        "deliveries_per_step": int(d), "direct_dropped_per_step": int(dropped),
        "algorithmic_GBps": ab / step_s / 1e9, "frac_of_hbm_peak": ab / step_s / 1e9 / peak,
        "config": dict(desc, setup_s=round(setup_s, 1), pack_variant=args.variant),
        "roofline": {"bound": "hbm", "kernel": "k_pack", "achieved": pack_bytes / (st["ms_pack"] * 1e-3) / 1e9 if st["ms_pack"] else None, "peak": peak, "unit": "GB/s",
                     "frac": pack_bytes / (st["ms_pack"] * 1e-3) / 1e9 / peak if st["ms_pack"] else None, "peak_source": peak_src, "stage_ms": st},
        "clocks": clocks,
        "verify": "engine counters == analytically expected deliveries (%d per step), no overflow, status 0" % int(d) if expect_deliveries is not None
                  else "engine counters consistent (hit rate < 1: dropped = %d), no overflow" % int(dropped),
    }
    print(json.dumps(line), flush=True)
    eng.close()
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
