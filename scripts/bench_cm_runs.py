#!/usr/bin/env python
"""Where a C2 step goes besides the pack: stage times and step time of the bench.py C2 engine on one GPU.

    python scripts/bench_cm_runs.py [--steps K] [--reps R] [--out FILE]

The engine, the batch and the loop are bench.py's C2 (2^20 subscribers on one topic, 8 x 1 KiB broadcasts per
batch resident in HBM, run-length span table, batch n released right after it is submitted).  In one process:
  step     ms per step with timing off (CUDA events around K steps), R repetitions, median and range;
  stages   with set_timing(True): match, plan_offsets (k_plan + k_offsets) and pack, each the median of R
           repetitions of K batches (every batch polled, so the stages of one batch are not overlapped by another);
  between  step - (match + plan_offsets + pack): what a step spends outside the three stages (counter zeroing and
           copies, k_release, launch gaps).
The card's name, power limit and max SM clock are read in the same run.  Prints one JSON object; with --out also
writes it there.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import __graft_entry__ as ge  # noqa: E402
from bench import KEY_LEN, MSGS_PER_STEP, N_CONNS, PAYLOAD, RING_RECORDS, broadcast_frame  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=60)
    return q.stdout.strip()


def c2_engine(pkg, stream):
    """bench.py's C2 engine (rings, run-length spans) with every user subscribed to topic 0"""
    N, M = N_CONNS, MSGS_PER_STEP
    frames = [broadcast_frame(0, bytes(((i * 131 + m * 7 + 1) & 0xFF) for i in range(PAYLOAD))) for m in range(M)]
    L = len(frames[0]); F = 4 + L
    rec = (F + 31) // 32 * 32
    eng = pkg.Engine(device=0, stream=stream.cuda_stream, max_conns=N, max_topics=256, max_keys=N, max_key_len=KEY_LEN,
                     ring_bytes_per_conn=RING_RECORDS * rec, max_batch_msgs=max(64, M), max_batch_bcast=max(16, M),
                     max_batch_bytes=max(1 << 20, 4 * M * (rec + 64)), max_batch_deliveries=M * N + 1024, batch_slots=4,
                     flags=pkg.FLAG_SPAN_RUNS)
    rng = np.random.default_rng(2)
    keys = rng.integers(0, 256, size=(N, KEY_LEN), dtype=np.uint8)
    keys[:, :8] = np.arange(N, dtype=np.uint64).view(np.uint8).reshape(N, 8)
    eng.add_users_bulk(keys, KEY_LEN, np.zeros(N, dtype=np.uint16), np.arange(N + 1, dtype=np.uint32))
    return eng, frames, F


def device_batches(pkg, frames, dev, stream):
    """two device-resident copies of the batch, alternated step by step as bench.py does"""
    M, L = len(frames), len(frames[0])
    slot = (4 + L + 15) // 16 * 16
    arena = np.zeros(M * slot + 64, dtype=np.uint8)
    for m, fr in enumerate(frames):
        arena[m * slot + 4:m * slot + 4 + L] = np.frombuffer(fr, dtype=np.uint8)
    with torch.cuda.stream(stream):
        t = dict(kind=torch.full((M,), 4, dtype=torch.uint8, device=dev), flags=torch.zeros(M, dtype=torch.uint8, device=dev),
                 slot=(torch.arange(M, device=dev) * (slot // 16)).to(torch.int32),
                 len=torch.full((M,), L, dtype=torch.int32, device=dev), aoff=torch.arange(M, dtype=torch.int32, device=dev),
                 alen=torch.ones(M, dtype=torch.int32, device=dev), topics=torch.zeros(M, dtype=torch.int16, device=dev),
                 bidx=torch.arange(M, dtype=torch.int32, device=dev))
        t["arenas"] = [torch.from_numpy(arena).to(dev) for _ in range(2)]
    torch.cuda.synchronize(dev)
    dbs = []
    for a in t["arenas"]:
        db = pkg.DeviceBatch(M, M, a.data_ptr(), a.numel(), t["kind"].data_ptr(), t["flags"].data_ptr(), t["slot"].data_ptr(),
                             t["len"].data_ptr(), t["aoff"].data_ptr(), t["alen"].data_ptr(), t["topics"].data_ptr(), M,
                             t["bidx"].data_ptr())
        db.hints = pkg.BATCH_READY
        dbs.append(db)
    return dbs, t


def time_steps(eng, dbs, stream, steps):
    """ms per step of the bench.py loop (submit_device, then release), CUDA events on the engine's stream"""
    with torch.cuda.stream(stream):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for i in range(steps):
            eng.release_batch(eng.submit_device(dbs[i & 1]))
        e1.record(stream)
        e1.synchronize()
    return e0.elapsed_time(e1) / steps


def stage_times(eng, dbs, stream, steps):
    eng.set_timing(True)
    s0 = eng.stats()
    with torch.cuda.stream(stream):
        for i in range(steps):
            b = eng.submit_device(dbs[i & 1])
            r = eng.poll(b)
            assert r.status == 0 and r.n_overflow == 0
            eng.release_batch(b)
    s1 = eng.stats()
    eng.set_timing(False)
    n = max(1, s1.timed_batches - s0.timed_batches)
    return {"match": (s1.ms_match - s0.ms_match) / n, "plan_offsets": (s1.ms_plan - s0.ms_plan) / n,
            "pack": (s1.ms_pack - s0.ms_pack) / n}


def spread(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "all": xs}


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
    eng, frames, F = c2_engine(pkg, stream)
    dbs, keep = device_batches(pkg, frames, dev, stream)
    time_steps(eng, dbs, stream, 5)
    stage_times(eng, dbs, stream, 3)
    steps, stages = [], {"match": [], "plan_offsets": [], "pack": []}
    for _ in range(args.reps):       # step time and stage times alternated
        steps.append(time_steps(eng, dbs, stream, args.steps))
        for k, v in stage_times(eng, dbs, stream, args.steps).items():
            stages[k].append(v)
    eng.close()
    step = statistics.median(steps)
    med = {k: statistics.median(v) for k, v in stages.items()}
    between = step - sum(med.values())
    res.update({
        "shape": "C2: %d subscribers, %d x %d B broadcasts per batch, rings, run-length spans" % (N_CONNS, MSGS_PER_STEP, PAYLOAD),
        "steps_per_rep": args.steps, "reps": args.reps,
        "step_ms": spread(steps), "stage_ms": {k: spread(v) for k, v in stages.items()},
        "between_ms": between,
        "plan_offsets_plus_between_pct_of_step": 100.0 * (med["plan_offsets"] + between) / step,
        "wire_gbs": MSGS_PER_STEP * N_CONNS * F / (step * 1e-3) / 1e9,
        "card_after": card()})
    s = json.dumps(res)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
