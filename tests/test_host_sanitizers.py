"""The host side of the engine (frame parser — the same source the device parse kernel compiles —,
table mirror, cuckoo table) built with AddressSanitizer + UndefinedBehaviorSanitizer and driven by a
mutation fuzzer / random operation sequences (tests/cpp/host_fuzz.cpp).  No GPU, no CUDA."""
import os
import random
import shutil
import struct
import subprocess

import pytest

from oracle import oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "push-cdn_b200", "csrc")


@pytest.mark.skipif(shutil.which("g++") is None, reason="g++ not available")
def test_host_code_under_asan_ubsan(tmp_path):
    exe = tmp_path / "host_fuzz"
    cmd = ["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined",
           "-fno-omit-frame-pointer", "-I", os.path.join(ROOT, "include"), "-I", CSRC,
           os.path.join(ROOT, "tests", "cpp", "host_fuzz.cpp"), os.path.join(CSRC, "host_state.cpp"),
           os.path.join(CSRC, "frame_parse.cpp"), "-o", str(exe)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    # seed corpus: every routed kind, field sizes around the word / segment boundaries, 2-segment frames
    rng = random.Random(5)
    seeds = []
    for kind in (3, 4, 5, 6, 7, 8):
        for f0n in (0, 1, 7, 8, 9, 128):
            for pn in (0, 1, 8, 100, 9000):
                f0 = bytes(rng.randrange(256) for _ in range(f0n))
                pl = bytes(rng.randrange(256) for _ in range(pn))
                if kind in (5, 6):
                    seeds.append(orc.serialize(kind, f0))
                elif kind in (7, 8):
                    seeds.append(orc.serialize(kind, b"", pl))
                else:
                    seeds.append(orc.serialize(kind, f0, pl))
    corpus = tmp_path / "seeds.bin"
    with open(corpus, "wb") as f:
        for s in seeds:
            f.write(struct.pack("<I", len(s)) + s)
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=0", UBSAN_OPTIONS="print_stacktrace=1")
    r = subprocess.run([str(exe), str(corpus), "120000", "7"], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, (r.stdout + r.stderr)[-6000:]
    assert "host_fuzz ok" in r.stdout


@pytest.mark.skipif(shutil.which("nvcc") is None, reason="nvcc not available")
def test_state_calls_under_tsan(tmp_path):
    """SURVEY 8b threading contract: state calls and lookups from many host threads.  The library is
    rebuilt with ThreadSanitizer (host code of engine.cu / kernels.cu included) and a C driver runs
    8 threads x 20 000 calls against a host-only engine; any data race report fails the test."""
    exe = tmp_path / "tsan_state_calls"
    srcs = [os.path.join(CSRC, f) for f in ("engine.cu", "kernels.cu", "egress.cu", "host_state.cpp", "frame_parse.cpp", "nccl_dl.cpp")]
    cmd = ["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-g", "-std=c++17",
           "-Xcompiler", "-fPIC,-pthread,-fsanitize=thread", "-I", os.path.join(ROOT, "include"), *srcs,
           os.path.join(ROOT, "tests", "cpp", "tsan_state_calls.c"), "-o", str(exe), "-lpthread", "-ltsan", "-ldl"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0 and "tsan" in r.stderr.lower():
        pytest.skip("libtsan not available: " + r.stderr[-300:])
    assert r.returncode == 0, r.stderr[-4000:]
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=0:exitcode=66")
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=900, env=env)
    assert "ThreadSanitizer" not in r.stderr, r.stderr[-6000:]
    assert r.returncode == 0 and "tsan driver ok" in r.stdout, (r.stdout + r.stderr)[-3000:]
