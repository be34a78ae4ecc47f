"""push-cdn_b200 — H100 (sm_90a) fan-out engine for Push-CDN's cdn-broker hot path.

This Python module is a thin ctypes binding over the C ABI (``include/pcdn_fanout.h``) of
``libpcdn_fanout.so`` (CUDA, sm_90a).  It mirrors the names of the reference's broker API
(`Connections::*`, `Inner::handle_broadcast_message`, `Inner::handle_direct_message`,
`user_receive_loop` / `broker_receive_loop` — cdn-broker/src/{connections/mod.rs,
tasks/broker/handler.rs, tasks/user/handler.rs}) so that tests read like the reference's own.

There is no Python or CPU implementation of the data path here: if the shared library is missing or
no CUDA device is present, constructing a routing ``Engine`` raises.
(The directory name has a hyphen; import it through ``__graft_entry__.load_package()`` which
registers it as ``push_cdn_b200``.)
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
CSRC = os.path.join(_HERE, "csrc")
LIB_PATH = os.path.join(_HERE, "libpcdn_fanout.so")
INCLUDE = os.path.join(_ROOT, "include")

SOURCES = ["engine.cu", "kernels.cu", "egress.cu", "host_state.cpp", "frame_parse.cpp", "nccl_dl.cpp"]
HEADERS = ["kernels.cuh", "host_state.h", "frame_parse.h", "frame_parse_core.h", "hash.h", "nccl_dl.h", "engine_internal.h"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC,-pthread", "-shared",
]

KIND_DIRECT, KIND_BROADCAST, KIND_SUBSCRIBE, KIND_UNSUBSCRIBE = 3, 4, 5, 6
TO_USERS_ONLY = 1
FLAG_DEVICE_PARSE = 1
FLAG_HOST_RINGS = 4     # rings in mapped pinned host memory: spans are readable in place (egress hand-off)
FLAG_OUTPUT_POOL = 16   # one shared output pool per GPU instead of a ring per connection (spans: 32-byte units relative to pool_base)
FLAG_SPAN_RUNS = 8      # run-length span table (BatchResult.runs): consecutive connections with identical spans
FLAG_STAGED_SPANS = 2   # force the large-engine span path (table in HBM + D2H) on a small engine
FLAG_SHARED_PAYLOAD = 32  # every delivery is one 32-byte reference record; the payload exists once per batch (batch_payload)
FLAG_INBATCH_SUBSCRIBE = 64  # subscription changes become events of the open batch instead of launching it
REF_MARK = 0xFFFFFFFF     # first 4 bytes of a reference record
BATCH_READY = 1         # DeviceBatch.hints: the arrays are already complete in device memory
INGEST_NCCL, INGEST_HOST = 0, 1   # sharded engines: NCCL broadcast over NVLink | every shard copies from host
RECORD_ALIGN = 32
CONN_NONE = 0xFFFFFFFF

ERRORS = {
    -1: "PCDN_EINVAL", -2: "PCDN_ENOMEM", -3: "PCDN_ENODEV", -4: "PCDN_ECUDA", -5: "PCDN_ENOSPC",
    -6: "PCDN_EKEYLEN", -7: "PCDN_EPARSE", -8: "PCDN_EPRUNE", -9: "PCDN_EKIND", -10: "PCDN_ENOENT",
    -11: "PCDN_EAGAIN", -12: "PCDN_E2BIG", -13: "PCDN_EHOOK",
}


class PcdnError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"{ERRORS.get(code, code)}: {msg}")
        self.code = code


def needs_build() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, f) for f in SOURCES + HEADERS] + [os.path.join(INCLUDE, "pcdn_fanout.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile every CUDA source for sm_90a into the in-tree shared library (nvcc cross-compiles
    without a GPU)."""
    if not force and not needs_build():
        return LIB_PATH
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc):
        nvcc = "nvcc"
    cmd = [nvcc] + NVCC_FLAGS + ["-I", INCLUDE, "-o", LIB_PATH] + [os.path.join(CSRC, s) for s in SOURCES] + ["-ldl"]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    subprocess.check_call(cmd, cwd=CSRC)
    return LIB_PATH


class Config(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("device", C.c_int32), ("max_conns", C.c_uint32), ("max_topics", C.c_uint32),
        ("max_keys", C.c_uint32), ("max_key_len", C.c_uint32), ("ring_bytes_per_conn", C.c_uint64),
        ("max_batch_msgs", C.c_uint32), ("max_batch_bcast", C.c_uint32), ("max_batch_bytes", C.c_uint64),
        ("max_batch_deliveries", C.c_uint64), ("batch_slots", C.c_uint32), ("n_valid_topics", C.c_uint32),
        ("hash_seed", C.c_uint64), ("stream", C.c_void_p), ("identity", C.c_char_p), ("pack_variant", C.c_uint32),
        ("flags", C.c_uint32),
        ("n_devices", C.c_uint32), ("ingest", C.c_uint32), ("devices", C.POINTER(C.c_int32)),
        ("world_shards", C.c_uint32), ("first_shard", C.c_uint32), ("nccl_unique_id", C.c_void_p),
        ("pool_bytes", C.c_uint64), ("global_memory_pool_size", C.c_uint64), ("ref_min_bytes", C.c_uint32),
    ]


class Msg(C.Structure):
    _fields_ = [
        ("kind", C.c_uint8), ("flags", C.c_uint8), ("n_topics", C.c_uint16), ("topics", C.POINTER(C.c_uint16)),
        ("recipient", C.c_char_p), ("recipient_len", C.c_uint32), ("raw_len", C.c_uint32), ("raw", C.c_char_p),
    ]


class Span(C.Structure):
    _fields_ = [("conn", C.c_uint32), ("ring_off", C.c_uint32), ("len", C.c_uint32), ("n_records", C.c_uint32)]


class SpanRun(C.Structure):
    _fields_ = [("conn0", C.c_uint32), ("n_conns", C.c_uint32), ("ring_off", C.c_uint32), ("len", C.c_uint32),
                ("n_records", C.c_uint32), ("off_stride", C.c_uint32)]


class BatchResult(C.Structure):
    _fields_ = [
        ("batch_id", C.c_uint64), ("n_msgs", C.c_uint32), ("n_spans", C.c_uint32), ("spans", C.POINTER(Span)),
        ("n_deliveries", C.c_uint64), ("bytes_out", C.c_uint64), ("n_overflow", C.c_uint32),
        ("overflow_conns", C.POINTER(C.c_uint32)), ("n_direct_dropped", C.c_uint32), ("status", C.c_uint32),
        ("msg_status", C.POINTER(C.c_int8)), ("n_msg_errors", C.c_uint32), ("reserved", C.c_uint32),
        ("runs", C.POINTER(SpanRun)), ("n_runs", C.c_uint32), ("pool_base", C.c_uint32),
    ]


class DeviceBatch(C.Structure):
    _fields_ = [
        ("n_msgs", C.c_uint32), ("n_bcast", C.c_uint32), ("arena", C.c_void_p), ("arena_bytes", C.c_uint64),
        ("kind", C.c_void_p), ("flags", C.c_void_p), ("slot_off16", C.c_void_p), ("raw_len", C.c_void_p),
        ("aux_off", C.c_void_p), ("aux_len", C.c_void_p), ("topics", C.c_void_p), ("n_topics_total", C.c_uint32),
        ("bcast_index", C.c_void_p), ("hints", C.c_uint32), ("reserved", C.c_uint32),
    ]


class ShardDesc(C.Structure):
    _fields_ = [("global_index", C.c_uint32), ("device", C.c_int32), ("conn_base", C.c_uint32), ("shard_stride", C.c_uint32),
                ("rings_dev", C.c_void_p), ("rings_host", C.c_void_p), ("ring_bytes", C.c_uint64), ("n_conns", C.c_uint32),
                ("nccl_ranks", C.c_uint32)]


class EgressConfig(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("n_threads", C.c_uint32), ("chunk_bytes", C.c_uint64),
                ("backlog_bytes_per_conn", C.c_uint64), ("backlog_bytes_total", C.c_uint64)]


EGRESS_CONFIG_NO_BACKLOG_SIZE = EgressConfig.backlog_bytes_per_conn.offset   # struct_size of callers built before the backlog fields


class EgressChunk(C.Structure):
    _fields_ = [("local_shard", C.c_uint32), ("n_spans", C.c_uint32), ("spans", C.POINTER(Span)),
                ("data_off", C.POINTER(C.c_uint64)), ("data", C.c_void_p), ("bytes", C.c_uint64)]


EGRESS_SINK = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(EgressChunk))


class EgressStats(C.Structure):
    _fields_ = [("bytes", C.c_uint64), ("spans", C.c_uint64), ("chunks", C.c_uint64), ("records", C.c_uint64),
                ("fd_bytes", C.c_uint64), ("fd_writes", C.c_uint64), ("unattached_spans", C.c_uint64),
                ("failed_conns", C.c_uint64), ("seconds", C.c_double)]


class HookMessage(C.Structure):
    _fields_ = [("kind", C.c_uint8), ("origin", C.c_uint8), ("n_topics", C.c_uint16), ("topics", C.POINTER(C.c_uint8)),
                ("recipient", C.c_void_p), ("recipient_len", C.c_uint32), ("raw_len", C.c_uint32), ("raw", C.c_void_p),
                ("sender", C.c_void_p), ("sender_len", C.c_uint32), ("reserved", C.c_uint32)]


MESSAGE_HOOK = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(HookMessage))
HOOK_PROCESS, HOOK_SKIP = 0, 1


class Stats(C.Structure):
    _fields_ = [
        ("batches", C.c_uint64), ("msgs", C.c_uint64), ("deliveries", C.c_uint64), ("bytes_out", C.c_uint64),
        ("ms_match", C.c_double), ("ms_plan", C.c_double), ("ms_direct", C.c_double), ("ms_pack", C.c_double),
        ("ms_total", C.c_double), ("timed_batches", C.c_uint64), ("inflight_bytes", C.c_uint64),
        ("released_batches", C.c_uint64), ("latency_ms_sum", C.c_double), ("bytes_in", C.c_uint64),
        ("latency_hist_us", C.c_uint64 * 16), ("kernel_launches", C.c_uint64),
    ]


class Frame(C.Structure):
    _fields_ = [("sender", C.c_char_p), ("sender_len", C.c_uint32), ("origin", C.c_uint32), ("raw", C.c_char_p),
                ("raw_len", C.c_uint32), ("reserved", C.c_uint32)]


class TopicSyncEntry(C.Structure):
    _fields_ = [("topic", C.c_uint16), ("status", C.c_uint8), ("reserved", C.c_uint8 * 5), ("version", C.c_uint64)]


class UserSyncEntry(C.Structure):
    _fields_ = [("key", C.c_char_p), ("key_len", C.c_uint32), ("version", C.c_uint64), ("owner", C.c_char_p)]


class UserSyncEntryOut(C.Structure):
    """same layout, for READING entries the engine returns: `key` may contain NUL bytes, so it must
    stay a raw address (a c_char_p field would hand back a truncated temporary copy)"""
    _fields_ = [("key", C.c_void_p), ("key_len", C.c_uint32), ("version", C.c_uint64), ("owner", C.c_char_p)]


# every symbol include/pcdn_fanout.h declares: name → (restype, argtypes)
_vp, _u8p, _u16p, _u32, _u64, _ci, _cp = C.c_void_p, C.c_char_p, C.POINTER(C.c_uint16), C.c_uint32, C.c_uint64, C.c_int, C.c_char_p
ABI = {
    "pcdn_abi_version": (_u32, []),
    "pcdn_config_default": (None, [C.POINTER(Config)]),
    "pcdn_create": (_ci, [C.POINTER(Config), C.POINTER(_vp)]),
    "pcdn_destroy": (None, [_vp]),
    "pcdn_last_error": (_cp, []),
    "pcdn_add_user": (_ci, [_vp, _u8p, _u32, _u16p, _u32, C.POINTER(_u32)]),
    "pcdn_remove_user": (_ci, [_vp, _u8p, _u32]),
    "pcdn_subscribe_user_to": (_ci, [_vp, _u8p, _u32, _u16p, _u32]),
    "pcdn_unsubscribe_user_from": (_ci, [_vp, _u8p, _u32, _u16p, _u32]),
    "pcdn_add_broker": (_ci, [_vp, _cp, C.POINTER(_u32)]),
    "pcdn_remove_broker": (_ci, [_vp, _cp]),
    "pcdn_subscribe_broker_to": (_ci, [_vp, _cp, _u16p, _u32]),
    "pcdn_unsubscribe_broker_from": (_ci, [_vp, _cp, _u16p, _u32]),
    "pcdn_apply_user_sync": (_ci, [_vp, _cp, C.POINTER(UserSyncEntry), _u32]),
    "pcdn_get_user_sync": (_ci, [_vp, _ci, C.POINTER(C.POINTER(UserSyncEntry)), C.POINTER(_u32)]),
    "pcdn_apply_topic_sync": (_ci, [_vp, _cp, _u32, C.POINTER(TopicSyncEntry), _u32]),
    "pcdn_get_topic_sync": (_ci, [_vp, _ci, C.POINTER(C.POINTER(TopicSyncEntry)), C.POINTER(_u32)]),
    "pcdn_add_users_bulk": (_ci, [_vp, _vp, _u32, _u32, _u32, _vp, _vp, _vp]),
    "pcdn_handle_broadcast_message": (_ci, [_vp, _u16p, _u32, _u8p, _u32, _ci]),
    "pcdn_handle_direct_message": (_ci, [_vp, _u8p, _u32, _u8p, _u32, _ci]),
    "pcdn_send_to_broker": (_ci, [_vp, _cp, _u8p, _u32]),
    "pcdn_send_to_brokers": (_ci, [_vp, _u8p, _u32]),
    "pcdn_user_receive": (_ci, [_vp, _u8p, _u32, _u8p, _u32]),
    "pcdn_broker_receive": (_ci, [_vp, _cp, _u8p, _u32]),
    "pcdn_set_message_hook": (_ci, [_vp, _ci, MESSAGE_HOOK, _vp]),
    "pcdn_receive_frames": (_ci, [_vp, C.POINTER(Frame), _u32, C.POINTER(C.c_int32)]),
    "pcdn_flush": (_ci, [_vp, C.POINTER(_u64)]),
    "pcdn_submit": (_ci, [_vp, C.POINTER(Msg), _u32, C.POINTER(_u64)]),
    "pcdn_submit_device": (_ci, [_vp, C.POINTER(DeviceBatch), C.POINTER(_u64)]),
    "pcdn_next_batch": (_ci, [_vp, C.POINTER(_u64)]),
    "pcdn_poll": (_ci, [_vp, _u64, C.POINTER(BatchResult), _ci]),
    "pcdn_read": (_ci, [_vp, _u32, _u32, _u32, _vp]),
    "pcdn_batch_payload": (_ci, [_vp, _u64, C.POINTER(_vp)]),
    "pcdn_release_batch": (_ci, [_vp, _u64]),
    "pcdn_retry_batch": (_ci, [_vp, _u64]),
    "pcdn_nccl_unique_id": (_ci, [_vp]),
    "pcdn_num_shards": (_ci, [_vp, C.POINTER(_u32), C.POINTER(_u32)]),
    "pcdn_shard_info": (_ci, [_vp, _u32, C.POINTER(ShardDesc)]),
    "pcdn_poll_shard": (_ci, [_vp, _u64, _u32, C.POINTER(BatchResult), _ci]),
    "pcdn_egress_create": (_ci, [_vp, C.POINTER(EgressConfig), C.POINTER(_vp)]),
    "pcdn_egress_destroy": (None, [_vp]),
    "pcdn_egress_drain": (_ci, [_vp, _u64, EGRESS_SINK, _vp, C.POINTER(EgressStats)]),
    "pcdn_egress_attach": (_ci, [_vp, _u32, _ci]),
    "pcdn_egress_detach": (_ci, [_vp, _u32]),
    "pcdn_egress_write_batch": (_ci, [_vp, _u64, C.POINTER(EgressStats)]),
    "pcdn_egress_failed": (_ci, [_vp, C.POINTER(C.POINTER(_u32)), C.POINTER(_u32)]),
    "pcdn_egress_soft_close": (_ci, [_vp, _u32, C.POINTER(_ci)]),
    "pcdn_egress_flush_backlog": (_ci, [_vp, _ci, C.POINTER(_u32)]),
    "pcdn_egress_backlog": (_ci, [_vp, C.POINTER(C.POINTER(_u32)), C.POINTER(_u32), C.POINTER(_u64)]),
    "pcdn_get_stats": (_ci, [_vp, C.POINTER(Stats)]),
    "pcdn_set_timing": (_ci, [_vp, _ci]),
    "pcdn_ring_info": (_ci, [_vp, C.POINTER(_vp), C.POINTER(_u64), C.POINTER(_u32)]),
    "pcdn_host_rings": (_ci, [_vp, C.POINTER(_vp)]),
    "pcdn_num_users": (_ci, [_vp, C.POINTER(_u32), C.POINTER(_u32)]),
    "pcdn_debug_interested": (_ci, [_vp, _u16p, _u32, _ci, C.POINTER(_u32), _u32, C.POINTER(_u32)]),
    "pcdn_debug_route": (_ci, [_vp, _u8p, _u32, C.POINTER(_ci), C.POINTER(_u32)]),
    "pcdn_parse_frame": (_ci, [_u8p, _u32, _u16p, C.POINTER(_u32), C.POINTER(_u32), C.POINTER(_u32)]),
}

_lib = None


def lib() -> C.CDLL:
    """Load the CUDA extension.  Raises if it is missing — there is no fallback."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(the product has no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in ABI.items():
            f = getattr(L, name)
            f.restype = res
            f.argtypes = args
        assert L.pcdn_abi_version() == 2
        _lib = L
    return _lib


def nccl_unique_id() -> bytes:
    """a fresh 128-byte ncclUniqueId for multi-process sharded engines (one process makes it, all use it)"""
    buf = C.create_string_buffer(128)
    rc = lib().pcdn_nccl_unique_id(C.cast(buf, C.c_void_p))
    if rc < 0:
        raise PcdnError(rc, lib().pcdn_last_error().decode())
    return buf.raw


def _t16(topics: Iterable[int]):
    t = [int(x) for x in topics]
    return (C.c_uint16 * max(1, len(t)))(*t), len(t)


def parse_frame(raw: bytes):
    """pcdn_parse_frame → (kind, topics list, (field_off, field_len)) or raises PcdnError(EPARSE)."""
    L = lib()
    t = (C.c_uint16 * 256)()
    n, off, ln = C.c_uint32(0), C.c_uint32(0), C.c_uint32(0)
    k = L.pcdn_parse_frame(raw, len(raw), t, C.byref(n), C.byref(off), C.byref(ln))
    if k < 0:
        raise PcdnError(k, L.pcdn_last_error().decode())
    return k, [t[i] for i in range(n.value)], (off.value, ln.value)


class Engine:
    """One fan-out engine on one CUDA device (or a host-only state mirror with ``device=-1``)."""

    def __init__(self, device: int = 0, stream: Optional[int] = None, identity: str = "/",
                 devices: Optional[Sequence[int]] = None, nccl_unique_id: Optional[bytes] = None, **kw):
        """devices=[0, 1, ...]: one connection shard per listed GPU (the engine stays one logical
        broker); world_shards / first_shard / nccl_unique_id: multi-process groups (see the header).
        Any other keyword sets the pcdn_config field of that name, e.g. ref_min_bytes=16384: messages of
        at least that many raw bytes are delivered by reference, shorter ones as framed copies."""
        self.L = lib()
        cfg = Config()
        self.L.pcdn_config_default(C.byref(cfg))
        cfg.device = device
        self._identity = identity.encode()
        cfg.identity = self._identity
        if stream is not None:
            cfg.stream = stream
        if devices is not None:
            self._devices = (C.c_int32 * len(devices))(*devices)
            cfg.n_devices = len(devices)
            cfg.devices = self._devices
        if nccl_unique_id is not None:
            assert len(nccl_unique_id) == 128
            self._uid = C.create_string_buffer(nccl_unique_id, 128)
            cfg.nccl_unique_id = C.cast(self._uid, C.c_void_p)
        for k, v in kw.items():
            if not hasattr(cfg, k):
                raise TypeError(f"unknown config field {k}")
            setattr(cfg, k, v)
        self.cfg = cfg
        h = C.c_void_p()
        self._chk(self.L.pcdn_create(C.byref(cfg), C.byref(h)))
        self.h = h
        self._shards = None

    # ---- connection shards --------------------------------------------------------------------
    def num_shards(self) -> Tuple[int, int]:
        a, b = C.c_uint32(), C.c_uint32()
        self._chk(self.L.pcdn_num_shards(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def shard_info(self, local_shard: int) -> ShardDesc:
        d = ShardDesc()
        self._chk(self.L.pcdn_shard_info(self.h, local_shard, C.byref(d)))
        return d

    def shards(self) -> List[ShardDesc]:
        if self._shards is None:
            self._shards = [self.shard_info(i) for i in range(max(1, self.num_shards()[0]))]
        return self._shards

    def poll_shard(self, batch_id: int, local_shard: int, block: bool = True) -> Optional[BatchResult]:
        r = BatchResult()
        rc = self._chk(self.L.pcdn_poll_shard(self.h, batch_id, local_shard, C.byref(r), int(block)))
        return None if rc == 1 else r

    def close(self):
        if getattr(self, "h", None):
            self.L.pcdn_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _chk(self, rc: int) -> int:
        if rc < 0:
            raise PcdnError(rc, self.L.pcdn_last_error().decode())
        return rc

    # ---- state: Connections::* --------------------------------------------------------------
    def add_user(self, key: bytes, topics: Iterable[int] = ()) -> int:
        t, n = _t16(topics)
        c = C.c_uint32()
        self._chk(self.L.pcdn_add_user(self.h, key, len(key), t, n, C.byref(c)))
        return c.value

    def add_users_bulk(self, keys, key_len: int, topics=None, topic_offsets=None):
        """keys: numpy uint8 [n, stride] (C-contiguous); topics/topic_offsets: CSR numpy arrays."""
        import numpy as np

        n, stride = keys.shape
        out = np.empty(n, dtype=np.uint32)
        tp = topics.ctypes.data if topics is not None else None
        op = topic_offsets.ctypes.data if topic_offsets is not None else None
        self._chk(self.L.pcdn_add_users_bulk(self.h, keys.ctypes.data, key_len, stride, n, tp, op, out.ctypes.data))
        return out

    def remove_user(self, key: bytes) -> None:
        self._chk(self.L.pcdn_remove_user(self.h, key, len(key)))

    def subscribe_user_to(self, key: bytes, topics: Iterable[int]) -> None:
        t, n = _t16(topics)
        self._chk(self.L.pcdn_subscribe_user_to(self.h, key, len(key), t, n))

    def unsubscribe_user_from(self, key: bytes, topics: Iterable[int]) -> None:
        t, n = _t16(topics)
        self._chk(self.L.pcdn_unsubscribe_user_from(self.h, key, len(key), t, n))

    def add_broker(self, ident: str) -> int:
        c = C.c_uint32()
        self._chk(self.L.pcdn_add_broker(self.h, ident.encode(), C.byref(c)))
        return c.value

    def remove_broker(self, ident: str) -> None:
        self._chk(self.L.pcdn_remove_broker(self.h, ident.encode()))

    def subscribe_broker_to(self, ident: str, topics: Iterable[int]) -> None:
        t, n = _t16(topics)
        self._chk(self.L.pcdn_subscribe_broker_to(self.h, ident.encode(), t, n))

    def unsubscribe_broker_from(self, ident: str, topics: Iterable[int]) -> None:
        t, n = _t16(topics)
        self._chk(self.L.pcdn_unsubscribe_broker_from(self.h, ident.encode(), t, n))

    def apply_user_sync(self, remote_identity: str, entries) -> None:
        ents = list(entries)
        arr = (UserSyncEntry * max(1, len(ents)))()
        keep = []
        for i, (key, version, owner) in enumerate(ents):
            ob = None if owner is None else owner.encode()
            keep.append((key, ob))
            arr[i] = UserSyncEntry(key, len(key), version, ob)
        self._chk(self.L.pcdn_apply_user_sync(self.h, remote_identity.encode(), arr, len(ents)))

    # ---- inter-broker sync (Connections::get_*_sync / apply_topic_sync) ----------------------
    def get_user_sync(self, full: bool = False):
        """→ [(key, version, owner or None)] — full map or the diff since the last call"""
        p, n = C.POINTER(UserSyncEntry)(), C.c_uint32()
        self._chk(self.L.pcdn_get_user_sync(self.h, int(full), C.byref(p), C.byref(n)))
        q = C.cast(p, C.POINTER(UserSyncEntryOut))
        return [(C.string_at(q[i].key, q[i].key_len) if q[i].key_len else b"", q[i].version,
                 q[i].owner.decode() if q[i].owner is not None else None) for i in range(n.value)]

    def apply_topic_sync(self, ident: str, entries, remote_identity: int = 0) -> None:
        """entries: [(topic, status 0|1|2, version)] — a peer's TopicSyncMap (or its diff)"""
        ents = list(entries)
        arr = (TopicSyncEntry * max(1, len(ents)))()
        for i, (t, st, ver) in enumerate(ents):
            arr[i].topic, arr[i].status, arr[i].version = t, st, ver
        self._chk(self.L.pcdn_apply_topic_sync(self.h, ident.encode(), remote_identity, arr, len(ents)))

    def get_topic_sync(self, full: bool = False):
        p, n = C.POINTER(TopicSyncEntry)(), C.c_uint32()
        self._chk(self.L.pcdn_get_topic_sync(self.h, int(full), C.byref(p), C.byref(n)))
        return [(p[i].topic, p[i].status, p[i].version) for i in range(n.value)]

    # ---- data in ----------------------------------------------------------------------------
    def handle_broadcast_message(self, topics: Iterable[int], raw: bytes, to_users_only: bool = False) -> None:
        t, n = _t16(topics)
        self._chk(self.L.pcdn_handle_broadcast_message(self.h, t, n, raw, len(raw), int(to_users_only)))

    def handle_direct_message(self, recipient: bytes, raw: bytes, to_user_only: bool = False) -> None:
        self._chk(self.L.pcdn_handle_direct_message(self.h, recipient, len(recipient), raw, len(raw), int(to_user_only)))

    # ---- data out: the broker's own frames to its peer brokers (tasks/broker/sender.rs) --------
    def send_to_broker(self, ident: str, raw: bytes) -> int:
        """Inner::try_send_to_broker: `raw` (e.g. a UserSync or TopicSync frame, forwarded verbatim) to the
        peer broker `ident`, in order with the open batch's routed messages.  0 = appended, 1 = no such broker."""
        return self._chk(self.L.pcdn_send_to_broker(self.h, ident.encode(), raw, len(raw)))

    def send_to_brokers(self, raw: bytes) -> int:
        """Inner::try_send_to_brokers: `raw` to every connected peer broker.  0 = appended, 1 = no broker."""
        return self._chk(self.L.pcdn_send_to_brokers(self.h, raw, len(raw)))

    def set_message_hook(self, origin: int, fn) -> None:
        """MessageHookDef (cdn-proto/src/def.rs:79-92).  fn(msg: HookMessage) -> HOOK_PROCESS | HOOK_SKIP | negative
        (error: the receive call returns PCDN_EHOOK and the host disconnects the peer); None removes the hook."""
        if not hasattr(self, "_hooks"):
            self._hooks = {}
        if fn is None:
            self._chk(self.L.pcdn_set_message_hook(self.h, origin, C.cast(None, MESSAGE_HOOK), None))
            self._hooks.pop(origin, None)
            return
        cb = MESSAGE_HOOK(lambda _u, m: int(fn(m.contents)))
        self._hooks[origin] = cb   # keep the trampoline alive
        self._chk(self.L.pcdn_set_message_hook(self.h, origin, cb, None))

    def user_receive(self, sender_key: bytes, raw: bytes) -> int:
        """One iteration of user_receive_loop; negative = the loop would have ended (disconnect)."""
        return self.L.pcdn_user_receive(self.h, sender_key, len(sender_key), raw, len(raw))

    def broker_receive(self, ident: str, raw: bytes) -> int:
        return self.L.pcdn_broker_receive(self.h, ident.encode(), raw, len(raw))

    def receive_frames(self, frames: Sequence[Tuple[bytes, int, bytes]]) -> List[int]:
        """frames: (sender key, origin 0=user/1=broker, raw) → per-frame return codes"""
        n = len(frames)
        arr = (Frame * max(1, n))()
        for i, (sender, origin, raw) in enumerate(frames):
            arr[i] = Frame(sender, len(sender), origin, raw, len(raw), 0)
        rcs = (C.c_int32 * max(1, n))()
        done = self._chk(self.L.pcdn_receive_frames(self.h, arr, n, rcs))
        if done != n:
            raise PcdnError(-11, f"only {done} of {n} frames consumed: drain a batch and resubmit the rest")
        return [rcs[i] for i in range(n)]

    def receive_frames_all(self, frames: Sequence[Tuple[bytes, int, bytes]]):
        """like receive_frames, but when the engine stops early (all batch slots in flight, memory
        pool exhausted) it drains the outstanding batches and resumes — the loop a broker's ingest
        task runs.  Returns (per-frame return codes, {conn: delivered frames})."""
        n = len(frames)
        arr = (Frame * max(1, n))()
        for i, (sender, origin, raw) in enumerate(frames):
            arr[i] = Frame(sender, len(sender), origin, raw, len(raw), 0)
        rcs = (C.c_int32 * max(1, n))()
        out: Dict[int, List[bytes]] = {}
        pos = 0
        while pos < n:
            done = self.L.pcdn_receive_frames(self.h, C.cast(C.byref(arr, pos * C.sizeof(Frame)), C.POINTER(Frame)), n - pos,
                                              C.cast(C.byref(rcs, pos * 4), C.POINTER(C.c_int32)))
            if done < 0 and done != -11:
                self._chk(done)
            pos += max(done, 0)
            if pos < n:
                for conn, fr in self.drain().items():
                    out.setdefault(conn, []).extend(fr)
        for conn, fr in self.drain().items():
            out.setdefault(conn, []).extend(fr)
        return [rcs[i] for i in range(n)], out

    def flush(self) -> int:
        b = C.c_uint64(0)
        self._chk(self.L.pcdn_flush(self.h, C.byref(b)))
        return b.value

    def submit(self, msgs: Sequence[Tuple]) -> int:
        """msgs: ('b', topics, raw, to_users_only) | ('d', recipient, raw, to_user_only)"""
        arr = (Msg * max(1, len(msgs)))()
        keep = []
        for i, m in enumerate(msgs):
            if m[0] == "b":
                t, n = _t16(m[1])
                keep.append(t)
                arr[i] = Msg(KIND_BROADCAST, TO_USERS_ONLY if m[3] else 0, n, t, None, 0, len(m[2]), m[2])
            else:
                arr[i] = Msg(KIND_DIRECT, TO_USERS_ONLY if m[3] else 0, 0, None, m[1], len(m[1]), len(m[2]), m[2])
        b = C.c_uint64(0)
        self._chk(self.L.pcdn_submit(self.h, arr, len(msgs), C.byref(b)))
        return b.value

    def submit_device(self, db: DeviceBatch) -> int:
        b = C.c_uint64(0)
        self._chk(self.L.pcdn_submit_device(self.h, C.byref(db), C.byref(b)))
        return b.value

    # ---- data out ---------------------------------------------------------------------------
    def next_batch(self) -> int:
        b = C.c_uint64(0)
        self._chk(self.L.pcdn_next_batch(self.h, C.byref(b)))
        return b.value

    def poll(self, batch_id: int, block: bool = True) -> Optional[BatchResult]:
        r = BatchResult()
        rc = self._chk(self.L.pcdn_poll(self.h, batch_id, C.byref(r), int(block)))
        return None if rc == 1 else r

    def read(self, conn: int, ring_off: int, length: int) -> bytes:
        buf = C.create_string_buffer(max(1, length))
        self._chk(self.L.pcdn_read(self.h, conn, ring_off, length, C.cast(buf, C.c_void_p)))
        return buf.raw[:length]

    def delivers_by_ref(self) -> bool:
        """some deliveries are reference records (FLAG_SHARED_PAYLOAD, or a ref_min_bytes threshold)"""
        return bool(self.cfg.flags & FLAG_SHARED_PAYLOAD) or self.cfg.ref_min_bytes > 0

    def batch_payload(self, batch_id: int) -> int:
        """host address of the batch's frames (pinned, valid until release): a reference record's raw
        bytes are at this address + the record's offset"""
        p = C.c_void_p()
        self._chk(self.L.pcdn_batch_payload(self.h, batch_id, C.byref(p)))
        return p.value or 0

    def release_batch(self, batch_id: int) -> None:
        self._chk(self.L.pcdn_release_batch(self.h, batch_id))

    def retry_batch(self, batch_id: int) -> None:
        """output-pool engines: run a batch again that was refused for space (status PCDN_EAGAIN)"""
        self._chk(self.L.pcdn_retry_batch(self.h, batch_id))

    def spans(self, res: BatchResult) -> List[Tuple[int, int, int, int]]:
        """(conn, ring_off, len, n_records) per span; a run-length table (FLAG_SPAN_RUNS) is expanded"""
        if res.runs:
            out = []
            for i in range(res.n_runs):
                r = res.runs[i]
                out.extend((r.conn0 + k, r.ring_off + k * r.off_stride, r.len, r.n_records) for k in range(r.n_conns))
            assert len(out) == res.n_spans, (len(out), res.n_spans)
            return out
        return [(res.spans[i].conn, res.spans[i].ring_off, res.spans[i].len, res.spans[i].n_records)
                for i in range(res.n_spans)]

    def collect_frames(self, res: BatchResult) -> Dict[int, List[bytes]]:
        """What the per-connection writer tasks would put on the wire for this batch: walk every
        span record by record (BE length prefix, 32-byte record stride; a reference record of a
        FLAG_SHARED_PAYLOAD or ref_min_bytes engine is resolved through batch_payload) and return the raw frames
        per connection in ring order.  A wrapped connection has two spans: the one that does not
        start at offset 0 comes first."""
        per: Dict[int, List[Tuple[int, int, int]]] = {}
        sh = self.shards()
        stride, rbytes = sh[0].shard_stride, sh[0].ring_bytes
        hosts = {d.global_index: d.rings_host for d in sh if d.rings_host}
        pool = bool(self.cfg.flags & FLAG_OUTPUT_POOL)   # offsets: 32-byte units relative to res.pool_base
        # engines that deliver by reference: reference records point into the batch's payload
        payload = self.batch_payload(res.batch_id) if self.delivers_by_ref() else 0
        for conn, off, ln, nrec in self.spans(res):
            per.setdefault(conn, []).append((off, ln, nrec))
        out: Dict[int, List[bytes]] = {}
        for conn, pieces in per.items():
            two = len(pieces) > 1  # (a list is empty while it is being sorted: take the length first)
            pieces.sort(key=lambda p: (p[0] == 0 and two, p[0]))
            frames = []
            for off, ln, nrec in pieces:
                # host rings: the bytes are read in place, exactly what a socket writer would do
                hb = hosts.get(conn // stride)
                if pool:
                    unit = res.pool_base + off
                    data = C.string_at(hb + unit * RECORD_ALIGN, ln) if hb else self.read(conn, unit, ln)
                else:
                    data = C.string_at(hb + (conn % stride) * rbytes + off, ln) if hb else self.read(conn, off, ln)
                p = 0
                for _ in range(nrec):
                    L = int.from_bytes(data[p:p + 4], "big")
                    if payload and L == REF_MARK:
                        L = int.from_bytes(data[p + 4:p + 8], "big")
                        assert int.from_bytes(data[p + 16:p + 24], "little") == res.batch_id, (conn, p)
                        frames.append(C.string_at(payload + int.from_bytes(data[p + 8:p + 16], "little"), L))
                        p += RECORD_ALIGN
                        continue
                    frames.append(data[p + 4:p + 4 + L])
                    p += (4 + L + RECORD_ALIGN - 1) // RECORD_ALIGN * RECORD_ALIGN
                assert p == ln, (conn, off, ln, nrec, p)
            out[conn] = frames
        return out

    def drain(self) -> Dict[int, List[bytes]]:
        """flush, then poll + collect + release every outstanding batch (oldest first)."""
        self.flush()
        out: Dict[int, List[bytes]] = {}
        while True:
            b = self.next_batch()
            if not b:
                return out
            res = self.poll(b)
            if res.status == 11:      # PCDN_EAGAIN: refused for space in the output pool; everything older is released by now
                self.retry_batch(b)
                res = self.poll(b)
            if res.status:
                self.release_batch(b)
                raise PcdnError(-int(res.status), "batch rejected on the device")
            for conn, fr in self.collect_frames(res).items():
                out.setdefault(conn, []).extend(fr)
            self.last_result = res
            self.release_batch(b)

    # ---- introspection ----------------------------------------------------------------------
    def stats(self) -> Stats:
        s = Stats()
        self._chk(self.L.pcdn_get_stats(self.h, C.byref(s)))
        return s

    def set_timing(self, on: bool) -> None:
        self._chk(self.L.pcdn_set_timing(self.h, int(on)))

    def ring_info(self) -> Tuple[int, int, int]:
        p, rb, mc = C.c_void_p(), C.c_uint64(), C.c_uint32()
        self._chk(self.L.pcdn_ring_info(self.h, C.byref(p), C.byref(rb), C.byref(mc)))
        return (p.value or 0), rb.value, mc.value

    def host_rings(self) -> int:
        """host address of the rings (FLAG_HOST_RINGS engines), else 0"""
        p = C.c_void_p()
        rc = self.L.pcdn_host_rings(self.h, C.byref(p))
        return (p.value or 0) if rc == 0 else 0

    def num_users(self) -> Tuple[int, int]:
        u, b = C.c_uint32(), C.c_uint32()
        self._chk(self.L.pcdn_num_users(self.h, C.byref(u), C.byref(b)))
        return u.value, b.value

    def debug_interested(self, topics: Iterable[int], to_users_only: bool = False) -> List[int]:
        t, n = _t16(topics)
        cap = self.shard_info(0).shard_stride * max(1, self.num_shards()[1])  # the whole id space (all shards)
        out = (C.c_uint32 * cap)()
        k = C.c_uint32()
        self._chk(self.L.pcdn_debug_interested(self.h, t, n, int(to_users_only), out, cap, C.byref(k)))
        return sorted(out[i] for i in range(min(k.value, cap)))

    def debug_route(self, key: bytes) -> Tuple[int, int]:
        kind, conn = C.c_int(), C.c_uint32()
        self._chk(self.L.pcdn_debug_route(self.h, key, len(key), C.byref(kind), C.byref(conn)))
        return kind.value, (-1 if conn.value == CONN_NONE else conn.value)


class Egress:
    """The consumer of span tables (pcdn_egress_*): drains a batch's framed records into host memory
    chunk by chunk and hands them to a sink — a Python callback, or the built-in writev sink that
    writes every connection's records to the file descriptor attached to it.  With a backlog budget
    (``backlog_bytes_per_conn`` / ``backlog_bytes_total``) that writer never waits for a slow peer:
    what the peer does not take is kept in host memory and written by ``flush_backlog``."""

    def __init__(self, engine: Engine, n_threads: int = 0, chunk_bytes: int = 0,
                 backlog_bytes_per_conn: int = 0, backlog_bytes_total: int = 0,
                 struct_size: Optional[int] = None):
        self.e, self.L = engine, engine.L
        cfg = EgressConfig(C.sizeof(EgressConfig) if struct_size is None else struct_size, n_threads, chunk_bytes,
                           backlog_bytes_per_conn, backlog_bytes_total)
        h = C.c_void_p()
        engine._chk(self.L.pcdn_egress_create(engine.h, C.byref(cfg), C.byref(h)))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.L.pcdn_egress_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def attach(self, conn: int, fd: int) -> None:
        self.e._chk(self.L.pcdn_egress_attach(self.h, conn, fd))

    def detach(self, conn: int) -> None:
        self.e._chk(self.L.pcdn_egress_detach(self.h, conn))

    def drain(self, batch_id: int, sink=None) -> EgressStats:
        """sink(chunk: EgressChunk) -> None, called once per chunk; None only stages the bytes"""
        st = EgressStats()
        err = []

        def tramp(_user, chunk):
            try:
                sink(chunk.contents)
                return 0
            except BaseException as ex:  # never unwind through the C frames
                err.append(ex)
                return 1

        cb = EGRESS_SINK(tramp) if sink is not None else C.cast(None, EGRESS_SINK)
        rc = self.L.pcdn_egress_drain(self.h, batch_id, cb, None, C.byref(st))
        if err:
            raise err[0]
        self.e._chk(rc)
        return st

    def write_batch(self, batch_id: int) -> EgressStats:
        st = EgressStats()
        self.e._chk(self.L.pcdn_egress_write_batch(self.h, batch_id, C.byref(st)))
        return st

    def failed(self) -> List[int]:
        p, n = C.POINTER(C.c_uint32)(), C.c_uint32()
        self.e._chk(self.L.pcdn_egress_failed(self.h, C.byref(p), C.byref(n)))
        return [p[i] for i in range(n.value)]

    def soft_close(self, conn: int) -> int:
        fd = C.c_int(-1)
        self.e._chk(self.L.pcdn_egress_soft_close(self.h, conn, C.byref(fd)))
        return fd.value

    def flush_backlog(self, timeout_ms: int = 0) -> int:
        """write what the backlogged descriptors accept (waiting up to timeout_ms; 0 = one pass, < 0 =
        until all are written or failed); returns the number of connections still backlogged"""
        n = C.c_uint32()
        self.e._chk(self.L.pcdn_egress_flush_backlog(self.h, timeout_ms, C.byref(n)))
        return n.value

    def backlog(self) -> Tuple[List[int], int]:
        """(connections with a backlog, bytes of all backlogs)"""
        p, n, b = C.POINTER(C.c_uint32)(), C.c_uint32(), C.c_uint64()
        self.e._chk(self.L.pcdn_egress_backlog(self.h, C.byref(p), C.byref(n), C.byref(b)))
        return [p[i] for i in range(n.value)], b.value
