/*
 * pcdn_fanout.h — C ABI of the broker fan-out engine (CUDA, H100 / sm_90a).
 *
 * This is the drop-in boundary for ONE hot path of EspressoSystems/Push-CDN: cdn-broker's
 * broadcast + direct-message routing and per-recipient replication with the cdn-proto
 * `u32 big-endian length ‖ raw bytes` framing fused in.  The reference (100 % safe Rust, no FFI)
 * has no plugin interface; the seam is cut where SURVEY.md §8(b) puts it.  Every entry point
 * below names the reference function it replaces (paths relative to the reference repo root).
 *
 * Threading: all calls on one engine are serialised internally by a mutex (mirrors the single
 * `parking_lot::RwLock<Connections>` of cdn-broker/src/lib.rs:98).  State calls issued before a
 * flush/submit are visible to that batch, later ones are not (R12, SURVEY Appendix A).
 *
 * Errors: every function returns 0 (PCDN_OK) or a negative PCDN_E* code; a human-readable message
 * for the calling thread is available from pcdn_last_error().  Nothing throws or aborts across
 * the ABI.  Unknown recipient / no subscribers is success with 0 deliveries (reference:
 * cdn-broker/src/tasks/broker/handler.rs:210 silently drops).
 *
 * There is NO CPU data path behind this ABI: with `device < 0` the engine is a host-only state
 * mirror (used by CPU unit tests of the table logic) and every data call fails with PCDN_ENODEV.
 *
 * Several GPUs (SURVEY 8e): ONE engine can spread its connections over the GPUs of a box
 * (pcdn_config.n_devices / devices).  Every state and data-in call below is unchanged — the engine
 * is still one logical broker with one connection-id space — and the library itself replicates
 * each batch to all GPUs (one ncclBroadcast over NVLink per batch, issued by the library on a side
 * stream) and lets every GPU fan out to its own connection shard.  The reference analogue is the
 * broker -> peer-broker forward with to_users_only (cdn-broker/src/tasks/broker/handler.rs:156-160,
 * 262-271): a message crosses once, each shard delivers to its own users.
 */
#ifndef PCDN_FANOUT_H
#define PCDN_FANOUT_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PCDN_ABI_VERSION 2u

/* ---- status codes ------------------------------------------------------------------------- */
enum {
  PCDN_OK = 0,
  PCDN_EINVAL = -1,    /* bad argument                                                          */
  PCDN_ENOMEM = -2,    /* host or device allocation failed                                      */
  PCDN_ENODEV = -3,    /* no CUDA device / host-only engine asked to route                      */
  PCDN_ECUDA = -4,     /* a CUDA runtime call failed (message has the cudaError string)         */
  PCDN_ENOSPC = -5,    /* a fixed-capacity table is full (conns, keys, batch arena, entries)    */
  PCDN_EKEYLEN = -6,   /* key longer than config.max_key_len                                    */
  PCDN_EPARSE = -7,    /* frame is not a valid cdn-proto message (=> caller disconnects peer)   */
  PCDN_EPRUNE = -8,    /* Topic::prune left no valid topic (=> caller disconnects peer)         */
  PCDN_EKIND = -9,     /* message kind not allowed on this connection type (=> disconnect)      */
  PCDN_ENOENT = -10,   /* unknown batch id / connection                                         */
  PCDN_EAGAIN = -11,   /* all batch slots in flight: poll + release one first                   */
  PCDN_E2BIG = -12,    /* batch exceeded max_batch_deliveries on the device; nothing was packed */
  PCDN_EHOOK = -13     /* the message hook returned an error (=> caller disconnects peer)       */
};

/* ---- vocabulary --------------------------------------------------------------------------- */
typedef struct pcdn_engine pcdn_engine; /* opaque */
typedef uint32_t pcdn_conn;            /* dense connection id; users and peer brokers share it */
#define PCDN_CONN_NONE 0xFFFFFFFFu

/* capnp union tags of cdn-proto/schema/messages.capnp (messages_capnp.rs:277,292) */
enum {
  PCDN_KIND_DIRECT = 3,
  PCDN_KIND_BROADCAST = 4,
  PCDN_KIND_SUBSCRIBE = 5,
  PCDN_KIND_UNSUBSCRIBE = 6,
  PCDN_KIND_USER_SYNC = 7,
  PCDN_KIND_TOPIC_SYNC = 8
};

/* pcdn_msg.flags — `to_users_only` / `to_user_only` of handler.rs:197,240 (R4) */
enum { PCDN_TO_USERS_ONLY = 1 };

/* Output records are 32-byte aligned inside a connection's ring; one record = one framed
 * delivery: u32 BE length ‖ raw bytes ‖ pad.  32 B = one DRAM sector, so two records never share
 * a sector and no store of the pack kernel is a partial-sector write. */
#define PCDN_RECORD_ALIGN 32u

typedef struct pcdn_config {
  uint32_t struct_size;         /* = sizeof(pcdn_config); ABI guard.  offsetof(pcdn_config, ref_min_bytes)
                                 * (the size before that field was added) is accepted as ref_min_bytes = 0 */
  int32_t device;               /* CUDA ordinal; < 0 = host-only state mirror (no data path)    */
  uint32_t max_conns;           /* capacity of the dense connection-id space (users + brokers)  */
  uint32_t max_topics;          /* rows of the subscription bitmap; 256 = wire-exact (Topic=u8) */
  uint32_t max_keys;            /* direct-map capacity (entries of the cuckoo table)            */
  uint32_t max_key_len;         /* longest user public key in bytes (prod BLS-BN254 G2 = 128)   */
  uint64_t ring_bytes_per_conn; /* output ring per connection, multiple of 32                   */
  uint32_t max_batch_msgs;      /* messages per batch                                           */
  uint32_t max_batch_bcast;     /* broadcast messages per batch (sizes the match matrix)        */
  uint64_t max_batch_bytes;     /* bytes of frames per batch (device arena + pinned staging)    */
  uint64_t max_batch_deliveries;/* capacity of the scatter list per batch                       */
  uint32_t batch_slots;         /* batches in flight (>=1)                                      */
  uint32_t n_valid_topics;      /* Topic::prune validity: topic t is valid iff t < this (def.rs:25-49); 0 = all */
  uint64_t hash_seed;           /* keys the direct-map hash (0 = default)                       */
  void* stream;                 /* optional cudaStream_t to run on (e.g. torch's); NULL = own   */
  const char* identity;         /* this broker's BrokerIdentifier string "public/private"       */
  uint32_t pack_variant;        /* pack launch geometry, 0 = engine default.  Bits 8-11 (k_pack) and
                                 * 12-15 (k_pack_direct), when non-zero, override the CTAs per SM;
                                 * any other bit set is PCDN_EINVAL.  Output does not depend on it. */
  uint32_t flags;               /* PCDN_FLAG_*                                                  */
  /* ---- connection shards over several GPUs (SURVEY 8e) ---------------------------------------
   * n_devices > 1 (or world_shards > 1): `max_conns`, `ring_bytes_per_conn` and the batch capacities
   * are PER SHARD; `max_keys`, `max_topics` describe the whole broker (the direct map is replicated
   * on every GPU: a direct message resolves identically everywhere and is packed by the GPU that
   * owns the target connection).  Connection ids are global: id = shard * shard_stride + local, a
   * new connection goes to the least-loaded shard (the marshal's policy for brokers,
   * cdn-proto/src/connection/auth/marshal.rs:108-118); pcdn_shard_info() gives shard_stride.
   * With n_devices >= 1 `device` is ignored and `stream` (optional) is the main stream of devices[0]. */
  uint32_t n_devices;           /* 0 = single device `device`; else number of entries of `devices`          */
  uint32_t ingest;              /* PCDN_INGEST_*: how a batch reaches every shard                           */
  const int32_t* devices;       /* CUDA ordinals; an ordinal may repeat (shards sharing one GPU: PCDN_INGEST_HOST only) */
  /* Multi-process groups (one process per GPU, e.g. torchrun): every process creates its engine with
   * the SAME config except devices/first_shard and then issues the SAME sequence of state and
   * data-in calls with the same arguments (SPMD, like the ranks of an NCCL job).  Each process keeps
   * the whole routing state, applies table updates to its own GPUs only, and polls / reads its own
   * shards.  The process that owns global shard 0 is the ingest root: only ITS copy of a batch's
   * bytes is used — it goes to every GPU of the group with the ncclBroadcast.                      */
  uint32_t world_shards;        /* total shards of the broker over all processes (0 = n_devices)            */
  uint32_t first_shard;         /* global index of devices[0]                                               */
  const void* nccl_unique_id;   /* world_shards > n_devices: the 128-byte id from pcdn_nccl_unique_id(), identical in every process */
  uint64_t pool_bytes;          /* PCDN_FLAG_OUTPUT_POOL: bytes of the output pool per shard (0 = max_conns * ring_bytes_per_conn; < 128 GiB) */
  uint64_t global_memory_pool_size; /* Limiter analogue (cdn-proto/src/connection/limiter/mod.rs:56-68,
                                 * cdn-broker/src/binaries/broker.rs:71-72 default 1 GiB): bytes of inbound frames
                                 * that may be in flight (accepted, their batch not yet released); 0 = unlimited.
                                 * The reference awaits the semaphore; here a frame that does not fit launches the
                                 * open batch and is refused with PCDN_EAGAIN: the caller retries after releasing a
                                 * batch (the launched one holds the permits it would wait for). */
  /* Delivery by reference above a size threshold: a routed message (broadcast or direct) whose raw length is
   * >= ref_min_bytes is delivered as ONE reference record per recipient (the layout of
   * PCDN_FLAG_SHARED_PAYLOAD below, its payload resolved through pcdn_batch_payload); every shorter message
   * keeps its framed copy, the wire bytes a consumer can send straight from the rings.  A message is
   * delivered one way or the other, never both, and a connection's span may hold both kinds of record, in
   * batch order.  Spans, runs, n_records, bytes_out (4 + L per delivery), pool_base, wrap, release and retry
   * keep their meaning.  0 = off (every delivery a framed copy).  The threshold decides which deliveries
   * need the host payload, so it is the host's to choose; pcdn_config_default leaves it 0.
   * pcdn_create refuses (PCDN_EINVAL) a non-zero value together with PCDN_FLAG_SHARED_PAYLOAD, a value
   * above 0x1FFFFFFF, and a value whose largest copied record, round_up(4 + ref_min_bytes - 1, 32) bytes,
   * does not fit an empty ring (ring_bytes_per_conn; with PCDN_FLAG_OUTPUT_POOL: the pool).  So with the
   * threshold set, no message overflows a connection by its size alone: only a connection that does not
   * drain its ring can overflow.                                                                   */
  uint32_t ref_min_bytes;
} pcdn_config;

/* pcdn_config.ingest — sharded engines: how the staged batch gets from the host into every GPU */
enum {
  PCDN_INGEST_NCCL = 0, /* host -> GPU of shard 0 (one H2D), then ONE ncclBroadcast over NVLink to all shards,
                         * issued by the library on a side stream so it overlaps the previous batch's pack
                         * (default; libnccl.so.2 is bound at run time and its absence is PCDN_ENODEV)  */
  PCDN_INGEST_HOST = 1  /* every shard copies the batch from pinned host memory itself (no NCCL needed;
                         * also the only mode for shards that share a GPU)                              */
};

/* pcdn_config.flags */
enum {
  /* Ingress parse on the device (SURVEY 8f-1): pcdn_user_receive / pcdn_broker_receive /
   * pcdn_receive_frames only peek the union tag of Broadcast/Direct frames and copy the raw bytes;
   * the Cap'n Proto walk, Topic::prune and the recipient extraction run in a kernel (k_parse) and
   * the per-message outcome comes back in pcdn_batch_result.msg_status.  Other kinds keep the host
   * path.  Deviation: a malformed / all-topics-invalid frame is reported after the batch instead of
   * synchronously, so later frames of that sender inside the same batch are still routed. */
  PCDN_FLAG_DEVICE_PARSE = 1,
  /* Engines with <= 65536 connection slots take the latency path for small batches: one fused
   * control launch, counters published into mapped pinned host memory, and the span table /
   * overflow list written there directly by the offsets kernel when few spans are expected
   * (no D2H copies, one event to wait for).  This flag forces the path of large engines (span
   * table built in HBM, copied out while the pack is still running) regardless of size. */
  PCDN_FLAG_STAGED_SPANS = 2,
  /* Egress hand-off without a device→host copy (SURVEY 8f-2): the per-connection rings live in
   * mapped pinned HOST memory and the pack kernel stores the framed records there over PCIe, so a
   * span is readable by the socket writer (writev / io_uring / MSG_ZEROCOPY) the moment pcdn_poll
   * returns: pcdn_host_rings() gives the base pointer, a span's bytes are at
   * base + conn * ring_bytes_per_conn + ring_off.  Egress is then bounded by PCIe (≈50 GB/s, above
   * any NIC) instead of HBM; rings in HBM (default) are for GPUDirect hand-off and measurement.   */
  PCDN_FLAG_HOST_RINGS = 4,
  /* Run-length span table: pcdn_batch_result.runs / n_runs instead of spans (spans == NULL; n_spans
   * still counts the spans the runs stand for).  A run = n_conns CONSECUTIVE connection ids that each
   * own an identical span.  A dense broadcast batch to 2^20 connections is 4096 runs (96 KB) instead
   * of a 16 MB table over PCIe per batch; sparse batches degrade to one run per span.              */
  PCDN_FLAG_SPAN_RUNS = 8,
  /* One shared OUTPUT POOL per GPU instead of a fixed ring per connection: every batch gets one
   * contiguous region of the pool, laid out connection by connection (each connection's records back
   * to back, in batch order), and the region is freed as a whole by pcdn_release_batch.  Memory is
   * sized by traffic (pcdn_config.pool_bytes), not by max_conns x the hottest connection, and no
   * connection can overflow: n_overflow is always 0.  A batch that does not fit the free part of the
   * pool is REFUSED AS A WHOLE — pcdn_batch_result.status = PCDN_EAGAIN (as a positive number), nothing
   * written — and so is every batch launched after it (order!); the host releases older batches and
   * calls pcdn_retry_batch, oldest first.  This is the reference Limiter's ingress back-pressure
   * (cdn-proto/src/connection/limiter/mod.rs:56-68) in place of a per-connection drop.
   * Span offsets in this mode: pcdn_span.ring_off is in units of PCDN_RECORD_ALIGN (32 B), relative to
   * pcdn_batch_result.pool_base; the bytes are at pool + (pool_base + ring_off) * 32 (pcdn_shard_info:
   * rings_dev / rings_host = the pool).  pcdn_read takes the absolute unit offset pool_base + ring_off. */
  PCDN_FLAG_OUTPUT_POOL = 16,
  /* Shared-payload delivery: EVERY routed message (broadcast and direct) is delivered by reference.
   * The payload exists once per batch, in pinned host memory (pcdn_batch_payload), and each delivery is
   * one 32-byte REFERENCE RECORD in the recipient's ring / the output pool instead of a framed copy (the
   * reference's fan-out clones a refcounted `Bytes`, it never copies per recipient).  Spans, runs,
   * n_records, pool_base, wrap, release and retry keep their meaning; bytes_out still counts the 4 + L
   * wire bytes of each delivery.  Records have no size limit in this mode (one unit each), so messages
   * far larger than a ring are delivered.  The CTA counts of pcdn_config.pack_variant do not apply
   * (the pack kernel is k_pack_ref).  Record layout (all fields fixed, so bytes compare exactly):
   *   bytes  0..3   PCDN_REF_MARK (no framed record starts with it: L <= 0x1FFFFFFF)
   *   bytes  4..7   u32 big-endian L: the 4 wire bytes of the length prefix
   *   bytes  8..15  u64 little-endian offset of the raw bytes from the batch's payload base
   *   bytes 16..23  u64 little-endian batch id (resolution is self-checking; a retry writes the same record)
   *   bytes 24..31  zero
   * A writer walks a span as usual: at p, if BE32(p) == PCDN_REF_MARK it sends p[4..8) ‖ the L bytes at
   * payload + offset and advances 32 bytes; otherwise it handles a framed record as before.          */
  PCDN_FLAG_SHARED_PAYLOAD = 32,
  /* In-batch subscription changes.  Without this flag every subscription change launches the open
   * batch first, so a receive window with k Subscribe / Unsubscribe frames becomes k + 1 batches.
   * With it, pcdn_subscribe_user_to, pcdn_unsubscribe_user_from, pcdn_subscribe_broker_to,
   * pcdn_unsubscribe_broker_from and a user's Subscribe / Unsubscribe frame on every receive path
   * (after Topic::prune and the hook) become an EVENT of the open batch instead.  The event's position
   * is the number of messages in the batch when it was recorded; it applies to exactly the batch's
   * messages at or after that position and to every later batch, so each connection's delivered byte
   * stream is identical to what the same calls produce without the flag: only batch boundaries differ.
   * The host mirror changes at once (pcdn_debug_interested, pcdn_get_topic_sync see it immediately).
   * Events are not messages: n_msgs, msg_status and the counters keep their meaning.
   * An event that does not fit the open batch (max_batch_msgs events already, or its topics would
   * overflow the descriptor block's topic entries) takes the path without the flag: the batch is
   * launched, then the change is applied.  Prune errors stay synchronous (PCDN_EPRUNE / PCDN_EPARSE,
   * no event).  Every other state call (add / remove of users and brokers, pcdn_apply_user_sync,
   * pcdn_apply_topic_sync) still launches the open batch first.                                   */
  PCDN_FLAG_INBATCH_SUBSCRIBE = 64
};
#define PCDN_REF_MARK 0xFFFFFFFFu

/* One routed message.  `raw` is the inbound frame body and is forwarded verbatim (R1). */
typedef struct pcdn_msg {
  uint8_t kind;  /* PCDN_KIND_BROADCAST or PCDN_KIND_DIRECT                                     */
  uint8_t flags; /* PCDN_TO_USERS_ONLY                                                          */
  uint16_t n_topics;
  const uint16_t* topics;   /* broadcast: already pruned (R6)                                   */
  const uint8_t* recipient; /* direct: recipient public key                                     */
  uint32_t recipient_len;
  uint32_t raw_len;
  const uint8_t* raw;
} pcdn_msg;

/* A contiguous run of records in one connection's ring.  The host walks it as the reference's
 * writer task walks its queue (cdn-proto/src/connection/protocols/mod.rs:156-186): at `p` read
 * L = BE32(p), write the 4+L bytes to the socket, advance p by round_up(4+L, 32). */
typedef struct pcdn_span {
  pcdn_conn conn;
  uint32_t ring_off;  /* byte offset of the first record inside the connection's ring; PCDN_FLAG_OUTPUT_POOL: offset in 32-byte units relative to pcdn_batch_result.pool_base */
  uint32_t len;       /* bytes covered (multiple of 32), padding included                      */
  uint32_t n_records; /* deliveries in this run                                                */
} pcdn_span;

/* PCDN_FLAG_SPAN_RUNS: connections conn0 .. conn0 + n_conns - 1 each have a span {ring_off, len, n_records} */
typedef struct pcdn_span_run {
  pcdn_conn conn0;
  uint32_t n_conns;
  uint32_t ring_off;   /* of conn0 */
  uint32_t len;
  uint32_t n_records;
  uint32_t off_stride; /* added to ring_off per following connection: 0 with per-connection rings (same offset in each
                        * connection's own ring), len / 32 units with PCDN_FLAG_OUTPUT_POOL (the regions follow each other) */
} pcdn_span_run;

typedef struct pcdn_batch_result {
  uint64_t batch_id;
  uint32_t n_msgs;
  uint32_t n_spans;
  const pcdn_span* spans;          /* engine-owned pinned host memory, valid until release      */
  uint64_t n_deliveries;           /* records written                                           */
  uint64_t bytes_out;              /* sum of 4+L over deliveries = bytes put on the wire (BYTES_SENT of protocols/mod.rs:388 counts L only: bytes_out - 4*n_deliveries) */
  uint32_t n_overflow;             /* connections whose ring was full: their deliveries from the overflow point on were dropped; the host must remove them (R13 analogue) */
  const pcdn_conn* overflow_conns; /* engine-owned                                              */
  uint32_t n_direct_dropped;       /* direct messages with no route (handler.rs:210,224)        */
  uint32_t status;                 /* 0, PCDN_E2BIG (scatter-list capacity, or larger than the whole output pool) or PCDN_EAGAIN (output pool full: release older batches, pcdn_retry_batch) — as positive numbers; a refused batch wrote nothing and reports zero counters */
  const int8_t* msg_status;        /* device-parse batches: per message 0 or PCDN_EPARSE / PCDN_EPRUNE (the reference would have ended that sender's receive loop); NULL otherwise */
  uint32_t n_msg_errors;           /* number of non-zero entries in msg_status                  */
  uint32_t reserved;               /* pcdn_poll_shard: global index of the shard                */
  const pcdn_span_run* runs;       /* PCDN_FLAG_SPAN_RUNS: the span table in run-length form (then spans == NULL) */
  uint32_t n_runs;
  uint32_t pool_base;              /* PCDN_FLAG_OUTPUT_POOL: first 32-byte unit of this batch's region; span offsets are relative to it (0 otherwise) */
} pcdn_batch_result;

/* Device-resident batch (inputs already in HBM; used by bench `value` and the NCCL ingest path).
 * Frame slot layout in `arena`: each message owns a 16-byte aligned slot; the raw bytes start at
 * slot+4 (the first 4 bytes are the hole the pack kernel fills with the BE length).  */
typedef struct pcdn_device_batch {
  uint32_t n_msgs;
  uint32_t n_bcast;              /* number of broadcast messages among them                    */
  const void* arena;             /* device: frame slots                                        */
  uint64_t arena_bytes;
  const uint8_t* kind;           /* device [n_msgs]                                            */
  const uint8_t* flags;          /* device [n_msgs]                                            */
  const uint32_t* slot_off16;    /* device [n_msgs] slot offset in arena, units of 16 B        */
  const uint32_t* raw_len;       /* device [n_msgs]                                            */
  const uint32_t* aux_off;       /* device [n_msgs] broadcast: index into `topics`; direct: byte offset of the recipient key in arena (4-byte aligned) */
  const uint32_t* aux_len;       /* device [n_msgs] broadcast: topic count; direct: key length */
  const uint16_t* topics;        /* device: concatenated topic lists                           */
  uint32_t n_topics_total;
  const uint32_t* bcast_index;   /* device [n_bcast]: batch index of the j-th broadcast, ascending */
  uint32_t hints;                /* PCDN_BATCH_*                                               */
  uint32_t reserved;
} pcdn_device_batch;
/* pcdn_device_batch.hints */
enum {
  /* The arrays are already complete in device memory (produced and synchronised earlier).  Without
   * this hint the engine orders the batch after everything queued on its (root shard's) main stream,
   * so that a caller sharing that stream can produce the batch with its own kernels; with it a sharded
   * engine may broadcast batch n+1 while batch n is still being packed. */
  PCDN_BATCH_READY = 1
};

typedef struct pcdn_stats {
  uint64_t batches, msgs, deliveries, bytes_out;
  double ms_match;   /* accumulated device time (CUDA events on the engine stream), when PCDN timing is on */
  double ms_plan;
  double ms_direct;
  double ms_pack;
  double ms_total;
  uint64_t timed_batches;
  uint64_t inflight_bytes;      /* bytes currently holding pool permits                               */
  uint64_t released_batches;
  double latency_ms_sum;        /* launch → release wall time per batch (the reference's LATENCY histogram observes the permit lifetime, limiter/pool.rs:44-52) */
  uint64_t bytes_in;            /* raw frame bytes accepted (metrics.rs BYTES_RECV; bytes_out above is BYTES_SENT + 4 per delivery) */
  /* the LATENCY histogram (metrics.rs:21-23) of the same launch → release time, log2 buckets in
   * microseconds: [0] < 16 us, [i] = [8 << i, 16 << i) us for i = 1..14, [15] >= 262 ms            */
  uint64_t latency_hist_us[16];
  uint64_t kernel_launches;     /* CUDA kernels launched by this library in this process (all engines) */
} pcdn_stats;

/* ---- lifecycle ---------------------------------------------------------------------------- */
uint32_t pcdn_abi_version(void);
void pcdn_config_default(pcdn_config* cfg);
int pcdn_create(const pcdn_config* cfg, pcdn_engine** out);
void pcdn_destroy(pcdn_engine* e);
const char* pcdn_last_error(void);

/* ---- state in: Connections::* (cdn-broker/src/connections/mod.rs) ------------------------- */
/* Connections::add_user mod.rs:278-304 — kicks an existing user with the same key, registers the
 * connection, direct_map[key]=self, subscribes to `topics`.  Returns the dense connection id.
 * Connection ids name rings and appear in spans: an id freed by a disconnect or a kick is not
 * handed out again until every batch launched before that removal has been released, so the host
 * can keep one id -> socket table.  PCDN_EAGAIN (before anything is changed) when the table is
 * full and the only free ids are still held back that way; PCDN_ENOSPC when it is simply full.   */
int pcdn_add_user(pcdn_engine* e, const uint8_t* key, uint32_t key_len, const uint16_t* topics,
                  uint32_t n_topics, pcdn_conn* out_conn);
/* Connections::remove_user mod.rs:330-351 */
int pcdn_remove_user(pcdn_engine* e, const uint8_t* key, uint32_t key_len);
/* Connections::subscribe_user_to mod.rs:365 / unsubscribe_user_from :383 (RelationalMap R10)   */
int pcdn_subscribe_user_to(pcdn_engine* e, const uint8_t* key, uint32_t key_len,
                           const uint16_t* topics, uint32_t n);
int pcdn_unsubscribe_user_from(pcdn_engine* e, const uint8_t* key, uint32_t key_len,
                               const uint16_t* topics, uint32_t n);
/* Connections::add_broker mod.rs:252-274 / remove_broker :308-324 */
int pcdn_add_broker(pcdn_engine* e, const char* identifier, pcdn_conn* out_conn);
int pcdn_remove_broker(pcdn_engine* e, const char* identifier);
/* Connections::subscribe_broker_to mod.rs:354 / unsubscribe_broker_from :372 */
int pcdn_subscribe_broker_to(pcdn_engine* e, const char* identifier, const uint16_t* topics,
                             uint32_t n);
int pcdn_unsubscribe_broker_from(pcdn_engine* e, const char* identifier, const uint16_t* topics,
                                 uint32_t n);
/* Connections::apply_user_sync mod.rs:154-162 = VersionedMap::merge (versioned_map.rs:193-269)
 * of a remote DirectMap followed by remove_user of every changed key.  One entry per key of the
 * remote map; owner == NULL is a tombstone.  `remote_identity` is the remote map's conflict id. */
typedef struct pcdn_user_sync_entry {
  const uint8_t* key;
  uint32_t key_len;
  uint64_t version;
  const char* owner; /* BrokerIdentifier string or NULL (tombstone) */
} pcdn_user_sync_entry;
int pcdn_apply_user_sync(pcdn_engine* e, const char* remote_identity,
                         const pcdn_user_sync_entry* entries, uint32_t n);
/* ---- inter-broker sync on the same tables (SURVEY 8f-4) ------------------------------------------
 * The CRDT side of Connections: what cdn-broker/src/tasks/broker/sync.rs sends and what
 * broker_receive_loop applies (handler.rs:164-188).  Serialisation of these maps on the wire (rkyv)
 * stays with the host; the engine exchanges plain arrays.  Returned arrays are engine-owned and stay
 * valid until the next pcdn_get_*_sync call on the same engine. */
typedef struct pcdn_topic_sync_entry {
  uint16_t topic;
  uint8_t status;   /* 0 Subscribed, 1 Unsubscribed, 2 tombstone */
  uint8_t reserved[5];
  uint64_t version;
} pcdn_topic_sync_entry;
/* Connections::get_full_user_sync mod.rs:131 (full != 0) / get_partial_user_sync :141 (= direct_map.diff()) */
int pcdn_get_user_sync(pcdn_engine* e, int full, const pcdn_user_sync_entry** out, uint32_t* n);
/* Connections::apply_topic_sync mod.rs:165-191: merge a peer's TopicSyncMap (conflict identity
 * `remote_identity`, TopicSyncMap::new(0) in the reference) and (un)subscribe that broker */
int pcdn_apply_topic_sync(pcdn_engine* e, const char* identifier, uint32_t remote_identity,
                          const pcdn_topic_sync_entry* entries, uint32_t n);
/* Connections::get_full_topic_sync mod.rs:194 / get_partial_topic_sync :205-237 */
int pcdn_get_topic_sync(pcdn_engine* e, int full, const pcdn_topic_sync_entry** out, uint32_t* n);
/* Bulk form of add_user for table loads (keys are fixed-stride); same semantics, one lock.      */
int pcdn_add_users_bulk(pcdn_engine* e, const uint8_t* keys, uint32_t key_len, uint32_t key_stride,
                        uint32_t n_users, const uint16_t* topics, const uint32_t* topic_offsets,
                        pcdn_conn* out_conns /* optional */);

/* ---- data in: the two routing functions of cdn-broker/src/tasks/broker/handler.rs ---------- */
/* Inner::handle_broadcast_message handler.rs:240-272 — appended to the open batch.              */
int pcdn_handle_broadcast_message(pcdn_engine* e, const uint16_t* topics, uint32_t n_topics,
                                  const uint8_t* raw, uint32_t raw_len, int to_users_only);
/* Inner::handle_direct_message handler.rs:197-237 */
int pcdn_handle_direct_message(pcdn_engine* e, const uint8_t* recipient, uint32_t recipient_len,
                               const uint8_t* raw, uint32_t raw_len, int to_user_only);
/* ---- data out: the broker's own frames to its peer brokers (cdn-broker/src/tasks/broker/sender.rs) -----
 * How a host sends the UserSync / TopicSync frames it builds (tasks/broker/sync.rs: the full syncs to a new
 * peer, the partial syncs to every peer every 10 s) in order with the routed traffic of the same link.
 *  - Bytes: `raw` is forwarded verbatim, framed as u32 BE len || raw (R1, R2).  The engine does not parse it
 *    and no message hook runs on it.  It is delivered by the rule of every routed message: a framed copy, or a
 *    32-byte reference record on PCDN_FLAG_SHARED_PAYLOAD engines and when raw_len >= ref_min_bytes.
 *  - Place: it is appended to the open batch as ONE message at its position, so every connection's stream
 *    follows call order together with routed messages (R9).  These are data calls: they do not launch the
 *    open batch (a full batch is launched and the frame opens the next one, as for any message).
 *  - Recipients: the peer brokers connected at the call (pcdn_add_broker / pcdn_remove_broker launch the open
 *    batch first, R12): a broker added after the send does not get the frame; a broker removed after it does
 *    (its id stays quarantined as usual); after a same-identifier re-add (kick) the frame stays with the old
 *    connection.  Users never get it; subscriptions, PCDN_FLAG_INBATCH_SUBSCRIBE events and to_users_only
 *    play no part.  A sharded engine delivers it from each shard to that shard's brokers.
 *  - Returns 0 = appended; 1 = nothing to send to (no broker `identifier` / no broker connected), nothing
 *    appended; else the negative codes of pcdn_handle_broadcast_message: PCDN_ENODEV (host-only engine),
 *    PCDN_EINVAL (length above MAX_MESSAGE_SIZE, or raw NULL with raw_len > 0), PCDN_ENOSPC (does not fit an
 *    empty batch), PCDN_EAGAIN (no batch slot free).
 *  - Capacity and counters: one broadcast slot (max_batch_bcast), its arena bytes and its deliveries; counted
 *    in msgs, deliveries and bytes_out.  It takes NO global_memory_pool_size permits and is not counted in
 *    bytes_in or inflight_bytes (the reference builds sync frames outside the Limiter, sync.rs:34), so a send
 *    succeeds while routed frames get PCDN_EAGAIN from the memory pool.  Overflow (overflow_conns), output-pool
 *    refusal and pcdn_retry_batch work as for any message; a retried batch delivers to the set at launch.
 *  - pcdn_submit, pcdn_submit_device and pcdn_receive_frames do not carry these messages.                  */
/* Inner::try_send_to_broker (cdn-broker/src/tasks/broker/sender.rs:17-45) */
int pcdn_send_to_broker(pcdn_engine* e, const char* identifier, const uint8_t* raw, uint32_t raw_len);
/* Inner::try_send_to_brokers (sender.rs:49-59): every connected peer broker */
int pcdn_send_to_brokers(pcdn_engine* e, const uint8_t* raw, uint32_t raw_len);
/* One iteration of Inner::user_receive_loop (cdn-broker/src/tasks/user/handler.rs:104-161):
 * Message::deserialize (cdn-proto/src/message.rs:212) → Topic::prune (def.rs:36-49) → dispatch.
 * Broadcast/Direct are appended to the open batch; Subscribe/Unsubscribe update the tables (the
 * open batch is flushed first so earlier messages do not see the change, R12).  A negative return
 * (PCDN_EPARSE/EPRUNE/EKIND) means the reference loop would have ended: the caller removes the user. */
int pcdn_user_receive(pcdn_engine* e, const uint8_t* sender_key, uint32_t key_len,
                      const uint8_t* raw, uint32_t raw_len);
/* One iteration of Inner::broker_receive_loop (tasks/broker/handler.rs:130-192), Direct and
 * Broadcast only (to_user(s)_only = true, no prune); other kinds return 1 = "not routed here". */
int pcdn_broker_receive(pcdn_engine* e, const char* identifier, const uint8_t* raw,
                        uint32_t raw_len);
/* ---- MessageHookDef (cdn-proto/src/def.rs:79-92) -------------------------------------------------
 * The reference calls `hook.on_message_received(&mut message)` after Message::deserialize and before
 * the dispatch, in user_receive_loop (cdn-broker/src/tasks/user/handler.rs:110-118) and in
 * broker_receive_loop (tasks/broker/handler.rs:137-144): Ok(SkipMessage) => the frame is ignored,
 * Ok(ProcessMessage) => dispatch (with whatever the hook changed in the parsed message), Err => the
 * receive loop ends (the peer is disconnected).  The hook sees the PARSED message and may rewrite its
 * routing fields; the bytes that are forwarded stay the inbound frame (the reference forwards
 * `raw_message`, not a re-serialisation).
 *
 * The callback runs on the thread that calls pcdn_user_receive / pcdn_broker_receive /
 * pcdn_receive_frames, with the engine lock held: it must not call back into the same engine.
 * A hooked origin is always parsed on the host: PCDN_FLAG_DEVICE_PARSE is bypassed for its frames
 * (the device parser never shows a message to the host).  While a hook is set, pcdn_receive_frames
 * parses each frame on the calling thread when it comes to it, so the hook sees the frames in order:
 * those the call consumes and the one it stops at, if it stops early (that frame is shown again when
 * the caller retries it).  pcdn_handle_*_message / pcdn_submit are below the hook, as in the
 * reference.                                                                                        */
enum { PCDN_HOOK_PROCESS = 0, PCDN_HOOK_SKIP = 1 };  /* HookResult; any negative return = Err */
typedef struct pcdn_hook_message {
  uint8_t kind;             /* PCDN_KIND_*                                                          */
  uint8_t origin;           /* 0 = user connection, 1 = broker connection                           */
  uint16_t n_topics;        /* Broadcast / Subscribe / Unsubscribe: entries of `topics`; may be lowered */
  uint8_t* topics;          /* the parsed topic list (wire values, before Topic::prune); rewritable  */
  const uint8_t* recipient; /* Direct: recipient key; may be re-pointed (read before the hook returns) */
  uint32_t recipient_len;
  uint32_t raw_len;
  const uint8_t* raw;       /* the inbound frame (read-only; forwarded verbatim)                    */
  const uint8_t* sender;    /* set_identifier analogue: the user's public key / the broker identifier string */
  uint32_t sender_len;
  uint32_t reserved;
} pcdn_hook_message;
typedef int (*pcdn_message_hook)(void* user, pcdn_hook_message* msg);
/* origin 0 = Inner::user_message_hook, 1 = Inner::broker_message_hook (cdn-broker/src/lib.rs); cb NULL removes it */
int pcdn_set_message_hook(pcdn_engine* e, int origin, pcdn_message_hook cb, void* user);

/* Many inbound frames in one call (one lock, no per-call FFI cost): frame i enters
 * user_receive_loop (origin 0, `sender` = that user's key) or broker_receive_loop (origin 1).
 * rc_out[i] (optional) gets what pcdn_user_receive / pcdn_broker_receive would have returned for
 * frame i, and pcdn_last_error is left as those calls, one per frame, would have left it.
 * Returns the number of frames consumed (== n unless a capacity condition — no free batch slot,
 * global memory pool exhausted — stopped it: drain a batch and call again with the rest) or a
 * negative code when not even the first frame could be taken.  Large calls are parsed and copied
 * by several host threads (PCDN_INGEST_THREADS, default min(16, cores)); order is preserved. */
typedef struct pcdn_frame {
  const uint8_t* sender;
  uint32_t sender_len;
  uint32_t origin;
  const uint8_t* raw;
  uint32_t raw_len;
  uint32_t reserved;
} pcdn_frame;
int pcdn_receive_frames(pcdn_engine* e, const pcdn_frame* frames, uint32_t n, int32_t* rc_out);
/* Close the open batch and launch it.  *batch_id = 0 when the batch was empty. */
int pcdn_flush(pcdn_engine* e, uint64_t* batch_id);
/* Submit an explicit ordered batch (R9: batch order = per-connection delivery order). */
int pcdn_submit(pcdn_engine* e, const pcdn_msg* msgs, uint32_t n, uint64_t* batch_id);
/* Same, inputs already resident in HBM (no host copy, no host parse).  PCDN_FLAG_SHARED_PAYLOAD or a
 * non-zero ref_min_bytes: the frame arena is copied once into the slot's pinned staging
 * (pcdn_batch_payload) before the batch runs, on the batch's stream (the main stream of the first local
 * shard), and polling the batch waits for that copy; an arena larger than that staging (max_batch_bytes)
 * is PCDN_ENOSPC. */
int pcdn_submit_device(pcdn_engine* e, const pcdn_device_batch* batch, uint64_t* batch_id);

/* ---- data out: replaces Connection::send_message_raw + the per-connection writer task
 *      (cdn-proto/src/connection/protocols/mod.rs:239-251,156-186,354-394) -------------------- */
/* Oldest batch that was launched and not yet released (0 = none).  State calls and full batches
 * launch the open batch implicitly, so a host drains with: while (next_batch) { poll; write; release }. */
int pcdn_next_batch(pcdn_engine* e, uint64_t* batch_id);
/* Wait for (block != 0) or test a batch; fills *out (span table is in pinned host memory). */
int pcdn_poll(pcdn_engine* e, uint64_t batch_id, pcdn_batch_result* out, int block);
/* Copy `len` ring bytes of a connection to host memory: its records, as a socket writer walks them
 * (PCDN_FLAG_SHARED_PAYLOAD or ref_min_bytes: reference records, resolved through pcdn_batch_payload).
 * With PCDN_FLAG_HOST_RINGS this is a plain memcpy; prefer pcdn_host_rings() and read in place.  */
int pcdn_read(pcdn_engine* e, pcdn_conn conn, uint32_t ring_off, uint32_t len, void* dst);
/* Pinned host memory holding the frames of a batch: a reference record's raw bytes are at
 * *host_base + its offset.  Valid until pcdn_release_batch of that batch; PCDN_ENOENT for an unknown or
 * released batch, and for a device-resident batch (pcdn_submit_device) of an engine without
 * PCDN_FLAG_SHARED_PAYLOAD or ref_min_bytes, whose frames never reach the host.  Sharded engines and multi-process
 * groups return this process's own staged copy (identical everywhere by the SPMD contract).       */
int pcdn_batch_payload(pcdn_engine* e, uint64_t batch_id, const uint8_t** host_base);
/* PCDN_FLAG_OUTPUT_POOL: run a refused batch (status PCDN_EAGAIN) again after older batches have been
 * released.  Only the oldest unreleased batch can be retried; its result is polled again afterwards.
 * The batch is routed against the tables as they were when it was launched, on every shard, like any
 * other batch: a state change made between the refusal and the retry applies to later batches only.
 * Shards that accepted their share keep it; the others place and pack theirs again. */
int pcdn_retry_batch(pcdn_engine* e, uint64_t batch_id);
/* The host has written every span of the batch: free its ring space and its slot.  This is the
 * analogue of dropping the last `Bytes` clone (limiter/pool.rs:44-52).  In order, oldest first. */
int pcdn_release_batch(pcdn_engine* e, uint64_t batch_id);

/* ---- connection shards (n_devices > 1) ------------------------------------------------------ */
/* A fresh ncclUniqueId (128 bytes) for pcdn_config.nccl_unique_id: one process generates it and
 * hands it to the others by whatever channel the host has (torch.distributed store, a file, MPI). */
#define PCDN_NCCL_UNIQUE_ID_BYTES 128
int pcdn_nccl_unique_id(void* out128);
typedef struct pcdn_shard_desc {
  uint32_t global_index;  /* shard number inside the broker (0 .. world_shards-1)                     */
  int32_t device;         /* CUDA ordinal                                                            */
  pcdn_conn conn_base;    /* ids [conn_base, conn_base + shard_stride) belong to this shard           */
  uint32_t shard_stride;  /* id range per shard (max_conns rounded up to a multiple of 8192)         */
  void* rings_dev;        /* device address of this shard's rings [max_conns][ring_bytes_per_conn]    */
  const void* rings_host; /* PCDN_FLAG_HOST_RINGS: host address of the same rings, else NULL          */
  uint64_t ring_bytes;    /* per-connection ring; PCDN_FLAG_OUTPUT_POOL: bytes of the whole pool      */
  uint32_t n_conns;       /* connections currently living on this shard                               */
  uint32_t nccl_ranks;    /* size of the ingest communicator this shard belongs to (0 = none)        */
} pcdn_shard_desc;
/* number of shards THIS process drives (1 for a single-GPU engine) */
int pcdn_num_shards(pcdn_engine* e, uint32_t* n_local, uint32_t* n_world);
int pcdn_shard_info(pcdn_engine* e, uint32_t local_shard, pcdn_shard_desc* out);
/* pcdn_poll for ONE local shard: spans (global connection ids, this shard's connections only) are
 * read in place from that shard's pinned result buffer — what the shard's egress writer uses.
 * pcdn_poll itself waits for all local shards and returns the summed counters with the shards'
 * span tables concatenated into one engine-owned array (a host copy: convenience, not the fast path). */
int pcdn_poll_shard(pcdn_engine* e, uint64_t batch_id, uint32_t local_shard, pcdn_batch_result* out, int block);

/* ---- egress: the consumer of the span table -------------------------------------------------
 * Replaces the per-connection writer task (cdn-proto/src/connection/protocols/mod.rs:156-186: pop a
 * queued message, write_length_delimited :354-394 to the socket) and Connection::soft_close
 * (:287-306).  pcdn_egress_drain makes one batch's framed records readable by the host: per local
 * shard a gather kernel packs the records of a chunk of spans into one contiguous device buffer, one
 * large DMA per chunk brings it into pinned host memory (double-buffered: PCIe stays busy while the
 * sink consumes), and the sink is called with the chunk.  With PCDN_FLAG_HOST_RINGS the sink reads the
 * rings in place (no copy).  The built-in sink (pcdn_egress_write_batch) writes every span to the file
 * descriptor attached to its connection with writev — u32 BE length + raw bytes per record, padding
 * skipped, per-connection order kept — on a small thread pool; a failed write detaches the
 * connection and reports it (pcdn_egress_failed), the analogue of the reference removing a peer
 * whose send failed (cdn-broker/src/tasks/user/sender.rs:24-30).
 * PCDN_FLAG_SHARED_PAYLOAD or ref_min_bytes: the chunks carry the reference records as stored; the fd sink sends each
 * as two iovecs (the 4 length bytes of the record, the L payload bytes from pcdn_batch_payload), and a
 * callback sink resolves them the same way through pcdn_batch_payload of the batch it drains.
 * Backlogs (backlog_bytes_per_conn / backlog_bytes_total, opt-in): without them a socket that cannot
 * take its bytes holds the fd sink in poll() for up to 30 s, and with it every other connection and
 * the release of the batch.  With a backlog the fd sink never waits on a peer: sockets are written
 * with MSG_DONTWAIT (other descriptors follow their own O_NONBLOCK mode), and on EAGAIN or a partial
 * write the unsent bytes of that connection's records — wire bytes, also the payload bytes of
 * reference records — are copied into a per-connection backlog in host memory.  The batch can be
 * released as soon as pcdn_egress_write_batch returns.  A connection with a backlog gets one
 * non-blocking attempt to flush it before its next records; whatever is left goes behind the backlog
 * (per-connection order is kept).  Growing a backlog past backlog_bytes_per_conn, or all backlogs
 * past backlog_bytes_total, is handled like a failed write: the connection is detached, its backlog
 * dropped, and it is reported once by pcdn_egress_failed.  The host moves backlogs on with
 * pcdn_egress_flush_backlog when their descriptors become writable (pcdn_egress_backlog lists them).*/
typedef struct pcdn_egress pcdn_egress;
typedef struct pcdn_egress_config {
  uint32_t struct_size; /* = sizeof(pcdn_egress_config); the size without the two backlog fields is
                           accepted too and means "no backlog"                                        */
  uint32_t n_threads;   /* writer threads of the fd sink (0 = min(16, cores))                         */
  uint64_t chunk_bytes; /* pinned staging per chunk (0 = 64 MiB); 3 host + 2 device chunks per shard  */
  uint64_t backlog_bytes_per_conn; /* bound of one connection's backlog (0 = only the total bounds it)  */
  uint64_t backlog_bytes_total;    /* bound of all backlogs together (0 = only the per-connection bound);
                                      both 0 = no backlog: the fd sink waits for slow peers (30 s bound) */
} pcdn_egress_config;
typedef struct pcdn_egress_chunk {
  uint32_t local_shard;
  uint32_t n_spans;
  const pcdn_span* spans;   /* this chunk's spans, span-table order (a wrapped connection's two spans are adjacent) */
  const uint64_t* data_off; /* [n_spans] byte offset of span i's first record inside `data`            */
  const uint8_t* data;      /* host memory, valid during the callback                                  */
  uint64_t bytes;           /* bytes of `data` covered by this chunk                                   */
} pcdn_egress_chunk;
typedef int (*pcdn_egress_sink)(void* user, const pcdn_egress_chunk* chunk); /* non-zero aborts the drain */
typedef struct pcdn_egress_stats {
  uint64_t bytes;            /* ring bytes made host-readable (record padding included)               */
  uint64_t spans, chunks;
  uint64_t records;          /* fd sink: records written                                               */
  uint64_t fd_bytes;         /* fd sink: bytes accepted by writev (= sum of 4+L)                       */
  uint64_t fd_writes;        /* fd sink: writev calls                                                  */
  uint64_t unattached_spans; /* fd sink: spans of connections without a file descriptor (skipped)      */
  uint64_t failed_conns;     /* connections reported by pcdn_egress_failed and not yet fetched         */
  double seconds;            /* wall time of the drain                                                 */
} pcdn_egress_stats;
int pcdn_egress_create(pcdn_engine* e, const pcdn_egress_config* cfg /* NULL = defaults */, pcdn_egress** out);
void pcdn_egress_destroy(pcdn_egress* g);
/* poll + hand every chunk of the batch (all local shards) to `sink` (NULL = only stage the bytes) */
int pcdn_egress_drain(pcdn_egress* g, uint64_t batch_id, pcdn_egress_sink sink, void* user, pcdn_egress_stats* out);
/* Connection::from_stream analogue: this connection's socket / pipe / memfd */
int pcdn_egress_attach(pcdn_egress* g, pcdn_conn conn, int fd);
int pcdn_egress_detach(pcdn_egress* g, pcdn_conn conn);
/* drain with the built-in writev sink */
int pcdn_egress_write_batch(pcdn_egress* g, uint64_t batch_id, pcdn_egress_stats* out);
/* connections whose write failed since the last call (engine-owned array): the host removes them (R13) */
int pcdn_egress_failed(pcdn_egress* g, const pcdn_conn** conns, uint32_t* n);
/* Connection::soft_close protocols/mod.rs:287-306: launches the open batch, writes and RELEASES every
 * batch in flight (oldest first), writes the connection's backlog (waiting up to 30 s at a time for
 * the peer), then detaches `conn` and hands its descriptor back for closing.  A write that fails on
 * the way reports the connection (pcdn_egress_failed) and *fd_out is then -2.                       */
int pcdn_egress_soft_close(pcdn_egress* g, pcdn_conn conn, int* fd_out);
/* backlogs: write what the backlogged descriptors accept, polling them together for POLLOUT for up to
 * timeout_ms (0 = one non-blocking pass; < 0 = until every backlog is written or failed).  A write
 * error reports the connection as failed.  *n_pending (may be NULL) = connections still backlogged. */
int pcdn_egress_flush_backlog(pcdn_egress* g, int timeout_ms, uint32_t* n_pending);
/* the connections that have a backlog (engine-owned array, valid until the next egress call) and the
 * bytes of all backlogs: the descriptors an event loop waits on for writability                      */
int pcdn_egress_backlog(pcdn_egress* g, const pcdn_conn** conns, uint32_t* n, uint64_t* bytes);

/* ---- introspection (tests, metrics: cdn-proto/src/connection/metrics.rs:12-28) ------------- */
int pcdn_get_stats(pcdn_engine* e, pcdn_stats* out);
/* the per-stage device times of the stats struct (ms_direct .. ms_pack) are accumulated while this is on:
 * CUDA events around the stages of the first local shard, read when the batch is polled.  Per-kernel
 * timestamps come from a profiler (e.g. torch.profiler with CUDA activities) in a run of its own. */
int pcdn_set_timing(pcdn_engine* e, int on);
/* device pointer + geometry of the rings (zero-copy verification / GPUDirect hand-off) */
int pcdn_ring_info(pcdn_engine* e, void** dev_base, uint64_t* ring_bytes, uint32_t* max_conns);
/* PCDN_FLAG_HOST_RINGS: host address of the rings (valid for the life of the engine); NULL and
 * PCDN_ENOENT when the rings live in device memory.  The rings hold records (with
 * PCDN_FLAG_SHARED_PAYLOAD or ref_min_bytes: reference records, see above). */
int pcdn_host_rings(pcdn_engine* e, const void** host_base);
/* number of connected users (Connections::num_users mod.rs:127) and brokers */
int pcdn_num_users(pcdn_engine* e, uint32_t* users, uint32_t* brokers);
/* Connections::get_interested_by_topic mod.rs:94-124 evaluated on the HOST MIRROR of the tables
 * (state-logic tests without a GPU).  Writes up to cap conn ids; returns the count via *n.       */
int pcdn_debug_interested(pcdn_engine* e, const uint16_t* topics, uint32_t n_topics,
                          int to_users_only, pcdn_conn* out, uint32_t cap, uint32_t* n);
/* Host-mirror route of a key, as the direct kernel would resolve it: 0 = none (drop),
 * 1 = local user (*conn), 2 = remote broker (*conn = that broker's conn or PCDN_CONN_NONE).     */
int pcdn_debug_route(pcdn_engine* e, const uint8_t* key, uint32_t key_len, int* kind,
                     pcdn_conn* conn);
/* Parse helper exported for tests: Message::deserialize restricted to the routed kinds.  Returns
 * the kind (>=0) or PCDN_EPARSE.  topics_out (cap 256) / recipient span are filled when relevant. */
int pcdn_parse_frame(const uint8_t* raw, uint32_t raw_len, uint16_t* topics_out,
                     uint32_t* n_topics, uint32_t* field_off, uint32_t* field_len);

#ifdef __cplusplus
}
#endif
#endif /* PCDN_FANOUT_H */
