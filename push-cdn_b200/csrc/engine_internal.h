// engine_internal.h — structures shared by the translation units of the host runtime
// (engine.cu: tables, batches, pipeline, C ABI; egress.cu: span consumers).  Not part of the ABI.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <thread>
#include <vector>

#include "frame_parse.h"
#include "host_state.h"
#include "kernels.cuh"
#include "nccl_dl.h"
#include "pcdn_fanout.h"

using namespace pcdn;

namespace pcdn_detail {

int fail(int code, const std::string& msg);   // sets the calling thread's pcdn_last_error text

#define CUDA_TRY(expr)                                                                         \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess)                                                                     \
      return fail(PCDN_ECUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));             \
  } while (0)
#define NCCL_TRY(api, expr)                                                                    \
  do {                                                                                         \
    int _r = (expr);                                                                           \
    if (_r != 0)                                                                               \
      return fail(PCDN_ECUDA, std::string(#expr) + ": NCCL " + ((api)->GetErrorString ? (api)->GetErrorString(_r) : "error")); \
  } while (0)

template <class T>
inline int dev_alloc(T** p, size_t n) {
  *p = nullptr;
  if (!n) n = 1;
  cudaError_t e = cudaMalloc((void**)p, n * sizeof(T));
  if (e != cudaSuccess) return fail(PCDN_ENOMEM, std::string("cudaMalloc ") + std::to_string(n * sizeof(T)) + " B: " + cudaGetErrorString(e));
  return 0;
}
template <class T>
inline int pin_alloc(T** p, size_t n) {
  *p = nullptr;
  if (!n) n = 1;
  cudaError_t e = cudaHostAlloc((void**)p, n * sizeof(T), cudaHostAllocPortable);
  if (e != cudaSuccess) return fail(PCDN_ENOMEM, std::string("cudaHostAlloc ") + std::to_string(n * sizeof(T)) + " B: " + cudaGetErrorString(e));
  return 0;
}

// pinned + mapped: the device writes through *dev_alias (same bytes the host reads through *p)
template <typename T>
inline int pin_alloc_mapped(T** p, T** dev_alias, size_t n) {
  *p = nullptr;
  if (!n) n = 1;
  cudaError_t e = cudaHostAlloc((void**)p, n * sizeof(T), cudaHostAllocMapped | cudaHostAllocPortable);
  if (e == cudaSuccess) e = cudaHostGetDevicePointer((void**)dev_alias, (void*)*p, 0);
  if (e != cudaSuccess) return fail(PCDN_ENOMEM, std::string("cudaHostAlloc(mapped) ") + std::to_string(n * sizeof(T)) + " B: " + cudaGetErrorString(e));
  return 0;
}

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

enum SlotState { SLOT_FREE = 0, SLOT_OPEN = 1, SLOT_INFLIGHT = 2 };
// shards up to this many connection slots publish spans directly into mapped host memory
constexpr uint32_t kDirectPublishMaxConns = 65536;  // = kSmallCtrlConns: the shards the fused control kernel serves

// One shard's share of a batch slot: the batch as it lies in that GPU's memory, the kernels' scratch
// and the result buffers the host reads.
struct ShardSlot {
  uint8_t* d_arena = nullptr;   // frames, and the descriptor block behind them (one ingest region)
  Work w{};
  BatchIn in{};
  // results
  BatchStats* h_stats = nullptr;      // pinned: final counters (after the pack)
  BatchStats* d_stats_pub = nullptr;  // direct publish: device alias of h_stats (mapped)
  // span table / overflow list of this batch: written by the device straight into mapped host memory
  // (few spans expected) or staged in HBM and copied out while the pack runs (up to 2 per connection)
  bool spans_mapped = false;
  Span* d_spans_map = nullptr; Span* d_spans_dev = nullptr;
  uint32_t* d_ovf_map = nullptr; uint32_t* d_ovf_dev = nullptr;
  BatchStats* h_early = nullptr;  // pinned: counters as of k_offsets (n_spans, n_overflow are final there)
  Span* h_spans = nullptr;        // pinned
  uint32_t* h_overflow = nullptr; // pinned
  int8_t* h_msg_status = nullptr; // pinned
  uint32_t n_msg_errors = 0;
  cudaEvent_t ev_done = nullptr;   // pack + final counters complete (pack stream)
  cudaEvent_t ev_ctrl = nullptr;   // match/plan/offsets complete (main stream)
  cudaEvent_t ev_early = nullptr;  // early counters are in h_early (copy stream)
  cudaEvent_t ev_ingest = nullptr; // the batch has arrived in d_arena (ingest stream)
  cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  bool timed = false;              // the stage events ev[] were recorded for this batch (pcdn_set_timing)
  bool polled = false;             // results of this shard have been fetched
};

// One connection shard: a CUDA device, its streams, its tables and rings.
struct Shard {
  int device = 0;
  uint32_t gindex = 0;           // global shard number inside the broker
  int n_sms = 132;
  bool direct_publish = false;   // spans / overflow list written by the device into mapped host memory
  uint8_t* h_rings = nullptr;    // PCDN_FLAG_HOST_RINGS: host address of the (mapped, pinned) rings
  // main stream: uploads, table updates, direct/match/plan/offsets, release.  pack stream: k_pack, so
  // that the control kernels of batch n+1 overlap the HBM-bound pack of batch n.  copy stream: D2H.
  // ingest stream (sharded): H2D of the staged batch + the NCCL broadcast, ahead of the main stream.
  cudaStream_t stream = nullptr, pack_stream = nullptr, copy_stream = nullptr, ingest_stream = nullptr;
  bool own_stream = false;
  DevState dev{};
  std::vector<ShardSlot> slots;
  // journal staging (pinned + device), reuse guarded by an event
  uint8_t* jstage_h = nullptr; uint8_t* jstage_d = nullptr; size_t jstage_cap = 0;
  cudaEvent_t ev_journal = nullptr; bool ev_journal_pending = false;
  std::vector<Upd32> h_u32;
  NcclComm comm = nullptr;
  int nccl_ranks = 0;
  int prev_slot[2] = {-1, -1};      // the two most recently launched slots (newest first)
  bool fat_only = false;            // the last completed batch packed message-major tiles only (no connection-major message)
  cudaEvent_t ev_submit = nullptr;  // device-input batches: "everything queued on the main stream so far"
  std::vector<void*> dev_allocs, pin_allocs;
};

// host side of a batch slot (shared by all shards)
struct Slot {
  int state = SLOT_FREE;
  uint64_t batch_id = 0;
  bool device_input = false;
  // host staging while open
  uint8_t* h_arena = nullptr;   // pinned: frames, and the descriptor block behind them once the batch is flushed
  size_t arena_used = 0;
  std::vector<uint8_t> kind, flags;
  std::vector<uint32_t> slot_off16, raw_len, aux_off, aux_len, bcast_index;
  std::vector<uint16_t> topics;
  std::vector<SubEvent> events;     // PCDN_FLAG_INBATCH_SUBSCRIBE: subscription events, in the order recorded
  std::vector<uint16_t> ev_topics;  // ... and their topics
  uint32_t n_direct = 0;
  uint32_t n_msgs = 0;
  uint64_t ingress_bytes = 0;   // pool permits held by this batch
  std::chrono::steady_clock::time_point t_launch;
  bool devparse = false;        // some messages carry MSGF_DEVPARSE (k_parse runs first)
  uint32_t max_raw_len = 0;     // host-staged: longest message (with ref_min_bytes: whether k_pack_ref runs)
  bool targeted = false;        // host-staged: some message carries MSGF_TARGET (pcdn_send_to_broker(s))
  bool counted = false;         // counters of this batch have been added to the engine stats
  // merged view of a sharded batch for pcdn_poll (host copy of the shards' span tables)
  std::vector<pcdn_span> merged_spans;
  std::vector<pcdn_span_run> merged_runs;
  std::vector<pcdn_conn> merged_overflow;
};

// One message on its way into a batch (an aggregate: InMsg{} is the empty message).
struct InMsg {
  uint8_t kind, flags;
  bool prune;                        // broadcast: apply Topic::prune to the wire topic list
  bool stage_key;                    // direct: the recipient is copied beside the frame, not read in place
  uint32_t raw_len, key_len;         // key_len: direct message's recipient length (routed_key_len)
  uint32_t target;                   // MSGF_TARGET: the recipient connection (global id), kConnNone = every peer broker
  uint32_t n_listed, n_topics;       // broadcast: entries of the topic list below, entries it adds to the batch
  const uint8_t* raw;
  const uint8_t* key;                // direct: the recipient
  const uint16_t* topic_ids;         // broadcast: the topic ids (API calls), or null and
  const uint8_t* wire_topics;        // a frame's wire topic list, pruned or verbatim
};

// What one message adds to a batch: a 16-byte frame slot (4-byte length hole, raw bytes, zero pad),
// `key_bytes` of recipient key staged beside it (0 when the key is read in place) and topic entries.
// `target`: a MSGF_TARGET message, which takes no memory-pool permits (the reference builds sync frames
// outside the Limiter, tasks/broker/sync.rs:34).
struct MsgShape {
  uint8_t kind;
  uint32_t raw_len, key_bytes, n_topics;
  bool target;
  uint64_t ingress() const { return target ? 0 : raw_len; }
  size_t bytes() const { return align_up(4 + (size_t)raw_len, 16) + key_bytes; }
};

// What the placement scan does with a classified frame or API message:
//   BATCH  place `InMsg` in the open batch;
//   EVENT  (PCDN_FLAG_INBATCH_SUBSCRIBE) a user's Subscribe / Unsubscribe, an event of the open batch;
//   STATE  a Subscribe / Unsubscribe through sub_change (the open batch is launched first, R12);
//   DONE   nothing to place: the result is `rc` (a protocol error with its text `why`, a hook's Skip,
//          1 for a broker frame of another kind).
enum Route : int8_t { ROUTE_BATCH, ROUTE_EVENT, ROUTE_STATE, ROUTE_DONE };
// what the serial placement scan reads and writes per entry (kept small: the scan streams through it;
// the InMsg of entry i lies beside it)
struct Entry {
  Route route;
  bool devparse;      // BATCH: the message carries MSGF_DEVPARSE
  int32_t rc;         // the entry's result, once the scan has handled it
  const char* why;    // DONE with rc < 0: the pcdn_last_error text
  MsgShape shape;     // BATCH; EVENT / STATE: shape.n_topics is the pruned topic count
  uint32_t msg_idx, bcast_pos, topic_off;   // BATCH: its place in the open batch, set by the scan
  uint64_t arena_off;
};

// make `dev` current for the calling thread for the lifetime of the guard (cheap when it already is)
struct DeviceGuard {
  int prev = -1; bool switched = false;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != dev) { cudaSetDevice(dev); switched = true; }
  }
  ~DeviceGuard() { if (switched && prev >= 0) cudaSetDevice(prev); }
};

}  // namespace pcdn_detail
using namespace pcdn_detail;

struct pcdn_engine {
  std::mutex mu;
  pcdn_config cfg{};
  std::string identity;
  std::vector<int32_t> devices;   // owned copy of cfg.devices
  Geometry geo{};                 // GLOBAL geometry (all shards of the broker, local or not)
  std::unique_ptr<HostTables> tables;
  std::unique_ptr<Connections> conns;
  bool has_device = false;
  bool sharded = false;           // the broker has more than one shard (in this or other processes)
  uint32_t world_shards = 1, first_shard = 0;
  uint32_t ingest = PCDN_INGEST_NCCL;
  const NcclApi* nccl = nullptr;
  std::vector<Shard> shards;      // LOCAL shards (global indices first_shard ..)
  std::vector<Slot> slots;
  int open_slot = -1;
  uint64_t next_batch_id = 1;
  std::vector<uint64_t> inflight;  // submit order
  size_t topics_cap = 0;
  size_t frames_cap = 0;          // frame bytes a slot's staging holds (bounds a shared-payload device batch's arena_bytes)
  size_t arena_cap = 0;           // a slot's staging / ingest region: frames_cap, 256-byte alignment, the largest descriptor block
  uint64_t pool_bytes = 0;        // PCDN_FLAG_OUTPUT_POOL: bytes of the output pool per shard
  std::vector<UpdSlot> h_slot; std::vector<uint32_t> h_kslot; std::vector<uint8_t> h_kbytes;  // journal parts common to all shards
  bool timing = false;
  // pcdn_config.pack_variant: CTAs per SM of k_pack (0 = chosen per batch, batch_pack) and of k_pack_direct
  uint32_t pack_ctas = 0, direct_ctas = 8;
  pcdn_message_hook hook[2] = {nullptr, nullptr};  // [origin]: MessageHookDef of user / broker connections
  void* hook_user[2] = {nullptr, nullptr};
  uint64_t inflight_bytes = 0;  // Limiter analogue: accepted frame bytes whose batch is not released yet
  pcdn_stats stats{};
  // receive / handle / submit scratch: the classified entries of a call and their messages.  Left
  // uninitialised (a large call pays no clearing); kept for the next call while they hold at most kRxKeep
  // entries, so small calls allocate nothing, and freed at the end of a larger call.
  static constexpr uint32_t kRxKeep = 1u << 16;
  std::unique_ptr<Entry[]> rx_plan;
  std::unique_ptr<InMsg[]> rx_msgs;
  uint32_t rx_cap = 0;
  void rx_reserve(uint32_t n) {
    if (n > rx_cap) { rx_plan.reset(new Entry[n]); rx_msgs.reset(new InMsg[n]); rx_cap = n; }
  }
  void rx_release() {
    if (rx_cap > kRxKeep) { rx_plan.reset(); rx_msgs.reset(); rx_cap = 0; }
  }
  std::vector<uint16_t> rx_topics;   // a Subscribe's pruned topics
  struct HookScratch {               // a hooked frame's private topic list, and the text of a hook's error
    std::vector<uint8_t> topics;
    std::string err;
  } rx_hook;
  // buffers behind pcdn_get_*_sync
  std::vector<UserSyncEntry> sync_users;
  std::vector<pcdn_user_sync_entry> sync_users_c;
  std::vector<TopicSyncEntry> sync_topics;
  std::vector<pcdn_topic_sync_entry> sync_topics_c;

  bool owns_root() const { return first_shard == 0; }   // this process holds global shard 0 (ingest root)
  // some deliveries are reference records, resolved through the batch's host payload (pcdn_batch_payload)
  bool delivers_by_ref() const { return (cfg.flags & PCDN_FLAG_SHARED_PAYLOAD) || cfg.ref_min_bytes; }
  uint32_t shard_N() const { return geo.shard_N; }
  uint32_t shard_W() const { return geo.shard_N / 32; }
};


namespace pcdn_detail {
int find_slot_index(pcdn_engine* e, uint64_t id);
// wait for (or test) one local shard's share of a batch and fetch its results (1 = not done yet)
int poll_one(pcdn_engine* e, uint64_t batch_id, uint32_t li, int block);
}  // namespace pcdn_detail
