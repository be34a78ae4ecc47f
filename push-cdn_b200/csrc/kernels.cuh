// kernels.cuh — device-side data layout and kernel launchers of the fan-out engine (sm_90a).
//
// Per batch the engine runs (all on one stream, no host round trip in between):
//   K0  k_parse         (device-parse mode) thread per frame: Cap'n Proto walk, Topic::prune, recipient
//   K3  k_direct_lookup 8 lanes per direct message: cuckoo probe pubkey → route → target connection,
//                       hit count per connection
//       k_dscan/k_dfill counts → segment starts (one scan launch), message indices dropped into their
//                       connection's segment (no sort: the connection's thread orders its few entries
//                       in k_offsets; k_dsort_hot orders connections with > 32 hits by bitmap)
//   K1a k_match         OR of subscription-bitmap rows per broadcast → match words + popcount ranks
//                       (bits of connections with in-batch subscription events re-evaluated per message;
//                       a MSGF_TARGET message's row is the broker mask or its one target connection's bit)
//   K1p k_plan_*        D_m per message, class (thin / message-major / connection-major), scatter-list
//                       bases and pack tiles by prefix sums (one launch when <= 256 messages)
//   K1b k_offsets       thread per connection walks the batch IN ORDER (R9), assigns ring offsets and
//                       writes each offset at its deterministic rank in the per-message scatter list
//   K2  k_pack          persistent CTAs, three phases: connection-major (groups of <= 8 small frames
//                       staged by TMA, one TMA bulk store per contiguous run of a connection's
//                       records), message-major (16 KiB chunks staged once per CTA, replicated to
//                       ~128 KB worth of recipients per tile), thin (warp per delivery), direct (warp
//                       per message; its own full-occupancy launch k_pack_direct for batches of >= 2048
//                       direct messages)
//   K2r k_pack_ref      thread per delivery over the three scatter lists, one 32-byte reference record for each
//                       delivery of a by-reference message (the payload stays once per batch).  Replaces K2 on
//                       PCDN_FLAG_SHARED_PAYLOAD engines; follows K2 on engines with a ref_min_bytes threshold
//   K1s k_ctrl_small    latency path (N <= 65536 connection slots, <= 256 messages): K3 + sort + K1a +
//                       K1p + K1b in ONE cluster launch, counters/spans published to mapped host memory
//   K4  k_apply_*       scatter of changed table words/slots (subscribe, add/remove, direct map)
//       k_release       ring space of a consumed batch goes back to the connections
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "hash.h"

namespace pcdn {

constexpr uint32_t kUnit = 32;               // record alignment in ring (bytes) = PCDN_RECORD_ALIGN
constexpr uint32_t kOffInvalid = 0xFFFFFFFFu;
// Work::cmrun: kCmBroken | p = the (group, connection) pair is one run up to group position p only.  Never a
// unit offset: a ring holds at most 2 GiB = 2^26 units, a connection's pool region less than 2^31.
constexpr uint32_t kCmBroken = 0xFFFFFFF0u;
constexpr uint32_t kConnNone = 0xFFFFFFFFu;
constexpr uint32_t kFatMin = 32;             // >= this many recipients → staged (fat) path
constexpr uint32_t kChunkBytes = 16384;      // shared-memory staging chunk of the fat path
constexpr uint32_t kTileRecipients = 1024;   // most recipients per fat tile
constexpr uint32_t kFatTileBytes = 131072;   // bytes of stores a fat tile aims at (kernels.cu: tile_recipients)
constexpr uint32_t kBlockWords = 256;        // bitmap words per match block (8192 connections)
// connection-major (cm) pack path: dense messages with small records are grouped and written
// connection by connection, so that one connection's records form ONE contiguous run in its ring
constexpr uint32_t kCmGroup = 8;             // messages staged together in shared memory
constexpr uint32_t kCmMaxBytes = 4096;       // largest padded record that takes the cm path
constexpr uint32_t kSmallCtrlConns = 65536;   // largest geometry served by the fused control kernel (<= 8 match blocks per message)
constexpr uint32_t kSmallCtrlMsgs = 256;      // largest batch it takes
constexpr uint32_t kSmallCtrlItems = 256;     // ... and at most this many (broadcast, 8192-connection block) match items
constexpr uint32_t kThinSeparateMin = 2048;  // direct messages in a batch from which the direct pack gets its own launch
constexpr uint32_t kPackRefCtas = 8;         // CTAs per SM of k_pack_ref (pack_variant does not set them)
constexpr uint32_t kHotMin = 32;             // more direct hits than this on one connection: ordered by k_dsort_hot
constexpr uint32_t kHotCtas = 32;            // CTAs (and bitmap scratch rows) of k_dsort_hot
constexpr uint32_t kCmTileWords = 16;        // bitmap words (512 connections) per cm tile
constexpr uint32_t kCmDenseShift = 4;        // cm needs D >= N/16 recipients
enum : uint8_t { CLS_THIN = 0, CLS_FAT = 1, CLS_CM = 2 };
// per-message flag bits (BatchIn::flags); bit 0 = PCDN_TO_USERS_ONLY
enum : uint8_t {
  MSGF_USERS_ONLY = 1,
  MSGF_DEVPARSE = 2,   // k_parse fills kind / aux_off / aux_len from the raw frame
  MSGF_TOPICS_U8 = 4,  // aux_off = byte offset in the arena of the wire topic list (u8 each)
  MSGF_PRUNE = 8,      // user-origin: apply Topic::prune while reading the wire topic list
  // pcdn_send_to_broker(s): a broadcast slot whose match row is its target, not topic rows: aux_off = the target's
  // global connection id, or kConnNone for every peer broker of the shard; aux_len = 0.  Read only by the
  // instantiations a batch holding such a message selects (launch_match / launch_ctrl_small: `targeted`)
  MSGF_TARGET = 16
};
constexpr int8_t kErrParse = -7, kErrPrune = -8;  // PCDN_EPARSE / PCDN_EPRUNE

// device-resident routing state + rings
struct DevState {
  uint32_t* sub;         // [T][W] subscription bitmap, row = topic
  uint32_t* brk;         // [W]    1 = connection is a peer broker
  uint32_t* owner_conn;  // [max_owners] broker owner index → its connection (or NONE)
  CuckooEntry* cuckoo;   // [nbuckets*4]
  uint8_t* keys;         // [max_keys][key_stride]
  uint32_t* ptail;       // [N] next free unit in the connection's ring
  uint32_t* used;        // [N] units not yet released
  uint8_t* rings;        // [max_conns][ring_bytes]
  uint32_t N, W, T, nblk;
  uint32_t bucket_mask, key_stride;
  uint32_t ring_units;   // ring_bytes / 32
  uint32_t n_valid_topics;  // Topic::prune validity bound (0 = all)
  uint32_t max_key_len;
  uint64_t seed;
  // (seed sits here so that the fields below keep their offsets: with them 12 bytes lower, k_offsets<false>
  //  compiled to 40 registers instead of 32, i.e. 6 CTAs per SM instead of 8, and ran measurably slower)
  // connection shards (SURVEY 8e): this GPU owns the connection ids [conn_base, conn_base + N).  The
  // bitmap / broker-mask words here are this shard's slice (local word index); the direct map and
  // owner_conn[] are replicated on every shard and name connections by GLOBAL id, so a direct
  // message resolves identically everywhere and is packed by the shard that owns the target.
  // PCDN_FLAG_OUTPUT_POOL: instead of one fixed ring per connection, `rings` is ONE output pool of
  // pool_units x 32 B shared by all connections of the shard.  Every batch gets a contiguous region,
  // laid out connection by connection (a connection's records back to back, in batch order); the
  // region is freed as a whole when the batch is released.  No connection can overflow; a batch
  // that does not fit is refused as a whole (status 2) and retried after older ones are released.
  uint32_t pool;
  uint32_t pool_units;       // capacity of the pool in 32-byte units
  struct PoolState* pool_state;
  uint32_t conn_base;
  uint32_t span_runs;    // PCDN_FLAG_SPAN_RUNS: the span table is run-length encoded (SpanRun entries)
  uint32_t count_drops;  // 1 on exactly one shard of the broker (global shard 0): it counts the unroutable directs
  // a message of raw_len >= ref_min is delivered as one 32-byte reference record (k_pack_ref), a shorter one as a
  // framed copy (kernels.cu: by_ref): 0 = every message (PCDN_FLAG_SHARED_PAYLOAD), 0xFFFFFFFF = none (copy mode),
  // else pcdn_config.ref_min_bytes
  uint32_t ref_min;
  uint64_t ring_bytes;
};

// PCDN_FLAG_INBATCH_SUBSCRIBE: a subscription change recorded inside a batch.  It applies to the batch's
// messages at index >= position; the match of every other message reads the bitmap as it was when the
// batch was opened.  Events are sorted by (conn, position), so a connection's events are one run.
struct SubEvent {
  uint32_t conn;     // global connection id
  uint32_t pos_op;   // bits 0..30: position (messages in the batch when it was recorded); bit 31: 1 = subscribe
  uint32_t toff;     // first topic in the batch's event topic list (u16 each)
  uint32_t tn;       // topics
};
constexpr uint32_t kEvSubscribe = 0x80000000u;

// inputs of one batch (device pointers) — same meaning as pcdn_device_batch
struct BatchIn {
  uint32_t n_msgs, n_bcast;
  const uint8_t* arena;
  const uint8_t* kind;
  const uint8_t* flags;
  const uint32_t* slot_off16;
  const uint32_t* raw_len;
  const uint32_t* aux_off;
  const uint32_t* aux_len;
  const uint16_t* topics;
  const uint32_t* bcast_index;
  // in-batch subscription events (0 unless PCDN_FLAG_INBATCH_SUBSCRIBE)
  uint32_t n_events;
  const SubEvent* events;
  const uint16_t* ev_topics;
};

struct BatchStats {
  unsigned long long n_deliveries;
  unsigned long long bytes_out;
  uint32_t n_spans;
  uint32_t n_overflow;
  uint32_t n_direct_dropped;
  uint32_t status;          // 0 ok, 1 = scatter list capacity exceeded (E2BIG)
  uint32_t n_fat_entries;
  uint32_t n_thin_entries;
  uint32_t n_fat_tiles;
  uint32_t tile_cursor;
  uint32_t n_cm;            // messages on the connection-major path
  uint32_t cm_cursor;
  uint32_t n_hot;           // connections with more than kHotMin direct hits in this batch
  uint32_t n_runs;          // run-length entries written to the span table (span_runs engines)
  uint32_t pool_base;       // pool mode: first unit of this batch's region (span offsets are relative to it)
  uint32_t pool_units;      // pool mode: units of the region
  uint32_t pool_skip;       // pool mode: units skipped at the end of the pool to keep the region contiguous
  uint32_t ctas_done;       // CTAs of the kernel that ends the batch that have finished (the last one publishes)
};

// ring buffer of batch regions inside the output pool (units of 32 B); batches are released in order
struct PoolState { uint32_t head, tail, used, blocked; };

struct Span { uint32_t conn, ring_off, len, n_records; };
// n_conns consecutive connection ids that each own an identical span (same offset, length, records):
// a dense broadcast batch is 1 run per 256 connections instead of one 16-byte span per connection
// (off_stride: units added to ring_off per connection — 0 with per-connection rings, where every
//  connection of the run has the records at the same offset of its own ring; len / 32 in pool mode,
//  where the connections' regions follow each other)
struct SpanRun { uint32_t conn0, n_conns, ring_off, len, n_records, off_stride; };

// per-slot scratch
struct Work {
  uint32_t* B;           // [max_bcast][W] match words
  uint16_t* wpre;        // [max_bcast][W] exclusive popcount prefix inside the 256-word block
  uint32_t* cnt;         // [max_bcast][nblk]
  uint32_t* base;        // [max_bcast][nblk] exclusive prefix of cnt over blocks
  uint32_t* done;        // [max_bcast] finished match blocks of a message (k_match; zero between batches)
  uint32_t* D;           // [max_msgs] recipients per message
  uint32_t* dconn;       // [max_msgs] direct: target connection or NONE
  uint32_t* eb_fat;      // [max_msgs+1] scatter-list base per message (fat list)
  uint32_t* eb_thin;     // [max_msgs+1]
  uint32_t* tbase;       // [max_msgs+1] fat tile base per message
  uint32_t* scan_tmp;    // [4 * nscanblk] block totals of the plan scan
  uint8_t* cls;          // [max_msgs] CLS_THIN / CLS_FAT / CLS_CM
  uint32_t* cm_rank;     // [max_msgs+1] rank among cm messages
  uint32_t* cm_list;     // [max_bcast] cm rank → message index
  uint32_t* jidx;        // [max_msgs] message index → broadcast slot j
  uint2* efat;           // [cap_fat]  {conn, ring offset in units} — message-major (fat) class
  uint32_t* ecm;         // [cap_fat]  ring offset in units — connection-major class (the connection is
                         //            implied by the rank, so 4 bytes per delivery instead of 8); written only
                         //            where cmrun says so
  uint32_t* cmrun;       // [min(MB/8 groups * N, 2 * cap_fat + N)] at g * N + c: the first unit of connection c's
                         //            records of connection-major group g (kCmGroup messages in cm rank order) when
                         //            they are ONE contiguous run in group order; kCmBroken | p when they are one
                         //            run only up to group position p (a wrap, another record of c in between, an
                         //            overflow): ecm then holds the first record's offset and those from p on.
                         //            Unset when c matches nothing of the group.
  uint4* ethin;          // [cap_thin] {conn, ring offset in units, slot_off16, raw_len}
  uint32_t cap_fat, cap_thin;
  // Direct hits grouped by target connection WITHOUT a sort: the lookup counts hits per connection
  // (dcount), one scan turns the counts into segment starts (dloc + dtile), a fill pass drops every
  // message index into its connection's segment of dlist (atomic slot: arbitrary order), and the
  // connection's own thread in k_offsets puts its handful of entries into batch order (R9).
  // Connections with more than kHotMin hits are ordered by k_dsort_hot before that.
  uint32_t* dcount;      // [N+2] hits per connection (zeroed per batch)
  uint32_t* dloc;        // [N+2] exclusive prefix of dcount inside its 1024-entry tile
  uint32_t* dtile;       // [N/1024+3] exclusive prefix of the tile totals (raw totals until the last CTA of k_dscan has run)
  uint32_t* dlist;       // [max_msgs] message indices grouped by connection
  uint32_t* hot_list;    // [max_msgs/kHotMin+1] connections with more than kHotMin hits
  uint32_t* hot_bitmap;  // [kHotCtas][max_msgs/32+1] scratch of k_dsort_hot
  uint32_t* scan_done;   // finished tiles of k_dscan (zero between batches)
  uint2* edir;           // [max_msgs] direct message m → {connection, ring offset in units}; offset invalid = not delivered by this shard
  // fused small-engine path: the (connection, message) order comes from a rank sort inside the kernel
  // and the segment bounds are sparse (valid iff dstamp == stamp: nothing to clear between batches)
  uint32_t* dstart;      // [N+1]
  uint32_t* dend;        // [N+1]
  uint32_t* dstamp;      // [N+1]
  uint32_t stamp;        // per-slot batch counter (never 0)
  // pool mode: connection c's region starts at pool_base + cbase[c]; the CTAs of k_offsets chain their
  // totals with a decoupled look-back (lb_state: stamp | flag | value per CTA, no clearing)
  uint32_t* cbase;       // [N]
  unsigned long long* lb_state;  // [N / 256 + 1] look-back words (fused small-engine kernel)
  uint32_t* lb_tot;      // [N / 256 + 1] units per k_offsets CTA (regular kernel; finished by k_pool_finish)
  uint32_t pool_unblock; // this launch is the retry of the oldest refused batch: clear PoolState::blocked
  unsigned long long batch_id;  // the batch this launch packs (k_pack_ref writes it into every reference record)
  // outputs
  uint32_t* batch_units; // [N] units consumed by this batch per connection (for release)
  Span* spans;           // [2*N] spans, or (span_runs) [2*N] SpanRun entries in the same buffer (sized for the larger)
  uint32_t* overflow;    // [max_conns]
  int8_t* msg_status;    // [max_msgs] device-parse outcome per message
  BatchStats* stats;
};

// table-update journal records (K4)
struct Upd32 { uint32_t arr, idx, val; };   // arr: 0 sub, 1 brk, 2 owner_conn
struct UpdSlot { uint32_t slot; CuckooEntry e; };

// ---- launchers (host functions defined in kernels.cu) -------------------------------------------
void launch_apply_updates(const DevState& s, const Upd32* u32, uint32_t n32, const UpdSlot* us,
                          uint32_t nslot, const uint32_t* key_slots, const uint8_t* key_bytes,
                          uint32_t nkeys, cudaStream_t st);
void launch_parse(const DevState& s, const Work& w, const BatchIn& b, cudaStream_t st);
void launch_direct(const DevState& s, const Work& w, const BatchIn& b, uint32_t n_direct, cudaStream_t st);
// zero: the batch's counters when k_match / k_ctrl_small zeroes them, else null (engine.cu: counters_zeroer)
// targeted: the batch holds a MSGF_TARGET message (host-staged batches only)
void launch_match(const DevState& s, const Work& w, const BatchIn& b, BatchStats* zero, bool targeted, cudaStream_t st);
void launch_plan(const DevState& s, const Work& w, const BatchIn& b, cudaStream_t st);
void launch_offsets(const DevState& s, const Work& w, const BatchIn& b, bool has_direct, int n_sms, cudaStream_t st);
// fused match + plan + offsets for N <= kSmallCtrlConns, n_msgs <= kSmallCtrlMsgs and at most kSmallCtrlItems
// match items (one cluster launch)
void launch_ctrl_small(const DevState& s, const Work& w, const BatchIn& b, bool has_direct, bool targeted, BatchStats* zero,
                       BatchStats* publish, bool offsets_only, cudaStream_t st);
// pool mode: reset what the offsets pass and the pack count before the retry of a refused batch
void launch_pool_retry_begin(const DevState& s, const Work& w, cudaStream_t st);
// publish (mapped host memory, or null): the last pack kernel copies the batch's final counters there, or a copy on `st`
// when the batch launches none.  pack_ctas / direct_ctas: CTAs per SM of k_pack / k_pack_direct (they change how the
// work is shared, not what is written).  has_ref: the batch may hold a message delivered by reference (k_pack_ref
// follows the copy packs; shared-payload engines ignore it)
void launch_pack(const DevState& s, const Work& w, const BatchIn& b, uint32_t n_direct, uint32_t pack_ctas, uint32_t direct_ctas,
                 int n_sms, bool has_ref, BatchStats* publish, cudaStream_t st);
void launch_release(const DevState& s, const uint32_t* batch_units, const BatchStats* stats, cudaStream_t st);
void launch_pool_init(const DevState& s, cudaStream_t st);
unsigned long long kernel_launches();   // launches issued by this library in this process so far
void count_kernel_launch();

}  // namespace pcdn
