// engine.cu — host runtime of the fan-out engine and the C ABI (include/pcdn_fanout.h).
//
// One engine = one logical broker: ONE host mirror of the routing tables (host_state.*) and ONE
// connection-id space, spread over one or more connection SHARDS.  A shard = one CUDA device with
// its streams, its slice of the subscription bitmap, a replica of the direct map, the output rings
// of its connections and its share of every batch slot.  A batch is staged in pinned memory while it
// is open, brought to every shard on flush (one H2D for a single shard; H2D to shard 0 + ONE
// ncclBroadcast over NVLink for several), routed there by the kernel pipeline of kernels.cuh, and
// its results (span table, counters) come back through pinned memory per shard.
// There is no CPU data path: without a device every routing call fails with PCDN_ENODEV.
#include "engine_internal.h"

namespace pcdn_detail {
thread_local std::string g_err;
int fail(int code, const std::string& msg) { g_err = msg; return code; }
}  // namespace pcdn_detail

namespace {

// Upload changed table words/slots/keys and apply them on every local shard's stream (K4).  Stream
// order gives R12: every earlier batch sees the old tables, every later batch the new ones.  A
// shard's bitmap / broker mask are its word slice of the global arrays; owner_conn, the cuckoo
// slots and the key arena are replicated.
int flush_journal(pcdn_engine* e) {
  HostTables& t = *e->tables;
  if (!e->has_device) { t.clear_dirty(); return 0; }
  const Geometry& g = e->geo;
  bool any = !t.dirty_sub.empty() || !t.dirty_brk.empty() || !t.dirty_owner.empty() || !t.dirty_slots.empty() ||
             !t.dirty_keys.empty();
  if (!any) return 0;
  const uint32_t Ws = e->shard_W(), W = g.W;
  const bool full_keys = t.dirty_keys.size() > (size_t)g.max_keys / 16 + 64;
  const bool full_sub = t.dirty_sub.size() > t.sub.size() / 16 + 64;
  const bool full_slots = t.dirty_slots.size() > t.cuckoo.size() / 16 + 64;
  // parts common to all shards
  e->h_slot.clear(); e->h_kslot.clear(); e->h_kbytes.clear();
  if (!full_slots) for (uint32_t i : t.dirty_slots) e->h_slot.push_back(UpdSlot{i, t.cuckoo[i]});
  if (!full_keys) for (uint32_t k : t.dirty_keys) {
    e->h_kslot.push_back(k);
    size_t at = e->h_kbytes.size();
    e->h_kbytes.resize(at + g.key_stride);
    std::memcpy(&e->h_kbytes[at], &t.keys[(size_t)k * g.key_stride], g.key_stride);
  }
  for (Shard& sh : e->shards) {
    DeviceGuard dg(sh.device);
    cudaStream_t st = sh.stream;
    const uint32_t w0 = sh.gindex * Ws;
    // keys first (slots reference them)
    if (full_keys) CUDA_TRY(cudaMemcpyAsync(sh.dev.keys, t.keys.data(), t.keys.size(), cudaMemcpyHostToDevice, st));
    sh.h_u32.clear();
    if (full_sub) {
      if (Ws == W) CUDA_TRY(cudaMemcpyAsync(sh.dev.sub, t.sub.data(), t.sub.size() * 4, cudaMemcpyHostToDevice, st));
      else CUDA_TRY(cudaMemcpy2DAsync(sh.dev.sub, (size_t)Ws * 4, t.sub.data() + w0, (size_t)W * 4, (size_t)Ws * 4, g.T, cudaMemcpyHostToDevice, st));
    } else {
      for (uint32_t i : t.dirty_sub) {
        const uint32_t row = i / W, wd = i % W;
        if (wd >= w0 && wd < w0 + Ws) sh.h_u32.push_back(Upd32{0, row * Ws + (wd - w0), t.sub_upload(i)});
      }
    }
    if (full_sub)   // words the open batch's events changed keep their value before the events (HostTables::hold)
      for (const auto& h : t.held_sub) {
        const uint32_t row = h.first / W, wd = h.first % W;
        if (wd >= w0 && wd < w0 + Ws) sh.h_u32.push_back(Upd32{0, row * Ws + (wd - w0), h.second});
      }
    for (uint32_t i : t.dirty_brk)
      if (i >= w0 && i < w0 + Ws) sh.h_u32.push_back(Upd32{1, i - w0, t.brk[i]});
    for (uint32_t i : t.dirty_owner) sh.h_u32.push_back(Upd32{2, i, t.owner_conn[i]});
    if (full_slots) CUDA_TRY(cudaMemcpyAsync(sh.dev.cuckoo, t.cuckoo.data(), t.cuckoo.size() * sizeof(CuckooEntry), cudaMemcpyHostToDevice, st));
    // One pinned staging block [Upd32 | UpdSlot | key slots | key bytes] → one H2D copy → apply kernels.
    // The staging block is reused by the next flush; an event (not a stream sync) guards it, so table
    // churn at control-plane rate never stalls the batches already queued on the stream.
    const size_t b_u32 = align_up(sh.h_u32.size() * sizeof(Upd32), 16), b_slot = align_up(e->h_slot.size() * sizeof(UpdSlot), 16);
    const size_t b_ks = align_up(e->h_kslot.size() * 4, 16), b_kb = align_up(e->h_kbytes.size(), 16);
    const size_t total = b_u32 + b_slot + b_ks + b_kb;
    if (total) {
      if (sh.ev_journal_pending) { CUDA_TRY(cudaEventSynchronize(sh.ev_journal)); sh.ev_journal_pending = false; }
      if (total > sh.jstage_cap) {
        const size_t ncap = std::max(total, sh.jstage_cap * 2 + (1 << 16));
        CUDA_TRY(cudaStreamSynchronize(st));
        if (sh.jstage_h) cudaFreeHost(sh.jstage_h);
        if (sh.jstage_d) cudaFree(sh.jstage_d);
        sh.jstage_h = nullptr; sh.jstage_d = nullptr; sh.jstage_cap = 0;
        CUDA_TRY(cudaMallocHost((void**)&sh.jstage_h, ncap));
        CUDA_TRY(cudaMalloc((void**)&sh.jstage_d, ncap));
        sh.jstage_cap = ncap;
      }
      uint8_t* h = sh.jstage_h;
      if (b_u32) std::memcpy(h, sh.h_u32.data(), sh.h_u32.size() * sizeof(Upd32));
      if (b_slot) std::memcpy(h + b_u32, e->h_slot.data(), e->h_slot.size() * sizeof(UpdSlot));
      if (b_ks) std::memcpy(h + b_u32 + b_slot, e->h_kslot.data(), e->h_kslot.size() * 4);
      if (b_kb) std::memcpy(h + b_u32 + b_slot + b_ks, e->h_kbytes.data(), e->h_kbytes.size());
      CUDA_TRY(cudaMemcpyAsync(sh.jstage_d, h, total, cudaMemcpyHostToDevice, st));
      uint8_t* d = sh.jstage_d;
      launch_apply_updates(sh.dev, (const Upd32*)d, (uint32_t)sh.h_u32.size(), (const UpdSlot*)(d + b_u32), (uint32_t)e->h_slot.size(),
                           (const uint32_t*)(d + b_u32 + b_slot), d + b_u32 + b_slot + b_ks, (uint32_t)e->h_kslot.size(), st);
      CUDA_TRY(cudaGetLastError());
      CUDA_TRY(cudaEventRecord(sh.ev_journal, st));
      sh.ev_journal_pending = true;
    }
    // whole-table uploads come from pageable vectors (staged by the runtime before the call returns);
    // they only happen on bulk loads, where one synchronisation is irrelevant
    if (full_keys || full_sub || full_slots) CUDA_TRY(cudaStreamSynchronize(st));
  }
  t.clear_dirty();
  return 0;
}

void slot_reset_open(Slot& s) {
  s.arena_used = 0; s.n_direct = 0; s.devparse = false; s.ingress_bytes = 0; s.n_msgs = 0; s.max_raw_len = 0; s.targeted = false;
  s.kind.clear(); s.flags.clear(); s.slot_off16.clear(); s.raw_len.clear(); s.aux_off.clear(); s.aux_len.clear();
  s.bcast_index.clear(); s.topics.clear(); s.events.clear(); s.ev_topics.clear();
  s.device_input = false; s.counted = false;
}

int acquire_open_slot(pcdn_engine* e) {
  if (e->open_slot >= 0) return 0;
  for (size_t i = 0; i < e->slots.size(); i++)
    if (e->slots[i].state == SLOT_FREE) {
      e->open_slot = (int)i;
      e->slots[i].state = SLOT_OPEN;
      slot_reset_open(e->slots[i]);
      return 0;
    }
  return fail(PCDN_EAGAIN, "all batch slots are in flight: poll and release a batch first");
}

// drop the open batch (nothing of it has been launched) and give its permits back
void abandon_open(pcdn_engine* e) {
  if (e->open_slot < 0) return;
  Slot& s = e->slots[e->open_slot];
  e->tables->release_held();   // its events' changes reach the device before the next batch
  e->inflight_bytes -= std::min(e->inflight_bytes, s.ingress_bytes);
  e->stats.bytes_in -= std::min(e->stats.bytes_in, s.ingress_bytes);
  slot_reset_open(s);
  s.state = SLOT_FREE;
  e->open_slot = -1;
}

// Descriptor block of a batch: its per-message arrays at these offsets from the block's base (host-staged
// batches, and device-resident ones as sharded engines replicate them)
// (PCDN_FLAG_INBATCH_SUBSCRIBE: the subscription events and their topics follow the message topics)
struct DescLayout {
  uint32_t n_msgs, n_bcast, n_events;
  size_t o_kind, o_flags, o_slot, o_len, o_aoff, o_alen, o_bidx, o_top, o_ev, o_etop, total;
  DescLayout(uint32_t n, uint32_t nb, size_t n_topics, uint32_t n_ev = 0, size_t n_ev_topics = 0) : n_msgs(n), n_bcast(nb), n_events(n_ev) {
    o_kind = 0; o_flags = align_up(o_kind + n, 16); o_slot = align_up(o_flags + n, 16);
    o_len = o_slot + (size_t)n * 4; o_aoff = o_len + (size_t)n * 4; o_alen = o_aoff + (size_t)n * 4;
    o_bidx = o_alen + (size_t)n * 4; o_top = align_up(o_bidx + (size_t)nb * 4, 16);
    o_ev = align_up(o_top + n_topics * 2, 16); o_etop = o_ev + (size_t)n_ev * sizeof(SubEvent);
    total = align_up(o_etop + n_ev_topics * 2, 16);
  }
};

// the kernels' view of a batch whose frames lie at `arena` and whose descriptor block lies at `desc`
BatchIn bind_batch(const uint8_t* arena, const uint8_t* desc, const DescLayout& L) {
  return BatchIn{L.n_msgs, L.n_bcast, arena, desc + L.o_kind, desc + L.o_flags, (const uint32_t*)(desc + L.o_slot),
                 (const uint32_t*)(desc + L.o_len), (const uint32_t*)(desc + L.o_aoff), (const uint32_t*)(desc + L.o_alen),
                 (const uint16_t*)(desc + L.o_top), (const uint32_t*)(desc + L.o_bidx),
                 L.n_events, (const SubEvent*)(desc + L.o_ev), (const uint16_t*)(desc + L.o_etop)};
}

// The adaptive pack-stream overlap applies to batches whose previous output was at most this many bytes.
// With every step queued ahead, overlapped packs can lose the launch race against the next control stage
// and run much longer; the overlap hides at most the short control stage, so it stops paying for long packs.
static constexpr unsigned long long kOverlapMaxBytes = 3ull << 29;

// Who zeroes a batch's counters (BatchStats): the first CTA of its first kernel, k_ctrl_small or k_match, unless k_parse
// or the regular direct lookup counts into them first from many CTAs, or no k_match runs: then a memset.  A retry zeroes
// nothing: the counters keep the plan's totals, and k_pool_retry_begin resets what offsets and pack count.
enum : uint8_t { ZERO_NONE, ZERO_MEMSET, ZERO_MATCH, ZERO_CTRL_SMALL };
uint8_t counters_zeroer(const Slot& hs, const BatchIn& in, bool fused, bool retry) {
  if (retry) return ZERO_NONE;
  if (hs.devparse || (!fused && (hs.n_direct || !in.n_bcast))) return ZERO_MEMSET;
  return fused ? ZERO_CTRL_SMALL : ZERO_MATCH;
}

// begin: the pack-stream prediction, the ingest wait, the launch's stamp and batch id, the span path
int batch_begin(pcdn_engine* e, Shard& sh, uint32_t si, bool fused, bool wait_ingest, bool retry) {
  ShardSlot& s = sh.slots[si];
  // Broadcast batches: running the next batch's control stage beside this batch's pack helps when the pack is short
  // and message-major (sparse fan-out, config 5) and hurts a long pack, which then shares SMs and HBM with it (config
  // 5 dense, C2).  Which one this batch will be is decided on the device, so the class mix and size of the most recent
  // COMPLETED batch of this shard predict it (a workload changes its mix rarely; a wrong guess costs a few percent).
  if (!sh.direct_publish && s.in.n_bcast > 0) {
    for (int k = 0; k < 2; k++) {
      const int pv = sh.prev_slot[k];
      if (pv < 0 || pv == (int)si) continue;
      const ShardSlot& o = sh.slots[pv];
      if (cudaEventQuery(o.ev_done) != cudaSuccess) { cudaGetLastError(); continue; }
      const BatchStats& ps_ = *o.h_stats;
      // (message-major entries, not tiles: a message delivered by reference has its entries but no tile)
      sh.fat_only = ps_.status == 0 && ps_.n_cm == 0 && ps_.n_fat_entries > 0 && ps_.bytes_out <= kOverlapMaxBytes;
      break;
    }
  }
  sh.prev_slot[1] = sh.prev_slot[0]; sh.prev_slot[0] = (int)si;
  if (wait_ingest) CUDA_TRY(cudaStreamWaitEvent(sh.stream, s.ev_ingest, 0));
  s.timed = e->timing; s.polled = false; s.n_msg_errors = 0;
  // validity stamp of the batch's direct buckets / look-back words (a retry keeps it: its direct bounds stay valid)
  if (!retry && ++s.w.stamp == 0) s.w.stamp = 1;
  if (!retry && sh.dev.pool && (s.w.stamp & 0x3FFFFFFFu) == 0) {   // the look-back words carry 30 bits of it
    s.w.stamp++;
    CUDA_TRY(cudaMemsetAsync(s.w.lb_state, 0, ((size_t)sh.dev.N / 256 + 1) * 8, sh.stream));
  }
  s.w.pool_unblock = retry ? 1u : 0u;
  s.w.batch_id = retry ? e->slots[si].batch_id : e->next_batch_id;   // (launch_pipeline hands out next_batch_id)
  // Spans go straight into mapped host memory when few are expected (16-byte PCIe writes: a table of 16 K spans is
  // slower than the staged copy): the smallest geometry, or a batch without broadcasts and with few messages (at most
  // one span per message).  Otherwise they are staged in HBM and copied out with one DMA of the exact size while the pack runs.
  s.spans_mapped = sh.direct_publish && (sh.dev.N <= 8192 || (s.in.n_bcast == 0 && s.in.n_msgs <= 4096));
  if (sh.dev.pool && !fused) s.spans_mapped = false;   // k_pool_finish patches the table: keep it in HBM until it is final
  s.w.spans = s.spans_mapped ? s.d_spans_map : s.d_spans_dev;
  s.w.overflow = s.spans_mapped ? s.d_ovf_map : s.d_ovf_dev;
  if (s.timed) CUDA_TRY(cudaEventRecord(s.ev[0], sh.stream));
  return 0;
}

// control: route the batch (parse, direct lookup, match, plan: everything that reads the tables) and place it
// (offsets).  retry: a batch the output pool refused keeps its routing; only the offsets (+ pool finish) run again.
int batch_control(Shard& sh, ShardSlot& s, const Slot& hs, bool fused, bool retry) {
  cudaStream_t st = sh.stream;
  const uint8_t zero = counters_zeroer(hs, s.in, fused, retry);
  if (retry) {
    launch_pool_retry_begin(sh.dev, s.w, st);
  } else {
    if (zero == ZERO_MEMSET) CUDA_TRY(cudaMemsetAsync(s.w.stats, 0, sizeof(BatchStats), st));
    if (hs.devparse) launch_parse(sh.dev, s.w, s.in, st);
    if (hs.n_direct && !fused) launch_direct(sh.dev, s.w, s.in, hs.n_direct, st);  // fused: lookup + sort inside k_ctrl_small
  }
  if (s.timed) CUDA_TRY(cudaEventRecord(s.ev[1], st));
  if (fused) {
    launch_ctrl_small(sh.dev, s.w, s.in, hs.n_direct > 0, hs.targeted, zero == ZERO_CTRL_SMALL ? s.w.stats : nullptr, s.d_stats_pub, retry, st);
    if (s.timed) { CUDA_TRY(cudaEventRecord(s.ev[2], st)); CUDA_TRY(cudaEventRecord(s.ev[3], st)); }
  } else {
    if (!retry) launch_match(sh.dev, s.w, s.in, zero == ZERO_MATCH ? s.w.stats : nullptr, hs.targeted, st);
    if (s.timed) CUDA_TRY(cudaEventRecord(s.ev[2], st));
    if (!retry) launch_plan(sh.dev, s.w, s.in, st);
    launch_offsets(sh.dev, s.w, s.in, hs.n_direct > 0, sh.n_sms, st);   // pool mode: a pure function of the scratch
    if (s.timed) CUDA_TRY(cudaEventRecord(s.ev[3], st));
  }
  return 0;
}

// pack: from the control stage's results to ev_done, which covers the batch's final counters in h_stats (published by
// k_ctrl_small on the fused path, else by launch_pack)
int batch_pack(pcdn_engine* e, Shard& sh, ShardSlot& s, const Slot& hs, bool fused) {
  // Only two kinds of batch pack on the high-priority pack stream, beside the next batch's control kernels (which slow
  // a long bulk-store pack): many direct messages alone, whose latency-bound lookup overlaps their bandwidth-bound pack
  // well (config C4), and broadcasts batch_begin predicts to be short and message-major (sh.fat_only).
  const bool fat_overlap = s.in.n_bcast > 0 && sh.fat_only;
  const bool direct_only = s.in.n_bcast == 0 && hs.n_direct >= kThinSeparateMin;
  cudaStream_t st = sh.stream, ps = (!sh.direct_publish && (direct_only || fat_overlap)) ? sh.pack_stream : st, cs = sh.copy_stream;
  if (!s.spans_mapped) {   // (mapped spans: k_offsets wrote them to host memory; the host waits for ev_done only)
    CUDA_TRY(cudaEventRecord(s.ev_ctrl, st));
    // the span table is final once k_offsets is done: its counters go home while the pack runs
    CUDA_TRY(cudaStreamWaitEvent(cs, s.ev_ctrl, 0));
    CUDA_TRY(cudaMemcpyAsync(s.h_early, s.w.stats, sizeof(BatchStats), cudaMemcpyDeviceToHost, cs));
    CUDA_TRY(cudaEventRecord(s.ev_early, cs));
    // pack on its own stream (packs of successive batches stay ordered among themselves)
    if (ps != st) CUDA_TRY(cudaStreamWaitEvent(ps, s.ev_ctrl, 0));
  }
  if (s.timed) CUDA_TRY(cudaEventRecord(s.ev[4], ps));
  // k_pack CTAs per SM unless pack_variant sets them: 4 when the pack has the GPU to itself, 3 when it overlaps the
  // next batch's control kernels (one H100: C2 +1.4 % with 4; the overlapped config-5 sparse shard +2 % with 3)
  const uint32_t pack_ctas = e->pack_ctas ? e->pack_ctas : fat_overlap ? 3u : 4u;
  // engines with ref_min_bytes: a host-staged batch runs k_pack_ref only when a message reaches the threshold; the
  // lengths of a device-resident batch are on the device, so it always does
  const bool has_ref = e->cfg.ref_min_bytes && (hs.device_input || hs.max_raw_len >= e->cfg.ref_min_bytes);
  launch_pack(sh.dev, s.w, s.in, hs.n_direct, pack_ctas, e->direct_ctas, sh.n_sms, has_ref, fused ? nullptr : s.d_stats_pub, ps);
  if (s.timed) CUDA_TRY(cudaEventRecord(s.ev[5], ps));
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaEventRecord(s.ev_done, ps));
  return 0;
}

// the kernel pipeline of one shard for slot `si` (wait_ingest: its BatchIn is ready once ev_ingest fires; retry: see batch_control)
int launch_shard_pipeline(pcdn_engine* e, Shard& sh, uint32_t si, bool wait_ingest, bool retry = false) {
  DeviceGuard dg(sh.device);
  ShardSlot& s = sh.slots[si];
  // latency path of the smallest geometry: match + plan + offsets in one cluster launch (kernels.cu: k_ctrl_small)
  // (one cluster of 8 CTAs: worth it while the whole match is a few passes — a 128-message batch on a
  //  65536-slot engine is 1024 (message, block) items and runs 10x faster through the regular kernels)
  const bool fused = sh.direct_publish && sh.dev.N <= kSmallCtrlConns && s.in.n_msgs <= kSmallCtrlMsgs &&
                     (uint64_t)s.in.n_bcast * sh.dev.nblk <= kSmallCtrlItems;
  if (int rc = batch_begin(e, sh, si, fused, wait_ingest, retry)) return rc;
  if (int rc = batch_control(sh, s, e->slots[si], fused, retry)) return rc;
  return batch_pack(e, sh, s, e->slots[si], fused);
}

// every local shard runs the pipeline on the open slot `si`; it becomes the newest in-flight batch
int launch_pipeline(pcdn_engine* e, uint32_t si, bool wait_ingest) {
  Slot& s = e->slots[si];
  for (Shard& sh : e->shards) {
    int rc = launch_shard_pipeline(e, sh, si, wait_ingest);
    if (rc) return rc;
  }
  s.state = SLOT_INFLIGHT;
  s.t_launch = std::chrono::steady_clock::now();
  s.batch_id = e->next_batch_id++;
  s.counted = false;
  e->inflight.push_back(s.batch_id);
  e->open_slot = -1;
  e->stats.batches++;
  e->stats.msgs += s.n_msgs;
  return 0;
}

// Sharded engines: bring a batch into every shard's d_arena, on the ingest streams — ahead of the main
// streams, so that it overlaps the pack of the previous batch.  The region may only be overwritten once
// the pack that last read this slot's arena is done (ev_done).  `regs`: the batch's pieces, regs[0] = the
// frames at offset 0, the descriptor block behind them (ascending dst_off).
//  - host-staged batch: one region, the slot's pinned staging (frames + descriptor block);
//  - device-resident batch (its arrays lie on the root GPU, global shard 0): the frames and the eight
//    descriptor arrays.  The root first GATHERS the descriptor arrays — and the frames too unless they are
//    large (`arena_in_place`) — into its own slot region with a few device-to-device copies, so that ONE
//    ncclBroadcast of one contiguous range (two with in-place frames) replicates the batch; nine separate
//    broadcasts per step cost C5-sparse 8 % at 8 GPUs.
// PCDN_INGEST_HOST (single process): every shard copies the regions itself (peer copies from the root's
// buffers).  PCDN_INGEST_NCCL: the root copies them, then ncclBroadcast over all shards of the broker
// (grouped over the local shards).  `wait_submit`: order the ingest after everything queued on the root's
// main stream (the caller's producer kernels); false when the caller says the buffers are already
// complete, so the broadcast of batch n+1 overlaps the pack of batch n.
struct IngestRegion { const void* src; size_t dst_off; size_t bytes; bool host = false; };  // src: pinned host memory, or device memory of the root
int ingest_batch(pcdn_engine* e, uint32_t si, const IngestRegion* regs, int nregs, bool arena_in_place, bool wait_submit) {
  const size_t all_hi = regs[nregs - 1].dst_off + regs[nregs - 1].bytes;
  if (e->ingest == PCDN_INGEST_HOST) {
    for (Shard& sh : e->shards) {
      DeviceGuard dg(sh.device);
      ShardSlot& ss = sh.slots[si];
      CUDA_TRY(cudaStreamWaitEvent(sh.ingest_stream, ss.ev_done, 0));
      if (wait_submit) CUDA_TRY(cudaStreamWaitEvent(sh.ingest_stream, e->shards[0].ev_submit, 0));
      for (int r = 0; r < nregs; r++) {
        const IngestRegion& g = regs[r];
        if (!g.bytes || (sh.gindex == 0 && r == 0 && arena_in_place)) continue;
        if (g.host || sh.gindex == 0)
          CUDA_TRY(cudaMemcpyAsync(ss.d_arena + g.dst_off, g.src, g.bytes, g.host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, sh.ingest_stream));
        else
          CUDA_TRY(cudaMemcpyPeerAsync(ss.d_arena + g.dst_off, sh.device, g.src, e->shards[0].device, g.bytes, sh.ingest_stream));
      }
      CUDA_TRY(cudaEventRecord(ss.ev_ingest, sh.ingest_stream));
    }
    return 0;
  }
  const NcclApi* nc = e->nccl;
  for (Shard& sh : e->shards) {
    DeviceGuard dg(sh.device);
    ShardSlot& ss = sh.slots[si];
    CUDA_TRY(cudaStreamWaitEvent(sh.ingest_stream, ss.ev_done, 0));
    if (sh.gindex != 0) continue;
    if (wait_submit) CUDA_TRY(cudaStreamWaitEvent(sh.ingest_stream, sh.ev_submit, 0));
    for (int r = arena_in_place ? 1 : 0; r < nregs; r++) {
      const IngestRegion& g = regs[r];
      if (g.bytes)
        CUDA_TRY(cudaMemcpyAsync(ss.d_arena + g.dst_off, g.src, g.bytes, g.host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, sh.ingest_stream));
    }
  }
  NCCL_TRY(nc, nc->GroupStart());
  for (Shard& sh : e->shards) {
    DeviceGuard dg(sh.device);
    ShardSlot& ss = sh.slots[si];
    int rc = 0;
    if (arena_in_place) {   // (device input only: regs[1] starts the descriptor arrays)
      const size_t desc_lo = regs[1].dst_off;
      if (regs[0].bytes) {
        void* buf = sh.gindex == 0 ? const_cast<void*>(regs[0].src) : (void*)ss.d_arena;   // the root sends from the caller's buffer
        rc = nc->Broadcast(buf, buf, regs[0].bytes, kNcclUint8, 0, sh.comm, sh.ingest_stream);
      }
      if (!rc) rc = nc->Broadcast(ss.d_arena + desc_lo, ss.d_arena + desc_lo, all_hi - desc_lo, kNcclUint8, 0, sh.comm, sh.ingest_stream);
    } else {
      rc = nc->Broadcast(ss.d_arena, ss.d_arena, all_hi, kNcclUint8, 0, sh.comm, sh.ingest_stream);
    }
    if (rc) { nc->GroupEnd(); return fail(PCDN_ECUDA, std::string("ncclBroadcast: ") + nc->GetErrorString(rc)); }
  }
  NCCL_TRY(nc, nc->GroupEnd());
  for (Shard& sh : e->shards) {
    DeviceGuard dg(sh.device);
    CUDA_TRY(cudaEventRecord(sh.slots[si].ev_ingest, sh.ingest_stream));
  }
  return 0;
}

// close the open batch: upload staging, launch
int flush_open(pcdn_engine* e, uint64_t* batch_id) {
  if (batch_id) *batch_id = 0;
  if (e->open_slot < 0) return 0;
  const uint32_t si = (uint32_t)e->open_slot;
  Slot& s = e->slots[si];
  const uint32_t n = (uint32_t)s.kind.size();
  if (n == 0) { abandon_open(e); return 0; }   // (events alone: no message sees them, they go up with the journal)
  if (!e->has_device) return fail(PCDN_ENODEV, "host-only engine cannot route messages");
  int rc = flush_journal(e);
  if (rc) return rc;
  const DescLayout L(n, (uint32_t)s.bcast_index.size(), s.topics.size(), (uint32_t)s.events.size(), s.ev_topics.size());
  // The descriptor block goes behind the frames in the slot's staging, so that the whole batch is one
  // host→device copy (one ingest region on a sharded engine); it fits arena_cap (init_device).
  const size_t doff = align_up(s.arena_used, 256);
  uint8_t* hd = s.h_arena + doff;
  std::memset(s.h_arena + s.arena_used, 0, doff - s.arena_used);
  std::memcpy(hd + L.o_kind, s.kind.data(), n);
  std::memcpy(hd + L.o_flags, s.flags.data(), n);
  std::memcpy(hd + L.o_slot, s.slot_off16.data(), (size_t)n * 4);
  std::memcpy(hd + L.o_len, s.raw_len.data(), (size_t)n * 4);
  std::memcpy(hd + L.o_aoff, s.aux_off.data(), (size_t)n * 4);
  std::memcpy(hd + L.o_alen, s.aux_len.data(), (size_t)n * 4);
  if (!s.bcast_index.empty()) std::memcpy(hd + L.o_bidx, s.bcast_index.data(), s.bcast_index.size() * 4);
  if (!s.topics.empty()) std::memcpy(hd + L.o_top, s.topics.data(), s.topics.size() * 2);
  if (!s.events.empty()) {   // by (connection, position): the match finds a connection's events by binary search
    std::stable_sort(s.events.begin(), s.events.end(), [](const SubEvent& a, const SubEvent& b) { return a.conn < b.conn; });
    std::memcpy(hd + L.o_ev, s.events.data(), s.events.size() * sizeof(SubEvent));
    std::memcpy(hd + L.o_etop, s.ev_topics.data(), s.ev_topics.size() * 2);
  }
  if (e->sharded) {
    const IngestRegion staged{s.h_arena, 0, doff + L.total, true};
    if ((rc = ingest_batch(e, si, &staged, 1, false, false))) return rc;
  } else {   // on the main stream: a wait for the ingest stream would lengthen the latency path
    Shard& sh = e->shards[0];
    DeviceGuard dg(sh.device);
    CUDA_TRY(cudaMemcpyAsync(sh.slots[si].d_arena, s.h_arena, doff + L.total, cudaMemcpyHostToDevice, sh.stream));
  }
  for (Shard& sh : e->shards) {
    ShardSlot& ss = sh.slots[si];
    ss.in = bind_batch(ss.d_arena, ss.d_arena + doff, L);
  }
  s.n_msgs = n;
  rc = launch_pipeline(e, si, e->sharded);
  e->tables->release_held();   // the events' words reach the device after this batch's control kernels
  if (rc) return rc;
  if (batch_id) *batch_id = s.batch_id;
  return 0;
}

// R12: a table mutation must not be visible to messages already handed to the engine
int before_state_change(pcdn_engine* e) {
  int rc = 0;
  if (e->open_slot >= 0 && (!e->slots[e->open_slot].kind.empty() || !e->slots[e->open_slot].events.empty())) rc = flush_open(e, nullptr);
  // connection-id quarantine (host_state.h): ids freed now may be named by spans of batches <= fence_now
  e->conns->fence_now = e->next_batch_id - 1;
  e->conns->oldest_unreleased = e->inflight.empty() ? ~0ull : e->inflight.front();
  return rc;
}

// What a batch holds.  `ingress`: bytes admitted to it that e->inflight_bytes does not count yet.
struct BatchFill {
  uint32_t msgs = 0, bcast = 0;
  uint64_t bytes = 0, topics = 0, ingress = 0;
  uint64_t ev_topics = 0;   // topic entries of the batch's subscription events (they share the topic capacity)
  uint32_t max_raw_len = 0;
  bool targeted = false;    // some message carries MSGF_TARGET
  void add(const MsgShape& m) {
    msgs++; bcast += m.kind == PCDN_KIND_BROADCAST ? 1 : 0;
    bytes += m.bytes(); topics += m.n_topics; ingress += m.ingress();
    max_raw_len = std::max(max_raw_len, m.raw_len);
    targeted |= m.target;
  }
};
BatchFill fill_of(const Slot& s) {
  return BatchFill{(uint32_t)s.kind.size(), (uint32_t)s.bcast_index.size(), s.arena_used, s.topics.size(), 0, s.ev_topics.size(),
                   s.max_raw_len, s.targeted};
}

// The per-batch limits: nullptr when `m` still fits a batch that holds `f`, else the limit it would
// break.  A message that does not fit an empty batch (BatchFill{}) never fits.
const char* batch_limit(const pcdn_engine* e, const BatchFill& f, const MsgShape& m) {
  const pcdn_config& c = e->cfg;
  if (f.msgs >= c.max_batch_msgs) return "max_batch_msgs";
  if (f.bytes + m.bytes() + 64 > c.max_batch_bytes) return "max_batch_bytes";
  if (m.kind == PCDN_KIND_BROADCAST && f.bcast >= c.max_batch_bcast) return "max_batch_bcast";
  if (f.topics + f.ev_topics + m.n_topics > e->topics_cap) return "the topic entries of the descriptor block";
  return nullptr;
}

// ---- subscription changes -----------------------------------------------------------------------
enum SubOp { SUB_USER, UNSUB_USER, SUB_BROKER, UNSUB_BROKER };

// `op` on the mirror for the user key / broker identifier `who`; *conn: its connection (or NONE)
int apply_sub(pcdn_engine* e, SubOp op, const std::string& who, const uint16_t* topics, uint32_t n, uint32_t* conn) {
  Connections& cn = *e->conns;
  switch (op) {
    case SUB_USER: *conn = cn.user_conn(who); return cn.subscribe_user_to(who, topics, n);
    case UNSUB_USER: *conn = cn.user_conn(who); return cn.unsubscribe_user_from(who, topics, n);
    case SUB_BROKER: *conn = cn.broker_conn(who.c_str()); return cn.subscribe_broker_to(who.c_str(), topics, n);
    default: *conn = cn.broker_conn(who.c_str()); return cn.unsubscribe_broker_from(who.c_str(), topics, n);
  }
}

// PCDN_FLAG_INBATCH_SUBSCRIBE: `op` as an event of the open batch, which holds `f`, at position f.msgs —
// or 1 when the batch cannot take one more event of n topics.  The mirror changes now, the device bitmap
// keeps the words' values before the batch's events until its control kernels have run (HostTables::hold),
// and the batch's match replays the event on the messages at or after f.msgs (kernels.cu: apply_events)
int record_event(pcdn_engine* e, const BatchFill& f, SubOp op, const std::string& who, const uint16_t* topics, uint32_t n) {
  HostTables& t = *e->tables;
  Slot& s = e->slots[e->open_slot];
  if (!(e->cfg.flags & PCDN_FLAG_INBATCH_SUBSCRIBE) || s.events.size() >= e->cfg.max_batch_msgs ||
      f.topics + f.ev_topics + n > e->topics_cap)
    return 1;
  const uint32_t pos = f.msgs;
  uint32_t conn;
  t.hold = true;
  const int rc = apply_sub(e, op, who, topics, n, &conn);
  t.hold = false;
  if (rc || conn == PCDN_CONN_NONE) return rc;   // (a connection not attached here changes no bit)
  SubEvent ev{conn, pos | (op == SUB_USER || op == SUB_BROKER ? kEvSubscribe : 0u), (uint32_t)s.ev_topics.size(), 0};
  for (uint32_t i = 0; i < n; i++)
    if (topics[i] < e->geo.T) { s.ev_topics.push_back(topics[i]); ev.tn++; }   // (no other id has a bitmap row)
  s.events.push_back(ev);
  return 0;
}

// A subscription change from the C ABI or a user's Subscribe / Unsubscribe frame: an event of the open
// batch when the flag is set and it fits there, else (R12) the open batch is launched first
int sub_change(pcdn_engine* e, SubOp op, const std::string& who, const uint16_t* topics, uint32_t n) {
  int rc = 1;
  if ((e->cfg.flags & PCDN_FLAG_INBATCH_SUBSCRIBE) && (e->open_slot >= 0 || acquire_open_slot(e) == 0))
    rc = record_event(e, fill_of(e->slots[e->open_slot]), op, who, topics, n);
  if (rc == 1) {
    if ((rc = before_state_change(e))) return rc;
    uint32_t conn;
    rc = apply_sub(e, op, who, topics, n, &conn);
  }
  return rc ? fail(rc, "topic id out of range") : 0;
}

// a frame this engine never accepts (PCDN_EINVAL): the reason, else nullptr
const char* msg_invalid(const pcdn_engine* e, const MsgShape& m) {
  if (m.raw_len > 0x1FFFFFFFu) return "message larger than MAX_MESSAGE_SIZE (cdn-proto/src/lib.rs:25)";
  if (e->cfg.global_memory_pool_size && m.ingress() > e->cfg.global_memory_pool_size) return "message larger than the global memory pool";
  return nullptr;
}

// limiter/mod.rs:56-68: the frames' length in permits must be available before they are accepted
bool pool_admits(const pcdn_engine* e, uint64_t bytes) {
  return !e->cfg.global_memory_pool_size || e->inflight_bytes + bytes <= e->cfg.global_memory_pool_size;
}

// A recipient longer than any key in the table cannot match (bytewise identity, R8): the message is
// dropped, but batch order bookkeeping still wants it.  It is staged as its first max_key_len + 1
// bytes, a length no table entry has, so the lookup finds no candidate and counts the drop.  (Length 0
// would not do: that is the key of a user whose key is empty.)
uint32_t routed_key_len(const pcdn_engine* e, uint32_t len) { return len > e->cfg.max_key_len ? e->cfg.max_key_len + 1 : len; }

// Entry `p` as the `batch` entry of message `m`.  A direct message's recipient is read in place when it lies
// inside the frame at a 4-byte aligned offset (the frame starts 4 bytes into a 16-byte slot), else (and
// whenever the caller set m.stage_key) it is staged beside the frame.
void as_batch(Entry& p, InMsg& m) {
  if (m.kind == PCDN_KIND_DIRECT)
    m.stage_key |= !(m.key && m.key >= m.raw && m.key + m.key_len <= m.raw + m.raw_len && ((m.key - m.raw) & 3) == 0);
  p.route = ROUTE_BATCH; p.devparse = (m.flags & MSGF_DEVPARSE) != 0; p.rc = 0; p.why = nullptr;
  p.shape = MsgShape{m.kind, m.raw_len, m.stage_key ? (uint32_t)align_up(m.key_len, 16) : 0u, m.n_topics, (m.flags & MSGF_TARGET) != 0};
}

// Scratch entry i as a message of the C ABI's handle / submit calls.  A multi-process group stages every
// recipient of these calls: the layout must not depend on how a process happens to hold the bytes (a
// parsed frame's recipient lies at the same offset in every process).
void api_entry(pcdn_engine* e, uint32_t i, uint8_t kind, uint8_t flags, const uint16_t* topics, uint32_t n_topics,
               const uint8_t* recipient, uint32_t recipient_len, const uint8_t* raw, uint32_t raw_len) {
  InMsg& m = e->rx_msgs[i];
  m = InMsg{};
  m.kind = kind; m.flags = flags; m.raw = raw; m.raw_len = raw_len;
  if (kind == PCDN_KIND_DIRECT) {
    m.key = recipient; m.key_len = routed_key_len(e, recipient_len);
    m.stage_key = e->world_shards != e->shards.size();
  } else {
    m.topic_ids = topics; m.n_listed = m.n_topics = n_topics;
  }
  as_batch(e->rx_plan[i], m);
}

// MessageHookDef::on_message_received on the parsed message (def.rs:79-92).  Returns 0 = process,
// 1 = skip, negative = error with its text in *why (the receive loop ends; the text may lie in hs.err).
// The hook may shrink / rewrite the topic list (a private copy in hs.topics) and re-point the recipient.
int run_hook(const pcdn_engine* e, uint32_t origin, const ParsedFrame& pf, const pcdn_frame& f, pcdn_engine::HookScratch& hs,
             const uint8_t** f0, uint32_t* f0_len, const char** why) {
  std::vector<uint8_t>& topic_copy = hs.topics;
  pcdn_hook_message m{};
  m.kind = (uint8_t)pf.kind; m.origin = (uint8_t)origin;
  m.raw = f.raw; m.raw_len = f.raw_len; m.sender = f.sender; m.sender_len = f.sender_len;
  const bool has_topics = pf.kind == PCDN_KIND_BROADCAST || pf.kind == PCDN_KIND_SUBSCRIBE || pf.kind == PCDN_KIND_UNSUBSCRIBE;
  if (has_topics) {
    if (pf.f0_len > 65535) { *why = "topic list too long"; return PCDN_EPARSE; }
    topic_copy.assign(*f0, *f0 + pf.f0_len);
    m.topics = topic_copy.data(); m.n_topics = (uint16_t)pf.f0_len;
  } else if (pf.kind == PCDN_KIND_DIRECT) {
    m.recipient = *f0; m.recipient_len = pf.f0_len;
  }
  const int r = e->hook[origin](e->hook_user[origin], &m);
  if (r < 0) { hs.err = "hook failed: " + std::to_string(r); *why = hs.err.c_str(); return PCDN_EHOOK; }
  if (r == PCDN_HOOK_SKIP) return 1;
  if (has_topics) {
    if (m.n_topics > topic_copy.size() || m.topics != topic_copy.data()) { *why = "hook returned an invalid topic list"; return PCDN_EHOOK; }
    *f0 = topic_copy.data(); *f0_len = m.n_topics;
  } else if (pf.kind == PCDN_KIND_DIRECT) {
    if (m.recipient_len && !m.recipient) { *why = "hook returned a null recipient"; return PCDN_EHOOK; }
    *f0 = m.recipient; *f0_len = m.recipient_len;
  }
  return 0;
}

// One iteration of user_receive_loop (origin 0, `sender` = the user's key) or broker_receive_loop
// (origin 1, `sender` = the peer's identifier) up to the dispatch: frame `f` as entry `p` with message `m`.
// It changes nothing in the engine, so phase A runs it on several threads.  A hook of f's origin runs in
// it, with `hook` as its scratch, so hooked frames are classified by the scan, one at a time (phase A runs
// only while no hook is set, and passes no scratch).
void classify_frame(const pcdn_engine* e, const pcdn_frame& f, Entry& p, InMsg& m, pcdn_engine::HookScratch* hook) {
  const uint32_t origin = f.origin ? 1 : 0;
  m = InMsg{};
  m.raw = f.raw; m.raw_len = f.raw_len; m.flags = origin ? MSGF_USERS_ONLY : 0;   // broker-origin messages go to users only
  p.route = ROUTE_DONE; p.rc = 0; p.why = nullptr;
  // device-parse engines without a hook for `origin`: a Direct or Broadcast frame is only tag-peeked and
  // copied; k_parse does the rest
  if ((e->cfg.flags & PCDN_FLAG_DEVICE_PARSE) && !e->hook[origin]) {
    const int k = peek_kind_core(f.raw, f.raw_len);
    if (k == PCDN_KIND_DIRECT || k == PCDN_KIND_BROADCAST) {
      m.kind = (uint8_t)k;
      m.flags |= MSGF_DEVPARSE | (k == PCDN_KIND_BROADCAST && !origin ? MSGF_PRUNE : 0);  // prune: user origin only (handler.rs:157 vs user/handler.rs:133)
      return as_batch(p, m);
    }
  }
  ParsedFrame pf;
  if (!parse_frame(f.raw, f.raw_len, &pf)) { p.rc = PCDN_EPARSE; p.why = "failed to deserialize message"; return; }
  const uint8_t* f0 = f.raw + pf.f0_off;   // field 0: the recipient or the wire topic list (a hook may replace it)
  uint32_t f0_len = pf.f0_len;
  if (e->hook[origin]) {
    const int hr = run_hook(e, origin, pf, f, *hook, &f0, &f0_len, &p.why);
    if (hr) { p.rc = hr < 0 ? hr : 0; return; }   // Ok(HookResult::SkipMessage) => continue
  }
  m.kind = (uint8_t)pf.kind;
  if (pf.kind == PCDN_KIND_DIRECT) { m.key = f0; m.key_len = routed_key_len(e, f0_len); return as_batch(p, m); }
  if (pf.kind != PCDN_KIND_BROADCAST) {
    if (origin) { p.rc = 1; return; }
    if (pf.kind != PCDN_KIND_SUBSCRIBE && pf.kind != PCDN_KIND_UNSUBSCRIBE) { p.rc = PCDN_EKIND; p.why = "invalid message received"; return; }
  }
  // A Broadcast or a user's Subscribe / Unsubscribe.  User-origin topic lists are pruned (Topic::prune,
  // user/handler.rs:133), broker-origin ones kept verbatim (handler.rs:157).  The wire list may be of any
  // length: what counts against a batch is the entries it adds (n_topics), which batch_limit judges.
  m.wire_topics = f0; m.n_listed = f0_len; m.prune = !origin;
  for (uint32_t t = 0; t < f0_len; t++) m.n_topics += !m.prune || topic_kept(f0, t, e->cfg.n_valid_topics) ? 1u : 0u;
  if (m.n_topics == 0 && m.prune) { p.rc = PCDN_EPRUNE; p.why = "supplied no valid topics"; return; }
  if (pf.kind == PCDN_KIND_BROADCAST) return as_batch(p, m);
  p.route = (e->cfg.flags & PCDN_FLAG_INBATCH_SUBSCRIBE) ? ROUTE_EVENT : ROUTE_STATE;
  p.shape = MsgShape{m.kind, 0, 0, m.n_topics};
}

void slot_resize(Slot& s, const BatchFill& f) {
  s.kind.resize(f.msgs); s.flags.resize(f.msgs); s.slot_off16.resize(f.msgs); s.raw_len.resize(f.msgs);
  s.aux_off.resize(f.msgs); s.aux_len.resize(f.msgs); s.bcast_index.resize(f.bcast); s.topics.resize(f.topics);
}

// Write message `m`, placed by `p`, into slot `s`: its frame at p.arena_off, a staged recipient behind
// the frame, and its descriptor entries (the arrays are sized already).  It touches only what this message
// owns, so threads may write distinct messages at once.
void write_msg(Slot& s, const Entry& p, const InMsg& m, uint32_t n_valid) {
  const size_t off = p.arena_off, slot = align_up(4 + (size_t)m.raw_len, 16);
  const uint32_t mi = p.msg_idx;
  uint8_t* dst = s.h_arena + off;
  std::memset(dst, 0, 4);
  if (m.raw_len) std::memcpy(dst + 4, m.raw, m.raw_len);
  std::memset(dst + 4 + m.raw_len, 0, slot - 4 - m.raw_len);
  s.kind[mi] = m.kind; s.flags[mi] = m.flags; s.slot_off16[mi] = (uint32_t)(off / 16); s.raw_len[mi] = m.raw_len;
  if (m.kind == PCDN_KIND_DIRECT) {
    if (m.stage_key) {
      if (m.key_len) std::memcpy(dst + slot, m.key, m.key_len);
      std::memset(dst + slot + m.key_len, 0, p.shape.key_bytes - m.key_len);
    }
    s.aux_off[mi] = (uint32_t)(m.stage_key ? off + slot : off + 4 + (size_t)(m.key - m.raw));
    s.aux_len[mi] = m.key_len;
    return;
  }
  s.aux_off[mi] = (m.flags & MSGF_TARGET) ? m.target : p.topic_off;
  s.aux_len[mi] = m.n_topics;
  s.bcast_index[p.bcast_pos] = mi;
  for (uint32_t t = 0, k = p.topic_off; t < m.n_listed; t++) {
    if (m.topic_ids) s.topics[k++] = m.topic_ids[t];
    else if (!m.prune || topic_kept(m.wire_topics, t, n_valid)) s.topics[k++] = m.wire_topics[t];
  }
}

// the open slot `s` now holds `f`: messages up to f.msgs are written
void slot_commit(pcdn_engine* e, Slot& s, const BatchFill& f, bool devparse) {
  s.arena_used = f.bytes; s.n_direct = f.msgs - f.bcast; s.devparse |= devparse; s.max_raw_len = f.max_raw_len;
  s.targeted = f.targeted;
  s.ingress_bytes += f.ingress; e->inflight_bytes += f.ingress; e->stats.bytes_in += f.ingress;
}

template <class F>
void parallel_for(uint32_t n, uint32_t nthreads, F f) {
  if (n < 2048 || nthreads <= 1) { f(0u, n); return; }
  std::vector<std::thread> th;
  const uint32_t per = (n + nthreads - 1) / nthreads;
  for (uint32_t t = 1; t < nthreads; t++) {
    const uint32_t lo = t * per, hi = std::min(n, lo + per);
    if (lo < hi) th.emplace_back([=] { f(lo, hi); });
  }
  f(0u, std::min(n, per));
  for (auto& x : th) x.join();
}

uint32_t ingest_threads() {
  static uint32_t n = [] {
    if (const char* e = std::getenv("PCDN_INGEST_THREADS")) return (uint32_t)std::max(1, atoi(e));
    return std::min(16u, std::max(1u, std::thread::hardware_concurrency()));
  }();
  return n;
}

// The placement scan: the scratch entries [0, n) in order, on the calling thread (each classified here
// first when `classify` is set; `frames`: the frames behind them, null for API messages).  An entry is
// placed in the open batch (launching a full one first), recorded as an event of it, applied through
// sub_change, or only reported.  Its result goes to Entry::rc and rc_out[i], a failure's text to
// pcdn_last_error.  The placed messages of a run are written by index (phase B, on several threads for
// long runs) before the batch is launched or anything else changes it.  Returns the number of entries
// consumed (a capacity condition, a CUDA error or a host-only engine stops early) or the code when not
// even the first one was.
int place_entries(pcdn_engine* e, const pcdn_frame* frames, uint32_t n, int32_t* rc_out, bool classify) {
  Entry* const plan = e->rx_plan.get();
  InMsg* const msgs = e->rx_msgs.get();
  const uint32_t n_valid = e->cfg.n_valid_topics;
  BatchFill fill;   // while `open`: the open batch, holding the messages placed by entries [run, i)
  bool open = false, devparse = false;
  uint32_t run = 0;
  auto end_run = [&](uint32_t end) {
    if (!open) return;
    Slot& s = e->slots[e->open_slot];
    slot_resize(s, fill);
    parallel_for(end - run, ingest_threads(), [&](uint32_t lo, uint32_t hi) {
      for (uint32_t q = run + lo; q < run + hi; q++)
        if (plan[q].route == ROUTE_BATCH) write_msg(s, plan[q], msgs[q], n_valid);
    });
    slot_commit(e, s, fill, devparse);
    open = devparse = false;
  };
  for (uint32_t i = 0; i < n; i++) {
    Entry& p = plan[i];
    if (classify) classify_frame(e, frames[i], p, msgs[i], &e->rx_hook);
    int rc = p.rc;
    if (p.route == ROUTE_BATCH) {
      const char* why;
      if (!e->has_device) rc = fail(PCDN_ENODEV, "host-only engine cannot route messages");
      else if ((why = msg_invalid(e, p.shape))) rc = fail(PCDN_EINVAL, why);
      else if ((why = batch_limit(e, BatchFill{}, p.shape))) rc = fail(PCDN_ENOSPC, std::string("message does not fit an empty batch: ") + why);
      else for (bool launched = false;; launched = true) {   // the open batch, else a new one behind it
        if (!open) {
          if ((rc = acquire_open_slot(e))) break;
          fill = fill_of(e->slots[e->open_slot]);
          open = true; run = i;
        }
        if (!batch_limit(e, fill, p.shape) && pool_admits(e, fill.ingress + p.shape.ingress())) {
          p.msg_idx = fill.msgs; p.arena_off = fill.bytes; p.bcast_pos = fill.bcast; p.topic_off = (uint32_t)fill.topics;
          fill.add(p.shape);
          devparse |= p.devparse;
          break;
        }
        // Only an exhausted memory pool refuses an empty batch.  Its permits come back when batches are
        // released, so the open batch is launched first: then draining a batch and calling again makes progress.
        if (launched) { rc = fail(PCDN_EAGAIN, "global memory pool exhausted: release a batch first"); break; }
        end_run(i);
        if ((rc = flush_open(e, nullptr))) break;
      }
      if (rc) p.route = ROUTE_DONE;   // (phase B skips it)
    } else if (p.route != ROUTE_DONE) {   // a user's Subscribe / Unsubscribe
      const InMsg& m = msgs[i];
      e->rx_topics.resize(m.n_listed);
      const uint32_t nt = prune_topics(m.wire_topics, m.n_listed, n_valid, e->rx_topics.data());
      const SubOp op = m.kind == PCDN_KIND_SUBSCRIBE ? SUB_USER : UNSUB_USER;
      const std::string who((const char*)frames[i].sender, frames[i].sender_len);
      rc = 1;
      if (p.route == ROUTE_EVENT && open) {   // an event at its place among the messages: the run goes on
        rc = record_event(e, fill, op, who, e->rx_topics.data(), nt);
        fill.ev_topics = e->slots[e->open_slot].ev_topics.size();
        if (rc < 0) fail(rc, "topic id out of range");
      }
      if (rc == 1) {
        end_run(i);
        rc = sub_change(e, op, who, e->rx_topics.data(), nt);
      }
    } else if (rc < 0) {
      fail(rc, p.why);
    }
    p.rc = rc;
    if (rc_out) rc_out[i] = rc;
    if (rc == PCDN_EAGAIN || rc == PCDN_ECUDA || rc == PCDN_ENODEV) {
      end_run(i);
      return i ? (int)i : rc;
    }
    if (classify) end_run(i + 1);   // (the next classification reuses the hook's scratch)
  }
  end_run(n);
  return (int)n;
}

// one message of pcdn_handle_*_message through the placement scan
int handle_msg(pcdn_engine* e, uint8_t kind, uint8_t flags, const uint16_t* topics, uint32_t n_topics,
               const uint8_t* recipient, uint32_t recipient_len, const uint8_t* raw, uint32_t raw_len) {
  e->rx_reserve(1);
  api_entry(e, 0, kind, flags, topics, n_topics, recipient, recipient_len, raw, raw_len);
  place_entries(e, nullptr, 1, nullptr, false);
  return e->rx_plan[0].rc;
}

// pcdn_receive_frames: phase A classifies every frame (on several threads for large calls), unless a hook
// is set: the scan then classifies each frame when it comes to it, so that the hook sees the frames in
// order and only those the call consumes
int receive_frames_locked(pcdn_engine* e, const pcdn_frame* frames, uint32_t n, int32_t* rc_out) {
  e->rx_reserve(n);
  const bool hooked = e->hook[0] || e->hook[1];
  if (!hooked)
    parallel_for(n, ingest_threads(), [&](uint32_t lo, uint32_t hi) {
      for (uint32_t i = lo; i < hi; i++) classify_frame(e, frames[i], e->rx_plan[i], e->rx_msgs[i], nullptr);
    });
  const int done = place_entries(e, frames, n, rc_out, hooked);
  e->rx_release();
  return done;
}

// one frame through pcdn_receive_frames: what it returns for that frame
int receive_one(pcdn_engine* e, uint32_t origin, const uint8_t* sender, uint32_t sender_len, const uint8_t* raw, uint32_t raw_len) {
  const pcdn_frame f{sender, sender_len, origin, raw, raw_len, 0};
  int32_t rc = 0;
  receive_frames_locked(e, &f, 1, &rc);
  return rc;
}

}  // namespace
int pcdn_detail::find_slot_index(pcdn_engine* e, uint64_t id) {
  for (size_t i = 0; i < e->slots.size(); i++)
    if (e->slots[i].state == SLOT_INFLIGHT && e->slots[i].batch_id == id) return (int)i;
  return -1;
}
namespace {

void destroy_shard(pcdn_engine* e, Shard& sh) {
  if (!sh.stream && sh.dev_allocs.empty() && sh.pin_allocs.empty()) return;  // never initialised (create failed earlier)
  if (cudaSetDevice(sh.device) != cudaSuccess) { cudaGetLastError(); return; }
  if (sh.stream) cudaStreamSynchronize(sh.stream);
  if (sh.pack_stream) cudaStreamSynchronize(sh.pack_stream);
  if (sh.copy_stream) cudaStreamSynchronize(sh.copy_stream);
  if (sh.ingest_stream) cudaStreamSynchronize(sh.ingest_stream);
  if (sh.comm && e->nccl) { e->nccl->CommDestroy(sh.comm); sh.comm = nullptr; }
  for (auto& s : sh.slots) {
    if (s.ev_done) cudaEventDestroy(s.ev_done);
    if (s.ev_ctrl) cudaEventDestroy(s.ev_ctrl);
    if (s.ev_early) cudaEventDestroy(s.ev_early);
    if (s.ev_ingest) cudaEventDestroy(s.ev_ingest);
    for (auto& ev : s.ev) if (ev) cudaEventDestroy(ev);
  }
  for (void* p : sh.dev_allocs) cudaFree(p);
  for (void* p : sh.pin_allocs) cudaFreeHost(p);
  if (sh.jstage_h) cudaFreeHost(sh.jstage_h);
  if (sh.jstage_d) cudaFree(sh.jstage_d);
  if (sh.ev_journal) cudaEventDestroy(sh.ev_journal);
  if (sh.ev_submit) cudaEventDestroy(sh.ev_submit);
  if (sh.copy_stream) cudaStreamDestroy(sh.copy_stream);
  if (sh.pack_stream) cudaStreamDestroy(sh.pack_stream);
  if (sh.ingest_stream) cudaStreamDestroy(sh.ingest_stream);
  if (sh.own_stream && sh.stream) cudaStreamDestroy(sh.stream);
}

void destroy_engine(pcdn_engine* e) {
  if (e->has_device) {
    int prev = -1;
    cudaGetDevice(&prev);
    for (Shard& sh : e->shards) destroy_shard(e, sh);
    for (Slot& s : e->slots)
      if (s.h_arena) cudaFreeHost(s.h_arena);
    if (prev >= 0) cudaSetDevice(prev);
    cudaGetLastError();  // a failed create must not leave its error behind for the next engine's launches
  }
  delete e;
}

#define DEV_ALLOC(ptr, n)                                 \
  do {                                                    \
    int _rc = dev_alloc(&(ptr), (n));                     \
    if (_rc) return _rc;                                  \
    sh.dev_allocs.push_back((void*)(ptr));                \
  } while (0)
#define PIN_ALLOC(ptr, n)                                 \
  do {                                                    \
    int _rc = pin_alloc(&(ptr), (n));                     \
    if (_rc) return _rc;                                  \
    sh.pin_allocs.push_back((void*)(ptr));                \
  } while (0)
#define PIN_ALLOC_MAPPED(ptr, alias, n)                   \
  do {                                                    \
    int _rc = pin_alloc_mapped(&(ptr), &(alias), (n));    \
    if (_rc) return _rc;                                  \
    sh.pin_allocs.push_back((void*)(ptr));                \
  } while (0)

// device side of one shard: streams, its table slices / replicas, rings, per-slot scratch + results
int init_shard(pcdn_engine* e, Shard& sh, int ndev, void* user_stream) {
  const pcdn_config& c = e->cfg;
  const Geometry& g = e->geo;
  if (sh.device < 0 || sh.device >= ndev) return fail(PCDN_ENODEV, "device ordinal " + std::to_string(sh.device) + " out of range (" + std::to_string(ndev) + " CUDA devices)");
  CUDA_TRY(cudaSetDevice(sh.device));
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, sh.device));
  sh.n_sms = prop.multiProcessorCount;
  if (user_stream) { sh.stream = (cudaStream_t)user_stream; sh.own_stream = false; }
  else { CUDA_TRY(cudaStreamCreateWithFlags(&sh.stream, cudaStreamNonBlocking)); sh.own_stream = true; }
  CUDA_TRY(cudaStreamCreateWithFlags(&sh.copy_stream, cudaStreamNonBlocking));
  CUDA_TRY(cudaEventCreateWithFlags(&sh.ev_journal, cudaEventDisableTiming));
  CUDA_TRY(cudaEventCreateWithFlags(&sh.ev_submit, cudaEventDisableTiming));
  {
    // highest priority: when a pack and the (small) control kernels of the next batch become
    // runnable together, the pack's persistent CTAs must be placed first and evenly over the SMs
    int lo = 0, hi = 0;
    CUDA_TRY(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    CUDA_TRY(cudaStreamCreateWithPriority(&sh.pack_stream, cudaStreamNonBlocking, hi));
    if (e->sharded) CUDA_TRY(cudaStreamCreateWithPriority(&sh.ingest_stream, cudaStreamNonBlocking, hi));
  }
  const uint32_t Ns = g.shard_N, Ws = Ns / 32;
  sh.direct_publish = Ns <= kDirectPublishMaxConns && !(c.flags & PCDN_FLAG_STAGED_SPANS);

  DevState& d = sh.dev;
  d.N = Ns; d.W = Ws; d.T = g.T; d.nblk = Ws / kBlockWords;
  d.bucket_mask = g.bucket_mask; d.key_stride = g.key_stride; d.seed = g.seed;
  d.ring_bytes = c.ring_bytes_per_conn; d.ring_units = (uint32_t)(c.ring_bytes_per_conn / kUnit);
  d.ref_min = (c.flags & PCDN_FLAG_SHARED_PAYLOAD) ? 0u : c.ref_min_bytes ? c.ref_min_bytes : 0xFFFFFFFFu;
  d.n_valid_topics = c.n_valid_topics;
  d.max_key_len = c.max_key_len;
  d.conn_base = sh.gindex * Ns;
  d.span_runs = (c.flags & PCDN_FLAG_SPAN_RUNS) ? 1u : 0u;
  d.pool = (c.flags & PCDN_FLAG_OUTPUT_POOL) ? 1u : 0u;
  d.pool_units = (uint32_t)(e->pool_bytes / kUnit);
  d.count_drops = sh.gindex == 0 ? 1u : 0u;
  DEV_ALLOC(d.sub, (size_t)g.T * Ws);
  DEV_ALLOC(d.brk, Ws);
  DEV_ALLOC(d.owner_conn, g.max_owners);
  DEV_ALLOC(d.cuckoo, (size_t)g.nbuckets * 4);
  DEV_ALLOC(d.keys, (size_t)g.max_keys * g.key_stride);
  DEV_ALLOC(d.ptail, Ns);
  DEV_ALLOC(d.used, Ns);
  const size_t out_bytes = d.pool ? (size_t)e->pool_bytes : (size_t)g.shard_max_conns * c.ring_bytes_per_conn;
  if (c.flags & PCDN_FLAG_HOST_RINGS) {
    // egress hand-off: the pack stores straight into host memory the socket writers read
    PIN_ALLOC_MAPPED(sh.h_rings, d.rings, out_bytes);
  } else {
    DEV_ALLOC(d.rings, out_bytes);
  }
  if (d.pool) {
    DEV_ALLOC(d.pool_state, 1);
    launch_pool_init(d, sh.stream);
  }
  CUDA_TRY(cudaMemsetAsync(d.sub, 0, (size_t)g.T * Ws * 4, sh.stream));
  CUDA_TRY(cudaMemsetAsync(d.brk, 0, (size_t)Ws * 4, sh.stream));
  CUDA_TRY(cudaMemsetAsync(d.owner_conn, 0xFF, (size_t)g.max_owners * 4, sh.stream));
  CUDA_TRY(cudaMemsetAsync(d.cuckoo, 0, (size_t)g.nbuckets * 4 * sizeof(CuckooEntry), sh.stream));
  CUDA_TRY(cudaMemsetAsync(d.keys, 0, (size_t)g.max_keys * g.key_stride, sh.stream));
  CUDA_TRY(cudaMemsetAsync(d.ptail, 0, (size_t)Ns * 4, sh.stream));
  CUDA_TRY(cudaMemsetAsync(d.used, 0, (size_t)Ns * 4, sh.stream));

  const uint32_t M = c.max_batch_msgs, MB = c.max_batch_bcast;
  const size_t cap_fat = (size_t)c.max_batch_deliveries;
  const size_t cap_thin = std::min<size_t>(c.max_batch_deliveries, (size_t)M * (kFatMin - 1));
  sh.slots.resize(c.batch_slots);
  for (ShardSlot& s : sh.slots) {
    DEV_ALLOC(s.d_arena, e->arena_cap);
    Work& w = s.w;
    DEV_ALLOC(w.B, (size_t)MB * Ws);
    DEV_ALLOC(w.wpre, (size_t)MB * Ws);
    DEV_ALLOC(w.cnt, (size_t)MB * d.nblk);
    DEV_ALLOC(w.base, (size_t)MB * d.nblk);
    DEV_ALLOC(w.done, MB);
    CUDA_TRY(cudaMemsetAsync(w.done, 0, (size_t)MB * 4, sh.stream));
    DEV_ALLOC(w.D, M);
    DEV_ALLOC(w.dconn, M);
    DEV_ALLOC(w.eb_fat, (size_t)M + 1);
    DEV_ALLOC(w.eb_thin, (size_t)M + 1);
    DEV_ALLOC(w.tbase, (size_t)M + 1);
    DEV_ALLOC(w.scan_tmp, 4 * ((size_t)M / 256 + 2));
    DEV_ALLOC(w.cls, M);
    DEV_ALLOC(w.cm_rank, (size_t)M + 1);
    DEV_ALLOC(w.cm_list, MB);
    DEV_ALLOC(w.jidx, M);
    DEV_ALLOC(w.efat, cap_fat);
    DEV_ALLOC(w.ecm, cap_fat);
    // A connection-major message has at least N/16 recipients (kCmDenseShift), and a batch past cap_fat
    // fat + cm deliveries is refused before k_offsets, so n_cm <= 16 * cap_fat / N and the run starts
    // need groups * N <= (n_cm / 8 + 1) * N <= 2 * cap_fat + N entries (and never more than MB / 8 groups).
    DEV_ALLOC(w.cmrun, std::min<size_t>(((size_t)MB + kCmGroup - 1) / kCmGroup * Ns, 2 * cap_fat + Ns));
    DEV_ALLOC(w.ethin, cap_thin);
    w.cap_fat = (uint32_t)std::min<size_t>(cap_fat, 0xFFFFFFFFu);
    w.cap_thin = (uint32_t)std::min<size_t>(cap_thin, 0xFFFFFFFFu);
    DEV_ALLOC(w.dcount, (size_t)Ns + 2);
    DEV_ALLOC(w.dloc, (size_t)Ns + 2);
    DEV_ALLOC(w.dtile, (size_t)Ns / 1024 + 3);
    DEV_ALLOC(w.dlist, M);
    DEV_ALLOC(w.hot_list, (size_t)M / kHotMin + 2);
    DEV_ALLOC(w.hot_bitmap, (size_t)kHotCtas * ((size_t)M / 32 + 1));
    DEV_ALLOC(w.scan_done, 1);
    CUDA_TRY(cudaMemsetAsync(w.scan_done, 0, 4, sh.stream));
    DEV_ALLOC(w.edir, M);
    DEV_ALLOC(w.dstart, (size_t)Ns + 1);
    DEV_ALLOC(w.dend, (size_t)Ns + 1);
    DEV_ALLOC(w.dstamp, (size_t)Ns + 1);
    CUDA_TRY(cudaMemsetAsync(w.dstamp, 0, ((size_t)Ns + 1) * 4, sh.stream));
    w.stamp = 0;
    DEV_ALLOC(w.batch_units, Ns);
    if (d.pool) {
      DEV_ALLOC(w.cbase, Ns);
      DEV_ALLOC(w.lb_state, (size_t)Ns / 256 + 1);
      DEV_ALLOC(w.lb_tot, (size_t)Ns / 256 + 1);
      CUDA_TRY(cudaMemsetAsync(w.lb_state, 0, ((size_t)Ns / 256 + 1) * 8, sh.stream));
    }
    w.pool_unblock = 0;
    const size_t span_entries = (size_t)2 * Ns * (d.span_runs ? 3 : 2) / 2;  // SpanRun = 24 B, Span = 16 B
    DEV_ALLOC(s.d_spans_dev, span_entries);
    DEV_ALLOC(s.d_ovf_dev, Ns);
    if (sh.direct_publish) {
      PIN_ALLOC_MAPPED(s.h_spans, s.d_spans_map, span_entries);
      PIN_ALLOC_MAPPED(s.h_overflow, s.d_ovf_map, (size_t)Ns);
    } else {
      PIN_ALLOC(s.h_spans, span_entries);
      PIN_ALLOC(s.h_overflow, g.shard_max_conns);
    }
    w.spans = s.d_spans_dev; w.overflow = s.d_ovf_dev;
    DEV_ALLOC(w.msg_status, M);
    PIN_ALLOC(s.h_msg_status, M);
    DEV_ALLOC(w.stats, 1);
    PIN_ALLOC_MAPPED(s.h_stats, s.d_stats_pub, 1);   // written by the kernel that ends the batch
    PIN_ALLOC(s.h_early, 1);
    CUDA_TRY(cudaEventCreateWithFlags(&s.ev_done, cudaEventDisableTiming));
    CUDA_TRY(cudaEventCreateWithFlags(&s.ev_ctrl, cudaEventDisableTiming));
    CUDA_TRY(cudaEventCreateWithFlags(&s.ev_early, cudaEventDisableTiming));
    CUDA_TRY(cudaEventCreateWithFlags(&s.ev_ingest, cudaEventDisableTiming));
    for (auto& ev : s.ev) CUDA_TRY(cudaEventCreate(&ev));
  }
  CUDA_TRY(cudaStreamSynchronize(sh.stream));
  return 0;
}

// the ingest communicator: one NCCL rank per shard of the broker, ranks of this process = its shards
int init_nccl(pcdn_engine* e) {
  const char* why = "";
  e->nccl = nccl_api(&why);
  if (!e->nccl) return fail(PCDN_ENODEV, std::string("PCDN_INGEST_NCCL needs libnccl.so.2: ") + why);
  NcclUniqueId id;
  if (e->cfg.nccl_unique_id) std::memcpy(&id, e->cfg.nccl_unique_id, sizeof(id));
  else NCCL_TRY(e->nccl, e->nccl->GetUniqueId(&id));
  NCCL_TRY(e->nccl, e->nccl->GroupStart());
  for (Shard& sh : e->shards) {
    cudaSetDevice(sh.device);
    int rc = e->nccl->CommInitRank(&sh.comm, (int)e->world_shards, id, (int)sh.gindex);
    if (rc) { e->nccl->GroupEnd(); return fail(PCDN_ECUDA, std::string("ncclCommInitRank: ") + e->nccl->GetErrorString(rc)); }
  }
  NCCL_TRY(e->nccl, e->nccl->GroupEnd());
  for (Shard& sh : e->shards) {
    int n = 0;
    if (e->nccl->CommCount && e->nccl->CommCount(sh.comm, &n) == 0) sh.nccl_ranks = n;
  }
  return 0;
}

int init_device(pcdn_engine* e) {
  const pcdn_config& c = e->cfg;
  int ndev = 0;
  cudaError_t err = cudaGetDeviceCount(&ndev);
  if (err != cudaSuccess || ndev == 0)
    return fail(PCDN_ENODEV, std::string("no CUDA device: ") + cudaGetErrorString(err));
  int prev = -1;
  cudaGetDevice(&prev);
  const uint32_t M = c.max_batch_msgs;
  e->topics_cap = (size_t)M * 4 + 4096;
  // in-batch subscription events: up to max_batch_msgs of them; their topics share topics_cap
  const uint32_t max_ev = (c.flags & PCDN_FLAG_INBATCH_SUBSCRIBE) ? M : 0;
  // The largest descriptor block: DescLayout grows with every count, so a full batch bounds every batch.
  // Splitting the topic entries between messages and events adds at most 16 bytes of alignment.
  const size_t desc_cap = DescLayout(M, std::min(M, c.max_batch_bcast), e->topics_cap, max_ev, 0).total + (max_ev ? 16 : 0);
  e->frames_cap = c.max_batch_bytes + 64;
  e->arena_cap = e->frames_cap + 256 + desc_cap;
  e->has_device = true;
  for (size_t i = 0; i < e->shards.size(); i++) {
    int rc = init_shard(e, e->shards[i], ndev, i == 0 ? c.stream : nullptr);
    if (rc) return rc;
  }
  e->slots.resize(c.batch_slots);
  for (Slot& s : e->slots) {
    int rc = pin_alloc(&s.h_arena, e->arena_cap);
    if (rc) return rc;
  }
  if (e->sharded && e->ingest == PCDN_INGEST_NCCL) {
    int rc = init_nccl(e);
    if (rc) return rc;
  }
  if (prev >= 0) cudaSetDevice(prev);
  return 0;
}

}  // namespace
// ================================================================================== C ABI
#define LOCK std::lock_guard<std::mutex> _g(e->mu)
#define GUARD_BEGIN try {
#define GUARD_END                                                          \
  } catch (const std::bad_alloc&) { return fail(PCDN_ENOMEM, "host allocation failed"); } \
  catch (const std::exception& ex) { return fail(PCDN_EINVAL, ex.what()); }

extern "C" {

uint32_t pcdn_abi_version(void) { return PCDN_ABI_VERSION; }
const char* pcdn_last_error(void) { return g_err.c_str(); }

void pcdn_config_default(pcdn_config* c) {
  std::memset(c, 0, sizeof(*c));
  c->struct_size = sizeof(pcdn_config);
  c->device = 0;
  c->max_conns = 1 << 16;
  c->max_topics = 256;
  c->max_keys = 1 << 17;
  c->max_key_len = 128;
  c->ring_bytes_per_conn = 1 << 16;
  c->max_batch_msgs = 4096;
  c->max_batch_bcast = 1024;
  c->max_batch_bytes = 64ull << 20;
  c->max_batch_deliveries = 16ull << 20;
  c->batch_slots = 4;
  c->n_valid_topics = 0;
  c->hash_seed = 0;
  c->identity = "/";
}

int pcdn_create(const pcdn_config* cfg, pcdn_engine** out) {
  GUARD_BEGIN
  if (!cfg || !out) return fail(PCDN_EINVAL, "null argument");
  // a config of the size before ref_min_bytes existed: the field is 0 (every delivery a framed copy)
  constexpr uint32_t kNoRefMinSize = offsetof(pcdn_config, ref_min_bytes);
  if (cfg->struct_size != sizeof(pcdn_config) && cfg->struct_size != kNoRefMinSize)
    return fail(PCDN_EINVAL, "pcdn_config.struct_size mismatch (ABI)");
  if (cfg->struct_size == kNoRefMinSize) {
    pcdn_config full{};
    std::memcpy(&full, cfg, kNoRefMinSize);
    full.struct_size = sizeof(pcdn_config);
    return pcdn_create(&full, out);
  }
  if (!cfg->max_conns || !cfg->max_topics || cfg->max_topics > 65536 || !cfg->max_keys || !cfg->max_key_len ||
      !cfg->max_batch_msgs || !cfg->batch_slots)
    return fail(PCDN_EINVAL, "zero or out-of-range capacity in pcdn_config");
  if (cfg->max_batch_bcast == 0 || cfg->max_batch_bcast > 65535) return fail(PCDN_EINVAL, "max_batch_bcast must be 1..65535");
  if (cfg->ring_bytes_per_conn % PCDN_RECORD_ALIGN || cfg->ring_bytes_per_conn == 0 || cfg->ring_bytes_per_conn > (1ull << 31))
    return fail(PCDN_EINVAL, "ring_bytes_per_conn must be a multiple of 32, at most 2 GiB");
  if (cfg->max_key_len > 4096) return fail(PCDN_EINVAL, "max_key_len > 4096");
  if (cfg->pack_variant & ~0xFF00u)
    return fail(PCDN_EINVAL, "pack_variant: only the CTA-count fields remain (bits 8-11: k_pack, bits 12-15: k_pack_direct CTAs per SM)");
  if (cfg->ref_min_bytes && (cfg->flags & PCDN_FLAG_SHARED_PAYLOAD))
    return fail(PCDN_EINVAL, "ref_min_bytes and PCDN_FLAG_SHARED_PAYLOAD exclude each other (the flag delivers every message by reference)");
  if (cfg->ref_min_bytes > 0x1FFFFFFFu) return fail(PCDN_EINVAL, "ref_min_bytes above MAX_MESSAGE_SIZE (0x1FFFFFFF)");
  // ---- connection shards
  const uint32_t n_local = cfg->n_devices ? cfg->n_devices : 1;
  const uint32_t world = cfg->world_shards ? cfg->world_shards : n_local;
  if (cfg->n_devices && !cfg->devices) return fail(PCDN_EINVAL, "n_devices > 0 but devices == NULL");
  if (n_local > 64 || world > 1024 || cfg->first_shard + n_local > world)
    return fail(PCDN_EINVAL, "shard layout: first_shard + n_devices must be <= world_shards");
  if (cfg->ingest != PCDN_INGEST_NCCL && cfg->ingest != PCDN_INGEST_HOST) return fail(PCDN_EINVAL, "unknown pcdn_config.ingest");
  const bool host_only = cfg->n_devices ? false : cfg->device < 0;
  if (world > n_local && cfg->ingest == PCDN_INGEST_NCCL && !cfg->nccl_unique_id && !host_only)
    return fail(PCDN_EINVAL, "a multi-process group needs pcdn_config.nccl_unique_id (pcdn_nccl_unique_id)");
  const uint64_t shard_N = align_up(cfg->max_conns, 32 * kBlockWords);
  if (shard_N * world > 0xFFFF0000ull) return fail(PCDN_EINVAL, "connection id space (max_conns x shards) exceeds 32 bits");
  if (cfg->n_devices && cfg->ingest == PCDN_INGEST_NCCL && world > 1)
    for (uint32_t i = 0; i < n_local; i++)
      for (uint32_t j = 0; j < i; j++)
        if (cfg->devices[i] == cfg->devices[j])
          return fail(PCDN_EINVAL, "PCDN_INGEST_NCCL needs one GPU per shard (use PCDN_INGEST_HOST for shards that share a device)");
  pcdn_engine* e = new pcdn_engine();
  e->cfg = *cfg;
  e->pack_ctas = (cfg->pack_variant >> 8) & 15u;
  if (const uint32_t d = (cfg->pack_variant >> 12) & 15u) e->direct_ctas = d;
  e->identity = cfg->identity ? cfg->identity : "/";
  e->cfg.identity = e->identity.c_str();
  e->world_shards = world;
  e->first_shard = cfg->first_shard;
  e->sharded = world > 1;
  e->ingest = cfg->ingest;
  if (cfg->n_devices) e->devices.assign(cfg->devices, cfg->devices + cfg->n_devices);
  else e->devices.assign(1, cfg->device);
  e->cfg.devices = e->devices.data();
  e->cfg.nccl_unique_id = nullptr;  // consumed below; never dereferenced after pcdn_create returns
  Geometry& g = e->geo;
  g.n_shards = world;
  g.shard_N = (uint32_t)shard_N;
  g.shard_max_conns = cfg->max_conns;
  g.max_conns = (world - 1) * g.shard_N + cfg->max_conns;
  g.N = world * g.shard_N;
  g.W = g.N / 32;
  g.T = cfg->max_topics;
  g.max_keys = cfg->max_keys;
  g.max_key_len = cfg->max_key_len;
  g.key_stride = (uint32_t)align_up(cfg->max_key_len, 16);
  uint32_t nb = 1;
  while ((uint64_t)nb * 2 < cfg->max_keys) nb <<= 1;  // 4 slots per bucket → load factor <= 50 %
  g.nbuckets = nb;
  g.bucket_mask = nb - 1;
  g.max_owners = 4096;
  g.seed = cfg->hash_seed ? cfg->hash_seed : 0x243F6A8885A308D3ULL;
  if (cfg->flags & PCDN_FLAG_OUTPUT_POOL) {
    e->pool_bytes = cfg->pool_bytes ? cfg->pool_bytes : (uint64_t)cfg->max_conns * cfg->ring_bytes_per_conn;
    e->pool_bytes = e->pool_bytes / PCDN_RECORD_ALIGN * PCDN_RECORD_ALIGN;
    if (e->pool_bytes < 4096 || e->pool_bytes / PCDN_RECORD_ALIGN >= 0xFFFFFFFFull) {
      delete e;
      return fail(PCDN_EINVAL, "pool_bytes must be between 4 KiB and 128 GiB");
    }
  }
  if (cfg->ref_min_bytes) {
    // the largest record still copied must fit an empty ring (the pool): then no message overflows by its size alone
    const uint64_t largest_copy = align_up(4 + (uint64_t)cfg->ref_min_bytes - 1, PCDN_RECORD_ALIGN);
    const bool pool = (cfg->flags & PCDN_FLAG_OUTPUT_POOL) != 0;
    if (largest_copy > (pool ? e->pool_bytes : cfg->ring_bytes_per_conn)) {
      delete e;
      return fail(PCDN_EINVAL, pool ? "ref_min_bytes: the largest copied record (4 + ref_min_bytes - 1, 32-byte aligned) exceeds pool_bytes"
                                    : "ref_min_bytes: the largest copied record (4 + ref_min_bytes - 1, 32-byte aligned) exceeds ring_bytes_per_conn");
    }
  }
  e->tables.reset(new HostTables(g));
  e->conns.reset(new Connections(*e->tables, e->identity.c_str()));
  if (!host_only) {
    e->shards.resize(n_local);
    for (uint32_t i = 0; i < n_local; i++) { e->shards[i].device = e->devices[i]; e->shards[i].gindex = cfg->first_shard + i; }
    e->cfg.nccl_unique_id = cfg->nccl_unique_id;
    int rc = init_device(e);
    e->cfg.nccl_unique_id = nullptr;
    if (rc) { destroy_engine(e); return rc; }
  }
  *out = e;
  return 0;
  GUARD_END
}

void pcdn_destroy(pcdn_engine* e) {
  if (e) destroy_engine(e);
}

// ---- state ------------------------------------------------------------------------------------
int pcdn_add_user(pcdn_engine* e, const uint8_t* key, uint32_t key_len, const uint16_t* topics, uint32_t n,
                  pcdn_conn* out_conn) {
  GUARD_BEGIN
  LOCK;
  int rc = before_state_change(e);
  if (rc) return rc;
  rc = e->conns->add_user(std::string((const char*)key, key_len), topics, n, out_conn);
  if (rc) return fail(rc, "add_user failed (capacity, key length or topic id)");
  return 0;
  GUARD_END
}
int pcdn_add_users_bulk(pcdn_engine* e, const uint8_t* keys, uint32_t key_len, uint32_t key_stride, uint32_t n_users,
                        const uint16_t* topics, const uint32_t* topic_offsets, pcdn_conn* out_conns) {
  GUARD_BEGIN
  LOCK;
  int rc = before_state_change(e);
  if (rc) return rc;
  for (uint32_t i = 0; i < n_users; i++) {
    uint32_t conn;
    const uint16_t* t = topics ? topics + topic_offsets[i] : nullptr;
    uint32_t nt = topics ? topic_offsets[i + 1] - topic_offsets[i] : 0;
    rc = e->conns->add_user(std::string((const char*)keys + (size_t)i * key_stride, key_len), t, nt, &conn);
    if (rc) return fail(rc, "add_users_bulk failed at user " + std::to_string(i));
    if (out_conns) out_conns[i] = conn;
  }
  return 0;
  GUARD_END
}
int pcdn_remove_user(pcdn_engine* e, const uint8_t* key, uint32_t key_len) {
  GUARD_BEGIN
  LOCK;
  int rc = before_state_change(e);
  if (rc) return rc;
  rc = e->conns->remove_user(std::string((const char*)key, key_len));
  return rc ? fail(rc, "remove_user failed") : 0;
  GUARD_END
}
int pcdn_subscribe_user_to(pcdn_engine* e, const uint8_t* key, uint32_t key_len, const uint16_t* topics, uint32_t n) {
  GUARD_BEGIN
  LOCK;
  return sub_change(e, SUB_USER, std::string((const char*)key, key_len), topics, n);
  GUARD_END
}
int pcdn_unsubscribe_user_from(pcdn_engine* e, const uint8_t* key, uint32_t key_len, const uint16_t* topics, uint32_t n) {
  GUARD_BEGIN
  LOCK;
  return sub_change(e, UNSUB_USER, std::string((const char*)key, key_len), topics, n);
  GUARD_END
}
int pcdn_add_broker(pcdn_engine* e, const char* identifier, pcdn_conn* out_conn) {
  GUARD_BEGIN
  LOCK;
  int rc = before_state_change(e);
  if (rc) return rc;
  rc = e->conns->add_broker(identifier, out_conn);
  return rc ? fail(rc, "add_broker failed") : 0;
  GUARD_END
}
int pcdn_remove_broker(pcdn_engine* e, const char* identifier) {
  GUARD_BEGIN
  LOCK;
  int rc = before_state_change(e);
  if (rc) return rc;
  return e->conns->remove_broker(identifier);
  GUARD_END
}
int pcdn_subscribe_broker_to(pcdn_engine* e, const char* identifier, const uint16_t* topics, uint32_t n) {
  GUARD_BEGIN
  LOCK;
  return sub_change(e, SUB_BROKER, std::string(identifier ? identifier : ""), topics, n);   // (BrokerIdent::parse reads null as "")
  GUARD_END
}
int pcdn_unsubscribe_broker_from(pcdn_engine* e, const char* identifier, const uint16_t* topics, uint32_t n) {
  GUARD_BEGIN
  LOCK;
  return sub_change(e, UNSUB_BROKER, std::string(identifier ? identifier : ""), topics, n);   // (BrokerIdent::parse reads null as "")
  GUARD_END
}
int pcdn_apply_user_sync(pcdn_engine* e, const char* remote_identity, const pcdn_user_sync_entry* entries, uint32_t n) {
  GUARD_BEGIN
  LOCK;
  int rc = before_state_change(e);
  if (rc) return rc;
  std::vector<UserSyncEntry> v;
  v.reserve(n);
  for (uint32_t i = 0; i < n; i++)
    v.push_back(UserSyncEntry{std::string((const char*)entries[i].key, entries[i].key_len), entries[i].version,
                              entries[i].owner != nullptr, entries[i].owner ? entries[i].owner : ""});
  rc = e->conns->apply_user_sync(remote_identity, v);
  return rc ? fail(rc, "apply_user_sync failed") : 0;
  GUARD_END
}

int pcdn_get_user_sync(pcdn_engine* e, int full, const pcdn_user_sync_entry** out, uint32_t* n) {
  GUARD_BEGIN
  LOCK;
  if (full) e->conns->get_full_user_sync(e->sync_users);
  else e->conns->get_partial_user_sync(e->sync_users);
  e->sync_users_c.clear();
  for (const UserSyncEntry& u : e->sync_users)
    e->sync_users_c.push_back(pcdn_user_sync_entry{(const uint8_t*)u.key.data(), (uint32_t)u.key.size(), u.version,
                                                   u.has_owner ? u.owner.c_str() : nullptr});
  *out = e->sync_users_c.data();
  *n = (uint32_t)e->sync_users_c.size();
  return 0;
  GUARD_END
}
int pcdn_apply_topic_sync(pcdn_engine* e, const char* identifier, uint32_t remote_identity,
                          const pcdn_topic_sync_entry* entries, uint32_t n) {
  GUARD_BEGIN
  LOCK;
  int rc = before_state_change(e);
  if (rc) return rc;
  std::vector<TopicSyncEntry> v;
  v.reserve(n);
  for (uint32_t i = 0; i < n; i++) v.push_back(TopicSyncEntry{entries[i].topic, entries[i].status, entries[i].version});
  rc = e->conns->apply_topic_sync(identifier, remote_identity, v);
  return rc ? fail(rc, "topic id out of range") : 0;
  GUARD_END
}
int pcdn_get_topic_sync(pcdn_engine* e, int full, const pcdn_topic_sync_entry** out, uint32_t* n) {
  GUARD_BEGIN
  LOCK;
  if (full) e->conns->get_full_topic_sync(e->sync_topics);
  else e->conns->get_partial_topic_sync(e->sync_topics);
  e->sync_topics_c.clear();
  for (const TopicSyncEntry& t : e->sync_topics) {
    pcdn_topic_sync_entry c{};
    c.topic = t.topic; c.status = t.status; c.version = t.version;
    e->sync_topics_c.push_back(c);
  }
  *out = e->sync_topics_c.data();
  *n = (uint32_t)e->sync_topics_c.size();
  return 0;
  GUARD_END
}

// ---- data in ----------------------------------------------------------------------------------
int pcdn_handle_broadcast_message(pcdn_engine* e, const uint16_t* topics, uint32_t n_topics, const uint8_t* raw,
                                  uint32_t raw_len, int to_users_only) {
  GUARD_BEGIN
  LOCK;
  return handle_msg(e, PCDN_KIND_BROADCAST, to_users_only ? PCDN_TO_USERS_ONLY : 0, topics, n_topics, nullptr, 0, raw, raw_len);
  GUARD_END
}
int pcdn_handle_direct_message(pcdn_engine* e, const uint8_t* recipient, uint32_t recipient_len, const uint8_t* raw,
                               uint32_t raw_len, int to_user_only) {
  GUARD_BEGIN
  LOCK;
  return handle_msg(e, PCDN_KIND_DIRECT, to_user_only ? PCDN_TO_USERS_ONLY : 0, nullptr, 0, recipient, recipient_len, raw, raw_len);
  GUARD_END
}

// ---- data out: frames the broker itself sends to its peer brokers ------------------------------
namespace {
// Inner::try_send_to_broker / try_send_to_brokers (tasks/broker/sender.rs:17-59): `raw` as one broadcast slot of
// the open batch whose recipients are the broker `identifier` (null: every peer broker) as connected now.  The
// mirror names the recipients: add_broker / remove_broker launch the open batch first (R12), so the batch is
// routed against this same set.  1 = nothing to send to (no such broker / no broker at all): nothing is appended.
int send_to_brokers(pcdn_engine* e, const char* identifier, const uint8_t* raw, uint32_t raw_len) {
  if (raw_len && !raw) return fail(PCDN_EINVAL, "null frame with non-zero length");
  if (const char* why = msg_invalid(e, MsgShape{PCDN_KIND_BROADCAST, raw_len, 0, 0, true})) return fail(PCDN_EINVAL, why);
  if (!e->has_device) return fail(PCDN_ENODEV, "host-only engine cannot route messages");
  uint32_t target = kConnNone;
  if (identifier) {
    target = e->conns->broker_conn(identifier);
    if (target == PCDN_CONN_NONE) return 1;   // if let Some(connection) = connection (sender.rs:29)
  } else if (e->conns->num_brokers() == 0) {
    return 1;                                 // the loop over no broker (sender.rs:52-57)
  }
  e->rx_reserve(1);
  api_entry(e, 0, PCDN_KIND_BROADCAST, MSGF_TARGET, nullptr, 0, nullptr, 0, raw, raw_len);
  e->rx_msgs[0].target = target;
  place_entries(e, nullptr, 1, nullptr, false);
  return e->rx_plan[0].rc;
}
}  // namespace

int pcdn_send_to_broker(pcdn_engine* e, const char* identifier, const uint8_t* raw, uint32_t raw_len) {
  GUARD_BEGIN
  LOCK;
  return send_to_brokers(e, identifier ? identifier : "", raw, raw_len);   // (BrokerIdent::parse reads null as "")
  GUARD_END
}
int pcdn_send_to_brokers(pcdn_engine* e, const uint8_t* raw, uint32_t raw_len) {
  GUARD_BEGIN
  LOCK;
  return send_to_brokers(e, nullptr, raw, raw_len);
  GUARD_END
}

int pcdn_user_receive(pcdn_engine* e, const uint8_t* sender_key, uint32_t key_len, const uint8_t* raw, uint32_t raw_len) {
  GUARD_BEGIN
  LOCK;
  return receive_one(e, 0, sender_key, key_len, raw, raw_len);
  GUARD_END
}

int pcdn_broker_receive(pcdn_engine* e, const char* identifier, const uint8_t* raw, uint32_t raw_len) {
  GUARD_BEGIN
  LOCK;
  return receive_one(e, 1, (const uint8_t*)identifier, identifier ? (uint32_t)std::strlen(identifier) : 0, raw, raw_len);
  GUARD_END
}

int pcdn_set_message_hook(pcdn_engine* e, int origin, pcdn_message_hook cb, void* user) {
  GUARD_BEGIN
  LOCK;
  if (origin != 0 && origin != 1) return fail(PCDN_EINVAL, "origin must be 0 (user) or 1 (broker)");
  e->hook[origin] = cb;
  e->hook_user[origin] = cb ? user : nullptr;
  return 0;
  GUARD_END
}

int pcdn_receive_frames(pcdn_engine* e, const pcdn_frame* frames, uint32_t n, int32_t* rc_out) {
  GUARD_BEGIN
  LOCK;
  return receive_frames_locked(e, frames, n, rc_out);
  GUARD_END
}

int pcdn_flush(pcdn_engine* e, uint64_t* batch_id) {
  GUARD_BEGIN
  LOCK;
  return flush_open(e, batch_id);
  GUARD_END
}

// All-or-nothing check of an explicit batch against every per-batch capacity, BEFORE anything is
// staged: a refused pcdn_submit leaves no message behind that a later flush would deliver (and a
// retry would deliver twice).  A dry run of the staging rule over the whole batch, with every
// recipient key counted as staged beside its frame (the worst case).
static int validate_explicit_batch(pcdn_engine* e, const pcdn_msg* msgs, uint32_t n) {
  const pcdn_config& c = e->cfg;
  if (!e->has_device) return fail(PCDN_ENODEV, "host-only engine cannot route messages");
  if (n > c.max_batch_msgs) return fail(PCDN_ENOSPC, "batch larger than max_batch_msgs");
  if (n && !msgs) return fail(PCDN_EINVAL, "null message array");
  BatchFill fill;
  const char* full = nullptr;
  for (uint32_t i = 0; i < n; i++) {
    const pcdn_msg& m = msgs[i];
    if (m.kind != PCDN_KIND_BROADCAST && m.kind != PCDN_KIND_DIRECT)
      return fail(PCDN_EINVAL, "message " + std::to_string(i) + ": kind must be broadcast or direct");
    if (m.flags & ~(uint8_t)PCDN_TO_USERS_ONLY)
      return fail(PCDN_EINVAL, "message " + std::to_string(i) + ": unknown bits in pcdn_msg.flags");
    if ((m.raw_len && !m.raw) || (m.kind == PCDN_KIND_BROADCAST && m.n_topics && !m.topics) ||
        (m.kind == PCDN_KIND_DIRECT && m.recipient_len && !m.recipient))
      return fail(PCDN_EINVAL, "message " + std::to_string(i) + ": null pointer with non-zero length");
    const bool direct = m.kind == PCDN_KIND_DIRECT;
    const MsgShape shape{m.kind, m.raw_len, direct ? (uint32_t)align_up(std::min<uint32_t>(m.recipient_len, c.max_key_len + 1), 16) : 0u,
                         direct ? 0u : m.n_topics};
    if (const char* why = msg_invalid(e, shape)) return fail(PCDN_EINVAL, "message " + std::to_string(i) + ": " + why);
    if (!full) full = batch_limit(e, fill, shape);
    fill.add(shape);
  }
  if (full) return fail(PCDN_ENOSPC, std::string("batch exceeds ") + full);
  if (!pool_admits(e, fill.ingress)) return fail(PCDN_EAGAIN, "global memory pool exhausted: release a batch first");
  return 0;
}

int pcdn_submit(pcdn_engine* e, const pcdn_msg* msgs, uint32_t n, uint64_t* batch_id) {
  GUARD_BEGIN
  LOCK;
  if (batch_id) *batch_id = 0;
  int rc = validate_explicit_batch(e, msgs, n);  // before anything is staged or launched
  if (rc) return rc;
  rc = flush_open(e, nullptr);  // keep explicit batches separate from the implicit open one
  if (rc) return rc;
  if (n == 0) return 0;
  if ((rc = acquire_open_slot(e))) return rc;  // PCDN_EAGAIN: nothing staged
  e->rx_reserve(n);
  for (uint32_t i = 0; i < n; i++) {
    const pcdn_msg& m = msgs[i];
    api_entry(e, i, m.kind, m.flags, m.topics, m.n_topics, m.recipient, m.recipient_len, m.raw, m.raw_len);
  }
  const uint64_t before = e->next_batch_id;
  place_entries(e, nullptr, n, nullptr, false);
  for (uint32_t i = 0; i < n && !rc; i++) rc = e->rx_plan[i].rc;
  e->rx_release();
  if (rc == 0 && e->next_batch_id != before) rc = fail(PCDN_ENOSPC, "batch exceeded a per-batch capacity and was split");
  if (rc) { abandon_open(e); return rc; }  // unreachable after validation; never leave a half batch open
  return flush_open(e, batch_id);
  GUARD_END
}

int pcdn_submit_device(pcdn_engine* e, const pcdn_device_batch* b, uint64_t* batch_id) {
  GUARD_BEGIN
  LOCK;
  if (batch_id) *batch_id = 0;
  if (!e->has_device) return fail(PCDN_ENODEV, "host-only engine cannot route messages");
  if (!b || b->n_msgs == 0 || b->n_msgs > e->cfg.max_batch_msgs || b->n_bcast > e->cfg.max_batch_bcast ||
      b->n_bcast > b->n_msgs)
    return fail(PCDN_EINVAL, "device batch exceeds configured capacities");
  const uint32_t n = b->n_msgs, nb = b->n_bcast;
  const bool shared = e->delivers_by_ref();   // the frames are staged on the host as the payload of reference records
  if (shared && b->arena_bytes > e->frames_cap)
    return fail(PCDN_ENOSPC, "device batch frames exceed the pinned payload staging (max_batch_bytes)");
  // sharded engines: the frames at the start of a receiving shard's arena, the descriptor block behind them
  const DescLayout L(n, nb, b->n_topics_total);
  const size_t doff = align_up(b->arena_bytes, 256);
  if (e->sharded) {
    if (doff + L.total > e->arena_cap) return fail(PCDN_ENOSPC, "device batch does not fit the shards' ingest region (max_batch_bytes)");
    if (e->ingest == PCDN_INGEST_HOST && e->world_shards != e->shards.size())
      return fail(PCDN_EINVAL, "device-resident batches in a multi-process group need PCDN_INGEST_NCCL");
  }
  int rc = flush_open(e, nullptr);
  if (rc) return rc;
  if ((rc = acquire_open_slot(e))) return rc;
  const uint32_t si = (uint32_t)e->open_slot;
  Slot& s = e->slots[si];
  if ((rc = flush_journal(e))) { abandon_open(e); return rc; }
  const bool ready = (b->hints & PCDN_BATCH_READY) != 0;
  const bool arena_in_place = b->arena_bytes > (4u << 20);   // large frame arenas are broadcast from the caller's buffer
  if (e->sharded) {
    // the batch lives on the root GPU (global shard 0): unless the caller says its buffers are complete,
    // everything queued so far on the root's main stream (the caller's producer kernels when it shares
    // that stream) comes before the broadcast
    if (e->owns_root() && !ready) {
      Shard& root = e->shards[0];
      DeviceGuard dg(root.device);
      CUDA_TRY(cudaEventRecord(root.ev_submit, root.stream));
    }
    const IngestRegion regs[9] = {
        {b->arena, 0, (size_t)b->arena_bytes}, {b->kind, doff + L.o_kind, n}, {b->flags, doff + L.o_flags, n},
        {b->slot_off16, doff + L.o_slot, (size_t)n * 4}, {b->raw_len, doff + L.o_len, (size_t)n * 4},
        {b->aux_off, doff + L.o_aoff, (size_t)n * 4}, {b->aux_len, doff + L.o_alen, (size_t)n * 4},
        {b->bcast_index, doff + L.o_bidx, (size_t)nb * 4}, {b->topics, doff + L.o_top, (size_t)b->n_topics_total * 2}};
    if ((rc = ingest_batch(e, si, regs, 9, arena_in_place, !ready))) { abandon_open(e); return rc; }
  }
  for (Shard& sh : e->shards) {
    ShardSlot& ss = sh.slots[si];
    if (e->sharded)   // the replicated copy in this shard's slot region (the root keeps large frames in place)
      ss.in = bind_batch((sh.gindex == 0 && arena_in_place) ? (const uint8_t*)b->arena : ss.d_arena, ss.d_arena + doff, L);
    else              // where the caller put it
      ss.in = BatchIn{n, nb, (const uint8_t*)b->arena, b->kind, b->flags, b->slot_off16, b->raw_len, b->aux_off, b->aux_len,
                      b->topics, b->bcast_index};
  }
  if (shared) {
    // the payload of the reference records: ONE D2H copy of the frames, from where the first local shard
    // reads them, on that shard's main stream ahead of the batch's kernels (so its ev_done covers it)
    Shard& sh = e->shards[0];
    ShardSlot& ss = sh.slots[si];
    DeviceGuard dg(sh.device);
    cudaError_t ce = e->sharded ? cudaStreamWaitEvent(sh.stream, ss.ev_ingest, 0) : cudaSuccess;
    if (ce == cudaSuccess && b->arena_bytes)
      ce = cudaMemcpyAsync(s.h_arena, ss.in.arena, b->arena_bytes, cudaMemcpyDeviceToHost, sh.stream);
    if (ce != cudaSuccess) { abandon_open(e); return fail(PCDN_ECUDA, std::string("payload staging copy: ") + cudaGetErrorString(ce)); }
  }
  s.device_input = true;
  s.n_msgs = n;
  s.n_direct = n - nb;
  if ((rc = launch_pipeline(e, si, e->sharded))) { abandon_open(e); return rc; }
  if (batch_id) *batch_id = s.batch_id;
  return 0;
  GUARD_END
}

// ---- data out ---------------------------------------------------------------------------------
int pcdn_next_batch(pcdn_engine* e, uint64_t* batch_id) {
  LOCK;
  *batch_id = e->inflight.empty() ? 0 : e->inflight.front();
  return 0;
}

extern "C++" {
namespace {

void fill_result(pcdn_engine* e, const Slot& s, const Shard& sh, const ShardSlot& ss, uint64_t batch_id, pcdn_batch_result* out) {
  const BatchStats& bs = *ss.h_stats;
  const uint32_t cap = e->geo.shard_max_conns;
  out->batch_id = batch_id;
  out->n_msgs = s.n_msgs;
  // a batch the device refused (scatter-list capacity, output pool) wrote nothing: its provisional
  // counters (the offsets pass counts before the pool says no) are not deliveries
  const bool refused = bs.status != 0;
  out->n_spans = refused ? 0 : std::min<uint32_t>(bs.n_spans, 2 * cap);
  out->spans = sh.dev.span_runs ? nullptr : reinterpret_cast<const pcdn_span*>(ss.h_spans);
  out->runs = sh.dev.span_runs ? reinterpret_cast<const pcdn_span_run*>(ss.h_spans) : nullptr;
  out->n_runs = (sh.dev.span_runs && !refused) ? std::min<uint32_t>(bs.n_runs, 2 * e->geo.shard_N) : 0;

  out->n_deliveries = refused ? 0 : bs.n_deliveries;
  out->bytes_out = refused ? 0 : bs.bytes_out;
  out->n_overflow = refused ? 0 : std::min<uint32_t>(bs.n_overflow, cap);
  out->overflow_conns = ss.h_overflow;
  out->n_direct_dropped = bs.n_direct_dropped;
  // device status: 1 = scatter list capacity, 3 = larger than the whole output pool (E2BIG); 2 = no room in the pool right now (EAGAIN)
  out->status = bs.status == 0 ? 0 : (bs.status == 2 ? (uint32_t)(-PCDN_EAGAIN) : (uint32_t)(-PCDN_E2BIG));
  out->pool_base = sh.dev.pool ? bs.pool_base : 0;
  out->msg_status = s.devparse ? ss.h_msg_status : nullptr;
  out->n_msg_errors = ss.n_msg_errors;
  out->reserved = sh.gindex;
}

// wait for (or test) one shard's share of a batch and fetch its results; returns 1 when !block and
// the shard is not done yet.  The blocking waits happen OUTSIDE the engine lock, so ingest threads
// keep appending to the next batch while an egress thread waits for this one (one poller per
// shard and batch).
}  // namespace
int pcdn_detail::poll_one(pcdn_engine* e, uint64_t batch_id, uint32_t li, int block) {
  cudaEvent_t ev_early = nullptr, ev_done = nullptr;
  bool mapped = false;
  int device = 0;
  {
    std::lock_guard<std::mutex> g(e->mu);
    const int si = find_slot_index(e, batch_id);
    if (si < 0) return fail(PCDN_ENOENT, "unknown batch id");
    if (li >= e->shards.size()) return fail(PCDN_EINVAL, "no such local shard");
    ShardSlot& ss = e->shards[li].slots[si];
    if (ss.polled) return 0;
    device = e->shards[li].device;
    if (!block) {
      DeviceGuard dg(device);
      cudaError_t q = cudaEventQuery(ss.ev_done);
      if (q == cudaErrorNotReady) return 1;
      CUDA_TRY(q);
    }
    ev_early = ss.ev_early; ev_done = ss.ev_done; mapped = ss.spans_mapped;
  }
  DeviceGuard dg(device);
  uint32_t nsp = 0, nov = 0;
  bool devparse = false;
  // 1. counters as of k_offsets → exact size of the span table; its D2H overlaps the pack
  //    (mapped spans: the table is already in host memory when ev_done fires)
  if (!mapped) CUDA_TRY(cudaEventSynchronize(ev_early));
  {
    std::lock_guard<std::mutex> g(e->mu);
    const int si = find_slot_index(e, batch_id);
    if (si < 0) return fail(PCDN_ENOENT, "batch released while it was being polled");
    Shard& sh = e->shards[li];
    ShardSlot& ss = sh.slots[si];
    devparse = e->slots[si].devparse;
    if (!mapped && !ss.polled) {
      const bool runs = sh.dev.span_runs != 0;
      nsp = std::min<uint32_t>(runs ? ss.h_early->n_runs : ss.h_early->n_spans, 2 * e->geo.shard_N);
      nov = std::min<uint32_t>(ss.h_early->n_overflow, e->geo.shard_max_conns);
      if (nsp) CUDA_TRY(cudaMemcpyAsync(ss.h_spans, ss.w.spans, (size_t)nsp * (runs ? sizeof(SpanRun) : sizeof(Span)), cudaMemcpyDeviceToHost, sh.copy_stream));
      if (nov) CUDA_TRY(cudaMemcpyAsync(ss.h_overflow, ss.w.overflow, (size_t)nov * 4, cudaMemcpyDeviceToHost, sh.copy_stream));
    }
  }
  // 2. the pack itself (ring bytes are valid after this)
  CUDA_TRY(cudaEventSynchronize(ev_done));
  std::lock_guard<std::mutex> _g(e->mu);
  const int si = find_slot_index(e, batch_id);
  if (si < 0) return fail(PCDN_ENOENT, "batch released while it was being polled");
  Shard& sh = e->shards[li];
  ShardSlot& ss = sh.slots[si];
  if (!ss.polled) {
    if (devparse) CUDA_TRY(cudaMemcpyAsync(ss.h_msg_status, ss.w.msg_status, ss.in.n_msgs, cudaMemcpyDeviceToHost, sh.copy_stream));
    if (nsp || nov || devparse) CUDA_TRY(cudaStreamSynchronize(sh.copy_stream));
    if (devparse) { ss.n_msg_errors = 0; for (uint32_t i = 0; i < ss.in.n_msgs; i++) ss.n_msg_errors += ss.h_msg_status[i] != 0; }
    const BatchStats& bs = *ss.h_stats;
    ss.polled = true;
    if (!bs.status) {
      e->stats.deliveries += bs.n_deliveries;
      e->stats.bytes_out += bs.bytes_out;
    }
    if (ss.timed && li == 0) {  // stage times of the first local shard (shards run the same pipeline side by side)
      float t[4] = {0, 0, 0, 0};
      for (int i = 0; i < 3; i++) cudaEventElapsedTime(&t[i], ss.ev[i], ss.ev[i + 1]);
      cudaEventElapsedTime(&t[3], ss.ev[4], ss.ev[5]);
      e->stats.ms_direct += t[0];
      e->stats.ms_match += t[1];
      e->stats.ms_plan += t[2];
      e->stats.ms_pack += t[3];
      e->stats.ms_total += t[0] + t[1] + t[2] + t[3];
      e->stats.timed_batches++;
    }
  }
  return 0;
}

}  // extern "C++"

int pcdn_poll_shard(pcdn_engine* e, uint64_t batch_id, uint32_t local_shard, pcdn_batch_result* out, int block) {
  GUARD_BEGIN
  if (!e->has_device) return fail(PCDN_ENODEV, "host-only engine");
  int rc = poll_one(e, batch_id, local_shard, block);
  if (rc) return rc;
  std::lock_guard<std::mutex> _g(e->mu);
  const int si = find_slot_index(e, batch_id);
  if (si < 0) return fail(PCDN_ENOENT, "batch released while it was being polled");
  if (out) fill_result(e, e->slots[si], e->shards[local_shard], e->shards[local_shard].slots[si], batch_id, out);
  return 0;
  GUARD_END
}

int pcdn_poll(pcdn_engine* e, uint64_t batch_id, pcdn_batch_result* out, int block) {
  GUARD_BEGIN
  if (!e->has_device) return fail(PCDN_ENODEV, "host-only engine");
  const uint32_t nl = (uint32_t)e->shards.size();
  if (nl == 1) return pcdn_poll_shard(e, batch_id, 0, out, block);
  for (uint32_t li = 0; li < nl; li++) {
    int rc = poll_one(e, batch_id, li, block);
    if (rc) return rc;  // error, or 1 = some shard still running
  }
  std::lock_guard<std::mutex> _g(e->mu);
  const int si = find_slot_index(e, batch_id);
  if (si < 0) return fail(PCDN_ENOENT, "batch released while it was being polled");
  Slot& s = e->slots[si];
  if (out) {
    // summed counters + the shards' span tables concatenated (ascending shard = ascending id range)
    s.merged_spans.clear(); s.merged_overflow.clear(); s.merged_runs.clear();
    pcdn_batch_result tot{};
    for (uint32_t li = 0; li < nl; li++) {
      pcdn_batch_result r{};
      fill_result(e, s, e->shards[li], e->shards[li].slots[si], batch_id, &r);
      // (output pool: every shard's offsets are relative to ITS region — the merged view carries absolute unit offsets)
      const size_t s0 = s.merged_spans.size(), r0 = s.merged_runs.size();
      if (r.spans) s.merged_spans.insert(s.merged_spans.end(), r.spans, r.spans + r.n_spans);
      if (r.runs) s.merged_runs.insert(s.merged_runs.end(), r.runs, r.runs + r.n_runs);
      if (r.pool_base) {
        for (size_t i = s0; i < s.merged_spans.size(); i++) s.merged_spans[i].ring_off += r.pool_base;
        for (size_t i = r0; i < s.merged_runs.size(); i++) s.merged_runs[i].ring_off += r.pool_base;
      }
      tot.n_spans += r.n_spans;
      s.merged_overflow.insert(s.merged_overflow.end(), r.overflow_conns, r.overflow_conns + r.n_overflow);
      tot.n_deliveries += r.n_deliveries; tot.bytes_out += r.bytes_out; tot.n_direct_dropped += r.n_direct_dropped;
      if (r.status == (uint32_t)(-PCDN_EAGAIN) || (r.status && !tot.status)) tot.status = r.status;   // "retry" wins over "too big"
      if (li == 0) { tot.msg_status = r.msg_status; tot.n_msg_errors = r.n_msg_errors; }  // identical on every shard
    }
    tot.batch_id = batch_id; tot.n_msgs = s.n_msgs;
    tot.spans = s.merged_runs.empty() && !(e->cfg.flags & PCDN_FLAG_SPAN_RUNS) ? s.merged_spans.data() : nullptr;
    tot.runs = (e->cfg.flags & PCDN_FLAG_SPAN_RUNS) ? s.merged_runs.data() : nullptr;
    tot.n_runs = (uint32_t)s.merged_runs.size();
    tot.n_overflow = (uint32_t)s.merged_overflow.size(); tot.overflow_conns = s.merged_overflow.data();
    *out = tot;
  }
  return 0;
  GUARD_END
}

int pcdn_read(pcdn_engine* e, pcdn_conn conn, uint32_t ring_off, uint32_t len, void* dst) {
  GUARD_BEGIN
  LOCK;
  if (!e->has_device) return fail(PCDN_ENODEV, "host-only engine");
  const uint32_t gs = conn / e->geo.shard_N, local = conn % e->geo.shard_N;
  if (gs < e->first_shard || gs >= e->first_shard + e->shards.size())
    return fail(PCDN_ENOENT, "connection lives on a shard of another process");
  Shard& sh = e->shards[gs - e->first_shard];
  size_t at;
  if (sh.dev.pool) {  // ring_off = absolute 32-byte unit inside the shard's output pool (pool_base + span offset)
    at = (size_t)ring_off * PCDN_RECORD_ALIGN;
    if (local >= e->geo.shard_max_conns || at + len > e->pool_bytes) return fail(PCDN_EINVAL, "read outside the output pool");
  } else {
    if (local >= e->geo.shard_max_conns || (uint64_t)ring_off + len > e->cfg.ring_bytes_per_conn)
      return fail(PCDN_EINVAL, "read outside the connection's ring");
    at = (size_t)local * e->cfg.ring_bytes_per_conn + ring_off;
  }
  if (sh.h_rings) {
    std::memcpy(dst, sh.h_rings + at, len);
    return 0;
  }
  DeviceGuard dg(sh.device);
  CUDA_TRY(cudaMemcpyAsync(dst, sh.dev.rings + at, len,
                           cudaMemcpyDeviceToHost, sh.copy_stream));
  CUDA_TRY(cudaStreamSynchronize(sh.copy_stream));
  return 0;
  GUARD_END
}

int pcdn_batch_payload(pcdn_engine* e, uint64_t batch_id, const uint8_t** host_base) {
  GUARD_BEGIN
  LOCK;
  if (host_base) *host_base = nullptr;
  if (!e->has_device) return fail(PCDN_ENODEV, "host-only engine");
  const int si = find_slot_index(e, batch_id);
  if (si < 0) return fail(PCDN_ENOENT, "unknown or released batch id");
  const Slot& s = e->slots[si];
  // host-staged batches keep their frames in the slot's pinned staging until release; device-resident
  // ones have them copied there only by engines that deliver by reference
  if (s.device_input && !e->delivers_by_ref())
    return fail(PCDN_ENOENT, "the frames of a device-resident batch are staged on the host only with PCDN_FLAG_SHARED_PAYLOAD or ref_min_bytes");
  if (host_base) *host_base = s.h_arena;
  return 0;
  GUARD_END
}

int pcdn_retry_batch(pcdn_engine* e, uint64_t batch_id) {
  GUARD_BEGIN
  LOCK;
  if (!e->has_device) return fail(PCDN_ENODEV, "host-only engine");
  if (!(e->cfg.flags & PCDN_FLAG_OUTPUT_POOL)) return fail(PCDN_EINVAL, "only batches of an output-pool engine can be refused for space");
  const int si = find_slot_index(e, batch_id);
  if (si < 0) return fail(PCDN_ENOENT, "unknown batch id");
  if (e->inflight.empty() || e->inflight.front() != batch_id)
    return fail(PCDN_EINVAL, "only the oldest unreleased batch can be retried (release the older ones first)");
  int rc = 0;
  uint32_t n = 0;
  for (Shard& sh : e->shards) {
    ShardSlot& ss = sh.slots[si];
    {
      DeviceGuard dg(sh.device);
      CUDA_TRY(cudaEventSynchronize(ss.ev_done));
    }
    if (ss.h_stats->status != 2) continue;   // this shard packed its share (or refused it for good): leave it alone
    if ((rc = launch_shard_pipeline(e, sh, (uint32_t)si, false, true))) return rc;
    n++;
  }
  if (!n) return fail(PCDN_EINVAL, "the batch was not refused for space");
  return 0;
  GUARD_END
}

int pcdn_release_batch(pcdn_engine* e, uint64_t batch_id) {
  GUARD_BEGIN
  LOCK;
  const int si = find_slot_index(e, batch_id);
  if (si < 0) return fail(PCDN_ENOENT, "unknown batch id");
  if (e->inflight.empty() || e->inflight.front() != batch_id)
    return fail(PCDN_EINVAL, "batches must be released oldest first");
  Slot& s = e->slots[si];
  for (Shard& sh : e->shards) {
    DeviceGuard dg(sh.device);
    ShardSlot& ss = sh.slots[si];
    // A slot released without having been polled may still have its host→device staging copy queued:
    // its pinned staging buffers must not be refilled before that copy ran (device-input batches have
    // no host staging and stay fully asynchronous — the pipelined submit_device/release loop — unless
    // their frames are being copied into the staging as the shared payload: ev_done comes after that copy).
    const bool payload_copy = s.device_input && e->delivers_by_ref();
    if (!ss.polled && (!s.device_input || payload_copy))
      CUDA_TRY(cudaEventSynchronize((e->sharded && !payload_copy) ? ss.ev_ingest : ss.ev_done));
    // ring space may be reused only after the pack that filled it has finished
    CUDA_TRY(cudaStreamWaitEvent(sh.stream, ss.ev_done, 0));
    launch_release(sh.dev, ss.w.batch_units, ss.w.stats, sh.stream);
    CUDA_TRY(cudaGetLastError());
  }
  e->inflight.erase(e->inflight.begin());
  s.state = SLOT_FREE;
  // the last 'clone' of every frame of this batch is gone: permits back to the pool (pool.rs:44-52)
  e->inflight_bytes -= std::min(e->inflight_bytes, s.ingress_bytes);
  s.ingress_bytes = 0;
  e->stats.released_batches++;
  {
    const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - s.t_launch).count();
    e->stats.latency_ms_sum += ms;
    const uint64_t us = (uint64_t)(ms * 1000.0);
    int bucket = 0;
    while (bucket < 15 && us >= (16ull << bucket)) bucket++;
    e->stats.latency_hist_us[bucket]++;
  }
  return 0;
  GUARD_END
}

// ---- connection shards -------------------------------------------------------------------------
int pcdn_nccl_unique_id(void* out128) {
  GUARD_BEGIN
  if (!out128) return fail(PCDN_EINVAL, "null argument");
  const char* why = "";
  const NcclApi* nc = nccl_api(&why);
  if (!nc) return fail(PCDN_ENODEV, std::string("libnccl.so.2 not available: ") + why);
  NcclUniqueId id;
  NCCL_TRY(nc, nc->GetUniqueId(&id));
  std::memcpy(out128, &id, sizeof(id));
  return 0;
  GUARD_END
}
int pcdn_num_shards(pcdn_engine* e, uint32_t* n_local, uint32_t* n_world) {
  LOCK;
  if (n_local) *n_local = e->has_device ? (uint32_t)e->shards.size() : 0;
  if (n_world) *n_world = e->world_shards;
  return 0;
}
int pcdn_shard_info(pcdn_engine* e, uint32_t local_shard, pcdn_shard_desc* out) {
  GUARD_BEGIN
  LOCK;
  if (!out) return fail(PCDN_EINVAL, "null argument");
  std::memset(out, 0, sizeof(*out));
  out->shard_stride = e->geo.shard_N;
  out->ring_bytes = (e->cfg.flags & PCDN_FLAG_OUTPUT_POOL) ? e->pool_bytes : e->cfg.ring_bytes_per_conn;
  if (!e->has_device) {  // host-only mirror: geometry only
    if (local_shard != 0) return fail(PCDN_EINVAL, "no such local shard");
    out->global_index = e->first_shard; out->device = -1; out->conn_base = e->first_shard * e->geo.shard_N;
    return 0;
  }
  if (local_shard >= e->shards.size()) return fail(PCDN_EINVAL, "no such local shard");
  const Shard& sh = e->shards[local_shard];
  out->global_index = sh.gindex;
  out->device = sh.device;
  out->conn_base = sh.dev.conn_base;
  out->rings_dev = sh.dev.rings;
  out->rings_host = sh.h_rings;
  out->nccl_ranks = (uint32_t)sh.nccl_ranks;
  std::vector<uint32_t> v;
  out->n_conns = e->conns->shard_load(sh.gindex);
  return 0;
  GUARD_END
}

// ---- introspection ----------------------------------------------------------------------------
int pcdn_get_stats(pcdn_engine* e, pcdn_stats* out) {
  LOCK;
  e->stats.inflight_bytes = e->inflight_bytes;
  e->stats.kernel_launches = kernel_launches();
  *out = e->stats;
  return 0;
}
int pcdn_set_timing(pcdn_engine* e, int on) {
  LOCK;
  e->timing = on != 0;
  return 0;
}
int pcdn_ring_info(pcdn_engine* e, void** dev_base, uint64_t* ring_bytes, uint32_t* max_conns) {
  LOCK;
  if (dev_base) *dev_base = e->has_device ? (void*)e->shards[0].dev.rings : nullptr;  // first local shard (pcdn_shard_info for the others)
  if (ring_bytes) *ring_bytes = e->cfg.ring_bytes_per_conn;
  if (max_conns) *max_conns = e->geo.shard_max_conns;
  return 0;
}
int pcdn_host_rings(pcdn_engine* e, const void** host_base) {
  LOCK;
  uint8_t* h = e->has_device ? e->shards[0].h_rings : nullptr;
  if (host_base) *host_base = h;
  return h ? 0 : fail(PCDN_ENOENT, "rings live in device memory (PCDN_FLAG_HOST_RINGS not set)");
}
int pcdn_num_users(pcdn_engine* e, uint32_t* users, uint32_t* brokers) {
  LOCK;
  if (users) *users = e->conns->num_users();
  if (brokers) *brokers = e->conns->num_brokers();
  return 0;
}
int pcdn_debug_interested(pcdn_engine* e, const uint16_t* topics, uint32_t n_topics, int to_users_only, pcdn_conn* out,
                          uint32_t cap, uint32_t* n) {
  GUARD_BEGIN
  LOCK;
  std::vector<uint32_t> v;
  e->conns->interested(topics, n_topics, to_users_only != 0, v);
  *n = (uint32_t)v.size();
  for (uint32_t i = 0; i < v.size() && i < cap; i++) out[i] = v[i];
  return 0;
  GUARD_END
}
int pcdn_debug_route(pcdn_engine* e, const uint8_t* key, uint32_t key_len, int* kind, pcdn_conn* conn) {
  GUARD_BEGIN
  LOCK;
  *kind = e->conns->route(std::string((const char*)key, key_len), conn);
  return 0;
  GUARD_END
}
int pcdn_parse_frame(const uint8_t* raw, uint32_t raw_len, uint16_t* topics_out, uint32_t* n_topics, uint32_t* field_off,
                     uint32_t* field_len) {
  ParsedFrame pf;
  if (!parse_frame(raw, raw_len, &pf)) return fail(PCDN_EPARSE, "failed to deserialize message");
  if (field_off) *field_off = pf.f0_off;
  if (field_len) *field_len = pf.f0_len;
  if (n_topics) *n_topics = 0;
  if ((pf.kind == PCDN_KIND_BROADCAST || pf.kind == PCDN_KIND_SUBSCRIBE || pf.kind == PCDN_KIND_UNSUBSCRIBE) && topics_out &&
      n_topics) {
    uint32_t n = std::min<uint32_t>(pf.f0_len, 256);
    for (uint32_t i = 0; i < n; i++) topics_out[i] = raw[pf.f0_off + i];
    *n_topics = n;
  }
  return pf.kind;
}

}  // extern "C"
