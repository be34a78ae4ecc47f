// kernels.cu — hand-written sm_90a kernels of the fan-out engine.  See kernels.cuh for the
// pipeline and DESIGN.md for the roofline of each kernel.  Everything here is integer/byte work
// bound by HBM bandwidth; there is deliberately no tensor-core code.
#include "kernels.cuh"

#include <atomic>

#include "frame_parse_core.h"

namespace pcdn {

// every kernel launch of the library is counted (pcdn_stats.kernel_launches: what bench.py reports as gpu_launches)
std::atomic<unsigned long long> g_kernel_launches{0};
#define PCDN_COUNT_LAUNCH (void)g_kernel_launches.fetch_add(1, std::memory_order_relaxed)

unsigned long long kernel_launches() { return g_kernel_launches.load(std::memory_order_relaxed); }
void count_kernel_launch() { PCDN_COUNT_LAUNCH; }

// =============================================================================== small helpers
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v) {
  const uint32_t lane = lane_id();
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    uint32_t n = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= (uint32_t)o) v += n;
  }
  return v;
}

// exclusive scan over a CTA of NW warps; *total = CTA sum.  `sm` needs NW+1 words (NW <= 32).
template <int NW>
__device__ __forceinline__ uint32_t cta_excl_scan(uint32_t v, uint32_t* total, uint32_t* sm) {
  const uint32_t lane = lane_id(), warp = threadIdx.x >> 5;
  uint32_t incl = warp_incl_scan(v);
  if (lane == 31) sm[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    uint32_t x = lane < NW ? sm[lane] : 0;
    uint32_t xi = warp_incl_scan(x);
    if (lane < NW) sm[lane] = xi - x;
    if (lane == NW - 1) sm[NW] = xi;
  }
  __syncthreads();
  uint32_t r = incl - v + sm[warp];
  *total = sm[NW];
  __syncthreads();
  return r;
}
// 256-thread block; `sm` needs 9 words
__device__ __forceinline__ uint32_t block256_excl_scan(uint32_t v, uint32_t* total, uint32_t* sm) {
  return cta_excl_scan<8>(v, total, sm);
}

__device__ __forceinline__ uint32_t bswap32(uint32_t x) { return __byte_perm(x, 0, 0x0123); }

// 16-byte streaming store: written once, never read back by the GPU
__device__ __forceinline__ void st_stream16(void* p, const uint4& v) {
  asm volatile("st.global.cs.v4.b32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}
__device__ __forceinline__ uint4 ld_nc16(const void* p) {
  uint4 v;
  asm volatile("ld.global.nc.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}

// ---- mbarrier / TMA bulk copy (cp.async.bulk → SASS UBLKCP) -----------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
  } while (!ok);
}
// global → shared, completion counted on the mbarrier
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// shared → global, bulk-group completion
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// =============================================================================== K4 table updates
__global__ void k_apply_u32(DevState s, const Upd32* __restrict__ u, uint32_t n) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Upd32 x = u[i];
  uint32_t* a = x.arr == 0 ? s.sub : (x.arr == 1 ? s.brk : s.owner_conn);
  a[x.idx] = x.val;
}
__global__ void k_apply_slots(DevState s, const UpdSlot* __restrict__ u, uint32_t n) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  s.cuckoo[u[i].slot] = u[i].e;
}
__global__ void k_apply_keys(DevState s, const uint32_t* __restrict__ slots, const uint8_t* __restrict__ bytes,
                             uint32_t n) {
  // one thread per 16 bytes of key
  uint32_t per = s.key_stride >> 4;
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (uint64_t)n * per) return;
  uint32_t k = (uint32_t)(i / per), v = (uint32_t)(i % per);
  const uint4* src = reinterpret_cast<const uint4*>(bytes + (size_t)k * s.key_stride) + v;
  uint4* dst = reinterpret_cast<uint4*>(s.keys + (size_t)slots[k] * s.key_stride) + v;
  *dst = *src;
}

void launch_apply_updates(const DevState& s, const Upd32* u32, uint32_t n32, const UpdSlot* us, uint32_t nslot,
                          const uint32_t* key_slots, const uint8_t* key_bytes, uint32_t nkeys, cudaStream_t st) {
  if (nkeys) {
    uint64_t th = (uint64_t)nkeys * (s.key_stride >> 4);
    PCDN_COUNT_LAUNCH, k_apply_keys<<<(unsigned)((th + 255) / 256), 256, 0, st>>>(s, key_slots, key_bytes, nkeys);
  }
  if (nslot) PCDN_COUNT_LAUNCH, k_apply_slots<<<(nslot + 255) / 256, 256, 0, st>>>(s, us, nslot);
  if (n32) PCDN_COUNT_LAUNCH, k_apply_u32<<<(n32 + 255) / 256, 256, 0, st>>>(s, u32, n32);
}

// =============================================================================== K0 ingress parse
// Thread per message (device-parse mode, SURVEY 8f-1): the same Cap'n Proto walk the host parser
// runs (frame_parse_core.h, compiled for both), on the raw frame already resident in the arena.
// Fills the routing fields the later kernels read — for a broadcast the wire topic list is used IN
// PLACE (byte offset + count, Topic::prune applied while matching), for a direct message the
// recipient key is read in place — and records a per-message outcome.  Host work per frame drops
// to a tag peek and one memcpy.
__global__ void __launch_bounds__(256) k_parse(DevState s, BatchIn b, Work w) {
  const uint32_t m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= b.n_msgs) return;
  uint8_t fl = b.flags[m];
  if (!(fl & MSGF_DEVPARSE)) return;
  const uint32_t slot_b = b.slot_off16[m] * 16u, len = b.raw_len[m];
  const uint8_t* raw = b.arena + slot_b + 4;
  uint8_t kind = b.kind[m];
  uint32_t aoff = 0, alen = 0;
  int8_t st = 0;
  ParsedFrame pf;
  if (!parse_frame_core(raw, len, &pf) || pf.kind != (int)kind) {
    st = kErrParse; kind = 0;
  } else if (kind == 4) {
    aoff = slot_b + 4 + pf.f0_off; alen = pf.f0_len; fl |= MSGF_TOPICS_U8;
    if (fl & MSGF_PRUNE) {
      uint32_t kept = 0;
      for (uint32_t i = 0; i < alen; i++) kept += topic_kept(raw + pf.f0_off, i, s.n_valid_topics) ? 1u : 0u;
      if (kept == 0) { st = kErrPrune; alen = 0; kind = 0; }  // Err("supplied no valid topics")
    }
  } else {  // direct: recipient key in place (word aligned in a valid message)
    aoff = slot_b + 4 + pf.f0_off; alen = pf.f0_len;
    if (aoff & 3) kind = 0;
    // longer than any registered key: its first max_key_len + 1 bytes match no entry, so the lookup
    // drops it and counts it, as the host staging does (engine.cu routed_key_len)
    else if (alen > s.max_key_len) alen = s.max_key_len + 1;
  }
  const_cast<uint8_t*>(b.kind)[m] = kind;
  const_cast<uint8_t*>(b.flags)[m] = fl;
  const_cast<uint32_t*>(b.aux_off)[m] = aoff;
  const_cast<uint32_t*>(b.aux_len)[m] = alen;
  w.msg_status[m] = st;
  if (kind == 0) w.D[m] = 0;
}
void launch_parse(const DevState& s, const Work& w, const BatchIn& b, cudaStream_t st) {
  cudaMemsetAsync(w.msg_status, 0, b.n_msgs, st);
  PCDN_COUNT_LAUNCH, k_parse<<<(b.n_msgs + 255) / 256, 256, 0, st>>>(s, b, w);
}

// =============================================================================== K3 direct lookup
__device__ __forceinline__ uint32_t key_word32(const uint8_t* kp, uint32_t j, uint32_t klen) {
  uint32_t o = j * 4;
  if (o >= klen) return 0;
  uint32_t w = *reinterpret_cast<const uint32_t*>(kp + o);  // kp is 4-byte aligned (engine contract)
  uint32_t rem = klen - o;
  if (rem < 4) w &= (1u << (8 * rem)) - 1u;
  return w;
}

// Eight lanes per message, four messages per warp (4x the memory-level parallelism of a warp per
// message: the kernel is a chain of three dependent DRAM accesses — key, buckets, stored key).
// Direct messages: hash the recipient key (64-bit words strided over the 8 lanes, xor-shuffle
// reduced inside the group), probe both 4-slot buckets with the 8 lanes, verify the full key
// against the key arena, resolve the route (handler.rs:204-236).  Also seeds the (conn, msg) sort.
// (gtid = global thread index: 8 consecutive threads serve message gtid / 8)
template <bool COUNT>
__device__ __forceinline__ void direct_lookup_body(const DevState& s, const BatchIn& b, const Work& w, uint32_t gtid) {
  const uint32_t lane = lane_id(), grp = lane >> 3, gl = lane & 7;
  const uint32_t m = (gtid >> 5) * 4 + grp;
  const bool valid = m < b.n_msgs;
  const bool is_direct = valid && b.kind[m] == 3;
  const uint32_t gshift = grp * 8;
  uint32_t target = kConnNone;
  const uint32_t klen = is_direct ? b.aux_len[m] : 0;
  const uint8_t* kp = b.arena + (is_direct ? b.aux_off[m] : 0);
  // hash
  const uint32_t nw = (klen + 7) >> 3;
  uint64_t acc = 0;
  for (uint32_t i = gl; i < nw; i += 8) {
    uint64_t wd = (uint64_t)key_word32(kp, 2 * i, klen) | ((uint64_t)key_word32(kp, 2 * i + 1, klen) << 32);
    acc += key_word_mix(wd, i, s.seed);
  }
#pragma unroll
  for (int o = 4; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  const uint64_t h = key_hash_finish(acc, klen);
  const uint32_t tag = key_tag(h), b1 = key_bucket(h, s.bucket_mask), b2 = alt_bucket(b1, tag, s.bucket_mask);
  CuckooEntry e{0, 0, ROUTE_NONE, 0};
  if (is_direct) {
    const uint4 raw = *reinterpret_cast<const uint4*>(&s.cuckoo[(size_t)(gl < 4 ? b1 : b2) * 4 + (gl & 3)]);
    e.tag = raw.x; e.key_slot = raw.y; e.route = raw.z; e.key_len = raw.w;
  }
  bool cand = is_direct && e.tag == tag && e.key_len == klen;
  if (b1 == b2 && gl >= 4) cand = false;
  uint32_t gmask = (__ballot_sync(0xffffffffu, cand) >> gshift) & 0xFFu;  // this group's candidates
  uint32_t route = ROUTE_NONE;
  const uint32_t nw32 = (klen + 3) >> 2;
  while (__any_sync(0xffffffffu, gmask != 0)) {  // groups advance through their own candidates in lockstep
    const bool active = gmask != 0;
    const int src = active ? (int)(gshift + __ffs(gmask) - 1) : (int)lane;
    if (active) gmask &= gmask - 1;
    const uint32_t kslot = __shfl_sync(0xffffffffu, e.key_slot, src);
    const uint32_t rt = __shfl_sync(0xffffffffu, e.route, src);
    bool eq = true;
    if (active) {
      const uint32_t* ak = reinterpret_cast<const uint32_t*>(s.keys + (size_t)kslot * s.key_stride);
      for (uint32_t i = gl; i < nw32; i += 8) eq = eq && (ak[i] == key_word32(kp, i, klen));
    }
    const bool all_eq = ((__ballot_sync(0xffffffffu, eq) >> gshift) & 0xFFu) == 0xFFu;
    if (active && all_eq) { route = rt; gmask = 0; }
  }
  if (route != ROUTE_NONE) {
    if (route & ROUTE_REMOTE) {
      // owner is another broker: forward unless the message came from a broker (to_user_only)
      if (!(b.flags[m] & 1)) target = s.owner_conn[route & ~ROUTE_REMOTE];
    } else {
      target = route;
    }
  }
  // `target` is a global connection id: count the unroutable message on one shard only, then keep
  // the message only if the target's ring lives on this shard
  const bool dropped = target == kConnNone;
  if (!dropped) { target -= s.conn_base; if (target >= s.N) target = kConnNone; }  // (unsigned wrap: below the base → NONE)
  if (valid && gl == 0) {
    w.dconn[m] = target;
    w.edir[m] = make_uint2(kConnNone, kOffInvalid);  // k_offsets fills in the ring offset of a delivered message
    if (is_direct) {
      w.D[m] = 0;  // direct messages never enter the broadcast classes' scatter lists
      if (dropped && s.count_drops) atomicAdd(&w.stats->n_direct_dropped, 1u);
      if (COUNT && target != kConnNone) atomicAdd(&w.dcount[target], 1u);
    }
  }
}
__global__ void __launch_bounds__(256) k_direct_lookup(DevState s, BatchIn b, Work w) {
  direct_lookup_body<true>(s, b, w, blockIdx.x * blockDim.x + threadIdx.x);
}

// ---- hits per connection → segments of dlist (no sort) ------------------------------------------
// start of connection c's segment of dlist (c may be N: the end of the last segment)
__device__ __forceinline__ uint32_t dseg_start(const Work& w, uint32_t c) { return w.dloc[c] + w.dtile[c >> 10]; }

// One launch: every CTA scans a tile of 1024 counts (exclusive, tile-local → dloc) and publishes the
// tile total; the CTA that finishes last turns the totals into tile bases in place (dtile).  Readers
// add the two (dseg_start).  Connections with more than kHotMin hits are listed for k_dsort_hot.
__global__ void __launch_bounds__(256) k_dscan(Work w, uint32_t n, uint32_t ntiles) {
  __shared__ uint32_t sm[9];
  __shared__ uint32_t is_last;
  const uint32_t base = blockIdx.x * 1024 + threadIdx.x * 4;
  uint32_t v[4], sum = 0;
#pragma unroll
  for (int k = 0; k < 4; k++) {
    v[k] = (base + k < n) ? w.dcount[base + k] : 0;
    sum += v[k];
    if (v[k] > kHotMin) w.hot_list[atomicAdd(&w.stats->n_hot, 1u)] = base + k;
  }
  uint32_t tot, ex = block256_excl_scan(sum, &tot, sm);
#pragma unroll
  for (int k = 0; k < 4; k++) { if (base + k < n) w.dloc[base + k] = ex; ex += v[k]; }
  if (threadIdx.x == 0) {
    w.dtile[blockIdx.x] = tot;
    __threadfence();
    is_last = atomicAdd(w.scan_done, 1u) == ntiles - 1 ? 1u : 0u;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  uint32_t carry = 0;
  for (uint32_t bb = 0; bb < ntiles; bb += 256) {
    const uint32_t i = bb + threadIdx.x;
    const uint32_t t = i < ntiles ? __ldcg(w.dtile + i) : 0;
    uint32_t tt, e2 = block256_excl_scan(t, &tt, sm);
    if (i < ntiles) w.dtile[i] = carry + e2;
    carry += tt;
  }
  if (threadIdx.x == 0) { w.dtile[ntiles] = carry; *w.scan_done = 0; }
}

// every delivered direct message drops its index into its connection's segment (arbitrary slot)
__global__ void __launch_bounds__(256) k_dfill(BatchIn b, Work w) {
  const uint32_t m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= b.n_msgs) return;
  const uint32_t t = w.dconn[m];
  if (t == kConnNone) return;
  const uint32_t slot = atomicSub(&w.dcount[t], 1u) - 1u;
  w.dlist[dseg_start(w, t) + slot] = m;
}

// Hot connections (votes to a leader: thousands of directs to ONE key in a batch): the segment's
// entries are distinct message indices below n_msgs, so "sorting" them is marking a bitmap of n_msgs
// bits and reading the set bits back in order — O(n_msgs / 32) per hot connection whatever its
// hit count.  One CTA per hot connection (grid-stride), its own bitmap row.
__global__ void __launch_bounds__(256) k_dsort_hot(BatchIn b, Work w, uint32_t words) {
  __shared__ uint32_t sm[9];
  const uint32_t nh = w.stats->n_hot;
  uint32_t* bm = w.hot_bitmap + (size_t)blockIdx.x * words;
  for (uint32_t h = blockIdx.x; h < nh; h += gridDim.x) {
    const uint32_t c = w.hot_list[h];
    const uint32_t s0 = dseg_start(w, c), e0 = dseg_start(w, c + 1);
    for (uint32_t i = threadIdx.x; i < words; i += 256) bm[i] = 0;
    __syncthreads();
    for (uint32_t i = s0 + threadIdx.x; i < e0; i += 256) {
      const uint32_t m = w.dlist[i];
      atomicOr(&bm[m >> 5], 1u << (m & 31));
    }
    __syncthreads();
    uint32_t carry = 0;
    for (uint32_t w0 = 0; w0 < words; w0 += 256) {
      uint32_t word = (w0 + threadIdx.x < words) ? bm[w0 + threadIdx.x] : 0;
      uint32_t tot, ex = block256_excl_scan(__popc(word), &tot, sm);
      uint32_t pos = s0 + carry + ex;
      while (word) {
        const uint32_t bit = __ffs(word) - 1;
        word &= word - 1;
        w.dlist[pos++] = (w0 + threadIdx.x) * 32 + bit;
      }
      carry += tot;
    }
    __syncthreads();
  }
}

void launch_direct(const DevState& s, const Work& w, const BatchIn& b, uint32_t n_direct, cudaStream_t st) {
  const uint32_t n = b.n_msgs;
  const uint32_t nseg = s.N + 1, ntiles = (nseg + 1023) / 1024;
  cudaMemsetAsync(w.dcount, 0, (size_t)(s.N + 2) * 4, st);
  PCDN_COUNT_LAUNCH, k_direct_lookup<<<(n * 8 + 255) / 256, 256, 0, st>>>(s, b, w);
  PCDN_COUNT_LAUNCH, k_dscan<<<ntiles, 256, 0, st>>>(w, nseg, ntiles);
  PCDN_COUNT_LAUNCH, k_dfill<<<(n + 255) / 256, 256, 0, st>>>(b, w);
  if (n_direct > kHotMin) PCDN_COUNT_LAUNCH, k_dsort_hot<<<kHotCtas, 256, 0, st>>>(b, w, (n + 31) / 32);
}

// =============================================================================== K1a topic match
// ---- in-batch subscription events (PCDN_FLAG_INBATCH_SUBSCRIBE).  The bitmap holds every connection's
// membership as it was when the batch was opened; a connection with events gets its bit of message m
// re-evaluated: per topic of m, its membership before the batch with its events at positions <= m
// replayed in order, ORed over the topics.  The match patches its words before the popcounts, so ranks,
// plan, offsets and pack see the patched bits like any other.

// every bitmap row message m names (fl, toff, tn: m's flags, aux_off, aux_len), in list order: the wire u8 list
// read in place with Topic::prune applied (device-parse mode), or the host's u16 list; a topic naming no row is
// skipped.  f(t) returns true to stop the walk.
template <class F>
__device__ __forceinline__ void for_each_topic(const DevState& s, const BatchIn& b, uint32_t fl, uint32_t toff, uint32_t tn, F&& f) {
  if (fl & MSGF_TOPICS_U8) {
    const uint8_t* tb = b.arena + toff;
    for (uint32_t i = 0; i < tn; i++) {
      if ((fl & MSGF_PRUNE) && !topic_kept(tb, i, s.n_valid_topics)) continue;
      const uint32_t t = tb[i];
      if (t < s.T && f(t)) return;
    }
  } else {
    for (uint32_t i = 0; i < tn; i++) {
      const uint32_t t = b.topics[toff + i];
      if (t < s.T && f(t)) return;
    }
  }
}

// bit k of local word wd for message m, with the connection's events [e0, e1) (its events at positions <= m)
__device__ uint32_t event_bit(const DevState& s, const BatchIn& b, uint32_t m, uint32_t wd, uint32_t k, uint32_t e0, uint32_t e1) {
  uint32_t bit = 0;
  for_each_topic(s, b, b.flags[m], b.aux_off[m], b.aux_len[m], [&](uint32_t t) {
    uint32_t on = (s.sub[(size_t)t * s.W + wd] >> k) & 1u;
    for (uint32_t e = e0; e < e1; e++) {
      const SubEvent ev = b.events[e];
      for (uint32_t q = 0; q < ev.tn; q++)
        if (b.ev_topics[ev.toff + q] == t) { on = ev.pos_op >> 31; break; }
    }
    bit = on;
    return on != 0;
  });
  return bit;
}

// patch NW consecutive match words v[] of message m, the first at local word wd0: one binary search for
// the first event of these 32 * NW connections, then the events of those connections only
template <int NW>
__device__ __forceinline__ void apply_events(const DevState& s, const BatchIn& b, uint32_t m, uint32_t wd0, uint32_t* v) {
  const uint32_t ne = b.n_events, c_lo = s.conn_base + wd0 * 32, c_hi = c_lo + NW * 32;
  uint32_t e = 0, hi = ne;
  while (e < hi) {
    const uint32_t mid = (e + hi) >> 1;
    if (b.events[mid].conn < c_lo) e = mid + 1; else hi = mid;
  }
  while (e < ne) {
    const uint32_t c = b.events[e].conn;
    if (c >= c_hi) break;
    uint32_t e1 = e;   // c's events at positions <= m
    while (e1 < ne && b.events[e1].conn == c && (b.events[e1].pos_op & ~kEvSubscribe) <= m) e1++;
    if (e1 > e) {
      const uint32_t q = (c - c_lo) >> 5, k = c & 31u;   // (c_lo is a multiple of 32)
      const uint32_t bit = event_bit(s, b, m, wd0 + q, k, e, e1);
#pragma unroll
      for (int x = 0; x < NW; x++)
        if ((uint32_t)x == q) v[x] = (v[x] & ~(1u << k)) | (bit << k);
    }
    while (e1 < ne && b.events[e1].conn == c) e1++;   // c's later events
    e = e1;
  }
}

// the batch's first kernel zeroes its counters (zero: null when a memset or an earlier kernel did); nothing else
// in that kernel's first CTA touches them before its next barrier
__device__ __forceinline__ void zero_stats(BatchStats* zero, bool first_cta) {
  if (zero && first_cta && threadIdx.x < sizeof(BatchStats) / 4) reinterpret_cast<uint32_t*>(zero)[threadIdx.x] = 0;
}
// copy of the final counters into the mapped host block: fenced after publish_if_last's count of finished CTAs, not
// after k_ctrl_small's cluster barrier (~0.8 us of its 15 us one-broadcast batch on an H100 80GB HBM3 at 700 W)
__device__ __forceinline__ void publish_stats(const Work& w, BatchStats* publish, bool fenced) {
  if (threadIdx.x < sizeof(BatchStats) / 4) {
    if (fenced) __threadfence();
    reinterpret_cast<uint32_t*>(publish)[threadIdx.x] = __ldcg(reinterpret_cast<const uint32_t*>(w.stats) + threadIdx.x);
    if (fenced) __threadfence_system();
  }
}

// Warp = one 256-word match block `blk` of broadcast j, lane = 8 consecutive words (32-byte vector
// loads of the bitmap rows, no block-level synchronisation: the popcount prefix of a 256-word block
// is a lane-local prefix plus one warp scan).  Run by k_match and by the fused small-engine kernel.
// (EVENTS: the batch holds in-batch subscription events; TARGET: it holds a MSGF_TARGET message, and only
//  that instantiation reads the flag)
template <bool EVENTS, bool TARGET>
__device__ __forceinline__ void match_block(const DevState& s, const BatchIn& b, const Work& w, uint32_t j, uint32_t blk) {
  const uint32_t lane = lane_id();
  const uint32_t m = b.bcast_index[j];
  const uint32_t w0 = blk * kBlockWords + lane * 8;
  const uint32_t toff = b.aux_off[m], fl = b.flags[m];
  uint4 lo = make_uint4(0, 0, 0, 0), hi = make_uint4(0, 0, 0, 0);
  for_each_topic(s, b, fl, toff, b.aux_len[m], [&](uint32_t t) {   // OR of the topics' bitmap rows
    const uint4* row = reinterpret_cast<const uint4*>(s.sub + (size_t)t * s.W + w0);
    const uint4 a = row[0], c = row[1];
    lo.x |= a.x; lo.y |= a.y; lo.z |= a.z; lo.w |= a.w;
    hi.x |= c.x; hi.y |= c.y; hi.z |= c.z; hi.w |= c.w;
    return false;
  });
  if (EVENTS && !(TARGET && (fl & MSGF_TARGET))) {
    uint32_t v[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
    apply_events<8>(s, b, m, w0, v);
    lo = make_uint4(v[0], v[1], v[2], v[3]); hi = make_uint4(v[4], v[5], v[6], v[7]);
  }
  if (fl & MSGF_USERS_ONLY) {  // to_users_only (connections/mod.rs:111)
    const uint4* br = reinterpret_cast<const uint4*>(s.brk + w0);
    const uint4 a = br[0], c = br[1];
    lo.x &= ~a.x; lo.y &= ~a.y; lo.z &= ~a.z; lo.w &= ~a.w;
    hi.x &= ~c.x; hi.y &= ~c.y; hi.z &= ~c.z; hi.w &= ~c.w;
  }
  // pcdn_send_to_broker(s): the row is the shard's broker mask for "every peer broker", else the bit of the one
  // target connection (none when it lies outside this shard's slice).  No topic rows, in-batch events or
  // to_users_only: the recipients are the brokers connected when it was sent.  A MSGF_TARGET message lists no
  // topic and is never to_users_only, so lo / hi are still zero here.
  if (TARGET && (fl & MSGF_TARGET)) {
    if (toff == kConnNone) {
      const uint4* br = reinterpret_cast<const uint4*>(s.brk + w0);
      lo = br[0]; hi = br[1];
    } else {
      const uint32_t local = toff - s.conn_base, bit = 1u << (local & 31u);
      const uint32_t q = local < s.N ? (local >> 5) - w0 : 8u;   // (unsigned: a word before w0 is >= 8 too)
      lo = make_uint4(q == 0 ? bit : 0u, q == 1 ? bit : 0u, q == 2 ? bit : 0u, q == 3 ? bit : 0u);
      hi = make_uint4(q == 4 ? bit : 0u, q == 5 ? bit : 0u, q == 6 ? bit : 0u, q == 7 ? bit : 0u);
    }
  }
  const uint32_t p0 = __popc(lo.x), p1 = p0 + __popc(lo.y), p2 = p1 + __popc(lo.z), p3 = p2 + __popc(lo.w);
  const uint32_t p4 = p3 + __popc(hi.x), p5 = p4 + __popc(hi.y), p6 = p5 + __popc(hi.z), p7 = p6 + __popc(hi.w);
  const uint32_t incl = warp_incl_scan(p7), ex = incl - p7;  // exclusive prefix over the lanes before this one
  // The warp that finishes a message last turns its block counts into exclusive bases and D_m
  // (no second launch).  `done[j]` counts finished blocks and is left at zero for the next batch.
  // (count published BEFORE the wide stores below, so the fence only has one store to wait for)
  uint32_t last = 0;
  if (lane == 31) {
    w.cnt[(size_t)j * s.nblk + blk] = incl;
    __threadfence();
    last = atomicAdd(&w.done[j], 1u) == s.nblk - 1 ? 1u : 0u;
  }
  uint4* Bo = reinterpret_cast<uint4*>(w.B + (size_t)j * s.W + w0);
  Bo[0] = lo; Bo[1] = hi;
  uint4 pre;  // eight u16 prefixes (a 256-word block holds at most 8192 recipients)
  pre.x = ex | ((ex + p0) << 16); pre.y = (ex + p1) | ((ex + p2) << 16);
  pre.z = (ex + p3) | ((ex + p4) << 16); pre.w = (ex + p5) | ((ex + p6) << 16);
  *reinterpret_cast<uint4*>(w.wpre + (size_t)j * s.W + w0) = pre;
  if (__shfl_sync(0xffffffffu, last, 31)) {
    __threadfence();
    uint32_t carry = 0;
    for (uint32_t bb = 0; bb < s.nblk; bb += 32) {
      const uint32_t i = bb + lane;
      const uint32_t v = i < s.nblk ? __ldcg(w.cnt + (size_t)j * s.nblk + i) : 0;
      const uint32_t in = warp_incl_scan(v);
      if (i < s.nblk) w.base[(size_t)j * s.nblk + i] = carry + in - v;
      carry += __shfl_sync(0xffffffffu, in, 31);
    }
    if (lane == 0) { w.D[m] = carry; w.jidx[m] = j; w.done[j] = 0; }
  }
}
// grid = (ceil(nblk / 8), n_bcast); zero: see zero_stats (the batch's first kernel when it has no direct message
// and no device parse)
template <bool EVENTS, bool TARGET>
__global__ void __launch_bounds__(256) k_match(DevState s, BatchIn b, Work w, BatchStats* zero) {
  zero_stats(zero, blockIdx.x == 0 && blockIdx.y == 0);
  const uint32_t blk = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (blk < s.nblk) match_block<EVENTS, TARGET>(s, b, w, blockIdx.y, blk);  // warp-uniform
}
void launch_match(const DevState& s, const Work& w, const BatchIn& b, BatchStats* zero, bool targeted, cudaStream_t st) {
  if (!b.n_bcast) return;
  dim3 grid((s.nblk + 7) / 8, b.n_bcast);
  // (a batch with in-batch subscription events, or with a targeted message, takes its own instantiation: the
  //  one without them keeps the registers and occupancy it has without the patch or the target rows)
  if (targeted) {
    if (b.n_events) PCDN_COUNT_LAUNCH, k_match<true, true><<<grid, 256, 0, st>>>(s, b, w, zero);
    else PCDN_COUNT_LAUNCH, k_match<false, true><<<grid, 256, 0, st>>>(s, b, w, zero);
  } else {
    if (b.n_events) PCDN_COUNT_LAUNCH, k_match<true, false><<<grid, 256, 0, st>>>(s, b, w, zero);
    else PCDN_COUNT_LAUNCH, k_match<false, false><<<grid, 256, 0, st>>>(s, b, w, zero);
  }
}

// =============================================================================== K1p plan
__device__ __forceinline__ uint32_t frame_vec_bytes(uint32_t raw_len) { return (4u + raw_len + 15u) & ~15u; }
__device__ __forceinline__ uint32_t frame_units(uint32_t raw_len) { return (4u + raw_len + kUnit - 1u) / kUnit; }
// The one delivery rule: a message is delivered by reference (one 32-byte record, k_pack_ref) when its raw
// length reaches DevState::ref_min, else as a framed copy.  Shared payload: always; copy mode: never.
__device__ __forceinline__ bool by_ref(const DevState& s, uint32_t raw_len) { return raw_len >= s.ref_min; }
// units one delivery takes in a ring / the output pool: the framed copy, or one 32-byte reference record.
// Every placement site (k_offsets, its direct path, k_ctrl_small) uses it.
__device__ __forceinline__ uint32_t rec_units(const DevState& s, uint32_t raw_len) {
  return by_ref(s, raw_len) ? 1u : frame_units(raw_len);
}
// recipients per message-major tile: about kFatTileBytes of stores per tile whatever the frame size, so a
// batch of large frames still splits into enough tiles to balance ~450 persistent CTAs
__device__ __forceinline__ uint32_t tile_recipients(uint32_t frame_bytes) {
  const uint32_t chunk = min(frame_bytes, kChunkBytes);
  return max(32u, min(kTileRecipients, kFatTileBytes / chunk));
}

// pack class of a message with d recipients, and its number of message-major tiles
__device__ __forceinline__ void plan_classify(const DevState& s, const BatchIn& b, uint32_t m, uint32_t d, uint32_t* cls_out,
                                              uint32_t* tiles_out) {
  uint32_t cls = CLS_THIN, tiles = 0;
  if (d >= kFatMin) {
    const uint32_t len = b.raw_len[m];
    // (by reference: every delivery is one 32-byte record with an explicit {conn, off} entry in efat, written by
    //  k_pack_ref.  The connection-major class and the message-major tiles stage frame copies: neither applies.)
    const bool ref = by_ref(s, len);
    const bool dense = !ref && ((uint64_t)d << kCmDenseShift) >= s.N && b.kind[m] == 4;
    if (dense && frame_units(len) * kUnit <= kCmMaxBytes) {
      cls = CLS_CM;
    } else {
      cls = CLS_FAT;
      const uint32_t nch = (frame_vec_bytes(len) + kChunkBytes - 1) / kChunkBytes;
      const uint32_t tr = tile_recipients(frame_vec_bytes(len));
      tiles = ref ? 0u : nch * ((d + tr - 1) / tr);
    }
  }
  *cls_out = cls; *tiles_out = tiles;
}

// Thread per message m of CTA vb of nvb (NW warps each): class, tiles, and the four CTA-local exclusive scans —
// fat entries, thin entries, tiles, connection-major rank — stored per message; thread 0 stores the CTA's totals
// into scan_tmp.  Returns m's connection-major rank; *cm: m is connection-major.
template <int NW>
__device__ __forceinline__ uint32_t plan_messages(const DevState& s, const BatchIn& b, const Work& w, uint32_t m, uint32_t vb,
                                                  uint32_t nvb, uint32_t* sm, bool* cm) {
  const bool valid = m < b.n_msgs;
  const uint32_t d = valid ? w.D[m] : 0;
  uint32_t cls, tiles;
  plan_classify(s, b, m, d, &cls, &tiles);
  uint32_t tot;
  uint32_t e0 = cta_excl_scan<NW>(cls != CLS_THIN ? d : 0, &tot, sm);
  if (threadIdx.x == 0) w.scan_tmp[vb] = tot;
  uint32_t e1 = cta_excl_scan<NW>(cls == CLS_THIN ? d : 0, &tot, sm);
  if (threadIdx.x == 0) w.scan_tmp[nvb + vb] = tot;
  uint32_t e2 = cta_excl_scan<NW>(tiles, &tot, sm);
  if (threadIdx.x == 0) w.scan_tmp[2 * nvb + vb] = tot;
  uint32_t e3 = cta_excl_scan<NW>(cls == CLS_CM ? 1u : 0u, &tot, sm);
  if (threadIdx.x == 0) w.scan_tmp[3 * nvb + vb] = tot;
  if (valid) { w.eb_fat[m] = e0; w.eb_thin[m] = e1; w.tbase[m] = e2; w.cm_rank[m] = e3; w.cls[m] = (uint8_t)cls; }
  *cm = valid && cls == CLS_CM;
  return e3;
}
// Whole batch in one CTA (<= 256 messages): its scans are already global, so the plan ends here — cm_list,
// the totals and cursors, the PCDN_E2BIG check and the [n] sentinels (what k_plan_b / k_plan_c do otherwise)
__device__ __forceinline__ void plan_finish(const BatchIn& b, const Work& w, uint32_t m, bool cm, uint32_t cm_rank) {
  if (cm) w.cm_list[cm_rank] = m;
  if (threadIdx.x == 0) {
    const uint32_t t0 = w.scan_tmp[0], t1 = w.scan_tmp[1], t2 = w.scan_tmp[2], t3 = w.scan_tmp[3];
    w.stats->n_fat_entries = t0; w.stats->n_thin_entries = t1; w.stats->n_fat_tiles = t2; w.stats->tile_cursor = 0;
    w.stats->n_cm = t3; w.stats->cm_cursor = 0;
    if (t0 > w.cap_fat || t1 > w.cap_thin) w.stats->status = 1;  // PCDN_E2BIG
    const uint32_t n = b.n_msgs;
    w.eb_fat[n] = t0; w.eb_thin[n] = t1; w.tbase[n] = t2; w.cm_rank[n] = t3;
  }
}

__global__ void __launch_bounds__(256) k_plan_a(DevState s, BatchIn b, Work w, uint32_t nblk) {
  __shared__ uint32_t sm[9];
  const uint32_t m = blockIdx.x * 256 + threadIdx.x;
  bool cm;
  const uint32_t r = plan_messages<8>(s, b, w, m, blockIdx.x, nblk, sm, &cm);
  // (one block: saves the k_plan_b / k_plan_c launches on the latency-critical small-batch path)
  if (gridDim.x == 1) plan_finish(b, w, m, cm, r);
}
// grid = 4: block q scans the block totals of one of the four planned quantities
__global__ void __launch_bounds__(256) k_plan_b(Work w, uint32_t nblk) {
  __shared__ uint32_t sm[9];
  const uint32_t q = blockIdx.x;
  uint32_t* t = w.scan_tmp + (size_t)q * nblk;
  uint32_t carry = 0;
  for (uint32_t bb = 0; bb < nblk; bb += 256) {
    const uint32_t i = bb + threadIdx.x;
    const uint32_t v = i < nblk ? t[i] : 0;
    uint32_t tot, ex = block256_excl_scan(v, &tot, sm);
    if (i < nblk) t[i] = ex + carry;
    carry += tot;
  }
  if (threadIdx.x == 0) {
    if (q == 0) { w.stats->n_fat_entries = carry; if (carry > w.cap_fat) w.stats->status = 1; }   // PCDN_E2BIG
    if (q == 1) { w.stats->n_thin_entries = carry; if (carry > w.cap_thin) w.stats->status = 1; }
    if (q == 2) { w.stats->n_fat_tiles = carry; w.stats->tile_cursor = 0; }
    if (q == 3) { w.stats->n_cm = carry; w.stats->cm_cursor = 0; }
  }
}
__global__ void __launch_bounds__(256) k_plan_c(BatchIn b, Work w, uint32_t nblk) {
  const uint32_t m = blockIdx.x * 256 + threadIdx.x;
  if (m < b.n_msgs) {
    w.eb_fat[m] += w.scan_tmp[blockIdx.x];
    w.eb_thin[m] += w.scan_tmp[nblk + blockIdx.x];
    w.tbase[m] += w.scan_tmp[2 * nblk + blockIdx.x];
    const uint32_t r = w.cm_rank[m] + w.scan_tmp[3 * nblk + blockIdx.x];
    w.cm_rank[m] = r;
    if (w.cls[m] == CLS_CM) w.cm_list[r] = m;
  } else if (m == b.n_msgs) {
    w.eb_fat[m] = w.stats->n_fat_entries;
    w.eb_thin[m] = w.stats->n_thin_entries;
    w.tbase[m] = w.stats->n_fat_tiles;
    w.cm_rank[m] = w.stats->n_cm;
  }
}
void launch_plan(const DevState& s, const Work& w, const BatchIn& b, cudaStream_t st) {
  // Direct messages need no plan: message m owns entry m of the direct list (edir).  A batch without
  // broadcasts has nothing to classify (the batch counters were zeroed at batch begin).
  if (b.n_bcast == 0) return;
  const uint32_t nblk = (b.n_msgs + 255) / 256;
  PCDN_COUNT_LAUNCH, k_plan_a<<<nblk, 256, 0, st>>>(s, b, w, nblk);
  if (nblk == 1) return;  // finished inside k_plan_a
  PCDN_COUNT_LAUNCH, k_plan_b<<<4, 256, 0, st>>>(w, nblk);
  PCDN_COUNT_LAUNCH, k_plan_c<<<(b.n_msgs + 1 + 255) / 256, 256, 0, st>>>(b, w, nblk);
}

// =============================================================================== K1b offsets
struct ConnCursor {
  uint32_t pt, us, bu;          // ring tail, units in use, units consumed by this batch
  uint32_t s1_off, s1_units, s1_rec, s2_units, s2_rec;
  uint32_t ovf, in2;
  uint32_t bytes;  // 4 + len summed over this batch's records: < ring bytes < 2^32
};
// reserve `u` units for one record; records never straddle the ring end
__device__ __forceinline__ uint32_t alloc_record(ConnCursor& k, uint32_t u, uint32_t R, uint32_t raw_len) {
  if (k.ovf) return kOffInvalid;
  const bool wrap = k.pt + u > R;
  // a drained ring (nothing in use) wraps for free: the space before its tail is free as well, so any
  // record of at most R units fits it (us == 0 also means no record of this batch is placed yet)
  const uint32_t pad = (wrap && k.us) ? R - k.pt : 0, at = wrap ? 0 : k.pt;
  if (u > R || k.us + pad + u > R) { k.ovf = 1; return kOffInvalid; }
  k.us += pad + u;
  k.bu += pad + u;
  if (wrap && k.s1_rec) k.in2 = 1;
  if (!k.in2) { if (!k.s1_rec) k.s1_off = at; k.s1_units += u; k.s1_rec++; }
  else { k.s2_units += u; k.s2_rec++; }
  k.pt = at + u;
  k.bytes += 4u + raw_len;
  return at;
}

// Thread per connection.  Walks the batch in order (broadcast matches from the match words, direct
// hits from the connection's sorted bucket), so a connection's records are laid out in batch order
// (R9) with no atomics, and writes each (conn, offset) into the per-message scatter list at its
// deterministic rank (block base + word prefix + lane rank).
// (body shared by k_offsets — 256-thread CTAs, any N — and the fused small-engine control kernel —
//  eight 1024-thread CTAs of one cluster, N = 8192; NT = threads per CTA, c = this thread's connection)
// Pool mode (DevState::pool): the CTAs of the offsets pass chain their unit totals in connection order
// with a decoupled look-back (one 64-bit word per CTA: batch stamp | flag | value, so nothing is
// cleared between batches).  Called by warp 0 of the CTA; returns the units of all CTAs before `vb`.
__device__ __forceinline__ uint32_t pool_lookback(const Work& w, uint32_t vb, uint32_t ctot) {
  const uint32_t lane = lane_id();
  volatile unsigned long long* st = w.lb_state;
  const unsigned long long tag = (unsigned long long)w.stamp << 34;
  auto pack = [&](uint32_t flag, uint32_t v) { return tag | ((unsigned long long)flag << 32) | v; };
  unsigned long long prefix64 = 0;
  if (vb > 0) {
    if (lane == 0) st[vb] = pack(1u, ctot);  // AGGREGATE: this CTA's own total
    int j = (int)vb - 1;
    for (;;) {
      const int idx = j - (int)lane;
      unsigned long long x = 0;
      if (idx >= 0) { do { x = st[idx]; } while ((x >> 34) != (tag >> 34)); }   // wait until that CTA has published this batch
      const uint32_t flag = idx >= 0 ? (uint32_t)(x >> 32) & 3u : 2u;             // before CTA 0: inclusive prefix 0
      const uint32_t val = idx >= 0 ? (uint32_t)x : 0u;
      const uint32_t pm = __ballot_sync(0xffffffffu, flag == 2u);
      const int first = pm ? __ffs(pm) - 1 : 32;                                  // nearest predecessor with an inclusive prefix
      const uint32_t v = (int)lane <= first ? val : 0u;
      // (32 values of up to 2^32 - 1: summed in two halves; a batch of more than 2^32 units saturates,
      //  which pool_allocate turns into "larger than the pool")
      const unsigned long long take = ((unsigned long long)__reduce_add_sync(0xffffffffu, v >> 16) << 16) + __reduce_add_sync(0xffffffffu, v & 0xFFFFu);
      prefix64 += take;
      if (pm) break;
      j -= 32;
    }
  }
  const uint32_t prefix = (uint32_t)(prefix64 > 0xFFFFFFFFull ? 0xFFFFFFFFull : prefix64);
  const unsigned long long incl = prefix64 + ctot;
  if (lane == 0) { __threadfence(); st[vb] = pack(2u, incl > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)incl); }  // PREFIX: inclusive
  return prefix;
}
// the CTA that holds the last connections knows the batch total: it takes the region out of the pool
__device__ __forceinline__ void pool_allocate(const DevState& s, const Work& w, unsigned long long total64) {
  PoolState* p = s.pool_state;
  BatchStats* bs = w.stats;
  if (w.pool_unblock) p->blocked = 0;
  if (total64 > s.pool_units) { bs->status = 3; return; }   // larger than the whole pool: can never fit (E2BIG)
  const uint32_t total = (uint32_t)total64;
  if (p->blocked) { bs->status = 2; return; }                // an older batch is waiting for space: keep the order
  if (p->used == 0) { p->head = 0; p->tail = 0; }
  uint32_t base = p->head, skip = 0;
  bool ok;
  if (p->head >= p->tail) {      // free: [head, cap) and [0, tail)
    if ((unsigned long long)p->head + total <= s.pool_units) ok = true;
    else if (total <= p->tail && p->used) { skip = s.pool_units - p->head; base = 0; ok = true; }
    else ok = false;
    if (p->used && p->head == p->tail) ok = false;   // completely full
  } else {
    ok = p->head + total <= p->tail;
  }
  if (!ok) { bs->status = 2; p->blocked = 1; return; }
  p->head = base + total;
  p->used += total + skip;
  bs->pool_base = base; bs->pool_units = total; bs->pool_skip = skip;
}

// FUSED: run by the fused small-engine kernel.  Its direct segments are rank-sorted with sparse bounds (valid
// iff stamped), and in pool mode its CTAs chain their unit totals with a look-back (they are co-resident, the
// chain is at most 64 long).  The regular kernel's CTAs instead keep CTA-local offsets and put the CTA total
// in lb_tot[], finished by k_pool_finish (one more launch instead of 4096 CTAs polling each other is slower
// at 2^20 connections).
template <bool HAS_DIRECT, int NT, bool FUSED>
__device__ __forceinline__ void offsets_body(const DevState& s, const BatchIn& b, const Work& w, uint32_t max_conns,
                                             uint32_t c, uint32_t vb, uint32_t nvb) {
  constexpr int NW = NT / 32;
  __shared__ uint32_t sm[NW + 1];
  __shared__ unsigned long long red[2][NW];
  __shared__ uint32_t span_base;
  if (w.stats->status) return;  // batch rejected (E2BIG): leave all cursors untouched (uniform over the grid)
  const uint32_t wd = c >> 5, lane = c & 31, lt = (1u << lane) - 1u;
  const uint32_t R = s.pool ? 0x7FFFFFFFu : s.ring_units;   // pool mode: a connection's region just grows
  ConnCursor k;
  k.pt = s.pool ? 0u : s.ptail[c]; k.us = s.pool ? 0u : s.used[c]; k.bu = 0;
  k.s1_off = 0; k.s1_units = 0; k.s1_rec = 0; k.s2_units = 0; k.s2_rec = 0; k.ovf = 0; k.in2 = 0; k.bytes = 0;
  uint32_t dp = 0, de = 0;
  if (HAS_DIRECT) {
    if (FUSED) {
      if (w.dstamp[c] == w.stamp) { dp = w.dstart[c]; de = w.dend[c]; }
    } else {
      dp = dseg_start(w, c); de = dseg_start(w, c + 1);
      // The fill pass left this connection's few hits in arbitrary order: put them into batch order
      // (R9) here, in place — the segment belongs to this thread alone.  Segments of more than
      // kHotMin entries were ordered by k_dsort_hot.
      if (de - dp >= 2 && de - dp <= kHotMin) {
        for (uint32_t i = dp + 1; i < de; i++) {
          const uint32_t x = w.dlist[i];
          uint32_t j = i;
          while (j > dp && w.dlist[j - 1] > x) { w.dlist[j] = w.dlist[j - 1]; j--; }
          w.dlist[j] = x;
        }
      }
    }
  }
  const uint32_t* dmsg = w.dlist;

  // direct hit: message m owns entry m of the direct list
  auto emit_direct = [&](uint32_t m) {
    const uint32_t len = b.raw_len[m];
    const uint32_t off = alloc_record(k, rec_units(s, len), R, len);
    w.edir[m] = make_uint2(c, off);
  };

  // Connection-major records: one cmrun word per (group, connection) instead of one ecm entry per
  // record when the connection's records of the group are one run, which is what the pack merges
  // into one bulk store anyway.  Per thread: cm_last = cm rank of its last connection-major record
  // (kOffInvalid: none yet), cm_start = that group's run start or kCmBroken | position, cm_first = the
  // ecm index of the group's first record, cm_next = the unit after the run.  (In shared memory, and
  // the cmrun row found through a pointer staged per message: kept in registers, or indexed with 64-bit
  // arithmetic here, they cost k_offsets<false> 8 more registers and with them 2 of its 8 CTAs per SM.)
  __shared__ uint32_t cm_last_[NT], cm_first_[NT], cm_start_[NT], cm_next_[NT];
  uint32_t& cm_start = cm_start_[threadIdx.x];
  uint32_t& cm_next = cm_next_[threadIdx.x];
  cm_last_[threadIdx.x] = kOffInvalid;

  // Broadcasts are taken 32 at a time: the block stages their per-message metadata in shared
  // memory once, and every warp fetches its 32 match words / rank prefixes with ONE load per lane
  // (lane i ↔ message j0+i) instead of a dependent chain of warp-uniform loads per message.
  __shared__ uint32_t m_mb[32], m_len[32], m_eb[32], m_slot[32], m_cls[32], m_cmr[32];
  __shared__ uint32_t* m_run[32];   // the cmrun row of the message's group (connection-major messages)
  for (uint32_t j0 = 0; j0 < b.n_bcast; j0 += 32) {
    const uint32_t nj = min(32u, b.n_bcast - j0);
    __syncthreads();
    if (threadIdx.x < nj) {
      const uint32_t m = b.bcast_index[j0 + threadIdx.x];
      const uint32_t cl = w.cls[m];
      m_mb[threadIdx.x] = m;
      m_len[threadIdx.x] = b.raw_len[m];
      m_cls[threadIdx.x] = cl;
      if (cl == CLS_CM) {
        const uint32_t r = w.cm_rank[m];
        m_cmr[threadIdx.x] = r;
        m_run[threadIdx.x] = w.cmrun + (size_t)(r / kCmGroup) * s.N;
      }
      m_eb[threadIdx.x] = cl != CLS_THIN ? w.eb_fat[m] : w.eb_thin[m];
      m_slot[threadIdx.x] = b.slot_off16[m];
    }
    uint32_t Bw = 0, pre = 0;
    if (lane < nj) {
      const size_t at = (size_t)(j0 + lane) * s.W + wd;
      Bw = w.B[at];
      pre = w.base[(size_t)(j0 + lane) * s.nblk + (wd / kBlockWords)] + w.wpre[at];
    }
    __syncthreads();
    uint32_t hits = __ballot_sync(0xffffffffu, Bw != 0);  // messages of this chunk that reach the warp
    while (hits) {
      const int i = __ffs(hits) - 1;
      hits &= hits - 1;
      const uint32_t word = __shfl_sync(0xffffffffu, Bw, i), p = __shfl_sync(0xffffffffu, pre, i);
      const uint32_t mb = m_mb[i];
      if (HAS_DIRECT) while (dp < de && dmsg[dp] < mb) { emit_direct(dmsg[dp]); dp++; }  // keep batch order (R9)
      if ((word >> lane) & 1u) {
        const uint32_t rank = p + __popc(word & lt), len = m_len[i];
        const uint32_t u = rec_units(s, len);
        const uint32_t off = alloc_record(k, u, R, len);
        const uint32_t cl = m_cls[i];
        if (cl == CLS_CM) {
          // The group stops being one run at the first record that does not follow the previous one (a
          // wrap, another record of this connection in between, an overflow): from there on its records
          // get ecm entries, and so does the first one (the run start); the pack follows the run up to
          // that position.
          uint32_t* row = m_run[i];
          const uint32_t r = m_cmr[i];
          if ((r ^ cm_last_[threadIdx.x]) >= kCmGroup) {   // first record of a group (cm ranks ascend with the batch order)
            cm_start = off != kOffInvalid ? off : kCmBroken | (r & (kCmGroup - 1));
            cm_first_[threadIdx.x] = m_eb[i] + rank;
            row[c] = cm_start;
          } else if (cm_start < kCmBroken && off != cm_next) {
            w.ecm[cm_first_[threadIdx.x]] = cm_start;
            cm_start = kCmBroken | (r & (kCmGroup - 1));
            row[c] = cm_start;
          }
          if (cm_start >= kCmBroken) w.ecm[m_eb[i] + rank] = off;
          cm_last_[threadIdx.x] = r;
          cm_next = off + u;
        } else if (cl == CLS_FAT) w.efat[m_eb[i] + rank] = make_uint2(c, off);
        else w.ethin[m_eb[i] + rank] = make_uint4(c, off, m_slot[i], len);
      }
    }
  }
  if (HAS_DIRECT) while (dp < de) { emit_direct(dmsg[dp]); dp++; }

  if (s.pool) {
    // connection-order prefix of the units: inside the CTA by a scan, across CTAs by the look-back
    __shared__ uint32_t cta_prefix;
    uint32_t ctot;
    const uint32_t cex = cta_excl_scan<NW>(k.bu, &ctot, sm);
    if (FUSED) {
      if (threadIdx.x < 32) {
        const uint32_t pre = pool_lookback(w, vb, ctot);
        if (threadIdx.x == 0) {
          cta_prefix = pre;
          if (vb == nvb - 1) pool_allocate(s, w, (unsigned long long)pre + ctot);
        }
      }
    } else if (threadIdx.x == 0) {
      cta_prefix = 0;            // CTA-local: k_pool_finish adds the CTA's base to cbase[] and to the span table
      w.lb_tot[vb] = ctot;
    }
    __syncthreads();
    k.s1_off = cta_prefix + cex;   // relative to the batch's region (BatchStats::pool_base)
    w.cbase[c] = k.s1_off;
  } else {
    s.ptail[c] = k.pt;
    s.used[c] = k.us;
  }
  w.batch_units[c] = k.bu;

  // spans: one per contiguous run (two when the ring wrapped inside the batch)
  const uint32_t nsp = (k.s1_rec ? 1u : 0u) + (k.s2_rec ? 1u : 0u);
  uint32_t tot, ex;
  uint32_t run_len = 1, my_runs = nsp, nsp_warp = 0;
  if (s.span_runs) {
    // Run-length form: a connection CONTINUES its left neighbour's run when both own exactly one span
    // with the same (offset, length, records) — the normal case of a dense broadcast batch, where
    // every connection of the CTA receives the same records at the same ring position.  Runs never
    // cross a CTA (<= NT connections per run).
    __shared__ uint32_t r_off[NT], r_len[NT], r_rec[NT], r_brk[NT + 1];
    const uint32_t t = threadIdx.x;
    r_off[t] = k.s1_off; r_len[t] = k.s1_units; r_rec[t] = nsp == 1 ? k.s1_rec : 0u;  // 0 = "not exactly one span"
    __syncthreads();
    const bool cont = t > 0 && nsp == 1 && r_rec[t - 1] == k.s1_rec && r_len[t - 1] == k.s1_units &&
                      (s.pool ? r_off[t - 1] + r_len[t - 1] == k.s1_off : r_off[t - 1] == k.s1_off);
    const uint32_t head = (nsp > 0 && !cont) ? 1u : 0u;
    my_runs = head ? nsp : 0u;
    // ONE scan carries both numbers (each <= 2 * NT < 65536): low half = run slots before this thread,
    // high half = threads before it that do NOT continue a run.  A run ends at the next such thread,
    // so its length is a subtraction — no counters (a dense batch would hit one counter 255 times).
    uint32_t ptot;
    const uint32_t pex = cta_excl_scan<NW>(my_runs | (cont ? 0u : 1u << 16), &ptot, sm);
    ex = pex & 0xFFFFu; tot = ptot & 0xFFFFu;
    const uint32_t brk = pex >> 16;                 // rank of this thread among the run breakers
    if (!cont) r_brk[brk] = t;
    if (t == 0) r_brk[ptot >> 16] = NT;             // sentinel after the last breaker
    __syncthreads();
    if (head) run_len = r_brk[brk + 1] - t;         // followers sit between this breaker and the next
    if (threadIdx.x == 0) span_base = tot ? atomicAdd(&w.stats->n_runs, tot) : 0;
    nsp_warp = __reduce_add_sync(0xffffffffu, nsp);                    // n_spans keeps counting expanded spans (added per CTA below)
  } else {
    ex = cta_excl_scan<NW>(nsp, &tot, sm);
    if (threadIdx.x == 0) span_base = tot ? atomicAdd(&w.stats->n_spans, tot) : 0;
  }
  // block reduction of deliveries / bytes
  // (redux.sync on 32-bit halves: a warp's record count fits 32 bits, its byte count may not)
  const unsigned long long nrec = __reduce_add_sync(0xffffffffu, k.s1_rec + k.s2_rec);
  const unsigned long long by = (unsigned long long)__reduce_add_sync(0xffffffffu, k.bytes & 0xFFFFu) +
                                ((unsigned long long)__reduce_add_sync(0xffffffffu, k.bytes >> 16) << 16);
  if (lane == 0) { red[0][threadIdx.x >> 5] = nrec | ((unsigned long long)nsp_warp << 48); red[1][threadIdx.x >> 5] = by; }
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long a = 0, bb = 0, sp = 0;
    for (int i = 0; i < NW; i++) { a += red[0][i] & 0xFFFFFFFFFFFFull; sp += red[0][i] >> 48; bb += red[1][i]; }
    if (a) { atomicAdd(&w.stats->n_deliveries, a); atomicAdd(&w.stats->bytes_out, bb); }
    if (sp) atomicAdd(&w.stats->n_spans, (uint32_t)sp);
  }
  if (s.span_runs) {
    if (my_runs) {
      SpanRun* runs = reinterpret_cast<SpanRun*>(w.spans);
      uint32_t at = span_base + ex;
      if (k.s1_rec) runs[at++] = SpanRun{s.conn_base + c, run_len, s.pool ? k.s1_off : k.s1_off * kUnit, k.s1_units * kUnit, k.s1_rec, s.pool ? k.s1_units : 0u};
      if (k.s2_rec) runs[at] = SpanRun{s.conn_base + c, 1, 0, k.s2_units * kUnit, k.s2_rec, 0};
    }
  } else if (nsp) {
    uint32_t at = span_base + ex;
    if (k.s1_rec) w.spans[at++] = Span{s.conn_base + c, s.pool ? k.s1_off : k.s1_off * kUnit, k.s1_units * kUnit, k.s1_rec};
    if (k.s2_rec) w.spans[at] = Span{s.conn_base + c, 0, k.s2_units * kUnit, k.s2_rec};
  }
  if (k.ovf) {
    uint32_t i = atomicAdd(&w.stats->n_overflow, 1u);
    if (i < max_conns) w.overflow[i] = s.conn_base + c;
  }
}
template <bool HAS_DIRECT>
__global__ void __launch_bounds__(256) k_offsets(DevState s, BatchIn b, Work w, uint32_t max_conns) {
  offsets_body<HAS_DIRECT, 256, false>(s, b, w, max_conns, blockIdx.x * 256 + threadIdx.x, blockIdx.x, gridDim.x);  // N is a multiple of 8192
}
// Pool mode, after k_offsets: every CTA scans the (at most a few thousand) CTA totals in shared memory
// — redundantly, 16 KB of reads each, cheaper than a second dependent launch — then the grid adds each
// connection's CTA base to cbase[] and to the span / run table (entries name their connection, hence
// their CTA); CTA 0 takes the region out of the pool.
__global__ void __launch_bounds__(1024) k_pool_finish(DevState s, Work w, uint32_t nblk) {
  extern __shared__ uint32_t tb[];   // [nblk] exclusive CTA bases
  __shared__ uint32_t sm[33];
  __shared__ unsigned long long total_s;
  if (w.stats->status) return;
  unsigned long long carry = 0;
  for (uint32_t b0 = 0; b0 < nblk; b0 += 1024) {
    const uint32_t i = b0 + threadIdx.x;
    const uint32_t v = i < nblk ? w.lb_tot[i] : 0;
    uint32_t tot, ex = cta_excl_scan<32>(v, &tot, sm);
    const unsigned long long at = carry + ex;
    if (i < nblk) tb[i] = at > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)at;
    carry += tot;
  }
  if (threadIdx.x == 0) total_s = carry;
  __syncthreads();
  if (blockIdx.x == 0 && threadIdx.x == 0) pool_allocate(s, w, total_s);
  const uint32_t gt = blockIdx.x * 1024 + threadIdx.x, gn = gridDim.x * 1024;
  for (uint32_t c = gt; c < s.N; c += gn) w.cbase[c] += tb[c >> 8];
  if (s.span_runs) {
    SpanRun* r = reinterpret_cast<SpanRun*>(w.spans);
    const uint32_t n = w.stats->n_runs;
    for (uint32_t i = gt; i < n; i += gn) r[i].ring_off += tb[(r[i].conn0 - s.conn_base) >> 8];
  } else {
    const uint32_t n = w.stats->n_spans;
    for (uint32_t i = gt; i < n; i += gn) w.spans[i].ring_off += tb[(w.spans[i].conn - s.conn_base) >> 8];
  }
}

void launch_offsets(const DevState& s, const Work& w, const BatchIn& b, bool has_direct, int n_sms, cudaStream_t st) {
  if (has_direct) PCDN_COUNT_LAUNCH, k_offsets<true><<<s.N / 256, 256, 0, st>>>(s, b, w, s.N);
  else PCDN_COUNT_LAUNCH, k_offsets<false><<<s.N / 256, 256, 0, st>>>(s, b, w, s.N);
  if (s.pool) {
    const uint32_t nblk = s.N / 256;
    if (nblk * 4 > 48u * 1024) cudaFuncSetAttribute(k_pool_finish, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(nblk * 4));  // > 3 M connections per shard
    PCDN_COUNT_LAUNCH, k_pool_finish<<<std::min<uint32_t>((uint32_t)n_sms, (s.N + 8191) / 8192), 1024, nblk * 4, st>>>(s, w, nblk);
  }
}

// =============================================================================== fused control (small engines)
// Small geometries (N <= kSmallCtrlConns connection slots, i.e. at most 8 match blocks per message)
// with a batch of at most kSmallCtrlMsgs messages are the latency regime of a real broker (a few
// hundred to a few thousand consensus nodes, one vote or proposal at a time).  There the regular pipeline is a chain of five
// tiny dependent launches; here match, plan and offsets run in ONE launch on one cluster of eight
// 1024-thread CTAs — a thread per connection and 8192-connection pass — with cluster barriers where the pipeline has kernel
// boundaries.  It runs the code of k_match (match_block), k_plan_a (plan_messages, plan_finish) and
// k_offsets (offsets_body), so it writes exactly the arrays they write (the pack kernel and the host
// cannot tell the difference), zeroes the batch counters itself when no earlier kernel of the batch
// needs them, and publishes the final counters into mapped host memory.
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// one warp per match item: the whole match of a batch the fused path takes is one pass of the cluster's warps
static_assert(kSmallCtrlItems == 8 * 1024 / 32, "kSmallCtrlItems = the warps of k_ctrl_small's 8 CTAs of 1024 threads");
// offsets_only: the retry of a batch the output pool refused — the routing of the first run (direct
// bounds, match words, plan) is still in the scratch, only the offsets pass runs again.
template <bool HAS_DIRECT, bool TARGET>
__global__ void __cluster_dims__(8, 1, 1) __launch_bounds__(1024, 1)
k_ctrl_small(DevState s, BatchIn b, Work w, BatchStats* zero, BatchStats* publish, int offsets_only) {
  __shared__ uint32_t sm[33];
  const uint32_t tid = threadIdx.x, rank = blockIdx.x;  // grid = one cluster
  zero_stats(zero, rank == 0);

  // ---- direct messages (= k_direct_lookup + the grouping by connection) on CTA 0; at most
  //      kSmallCtrlMsgs of them, so the (connection, message) order is a rank count
  if (HAS_DIRECT && rank == 0 && !offsets_only) {
    __shared__ uint32_t skey_s[kSmallCtrlMsgs], sorted_s[kSmallCtrlMsgs];
    __syncthreads();  // counters are zero before the lookup counts dropped messages
    for (uint32_t g0 = 0; g0 < b.n_msgs * 8; g0 += 1024) direct_lookup_body<false>(s, b, w, g0 + tid);  // 128 messages per pass
    __syncthreads();
    const uint32_t n = b.n_msgs;
    if (tid < n) { const uint32_t t = w.dconn[tid]; skey_s[tid] = t == kConnNone ? s.N : t; }
    __syncthreads();
    if (tid < n) {
      const uint32_t key = skey_s[tid];
      uint32_t r = 0;
      for (uint32_t o = 0; o < n; o++) r += (skey_s[o] < key || (skey_s[o] == key && o < tid)) ? 1u : 0u;
      sorted_s[r] = key;
      w.dlist[r] = tid;
    }
    __syncthreads();
    if (tid < n) {
      const uint32_t key = sorted_s[tid];
      if (tid == 0 || sorted_s[tid - 1] != key) { w.dstart[key] = tid; w.dstamp[key] = w.stamp; }
      if (tid + 1 == n || sorted_s[tid + 1] != key) w.dend[key] = tid + 1;
    }
  }

  // ---- match (= k_match): warp = one (broadcast, 256-word block) item, the last warp of a broadcast
  //      writes its block bases and D_m
  if (!offsets_only) {
    const uint32_t item = rank * 32 + (tid >> 5), nblk = s.nblk;
    if (item < b.n_bcast * nblk) {   // warp-uniform
      if (b.n_events) match_block<true, TARGET>(s, b, w, item / nblk, item % nblk);
      else match_block<false, TARGET>(s, b, w, item / nblk, item % nblk);
    }
  }
  cluster_sync_all();

  // ---- plan (= k_plan_a of a one-block batch) on CTA 0
  if (rank == 0 && !offsets_only) {
    bool cm;
    const uint32_t r = plan_messages<32>(s, b, w, tid, 0, 1, sm, &cm);
    plan_finish(b, w, tid, cm, r);
  }
  cluster_sync_all();

  // ---- offsets: thread = connection (one pass per 8192 connections)
  // (pool mode: the CTA's position in connection order is pass * 8 + rank; the eight CTAs of the
  //  cluster are co-resident and earlier passes are complete, so the look-back never waits on a CTA
  //  that has not started)
  for (uint32_t c0 = 0; c0 < s.N; c0 += 8192)
    offsets_body<HAS_DIRECT, 1024, true>(s, b, w, s.N, c0 + rank * 1024 + tid, c0 / 1024 + rank, s.N / 1024);

  if (publish) {   // ---- final counters straight into the host's (mapped, pinned) result block
    cluster_sync_all();
    if (rank == 0) publish_stats(w, publish, false);
  }
}
void launch_ctrl_small(const DevState& s, const Work& w, const BatchIn& b, bool has_direct, bool targeted, BatchStats* zero,
                       BatchStats* publish, bool offsets_only, cudaStream_t st) {
  const int oo = offsets_only ? 1 : 0;
  if (targeted) {   // (as in launch_match: the instantiations without target rows stay as they are)
    if (has_direct) PCDN_COUNT_LAUNCH, k_ctrl_small<true, true><<<8, 1024, 0, st>>>(s, b, w, zero, publish, oo);
    else PCDN_COUNT_LAUNCH, k_ctrl_small<false, true><<<8, 1024, 0, st>>>(s, b, w, zero, publish, oo);
  } else {
    if (has_direct) PCDN_COUNT_LAUNCH, k_ctrl_small<true, false><<<8, 1024, 0, st>>>(s, b, w, zero, publish, oo);
    else PCDN_COUNT_LAUNCH, k_ctrl_small<false, false><<<8, 1024, 0, st>>>(s, b, w, zero, publish, oo);
  }
}

// Pool mode, retry of a refused batch: the offsets pass runs again from the counters as the plan left
// them (no refusal, nothing added yet by the offsets pass, whose counters are atomic sums; pack cursors
// at 0), and with cleared look-back words, so the fused kernel's look-back waits for this run's totals.
__global__ void k_pool_retry_begin(BatchStats* bs) {
  bs->status = 0;
  bs->n_deliveries = 0; bs->bytes_out = 0;
  bs->n_spans = 0; bs->n_runs = 0; bs->n_overflow = 0;
  bs->tile_cursor = 0; bs->cm_cursor = 0; bs->ctas_done = 0;
}
void launch_pool_retry_begin(const DevState& s, const Work& w, cudaStream_t st) {
  cudaMemsetAsync(w.lb_state, 0, ((size_t)s.N / 256 + 1) * 8, st);
  PCDN_COUNT_LAUNCH, k_pool_retry_begin<<<1, 1, 0, st>>>(w.stats);
}

// where a record goes: `off` units into the connection's own ring, or (pool mode) into the
// connection's region of this batch's slice of the output pool
__device__ __forceinline__ uint8_t* conn_out(const DevState& s, const Work& w, uint32_t conn, uint32_t pool_base) {
  return s.pool ? s.rings + ((size_t)pool_base + w.cbase[conn]) * kUnit : s.rings + (size_t)conn * s.ring_bytes;
}

// =============================================================================== K2a pack (fat)
// Persistent CTAs pull tiles (message, frame chunk, group of <=1024 recipients) from a counter.
// The chunk is staged ONCE per CTA into shared memory with a TMA bulk copy (mbarrier-completed),
// the 4-byte hole at the front of the slot is overwritten with the big-endian length (the
// cdn-proto framing, protocols/mod.rs:366-385), then every recipient gets the chunk with one TMA
// bulk store (shared → global), one lane per recipient.
__device__ __forceinline__ void pack_fat_phase(const DevState& s, const BatchIn& b, const Work& w, uint8_t* buf,
                                               uint64_t* barp) {
  uint64_t& bar = *barp;
  __shared__ uint32_t t_info[8];  // tile, m, chunk, r0, r1, nbytes, need_load
  const uint32_t tid = threadIdx.x;
  const uint32_t ntiles = w.stats->n_fat_tiles;
  if (ntiles == 0) return;
  const uint32_t pool_base = w.stats->pool_base;
  uint32_t phase = 0;
  uint32_t staged_m = 0xFFFFFFFFu, staged_k = 0xFFFFFFFFu;  // meaningful in thread 0 only

  for (;;) {
    if (tid == 0) {
      const uint32_t t = atomicAdd(&w.stats->tile_cursor, 1u);
      t_info[0] = t;
      if (t < ntiles) {
        uint32_t lo = 0, hi = b.n_msgs;  // largest m with tbase[m] <= t
        while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (w.tbase[mid] <= t) lo = mid; else hi = mid; }
        const uint32_t m = lo, ltile = t - w.tbase[m], d = w.D[m];
        const uint32_t fb = frame_vec_bytes(b.raw_len[m]);
        const uint32_t tr = tile_recipients(fb);
        const uint32_t ngrp = (d + tr - 1) / tr;
        const uint32_t ch = ltile / ngrp, grp = ltile % ngrp;
        const uint32_t nbytes = min(kChunkBytes, fb - ch * kChunkBytes);
        t_info[1] = m; t_info[2] = ch; t_info[3] = grp * tr;
        t_info[4] = min(d, (grp + 1) * tr); t_info[5] = nbytes;
        t_info[6] = (m != staged_m || ch != staged_k) ? 1u : 0u;
        staged_m = m; staged_k = ch;
      }
    }
    __syncthreads();
    if (t_info[0] >= ntiles) break;
    const uint32_t m = t_info[1], ch = t_info[2], r0 = t_info[3], r1 = t_info[4], nbytes = t_info[5];
    if (t_info[6]) {
      // re-stage: drain the bulk stores that still read the old chunk (only here, not per tile)
      bulk_wait_read0();
      __syncthreads();
      if (tid == 0) {
        mbar_arrive_expect_tx(&bar, nbytes);
        bulk_g2s(buf, b.arena + (size_t)b.slot_off16[m] * 16 + (size_t)ch * kChunkBytes, nbytes, &bar);
      }
      mbar_wait(&bar, phase);
      phase ^= 1;
      if (ch == 0) {  // fused framing: BE length prefix
        if (tid == 0) {
          *reinterpret_cast<uint32_t*>(buf) = bswap32(b.raw_len[m]);
          fence_proxy_async_smem();
        }
        __syncthreads();
      }
    }
    const uint2* E = w.efat + w.eb_fat[m];
    const size_t chunk_off = (size_t)ch * kChunkBytes;
    for (uint32_t r = r0 + tid; r < r1; r += 256) {
      const uint2 ent = E[r];
      if (ent.y != kOffInvalid)
        bulk_s2g(conn_out(s, w, ent.x, pool_base) + (size_t)ent.y * kUnit + chunk_off, buf, nbytes);
    }
    bulk_commit();
    __syncthreads();  // all reads of t_info done before thread 0 starts the next tile
  }
  bulk_wait_read0();
}

// =============================================================================== K2c pack (connection-major)
// Dense messages with small records (class CLS_CM) are taken in groups of up to kCmGroup in batch
// order.  A CTA stages the whole group in shared memory (one TMA bulk copy per frame, all counted
// on one mbarrier) in exactly the layout the records have in a ring (32-byte padded, back to back),
// patches the big-endian length prefixes, and then walks a tile of 512 connections.  For every
// connection the offsets of its matched records come from the scatter list (rank = block base +
// word prefix + lane rank, the same formula k_offsets used); records that are adjacent in the ring
// are written as ONE contiguous run — for the all-subscribed case that is the whole batch
// (8 x 1088 B = 8.7 KB) per connection instead of eight separate 1 KB writes, which is what the
// HBM row buffers want (scattered 1 KB granules are written well below the copy rate, runs of several KB close to it).
// Every lane issues one TMA bulk store (shared → global) per run of ITS connection.
__device__ __forceinline__ void pack_cm_phase(const DevState& s, const BatchIn& b, const Work& w, uint8_t* buf,
                                              uint64_t* barp) {
  uint64_t& bar = *barp;
  __shared__ uint32_t g_m[kCmGroup], g_j[kCmGroup], g_soff[kCmGroup], g_units[kCmGroup], g_eb[kCmGroup];
  __shared__ uint32_t t_info[4];  // tile, group, gcount, need_load
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (w.stats->status) return;
  const uint32_t ncm = w.stats->n_cm;
  if (ncm == 0) return;
  const uint32_t pool_base = w.stats->pool_base;
  const uint32_t ngroups = (ncm + kCmGroup - 1) / kCmGroup;
  const uint32_t tpg = s.W / kCmTileWords;  // tiles per group (W is a multiple of 256)
  const uint32_t ntiles = ngroups * tpg;
  uint32_t phase = 0;
  uint32_t staged_g = 0xFFFFFFFFu;  // meaningful in thread 0 only

  for (;;) {
    if (tid == 0) {
      const uint32_t t = atomicAdd(&w.stats->cm_cursor, 1u);
      t_info[0] = t;
      if (t < ntiles) {
        const uint32_t g = t / tpg;
        const uint32_t gcount = min(kCmGroup, ncm - g * kCmGroup);
        t_info[1] = g; t_info[2] = gcount;
        t_info[3] = g != staged_g ? 1u : 0u;
        staged_g = g;
      }
    }
    __syncthreads();
    if (t_info[0] >= ntiles) break;
    const uint32_t grp = t_info[1], gcount = t_info[2];
    if (t_info[3]) {
      // New group: shared memory is re-staged.  Bulk stores issued for earlier tiles only have to
      // be drained HERE (they read the old frames) — not after every tile, so the TMA store
      // queue never runs dry while the next tile's offsets are being fetched.
      bulk_wait_read0();
      __syncthreads();
      if (tid == 0) {
        const uint32_t g = t_info[1];
        uint32_t soff = 0, total = 0;
        for (uint32_t i = 0; i < gcount; i++) {
          const uint32_t m = w.cm_list[g * kCmGroup + i];
          const uint32_t len = b.raw_len[m];
          g_m[i] = m; g_j[i] = w.jidx[m]; g_soff[i] = soff; g_units[i] = frame_units(len); g_eb[i] = w.eb_fat[m];
          soff += frame_units(len) * kUnit;
          total += frame_vec_bytes(len);
        }
        mbar_arrive_expect_tx(&bar, total);
        for (uint32_t i = 0; i < gcount; i++)
          bulk_g2s(buf + g_soff[i], b.arena + (size_t)b.slot_off16[g_m[i]] * 16, frame_vec_bytes(b.raw_len[g_m[i]]), &bar);
      }
      __syncthreads();
      mbar_wait(&bar, phase);
      phase ^= 1;
      if (tid < gcount) {  // fused framing: one BE length prefix per staged frame
        *reinterpret_cast<uint32_t*>(buf + g_soff[tid]) = bswap32(b.raw_len[g_m[tid]]);
        fence_proxy_async_smem();
      }
      __syncthreads();
    }
    const uint32_t wt = t_info[0] % tpg;
    for (uint32_t wi = warp; wi < kCmTileWords; wi += 8) {
      const uint32_t wd = wt * kCmTileWords + wi;
      const uint32_t myword = lane < gcount ? w.B[(size_t)g_j[lane] * s.W + wd] : 0u;
      const uint32_t any = __reduce_or_sync(0xffffffffu, myword);
      if (!any) continue;
      uint32_t mine = 0;  // bit i: connection wd*32+lane receives message i of the group
#pragma unroll
      for (int i = 0; i < (int)kCmGroup; i++)
        mine |= ((__shfl_sync(0xffffffffu, myword, i) >> lane) & 1u) << i;
      mine &= (1u << gcount) - 1u;
      // ring offset of (connection = wd*32+lane, message i of the group), or invalid: from the run start
      // (k_offsets' cmrun) while the connection's records of the group follow each other, from the scatter
      // list for its first record and from the position where they stop following each other
      uint32_t offs[kCmGroup];
      const uint32_t run = mine ? w.cmrun[(size_t)grp * s.N + wd * 32 + lane] : kOffInvalid;
      const uint32_t brk = run >= kCmBroken ? run - kCmBroken : kCmGroup;
      uint32_t cur = run;
      bool first = true;
#pragma unroll
      for (int i = 0; i < (int)kCmGroup; i++) {
        offs[i] = kOffInvalid;
        if ((mine >> i) & 1u) {
          if (brk < kCmGroup && (first || (uint32_t)i >= brk)) {   // (rare: lanes of one warp may get here apart, so the match word is re-read)
            const uint32_t j = g_j[i];
            const size_t at = (size_t)j * s.W + wd;
            cur = w.ecm[g_eb[i] + w.base[(size_t)j * s.nblk + wd / kBlockWords] + w.wpre[at] + __popc(w.B[at] & ((1u << lane) - 1u))];
          }
          offs[i] = cur;
          first = false;
          if (cur != kOffInvalid) cur += g_units[i];
        }
      }
      // one lane = one connection: merge adjacent records into runs, one bulk store per run
      uint8_t* ring = conn_out(s, w, wd * 32 + lane, pool_base);
      uint32_t run_o = kOffInvalid, run_units = 0, run_s = 0;
#pragma unroll
      for (int i = 0; i < (int)kCmGroup; i++) {
        const uint32_t o = offs[i];
        if (o != kOffInvalid && run_o != kOffInvalid && o == run_o + run_units) {
          run_units += g_units[i];
        } else {
          if (run_o != kOffInvalid) bulk_s2g(ring + (size_t)run_o * kUnit, buf + run_s, run_units * kUnit);
          run_o = o; run_s = g_soff[i]; run_units = (o != kOffInvalid) ? g_units[i] : 0;
        }
      }
      if (run_o != kOffInvalid) bulk_s2g(ring + (size_t)run_o * kUnit, buf + run_s, run_units * kUnit);
    }
    bulk_commit();
    __syncthreads();  // all reads of g_* / t_info done before thread 0 starts the next tile
  }
  bulk_wait_read0();  // the next phase reuses buf
}

// =============================================================================== K2b pack (thin / direct)
// warp copies one framed record: 16-byte read-only loads from the frame slot, length prefix patched
// into the first vector, 16-byte streaming stores (four vectors per lane in flight)
__device__ __forceinline__ void copy_record(const uint4* __restrict__ src, uint4* __restrict__ dst, uint32_t raw_len, uint32_t lane) {
  const uint32_t nvec = (4u + raw_len + 15u) >> 4;
  const uint32_t hdr = bswap32(raw_len);
  for (uint32_t v = lane; v < nvec; v += 128) {
    uint4 x0, x1, x2, x3;
    const bool p1 = v + 32 < nvec, p2 = v + 64 < nvec, p3 = v + 96 < nvec;
    x0 = ld_nc16(src + v);
    if (p1) x1 = ld_nc16(src + v + 32);
    if (p2) x2 = ld_nc16(src + v + 64);
    if (p3) x3 = ld_nc16(src + v + 96);
    if (v == 0) x0.x = hdr;
    st_stream16(dst + v, x0);
    if (p1) st_stream16(dst + v + 32, x1);
    if (p2) st_stream16(dst + v + 64, x2);
    if (p3) st_stream16(dst + v + 96, x3);
  }
}
// Warp per scatter-list entry (broadcasts with < kFatMin recipients); k_pack_ref writes the entries of
// messages delivered by reference.
__device__ __forceinline__ void pack_thin_phase(const DevState& s, const BatchIn& b, const Work& w) {
  const uint32_t n = w.stats->n_thin_entries;
  const uint32_t pool_base = w.stats->pool_base;
  const uint32_t lane = lane_id();
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t e = gw; e < n; e += nw) {
    const uint4 ent = w.ethin[e];
    if (ent.y == kOffInvalid || by_ref(s, ent.w)) continue;
    copy_record(reinterpret_cast<const uint4*>(b.arena + (size_t)ent.z * 16),
                reinterpret_cast<uint4*>(conn_out(s, w, ent.x, pool_base) + (size_t)ent.y * kUnit), ent.w, lane);
  }
}
// Direct messages: warp per MESSAGE — entry m of the direct list, the frame slot and the length are
// all indexed by the message, so the warps of a CTA stream the arena in order; only the record
// stores are scattered (one ~700 B record per ring).
// (a variant with four entries in flight per warp measured no faster: the phase is bound by the
// scattered sub-KB writes, not by load latency)
__device__ __forceinline__ void pack_direct_phase(const DevState& s, const BatchIn& b, const Work& w) {
  const uint32_t n = b.n_msgs;
  const uint32_t pool_base = w.stats->pool_base;
  const uint32_t lane = lane_id();
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  // The three per-message words (list entry, slot, length) of the NEXT message are fetched while the
  // current record is being copied: the chain entry → frame → stores loses its first DRAM round trip.
  uint2 ent = make_uint2(0, kOffInvalid);
  uint32_t so = 0, len = 0;
  if (gw < n) { ent = w.edir[gw]; so = b.slot_off16[gw]; len = b.raw_len[gw]; }
  for (uint32_t m = gw; m < n; m += nw) {
    const uint2 cur = ent;
    const uint32_t cso = so, clen = len;
    const uint32_t nx = m + nw;
    if (nx < n) { ent = w.edir[nx]; so = b.slot_off16[nx]; len = b.raw_len[nx]; }
    if (cur.y == kOffInvalid || by_ref(s, clen)) continue;   // (by reference: k_pack_ref)
    copy_record(reinterpret_cast<const uint4*>(b.arena + (size_t)cso * 16),
                reinterpret_cast<uint4*>(conn_out(s, w, cur.x, pool_base) + (size_t)cur.y * kUnit), clen, lane);
  }
}

// The pack kernel that ends a batch publishes its final counters into mapped host memory, so that the batch's
// ev_done covers them without a device-to-host copy on the stream between one pack and the next batch.
// Every CTA counts itself done (also when the batch was refused); the last one copies the counters.
__device__ __forceinline__ void publish_if_last(const Work& w, BatchStats* publish) {
  if (!publish) return;
  __shared__ uint32_t last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    last = atomicAdd(&w.stats->ctas_done, 1u) == gridDim.x - 1 ? 1u : 0u;
  }
  __syncthreads();
  if (last) publish_stats(w, publish, true);
}

// One launch runs the pack phases back to back in persistent CTAs (each phase pulls its own
// work from its own cursor, so CTAs drift from phase to phase without a grid barrier; the phases
// write disjoint records).
__global__ void __launch_bounds__(256) k_pack(DevState s, BatchIn b, Work w, int do_direct, BatchStats* publish) {
  __shared__ __align__(128) uint8_t buf[kCmGroup * kCmMaxBytes];  // 32 KB; the fat phase uses the first 16 KB
  __shared__ __align__(8) uint64_t bars[2];
  if (!w.stats->status) {
    if (threadIdx.x == 0) {
      mbar_init(&bars[0], 1);
      mbar_init(&bars[1], 1);
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    pack_cm_phase(s, b, w, buf, &bars[0]);
    __syncthreads();
    pack_fat_phase(s, b, w, buf, &bars[1]);
    pack_thin_phase(s, b, w);
    if (do_direct) pack_direct_phase(s, b, w);
  }
  publish_if_last(w, publish);
}
// Batches dominated by direct messages run the direct phase as its own launch at full occupancy
// (no shared memory, 8 CTAs per SM): a warp per record is a chain of two dependent DRAM reads
// (list entry, frame) before its stores, so the phase scales with warps in flight — 24 → 48
// warps per SM is faster on the 1 M x 512 B direct workload (config C4).
__global__ void __launch_bounds__(256, 8) k_pack_direct(DevState s, BatchIn b, Work w, BatchStats* publish) {
  if (!w.stats->status) pack_direct_phase(s, b, w);
  publish_if_last(w, publish);
}

// =============================================================================== K2r pack (reference records)
// A message delivered by reference (by_ref: every message of a PCDN_FLAG_SHARED_PAYLOAD engine, those of at
// least ref_min_bytes on an engine with that threshold) gets ONE 32-byte reference record (pcdn_fanout.h) per
// delivery instead of a framed copy: marker, BE length, offset of the raw bytes in the batch's frame arena, batch id, zero.
// One sector, two 16-byte streaming stores, no partial-sector write.  The record depends on the message
// and the batch only, so a retried batch writes identical records wherever the pool places them.
__device__ __forceinline__ void st_ref_record(uint8_t* dst, uint32_t raw_len, uint32_t slot_off16, unsigned long long batch_id) {
  const unsigned long long off = (unsigned long long)slot_off16 * 16u + 4u;
  st_stream16(dst, make_uint4(0xFFFFFFFFu, bswap32(raw_len), (uint32_t)off, (uint32_t)(off >> 32)));
  st_stream16(dst + 16, make_uint4((uint32_t)batch_id, (uint32_t)(batch_id >> 32), 0u, 0u));
}
// Thread per delivery over the three scatter lists back to back: message-major (efat: the owning message
// is found by a binary search of eb_fat), thin (ethin carries everything) and direct (edir, entry m =
// message m).  Entries of one message are in connection order, so a warp's 32 stores go to 32
// consecutive connections; a connection's records of successive messages are adjacent in its ring.  Entries of
// messages delivered as copies are k_pack's: skipped here (never on a shared-payload engine).
__global__ void __launch_bounds__(256) k_pack_ref(DevState s, BatchIn b, Work w, int do_direct, BatchStats* publish) {
  if (w.stats->status) { publish_if_last(w, publish); return; }
  const uint32_t nfat = w.stats->n_fat_entries, nthin = w.stats->n_thin_entries;
  const uint64_t nft = (uint64_t)nfat + nthin, total = nft + (do_direct ? b.n_msgs : 0u);
  const uint32_t pool_base = w.stats->pool_base;
  const unsigned long long bid = w.batch_id;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    uint32_t conn, off, m = 0, slot = 0, len = 0;
    bool thin = false;
    if (i < nfat) {
      const uint32_t e = (uint32_t)i;
      uint32_t lo = 0, hi = b.n_msgs;  // largest m with eb_fat[m] <= e: the message that owns entry e
      while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (w.eb_fat[mid] <= e) lo = mid; else hi = mid; }
      const uint2 ent = w.efat[e];
      conn = ent.x; off = ent.y; m = lo;
    } else if (i < nft) {
      const uint4 ent = w.ethin[i - nfat];
      conn = ent.x; off = ent.y; slot = ent.z; len = ent.w; thin = true;
    } else {
      m = (uint32_t)(i - nft);
      const uint2 ent = w.edir[m];
      conn = ent.x; off = ent.y;
    }
    if (off == kOffInvalid) continue;   // ring overflow, or a direct message this shard does not deliver
    if (!thin) { slot = b.slot_off16[m]; len = b.raw_len[m]; }
    // (a copied message's entries are k_pack's; those of a connection-major one are not even in efat, whose
    //  slots in its range hold nothing meaningful: this test comes before conn / off are used)
    if (!by_ref(s, len)) continue;
    st_ref_record(conn_out(s, w, conn, pool_base) + (size_t)off * kUnit, len, slot, bid);
  }
  publish_if_last(w, publish);
}

void launch_pack(const DevState& s, const Work& w, const BatchIn& b, uint32_t n_direct, uint32_t pack_ctas, uint32_t direct_ctas,
                 int n_sms, bool has_ref, BatchStats* publish, cudaStream_t st) {
  if (!b.n_bcast && !n_direct) {   // no pack kernel: the counters are final as the control stage left them
    if (publish) cudaMemcpyAsync(publish, w.stats, sizeof(BatchStats), cudaMemcpyDefault, st);
    return;
  }
  const uint32_t ref_grid = (uint32_t)n_sms * kPackRefCtas;
  if (s.ref_min == 0) {   // shared payload: k_pack_ref is the whole pack
    PCDN_COUNT_LAUNCH, k_pack_ref<<<ref_grid, 256, 0, st>>>(s, b, w, n_direct ? 1 : 0, publish);
    return;
  }
  // copies; with a message delivered by reference in the batch, k_pack_ref follows on the same stream and is the
  // kernel that publishes the counters
  BatchStats* copy_publish = has_ref ? nullptr : publish;
  const bool direct_separate = n_direct >= kThinSeparateMin;
  const int do_direct = (n_direct && !direct_separate) ? 1 : 0;
  if (b.n_bcast || do_direct)  // (a batch of nothing but many direct messages has no work for this kernel)
    PCDN_COUNT_LAUNCH, k_pack<<<(uint32_t)n_sms * pack_ctas, 256, 0, st>>>(s, b, w, do_direct, direct_separate ? nullptr : copy_publish);
  if (direct_separate) PCDN_COUNT_LAUNCH, k_pack_direct<<<(uint32_t)n_sms * direct_ctas, 256, 0, st>>>(s, b, w, copy_publish);
  if (has_ref) PCDN_COUNT_LAUNCH, k_pack_ref<<<ref_grid, 256, 0, st>>>(s, b, w, n_direct ? 1 : 0, publish);
}

// =============================================================================== release
// four connections per thread (N is a multiple of 8192; both arrays are separate allocations)
// (a batch the device rejected — BatchStats::status — reserved nothing: its batch_units are stale)
__global__ void __launch_bounds__(256) k_release(DevState s, const uint32_t* __restrict__ batch_units,
                                                 const BatchStats* __restrict__ stats) {
  if (stats->status) return;
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i * 4 < s.N) {
    const uint4 u = reinterpret_cast<const uint4*>(batch_units)[i];
    if (u.x | u.y | u.z | u.w) {
      uint4* p = reinterpret_cast<uint4*>(s.used) + i;
      uint4 v = *p;
      v.x -= u.x; v.y -= u.y; v.z -= u.z; v.w -= u.w;
      *p = v;
    }
  }
}
// pool mode: the region of the oldest batch goes back (batches are released in order)
__global__ void k_pool_release(PoolState* p, const BatchStats* __restrict__ stats) {
  if (stats->status) return;  // a refused batch holds nothing
  p->used -= stats->pool_units + stats->pool_skip;
  p->tail = stats->pool_base + stats->pool_units;
  if (p->used == 0) { p->head = 0; p->tail = 0; }
}
__global__ void k_pool_init(PoolState* p) { p->head = 0; p->tail = 0; p->used = 0; p->blocked = 0; }
void launch_pool_init(const DevState& s, cudaStream_t st) {
  if (s.pool) PCDN_COUNT_LAUNCH, k_pool_init<<<1, 1, 0, st>>>(s.pool_state);
}
void launch_release(const DevState& s, const uint32_t* batch_units, const BatchStats* stats, cudaStream_t st) {
  if (s.pool) { PCDN_COUNT_LAUNCH, k_pool_release<<<1, 1, 0, st>>>(s.pool_state, stats); return; }
  PCDN_COUNT_LAUNCH, k_release<<<(s.N / 4 + 255) / 256, 256, 0, st>>>(s, batch_units, stats);
}

}  // namespace pcdn
