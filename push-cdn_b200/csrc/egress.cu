// egress.cu — the consumer side of the span table: what the reference's per-connection writer task
// does with its queue (cdn-proto/src/connection/protocols/mod.rs:156-186: pop a message, write the
// u32 BE length and the bytes to the socket, :354-394) and its soft_close (:287-306: everything queued
// before the close still goes out).
//
// The pack kernel leaves a batch as framed records in the per-connection rings (HBM by default).
// pcdn_egress_drain turns one batch into bytes a socket writer can read: per local shard the spans are
// cut into chunks, a gather kernel (k_gather_spans) copies each chunk's records into ONE contiguous
// device buffer, one large DMA per chunk brings it into pinned host memory (two device and three
// host buffers in flight: the gather of chunk c+1 and the DMA of chunk c overlap the consumer of chunk
// c-1), and the sink gets {host bytes, spans, offset of every span}.  Engines with PCDN_FLAG_HOST_RINGS
// skip all of that: the sink sees the rings in place.  The built-in sink writes every span to the
// file descriptor attached to its connection with writev (length prefix + raw bytes per record, the
// padding between records skipped), on a small thread pool, keeping per-connection order.  On an engine
// that delivers by reference (PCDN_FLAG_SHARED_PAYLOAD, or messages of at least ref_min_bytes) a reference
// record becomes two iovecs: its 4 length bytes and the L
// bytes of the batch's payload (pcdn_batch_payload) it points to.
//
// With backlogs configured (pcdn_egress_config.backlog_bytes_*) the built-in sink never waits for a
// peer: what a socket does not take is copied into that connection's backlog in host memory and
// written later (before its next records, by pcdn_egress_flush_backlog, or by soft_close).  The
// backlog is host memory rather than unreleased ring space because a ring is released per batch for
// all its connections (k_release), the output pool frees a batch's region as a whole, and a shared
// payload is freed when its batch is released: none of them can hold one slow connection's bytes.
#include <errno.h>
#include <poll.h>
#include <sys/socket.h>
#include <sys/uio.h>
#include <unistd.h>

#include <atomic>
#include <condition_variable>
#include <cstddef>
#include <functional>

#include "engine_internal.h"

namespace pcdn {

struct GatherDesc { unsigned long long src_off, dst_off; uint32_t len, pad; };  // bytes; len is a multiple of 32

// warp per span: 16-byte read-only loads from the ring, 16-byte stores into the staging chunk
__global__ void __launch_bounds__(256) k_gather_spans(const uint8_t* __restrict__ rings, const GatherDesc* __restrict__ d,
                                                       uint32_t n, uint8_t* __restrict__ dst) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t i = gw; i < n; i += nw) {
    const GatherDesc g = d[i];
    const uint4* s = reinterpret_cast<const uint4*>(rings + g.src_off);
    uint4* o = reinterpret_cast<uint4*>(dst + g.dst_off);
    const uint32_t nvec = g.len >> 4;
    for (uint32_t v = lane; v < nvec; v += 128) {
      uint4 x0, x1, x2, x3;
      const bool p1 = v + 32 < nvec, p2 = v + 64 < nvec, p3 = v + 96 < nvec;
      asm volatile("ld.global.nc.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(x0.x), "=r"(x0.y), "=r"(x0.z), "=r"(x0.w) : "l"(s + v));
      if (p1) asm volatile("ld.global.nc.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(x1.x), "=r"(x1.y), "=r"(x1.z), "=r"(x1.w) : "l"(s + v + 32));
      if (p2) asm volatile("ld.global.nc.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(x2.x), "=r"(x2.y), "=r"(x2.z), "=r"(x2.w) : "l"(s + v + 64));
      if (p3) asm volatile("ld.global.nc.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(x3.x), "=r"(x3.y), "=r"(x3.z), "=r"(x3.w) : "l"(s + v + 96));
      o[v] = x0;
      if (p1) o[v + 32] = x1;
      if (p2) o[v + 64] = x2;
      if (p3) o[v + 96] = x3;
    }
  }
}

}  // namespace pcdn

using namespace pcdn;

namespace {

constexpr int kHostBufs = 3, kDevBufs = 2;
constexpr uint32_t kMaxChunkSpans = 1u << 18;

struct ShardEgress {
  uint8_t* d_stage[kDevBufs] = {nullptr, nullptr};
  GatherDesc* d_desc[kDevBufs] = {nullptr, nullptr};
  uint8_t* h_stage[kHostBufs] = {nullptr, nullptr, nullptr};
  GatherDesc* h_desc[kHostBufs] = {nullptr, nullptr, nullptr};
  std::vector<uint64_t> data_off[kHostBufs];
  std::vector<pcdn_span> expanded;
  cudaStream_t gs = nullptr, cs = nullptr;
  cudaEvent_t ev_gather[kDevBufs] = {nullptr, nullptr};
  cudaEvent_t ev_chunk[kHostBufs] = {nullptr, nullptr, nullptr};  // chunk is in host memory (also: its device buffer is free)
  cudaEvent_t ev_dev_free[kDevBufs] = {nullptr, nullptr};
  bool dev_used[kDevBufs] = {false, false};
};

// a tiny persistent pool: run(n, f) calls f(0..n-1) on the workers and the caller, returns when all are done
struct Pool {
  std::vector<std::thread> th;
  std::mutex mu;
  std::condition_variable cv, done_cv;
  std::function<void(uint32_t)> job;
  uint32_t n_parts = 0, next = 0, running = 0;
  uint64_t gen = 0;
  bool stop = false;
  explicit Pool(uint32_t n) {
    for (uint32_t i = 1; i < n; i++) th.emplace_back([this] { loop(); });
  }
  ~Pool() {
    { std::lock_guard<std::mutex> g(mu); stop = true; }
    cv.notify_all();
    for (auto& t : th) t.join();
  }
  void loop() {
    uint64_t seen = 0;
    for (;;) {
      std::unique_lock<std::mutex> lk(mu);
      cv.wait(lk, [&] { return stop || (gen != seen && next < n_parts); });
      if (stop) return;
      seen = gen;
      while (next < n_parts) {
        const uint32_t p = next++;
        running++;
        lk.unlock();
        job(p);
        lk.lock();
        running--;
      }
      if (running == 0) done_cv.notify_all();
    }
  }
  void run(uint32_t n, std::function<void(uint32_t)> f) {
    if (n == 0) return;
    if (th.empty() || n == 1) { for (uint32_t i = 0; i < n; i++) f(i); return; }
    std::unique_lock<std::mutex> lk(mu);
    job = std::move(f); n_parts = n; next = 0; gen++;
    cv.notify_all();
    while (next < n_parts) {
      const uint32_t p = next++;
      running++;
      lk.unlock();
      job(p);
      lk.lock();
      running--;
    }
    done_cv.wait(lk, [&] { return running == 0; });
    n_parts = 0;
  }
};

inline uint32_t be32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }

// one connection's backlog (pcdn_egress_config.backlog_bytes_*): wire bytes its peer has not taken
// yet, buf[head..).  Copies, never pointers: the chunk and the shared payload the bytes came from are
// gone once the sink returns / the batch is released.
struct Backlog {
  std::vector<uint8_t> buf;
  size_t head = 0;
  bool listed = false;  // in pcdn_egress::bl_list
  uint64_t pending() const { return buf.size() - head; }
};

}  // namespace

struct pcdn_egress {
  pcdn_engine* e = nullptr;
  pcdn_egress_config cfg{};
  std::mutex mu;       // one drain at a time
  std::mutex sink_mu;  // shards drain side by side, but the sink sees one chunk at a time
  std::vector<ShardEgress> sh;
  std::unique_ptr<Pool> pool;
  // fd table of the built-in sink: index = global connection id; -1 = not attached, -2 = failed
  std::vector<int> fds;
  std::mutex fail_mu;
  std::vector<pcdn_conn> failed, failed_out;
  pcdn_egress_stats last{};
  std::atomic<uint64_t> fd_bytes{0}, fd_writes{0}, unattached{0}, records{0};
  // engines that deliver by reference: the batch being drained and its payload base (reference records point into it)
  const uint8_t* payload = nullptr;
  uint64_t batch_id = 0;
  std::atomic<bool> bad_ref{false};
  // backlogs (index = global connection id, allocated on a connection's first backlog).  During a
  // drain only the writer-pool part that owns a connection touches its entry; the total is shared by
  // every part of every shard thread.  bl_list: the connections with a backlog (a few stale entries
  // whose backlog emptied are dropped under `mu`, where no drain runs).
  bool backlog_on = false;
  std::vector<std::unique_ptr<Backlog>> bl;
  std::atomic<uint64_t> bl_total{0};
  std::mutex bl_mu;  // bl_list during a drain
  std::vector<pcdn_conn> bl_list, bl_out;
};

namespace {

int init_shard_egress(pcdn_egress* g, uint32_t li) {
  pcdn_engine* e = g->e;
  Shard& sh = e->shards[li];
  if (sh.h_rings) return 0;  // rings already live in host memory
  ShardEgress& s = g->sh[li];
  DeviceGuard dg(sh.device);
  const size_t cb = g->cfg.chunk_bytes;
  for (int i = 0; i < kDevBufs; i++) {
    CUDA_TRY(cudaMalloc((void**)&s.d_stage[i], cb));
    CUDA_TRY(cudaMalloc((void**)&s.d_desc[i], (size_t)kMaxChunkSpans * sizeof(GatherDesc)));
    CUDA_TRY(cudaEventCreateWithFlags(&s.ev_gather[i], cudaEventDisableTiming));
    CUDA_TRY(cudaEventCreateWithFlags(&s.ev_dev_free[i], cudaEventDisableTiming));
  }
  for (int i = 0; i < kHostBufs; i++) {
    CUDA_TRY(cudaHostAlloc((void**)&s.h_stage[i], cb, cudaHostAllocPortable));
    CUDA_TRY(cudaHostAlloc((void**)&s.h_desc[i], (size_t)kMaxChunkSpans * sizeof(GatherDesc), cudaHostAllocPortable));
    CUDA_TRY(cudaEventCreateWithFlags(&s.ev_chunk[i], cudaEventDisableTiming));
  }
  CUDA_TRY(cudaStreamCreateWithFlags(&s.gs, cudaStreamNonBlocking));
  CUDA_TRY(cudaStreamCreateWithFlags(&s.cs, cudaStreamNonBlocking));
  return 0;
}

void free_shard_egress(pcdn_egress* g, uint32_t li) {
  ShardEgress& s = g->sh[li];
  cudaSetDevice(g->e->shards[li].device);
  if (s.gs) cudaStreamSynchronize(s.gs);
  if (s.cs) cudaStreamSynchronize(s.cs);
  for (int i = 0; i < kDevBufs; i++) {
    if (s.d_stage[i]) cudaFree(s.d_stage[i]);
    if (s.d_desc[i]) cudaFree(s.d_desc[i]);
    if (s.ev_gather[i]) cudaEventDestroy(s.ev_gather[i]);
    if (s.ev_dev_free[i]) cudaEventDestroy(s.ev_dev_free[i]);
  }
  for (int i = 0; i < kHostBufs; i++) {
    if (s.h_stage[i]) cudaFreeHost(s.h_stage[i]);
    if (s.h_desc[i]) cudaFreeHost(s.h_desc[i]);
    if (s.ev_chunk[i]) cudaEventDestroy(s.ev_chunk[i]);
  }
  if (s.gs) cudaStreamDestroy(s.gs);
  if (s.cs) cudaStreamDestroy(s.cs);
}

// one local shard's share of a batch → chunks → sink
int drain_shard(pcdn_egress* g, uint64_t batch_id, uint32_t li, pcdn_egress_sink sink, void* user, pcdn_egress_stats* st) {
  pcdn_engine* e = g->e;
  pcdn_batch_result res{};
  int rc = pcdn_poll_shard(e, batch_id, li, &res, 1);
  if (rc) return rc;
  if (res.status == (uint32_t)(-PCDN_EAGAIN))
    return fail(PCDN_EAGAIN, "the batch was refused for space in the output pool: release older batches, pcdn_retry_batch, drain again");
  if (res.status) return fail(PCDN_E2BIG, "batch was rejected on the device: nothing to drain");
  Shard& sh = e->shards[li];
  ShardEgress& s = g->sh[li];
  const uint64_t ring_bytes = e->cfg.ring_bytes_per_conn;
  const uint32_t base = sh.dev.conn_base;
  // run-length span tables (PCDN_FLAG_SPAN_RUNS) are expanded here: the sink always sees plain spans
  if (res.runs) {
    s.expanded.clear();
    for (uint32_t i = 0; i < res.n_runs; i++) {
      const pcdn_span_run& r = res.runs[i];
      for (uint32_t k = 0; k < r.n_conns; k++) s.expanded.push_back(pcdn_span{r.conn0 + k, r.ring_off + k * r.off_stride, r.len, r.n_records});
    }
  }
  const pcdn_span* sp = res.runs ? s.expanded.data() : res.spans;
  const uint32_t ns = res.runs ? (uint32_t)s.expanded.size() : res.n_spans;
  st->spans += ns;
  // where a span's records lie inside the shard's ring array / output pool
  const bool pool = sh.dev.pool != 0;
  const uint64_t pool_base = res.pool_base;
  auto src_of = [&](const pcdn_span& x) -> uint64_t {
    return pool ? (pool_base + x.ring_off) * (uint64_t)PCDN_RECORD_ALIGN : (uint64_t)(x.conn - base) * ring_bytes + x.ring_off;
  };
  if (sh.h_rings) {
    // egress hand-off mode: one chunk, the records are read where the pack kernel stored them
    std::vector<uint64_t>& off = s.data_off[0];
    off.resize(ns);
    uint64_t bytes = 0;
    for (uint32_t i = 0; i < ns; i++) { off[i] = src_of(sp[i]); bytes += sp[i].len; }
    pcdn_egress_chunk ch{li, ns, sp, off.data(), sh.h_rings, sh.dev.pool ? e->pool_bytes : (uint64_t)e->geo.shard_max_conns * ring_bytes};
    st->bytes += bytes; st->chunks += 1;
    if (ns && sink) {
      std::lock_guard<std::mutex> sl(g->sink_mu);
      if ((rc = sink(user, &ch))) return fail(PCDN_EINVAL, "egress sink returned " + std::to_string(rc));
    }
    return 0;
  }
  DeviceGuard dg(sh.device);
  const uint64_t cb = g->cfg.chunk_bytes;
  struct ChunkRange { uint32_t i0, i1; uint64_t bytes; };
  auto issue = [&](uint32_t c, const ChunkRange& r) -> int {
    const int hb = (int)(c % kHostBufs), db = (int)(c % kDevBufs);
    GatherDesc* hd = s.h_desc[hb];
    std::vector<uint64_t>& off = s.data_off[hb];
    off.resize(r.i1 - r.i0);
    uint64_t at = 0;
    for (uint32_t i = r.i0; i < r.i1; i++) {
      hd[i - r.i0] = GatherDesc{(unsigned long long)src_of(sp[i]), at, sp[i].len, 0};
      off[i - r.i0] = at;
      at += sp[i].len;
    }
    const uint32_t n = r.i1 - r.i0;
    if (s.dev_used[db]) CUDA_TRY(cudaStreamWaitEvent(s.gs, s.ev_dev_free[db], 0));  // the DMA that last read this device buffer
    CUDA_TRY(cudaMemcpyAsync(s.d_desc[db], hd, (size_t)n * sizeof(GatherDesc), cudaMemcpyHostToDevice, s.gs));
    const uint32_t grid = (uint32_t)std::min<uint64_t>((uint64_t)sh.n_sms * 8, ((uint64_t)n * 32 + 255) / 256);
    count_kernel_launch();
    k_gather_spans<<<grid, 256, 0, s.gs>>>(sh.dev.rings, s.d_desc[db], n, s.d_stage[db]);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaEventRecord(s.ev_gather[db], s.gs));
    CUDA_TRY(cudaStreamWaitEvent(s.cs, s.ev_gather[db], 0));
    CUDA_TRY(cudaMemcpyAsync(s.h_stage[hb], s.d_stage[db], r.bytes, cudaMemcpyDeviceToHost, s.cs));
    CUDA_TRY(cudaEventRecord(s.ev_chunk[hb], s.cs));
    CUDA_TRY(cudaEventRecord(s.ev_dev_free[db], s.cs));
    s.dev_used[db] = true;
    return 0;
  };
  // cut the span table into chunks (a connection's two wrap spans stay in one chunk)
  std::vector<ChunkRange> chunks;
  for (uint32_t i = 0; i < ns;) {
    ChunkRange r{i, i, 0};
    while (r.i1 < ns && r.i1 - r.i0 < kMaxChunkSpans) {
      uint32_t take = 1;
      uint64_t b = sp[r.i1].len;
      if (r.i1 + 1 < ns && sp[r.i1 + 1].conn == sp[r.i1].conn) { take = 2; b += sp[r.i1 + 1].len; }
      if (b > cb) return fail(PCDN_ENOSPC, "a connection's spans exceed pcdn_egress_config.chunk_bytes");
      if (r.bytes + b > cb || r.i1 - r.i0 + take > kMaxChunkSpans) break;
      r.bytes += b; r.i1 += take;
    }
    chunks.push_back(r);
    i = r.i1;
  }
  const uint32_t nc = (uint32_t)chunks.size();
  for (uint32_t c = 0; c < nc && c < 2; c++) if ((rc = issue(c, chunks[c]))) return rc;
  for (uint32_t c = 0; c < nc; c++) {
    const int hb = (int)(c % kHostBufs);
    CUDA_TRY(cudaEventSynchronize(s.ev_chunk[hb]));
    pcdn_egress_chunk ch{li, chunks[c].i1 - chunks[c].i0, sp + chunks[c].i0, s.data_off[hb].data(), s.h_stage[hb], chunks[c].bytes};
    st->bytes += chunks[c].bytes; st->chunks += 1;
    // the next chunk but one reuses neither this chunk's host buffer (3 in rotation) nor a device
    // buffer still being read (ev_dev_free): issue it before running the sink so the link stays busy
    if (c + 2 < nc && (rc = issue(c + 2, chunks[c + 2]))) return rc;
    if (sink) {
      std::lock_guard<std::mutex> sl(g->sink_mu);
      rc = sink(user, &ch);
    }
    if (rc) {
      cudaStreamSynchronize(s.cs);
      return fail(PCDN_EINVAL, "egress sink returned " + std::to_string(rc));
    }
  }
  return 0;
}

// ---- built-in sink: writev to the connection's file descriptor --------------------------------
// sockets are written with sendmsg(MSG_NOSIGNAL) so a peer that went away is an error return (EPIPE),
// not a SIGPIPE for the host process; pipes / memfds / files (ENOTSOCK) fall back to writev
bool write_all(int fd, struct iovec* iov, int cnt, uint64_t* nbytes, uint64_t* nwrites) {
  bool is_sock = true;
  while (cnt > 0) {
    const int take = std::min(cnt, 1024);  // IOV_MAX
    ssize_t w;
    if (is_sock) {
      struct msghdr mh{};
      mh.msg_iov = iov; mh.msg_iovlen = (size_t)take;
      w = ::sendmsg(fd, &mh, MSG_NOSIGNAL);
      if (w < 0 && errno == ENOTSOCK) { is_sock = false; continue; }
    } else {
      w = ::writev(fd, iov, take);
    }
    if (w < 0) {
      if (errno == EINTR) continue;
      if (errno == EAGAIN || errno == EWOULDBLOCK) {  // non-blocking socket with a full send buffer: wait for the peer
        struct pollfd p{fd, POLLOUT, 0};
        if (::poll(&p, 1, 30000) <= 0) return false;
        continue;
      }
      return false;
    }
    (*nwrites)++;
    *nbytes += (uint64_t)w;
    size_t left = (size_t)w;
    while (cnt > 0 && left >= iov->iov_len) { left -= iov->iov_len; iov++; cnt--; }
    if (left && cnt > 0) { iov->iov_base = (uint8_t*)iov->iov_base + left; iov->iov_len -= left; }
  }
  return true;
}

// ---- backlogs: the fd sink never waits for a peer ---------------------------------------------
// one write that does not wait: sockets with MSG_DONTWAIT whatever the descriptor's mode, other
// descriptors as their O_NONBLOCK mode says.  Bytes written, 0 = the peer takes nothing now, -1 = error.
ssize_t write_nowait(int fd, const struct iovec* iov, int cnt, bool* is_sock) {
  for (;;) {
    ssize_t w;
    if (*is_sock) {
      struct msghdr mh{};
      mh.msg_iov = const_cast<struct iovec*>(iov); mh.msg_iovlen = (size_t)cnt;
      w = ::sendmsg(fd, &mh, MSG_DONTWAIT | MSG_NOSIGNAL);
      if (w < 0 && errno == ENOTSOCK) { *is_sock = false; continue; }
    } else {
      w = ::writev(fd, iov, cnt);
    }
    if (w >= 0) return w;
    if (errno == EINTR) continue;
    return (errno == EAGAIN || errno == EWOULDBLOCK) ? 0 : -1;
  }
}

void drop_backlog(pcdn_egress* g, pcdn_conn c) {
  if (g->bl.empty() || !g->bl[c]) return;
  Backlog& b = *g->bl[c];
  g->bl_total -= b.pending();
  std::vector<uint8_t>().swap(b.buf);
  b.head = 0;  // stays listed until the list is compacted
}

// a failed write: detach, drop the backlog, report once (sender.rs:24-30)
void fail_conn(pcdn_egress* g, pcdn_conn c) {
  g->fds[c] = -2;
  drop_backlog(g, c);
  std::lock_guard<std::mutex> lk(g->fail_mu);
  g->failed.push_back(c);
}

// writes what the peer takes of a backlog now; false on a write error
bool flush_nowait(pcdn_egress* g, int fd, Backlog& b, uint64_t* nbytes, uint64_t* nwrites) {
  bool is_sock = true;
  while (b.pending()) {
    const struct iovec v{b.buf.data() + b.head, (size_t)b.pending()};
    const ssize_t w = write_nowait(fd, &v, 1, &is_sock);
    if (w < 0) return false;
    if (w == 0) break;
    (*nwrites)++;
    *nbytes += (uint64_t)w;
    b.head += (size_t)w;
    g->bl_total -= (uint64_t)w;
  }
  if (!b.pending()) {
    b.buf.clear(); b.head = 0;
    if (b.buf.capacity() > (1u << 20)) std::vector<uint8_t>().swap(b.buf);
  }
  return true;
}

// copies iov[0..cnt) behind the connection's backlog; false when that would break a budget
bool append_backlog(pcdn_egress* g, pcdn_conn c, const struct iovec* iov, int cnt) {
  uint64_t add = 0;
  for (int i = 0; i < cnt; i++) add += iov[i].iov_len;
  if (!add) return true;
  if (!g->bl[c]) g->bl[c].reset(new Backlog());
  Backlog& b = *g->bl[c];
  if (g->cfg.backlog_bytes_per_conn && b.pending() + add > g->cfg.backlog_bytes_per_conn) return false;
  const uint64_t cap = g->cfg.backlog_bytes_total;
  uint64_t cur = g->bl_total.load();
  do {
    if (cap && cur + add > cap) return false;
  } while (!g->bl_total.compare_exchange_weak(cur, cur + add));
  if (b.head && b.head >= b.buf.size() / 2) { b.buf.erase(b.buf.begin(), b.buf.begin() + (ptrdiff_t)b.head); b.head = 0; }
  const uint64_t before = b.pending();
  try {
    for (int i = 0; i < cnt; i++) {
      const uint8_t* p = (const uint8_t*)iov[i].iov_base;
      b.buf.insert(b.buf.end(), p, p + iov[i].iov_len);
    }
  } catch (const std::bad_alloc&) {  // the bytes that did go in are dropped with the failed connection
    g->bl_total -= add - (b.pending() - before);
    return false;
  }
  if (!b.listed) {
    b.listed = true;
    std::lock_guard<std::mutex> lk(g->bl_mu);
    g->bl_list.push_back(c);
  }
  return true;
}

// the fd sink's write with backlogs: older backlog first (one pass), then the span's records; what
// the peer does not take goes behind the backlog.  false = the connection failed.
bool write_or_queue(pcdn_egress* g, pcdn_conn c, int fd, struct iovec* iov, int cnt, uint64_t* nbytes, uint64_t* nwrites) {
  if (Backlog* b = g->bl[c].get(); b && b->pending()) {
    if (!flush_nowait(g, fd, *b, nbytes, nwrites)) return false;
    if (b->pending()) return append_backlog(g, c, iov, cnt);  // per-connection FIFO (R9)
  }
  bool is_sock = true;
  while (cnt > 0) {
    const int take = std::min(cnt, 1024);  // IOV_MAX
    const ssize_t w = write_nowait(fd, iov, take, &is_sock);
    if (w < 0) return false;
    if (w == 0) return append_backlog(g, c, iov, cnt);
    (*nwrites)++;
    *nbytes += (uint64_t)w;
    size_t left = (size_t)w;
    while (cnt > 0 && left >= iov->iov_len) { left -= iov->iov_len; iov++; cnt--; }
    if (left && cnt > 0) { iov->iov_base = (uint8_t*)iov->iov_base + left; iov->iov_len -= left; }
  }
  return true;
}

// drops bl_list entries whose backlog emptied; only where no drain runs (under pcdn_egress::mu)
void compact_backlog_list(pcdn_egress* g) {
  size_t k = 0;
  for (pcdn_conn c : g->bl_list) {
    Backlog& b = *g->bl[c];
    if (b.pending()) g->bl_list[k++] = c;
    else b.listed = false;
  }
  g->bl_list.resize(k);
}

int fd_sink(void* user, const pcdn_egress_chunk* ch) {
  pcdn_egress* g = (pcdn_egress*)user;
  const uint32_t n = ch->n_spans;
  const uint32_t parts = std::max<uint32_t>(1, std::min<uint32_t>((uint32_t)g->pool->th.size() + 1, n / 64 + 1));
  g->pool->run(parts, [&](uint32_t p) {
    uint32_t lo = (uint32_t)((uint64_t)n * p / parts), hi = (uint32_t)((uint64_t)n * (p + 1) / parts);
    // a connection's two spans of one batch (ring wrap) are adjacent in the table: keep them in one part
    while (lo > 0 && lo < n && ch->spans[lo].conn == ch->spans[lo - 1].conn) lo++;
    while (hi < n && hi > 0 && ch->spans[hi].conn == ch->spans[hi - 1].conn) hi++;
    std::vector<struct iovec> iov;
    uint64_t nb = 0, nw = 0, nrec = 0, una = 0;
    for (uint32_t i = lo; i < hi; i++) {
      const pcdn_span& s = ch->spans[i];
      const int fd = s.conn < g->fds.size() ? g->fds[s.conn] : -1;
      if (fd < 0) { una += fd == -1; continue; }
      // walk the records exactly like the writer task walks its queue: u32 BE length, then the bytes
      // (a reference record: its 4 length bytes, then the L bytes of the shared payload)
      iov.clear();
      const uint8_t* q = ch->data + ch->data_off[i];
      bool ok = true;
      for (uint32_t r = 0; r < s.n_records; r++) {
        if (g->payload && be32(q) == PCDN_REF_MARK) {
          uint64_t off, bid;
          std::memcpy(&off, q + 8, 8); std::memcpy(&bid, q + 16, 8);
          if (bid != g->batch_id) { ok = false; break; }
          iov.push_back({(void*)(q + 4), 4});
          iov.push_back({(void*)(g->payload + off), be32(q + 4)});
          q += PCDN_RECORD_ALIGN;
          continue;
        }
        const uint32_t F = 4 + be32(q);
        if (!iov.empty() && (const uint8_t*)iov.back().iov_base + iov.back().iov_len == q) iov.back().iov_len += F;
        else iov.push_back({(void*)q, F});
        q += (F + PCDN_RECORD_ALIGN - 1) / PCDN_RECORD_ALIGN * PCDN_RECORD_ALIGN;
      }
      if (!ok) { g->bad_ref = true; continue; }   // a record of another batch: nothing of this span is written
      nrec += s.n_records;
      const bool written = g->backlog_on ? write_or_queue(g, s.conn, fd, iov.data(), (int)iov.size(), &nb, &nw)
                                         : write_all(fd, iov.data(), (int)iov.size(), &nb, &nw);
      // Err ⇒ the reference's sender removes the peer (tasks/user/sender.rs:24-30): report it, stop writing to it
      if (!written) fail_conn(g, s.conn);
    }
    g->fd_bytes += nb; g->fd_writes += nw; g->records += nrec; g->unattached += una;
  });
  return g->bad_ref ? 1 : 0;
}

int drain_locked(pcdn_egress* g, uint64_t batch_id, pcdn_egress_sink sink, void* user, pcdn_egress_stats* out) {
  pcdn_engine* e = g->e;
  pcdn_egress_stats st{};
  g->fd_bytes = 0; g->fd_writes = 0; g->unattached = 0; g->records = 0;
  const auto t0 = std::chrono::steady_clock::now();
  const uint32_t nl = (uint32_t)e->shards.size();
  int rc = 0;
  g->payload = nullptr; g->batch_id = batch_id; g->bad_ref = false;
  if (e->delivers_by_ref() && (rc = pcdn_batch_payload(e, batch_id, &g->payload))) return rc;
  if (nl == 1) {
    rc = drain_shard(g, batch_id, 0, sink, user, &st);
  } else {
    // A batch the output pool refused on some shard goes to the sink from no shard: the recovery
    // (release older batches, pcdn_retry_batch, drain again) then hands every shard's share over once.
    for (uint32_t li = 0; li < nl && !rc; li++) {
      pcdn_batch_result res{};
      rc = pcdn_poll_shard(e, batch_id, li, &res, 1);
      if (!rc && res.status == (uint32_t)(-PCDN_EAGAIN))
        rc = fail(PCDN_EAGAIN, "the batch was refused for space in the output pool: release older batches, pcdn_retry_batch, drain again");
    }
    // every GPU has its own PCIe link: the shards drain side by side
    std::vector<pcdn_egress_stats> ps(nl);
    std::vector<int> rcs(nl, 0);
    std::vector<std::string> errs(nl);
    std::vector<std::thread> th;
    for (uint32_t li = 0; li < nl && !rc; li++)
      th.emplace_back([&, li] { rcs[li] = drain_shard(g, batch_id, li, sink, user, &ps[li]); if (rcs[li]) errs[li] = pcdn_last_error(); });
    for (auto& t : th) t.join();
    for (uint32_t li = 0; li < nl; li++) {
      st.bytes += ps[li].bytes; st.spans += ps[li].spans; st.chunks += ps[li].chunks;
      if (rcs[li] && !rc) rc = fail(rcs[li], errs[li]);
    }
  }
  st.seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  st.fd_bytes = g->fd_bytes; st.fd_writes = g->fd_writes; st.unattached_spans = g->unattached; st.records = g->records;
  { std::lock_guard<std::mutex> lk(g->fail_mu); st.failed_conns = g->failed.size(); }
  g->last = st;
  if (out) *out = st;
  return rc;
}

}  // namespace

#define GUARD_BEGIN try {
#define GUARD_END                                                          \
  } catch (const std::bad_alloc&) { return fail(PCDN_ENOMEM, "host allocation failed"); } \
  catch (const std::exception& ex) { return fail(PCDN_EINVAL, ex.what()); }

extern "C" {

int pcdn_egress_create(pcdn_engine* e, const pcdn_egress_config* cfg, pcdn_egress** out) {
  GUARD_BEGIN
  if (!e || !out) return fail(PCDN_EINVAL, "null argument");
  // callers built before the backlog fields pass the shorter struct: no backlog
  constexpr uint32_t kNoBacklogSize = offsetof(pcdn_egress_config, backlog_bytes_per_conn);
  if (cfg && cfg->struct_size != sizeof(pcdn_egress_config) && cfg->struct_size != kNoBacklogSize)
    return fail(PCDN_EINVAL, "pcdn_egress_config.struct_size mismatch (ABI)");
  if (!e->has_device) return fail(PCDN_ENODEV, "host-only engine has nothing to drain");
  pcdn_egress* g = new pcdn_egress();
  g->e = e;
  if (cfg) std::memcpy(&g->cfg, cfg, cfg->struct_size);
  g->cfg.struct_size = sizeof(pcdn_egress_config);
  g->backlog_on = g->cfg.backlog_bytes_per_conn || g->cfg.backlog_bytes_total;
  if (g->backlog_on) g->bl.resize(e->geo.N);
  if (!g->cfg.chunk_bytes) g->cfg.chunk_bytes = 64ull << 20;
  if (!(e->cfg.flags & PCDN_FLAG_OUTPUT_POOL)) g->cfg.chunk_bytes = std::max<uint64_t>(g->cfg.chunk_bytes, 2 * e->cfg.ring_bytes_per_conn);
  g->cfg.chunk_bytes = align_up(g->cfg.chunk_bytes, 4096);
  if (!g->cfg.n_threads) g->cfg.n_threads = std::min(16u, std::max(1u, std::thread::hardware_concurrency()));
  g->pool.reset(new Pool(g->cfg.n_threads));
  g->fds.assign(e->geo.N, -1);
  g->sh.resize(e->shards.size());
  for (uint32_t li = 0; li < e->shards.size(); li++) {
    int rc = init_shard_egress(g, li);
    if (rc) { pcdn_egress_destroy(g); return rc; }
  }
  *out = g;
  return 0;
  GUARD_END
}

void pcdn_egress_destroy(pcdn_egress* g) {
  if (!g) return;
  int prev = -1;
  cudaGetDevice(&prev);
  for (uint32_t li = 0; li < g->sh.size(); li++) free_shard_egress(g, li);
  if (prev >= 0) cudaSetDevice(prev);
  delete g;
}

int pcdn_egress_drain(pcdn_egress* g, uint64_t batch_id, pcdn_egress_sink sink, void* user, pcdn_egress_stats* out) {
  GUARD_BEGIN
  std::lock_guard<std::mutex> lk(g->mu);
  return drain_locked(g, batch_id, sink, user, out);
  GUARD_END
}

int pcdn_egress_attach(pcdn_egress* g, pcdn_conn conn, int fd) {
  std::lock_guard<std::mutex> lk(g->mu);
  if (conn >= g->fds.size() || fd < 0) return fail(PCDN_EINVAL, "connection id or file descriptor out of range");
  drop_backlog(g, conn);  // a reused connection id never inherits the bytes of an earlier peer
  g->fds[conn] = fd;
  return 0;
}
int pcdn_egress_detach(pcdn_egress* g, pcdn_conn conn) {
  std::lock_guard<std::mutex> lk(g->mu);
  if (conn >= g->fds.size()) return fail(PCDN_EINVAL, "connection id out of range");
  drop_backlog(g, conn);
  g->fds[conn] = -1;
  return 0;
}

int pcdn_egress_write_batch(pcdn_egress* g, uint64_t batch_id, pcdn_egress_stats* out) {
  GUARD_BEGIN
  std::lock_guard<std::mutex> lk(g->mu);
  return drain_locked(g, batch_id, fd_sink, g, out);
  GUARD_END
}

int pcdn_egress_failed(pcdn_egress* g, const pcdn_conn** conns, uint32_t* n) {
  GUARD_BEGIN
  std::lock_guard<std::mutex> lk(g->mu);
  std::lock_guard<std::mutex> lk2(g->fail_mu);
  g->failed_out.swap(g->failed);
  g->failed.clear();
  if (conns) *conns = g->failed_out.data();
  if (n) *n = (uint32_t)g->failed_out.size();
  return 0;
  GUARD_END
}

int pcdn_egress_soft_close(pcdn_egress* g, pcdn_conn conn, int* fd_out) {
  GUARD_BEGIN
  std::lock_guard<std::mutex> lk(g->mu);
  if (conn >= g->fds.size()) return fail(PCDN_EINVAL, "connection id out of range");
  // everything handed to the engine before the close still goes out (protocols/mod.rs:287-306):
  // launch the open batch, then write and release every batch in flight, oldest first
  int rc = pcdn_flush(g->e, nullptr);
  if (rc) return rc;
  for (;;) {
    uint64_t b = 0;
    if ((rc = pcdn_next_batch(g->e, &b))) return rc;
    if (!b) break;
    rc = drain_locked(g, b, fd_sink, g, nullptr);
    if (rc == PCDN_EAGAIN) {   // output pool: everything older is released by now, so the refused batch fits
      if ((rc = pcdn_retry_batch(g->e, b))) return rc;
      rc = drain_locked(g, b, fd_sink, g, nullptr);
    }
    if (rc) return rc;
    if ((rc = pcdn_release_batch(g->e, b))) return rc;
  }
  // then the connection's backlog, waiting for the peer as the writer without backlogs does
  if (const int fd = g->fds[conn]; fd >= 0 && g->backlog_on && g->bl[conn]) {
    Backlog& b = *g->bl[conn];
    uint64_t nb = 0, nw = 0;
    bool ok = true;
    while (ok && b.pending()) {
      ok = flush_nowait(g, fd, b, &nb, &nw);
      if (ok && b.pending()) {
        struct pollfd p{fd, POLLOUT, 0};
        const int r = ::poll(&p, 1, 30000);
        ok = r > 0 || (r < 0 && errno == EINTR);
      }
    }
    if (!ok) fail_conn(g, conn);
    compact_backlog_list(g);
  }
  if (fd_out) *fd_out = g->fds[conn];
  g->fds[conn] = -1;
  return 0;
  GUARD_END
}

int pcdn_egress_flush_backlog(pcdn_egress* g, int timeout_ms, uint32_t* n_pending) {
  GUARD_BEGIN
  std::lock_guard<std::mutex> lk(g->mu);
  const auto t_end = std::chrono::steady_clock::now() + std::chrono::milliseconds(std::max(timeout_ms, 0));
  std::vector<struct pollfd> pf;
  for (;;) {
    uint64_t nb = 0, nw = 0;
    for (pcdn_conn c : g->bl_list) {
      Backlog& b = *g->bl[c];
      if (b.pending() && !flush_nowait(g, g->fds[c], b, &nb, &nw)) fail_conn(g, c);
    }
    compact_backlog_list(g);
    if (g->bl_list.empty() || timeout_ms == 0) break;
    int wait = -1;
    if (timeout_ms > 0) {
      const auto left = std::chrono::duration_cast<std::chrono::milliseconds>(t_end - std::chrono::steady_clock::now()).count();
      if (left <= 0) break;
      wait = (int)left;
    }
    pf.clear();
    for (pcdn_conn c : g->bl_list) pf.push_back({g->fds[c], POLLOUT, 0});
    const int r = ::poll(pf.data(), (nfds_t)pf.size(), wait);
    if (r < 0 && errno != EINTR) return fail(PCDN_EINVAL, std::string("poll: ") + std::strerror(errno));
    if (r == 0) break;
  }
  if (n_pending) *n_pending = (uint32_t)g->bl_list.size();
  return 0;
  GUARD_END
}

int pcdn_egress_backlog(pcdn_egress* g, const pcdn_conn** conns, uint32_t* n, uint64_t* bytes) {
  GUARD_BEGIN
  std::lock_guard<std::mutex> lk(g->mu);
  compact_backlog_list(g);
  g->bl_out = g->bl_list;
  std::sort(g->bl_out.begin(), g->bl_out.end());
  if (conns) *conns = g->bl_out.data();
  if (n) *n = (uint32_t)g->bl_out.size();
  if (bytes) *bytes = g->bl_total;
  return 0;
  GUARD_END
}

}  // extern "C"
