// ORACLE — test infrastructure only.  Nothing under oracle/ is linked into, imported by or
// executed from the product (push-cdn_b200/); only tests/, __graft_entry__.smoke() and bench.py's
// cpu_baseline / --impl reference legs use it, and only as the checker / CPU baseline.
//
// capnp_lite.hpp — encoder/decoder for the cdn-proto wire messages the broker routes.
//
// PARITY UNPINNED: the reference serialises with the third-party crate `capnp` 0.20.6
// (Cargo.lock:799-800, NOT vendored in the reference repository; call sites cdn-proto/src/message.rs:
// 118-119,203,214-228) and its only test at this boundary is a round trip without golden bytes
// (message.rs:397-457).  The layout below is restated from the public Cap'n Proto encoding spec and
// the struct sizes/discriminants in the reference's generated code:
//   Message   1 data word + 1 pointer            cdn-proto/schema/messages_capnp.rs:175
//   Direct    0 data + 2 pointers (recipient, message)              messages_capnp.rs:1438
//   Broadcast 0 data + 2 pointers (topics List(UInt8), message)     messages_capnp.rs:1687
//   union tag u16 @ data offset 0: direct=3 (:277) broadcast=4 (:292) subscribe=5 unsubscribe=6
//   userSync=7 topicSync=8                       cdn-proto/schema/messages.capnp:5-76
// Build order root → variant struct → field0 → field1 (message.rs:151-174); first segment is
// 1024 words (capnp-rust Builder::new_default), an object that does not fit goes to a new segment
// behind a single far pointer + landing pad.  Routing never depends on these bytes being what the
// Rust client would emit: the broker forwards the inbound bytes verbatim (SURVEY Appendix A, R1).
#pragma once
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

namespace capnp_lite {

using Bytes = std::vector<uint8_t>;

enum Kind : int {
  AuthenticateWithKey = 0, AuthenticateWithPermit = 1, AuthenticateResponse = 2,
  Direct = 3, Broadcast = 4, Subscribe = 5, Unsubscribe = 6, UserSync = 7, TopicSync = 8
};

struct Message {
  int kind = -1;
  Bytes topics;     // Broadcast / Subscribe / Unsubscribe (Topic = u8, message.rs:26)
  Bytes recipient;  // Direct
  Bytes payload;    // Direct.message / Broadcast.message / UserSync / TopicSync blob
};

// ---------------------------------------------------------------- encoder
namespace detail {
struct Builder {
  // segments of 64-bit words, little-endian on the wire
  std::vector<std::vector<uint64_t>> segs;
  size_t first_cap = 1024;  // capnp-rust SUGGESTED_FIRST_SEGMENT_WORDS
  Builder() { segs.emplace_back(); }
  size_t cap(size_t seg) const { return seg == 0 ? first_cap : SIZE_MAX; }
  // allocate `n` words in segment `seg` if they fit; returns word index or SIZE_MAX
  size_t try_alloc(size_t seg, size_t n) {
    if (segs[seg].size() + n > cap(seg)) return SIZE_MAX;
    size_t at = segs[seg].size();
    segs[seg].resize(at + n, 0);
    return at;
  }
};
inline uint64_t struct_ptr(int32_t off, uint16_t data, uint16_t ptrs) {
  return (uint64_t)((uint32_t)(off << 2) | 0u) | ((uint64_t)data << 32) | ((uint64_t)ptrs << 48);
}
inline uint64_t list_ptr(int32_t off, uint32_t elem_code, uint32_t count) {
  return (uint64_t)((uint32_t)(off << 2) | 1u) | ((uint64_t)(elem_code | (count << 3)) << 32);
}
inline uint64_t far_ptr(uint32_t pad_word, uint32_t seg) {
  return (uint64_t)((pad_word << 3) | 2u) | ((uint64_t)seg << 32);
}
// write a byte list reachable from pointer slot (pseg, pidx)
inline void set_bytes(Builder& b, size_t pseg, size_t pidx, const uint8_t* p, size_t n) {
  size_t words = (n + 7) / 8;
  size_t at = b.try_alloc(pseg, words);
  if (at != SIZE_MAX) {
    if (n) std::memcpy(b.segs[pseg].data() + at, p, n);
    b.segs[pseg][pidx] = list_ptr((int32_t)(at - pidx - 1), 2, (uint32_t)n);
    return;
  }
  // new segment: landing pad + content, far pointer at the original slot
  b.segs.emplace_back();
  size_t s = b.segs.size() - 1;
  b.segs[s].resize(1 + words, 0);
  if (n) std::memcpy(b.segs[s].data() + 1, p, n);
  b.segs[s][0] = list_ptr(0, 2, (uint32_t)n);
  b.segs[pseg][pidx] = far_ptr(0, (uint32_t)s);
}
inline Bytes finish(const Builder& b) {
  Bytes out;
  uint32_t nseg = (uint32_t)b.segs.size();
  auto put32 = [&](uint32_t v) { for (int i = 0; i < 4; i++) out.push_back((uint8_t)(v >> (8 * i))); };
  put32(nseg - 1);
  for (auto& s : b.segs) put32((uint32_t)s.size());
  if (nseg % 2 == 0) put32(0);  // pad table to 8 bytes
  for (auto& s : b.segs)
    for (uint64_t w : s)
      for (int i = 0; i < 8; i++) out.push_back((uint8_t)(w >> (8 * i)));
  return out;
}
}  // namespace detail

// Message::serialize (cdn-proto/src/message.rs:116-204) for the kinds the broker routes.
inline Bytes serialize(const Message& m) {
  using namespace detail;
  Builder b;
  size_t root = b.try_alloc(0, 1);          // root pointer
  size_t st = b.try_alloc(0, 2);            // Message: 1 data word + 1 pointer
  b.segs[0][root] = struct_ptr((int32_t)(st - root - 1), 1, 1);
  b.segs[0][st] = (uint64_t)(uint16_t)m.kind;  // union discriminant
  size_t p = st + 1;
  switch (m.kind) {
    case Direct:
    case Broadcast: {
      size_t v = b.try_alloc(0, 2);         // variant struct: 0 data + 2 pointers
      b.segs[0][p] = struct_ptr((int32_t)(v - p - 1), 0, 2);
      const Bytes& f0 = (m.kind == Direct) ? m.recipient : m.topics;
      set_bytes(b, 0, v, f0.data(), f0.size());
      set_bytes(b, 0, v + 1, m.payload.data(), m.payload.size());
      break;
    }
    case Subscribe:
    case Unsubscribe:
      set_bytes(b, 0, p, m.topics.data(), m.topics.size());
      break;
    case UserSync:
    case TopicSync:
      set_bytes(b, 0, p, m.payload.data(), m.payload.size());
      break;
    default:
      break;  // auth messages are not on the routed path
  }
  return finish(b);
}

// ---------------------------------------------------------------- decoder
namespace detail {
struct Reader {
  const uint8_t* base = nullptr;
  std::vector<std::pair<size_t, size_t>> seg;  // (byte offset, words)
  bool word(size_t s, size_t idx, uint64_t& w) const {
    if (s >= seg.size() || idx >= seg[s].second) return false;
    std::memcpy(&w, base + seg[s].first + idx * 8, 8);  // little-endian host
    return true;
  }
};
struct Loc { size_t seg, idx; };
// Resolve far pointers: on return `w` is a near pointer and `tgt` is the word its offset is
// relative to (i.e. offset is applied to tgt), or the object start for double-far.
inline bool follow(const Reader& r, Loc at, uint64_t& w, Loc& rel, bool& dbl, Loc& obj) {
  dbl = false;
  if (!r.word(at.seg, at.idx, w)) return false;
  rel = {at.seg, at.idx + 1};
  if ((w & 3) != 2) return true;
  bool two = (w >> 2) & 1;
  size_t pad = (size_t)((uint32_t)w >> 3), s = (size_t)(w >> 32);
  if (!two) {
    uint64_t pw;
    if (!r.word(s, pad, pw)) return false;
    if ((pw & 3) == 2) return false;  // landing pad must not be far
    w = pw;
    rel = {s, pad + 1};
    return true;
  }
  uint64_t f, tag;
  if (!r.word(s, pad, f) || !r.word(s, pad + 1, tag)) return false;
  if ((f & 3) != 2 || ((f >> 2) & 1)) return false;
  dbl = true;
  obj = {(size_t)(f >> 32), (size_t)((uint32_t)f >> 3)};
  w = tag;
  return true;
}
inline bool read_bytes(const Reader& r, Loc at, Bytes& out) {
  uint64_t w; Loc rel, obj; bool dbl;
  if (!follow(r, at, w, rel, dbl, obj)) return false;
  out.clear();
  if (w == 0) return true;  // null pointer = empty default
  if ((w & 3) != 1) return false;
  uint32_t hi = (uint32_t)(w >> 32);
  if ((hi & 7) != 2) return false;  // element size must be BYTE
  size_t n = hi >> 3;
  Loc start = dbl ? obj : Loc{rel.seg, (size_t)((int64_t)rel.idx + ((int32_t)(uint32_t)w >> 2))};
  size_t words = (n + 7) / 8;
  if (start.seg >= r.seg.size() || start.idx > r.seg[start.seg].second ||
      words > r.seg[start.seg].second - start.idx)
    return false;
  const uint8_t* p = r.base + r.seg[start.seg].first + start.idx * 8;
  out.assign(p, p + n);
  return true;
}
}  // namespace detail

// Message::deserialize (cdn-proto/src/message.rs:212-312).  false = Error::Deserialize.
inline bool deserialize(const uint8_t* p, size_t len, Message& m) {
  using namespace detail;
  if (len < 8) return false;
  uint32_t nm1; std::memcpy(&nm1, p, 4);
  uint64_t nseg = (uint64_t)nm1 + 1;
  if (nseg >= 512) return false;  // capnp-rust serialize.rs: "Too many segments"
  size_t table = 4 + 4 * nseg;
  table = (table + 7) & ~(size_t)7;
  if (len < table) return false;
  Reader r; r.base = p;
  size_t off = table;
  for (uint64_t i = 0; i < nseg; i++) {
    uint32_t sz; std::memcpy(&sz, p + 4 + 4 * i, 4);
    if ((uint64_t)sz * 8 > len - off) return false;  // premature end of message
    r.seg.push_back({off, sz});
    off += (size_t)sz * 8;
  }
  // root struct
  uint64_t w; Loc rel, obj; bool dbl;
  if (!follow(r, {0, 0}, w, rel, dbl, obj)) return false;
  m = Message();
  if (w == 0) { m.kind = 0; return true; }  // default struct, tag 0
  if ((w & 3) != 0) return false;
  Loc st = dbl ? obj : Loc{rel.seg, (size_t)((int64_t)rel.idx + ((int32_t)(uint32_t)w >> 2))};
  size_t dw = (w >> 32) & 0xFFFF, pw = (w >> 48) & 0xFFFF;
  if (st.seg >= r.seg.size() || st.idx > r.seg[st.seg].second ||
      dw + pw > r.seg[st.seg].second - st.idx)
    return false;
  uint16_t tag = 0;
  if (dw >= 1) { uint64_t d = 0; r.word(st.seg, st.idx, d); tag = (uint16_t)d; }
  if (tag > 8) return false;  // "message not in schema"
  m.kind = tag;
  bool has_ptr = pw >= 1;
  Loc ptr = {st.seg, st.idx + dw};
  switch (tag) {
    case Direct:
    case Broadcast: {
      if (!has_ptr) return true;  // null → default (empty) variant
      uint64_t vw; Loc vrel, vobj; bool vdbl;
      if (!follow(r, ptr, vw, vrel, vdbl, vobj)) return false;
      if (vw == 0) return true;
      if ((vw & 3) != 0) return false;
      Loc v = vdbl ? vobj : Loc{vrel.seg, (size_t)((int64_t)vrel.idx + ((int32_t)(uint32_t)vw >> 2))};
      size_t vd = (vw >> 32) & 0xFFFF, vp = (vw >> 48) & 0xFFFF;
      if (v.seg >= r.seg.size() || v.idx > r.seg[v.seg].second ||
          vd + vp > r.seg[v.seg].second - v.idx)
        return false;
      Bytes f0, f1;
      if (vp >= 1 && !read_bytes(r, {v.seg, v.idx + vd}, f0)) return false;
      if (vp >= 2 && !read_bytes(r, {v.seg, v.idx + vd + 1}, f1)) return false;
      if (tag == Direct) m.recipient = f0; else m.topics = f0;
      m.payload = f1;
      return true;
    }
    case Subscribe:
    case Unsubscribe:
      return !has_ptr || read_bytes(r, ptr, m.topics);
    case UserSync:
    case TopicSync:
      return !has_ptr || read_bytes(r, ptr, m.payload);
    default:
      return true;  // auth kinds: fields not needed by the broker hot path
  }
}

}  // namespace capnp_lite
