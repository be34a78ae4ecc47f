// host_state.cpp — see host_state.h.  Pure host C++ (no CUDA), unit-tested on CPU through the
// C ABI with a host-only engine (pcdn_config.device < 0).
#include "host_state.h"

#include <algorithm>
#include <cstring>

#include "pcdn_fanout.h"

namespace pcdn {

// ============================================================================ HostTables
HostTables::HostTables(const Geometry& geo) : g(geo) {
  sub.assign((size_t)g.T * g.W, 0);
  brk.assign(g.W, 0);
  owner_conn.assign(g.max_owners, PCDN_CONN_NONE);
  cuckoo.assign((size_t)g.nbuckets * 4, CuckooEntry{0, 0, ROUTE_NONE, 0});
  keys.assign((size_t)g.max_keys * g.key_stride, 0);
  f_sub_.assign(sub.size(), 0);
  f_brk_.assign(brk.size(), 0);
  f_owner_.assign(owner_conn.size(), 0);
  f_slot_.assign(cuckoo.size(), 0);
  f_key_.assign(g.max_keys, 0);
}

void HostTables::mark(std::vector<uint32_t>& list, std::vector<uint8_t>& flag, uint32_t idx) {
  if (!flag[idx]) { flag[idx] = 1; list.push_back(idx); }
}

void HostTables::clear_dirty() {
  for (uint32_t i : dirty_sub) f_sub_[i] = 0;
  for (uint32_t i : dirty_brk) f_brk_[i] = 0;
  for (uint32_t i : dirty_owner) f_owner_[i] = 0;
  for (uint32_t i : dirty_slots) f_slot_[i] = 0;
  for (uint32_t i : dirty_keys) f_key_[i] = 0;
  dirty_sub.clear(); dirty_brk.clear(); dirty_owner.clear(); dirty_slots.clear(); dirty_keys.clear();
}

void HostTables::set_bit(uint32_t topic, uint32_t conn, bool on) {
  size_t i = (size_t)topic * g.W + (conn >> 5);
  uint32_t m = 1u << (conn & 31), old = sub[i];
  uint32_t nw = on ? (old | m) : (old & ~m);
  if (nw != old) {
    if (hold) held_sub.emplace((uint32_t)i, old);   // (keeps the value before the first change)
    sub[i] = nw;
    mark(dirty_sub, f_sub_, (uint32_t)i);
  }
}
void HostTables::release_held() {
  for (const auto& h : held_sub) mark(dirty_sub, f_sub_, h.first);
  held_sub.clear();
}
bool HostTables::get_bit(uint32_t topic, uint32_t conn) const {
  return (sub[(size_t)topic * g.W + (conn >> 5)] >> (conn & 31)) & 1u;
}
void HostTables::set_broker(uint32_t conn, bool on) {
  uint32_t i = conn >> 5, m = 1u << (conn & 31), old = brk[i];
  uint32_t nw = on ? (old | m) : (old & ~m);
  if (nw != old) { brk[i] = nw; mark(dirty_brk, f_brk_, i); }
}
void HostTables::set_owner_conn(uint32_t owner, uint32_t conn) {
  if (owner_conn[owner] != conn) { owner_conn[owner] = conn; mark(dirty_owner, f_owner_, owner); }
}

void HostTables::write_slot(uint32_t slot, const CuckooEntry& e) {
  cuckoo[slot] = e;
  mark(dirty_slots, f_slot_, slot);
}

int HostTables::find_slot(const uint8_t* key, uint32_t len, uint64_t h) const {
  uint32_t tag = key_tag(h), b1 = key_bucket(h, g.bucket_mask), b2 = alt_bucket(b1, tag, g.bucket_mask);
  for (uint32_t b : {b1, b2}) {
    for (uint32_t s = 0; s < 4; s++) {
      const CuckooEntry& e = cuckoo[(size_t)b * 4 + s];
      if (e.tag == tag && e.key_len == len &&
          std::memcmp(&keys[(size_t)e.key_slot * g.key_stride], key, len) == 0)
        return (int)(b * 4 + s);
    }
    if (b1 == b2) break;
  }
  return -1;
}

bool HostTables::route_find(const uint8_t* key, uint32_t len, uint32_t* route) const {
  if (len > g.max_key_len) return false;
  int s = find_slot(key, len, key_hash_host(key, len, g.seed));
  if (s < 0) return false;
  *route = cuckoo[s].route;
  return true;
}

int HostTables::place(CuckooEntry e, uint32_t bucket) {
  // random-walk cuckoo insertion; the alternate bucket depends on (bucket, tag) only.  Every eviction
  // is logged so that a walk that ends without a free slot can be undone: a failed insert must not
  // leave some OTHER key (the last victim) without a slot.
  std::vector<std::pair<uint32_t, CuckooEntry>> undo;
  for (int kick = 0; kick < 512; kick++) {
    uint32_t alt = alt_bucket(bucket, e.tag, g.bucket_mask);
    for (uint32_t b : {bucket, alt})
      for (uint32_t s = 0; s < 4; s++)
        if (cuckoo[(size_t)b * 4 + s].tag == 0) { write_slot(b * 4 + s, e); return 0; }
    // evict a pseudo-random victim from the alternate bucket and continue with it
    kick_rng_ = kick_rng_ * 1664525u + 1013904223u;
    uint32_t victim = alt * 4 + ((kick_rng_ >> 16) & 3);
    CuckooEntry v = cuckoo[victim];
    undo.emplace_back(victim, v);
    write_slot(victim, e);
    e = v;
    bucket = alt;  // the victim lived in `alt`; its other choice is alt_bucket(alt, v.tag)
  }
  // Could not place `e`.  Callers size the table at <= 50 % load where this is not reached in
  // practice; put every evicted entry back where it was (newest first) and report it loudly.
  for (size_t i = undo.size(); i-- > 0;) write_slot(undo[i].first, undo[i].second);
  return PCDN_ENOSPC;
}

int HostTables::route_upsert(const uint8_t* key, uint32_t len, uint32_t route) {
  if (len > g.max_key_len) return PCDN_EKEYLEN;
  uint64_t h = key_hash_host(key, len, g.seed);
  int s = find_slot(key, len, h);
  if (s >= 0) {
    if (cuckoo[s].route != route) { CuckooEntry e = cuckoo[s]; e.route = route; write_slot((uint32_t)s, e); }
    return 0;
  }
  if (n_keys_ >= g.max_keys) return PCDN_ENOSPC;
  uint32_t ks;
  if (!free_key_slots_.empty()) { ks = free_key_slots_.back(); free_key_slots_.pop_back(); }
  else ks = next_key_slot_++;
  uint8_t* dst = &keys[(size_t)ks * g.key_stride];
  std::memset(dst, 0, g.key_stride);
  std::memcpy(dst, key, len);
  mark(dirty_keys, f_key_, ks);
  CuckooEntry e{key_tag(h), ks, route, len};
  int rc = place(e, key_bucket(h, g.bucket_mask));
  if (rc == 0) n_keys_++;
  else free_key_slots_.push_back(ks);  // the key slot goes back (its bytes are never referenced)
  return rc;
}

void HostTables::route_erase(const uint8_t* key, uint32_t len) {
  if (len > g.max_key_len) return;
  int s = find_slot(key, len, key_hash_host(key, len, g.seed));
  if (s < 0) return;
  free_key_slots_.push_back(cuckoo[s].key_slot);
  write_slot((uint32_t)s, CuckooEntry{0, 0, ROUTE_NONE, 0});
  n_keys_--;
}

// ============================================================================ BrokerIdent
BrokerIdent BrokerIdent::parse(const char* s) {
  // TryFrom<String> discovery/mod.rs:104-129: split on '/', first two parts
  BrokerIdent b;
  std::string v(s ? s : "");
  size_t a = v.find('/');
  if (a == std::string::npos) { b.pub = v; return b; }
  b.pub = v.substr(0, a);
  size_t c = v.find('/', a + 1);
  b.priv = v.substr(a + 1, c == std::string::npos ? std::string::npos : c - a - 1);
  return b;
}

// ============================================================================ Connections
Connections::Connections(HostTables& t, const char* identity)
    : t_(t), identity_(BrokerIdent::parse(identity)) {
  owners_.push_back(identity_);
  owner_ids_[identity_.str()] = 0;
  conn_kind_.assign(t_.g.N, CONN_FREE);
  topic_key_count_.assign(t_.g.T, 0);
  free_conns_.resize(t_.g.n_shards);
  next_conn_.assign(t_.g.n_shards, 0);
  shard_load_.assign(t_.g.n_shards, 0);
}

void Connections::drain_quarantine() {
  while (!quarantine_.empty() && quarantine_.front().second < oldest_unreleased) {
    const uint32_t c = quarantine_.front().first;
    free_conns_[c / t_.g.shard_N].push_back(c);
    quarantine_.pop_front();
  }
}
bool Connections::id_available() const {
  for (uint32_t s = 0; s < t_.g.n_shards; s++)
    if (!free_conns_[s].empty() || next_conn_[s] < t_.g.shard_max_conns) return true;
  return false;
}
int Connections::alloc_conn(int kind, uint32_t* conn) {
  drain_quarantine();
  // least-loaded shard that can hand out an id (ties: lowest shard index, so every process of a
  // multi-process group that replays the same calls picks the same id)
  int best = -1;
  for (uint32_t s = 0; s < t_.g.n_shards; s++) {
    if (free_conns_[s].empty() && next_conn_[s] >= t_.g.shard_max_conns) continue;
    if (best < 0 || shard_load_[s] < shard_load_[best]) best = (int)s;
  }
  if (best < 0) return quarantine_.empty() ? PCDN_ENOSPC : PCDN_EAGAIN;  // ids come back when older batches are released
  uint32_t c;
  if (!free_conns_[best].empty()) { c = free_conns_[best].back(); free_conns_[best].pop_back(); }
  else c = (uint32_t)best * t_.g.shard_N + next_conn_[best]++;
  shard_load_[best]++;
  conn_kind_[c] = (uint8_t)kind;
  *conn = c;
  return 0;
}
void Connections::free_conn(uint32_t conn) {
  conn_kind_[conn] = CONN_FREE;
  shard_load_[conn / t_.g.shard_N]--;
  if (oldest_unreleased <= fence_now) quarantine_.emplace_back(conn, fence_now);  // an unreleased batch may name it
  else free_conns_[conn / t_.g.shard_N].push_back(conn);
}
int Connections::owner_id(const BrokerIdent& b, uint32_t* id) {
  std::string s = b.str();
  auto it = owner_ids_.find(s);
  if (it != owner_ids_.end()) { *id = it->second; return 0; }
  if (owners_.size() >= t_.g.max_owners) return PCDN_ENOSPC;
  *id = (uint32_t)owners_.size();
  owners_.push_back(b);
  owner_ids_[s] = *id;
  return 0;
}
int Connections::check_topics(const uint16_t* topics, uint32_t n) const {
  for (uint32_t i = 0; i < n; i++)
    if (topics[i] >= t_.g.T) return PCDN_EINVAL;
  return 0;
}
bool Connections::has_broker(const char* ident) const {
  return brokers_.count(BrokerIdent::parse(ident).str()) != 0;
}
uint32_t Connections::user_conn(const std::string& key) const {
  auto u = users_.find(key);
  return u == users_.end() ? PCDN_CONN_NONE : u->second;
}
uint32_t Connections::broker_conn(const char* ident) const {
  auto b = brokers_.find(BrokerIdent::parse(ident).str());
  return b == brokers_.end() ? PCDN_CONN_NONE : b->second.conn;
}

// VersionedMap::modify_local versioned_map.rs:84-113
void Connections::dm_modify_local(const std::string& key, bool has, uint32_t owner) {
  auto it = direct_map_.find(key);
  if (it != direct_map_.end()) {
    if (!locally_modified_.count(key)) it->second.version += 1;
    it->second.has = has;
    it->second.owner = owner;
  } else {
    direct_map_.emplace(key, VV{1, has, owner});
  }
  locally_modified_.insert(key);
}

// What handle_direct_message would resolve for `key` (handler.rs:204-236 + sender.rs:18-21),
// collapsed into one table entry: LOCAL(conn) | REMOTE(owner) | absent.
int Connections::update_route(const std::string& key) {
  const uint8_t* k = (const uint8_t*)key.data();
  uint32_t len = (uint32_t)key.size();
  // keys longer than max_key_len cannot be connected users (add_user refuses them) and have no slot
  // in the key arena: they live in the CRDT map only (sync parity) and never get a device route
  if (len > t_.g.max_key_len) return 0;
  auto it = direct_map_.find(key);
  if (it == direct_map_.end() || !it->second.has) { t_.route_erase(k, len); return 0; }
  if (it->second.owner == 0) {
    auto u = users_.find(key);
    if (u == users_.end()) { t_.route_erase(k, len); return 0; }
    return t_.route_upsert(k, len, u->second);
  }
  return t_.route_upsert(k, len, ROUTE_REMOTE | it->second.owner);
}

static void set_insert(std::vector<uint16_t>& v, uint16_t t, bool* added) {
  auto it = std::lower_bound(v.begin(), v.end(), t);
  if (it != v.end() && *it == t) { *added = false; return; }
  v.insert(it, t);
  *added = true;
}

// Connections::remove_user mod.rs:330-351
int Connections::remove_user(const std::string& key) {
  auto u = users_.find(key);
  auto kt = user_topics_.find(key);
  if (u != users_.end()) {
    uint32_t conn = u->second;
    if (kt != user_topics_.end())
      for (uint16_t t : kt->second) t_.set_bit(t, conn, false);
    free_conn(conn);
    users_.erase(u);
  }
  if (kt != user_topics_.end()) {  // broadcast_map.users.remove_key
    for (uint16_t t : kt->second) topic_key_count_[t]--;
    user_topics_.erase(kt);
  }
  // direct_map.remove_if_equals(key, identity) versioned_map.rs:128-136
  auto d = direct_map_.find(key);
  if (d != direct_map_.end() && d->second.has && d->second.owner == 0) dm_modify_local(key, false, 0);
  return update_route(key);
}

// Connections::add_user mod.rs:278-304
int Connections::add_user(const std::string& key, const uint16_t* topics, uint32_t n, uint32_t* conn) {
  if (key.size() > t_.g.max_key_len) return PCDN_EKEYLEN;
  int rc = check_topics(topics, n);
  if (rc) return rc;
  {  // refuse BEFORE kicking the same-key user when no connection id could be handed out afterwards
    const bool quarantining = oldest_unreleased <= fence_now;
    const bool have = id_available() ||
                      (!quarantine_.empty() && quarantine_.front().second < oldest_unreleased) ||
                      (users_.count(key) && !quarantining);
    if (!have) return (quarantine_.empty() && !users_.count(key)) ? PCDN_ENOSPC : PCDN_EAGAIN;
  }
  remove_user(key);
  uint32_t c;
  if ((rc = alloc_conn(CONN_USER, &c))) return rc;
  users_[key] = c;
  dm_modify_local(key, true, 0);  // direct_map.insert(key, identity)
  auto& set = user_topics_[key];   // associate_key_with_values: entry created even when empty
  for (uint32_t i = 0; i < n; i++) {
    bool added;
    set_insert(set, topics[i], &added);
    if (added) topic_key_count_[topics[i]]++;
    t_.set_bit(topics[i], c, true);
  }
  if ((rc = update_route(key))) {
    // table full: undo so the engine state stays consistent with what we report
    remove_user(key);
    return rc;
  }
  if (conn) *conn = c;
  return 0;
}

// Connections::subscribe_user_to mod.rs:365 → RelationalMap::associate_key_with_values :57-68
int Connections::subscribe_user_to(const std::string& key, const uint16_t* topics, uint32_t n) {
  int rc = check_topics(topics, n);
  if (rc) return rc;
  auto& set = user_topics_[key];
  auto u = users_.find(key);
  for (uint32_t i = 0; i < n; i++) {
    bool added;
    set_insert(set, topics[i], &added);
    if (added) topic_key_count_[topics[i]]++;
    if (u != users_.end()) t_.set_bit(topics[i], u->second, true);
  }
  return 0;
}

// Connections::unsubscribe_user_from mod.rs:383 → dissociate_keys_from_value :71-96
int Connections::unsubscribe_user_from(const std::string& key, const uint16_t* topics, uint32_t n) {
  auto kt = user_topics_.find(key);
  if (kt == user_topics_.end()) return 0;
  auto u = users_.find(key);
  for (uint32_t i = 0; i < n; i++) {
    auto& v = kt->second;
    auto it = std::lower_bound(v.begin(), v.end(), topics[i]);
    if (it != v.end() && *it == topics[i]) {
      v.erase(it);
      topic_key_count_[topics[i]]--;
      if (u != users_.end() && topics[i] < t_.g.T) t_.set_bit(topics[i], u->second, false);
    }
  }
  if (kt->second.empty()) user_topics_.erase(kt);
  return 0;
}

// Connections::remove_broker mod.rs:308-324
int Connections::remove_broker(const char* ident) {
  std::string id = BrokerIdent::parse(ident).str();
  auto b = brokers_.find(id);
  auto kt = broker_topics_.find(id);
  if (b != brokers_.end()) {
    uint32_t conn = b->second.conn;
    if (kt != broker_topics_.end())
      for (uint16_t t : kt->second) t_.set_bit(t, conn, false);
    t_.set_broker(conn, false);
    t_.set_owner_conn(b->second.owner, PCDN_CONN_NONE);
    free_conn(conn);
    brokers_.erase(b);
  }
  if (kt != broker_topics_.end()) broker_topics_.erase(kt);  // broadcast_map.brokers.remove_key
  return 0;
}

// Connections::add_broker mod.rs:252-274
int Connections::add_broker(const char* ident, uint32_t* conn) {
  BrokerIdent bi = BrokerIdent::parse(ident);
  std::string id = bi.str();
  uint32_t owner;
  int rc = owner_id(bi, &owner);
  if (rc) return rc;
  if (owner == 0) return PCDN_EINVAL;  // a broker never connects to itself (heartbeat.rs:66-70)
  {  // refuse BEFORE dropping the existing connection when no id could be handed out afterwards (as add_user)
    const bool quarantining = oldest_unreleased <= fence_now;
    const bool reconnect = brokers_.count(id) != 0;
    const bool have = id_available() ||
                      (!quarantine_.empty() && quarantine_.front().second < oldest_unreleased) ||
                      (reconnect && !quarantining);
    if (!have) return (quarantine_.empty() && !reconnect) ? PCDN_ENOSPC : PCDN_EAGAIN;
  }
  remove_broker(ident);
  uint32_t c;
  if ((rc = alloc_conn(CONN_BROKER, &c))) return rc;
  brokers_[id] = BrokerRec{c, owner, TopicVersionedMap()};  // topic_sync_map: TopicSyncMap::new(0) mod.rs:271
  t_.set_broker(c, true);
  t_.set_owner_conn(owner, c);
  if (conn) *conn = c;
  return 0;
}

// Connections::subscribe_broker_to mod.rs:354
int Connections::subscribe_broker_to(const char* ident, const uint16_t* topics, uint32_t n) {
  int rc = check_topics(topics, n);
  if (rc) return rc;
  std::string id = BrokerIdent::parse(ident).str();
  auto& set = broker_topics_[id];
  auto b = brokers_.find(id);
  for (uint32_t i = 0; i < n; i++) {
    bool added;
    set_insert(set, topics[i], &added);
    if (b != brokers_.end()) t_.set_bit(topics[i], b->second.conn, true);
  }
  return 0;
}

// Connections::unsubscribe_broker_from mod.rs:372
int Connections::unsubscribe_broker_from(const char* ident, const uint16_t* topics, uint32_t n) {
  std::string id = BrokerIdent::parse(ident).str();
  auto kt = broker_topics_.find(id);
  if (kt == broker_topics_.end()) return 0;
  auto b = brokers_.find(id);
  for (uint32_t i = 0; i < n; i++) {
    auto& v = kt->second;
    auto it = std::lower_bound(v.begin(), v.end(), topics[i]);
    if (it != v.end() && *it == topics[i]) {
      v.erase(it);
      if (b != brokers_.end() && topics[i] < t_.g.T) t_.set_bit(topics[i], b->second.conn, false);
    }
  }
  if (kt->second.empty()) broker_topics_.erase(kt);
  return 0;
}

// Connections::apply_user_sync mod.rs:154-162 = VersionedMap::merge versioned_map.rs:202-269,
// then remove_user for every changed key.
int Connections::apply_user_sync(const char* remote_identity, const std::vector<UserSyncEntry>& es) {
  BrokerIdent remote = BrokerIdent::parse(remote_identity);
  bool remote_wins_ties = remote > identity_;
  // Resolve every owner BEFORE touching the map: the only failure that can refuse the merge as a
  // whole (owner table full) must happen while nothing has changed.  The reference's merge cannot
  // fail at all (versioned_map.rs:202-269), so from here on every entry is merged and every changed
  // key gets its remove_user (mod.rs:157-161), whatever happens to an individual device route.
  std::vector<uint32_t> owners(es.size(), 0);
  {
    const size_t owners_before = owners_.size();
    for (size_t i = 0; i < es.size(); i++) {
      if (!es[i].has_owner) continue;
      int rc = owner_id(BrokerIdent::parse(es[i].owner.c_str()), &owners[i]);
      if (rc) {  // undo the owner ids handed out by this call
        while (owners_.size() > owners_before) { owner_ids_.erase(owners_.back().str()); owners_.pop_back(); }
        return rc;
      }
    }
  }
  std::vector<std::string> changed;
  for (size_t i = 0; i < es.size(); i++) {
    const UserSyncEntry& e = es[i];
    const uint32_t owner = owners[i];
    auto it = direct_map_.find(e.key);
    if (it != direct_map_.end()) {
      bool take = e.version > it->second.version ||
                  (e.version == it->second.version && remote_wins_ties);
      if (!take) continue;
      if (e.has_owner) { it->second.has = true; it->second.owner = owner; it->second.version = e.version; }
      else direct_map_.erase(it);
      locally_modified_.erase(e.key);
      changed.push_back(e.key);
    } else if (e.has_owner) {
      direct_map_.emplace(e.key, VV{e.version, true, owner});
      changed.push_back(e.key);
    }
  }
  int rc = 0;
  for (const std::string& k : changed) {
    int r = remove_user(k);  // ends with update_route(k)
    if (r && !rc) rc = r;    // (route table full: the CRDT state is still complete and consistent)
  }
  return rc;
}

// ---- TopicVersionedMap = VersionedMap<Topic, SubscriptionStatus, u32> ---------------------------
void TopicVersionedMap::insert(uint16_t t, uint8_t status) {
  auto it = map.find(t);
  if (it != map.end()) {
    if (!locally_modified.count(t)) it->second.version += 1;
    it->second.status = status;
  } else {
    map.emplace(t, VV{1, status});
  }
  locally_modified.insert(t);
}
void TopicVersionedMap::diff(std::vector<TopicSyncEntry>& out) {
  out.clear();
  std::unordered_set<uint16_t> mod;
  mod.swap(locally_modified);
  for (uint16_t t : mod) {
    auto it = map.find(t);
    if (it == map.end()) continue;
    out.push_back(TopicSyncEntry{t, it->second.status, it->second.version});
    if (it->second.status == 2) map.erase(it);
  }
}
void TopicVersionedMap::full(std::vector<TopicSyncEntry>& out) const {
  out.clear();
  for (auto& kv : map) out.push_back(TopicSyncEntry{kv.first, kv.second.status, kv.second.version});
}
void TopicVersionedMap::merge(uint32_t remote_identity, const std::vector<TopicSyncEntry>& remote,
                              std::vector<std::pair<uint16_t, uint8_t>>& changes) {
  changes.clear();
  for (const TopicSyncEntry& r : remote) {
    auto it = map.find(r.topic);
    if (it != map.end()) {
      const bool take = r.version > it->second.version ||
                        (r.version == it->second.version && remote_identity > conflict_identity);
      if (!take) continue;
      if (r.status != 2) { it->second.status = r.status; it->second.version = r.version; }
      else map.erase(it);
      locally_modified.erase(r.topic);
      changes.emplace_back(r.topic, r.status);
    } else if (r.status != 2) {
      map.emplace(r.topic, VV{r.version, r.status});
      changes.emplace_back(r.topic, r.status);
    }
  }
}

// Connections::get_full_user_sync mod.rs:131-137 (None when empty = empty list)
void Connections::get_full_user_sync(std::vector<UserSyncEntry>& out) const {
  out.clear();
  for (auto& kv : direct_map_)
    out.push_back(UserSyncEntry{kv.first, kv.second.version, kv.second.has, kv.second.has ? owners_[kv.second.owner].str() : ""});
}
// Connections::get_partial_user_sync mod.rs:141-148 = VersionedMap::diff versioned_map.rs:169-195
void Connections::get_partial_user_sync(std::vector<UserSyncEntry>& out) {
  out.clear();
  std::unordered_set<std::string> mod;
  mod.swap(locally_modified_);
  for (const std::string& k : mod) {
    auto it = direct_map_.find(k);
    if (it == direct_map_.end()) continue;
    out.push_back(UserSyncEntry{k, it->second.version, it->second.has, it->second.has ? owners_[it->second.owner].str() : ""});
    if (!it->second.has) direct_map_.erase(it);  // tombstones are dropped once they have been sent
  }
}
// Connections::apply_topic_sync mod.rs:165-191
int Connections::apply_topic_sync(const char* ident, uint32_t remote_identity, const std::vector<TopicSyncEntry>& e) {
  std::string id = BrokerIdent::parse(ident).str();
  auto b = brokers_.find(id);
  if (b == brokers_.end()) { remove_broker(ident); return 0; }
  for (const TopicSyncEntry& x : e)
    if (x.topic >= t_.g.T) return PCDN_EINVAL;
  std::vector<std::pair<uint16_t, uint8_t>> changed;
  b->second.topic_sync_map.merge(remote_identity, e, changed);
  for (auto& c : changed) {
    if (c.second == 0) subscribe_broker_to(ident, &c.first, 1);
    else unsubscribe_broker_from(ident, &c.first, 1);
  }
  return 0;
}
// Connections::get_full_topic_sync mod.rs:194-200
void Connections::get_full_topic_sync(std::vector<TopicSyncEntry>& out) const { topic_sync_map_.full(out); }
// Connections::get_partial_topic_sync mod.rs:205-237
void Connections::get_partial_topic_sync(std::vector<TopicSyncEntry>& out) {
  out.clear();
  std::vector<uint16_t> added, removed;
  for (uint32_t t = 0; t < t_.g.T; t++) {
    const bool now = topic_key_count_[t] != 0, before = previous_subscribed_topics_.count((uint16_t)t) != 0;
    if (now && !before) added.push_back((uint16_t)t);
    if (!now && before) removed.push_back((uint16_t)t);
  }
  if (added.empty() && removed.empty()) return;
  for (uint16_t t : added) { previous_subscribed_topics_.insert(t); topic_sync_map_.insert(t, 0); }
  for (uint16_t t : removed) { previous_subscribed_topics_.erase(t); topic_sync_map_.insert(t, 1); }
  topic_sync_map_.diff(out);
}

// Connections::get_interested_by_topic mod.rs:94-124 on the bitmap mirror
void Connections::interested(const uint16_t* topics, uint32_t n, bool to_users_only,
                             std::vector<uint32_t>& conns) const {
  conns.clear();
  for (uint32_t w = 0; w < t_.g.W; w++) {
    uint32_t m = 0;
    for (uint32_t i = 0; i < n; i++)
      if (topics[i] < t_.g.T) m |= t_.sub[(size_t)topics[i] * t_.g.W + w];
    if (to_users_only) m &= ~t_.brk[w];
    while (m) {
      uint32_t b = (uint32_t)__builtin_ctz(m);
      conns.push_back(w * 32 + b);
      m &= m - 1;
    }
  }
}

int Connections::route(const std::string& key, uint32_t* conn) const {
  uint32_t r;
  *conn = PCDN_CONN_NONE;
  if (!t_.route_find((const uint8_t*)key.data(), (uint32_t)key.size(), &r) || r == ROUTE_NONE) return 0;
  if (r & ROUTE_REMOTE) { *conn = t_.owner_conn[r & ~ROUTE_REMOTE]; return 2; }
  *conn = r;
  return 1;
}

}  // namespace pcdn
