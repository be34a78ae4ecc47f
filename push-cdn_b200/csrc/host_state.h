// host_state.h — host-side mirror of the broker's routing state.
//
// `Connections` restates cdn-broker/src/connections/mod.rs:40-388 (with RelationalMap
// broadcast/relational_map.rs:13-116 and VersionedMap versioned_map.rs:39-270 folded in) but keeps
// its results in the layout the GPU kernels read: a topic→connection subscription bitmap, a broker
// mask, an owner→connection table and a cuckoo hash from user public key to route.  `HostTables`
// owns those arrays and remembers which words/slots changed since the last upload, so that a state
// call costs O(1) host work and a few scattered device words (R12 ordering: the journal is applied
// on the engine stream before the next batch's kernels).
#pragma once
#include <cstdint>
#include <deque>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

#include "hash.h"

namespace pcdn {

struct Geometry {
  // Connection shards (SURVEY 8e): the id space is n_shards contiguous ranges of shard_N ids, range s
  // = the connections whose rings live on shard s's GPU; ids [s*shard_N, s*shard_N + shard_max_conns)
  // are usable.  A single-GPU engine is one shard.
  uint32_t n_shards = 1;
  uint32_t shard_N = 0;          // per-shard id range: shard_max_conns rounded up to a multiple of 8192
  uint32_t shard_max_conns = 0;  // usable connection ids per shard (pcdn_config.max_conns)
  uint32_t max_conns = 0;   // exclusive upper bound of the usable connection ids (all shards)
  uint32_t N = 0;           // n_shards * shard_N (a multiple of 8192 = 256 bitmap words)
  uint32_t W = 0;           // N / 32 bitmap words per topic row
  uint32_t T = 0;           // topic rows
  uint32_t max_keys = 0;
  uint32_t max_key_len = 0;
  uint32_t key_stride = 0;  // bytes per key-arena slot (multiple of 16)
  uint32_t nbuckets = 0;    // power of two, 4 slots each
  uint32_t bucket_mask = 0;
  uint32_t max_owners = 0;
  uint64_t seed = 0;
};

enum { CONN_FREE = 0, CONN_USER = 1, CONN_BROKER = 2 };

class HostTables {
 public:
  explicit HostTables(const Geometry& g);
  Geometry g;
  std::vector<uint32_t> sub;         // [T][W]
  std::vector<uint32_t> brk;         // [W]
  std::vector<uint32_t> owner_conn;  // [max_owners]
  std::vector<CuckooEntry> cuckoo;   // [nbuckets*4]
  std::vector<uint8_t> keys;         // [max_keys][key_stride]

  // dirty sets since the last take_*()
  std::vector<uint32_t> dirty_sub, dirty_brk, dirty_owner, dirty_slots, dirty_keys;

  // In-batch subscription events (PCDN_FLAG_INBATCH_SUBSCRIBE): while `hold` is set, set_bit keeps the
  // value a bitmap word had before its first change.  The device must keep that value while the batch
  // that holds the events runs (its match replays the events per message); the held words' current
  // values go up with the upload after it (release_held).
  bool hold = false;
  std::unordered_map<uint32_t, uint32_t> held_sub;   // word index → value before the open batch's events
  uint32_t sub_upload(uint32_t i) const {             // what the next upload writes for dirty word i
    auto it = held_sub.find(i);
    return it == held_sub.end() ? sub[i] : it->second;
  }
  void release_held();

  void set_bit(uint32_t topic, uint32_t conn, bool on);
  bool get_bit(uint32_t topic, uint32_t conn) const;
  void set_broker(uint32_t conn, bool on);
  void set_owner_conn(uint32_t owner, uint32_t conn);
  // cuckoo: returns 0, PCDN_ENOSPC or PCDN_EKEYLEN
  int route_upsert(const uint8_t* key, uint32_t len, uint32_t route);
  void route_erase(const uint8_t* key, uint32_t len);
  bool route_find(const uint8_t* key, uint32_t len, uint32_t* route) const;
  uint32_t n_keys() const { return n_keys_; }
  void clear_dirty();

 private:
  std::vector<uint8_t> f_sub_, f_brk_, f_owner_, f_slot_, f_key_;
  std::vector<uint32_t> free_key_slots_;
  uint32_t next_key_slot_ = 0, n_keys_ = 0;
  uint32_t kick_rng_ = 0x9E3779B9u;
  void mark(std::vector<uint32_t>& list, std::vector<uint8_t>& flag, uint32_t idx);
  int find_slot(const uint8_t* key, uint32_t len, uint64_t h) const;  // slot index or -1
  int place(CuckooEntry e, uint32_t bucket);                          // with eviction
  void write_slot(uint32_t slot, const CuckooEntry& e);
};

// BrokerIdentifier (cdn-proto/src/discovery/mod.rs:80-129): "public/private", ordered as the tuple
struct BrokerIdent {
  std::string pub, priv;
  static BrokerIdent parse(const char* s);
  std::string str() const { return pub + "/" + priv; }
  bool operator>(const BrokerIdent& o) const { return pub != o.pub ? pub > o.pub : priv > o.priv; }
};

struct UserSyncEntry {
  std::string key;
  uint64_t version;
  bool has_owner;
  std::string owner;
};

// one entry of a TopicSyncMap = VersionedMap<Topic, SubscriptionStatus, u32> (broadcast/mod.rs:19-25)
struct TopicSyncEntry {
  uint16_t topic;
  uint8_t status;    // 0 Subscribed, 1 Unsubscribed, 2 tombstone (value None)
  uint64_t version;
};

// VersionedMap<Topic, SubscriptionStatus, u32> (versioned_map.rs:39-270), small and dense
struct TopicVersionedMap {
  struct VV { uint64_t version; uint8_t status; };  // status 2 = None
  std::unordered_map<uint16_t, VV> map;
  std::unordered_set<uint16_t> locally_modified;
  uint32_t conflict_identity = 0;
  void insert(uint16_t t, uint8_t status);                                  // modify_local :84-113
  void diff(std::vector<TopicSyncEntry>& out);                              // :169-195
  void full(std::vector<TopicSyncEntry>& out) const;
  // merge :202-269 → changed (topic, new status or 2)
  void merge(uint32_t remote_identity, const std::vector<TopicSyncEntry>& remote,
             std::vector<std::pair<uint16_t, uint8_t>>& changes);
};

class Connections {
 public:
  Connections(HostTables& t, const char* identity);

  // -- the reference's mutation API (connections/mod.rs) ---------------------------------------
  int add_user(const std::string& key, const uint16_t* topics, uint32_t n, uint32_t* conn);  // :278
  int remove_user(const std::string& key);                                                   // :330
  int subscribe_user_to(const std::string& key, const uint16_t* topics, uint32_t n);         // :365
  int unsubscribe_user_from(const std::string& key, const uint16_t* topics, uint32_t n);     // :383
  int add_broker(const char* ident, uint32_t* conn);                                         // :252
  int remove_broker(const char* ident);                                                      // :308
  int subscribe_broker_to(const char* ident, const uint16_t* topics, uint32_t n);            // :354
  int unsubscribe_broker_from(const char* ident, const uint16_t* topics, uint32_t n);        // :372
  int apply_user_sync(const char* remote_identity, const std::vector<UserSyncEntry>& e);     // :154
  // -- inter-broker sync (SURVEY 8f-4): what the sync task sends / receives -----------------------
  void get_full_user_sync(std::vector<UserSyncEntry>& out) const;                             // :131
  void get_partial_user_sync(std::vector<UserSyncEntry>& out);                                // :141 (direct_map.diff())
  int apply_topic_sync(const char* ident, uint32_t remote_identity, const std::vector<TopicSyncEntry>& e);  // :165
  void get_full_topic_sync(std::vector<TopicSyncEntry>& out) const;                           // :194
  void get_partial_topic_sync(std::vector<TopicSyncEntry>& out);                              // :205

  // -- connection-id quarantine ------------------------------------------------------------------
  // Spans of an unreleased batch name connections by id.  An id freed by remove_user / a kick /
  // remove_broker is therefore not handed out again until every batch launched before the removal
  // has been released (the analogue of the reference dropping a Connection only after its queued
  // Bytes are gone, protocols/mod.rs:287-306).  The engine sets both values before each state call.
  uint64_t fence_now = 0;                  // id of the newest launched batch
  uint64_t oldest_unreleased = ~0ull;      // id of the oldest batch not yet released (~0: none)

  // -- lookups on the mirror (tests / debug; the data path does these on the GPU) --------------
  void interested(const uint16_t* topics, uint32_t n, bool to_users_only,
                  std::vector<uint32_t>& conns) const;                                       // :94
  // 0 none, 1 local user, 2 remote broker (conn may be NONE)
  int route(const std::string& key, uint32_t* conn) const;                                   // :69,:84,:74
  uint32_t num_users() const { return (uint32_t)users_.size(); }
  uint32_t num_brokers() const { return (uint32_t)brokers_.size(); }
  uint32_t shard_load(uint32_t shard) const { return shard < shard_load_.size() ? shard_load_[shard] : 0; }
  bool has_user(const std::string& key) const { return users_.count(key) != 0; }
  bool has_broker(const char* ident) const;
  uint32_t user_conn(const std::string& key) const;   // PCDN_CONN_NONE when the user is not connected here
  uint32_t broker_conn(const char* ident) const;      // PCDN_CONN_NONE when the broker is not connected

 private:
  struct VV { uint64_t version; bool has; uint32_t owner; };  // VersionedValue<BrokerIdentifier>
  struct BrokerRec { uint32_t conn; uint32_t owner; TopicVersionedMap topic_sync_map; };  // Broker mod.rs:34-38
  HostTables& t_;
  BrokerIdent identity_;
  std::unordered_map<std::string, uint32_t> users_;                         // users :45
  std::unordered_map<std::string, BrokerRec> brokers_;                      // brokers :47
  std::unordered_map<std::string, VV> direct_map_;                          // direct_map :50
  std::unordered_set<std::string> locally_modified_;                        // versioned_map.rs:47
  std::unordered_map<std::string, std::vector<uint16_t>> user_topics_;      // broadcast_map.users key_to_values
  std::unordered_map<std::string, std::vector<uint16_t>> broker_topics_;    // broadcast_map.brokers key_to_values
  std::unordered_map<std::string, uint32_t> owner_ids_;                     // identifier → owner index (0 = self)
  std::vector<BrokerIdent> owners_;
  std::vector<uint32_t> topic_key_count_;   // |value_to_keys[t]| of broadcast_map.users (keys, connected or not)
  TopicVersionedMap topic_sync_map_;        // broadcast_map.topic_sync_map
  std::unordered_set<uint16_t> previous_subscribed_topics_;
  std::vector<uint8_t> conn_kind_;
  // connection ids are handed out per shard, to the least-loaded shard that has one (the reference's
  // marshal hands a user to the least-loaded broker, cdn-proto/src/connection/auth/marshal.rs:108-118)
  std::vector<std::vector<uint32_t>> free_conns_;   // [shard] freed ids, LIFO
  std::vector<uint32_t> next_conn_;                 // [shard] next never-used local id
  std::vector<uint32_t> shard_load_;                // [shard] ids in use
  std::deque<std::pair<uint32_t, uint64_t>> quarantine_;  // (conn, fence): reusable once oldest_unreleased > fence

  bool id_available() const;   // some shard can hand out an id right now (quarantine already drained)
  void drain_quarantine();
  int alloc_conn(int kind, uint32_t* conn);
  void free_conn(uint32_t conn);
  int owner_id(const BrokerIdent& b, uint32_t* id);
  int update_route(const std::string& key);
  void dm_modify_local(const std::string& key, bool has, uint32_t owner);   // versioned_map.rs:84-113
  int check_topics(const uint16_t* topics, uint32_t n) const;
};

}  // namespace pcdn
