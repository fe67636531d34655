// store.h -- host side of the relationship store: object interning, the mutable
// relationship set (what WriteRelationships / DeleteRelationships act on,
// pkg/authz/distributedtx/activity.go:54-76) and the CSR snapshot builder whose
// output the engine uploads to HBM.
#pragma once
#include <algorithm>
#include <cstdint>
#include <string>
#include <string_view>
#include <unordered_map>
#include <vector>

#include "../../include/zgpu.h"
#include "schema.h"

namespace zg {

struct Key {
  uint64_t hi, lo;  // hi = rel<<32 | stype<<16 | srel ; lo = res<<32 | subj
  bool operator==(const Key& o) const { return hi == o.hi && lo == o.lo; }
};
struct KeyHash {
  size_t operator()(const Key& k) const {
    uint64_t x = k.hi * 0x9E3779B97F4A7C15ull ^ (k.lo + 0xD6E8FEB86659FD93ull);
    x ^= x >> 32;
    x *= 0xD6E8FEB86659FD93ull;
    x ^= x >> 29;
    return static_cast<size_t>(x);
  }
};
inline Key key_of(const zg_tuple& t) {
  return Key{(uint64_t(t.rel) << 32) | (uint64_t(t.stype) << 16) | t.srel,
             (uint64_t(t.res) << 32) | (t.srel == kWildcard ? 0u : t.subj)};
}

// The order of pages (zg_read_relationships_page): K = (resource type, resource, class position, subject), a wildcard
// relationship's subject 0. It depends on the schema and the ids alone, so every engine kind and both paths agree.
struct PageKey {
  uint32_t type, res, pos, subj;
  bool operator<(const PageKey& o) const {
    if (type != o.type) return type < o.type;
    if (res != o.res) return res < o.res;
    if (pos != o.pos) return pos < o.pos;
    return subj < o.subj;
  }
};

// The class position of the relationships (rel_slot, stype, srel): where Store::layout puts their rows in the forward
// block of their resource type. It depends on the schema alone. -1 when the schema has no such class.
inline int page_class_pos(const Schema& sc, int rel_slot, uint16_t stype, uint16_t srel) {
  const int k = sc.class_of(rel_slot, stype, srel);
  if (k < 0) return -1;
  int pos = k;
  for (int rs : sc.rel_slots) {
    if (rs == rel_slot) return pos;
    if (sc.slots[rs].type == sc.slots[rel_slot].type) pos += static_cast<int>(sc.slots[rs].classes.size());
  }
  return -1;
}

inline PageKey page_key(const Schema& sc, const zg_tuple& t) {
  return PageKey{sc.slots[t.rel].type, t.res, static_cast<uint32_t>(page_class_pos(sc, t.rel, t.stype, t.srel)),
                 t.srel == kWildcard ? 0u : t.subj};
}

// CSR snapshot in host memory, ready to upload. Layout: DESIGN.md "Data layout in HBM".
struct HostSnapshot {
  std::vector<uint32_t> row_ptr;  // pool: per data relation, nres x ncls offsets, +1 sentinel
  std::vector<uint32_t> col;      // subject object ids, sorted within (object, class)
  std::vector<uint32_t> exp;      // parallel to col when the schema uses expiration, else empty
  std::vector<DRel> rels;
  std::vector<DCls> cls;          // schema classes + rrow_base / CF_EMPTY for this snapshot
  std::vector<uint32_t> rrow_ptr; // reverse CSR: per class, one row per SUBJECT object (+1 sentinel)
  std::vector<uint32_t> rcol;     // resource object ids, ascending within a row
  std::vector<std::vector<uint32_t>> resources;  // per type: ids that are the resource of >= 1 relationship
  std::vector<uint32_t> n_objects;               // per type
  uint64_t n_tuples = 0;
  uint64_t pool = 0, rpool = 0;            // entries of row_ptr / rrow_ptr (each has +1 sentinel)
  std::vector<uint64_t> type_base;         // per type: first row_ptr index of its objects
  std::vector<uint32_t> type_ncls;         // per type: row stride (classes of all its relations)
  std::string err;  // non-empty: build failed
};

class Store {
 public:
  void reset(const Schema* s);
  // Drops every relationship; interned object names (and therefore ids) stay.
  void clear_relationships();

  uint32_t intern(int type, const std::string& id);
  uint32_t find(int type, const std::string& id) const;  // ZG_NO_OBJECT
  uint32_t find(int type, const char* id, size_t len) const;  // no temporary string: the check-ingress path
  // false for a numeric-only object (bulk loads) or an id out of range
  bool name(int type, uint32_t id, std::string_view* out) const;
  // Read-only view of a type's interned names, for the device mirror (ingress.cuh): the records
  // [u32 id][u32 len][bytes] back to back (appended to; rewritten only by retire() and reset) and how many there are.
  size_t n_types() const { return objs_.size(); }
  const std::vector<char>& name_arena(int type) const { return objs_[type].arena; }
  uint32_t n_interned(int type) const { return objs_[type].n_interned; }

  // ---- retiring names no relationship mentions (zg_retire_unused_names) ----
  // Per type, one bit per id: set where a live or expired relationship of the store names the id as its resource or
  // its subject (what Device::scan_mentions reads from a snapshot of this store). Bitmaps cover the id extent.
  using IdBits = std::vector<std::vector<uint32_t>>;
  void mentioned(IdBits* bits) const;
  static void mark(IdBits* bits, int type, uint32_t id);
  // Retires every name whose bit in `keep` is clear (bits past a bitmap's end are clear): the record leaves the
  // type's arena, which is rewritten with the kept records (ids unchanged) and its table rebuilt; the id goes on the
  // type's free list, which intern() hands out lowest first. Numeric-only ids are never touched. Returns how many.
  uint64_t retire(const IdBits& keep);
  uint64_t retired_names = 0;  // since reset()
  struct NameCounts {
    uint64_t named = 0, free_ids = 0, extent = 0, arena_bytes = 0;
  };
  NameCounts name_counts() const;
  uint32_t capacity(int type) const { return type >= 0 && type < static_cast<int>(obj_cap_.size()) ? obj_cap_[type] : 0; }

  // ---- importing named relationships (zg_import_relationships) ----
  // The id space of a type: ids below it are named or used by a bulk load; interning extends it.
  uint32_t extent(int type) const { return std::max<uint32_t>(objs_[type].n_ids(), objs_[type].n_numeric); }
  // The ids that interning `count` new names of `type` hands out, in order: free ids lowest first, then the extent.
  // Changes nothing.
  void next_ids(int type, uint64_t count, std::vector<uint32_t>* out) const;
  // Interns a name known not to be interned, whose hash_bytes() is `hash` (computed on the device): the id intern()
  // would give it. Returns the id.
  uint32_t intern_new(int type, const char* s, uint32_t len, uint64_t hash);
  // Appends n relationships known to be valid and new (no duplicate among them or in the store), whose names are
  // interned. A current relationship index stays current; the journal records them while it can.
  void import(const zg_tuple* t, const uint32_t* expires, uint64_t n);
  // true when the store holds a live relationship with t's key; builds the index when a bulk load left it behind
  bool contains(const zg_tuple& t);
  // the most changes the journal holds for an incremental publish (Device::publish_delta); more rebuild
  static constexpr size_t kMaxJournal = 1u << 16;

  // Returns "" or an error message; `code` receives the ZG_* code.
  std::string validate(const zg_tuple& t, bool has_expiry) const;
  std::string load(const zg_tuple* t, const uint32_t* expires, uint64_t n);
  // `changed` (optional, n entries): nonzero where the update took effect (a DELETE of a relationship that
  // does not exist changes nothing; TOUCH and CREATE always count): kTouched = the relationship existed
  // (only its expiration may differ), kInserted, kDeleted.
  enum : uint8_t { kUnchanged = 0, kTouched = 1, kInserted = 2, kDeleted = 3 };
  std::string apply(const zg_update* u, uint64_t n, int* code, std::vector<uint8_t>* changed = nullptr);

  // Journal of what apply() changed since journal_clear(): what an incremental publish merges into the
  // device snapshot instead of rebuilding it (build.cu gpu_apply_delta). journal_ok turns false when
  // something the journal cannot express happened (bulk load, clear, re-layout).
  struct JournalEntry {
    zg_tuple t;
    uint32_t expires;
    uint8_t kind;  // kTouched / kInserted / kDeleted
  };
  std::vector<JournalEntry> journal;
  bool journal_ok = false;
  void journal_clear() {
    journal.clear();
    journal_ok = true;
  }

  // Live relationships matching a filter (unset field = -1 / ZG_NO_OBJECT-1 sentinel via has_*).
  struct Filter {
    int res_type = -1;
    bool has_res = false;
    uint32_t res = 0;
    int rel = -1;  // slot
    int subj_type = -1;
    bool has_subj = false;
    uint32_t subj = 0;
    bool subj_wildcard = false;
    bool has_srel = false;
    uint16_t srel = kNone;
    bool impossible = false;  // names an object/relation that does not exist
    // optional_resource_id_prefix: only resources whose interned name starts with these bytes (empty = unset)
    std::string prefix;
  };
  // true when (type, id) has an interned name that starts with `prefix` (byte-wise, case-sensitive)
  bool name_has_prefix(int type, uint32_t id, const std::string& prefix) const;
  void match(const Filter& f, uint32_t now, std::vector<uint64_t>* idx) const;
  // The host path of a page: the first `want` relationships match() lists whose key follows *after (nullptr: from
  // the start), in K order (PageKey), as positions in `tuples`.
  void page(const Filter& f, uint32_t now, const PageKey* after, uint64_t want, std::vector<uint64_t>* idx) const;
  // Where the n live relationships t[] sit in `tuples`, ascending: the order match() lists them in. Builds the
  // relationship index when a bulk load left it behind. false when one of them is not in the store.
  bool locate(const zg_tuple* t, uint64_t n, std::vector<uint64_t>* idx);
  // Where the live relationships whose expiration is set and <= before sit in `tuples`, ascending: what
  // zg_collect_expired removes. Folds the duplicates of bulk loads first, as match() does.
  void expired(uint32_t before, std::vector<uint64_t>* idx);

  // Sizes and bases only (n_objects, rels, cls with rrow_base / nsubj and CF_EMPTY set on every
  // class): what both the host builder and the GPU builder (build.cu) start from.
  // Object counts are CAPACITIES: they grow in steps (1/8 + 4096 beyond what is needed) and never shrink, so
  // that relationships on newly created objects -- the proxy's common write -- do not move any row table.
  HostSnapshot layout() const;
  // true when layout() would still return the capacities it returned last time
  bool layout_stable() const;
  // owner filter (rank, count): only the relationships whose resource id % count == rank, with the capacities of the
  // whole store -- one shard of a sharded handle, whose store holds every shard's relationships. count = 1: all.
  HostSnapshot build(uint32_t owner_rank = 0, uint32_t owner_count = 1) const;
  uint64_t size() const { return live_; }

  const Schema* schema = nullptr;
  // object-hash sharding: relationships whose resource id % shard_count != shard_rank are dropped
  // (object counts still follow every relationship seen, so ids mean the same on all shards)
  uint32_t shard_count = 1, shard_rank = 0;
  std::vector<zg_tuple> tuples;  // flags bit0 = dead (tombstone)
  std::vector<uint32_t> expires; // parallel to tuples (always sized like tuples)

 private:
  void ensure_index();
  // Interned names of one type. Each name lives once, in `arena`, as a record [u32 id][u32 len][bytes];
  // `table` is an open-addressing index over the records (slot = record offset + 1, 0 = empty, power-of-two
  // size, load <= 1/2), so a lookup hashes the caller's bytes in place and touches two cache lines on a hit:
  // the slot and the record. `rec_of` maps an id back to its record (0 = no name) for the output paths.
  struct TypeObjs {
    std::vector<char> arena;
    std::vector<uint64_t> table;
    std::vector<uint64_t> rec_of;
    uint32_t n_interned = 0;
    uint32_t n_numeric = 0;  // max numeric id seen in bulk loads + 1
    // ids of retired names that no relationship has named since: one bit per id below n_ids()
    std::vector<uint32_t> free_bits;
    uint32_t n_free = 0, free_word = 0;  // free_word: no free id lies in an earlier word
    uint32_t lookup(const char* s, size_t n) const;
    void insert(uint64_t rec);  // record offset
    void place(uint64_t rec);   // into a table with room
    void place(uint64_t rec, uint64_t hash);
    uint32_t n_ids() const { return static_cast<uint32_t>(rec_of.size()); }
    uint32_t take_free();  // the lowest free id, off the list
    // a relationship names `id` directly (bulk load, raw update): it is no longer free
    void claim(uint32_t id) {
      if (n_free && (id >> 5) < free_bits.size() && (free_bits[id >> 5] >> (id & 31) & 1u)) {
        free_bits[id >> 5] &= ~(1u << (id & 31));
        --n_free;
      }
    }
  };
  std::vector<TypeObjs> objs_;
  mutable std::vector<uint32_t> obj_cap_;  // per type: capacity handed out by the last layout()
  std::unordered_map<Key, uint64_t, KeyHash> index_;
  bool indexed_ = true;  // index_ covers every live tuple
  uint64_t live_ = 0;
};

}  // namespace zg
