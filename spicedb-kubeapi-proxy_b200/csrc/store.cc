// store.cc -- see store.h.
#include "store.h"

#include <algorithm>
#include <cstring>
#include <numeric>

#include "hash_bytes.h"

namespace zg {

void Store::reset(const Schema* s) {
  schema = s;
  tuples.clear();
  expires.clear();
  objs_.assign(s ? s->types.size() : 0, TypeObjs{});
  obj_cap_.assign(s ? s->types.size() : 0, 0);
  journal.clear();
  journal_ok = false;
  index_.clear();
  indexed_ = true;
  live_ = 0;
  retired_names = 0;
}

void Store::clear_relationships() {
  journal.clear();
  journal_ok = false;
  tuples.clear();
  expires.clear();
  index_.clear();
  indexed_ = true;
  live_ = 0;
}

static inline void rec_read(const std::vector<char>& arena, uint64_t off, uint32_t* id, uint32_t* len) {
  std::memcpy(id, arena.data() + off, 4);
  std::memcpy(len, arena.data() + off + 4, 4);
}

uint32_t Store::TypeObjs::lookup(const char* s, size_t n) const {
  if (table.empty()) return ZG_NO_OBJECT;
  const size_t mask = table.size() - 1;
  for (size_t i = hash_bytes(s, n) & mask;; i = (i + 1) & mask) {
    const uint64_t v = table[i];
    if (!v) return ZG_NO_OBJECT;
    uint32_t id, len;
    rec_read(arena, v - 1, &id, &len);
    if (len == n && std::memcmp(arena.data() + (v - 1) + 8, s, n) == 0) return id;
  }
}

void Store::TypeObjs::place(uint64_t off) {
  uint32_t id, len;
  rec_read(arena, off, &id, &len);
  place(off, hash_bytes(arena.data() + off + 8, len));
}
void Store::TypeObjs::place(uint64_t off, uint64_t hash) {
  const size_t mask = table.size() - 1;
  size_t i = hash & mask;
  while (table[i]) i = (i + 1) & mask;
  table[i] = off + 1;
}

void Store::TypeObjs::insert(uint64_t rec) {
  if ((n_interned + 1) * 2 > table.size()) {  // grow and re-index from the records
    std::vector<uint64_t> old;
    old.swap(table);
    table.assign(old.empty() ? 64 : old.size() * 2, 0);
    for (uint64_t v : old)
      if (v) place(v - 1);
  }
  place(rec);
  ++n_interned;
}

uint32_t Store::intern(int type, const std::string& id) {
  const uint32_t have = objs_[type].lookup(id.data(), id.size());
  if (have != ZG_NO_OBJECT) return have;
  return intern_new(type, id.data(), static_cast<uint32_t>(id.size()), hash_bytes(id.data(), id.size()));
}
void Store::next_ids(int type, uint64_t count, std::vector<uint32_t>* out) const {
  const TypeObjs& t = objs_[type];
  out->clear();
  out->reserve(count);
  for (uint32_t w = t.free_word; t.n_free && w < t.free_bits.size() && out->size() < count; ++w)
    for (uint32_t b = t.free_bits[w]; b && out->size() < count; b &= b - 1)
      out->push_back(w * 32 + static_cast<uint32_t>(__builtin_ctz(b)));
  for (uint32_t id = extent(type); out->size() < count; ++id) out->push_back(id);
}

uint32_t Store::intern_new(int type, const char* s, uint32_t len, uint64_t hash) {
  TypeObjs& t = objs_[type];
  // keep string ids and bulk numeric ids in one id space; the ids of retired names go first, lowest first
  const uint32_t nid = t.n_free ? t.take_free() : std::max<uint32_t>(t.n_ids(), t.n_numeric);
  if (nid >= t.n_ids()) t.rec_of.resize(nid + 1, 0);
  const uint64_t rec = t.arena.size();
  t.arena.resize(rec + 8 + len);
  std::memcpy(t.arena.data() + rec, &nid, 4);
  std::memcpy(t.arena.data() + rec + 4, &len, 4);
  std::memcpy(t.arena.data() + rec + 8, s, len);
  t.rec_of[nid] = rec + 1;
  if ((t.n_interned + 1) * 2 > t.table.size()) {
    t.insert(rec);  // grows the table, re-hashing every record
  } else {
    t.place(rec, hash);
    ++t.n_interned;
  }
  return nid;
}

void Store::import(const zg_tuple* t, const uint32_t* ex, uint64_t n) {
  if (journal_ok && journal.size() + n > kMaxJournal) {  // only a rebuild publishes this many
    journal.clear();
    journal_ok = false;
  }
  if (indexed_) index_.reserve(index_.size() + n);
  tuples.reserve(tuples.size() + n);
  expires.reserve(tuples.capacity());
  for (uint64_t i = 0; i < n; ++i) {
    zg_tuple x = t[i];
    x.flags = 0;
    if (x.srel == kWildcard) x.subj = 0;
    const uint32_t e = ex ? ex[i] : 0;
    if (indexed_) index_.emplace(key_of(x), tuples.size());
    if (journal_ok) journal.push_back(JournalEntry{x, e, kInserted});
    tuples.push_back(x);
    expires.push_back(e);
  }
  live_ += n;
}

bool Store::contains(const zg_tuple& t) {
  ensure_index();
  return index_.count(key_of(t)) != 0;
}

uint32_t Store::find(int type, const std::string& id) const { return find(type, id.data(), id.size()); }
uint32_t Store::find(int type, const char* id, size_t len) const {
  if (type < 0 || type >= static_cast<int>(objs_.size())) return ZG_NO_OBJECT;
  return objs_[type].lookup(id, len);
}
bool Store::name(int type, uint32_t id, std::string_view* out) const {
  if (type < 0 || type >= static_cast<int>(objs_.size())) return false;
  const TypeObjs& t = objs_[type];
  if (id >= t.rec_of.size() || !t.rec_of[id]) return false;  // numeric-only object
  uint32_t rid, len;
  rec_read(t.arena, t.rec_of[id] - 1, &rid, &len);
  if (!len) return false;  // the empty name reads as "no name", as it always did
  *out = std::string_view(t.arena.data() + (t.rec_of[id] - 1) + 8, len);
  return true;
}

bool Store::name_has_prefix(int type, uint32_t id, const std::string& prefix) const {
  std::string_view n;
  return name(type, id, &n) && n.size() >= prefix.size() && std::memcmp(n.data(), prefix.data(), prefix.size()) == 0;
}

std::string Store::validate(const zg_tuple& t, bool has_expiry) const {
  const Schema& sc = *schema;
  if (t.rel >= sc.slots.size() || sc.slots[t.rel].is_perm) return "relationship does not name a relation";
  if (t.stype >= sc.types.size()) return "unknown subject type";
  int k = sc.class_of(t.rel, t.stype, t.srel);
  if (k < 0) {
    const SlotInfo& r = sc.slots[t.rel];
    std::string what = sc.types[t.stype].name;
    if (t.srel == kWildcard) what += ":*";
    else if (t.srel != kNone) what += t.srel < sc.slots.size() ? "#" + sc.slots[t.srel].name : "#?";
    return "subjects of type " + what + " are not allowed on relation " + sc.types[r.type].name + "#" + r.name;
  }
  if (has_expiry && !sc.slots[t.rel].classes[k].expiry)
    return "relation " + sc.types[sc.slots[t.rel].type].name + "#" + sc.slots[t.rel].name +
           " does not allow expiration for this subject type";
  if (t.res == ZG_NO_OBJECT || (t.srel != kWildcard && t.subj == ZG_NO_OBJECT)) return "invalid object id";
  return "";
}

std::string Store::load(const zg_tuple* t, const uint32_t* ex, uint64_t n) {
  // validate per distinct (rel, stype, srel, has_exp) combination: cache the last one
  uint64_t last = ~0ull;
  for (uint64_t i = 0; i < n; ++i) {
    uint64_t sig = (uint64_t(t[i].rel) << 33) | (uint64_t(t[i].stype) << 17) | (uint64_t(t[i].srel) << 1) |
                   (ex && ex[i] ? 1u : 0u);
    if (sig != last || t[i].res == ZG_NO_OBJECT || t[i].subj == ZG_NO_OBJECT) {
      std::string err = validate(t[i], ex && ex[i]);
      if (!err.empty()) return "relationship " + std::to_string(i) + ": " + err;
      last = sig;
    }
  }
  tuples.reserve(tuples.size() + (shard_count > 1 ? n / shard_count + 1 : n));
  expires.reserve(tuples.capacity());
  uint64_t kept = 0;
  for (uint64_t i = 0; i < n; ++i) {
    zg_tuple x = t[i];
    x.flags = 0;
    if (x.srel == kWildcard) x.subj = 0;
    TypeObjs& rt = objs_[schema->slots[x.rel].type];
    if (x.res + 1 > rt.n_numeric) rt.n_numeric = x.res + 1;
    rt.claim(x.res);
    if (x.srel != kWildcard) {
      TypeObjs& st = objs_[x.stype];
      if (x.subj + 1 > st.n_numeric) st.n_numeric = x.subj + 1;
      st.claim(x.subj);
    }
    if (shard_count > 1 && x.res % shard_count != shard_rank) continue;  // another shard owns it
    tuples.push_back(x);
    expires.push_back(ex ? ex[i] : 0);
    ++kept;
  }
  live_ += kept;  // upper bound until duplicates are folded by ensure_index()/build()
  indexed_ = false;
  journal.clear();
  journal_ok = false;  // bulk loads may hold duplicates: only a full build folds them
  return "";
}

void Store::ensure_index() {
  if (indexed_) return;
  index_.clear();
  index_.reserve(tuples.size() * 2);
  live_ = 0;
  for (uint64_t i = 0; i < tuples.size(); ++i) {
    if (tuples[i].flags & 1) continue;
    auto res = index_.emplace(key_of(tuples[i]), i);
    if (!res.second) {  // later TOUCH wins
      tuples[res.first->second].flags |= 1;
      res.first->second = i;
    } else {
      ++live_;
    }
  }
  indexed_ = true;
}

std::string Store::apply(const zg_update* u, uint64_t n, int* code, std::vector<uint8_t>* changed) {
  *code = ZG_EINVAL;
  if (changed) changed->assign(n, 0);
  for (uint64_t i = 0; i < n; ++i) {
    if (u[i].op > ZG_OP_DELETE) return "update " + std::to_string(i) + ": unknown operation";
    if (u[i].op == ZG_OP_DELETE) {
      if (u[i].t.rel >= schema->slots.size() || schema->slots[u[i].t.rel].is_perm) return "update names no relation";
      continue;
    }
    std::string err = validate(u[i].t, u[i].expires_at != 0);
    if (!err.empty()) return "update " + std::to_string(i) + ": " + err;
  }
  ensure_index();
  // CREATE must not collide with an existing relationship or with an earlier update
  for (uint64_t i = 0; i < n; ++i)
    if (u[i].op == ZG_OP_CREATE) {
      zg_tuple t = u[i].t;
      if (index_.count(key_of(t))) {
        *code = ZG_EEXIST;
        return "update " + std::to_string(i) + ": relationship already exists";
      }
    }
  for (uint64_t i = 0; i < n; ++i) {
    zg_tuple t = u[i].t;
    t.flags = 0;
    if (t.srel == kWildcard) t.subj = 0;
    if (shard_count > 1) {  // keep id spaces aligned across shards, store only what this shard owns
      TypeObjs& rt0 = objs_[schema->slots[t.rel].type];
      if (t.res + 1 > rt0.n_numeric) rt0.n_numeric = t.res + 1;
      if (t.srel != kWildcard && t.subj + 1 > objs_[t.stype].n_numeric) objs_[t.stype].n_numeric = t.subj + 1;
      if (t.res % shard_count != shard_rank) continue;
    }
    Key k = key_of(t);
    auto it = index_.find(k);
    if (u[i].op == ZG_OP_DELETE) {
      if (it != index_.end()) {
        tuples[it->second].flags |= 1;
        index_.erase(it);
        --live_;
        if (changed) (*changed)[i] = kDeleted;
        if (journal_ok) journal.push_back(JournalEntry{t, 0, kDeleted});
      }
      continue;
    }
    if (it != index_.end()) {
      if (changed) (*changed)[i] = kTouched;
      if (journal_ok && expires[it->second] != u[i].expires_at) journal.push_back(JournalEntry{t, u[i].expires_at, kTouched});
      expires[it->second] = u[i].expires_at;
      continue;
    }
    if (changed) (*changed)[i] = kInserted;
    if (journal_ok) journal.push_back(JournalEntry{t, u[i].expires_at, kInserted});
    index_.emplace(k, tuples.size());
    tuples.push_back(t);
    expires.push_back(u[i].expires_at);
    ++live_;
    TypeObjs& rt = objs_[schema->slots[t.rel].type];
    if (t.res + 1 > rt.n_numeric) rt.n_numeric = t.res + 1;
    rt.claim(t.res);
    if (t.srel != kWildcard) {
      TypeObjs& st = objs_[t.stype];
      if (t.subj + 1 > st.n_numeric) st.n_numeric = t.subj + 1;
      st.claim(t.subj);
    }
  }
  // compact tombstones when they dominate
  if (tuples.size() > 1024 && live_ * 2 < tuples.size()) {
    size_t w = 0;
    for (size_t i = 0; i < tuples.size(); ++i)
      if (!(tuples[i].flags & 1)) {
        tuples[w] = tuples[i];
        expires[w] = expires[i];
        ++w;
      }
    tuples.resize(w);
    expires.resize(w);
    indexed_ = false;
    ensure_index();
  }
  *code = ZG_OK;
  return "";
}

void Store::match(const Filter& f, uint32_t now, std::vector<uint64_t>* idx) const {
  idx->clear();
  if (f.impossible) return;
  const_cast<Store*>(this)->ensure_index();
  for (uint64_t i = 0; i < tuples.size(); ++i) {
    const zg_tuple& t = tuples[i];
    if (t.flags & 1) continue;
    if (expires[i] != 0 && expires[i] <= now) continue;
    if (f.res_type >= 0 && schema->slots[t.rel].type != f.res_type) continue;
    if (f.has_res && t.res != f.res) continue;
    if (!f.prefix.empty() && !name_has_prefix(schema->slots[t.rel].type, t.res, f.prefix)) continue;
    if (f.rel >= 0 && t.rel != f.rel) continue;
    if (f.subj_type >= 0 && t.stype != f.subj_type) continue;
    if (f.subj_wildcard && t.srel != kWildcard) continue;
    if (f.has_subj && (t.srel == kWildcard || t.subj != f.subj)) continue;
    if (f.has_srel && t.srel != f.srel) continue;
    idx->push_back(i);
  }
}

void Store::page(const Filter& f, uint32_t now, const PageKey* after, uint64_t want, std::vector<uint64_t>* idx) const {
  std::vector<uint64_t> all;
  match(f, now, &all);
  std::vector<std::pair<PageKey, uint64_t>> keys;
  keys.reserve(all.size());
  for (uint64_t i : all) {
    const PageKey k = page_key(*schema, tuples[i]);
    if (!after || *after < k) keys.push_back({k, i});
  }
  const size_t n = static_cast<size_t>(std::min<uint64_t>(want, keys.size()));
  std::partial_sort(keys.begin(), keys.begin() + n, keys.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
  idx->resize(n);
  for (size_t i = 0; i < n; ++i) (*idx)[i] = keys[i].second;
}

bool Store::locate(const zg_tuple* t, uint64_t n, std::vector<uint64_t>* idx) {
  ensure_index();
  idx->resize(n);
  for (uint64_t i = 0; i < n; ++i) {
    auto it = index_.find(key_of(t[i]));
    if (it == index_.end()) return false;
    (*idx)[i] = it->second;
  }
  std::sort(idx->begin(), idx->end());
  return true;
}

void Store::expired(uint32_t before, std::vector<uint64_t>* idx) {
  idx->clear();
  ensure_index();
  for (uint64_t i = 0; i < tuples.size(); ++i)
    if (!(tuples[i].flags & 1) && expires[i] != 0 && expires[i] <= before) idx->push_back(i);
}

void Store::mark(IdBits* bits, int type, uint32_t id) {
  std::vector<uint32_t>& b = (*bits)[type];
  if ((id >> 5) >= b.size()) b.resize((id >> 5) + 1, 0);
  b[id >> 5] |= 1u << (id & 31);
}

void Store::mentioned(IdBits* bits) const {
  bits->assign(objs_.size(), {});
  for (size_t t = 0; t < objs_.size(); ++t)
    (*bits)[t].assign((std::max<uint32_t>(objs_[t].n_ids(), objs_[t].n_numeric) + 31) / 32, 0);
  for (const zg_tuple& t : tuples) {  // a duplicate of a bulk load names the same ids as the copy it folds into
    if (t.flags & 1) continue;
    mark(bits, schema->slots[t.rel].type, t.res);
    if (t.srel != kWildcard) mark(bits, t.stype, t.subj);
  }
}

uint32_t Store::TypeObjs::take_free() {
  while (!free_bits[free_word]) ++free_word;
  const uint32_t b = static_cast<uint32_t>(__builtin_ctz(free_bits[free_word]));
  free_bits[free_word] &= ~(1u << b);
  --n_free;
  return free_word * 32 + b;
}

uint64_t Store::retire(const IdBits& keep) {
  uint64_t total = 0;
  for (size_t ty = 0; ty < objs_.size(); ++ty) {
    TypeObjs& t = objs_[ty];
    const std::vector<uint32_t>* k = ty < keep.size() ? &keep[ty] : nullptr;
    const uint32_t n = t.n_ids();
    t.free_bits.resize((n + 31) / 32, 0);
    uint32_t gone = 0, first_word = ~0u;
    for (uint32_t w = 0; w * 32 < n; ++w) {
      uint32_t named = 0;
      for (uint32_t b = 0; b < 32 && w * 32 + b < n; ++b)
        if (t.rec_of[w * 32 + b]) named |= 1u << b;
      uint32_t drop = named & ~(k && w < k->size() ? (*k)[w] : 0u);
      if (!drop) continue;
      first_word = std::min(first_word, w);
      t.free_bits[w] |= drop;
      for (; drop; drop &= drop - 1) {
        t.rec_of[w * 32 + static_cast<uint32_t>(__builtin_ctz(drop))] = 0;
        ++gone;
      }
    }
    if (!gone) continue;
    // the arena keeps only the records rec_of still points at, in their old order; ids do not move
    std::vector<char> arena;
    arena.reserve(t.arena.size());
    for (uint64_t off = 0; off < t.arena.size();) {
      uint32_t id, len;
      rec_read(t.arena, off, &id, &len);
      if (t.rec_of[id] == off + 1) {
        t.rec_of[id] = arena.size() + 1;
        arena.insert(arena.end(), t.arena.begin() + off, t.arena.begin() + off + 8 + len);
      }
      off += 8 + len;
    }
    t.arena.swap(arena);
    t.n_interned -= gone;
    size_t cap = 64;
    while (cap < uint64_t(t.n_interned) * 2 + 2) cap *= 2;
    t.table.assign(cap, 0);
    for (uint64_t off = 0; off < t.arena.size();) {
      t.place(off);
      uint32_t len;
      std::memcpy(&len, t.arena.data() + off + 4, 4);
      off += 8 + len;
    }
    t.n_free += gone;
    t.free_word = std::min(t.free_word, first_word);
    total += gone;
  }
  retired_names += total;
  return total;
}

Store::NameCounts Store::name_counts() const {
  NameCounts c;
  for (const TypeObjs& t : objs_) {
    c.named += t.n_interned;
    c.free_ids += t.n_free;
    c.extent += std::max<uint32_t>(t.n_ids(), t.n_numeric);
    c.arena_bytes += t.arena.size();
  }
  return c;
}

HostSnapshot Store::layout() const {
  const Schema& sc = *schema;
  HostSnapshot h;
  const size_t nt = sc.types.size();
  h.n_objects.resize(nt);
  obj_cap_.resize(nt, 0);
  for (size_t t = 0; t < nt; ++t) {
    const uint32_t need = std::max<uint32_t>(objs_[t].n_ids(), objs_[t].n_numeric);
    if (need > obj_cap_[t]) {
      const uint64_t want = uint64_t(need) + need / 8 + 4096;
      obj_cap_[t] = static_cast<uint32_t>(std::min<uint64_t>(want, 0xFFFFFFF0ull));
    }
    h.n_objects[t] = obj_cap_[t];
  }

  // row table: per resource type, objects x (all classes of all relations of the type)
  h.type_ncls.assign(nt, 0);
  for (int rs : sc.rel_slots) h.type_ncls[sc.slots[rs].type] += static_cast<uint32_t>(sc.slots[rs].classes.size());
  h.type_base.assign(nt + 1, 0);
  for (size_t t = 0; t < nt; ++t) h.type_base[t + 1] = h.type_base[t] + uint64_t(h.n_objects[t]) * h.type_ncls[t];
  h.pool = h.type_base[nt];
  std::vector<uint32_t> type_used(nt, 0);
  uint16_t cls_begin = 0;
  for (int rs : sc.rel_slots) {
    const SlotInfo& s = sc.slots[rs];
    DRel r{};
    r.row_base = h.type_base[s.type] + type_used[s.type];
    r.nres = h.n_objects[s.type];
    r.ncls = static_cast<uint16_t>(s.classes.size());
    r.stride = h.type_ncls[s.type];
    r.cls_begin = cls_begin;
    cls_begin = static_cast<uint16_t>(cls_begin + r.ncls);
    type_used[s.type] += r.ncls;
    h.rels.push_back(r);
  }
  // reverse CSR: one row per (SUBJECT object, class). All classes of one subject type are
  // interleaved per subject (row = rrow_base + subject * rstride), classes whose probes may be
  // answered from the subject's reverse rows (CF_INVERT) first: a check's admission reads every
  // offset of its subject from one or two sectors, and the subject's entries are contiguous in
  // rcol. A wildcard class has a single row of its own.
  h.cls = sc.d_cls;
  h.rpool = 0;
  for (size_t t = 0; t < nt; ++t) {
    std::vector<size_t> order;
    for (int pass = 0; pass < 2; ++pass)
      for (size_t c = 0; c < h.cls.size(); ++c)
        if (h.cls[c].stype == t && h.cls[c].sslot != kWildcard && ((h.cls[c].flags & CF_INVERT) != 0) == (pass == 0))
          order.push_back(c);
    for (size_t k = 0; k < order.size(); ++k) {
      DCls& c = h.cls[order[k]];
      c.rrow_base = h.rpool + k;
      c.rstride = static_cast<uint16_t>(order.size());
      c.nsubj = h.n_objects[t];
    }
    h.rpool += uint64_t(order.size()) * h.n_objects[t];
  }
  for (auto& c : h.cls) {
    if (c.sslot == kWildcard) {
      c.rrow_base = h.rpool;
      c.rstride = 0;
      c.nsubj = 1;
      h.rpool += 1;
    }
    c.flags |= CF_EMPTY;  // cleared by the builder for every class that has a relationship
  }
  return h;
}

bool Store::layout_stable() const {
  if (obj_cap_.size() != objs_.size()) return false;
  for (size_t t = 0; t < objs_.size(); ++t)
    if (std::max<uint32_t>(objs_[t].n_ids(), objs_[t].n_numeric) > obj_cap_[t]) return false;
  return true;
}

HostSnapshot Store::build(uint32_t owner_rank, uint32_t owner_count) const {
  const Schema& sc = *schema;
  HostSnapshot h = layout();
  const size_t nt = sc.types.size();
  const uint64_t pool = h.pool;
  h.row_ptr.assign(pool + 1, 0);
  const bool with_exp = sc.has_expiry;

  // class lookup table per data relation
  auto row_index = [&](const zg_tuple& t) -> uint64_t {
    const DRel& r = h.rels[sc.slots[t.rel].rel_index];
    int k = sc.class_of(t.rel, t.stype, t.srel);
    return r.row_base + uint64_t(t.res) * r.stride + static_cast<uint64_t>(k);
  };

  std::vector<std::vector<uint8_t>> seen(nt);
  for (size_t t = 0; t < nt; ++t) seen[t].assign(h.n_objects[t], 0);
  auto skip = [&](const zg_tuple& t) { return (t.flags & 1) || (owner_count > 1 && t.res % owner_count != owner_rank); };
  uint64_t n_live = 0;
  for (size_t i = 0; i < tuples.size(); ++i) {
    const zg_tuple& t = tuples[i];
    if (skip(t)) continue;
    ++h.row_ptr[row_index(t) + 1];
    seen[sc.slots[t.rel].type][t.res] = 1;
    ++n_live;
  }
  for (uint64_t i = 0; i < pool; ++i) h.row_ptr[i + 1] += h.row_ptr[i];
  if (n_live >= 0xFFFFFFF0ull) {
    h.err = "more than 2^32 relationships in one snapshot";
    return h;
  }
  h.col.resize(n_live);
  if (with_exp) h.exp.resize(n_live);
  {
    std::vector<uint32_t> cur(h.row_ptr.begin(), h.row_ptr.end() - 1);
    for (size_t i = 0; i < tuples.size(); ++i) {
      const zg_tuple& t = tuples[i];
      if (skip(t)) continue;
      uint32_t pos = cur[row_index(t)]++;
      h.col[pos] = t.srel == kWildcard ? 0u : t.subj;
      if (with_exp) h.exp[pos] = expires[i];
    }
  }
  // sort each (object, class) row; fold duplicates (bulk loads are TOUCH: last wins)
  bool dup = false;
  std::vector<std::pair<uint32_t, uint32_t>> tmp;
  for (uint64_t r = 0; r < pool; ++r) {
    uint32_t b = h.row_ptr[r], e = h.row_ptr[r + 1];
    if (e - b < 2) continue;
    if (!with_exp) {
      std::sort(h.col.begin() + b, h.col.begin() + e);
    } else {
      tmp.resize(e - b);
      for (uint32_t i = b; i < e; ++i) tmp[i - b] = {h.col[i], h.exp[i]};
      std::stable_sort(tmp.begin(), tmp.end(), [](const auto& x, const auto& y) { return x.first < y.first; });
      for (uint32_t i = b; i < e; ++i) {
        h.col[i] = tmp[i - b].first;
        h.exp[i] = tmp[i - b].second;
      }
    }
    for (uint32_t i = b + 1; i < e && !dup; ++i) dup = h.col[i] == h.col[i - 1];
  }
  if (dup) {
    std::vector<uint32_t> nrow(pool + 1, 0);
    uint32_t w = 0;
    for (uint64_t r = 0; r < pool; ++r) {
      uint32_t b = h.row_ptr[r], e = h.row_ptr[r + 1];
      nrow[r] = w;
      for (uint32_t i = b; i < e; ++i) {
        if (i + 1 < e && h.col[i + 1] == h.col[i]) continue;  // keep the last of a run
        h.col[w] = h.col[i];
        if (with_exp) h.exp[w] = h.exp[i];
        ++w;
      }
    }
    nrow[pool] = w;
    h.row_ptr.swap(nrow);
    h.col.resize(w);
    if (with_exp) h.exp.resize(w);
  }
  h.n_tuples = h.col.size();

  // ---- reverse CSR (subject -> resources), per edge class; built from the deduplicated
  // forward rows in ascending resource order, so every reverse row comes out sorted
  const uint64_t rpool = h.rpool;
  h.rrow_ptr.assign(rpool + 1, 0);
  h.rcol.resize(h.col.size());
  for (int pass = 0; pass < 2; ++pass) {
    std::vector<uint32_t> cur;
    if (pass == 1) {
      for (uint64_t i = 0; i < rpool; ++i) h.rrow_ptr[i + 1] += h.rrow_ptr[i];
      cur.assign(h.rrow_ptr.begin(), h.rrow_ptr.end() - 1);
    }
    for (const DRel& r : h.rels)
      for (uint32_t res = 0; res < r.nres; ++res)
        for (uint32_t k = 0; k < r.ncls; ++k) {
          const uint64_t idx = r.row_base + uint64_t(res) * r.stride + k;
          const uint32_t b = h.row_ptr[idx], e = h.row_ptr[idx + 1];
          if (b == e) continue;
          DCls& c = h.cls[r.cls_begin + k];
          c.flags &= static_cast<uint16_t>(~CF_EMPTY);
          for (uint32_t i = b; i < e; ++i) {
            const uint64_t ridx = c.rrow_base + (c.sslot == kWildcard ? 0ull : uint64_t(h.col[i]) * c.rstride);
            if (pass == 0) ++h.rrow_ptr[ridx + 1];
            else h.rcol[cur[ridx]++] = res;
          }
        }
  }
  h.resources.resize(nt);
  for (size_t t = 0; t < nt; ++t)
    for (uint32_t i = 0; i < seen[t].size(); ++i)
      if (seen[t][i]) h.resources[t].push_back(i);
  return h;
}

}  // namespace zg
