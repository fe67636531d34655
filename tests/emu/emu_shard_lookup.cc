// emu_shard_lookup.cc -- LookupResources on the object-hash sharded store (device.cu Device::shard_lookup_*) under the
// CPU SIMT emulator. TEST INFRASTRUCTURE ONLY (built by tests/emu/emu_shard_lookup.py into its own .so; never part of
// libzgpu.so). The emulator driver emu_main.cc is compiled into this translation unit unchanged: its engine model and
// every emu_* entry point (the sharded check protocol included) come with it. Added here: the round of lookups (begin,
// level expand, candidates, answer keys routed home, final sort and split) over host memory; pointers are those of
// CPU tensors, as in emu_shard_route.
#include "emu_main.cc"

#include <map>
#include <mutex>

namespace {

struct SlState {
  std::vector<uint16_t> res_types;
  std::vector<zg_check> protos;
  std::vector<LookupParam> lp;
  std::vector<uint8_t> home;
  uint64_t cap = 0, n_cand = 0, n_walk = 0;  // n_walk: candidates before the self-membership ones
  unsigned long long words = 0;
  std::vector<unsigned long long> base;  // type_bit_base
  std::vector<uint32_t> visited;
  std::vector<zg_check> cand;
  std::vector<uint8_t> owner;
  std::vector<unsigned long long> counts, keys;
  unsigned long long cand_count = 0;
  uint32_t flags = 0;
};

std::mutex g_mu;
std::map<void*, SlState> g_state;  // one round per emulated engine (ranks run in threads)

SlState& state(void* h) {
  std::lock_guard<std::mutex> g(g_mu);
  return g_state[h];
}

// Snapshot::resources[t]: objects of type t with a non-empty forward row (build.cu gpu_resource_lists), ascending
std::vector<uint32_t> resources(const Emu* e, uint16_t t) {
  std::vector<uint32_t> out;
  const HostSnapshot& h = e->h;
  const uint32_t ncls = h.type_ncls[t];
  if (!ncls) return out;
  for (uint32_t o = 0; o < h.n_objects[t]; ++o) {
    const uint64_t b = h.type_base[t] + uint64_t(o) * ncls;
    if (h.row_ptr[b + ncls] > h.row_ptr[b]) out.push_back(o);
  }
  return out;
}

}  // namespace

extern "C" {

void emu_sl_release(void* h) {
  std::lock_guard<std::mutex> g(g_mu);
  g_state.erase(h);
}

int emu_sl_begin(void* h, const uint16_t* res_types, const zg_check* protos, const uint8_t* home, uint32_t K, uint64_t walk_cap,
                 unsigned long long* seeds) {
  Emu* e = static_cast<Emu*>(h);
  if (!e->published || K == 0 || K > kMaxLookupBatch || walk_cap == 0 || e->shard_count > kMaxRouteDest) return ZG_EINVAL;
  for (uint32_t k = 0; k < K; ++k)
    if (res_types[k] >= e->h.n_objects.size() || protos[k].stype >= e->h.n_objects.size() || home[k] >= e->shard_count) return ZG_EINVAL;
  SlState& s = state(h);
  s = SlState{};
  s.res_types.assign(res_types, res_types + K);
  s.protos.assign(protos, protos + K);
  s.home.assign(home, home + K);
  s.cap = walk_cap;
  s.base.assign(e->h.n_objects.size() + 1, 0);
  for (size_t t = 0; t < e->h.n_objects.size(); ++t) s.base[t + 1] = s.base[t] + ((uint64_t(e->h.n_objects[t]) + 31) & ~31ull);
  s.words = (s.base.back() + 31) / 32 + 4;
  s.visited.assign(s.words * K, 0);
  s.cand.assign(walk_cap + K, zg_check{});
  s.owner.assign(walk_cap + K, 0);
  s.counts.assign(ZG_MAX_DEPTH + 4, 0);
  for (uint32_t i = 0; i < K; ++i) {
    s.lp.push_back(LookupParam{protos[i].subj, res_types[i], protos[i].perm, protos[i].stype, protos[i].srel});
    seeds[i] = (static_cast<unsigned long long>(i) << 48) | (static_cast<unsigned long long>(protos[i].stype) << 32) | protos[i].subj;
  }
  return 0;
}

int emu_sl_expand(void* h, const unsigned long long* front, uint64_t n_in, int level, unsigned long long* next, uint64_t* n_next,
                  int* overflow) {
  Emu* e = static_cast<Emu*>(h);
  SlState& s = state(h);
  *n_next = 0;
  *overflow = 0;
  if (s.lp.empty() || level < 0 || level > ZG_MAX_DEPTH + 1) return ZG_EINVAL;
  if (n_in > s.cap) {
    *overflow = 1;
    return 0;
  }
  if (n_in == 0) return 0;
  static const uint32_t zero = 0;
  s.counts[level] = n_in;
  s.counts[level + 1] = 0;
  MrbfsParams p{};
  p.rrow_ptr = e->h.rrow_ptr.empty() ? &zero : e->h.rrow_ptr.data();
  p.rcol = e->h.rcol.empty() ? &zero : e->h.rcol.data();
  p.prog = e->blob.data();
  p.lk = s.lp.data();
  p.in = front;
  p.out = next;
  p.counts = s.counts.data();
  p.level = level;
  p.cap = s.cap;
  p.visited = s.visited.data();
  p.words = s.words;
  p.type_bit_base = s.base.data();
  p.cand = s.cand.data();
  p.cand_owner = s.owner.data();
  p.cand_count = &s.cand_count;
  p.cand_cap = s.cap;
  p.flags = &s.flags;
  zg_emu::launch(mrbfs_expand_kernel, p, 2, 256, 0);
  *overflow = (s.flags & 16u) ? 1 : 0;
  *n_next = std::min<uint64_t>(s.counts[level + 1], s.cap);
  return 0;
}

int emu_sl_candidates(void* h, int exhaustive, zg_check* items, uint64_t cap, uint64_t* n) {
  Emu* e = static_cast<Emu*>(h);
  SlState& s = state(h);
  *n = 0;
  const size_t K = s.lp.size();
  if (!K) return ZG_EINVAL;
  std::vector<SelfCand> self;
  for (size_t k = 0; k < K; ++k) {
    const zg_check& q = s.protos[k];
    const uint16_t T = s.res_types[k];
    if (q.srel == kNone || q.stype != T || q.subj >= ZG_NO_OBJECT - 1 || q.subj % e->shard_count != e->shard_rank) continue;
    self.push_back(SelfCand{static_cast<uint32_t>(k), 0, q.subj < e->h.n_objects[T] ? s.base[T] + q.subj : ~0ull});
  }
  std::vector<std::vector<uint32_t>> res(K);
  uint64_t need = self.size();
  if (exhaustive) {
    for (size_t k = 0; k < K; ++k) {
      res[k] = resources(e, s.res_types[k]);
      need += res[k].size();
    }
  } else {
    if (s.cand_count > s.cap) return ZG_EINVAL;
    need += s.cand_count;
  }
  if (!items) {
    *n = need;
    return 0;
  }
  if (cap < need) return ZG_E2BIG;
  if (exhaustive) {
    s.cand.assign(std::max<uint64_t>(need, 1), zg_check{});
    s.owner.assign(std::max<uint64_t>(need, 1), 0);
    std::fill(s.visited.begin(), s.visited.end(), 0u);
    uint64_t at = 0;
    struct FillArgs {
      const uint32_t* res;
      unsigned long long n;
      LookupParam l;
      uint32_t k;
      uint32_t* vis;
      unsigned long long bit_base;
      zg_check* cand;
      uint8_t* owner;
    };
    for (size_t k = 0; k < K; ++k) {
      const uint64_t nr = res[k].size();
      if (!nr) continue;
      FillArgs fa{res[k].data(), nr, s.lp[k], static_cast<uint32_t>(k), s.visited.data() + k * s.words, s.base[s.res_types[k]],
                  s.cand.data() + at, s.owner.data() + at};
      zg_emu::launch(+[](const FillArgs& a) { lookup_fill_owned_kernel(a.res, a.n, a.l, a.k, a.vis, a.bit_base, a.cand, a.owner); }, fa,
                     static_cast<unsigned>((nr + 255) / 256), 256, 0);
      at += nr;
    }
    s.cand_count = at;
  }
  s.n_walk = s.cand_count;
  if (!self.empty()) {
    struct SelfArgs {
      const LookupParam* lk;
      const SelfCand* self;
      uint32_t n;
      const uint32_t* vis;
      unsigned long long words;
      zg_check* cand;
      uint8_t* owner;
      unsigned long long* count;
    } sa{s.lp.data(), self.data(), static_cast<uint32_t>(self.size()), s.visited.data(), s.words, s.cand.data(), s.owner.data(), &s.cand_count};
    zg_emu::launch(+[](const SelfArgs& a) { lookup_self_kernel(a.lk, a.self, a.n, a.vis, a.words, a.cand, a.owner, a.count); }, sa, 1,
                   kMaxLookupBatch, 0);
  }
  std::copy(s.cand.begin(), s.cand.begin() + s.cand_count, items);
  s.n_cand = s.cand_count;
  *n = s.cand_count;
  return 0;
}

int emu_sl_route(void* h, const uint8_t* codes, uint64_t n, uint32_t n_dest, unsigned long long* routed, uint64_t* counts) {
  Emu* e = static_cast<Emu*>(h);
  SlState& s = state(h);
  for (uint32_t d = 0; d < n_dest && d < kMaxRouteDest; ++d) counts[d] = 0;
  if (s.lp.empty() || n != s.n_cand || n_dest != e->shard_count) return ZG_EINVAL;
  if (n == 0) return 0;
  s.keys.assign(n, 0);
  std::vector<unsigned long long> per(kMaxLookupBatch, 0);
  unsigned long long n_keys = 0, err_mask = 0;
  struct KeyArgs {
    const zg_check* cand;
    const uint8_t* owner;
    const uint8_t* codes;
    unsigned long long n;
    unsigned long long *keys, *n_keys, *per, *err;
    unsigned long long err_below;
  } ka{s.cand.data(), s.owner.data(), codes, n, s.keys.data(), &n_keys, per.data(), &err_mask, s.n_walk};
  zg_emu::launch(+[](const KeyArgs& a) { lookup_keys_kernel(a.cand, a.owner, a.codes, a.n, a.keys, a.n_keys, a.per, a.err, a.err_below); }, ka,
                 static_cast<unsigned>((n + 255) / 256), 256, 0);
  std::vector<unsigned long long> cnt(kMaxRouteDest, 0), cursor(kMaxRouteDest, 0);
  const KeyHomeOwner own{s.home.data()};
  struct CntArgs {
    const unsigned long long* keys;
    unsigned long long n;
    uint32_t n_dest;
    unsigned long long* counts;
    KeyHomeOwner own;
  } ca{s.keys.data(), n_keys, n_dest, cnt.data(), own};
  zg_emu::launch(+[](const CntArgs& a) { route_count_kernel(a.keys, a.n, a.n_dest, a.counts, a.own); }, ca, 2, 256, 0);
  unsigned long long acc = 0;
  for (uint32_t d = 0; d < n_dest; ++d) {
    counts[d] = cnt[d];
    cursor[d] = acc;
    acc += cnt[d];
  }
  struct ScArgs {
    const unsigned long long* keys;
    unsigned long long n;
    uint32_t n_dest;
    unsigned long long* cursor;
    unsigned long long* routed;
    KeyHomeOwner own;
  } sa{s.keys.data(), n_keys, n_dest, cursor.data(), routed, own};
  zg_emu::launch(+[](const ScArgs& a) { route_scatter_kernel<unsigned long long, KeyHomeOwner, false>(a.keys, a.n, a.n_dest, a.cursor, a.routed, nullptr, a.own); },
                 sa, 2, 256, 0);
  return 0;
}

int emu_sl_finish(void* h, const unsigned long long* keys, uint64_t n, uint32_t* ids, uint64_t* per_lookup, uint64_t* err_mask) {
  SlState& s = state(h);
  *err_mask = 0;
  const size_t K = s.lp.size();
  if (!K) return ZG_EINVAL;
  for (size_t k = 0; k < K; ++k) per_lookup[k] = 0;
  if (n == 0) return 0;
  std::vector<unsigned long long> sorted(keys, keys + n), first(kMaxLookupBatch, 0), end(kMaxLookupBatch, 0);
  std::sort(sorted.begin(), sorted.end());  // sort_u64 over the low kErrKeyBit + 1 bits: the keys have no others
  unsigned long long mask = 0;
  struct SplitArgs {
    const unsigned long long* keys;
    unsigned long long n;
    uint32_t* ids;
    unsigned long long *first, *end, *err;
  } sp{sorted.data(), n, ids, first.data(), end.data(), &mask};
  zg_emu::launch(+[](const SplitArgs& a) { lookup_split_kernel(a.keys, a.n, a.ids, a.first, a.end, a.err); }, sp,
                 static_cast<unsigned>((n + 255) / 256), 256, 0);
  *err_mask = mask;
  for (size_t k = 0; k < K; ++k) per_lookup[k] = end[k] - first[k];
  return 0;
}

}  // extern "C"
