// emu_shard_subjects.cc -- LookupSubjects on the object-hash sharded store (device.cu Device::shard_subjects_* and
// shard_pass_nowild_dev) under the CPU SIMT emulator. TEST INFRASTRUCTURE ONLY (built by tests/emu/emu_shard_subjects.py
// into its own .so; never part of libzgpu.so). emu_subjects.cc is compiled into this translation unit unchanged: it
// brings the emulator driver emu_main.cc (the engine model and every emu_* entry point, the sharded check protocol
// included) and a pass with KParams::no_wildcards. Added here: the sharded pass with no_wildcards and the round of
// lookups (begin, expand and route to the owners, admission, candidates, verdicts, no-wildcards items, answer keys
// routed home, final sort and split) over host memory; pointers are those of CPU tensors, as in emu_shard_route.
#include "emu_subjects.cc"

#include <map>
#include <mutex>

namespace {

struct SsState {
  std::vector<SubjectsParam> lp;
  std::vector<uint8_t> home;
  uint64_t cap = 0, include = 0, n_cand = 0, n_nw = 0;
  unsigned long long words = 0;
  std::vector<unsigned long long> base;  // type_bit_base
  std::vector<FwdClass> fwd;
  std::vector<uint32_t> type_off, visited;
  std::vector<zg_check> probes, cand, nw;
  std::vector<uint8_t> probe_owner, owner, nw_owner;
  std::vector<unsigned long long> out, keys;
  unsigned long long out_count = 0, cand_count = 0, n_keys = 0;
  uint32_t flags = 0;
};

std::mutex g_mu;
std::map<void*, SsState> g_state;  // one round per emulated engine (ranks run in threads)

SsState& state(void* h) {
  std::lock_guard<std::mutex> g(g_mu);
  return g_state[h];
}

SsWalkParams walk_params(Emu* e, SsState& s) {
  static const uint32_t zero = 0;
  SsWalkParams p{};
  p.row_ptr = e->h.row_ptr.empty() ? &zero : e->h.row_ptr.data();
  p.col = e->h.col.empty() ? &zero : e->h.col.data();
  p.fwd = s.fwd.data();
  p.type_off = s.type_off.data();
  p.mask = e->sc.fwd_mask.data();
  p.mask_words = e->sc.fwd_mask_words;
  p.shard_rank = e->shard_rank;
  p.shard_count = e->shard_count;
  p.lk = s.lp.data();
  p.visited = s.visited.data();
  p.words = s.words;
  p.type_bit_base = s.base.data();
  p.flags = &s.flags;
  return p;
}

// device.cu route_ over host memory, for 8-byte entries with an owner functor
template <class Owner>
void route(const unsigned long long* items, uint64_t n, uint32_t n_dest, Owner own, unsigned long long* routed, uint64_t* counts) {
  std::vector<unsigned long long> cnt(kMaxRouteDest, 0), cursor(kMaxRouteDest, 0);
  struct CntArgs {
    const unsigned long long* items;
    unsigned long long n;
    uint32_t n_dest;
    unsigned long long* counts;
    Owner own;
  } ca{items, n, n_dest, cnt.data(), own};
  zg_emu::launch(+[](const CntArgs& a) { route_count_kernel(a.items, a.n, a.n_dest, a.counts, a.own); }, ca, 2, 256, 0);
  unsigned long long acc = 0;
  for (uint32_t d = 0; d < n_dest; ++d) {
    counts[d] = cnt[d];
    cursor[d] = acc;
    acc += cnt[d];
  }
  struct ScArgs {
    const unsigned long long* items;
    unsigned long long n;
    uint32_t n_dest;
    unsigned long long* cursor;
    unsigned long long* routed;
    Owner own;
  } sa{items, n, n_dest, cursor.data(), routed, own};
  zg_emu::launch(+[](const ScArgs& a) { route_scatter_kernel<unsigned long long, Owner, false>(a.items, a.n, a.n_dest, a.cursor, a.routed, nullptr, a.own); },
                 sa, 2, 256, 0);
}

struct KeyArgs {
  const zg_check* cand;
  const uint8_t* owner;
  const uint8_t* codes;
  unsigned long long n, granted, failed, include;
  unsigned long long *keys, *n_keys;
  zg_check* nw;
  uint8_t* nw_owner;
  unsigned long long* n_nw;
};
void keys(const KeyArgs& ka) {
  zg_emu::launch(+[](const KeyArgs& a) { ss_keys_kernel(a.cand, a.owner, a.codes, a.n, a.granted, a.failed, a.include, a.keys, a.n_keys, a.nw, a.nw_owner, a.n_nw); },
                 ka, static_cast<unsigned>((ka.n + 255) / 256), 256, 0);
}

}  // namespace

extern "C" {

void emu_ss_release(void* h) {
  std::lock_guard<std::mutex> g(g_mu);
  g_state.erase(h);
}

// emu_shard_pass with KParams::no_wildcards (device.cu shard_pass_nowild_dev)
int emu_ss_pass_nowild(void* h, const zg_check* queries, uint64_t n, int level, const EmuOpts* o, uint64_t* n_sub) {
  Emu* e = static_cast<Emu*>(h);
  if (!e->published) return -1;
  if (e->levels.size() <= static_cast<size_t>(level)) e->levels.resize(level + 1);
  ShardLevel& L = e->levels[level];
  L.nq = n;
  L.nsub = 0;
  *n_sub = 0;
  if (n == 0) return 0;
  L.q.assign(queries, queries + n);
  L.val.assign(n * e->sc.max_leaves + 4, 0);
  L.raised.assign(o->subq_cap, zg_check{});
  L.parent.assign(o->subq_cap, 0);
  uint64_t ns = 0;
  run_pass_ls(e, *o, L.q.data(), n, L.val.data(), nullptr, level == 0, L.raised.data(), L.parent.data(), &ns, false, true);
  if (ns > o->subq_cap) return -3;
  L.nsub = ns;
  *n_sub = ns;
  return 0;
}

int emu_ss_admit(void* h, const unsigned long long* in, uint64_t n_in, unsigned long long* next, uint64_t* n_next) {
  Emu* e = static_cast<Emu*>(h);
  SsState& s = state(h);
  *n_next = 0;
  if (s.lp.empty()) return ZG_EINVAL;
  if (n_in == 0) return 0;
  unsigned long long admitted = 0;
  SsWalkParams p = walk_params(e, s);
  p.in = in;
  p.n_in = n_in;
  p.out = next;
  p.out_count = &admitted;
  p.cap = s.cap;
  p.cand = s.cand.data();
  p.cand_owner = s.owner.data();
  p.cand_count = &s.cand_count;
  p.cand_cap = s.cap + s.probes.size();
  zg_emu::launch(ss_admit_kernel, p, static_cast<unsigned>((n_in + 255) / 256), 256, 0);
  *n_next = std::min<uint64_t>(admitted, s.cap);
  return 0;
}

int emu_ss_begin(void* h, const uint16_t* res_types, const zg_check* reqs, const uint32_t* options, const uint8_t* home, uint32_t K,
                 uint64_t walk_cap, unsigned long long* front, uint64_t* n_front) {
  Emu* e = static_cast<Emu*>(h);
  *n_front = 0;
  if (!e->published || K == 0 || K > kMaxLookupBatch || walk_cap == 0 || e->shard_count > kMaxRouteDest) return ZG_EINVAL;
  for (uint32_t k = 0; k < K; ++k)
    if (res_types[k] >= e->h.n_objects.size() || reqs[k].stype >= e->h.n_objects.size() || home[k] >= e->shard_count ||
        reqs[k].perm >= e->sc.slots.size() || e->sc.slots[reqs[k].perm].type != res_types[k])
      return ZG_EINVAL;
  SsState& s = state(h);
  s = SsState{};
  s.home.assign(home, home + K);
  s.cap = walk_cap;
  s.base.assign(e->h.n_objects.size() + 1, 0);
  for (size_t t = 0; t < e->h.n_objects.size(); ++t) s.base[t + 1] = s.base[t] + ((uint64_t(e->h.n_objects[t]) + 31) & ~31ull);
  s.words = (s.base.back() + 31) / 32 + 4;
  s.visited.assign(s.words * K, 0);
  e->sc.forward_tables(e->h.rels, &s.fwd, &s.type_off);
  s.cand.assign(walk_cap + K, zg_check{});
  s.owner.assign(walk_cap + K, 0);
  s.out.assign(std::max<uint64_t>(walk_cap, K), 0);
  std::vector<unsigned long long> seeds;
  for (uint32_t k = 0; k < K; ++k) {
    const zg_check& q = reqs[k];
    s.lp.push_back(SubjectsParam{q.res, res_types[k], q.perm, q.stype, q.srel});
    if (options[k] == ZG_WILDCARDS_INCLUDE) s.include |= 1ull << k;
    if (q.res >= e->h.n_objects[res_types[k]] || q.res % e->shard_count != e->shard_rank) continue;
    zg_check probe{};
    probe.res = q.res;
    probe.subj = ZG_NO_OBJECT - 1;
    probe.perm = q.perm;
    probe.stype = q.stype;
    probe.srel = q.srel;
    s.cand[s.probes.size()] = probe;
    s.owner[s.probes.size()] = static_cast<uint8_t>(k);
    s.probes.push_back(probe);
    s.probe_owner.push_back(static_cast<uint8_t>(k));
    seeds.push_back((static_cast<unsigned long long>(k) << 48) | (static_cast<unsigned long long>(res_types[k]) << 32) | q.res);
  }
  s.cand_count = s.probes.size();
  return emu_ss_admit(h, seeds.data(), seeds.size(), front, n_front);
}

int emu_ss_expand(void* h, const unsigned long long* front, uint64_t n_in, uint32_t n_dest, unsigned long long* routed, uint64_t* counts,
                  int* overflow) {
  Emu* e = static_cast<Emu*>(h);
  SsState& s = state(h);
  *overflow = 0;
  for (uint32_t d = 0; d < n_dest && d < kMaxRouteDest; ++d) counts[d] = 0;
  if (s.lp.empty() || n_dest != e->shard_count || n_in > s.cap) return ZG_EINVAL;
  s.out_count = 0;
  if (n_in) {
    SsWalkParams p = walk_params(e, s);
    p.in = front;
    p.n_in = n_in;
    p.out = s.out.data();
    p.out_count = &s.out_count;
    p.cap = s.cap;
    zg_emu::launch(ss_expand_kernel, p, 2, 256, 0);
  }
  if (s.flags & 16u) {
    *overflow = 1;
    return 0;
  }
  if (s.out_count) route(s.out.data(), s.out_count, n_dest, EntryOwner{}, routed, counts);
  return 0;
}

int emu_ss_candidates(void* h, int exhaustive, zg_check* items, uint64_t cap, uint64_t* n) {
  Emu* e = static_cast<Emu*>(h);
  SsState& s = state(h);
  *n = 0;
  const size_t K = s.lp.size();
  if (!K) return ZG_EINVAL;
  std::vector<uint64_t> owned(K, 0);
  uint64_t need = s.probes.size();
  if (exhaustive) {
    for (size_t k = 0; k < K; ++k) {
      const uint64_t no = e->h.n_objects[s.lp[k].stype];
      owned[k] = no > e->shard_rank ? (no - e->shard_rank - 1) / e->shard_count + 1 : 0;
      need += owned[k];
    }
  } else {
    if (s.cand_count > s.cap + s.probes.size()) return ZG_EINVAL;
    need = s.cand_count;
  }
  if (!items) {
    *n = need;
    return 0;
  }
  if (cap < need) return ZG_E2BIG;
  if (exhaustive) {
    s.cand.assign(std::max<uint64_t>(need, 1), zg_check{});
    s.owner.assign(std::max<uint64_t>(need, 1), 0);
    std::copy(s.probes.begin(), s.probes.end(), s.cand.begin());
    std::copy(s.probe_owner.begin(), s.probe_owner.end(), s.owner.begin());
    uint64_t at = s.probes.size();
    struct FillArgs {
      SubjectsParam l;
      uint32_t k;
      unsigned long long n;
      uint32_t rank, count;
      zg_check* cand;
      uint8_t* owner;
    };
    for (size_t k = 0; k < K; ++k) {
      if (!owned[k]) continue;
      FillArgs fa{s.lp[k], static_cast<uint32_t>(k), owned[k], e->shard_rank, e->shard_count, s.cand.data() + at, s.owner.data() + at};
      zg_emu::launch(+[](const FillArgs& a) { ss_fill_owned_kernel(a.l, a.k, a.n, a.rank, a.count, a.cand, a.owner); }, fa,
                     static_cast<unsigned>((owned[k] + 255) / 256), 256, 0);
      at += owned[k];
    }
  }
  std::copy(s.cand.begin(), s.cand.begin() + need, items);
  s.n_cand = need;
  *n = need;
  return 0;
}

int emu_ss_verdicts(void* h, const uint8_t* codes, uint64_t n, uint64_t* granted, uint64_t* failed) {
  SsState& s = state(h);
  *granted = *failed = 0;
  if (s.lp.empty() || n != s.n_cand) return ZG_EINVAL;
  if (n == 0) return 0;
  unsigned long long g = 0, f = 0;
  struct VArgs {
    const zg_check* cand;
    const uint8_t* owner;
    const uint8_t* codes;
    unsigned long long n;
    unsigned long long *g, *f;
  } va{s.cand.data(), s.owner.data(), codes, n, &g, &f};
  zg_emu::launch(+[](const VArgs& a) { ss_verdict_kernel(a.cand, a.owner, a.codes, a.n, a.g, a.f); }, va,
                 static_cast<unsigned>((n + 255) / 256), 256, 0);
  *granted = g;
  *failed = f;
  return 0;
}

int emu_ss_nowild(void* h, const uint8_t* codes, uint64_t n, uint64_t granted, uint64_t failed, zg_check* items, uint64_t cap,
                  uint64_t* n_nw) {
  SsState& s = state(h);
  *n_nw = 0;
  if (s.lp.empty() || n != s.n_cand) return ZG_EINVAL;
  if (cap < n) return ZG_E2BIG;
  const uint64_t m = std::max<uint64_t>(n, 1);
  s.keys.assign(m, 0);
  s.nw.assign(m, zg_check{});
  s.nw_owner.assign(m, 0);
  s.n_keys = 0;
  unsigned long long nw = 0;
  if (n) keys(KeyArgs{s.cand.data(), s.owner.data(), codes, n, granted, failed, s.include, s.keys.data(), &s.n_keys, s.nw.data(), s.nw_owner.data(), &nw});
  std::copy(s.nw.begin(), s.nw.begin() + nw, items);
  s.n_nw = nw;
  *n_nw = nw;
  return 0;
}

int emu_ss_route(void* h, const uint8_t* codes, uint64_t n, uint32_t n_dest, unsigned long long* routed, uint64_t* counts) {
  Emu* e = static_cast<Emu*>(h);
  SsState& s = state(h);
  for (uint32_t d = 0; d < n_dest && d < kMaxRouteDest; ++d) counts[d] = 0;
  if (s.lp.empty() || n != s.n_nw || n_dest != e->shard_count) return ZG_EINVAL;
  unsigned long long unused = 0;
  if (n) keys(KeyArgs{s.nw.data(), s.nw_owner.data(), codes, n, 0, 0, 0, s.keys.data(), &s.n_keys, nullptr, nullptr, &unused});
  if (s.n_keys) route(s.keys.data(), s.n_keys, n_dest, KeyHomeOwner{s.home.data()}, routed, counts);
  return 0;
}

// The objects a replica's forward walk marks for one lookup (device.cu lookup_subjects' fwalk_seed_kernel and
// fwalk_expand_kernel, levels 0 .. ZG_MAX_DEPTH + 1, on an unsharded emulated engine): *marked = the resource plus
// every object the walk reaches, 0 for a resource no relationship names. Returns -7 when the walk overflows walk_cap.
int emu_ss_replica_marks(void* h, uint16_t res_type, uint32_t res, uint16_t perm, uint16_t stype, uint16_t srel, uint64_t walk_cap,
                         uint64_t* marked) {
  Emu* e = static_cast<Emu*>(h);
  *marked = 0;
  if (!e->published || e->shard_count != 1 || res_type >= e->h.n_objects.size() || stype >= e->h.n_objects.size()) return ZG_EINVAL;
  if (res >= e->h.n_objects[res_type]) return 0;
  static const uint32_t zero = 0;
  std::vector<unsigned long long> base(e->h.n_objects.size() + 1, 0);
  for (size_t t = 0; t < e->h.n_objects.size(); ++t) base[t + 1] = base[t] + ((uint64_t(e->h.n_objects[t]) + 31) & ~31ull);
  std::vector<uint32_t> visited((base.back() + 31) / 32 + 4, 0), type_off;
  std::vector<unsigned long long> front[2] = {std::vector<unsigned long long>(walk_cap + 1), std::vector<unsigned long long>(walk_cap + 1)};
  std::vector<unsigned long long> counts(ZG_MAX_DEPTH + 4, 0);
  std::vector<FwdClass> fwd;
  e->sc.forward_tables(e->h.rels, &fwd, &type_off);
  std::vector<zg_check> jobs(walk_cap + 2);
  unsigned long long cand_count = 0;
  uint32_t flags = 0;
  FwalkParams p{};
  p.row_ptr = e->h.row_ptr.empty() ? &zero : e->h.row_ptr.data();
  p.col = e->h.col.empty() ? &zero : e->h.col.data();
  p.fwd = fwd.data();
  p.type_off = type_off.data();
  p.mask = e->sc.fwd_mask.data() + size_t(perm) * e->sc.fwd_mask_words;
  p.counts = counts.data();
  p.cap = walk_cap;
  p.visited = visited.data();
  p.type_bit_base = base.data();
  p.proto.res = res;
  p.proto.perm = perm;
  p.proto.stype = stype;
  p.proto.srel = srel;
  p.cand = jobs.data();
  p.cand_count = &cand_count;
  p.cand_cap = walk_cap + 2;
  p.flags = &flags;
  p.in = front[0].data();
  struct SeedArgs {
    FwalkParams p;
    uint32_t rt;
  } sa{p, res_type};
  zg_emu::launch(+[](const SeedArgs& a) { fwalk_seed_kernel(a.p, a.rt); }, sa, 1, 32, 0);
  uint64_t n = 1;
  for (int level = 0, cur = 0; level <= ZG_MAX_DEPTH + 1; ++level, cur ^= 1) {
    p.in = front[cur].data();
    p.out = front[cur ^ 1].data();
    p.level = level;
    zg_emu::launch(fwalk_expand_kernel, p, 2, 256, 0);
    if (flags & 16u) return -7;
    n += counts[level + 1];
    if (counts[level + 1] == 0) break;
  }
  *marked = n;
  return 0;
}

int emu_ss_finish(void* h, const unsigned long long* keys_in, uint64_t n, uint32_t* ids, uint64_t* listed, uint64_t* excluded) {
  SsState& s = state(h);
  const size_t K = s.lp.size();
  if (!K) return ZG_EINVAL;
  for (size_t k = 0; k < K; ++k) listed[k] = excluded[k] = 0;
  if (n == 0) return 0;
  // sort_u64 over the low kExclKeyBit + 1 bits: the keys have no others
  std::vector<unsigned long long> sorted(keys_in, keys_in + n), first(2 * kMaxLookupBatch, 0), end(2 * kMaxLookupBatch, 0);
  std::sort(sorted.begin(), sorted.end());
  struct SplitArgs {
    const unsigned long long* keys;
    unsigned long long n;
    uint32_t* ids;
    unsigned long long *first, *end;
  } sp{sorted.data(), n, ids, first.data(), end.data()};
  zg_emu::launch(+[](const SplitArgs& a) { ss_split_kernel(a.keys, a.n, a.ids, a.first, a.end); }, sp,
                 static_cast<unsigned>((n + 255) / 256), 256, 0);
  for (size_t k = 0; k < K; ++k) {
    listed[k] = end[k] - first[k];
    excluded[k] = end[kMaxLookupBatch + k] - first[kMaxLookupBatch + k];
  }
  return 0;
}

}  // extern "C"
