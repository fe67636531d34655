// emu_subjects.cc -- LookupSubjects' launch sequence (device.cu Device::lookup_subjects) under the CPU SIMT emulator.
// TEST INFRASTRUCTURE ONLY (built by tests/emu_subjects.py into its own .so; never part of libzgpu.so).
// The emulator driver emu_main.cc is compiled into this translation unit unchanged: its engine model (the product's
// schema compiler, store and host snapshot) and every emu_* entry point come with it. Added here: the pass loop
// with KParams::no_wildcards (the second verification), the forward walk, the fallback fill, the split kernel.
#include "emu_main.cc"

namespace {

int run_pass_ls(Emu* e, const EmuOpts& o, const zg_check* queries, uint64_t nq, uint8_t* val, uint8_t* out, bool raw,
                zg_check* subq, uint32_t* subq_parent, uint64_t* n_sub, bool count, bool no_wild) {
  KParams p{};
  static const uint32_t zero = 0;
  auto ptr = [&](const std::vector<uint32_t>& v) { return v.empty() ? &zero : v.data(); };
  p.row_ptr = ptr(e->h.row_ptr);
  p.col = ptr(e->h.col);
  p.exp = e->sc.has_expiry ? ptr(e->h.exp) : nullptr;
  p.rrow_ptr = ptr(e->h.rrow_ptr);
  p.rcol = ptr(e->h.rcol);
  p.invert = o.invert;
  p.prog = e->blob.data();
  p.prog_bytes = static_cast<uint32_t>(e->blob.size());
  p.queries = queries;
  p.nq = nq;
  p.L = e->sc.max_leaves;
  p.val = val;
  p.out = out;
  p.final_codes = 1;
  Ctrl c;
  p.next = &c.next;
  p.subq_count = &c.subq_count;
  p.alg_bytes = &c.alg_bytes;
  p.flags = &c.flags;
  p.events = c.events;
  p.ready = &c.ready;
  const uint32_t grid = o.grid ? o.grid : 2;
  const size_t warps = size_t(grid) * kWarpsPerBlock;
  std::vector<uint4> spill(warps * o.spill_cap);
  std::vector<unsigned long long> memo(warps * std::max<uint32_t>(o.memo_entries, 1));
  p.spill = spill.data();
  p.spill_cap = o.spill_cap;
  p.subq = subq;
  p.subq_parent = subq_parent;
  p.subq_cap = subq ? o.subq_cap : 0;
  p.now = o.now;
  p.budget = o.budget;
  p.raw_items = raw;
  p.memo = memo.data();
  p.memo_entries = o.memo_entries;
  p.memo_after = o.memo_after;
  p.shard_count = e->shard_count;
  p.shard_rank = e->shard_rank;
  p.no_wildcards = no_wild ? 1 : 0;
  if (e->shard_count > 1) p.invert = 0;  // a shard does not hold the subject's reverse rows
  const size_t sm = p.prog_bytes + size_t(kWarpsPerBlock) * kWarpSmem;
  if (count) zg_emu::launch(check_kernel<true, false>, p, grid, kThreads, sm);
  else if (o.streamed) zg_emu::launch(check_kernel<false, true>, p, grid, kThreads, sm);
  else zg_emu::launch(check_kernel<false, false>, p, grid, kThreads, sm);
  e->alg_bytes += c.alg_bytes;
  e->spills += c.events[0];
  e->memo_batches += c.events[1];
  e->flags |= c.flags;
  if (n_sub) *n_sub = c.subq_count;
  return 0;
}

// device.cu check_device over host memory, with KParams::no_wildcards on every pass when no_wild is set
int check_ls(Emu* e, const EmuOpts& o, const zg_check* items, uint64_t n, uint8_t* out, bool no_wild) {
  const bool count = false;
  if (n == 0) return 0;
  const uint32_t L = e->sc.max_leaves;
  if (!e->sc.has_nonpure) return run_pass_ls(e, o, items, n, nullptr, out, true, nullptr, nullptr, nullptr, count, no_wild);
  std::vector<std::vector<zg_check>> q(1);
  std::vector<std::vector<uint32_t>> parent(1);
  std::vector<std::vector<uint8_t>> val;
  std::vector<uint64_t> nq;
  const zg_check* queries = items;
  uint64_t cur = n;
  bool raw = true;
  for (size_t lv = 0; cur > 0; ++lv) {
    if (lv > ZG_MAX_DEPTH + 1) return -2;
    nq.push_back(cur);
    val.emplace_back(cur * L + 4, 0);
    q.emplace_back(o.subq_cap);
    parent.emplace_back(o.subq_cap);
    uint64_t n_sub = 0;
    run_pass_ls(e, o, queries, cur, val[lv].data(), lv == 0 ? out : nullptr, raw, q[lv + 1].data(), parent[lv + 1].data(), &n_sub, count, no_wild);
    if (n_sub > o.subq_cap) {
      if (n < 2) return -3;
      ++e->splits;
      const uint64_t half = n / 2;
      int r = check_ls(e, o, items, half, out, no_wild);
      if (r) return r;
      return check_ls(e, o, items + half, n - half, out + half, no_wild);
    }
    cur = n_sub;
    queries = q[lv + 1].data();
    raw = false;
    if (cur) ++e->passes;
  }
  if (nq.size() > 1) {
    struct FoldArgs {
      const uint8_t* prog;
      const zg_check* queries;
      unsigned long long n;
      uint32_t L;
      const uint8_t* val;
      uint8_t* out;
      const uint32_t* parent;
      uint8_t* parent_val;
    };
    for (size_t lv = nq.size(); lv-- > 0;) {
      FoldArgs a{e->blob.data(), lv == 0 ? items : q[lv].data(), nq[lv], L, val[lv].data(), lv == 0 ? out : nullptr,
                 lv == 0 ? nullptr : parent[lv].data(), lv == 0 ? nullptr : val[lv - 1].data()};
      zg_emu::launch(+[](const FoldArgs& f) { fold_kernel(f.prog, f.queries, f.n, f.L, f.val, f.out, f.parent, f.parent_val, 0); },
                     a, static_cast<unsigned>((nq[lv] + 255) / 256), 256, 0);
    }
  }
  return 0;
}

}  // namespace

// device.cu lookup_subjects over host memory: forward walk (or, forced or on overflow, every object of stype), the
// probe item, one verification, the no-wildcards verification when the wildcard is granted, compaction, sort.
// out: concrete ids then excluded ids, ascending each. info: [0] concrete, [1] excluded, [2] wildcard entry,
// [3] fell back to every object, [4] items of the first verification. Returns 0, ZG_EDEPTH, -7 (cap too small).
extern "C" int emu_lookup_subjects(void* h, uint16_t res_type, uint32_t res, uint16_t perm, uint16_t stype, uint16_t srel,
                                   int include_wildcard, int force_fallback, uint64_t walk_cap, const EmuOpts* o,
                                   uint32_t* out, uint64_t cap, uint64_t* info) {
  Emu* e = static_cast<Emu*>(h);
  if (!e->published) return -1;
  for (int i = 0; i < 5; ++i) info[i] = 0;
  if (res_type >= e->h.n_objects.size() || stype >= e->h.n_objects.size()) return ZG_EINVAL;
  if (res >= e->h.n_objects[res_type]) return 0;
  zg_check proto{};
  proto.res = res;
  proto.perm = perm;
  proto.stype = stype;
  proto.srel = srel;
  static const uint32_t zero = 0;
  std::vector<zg_check> jobs;
  bool walked = false;
  if (!force_fallback) {
    std::vector<unsigned long long> base(e->h.n_objects.size() + 1, 0);
    for (size_t t = 0; t < e->h.n_objects.size(); ++t) base[t + 1] = base[t] + ((uint64_t(e->h.n_objects[t]) + 31) & ~31ull);
    std::vector<uint32_t> visited((base.back() + 31) / 32 + 4, 0);
    std::vector<unsigned long long> front[2] = {std::vector<unsigned long long>(walk_cap + 1),
                                                std::vector<unsigned long long>(walk_cap + 1)};
    std::vector<unsigned long long> counts(ZG_MAX_DEPTH + 4, 0);
    std::vector<FwdClass> fwd;
    std::vector<uint32_t> type_off;
    e->sc.forward_tables(e->h.rels, &fwd, &type_off);
    jobs.resize(walk_cap + 2);
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
    p.proto = proto;
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
    int cur = 0;
    for (int level = 0; level <= ZG_MAX_DEPTH + 1; ++level) {
      p.in = front[cur].data();
      p.out = front[cur ^ 1].data();
      p.level = level;
      zg_emu::launch(fwalk_expand_kernel, p, 2, 256, 0);
      cur ^= 1;
      if (flags & 16u) break;
      if (counts[level + 1] == 0 || level == ZG_MAX_DEPTH + 1) {
        walked = true;
        break;
      }
    }
    if (walked) jobs.resize(cand_count);
  }
  if (!walked) {
    const uint64_t no = e->h.n_objects[stype];
    jobs.assign(no + 1, zg_check{});
    struct FillArgs {
      zg_check proto;
      unsigned long long n;
      zg_check* jobs;
    } fa{proto, no, jobs.data()};
    zg_emu::launch(+[](const FillArgs& a) { ls_fill_kernel(a.proto, a.n, a.jobs); }, fa, static_cast<unsigned>((no + 1 + 255) / 256), 256, 0);
  }
  const uint64_t n = jobs.size();
  info[3] = walked ? 0 : 1;
  info[4] = n;
  std::vector<uint8_t> codes(n);
  e->flags = 0;
  int rc = check_ls(e, *o, jobs.data(), n, codes.data(), false);
  if (rc) return rc;
  std::vector<uint32_t> has_ids(n), no_ids(n);
  std::vector<zg_check> has_items(n);
  unsigned long long cnt[2] = {0, 0};
  uint32_t sflags = 0;
  struct SplitArgs {
    const zg_check* items;
    const uint8_t* codes;
    unsigned long long n;
    uint32_t *has_ids;
    zg_check* has_items;
    uint32_t* no_ids;
    unsigned long long* counts;
    uint32_t* flags;
  } spa{jobs.data(), codes.data(), n, has_ids.data(), has_items.data(), no_ids.data(), cnt, &sflags};
  if (n > 1)
    zg_emu::launch(+[](const SplitArgs& a) { ls_split_kernel(a.items, a.codes, a.n, a.has_ids, a.has_items, a.no_ids, a.counts, a.flags); },
                   spa, static_cast<unsigned>((n - 1 + 255) / 256), 256, 0);
  if (codes[0] == ZG_ITEM_ERROR || (sflags & 8u)) return ZG_EDEPTH;
  const bool granted = srel == kNone && codes[0] == ZG_HAS_PERMISSION;
  std::vector<uint32_t> concrete(has_ids.begin(), has_ids.begin() + cnt[0]);
  if (granted && cnt[0]) {
    std::vector<uint8_t> codes2(cnt[0]);
    rc = check_ls(e, *o, has_items.data(), cnt[0], codes2.data(), true);
    if (rc) return rc;
    std::vector<uint32_t> kept(cnt[0]);
    unsigned long long nk = 0;
    uint32_t scratch = 0;
    struct CompactArgs {
      const uint32_t* cand;
      const uint8_t* codes;
      unsigned long long n;
      uint32_t* out;
      unsigned long long* count;
      uint32_t* flags;
    } ca{has_ids.data(), codes2.data(), cnt[0], kept.data(), &nk, &scratch};
    zg_emu::launch(+[](const CompactArgs& a) { lookup_compact_kernel(a.cand, a.codes, a.n, a.out, a.n, a.count, a.flags); }, ca,
                   static_cast<unsigned>((cnt[0] + 255) / 256), 256, 0);
    concrete.assign(kept.begin(), kept.begin() + nk);
  }
  std::sort(concrete.begin(), concrete.end());
  std::vector<uint32_t> excluded;
  if (granted && include_wildcard) {
    excluded.assign(no_ids.begin(), no_ids.begin() + cnt[1]);
    std::sort(excluded.begin(), excluded.end());
  }
  info[0] = concrete.size();
  info[1] = excluded.size();
  info[2] = granted && include_wildcard ? 1 : 0;
  if (concrete.size() + excluded.size() > cap) return -7;
  std::copy(concrete.begin(), concrete.end(), out);
  std::copy(excluded.begin(), excluded.end(), out + concrete.size());
  return 0;
}

