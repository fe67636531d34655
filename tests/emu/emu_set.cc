// emu_set.cc -- the check kernel's signature meet with set tables (kernels.cuh sig_meet, MEET = kMeetSet16) under the
// CPU SIMT emulator (cuda_emu.h): emu_sig.cc's host-built closure indexes and signatures, plus the set table of every row, chosen and
// filled in the order build.cu closure_table_kernel takes (bucket counts from table_first_nb, `seeds` seeds each, each
// bucket's entries ascending). A pair whose target type holds 65 536 objects, or whose rows need more than
// kTableMaxBuckets buckets, has no table, and the check then runs kMeetSig16 as a publish's run_pass would. TEST
// INFRASTRUCTURE ONLY (built by tests/test_closure_set_emulation.py into its own .so; never part of libzgpu.so).
#include "emu_sig.cc"

namespace {

struct Tabled {
  Signed* s = nullptr;
  struct Pair {
    bool built = false;
    std::vector<unsigned long long> hdr, tab;
  };
  std::vector<Pair> pairs;
};

// places row[0, len) into nb buckets under seed: false when a bucket would get a fifth entry; fills tab when given
bool place(const uint16_t* row, uint32_t len, uint32_t nb, uint32_t seed, unsigned long long* tab) {
  std::vector<uint32_t> cnt(nb, 0);
  for (uint32_t i = 0; i < len; ++i) {
    const uint32_t k = table_bucket(row[i], seed, nb), slot = cnt[k]++;
    if (slot >= kTableSlots) return false;
    if (tab) {
      const unsigned long long sh = 16ull * slot;
      tab[k] = (tab[k] & ~(0xFFFFull << sh)) | (static_cast<unsigned long long>(row[i]) << sh);
    }
  }
  return true;
}

}  // namespace

extern "C" {

// Set tables of every pair of the signed index s (emu_sig_create, width 2), `seeds` seeds per bucket count; none when
// `capacity` (the target type's objects) is 65 536 or more.
void* emu_set_create(void* sp, uint32_t seeds, uint32_t capacity) {
  Signed* s = static_cast<Signed*>(sp);
  Tabled* t = new Tabled();
  t->s = s;
  for (const auto& c : s->x->cl) {
    Tabled::Pair q;
    q.built = capacity < 65536u && seeds > 0;
    for (uint32_t u = 0; u < c.nsubj && q.built; ++u) {
      const uint16_t* row = c.col + c.row_ptr[u];
      const uint32_t len = c.row_ptr[u + 1] - c.row_ptr[u];
      uint32_t nb = table_first_nb(len), seed = 0;
      bool ok = len == 0;
      while (!ok && nb <= kTableMaxBuckets) {
        for (seed = 0; seed < seeds; ++seed)
          if ((ok = place(row, len, nb, seed, nullptr))) break;
        if (!ok) nb = table_grow_nb(nb);
      }
      if (!ok) {
        q.built = false;
        break;
      }
      const uint32_t off = static_cast<uint32_t>(q.tab.size());
      q.hdr.push_back(table_header(off, nb, seed));
      q.tab.resize(size_t(off) + nb, ~0ull);
      place(row, len, nb, seed, q.tab.data() + off);
    }
    if (!q.built) q.hdr.clear(), q.tab.clear();
    t->pairs.push_back(std::move(q));
  }
  return t;
}

void emu_set_destroy(void* t) { delete static_cast<Tabled*>(t); }

// The meet emu_set_check runs: kMeetSet16 when every pair has a table, else kMeetSig16.
int emu_set_meet(void* t) {
  for (const auto& q : static_cast<Tabled*>(t)->pairs)
    if (!q.built) return kMeetSig16;
  return kMeetSet16;
}

int emu_set_built(void* t, int pair) { return static_cast<Tabled*>(t)->pairs[pair].built; }

uint64_t emu_set_buckets(void* t, int pair) { return static_cast<Tabled*>(t)->pairs[pair].tab.size(); }

// The header word of every row and the buckets of `pair` (rows and emu_set_buckets words).
void emu_set_copy(void* t, int pair, unsigned long long* hdr, unsigned long long* tab) {
  const auto& q = static_cast<Tabled*>(t)->pairs[pair];
  std::copy(q.hdr.begin(), q.hdr.end(), hdr);
  std::copy(q.tab.begin(), q.tab.end(), tab);
}

// One pass of check_kernel<COUNT, false, kMeetSet16> (pure permissions) when every pair has a table, else of
// kMeetSig16, as emu_sig_check.
uint32_t emu_set_check(void* tp, const zg_check* items, uint64_t n, uint8_t* out, int raw, int count, uint64_t* bytes) {
  Tabled* t = static_cast<Tabled*>(tp);
  Signed* s = t->s;
  Indexed* d = s->x;
  Emu* e = d->e;
  KParams p{};
  static const uint32_t zero = 0;
  auto ptr = [&](const std::vector<uint32_t>& v) { return v.empty() ? &zero : v.data(); };
  p.row_ptr = ptr(e->h.row_ptr);
  p.col = ptr(e->h.col);
  p.rrow_ptr = ptr(e->h.rrow_ptr);
  p.rcol = ptr(e->h.rcol);
  p.invert = 1;
  p.prog = d->blob.data();
  p.prog_bytes = static_cast<uint32_t>(d->blob.size());
  p.queries = items;
  p.nq = n;
  p.L = e->sc.max_leaves;
  p.out = out;
  p.final_codes = 1;
  Ctrl c;
  p.next = &c.next;
  p.subq_count = &c.subq_count;
  p.alg_bytes = &c.alg_bytes;
  p.flags = &c.flags;
  p.events = c.events;
  const uint32_t grid = 2, spill_cap = 4096;
  std::vector<uint4> spill(size_t(grid) * kWarpsPerBlock * spill_cap);
  std::vector<unsigned long long> memo(size_t(grid) * kWarpsPerBlock);
  std::vector<zg_check> subq(1 << 12);
  std::vector<uint32_t> subq_parent(1 << 12);
  p.spill = spill.data();
  p.spill_cap = spill_cap;
  p.subq = subq.data();
  p.subq_parent = subq_parent.data();
  p.subq_cap = subq.size();
  p.budget = 1 << 20;
  p.raw_items = raw;
  p.memo = memo.data();
  bool all = true;
  static const unsigned long long none = ~0ull;
  for (size_t i = 0; i < d->cl.size(); ++i) {
    const auto& cl = d->cl[i];
    const auto& q = s->pairs[i];
    const auto& x = t->pairs[i];
    all = all && x.built;
    p.closure[p.n_closure++] =
        ClosureRef{cl.row_ptr.data(), cl.col, cl.nsubj, cl.tgc, 2, q.sig.empty() ? nullptr : q.sig.data(), q.words,
                   x.built ? (x.hdr.empty() ? &none : x.hdr.data()) : nullptr,
                   x.built ? (x.tab.empty() ? &none : x.tab.data()) : nullptr};
  }
  const size_t sm = p.prog_bytes + size_t(kWarpsPerBlock) * kWarpSmem;
  if (all && p.n_closure) {
    if (count) zg_emu::launch(check_kernel<true, false, kMeetSet16>, p, grid, kThreads, sm);
    else zg_emu::launch(check_kernel<false, false, kMeetSet16>, p, grid, kThreads, sm);
  } else {
    if (count) zg_emu::launch(check_kernel<true, false, kMeetSig16>, p, grid, kThreads, sm);
    else zg_emu::launch(check_kernel<false, false, kMeetSig16>, p, grid, kThreads, sm);
  }
  *bytes = c.alg_bytes;
  return c.flags;
}

}  // extern "C"
