// emu_flat.cc -- the lean check kernel (kernels.cuh flat_check_kernel) and the residual pass of check_kernel<kMeetSet16>
// behind it, under the CPU SIMT emulator (cuda_emu.h), as device.cu run_pass launches them on a snapshot with SF_FLAT
// slots: emu_set.cc's host-built closure indexes, signatures and set tables, and the program's SF_FLAT flags marked by
// schema.cc mark_flat_slots over every pair with a table. TEST INFRASTRUCTURE ONLY (built by
// tests/test_flat_check_emulation.py into its own .so; never part of libzgpu.so).
#include "emu_set.cc"

extern "C" {

// SF_FLAT of every slot of the set-tabled index t's program (after mark_flat_slots), and the number marked.
int emu_flat_mark(void* tp, uint16_t* flags, int n_slots) {
  Tabled* t = static_cast<Tabled*>(tp);
  Indexed* d = t->s->x;
  std::vector<uint16_t> tgcs;
  for (size_t i = 0; i < d->cl.size(); ++i)
    if (t->pairs[i].built) tgcs.push_back(d->cl[i].tgc);
  std::vector<uint8_t> blob = d->blob;
  const int marked = mark_flat_slots(&blob, tgcs);
  const DHeader* ph = reinterpret_cast<const DHeader*>(blob.data());
  for (int s = 0; s < n_slots && s < static_cast<int>(ph->n_slots); ++s)
    flags[s] = reinterpret_cast<const DSlot*>(blob.data() + ph->off_slots)[s].flags;
  return marked;
}

// flat_check_kernel<COUNT> over the items, then check_kernel<COUNT, false, kMeetSet16, true> over its residual list
// (pure permissions). lean = 0: no slot is marked SF_FLAT, so every item is residual; lean < 0: the plain
// check_kernel<COUNT, false, kMeetSet16> over the items alone, as a snapshot without flat slots runs them (the
// reference). now: the expiration clock; no_wildcards: KParams::no_wildcards. val (may be null): [n] leaf values.
// *residual: the items the lean kernel left. Returns the check kernel's flags word; *bytes: the COUNT variants' bytes.
uint32_t emu_flat_check(void* tp, const zg_check* items, uint64_t n, uint8_t* out, uint8_t* val, int raw, int count,
                        int lean, uint32_t now, int no_wildcards, uint64_t* bytes, uint64_t* residual) {
  Tabled* t = static_cast<Tabled*>(tp);
  Signed* s = t->s;
  Indexed* d = s->x;
  Emu* e = d->e;
  std::vector<uint16_t> tgcs;
  for (size_t i = 0; i < d->cl.size(); ++i)
    if (t->pairs[i].built && lean > 0) tgcs.push_back(d->cl[i].tgc);
  std::vector<uint8_t> blob = d->blob;
  mark_flat_slots(&blob, tgcs);
  KParams p{};
  static const uint32_t zero = 0;
  auto ptr = [&](const std::vector<uint32_t>& v) { return v.empty() ? &zero : v.data(); };
  p.row_ptr = ptr(e->h.row_ptr);
  p.col = ptr(e->h.col);
  p.exp = e->sc.has_expiry ? ptr(e->h.exp) : nullptr;
  p.rrow_ptr = ptr(e->h.rrow_ptr);
  p.rcol = ptr(e->h.rcol);
  p.invert = 1;
  p.prog = blob.data();
  p.prog_bytes = static_cast<uint32_t>(blob.size());
  p.queries = items;
  p.nq = n;
  p.L = e->sc.max_leaves;
  p.out = out;
  p.val = val;
  p.final_codes = 1;
  p.now = now;
  p.no_wildcards = no_wildcards;
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
  static const unsigned long long none = ~0ull;
  for (size_t i = 0; i < d->cl.size(); ++i) {
    const auto& cl = d->cl[i];
    const auto& q = s->pairs[i];
    const auto& x = t->pairs[i];
    if (!x.built || q.sig.empty()) return ~0u;  // the lean kernel runs only where every pair has both (kMeetSet16)
    p.closure[p.n_closure++] = ClosureRef{cl.row_ptr.data(), cl.col, cl.nsubj, cl.tgc, 2, q.sig.data(), q.words,
                                          x.hdr.empty() ? &none : x.hdr.data(), x.tab.empty() ? &none : x.tab.data()};
  }
  const size_t sm = p.prog_bytes + size_t(kWarpsPerBlock) * kWarpSmem;
  if (lean < 0) {
    if (count) zg_emu::launch(check_kernel<true, false, kMeetSet16>, p, grid, kThreads, sm);
    else zg_emu::launch(check_kernel<false, false, kMeetSet16>, p, grid, kThreads, sm);
    *bytes = c.alg_bytes;
    *residual = n;
    return c.flags;
  }
  std::vector<uint32_t> idx(std::max<uint64_t>(n, 1));
  unsigned long long nq_dev[2] = {0, 0};
  p.idx = idx.data();
  p.nq_dev = nq_dev;
  const unsigned fgrid = static_cast<unsigned>((n + kFlatThreads - 1) / kFlatThreads);
  if (count) zg_emu::launch(flat_check_kernel<true>, p, fgrid, kFlatThreads, 0);
  else zg_emu::launch(flat_check_kernel<false>, p, fgrid, kFlatThreads, 0);
  if (count) zg_emu::launch(check_kernel<true, false, kMeetSet16, true>, p, grid, kThreads, sm);
  else zg_emu::launch(check_kernel<false, false, kMeetSet16, true>, p, grid, kThreads, sm);
  *bytes = c.alg_bytes;
  *residual = nq_dev[0];
  return nq_dev[1] == nq_dev[0] ? c.flags : ~0u;
}

}  // extern "C"
