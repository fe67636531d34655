// emu_flat_record.cc -- the lean check kernel (kernels.cuh flat_check_kernel) with range records (closure_sig.cuh
// kRecSlots) built on the host from the forward CSR, and the residual pass behind it, under the CPU SIMT emulator
// (cuda_emu.h). Otherwise as emu_flat.cc's emu_flat_check with every pair tabled. TEST INFRASTRUCTURE ONLY (built by
// tests/test_flat_record_emulation.py into its own .so; never part of libzgpu.so).
#include "emu_flat.cc"

extern "C" {

// flat_check_kernel<COUNT> over the items with the range records of every SF_FLAT push step's class (records = 0:
// none), then check_kernel<COUNT, false, kMeetSet16, true> over its residual list. *n_records: the classes given
// records, *n_long: their rows read from the CSR. Returns the check kernel's flags word (~0: the residual counts
// disagree, or a pair has no table); *bytes: the COUNT variants' bytes; *residual: the items the lean kernel left.
uint32_t emu_flat_record_check(void* tp, const zg_check* items, uint64_t n, uint8_t* out, int raw, int count,
                               int records, uint32_t now, int no_wildcards, uint64_t* bytes, uint64_t* residual,
                               uint32_t* n_records, uint64_t* n_long) {
  Tabled* t = static_cast<Tabled*>(tp);
  Signed* s = t->s;
  Indexed* d = s->x;
  Emu* e = d->e;
  std::vector<uint16_t> tgcs;
  for (size_t i = 0; i < d->cl.size(); ++i)
    if (t->pairs[i].built) tgcs.push_back(d->cl[i].tgc);
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
    if (!x.built || q.sig.empty()) return ~0u;
    p.closure[p.n_closure++] = ClosureRef{cl.row_ptr.data(), cl.col, cl.nsubj, cl.tgc, 2, q.sig.data(), q.words,
                                          x.hdr.empty() ? &none : x.hdr.data(), x.tab.empty() ? &none : x.tab.data()};
  }
  // the records, as device.cu finish_publish picks their classes and build.cu flat_record_kernel fills them
  std::vector<std::vector<uint4>> recs;
  *n_long = 0;
  const DHeader* ph = reinterpret_cast<const DHeader*>(blob.data());
  const DSlot* slots = reinterpret_cast<const DSlot*>(blob.data() + ph->off_slots);
  const DUnit* units = reinterpret_cast<const DUnit*>(blob.data() + ph->off_units);
  const DStep* steps = reinterpret_cast<const DStep*>(blob.data() + ph->off_steps);
  for (uint32_t sl = 0; records && sl < ph->n_slots; ++sl) {
    if (!(slots[sl].flags & SF_FLAT)) continue;
    const DUnit& u = units[slots[sl].unit];
    for (int i = u.push_begin; i < u.step_end; ++i) {
      const DStep& st = steps[i];
      bool seen = false;
      for (uint32_t k = 0; k < p.n_rec; ++k) seen = seen || p.rec[k].gc == st.gc;
      if (seen || p.n_rec == static_cast<uint32_t>(kMaxFlatRecords)) continue;
      recs.emplace_back(size_t(st.nres) * kRecSlots / 8 + 1);
      uint16_t* r = reinterpret_cast<uint16_t*>(recs.back().data());
      for (uint32_t o = 0; o < st.nres; ++o) {
        const uint64_t row = st.row_base + uint64_t(o) * st.ncls;
        const uint32_t lo = e->h.row_ptr[row], len = e->h.row_ptr[row + 1] - lo;
        uint16_t* x = r + size_t(o) * kRecSlots;
        for (uint32_t k = 0; k < kRecSlots; ++k) x[k] = static_cast<uint16_t>(kRecLong);
        if (len < kRecSlots) {
          x[0] = static_cast<uint16_t>(len);
          for (uint32_t k = 0; k < len; ++k) x[k + 1] = static_cast<uint16_t>(e->h.col[lo + k]);
        } else {
          ++*n_long;
        }
      }
      p.rec[p.n_rec++] = FlatRecordRef{recs.back().data(), st.nres, st.gc};
    }
  }
  *n_records = p.n_rec;
  const size_t sm = p.prog_bytes + size_t(kWarpsPerBlock) * kWarpSmem;
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
