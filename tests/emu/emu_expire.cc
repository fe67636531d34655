// emu_expire.cc -- the collection scan (filter.cuh filter_expired_kernel) and its plan (device.cu
// Device::match_expired) under the CPU SIMT emulator. TEST INFRASTRUCTURE ONLY (built by tests/emu/emu_expire.py into
// its own .so; never part of libzgpu.so). The emulator driver emu_main.cc is compiled into this translation unit
// unchanged: its engine model (the product's schema compiler, store and host snapshot) comes with it. Added here: the
// class selection, the count launch and the emit launch over host memory, and Store::expired as the answer to compare
// with.
#include "emu_main.cc"

#include "../../spicedb-kubeapi-proxy_b200/csrc/filter.cuh"

// Store::expired: the relationships it selects, in store order. Returns their number (cap too small: nothing is
// written past it).
extern "C" uint64_t emu_expired_host(void* h, uint32_t before, zg_tuple* out, uint32_t* out_exp, uint64_t cap) {
  Emu* e = static_cast<Emu*>(h);
  std::vector<uint64_t> idx;
  e->st.expired(before, &idx);
  for (uint64_t i = 0; i < idx.size() && i < cap; ++i) {
    out[i] = e->st.tuples[idx[i]];
    out_exp[i] = e->st.expires[idx[i]];
  }
  return idx.size();
}

// device.cu match_expired over host memory. max_sel: selected classes per launch. poison != 0: every expiration in a
// row of a class WITHOUT CF_EXPIRY is set to 1 in a copy of the snapshot first, so that a kernel reading such a row
// would report it. info: [0] count of the count launch, [1] count of the emit launch, [2] selected classes,
// [3] launches. Returns 0, -1 (not published), -7 (cap too small).
extern "C" int emu_expired_device(void* h, uint32_t before, uint32_t grid, uint32_t max_sel, int emit, int poison,
                                  zg_tuple* out, uint32_t* out_exp, uint64_t cap, uint64_t* info) {
  Emu* e = static_cast<Emu*>(h);
  if (!e->published) return -1;
  for (int i = 0; i < 4; ++i) info[i] = 0;
  const Schema& sc = e->sc;
  std::vector<uint32_t> exp = e->h.exp;
  std::vector<FilterSel> sel;
  for (size_t ri = 0; ri < sc.rel_slots.size(); ++ri) {
    const DRel& r = e->h.rels[ri];
    for (uint16_t k = 0; k < r.ncls; ++k) {
      const DCls& c = e->h.cls[r.cls_begin + k];
      if (!(c.flags & CF_EXPIRY)) {
        if (poison && !exp.empty())
          for (uint64_t o = 0; o < r.nres; ++o) {
            const uint64_t ri2 = r.row_base + k + o * r.stride;
            for (uint32_t i = e->h.row_ptr[ri2]; i < e->h.row_ptr[ri2 + 1]; ++i) exp[i] = 1;
          }
        continue;
      }
      FilterSel s{};
      s.row_base = r.row_base + k;
      s.nres = r.nres;
      s.stride = r.stride;
      s.rel = static_cast<uint16_t>(sc.rel_slots[ri]);
      s.stype = c.stype;
      s.srel = c.sslot;
      sel.push_back(s);
    }
  }
  info[2] = sel.size();
  static const uint32_t zero = 0;
  auto ptr = [&](const std::vector<uint32_t>& v) { return v.empty() ? &zero : v.data(); };
  unsigned long long count = 0;
  FilterPlan p{};
  p.row_ptr = ptr(e->h.row_ptr);
  p.col = ptr(e->h.col);
  p.exp = sc.has_expiry ? ptr(exp) : nullptr;
  p.rrow_ptr = ptr(e->h.rrow_ptr);
  p.rcol = ptr(e->h.rcol);
  p.now = before;
  p.count = &count;
  auto run = [&](bool em) {
    count = 0;
    for (size_t at = 0; at < sel.size(); at += max_sel) {
      p.n_sel = static_cast<uint32_t>(std::min<size_t>(max_sel, sel.size() - at));
      std::copy(sel.begin() + at, sel.begin() + at + p.n_sel, p.sel);
      if (em) zg_emu::launch(filter_expired_kernel<true>, p, grid, 64, 0);
      else zg_emu::launch(filter_expired_kernel<false>, p, grid, 64, 0);
      ++info[3];
    }
  };
  if (sel.empty()) return 0;
  run(false);
  info[0] = count;
  if (!emit || count == 0) return 0;
  if (count > cap) return -7;
  std::vector<zg_tuple> rec(count);
  std::vector<uint32_t> ex(count);
  p.out = rec.data();
  p.out_exp = ex.data();
  p.cap = count;
  run(true);
  info[1] = count;
  std::copy(rec.begin(), rec.end(), out);
  std::copy(ex.begin(), ex.end(), out_exp);
  return 0;
}
