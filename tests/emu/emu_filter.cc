// emu_filter.cc -- the relationship-filter kernels (filter.cuh) and their plan (device.cu Device::match_filter) under
// the CPU SIMT emulator. TEST INFRASTRUCTURE ONLY (built by tests/emu/emu_filter.py into its own .so; never part of
// libzgpu.so). The emulator driver emu_main.cc is compiled into this translation unit unchanged: its engine model (the
// product's schema compiler, store and host snapshot) comes with it. Added here: the class selection, the count
// launch and the emit launch over host memory, and Store::match as the answer to compare with.
#include "emu_main.cc"

#include "../../spicedb-kubeapi-proxy_b200/csrc/filter.cuh"

namespace {

struct EmuFilter {  // Store::Filter, flat
  int32_t res_type, rel, subj_type;
  uint32_t has_res, res, has_subj, subj, subj_wildcard, has_srel, srel;
};

Store::Filter to_filter(const EmuFilter& x) {
  Store::Filter f;
  f.res_type = x.res_type;
  f.has_res = x.has_res;
  f.res = x.res;
  f.rel = x.rel;
  f.subj_type = x.subj_type;
  f.has_subj = x.has_subj;
  f.subj = x.subj;
  f.subj_wildcard = x.subj_wildcard;
  f.has_srel = x.has_srel;
  f.srel = static_cast<uint16_t>(x.srel);
  return f;
}

}  // namespace

// Store::match: the matching relationships and their expirations in store order. Returns their number (cap too
// small: nothing is written past it).
extern "C" uint64_t emu_filter_host(void* h, const EmuFilter* x, uint32_t now, zg_tuple* out, uint32_t* out_exp, uint64_t cap) {
  Emu* e = static_cast<Emu*>(h);
  std::vector<uint64_t> idx;
  e->st.match(to_filter(*x), now, &idx);
  for (uint64_t i = 0; i < idx.size() && i < cap; ++i) {
    out[i] = e->st.tuples[idx[i]];
    out_exp[i] = e->st.expires[idx[i]];
  }
  return idx.size();
}

// device.cu match_filter over host memory. max_sel: selected classes per launch (kMaxFilterSel on the device; smaller
// here to run a filter in several launches). emit == 0: the count launch only. info: [0] count of the count launch,
// [1] count of the emit launch, [2] shape, [3] launches. Returns 0, -1 (not published), -7 (cap too small).
extern "C" int emu_filter_device(void* h, const EmuFilter* x, uint32_t now, uint32_t grid, uint32_t max_sel, int emit,
                                 zg_tuple* out, uint32_t* out_exp, uint64_t cap, uint64_t* info) {
  Emu* e = static_cast<Emu*>(h);
  if (!e->published) return -1;
  for (int i = 0; i < 4; ++i) info[i] = 0;
  const Store::Filter f = to_filter(*x);
  const Schema& sc = e->sc;
  std::vector<FilterSel> sel;
  for (size_t ri = 0; ri < sc.rel_slots.size(); ++ri) {
    const int slot = sc.rel_slots[ri];
    if ((f.res_type >= 0 && sc.slots[slot].type != f.res_type) || (f.rel >= 0 && slot != f.rel)) continue;
    const DRel& r = e->h.rels[ri];
    for (uint16_t k = 0; k < r.ncls; ++k) {
      const DCls& c = e->h.cls[r.cls_begin + k];
      if (f.subj_type >= 0 && c.stype != f.subj_type) continue;
      if (f.subj_wildcard && c.sslot != kWildcard) continue;
      if (f.has_subj && c.sslot == kWildcard) continue;
      if (f.has_srel && c.sslot != f.srel) continue;
      FilterSel s{};
      s.row_base = r.row_base + k;
      s.rrow_base = c.rrow_base;
      s.nres = r.nres;
      s.nsubj = c.nsubj;
      s.stride = r.stride;
      s.rstride = c.rstride;
      s.rel = static_cast<uint16_t>(slot);
      s.stype = c.stype;
      s.srel = c.sslot;
      sel.push_back(s);
    }
  }
  const int shape = f.has_res ? 0 : (f.has_subj || f.subj_wildcard) ? 1 : 2;
  info[2] = static_cast<uint64_t>(shape);
  static const uint32_t zero = 0;
  auto ptr = [&](const std::vector<uint32_t>& v) { return v.empty() ? &zero : v.data(); };
  unsigned long long count = 0;
  FilterPlan p{};
  p.row_ptr = ptr(e->h.row_ptr);
  p.col = ptr(e->h.col);
  p.exp = sc.has_expiry ? ptr(e->h.exp) : nullptr;
  p.rrow_ptr = ptr(e->h.rrow_ptr);
  p.rcol = ptr(e->h.rcol);
  p.has_subj = f.has_subj;
  p.res = f.res;
  p.subj = f.has_subj ? f.subj : 0;
  p.now = now;
  p.count = &count;
  auto run = [&](bool em) {
    count = 0;
    for (size_t at = 0; at < sel.size(); at += max_sel) {
      p.n_sel = static_cast<uint32_t>(std::min<size_t>(max_sel, sel.size() - at));
      std::copy(sel.begin() + at, sel.begin() + at + p.n_sel, p.sel);
      if (shape == 0) {
        if (em) zg_emu::launch(filter_resource_kernel<true>, p, grid, 64, 0);
        else zg_emu::launch(filter_resource_kernel<false>, p, grid, 64, 0);
      } else if (shape == 1) {
        if (em) zg_emu::launch(filter_subject_kernel<true>, p, grid, 64, 0);
        else zg_emu::launch(filter_subject_kernel<false>, p, grid, 64, 0);
      } else {
        if (em) zg_emu::launch(filter_scan_kernel<true>, p, grid, 64, 0);
        else zg_emu::launch(filter_scan_kernel<false>, p, grid, 64, 0);
      }
      ++info[3];
    }
  };
  if (f.impossible || sel.empty()) return 0;
  run(false);
  info[0] = count;
  if (!emit) return 0;
  if (count > cap) return -7;
  // the output is exactly as large as the count: a kernel that appended more would write past it (guarded by cap)
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
