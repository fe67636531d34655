// emu_page.cc -- the page kernels (filter.cuh page_*) and their host side (page_walk, page_merge) under the CPU SIMT
// emulator. TEST INFRASTRUCTURE ONLY (built by tests/emu/emu_page.py into its own .so; never part of libzgpu.so).
// emu_filter.cc (and through it the emulator driver and the product's schema compiler and store) is compiled into this
// translation unit unchanged. Added here: device.cu Device::page_filter over host memory (its launches restated, the
// scan of the tile counts done on the host), and Store::page as the answer to compare with.
#include "emu_filter.cc"

namespace {

// device.cu select_classes, sorted as Device::page_filter sorts them
std::vector<FilterSel> page_select(const Emu* e, const Store::Filter& f) {
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
      s.pos = static_cast<uint16_t>(page_class_pos(sc, slot, c.stype, c.sslot));
      s.rtype = sc.slots[slot].type;
      sel.push_back(s);
    }
  }
  std::sort(sel.begin(), sel.end(), [](const FilterSel& a, const FilterSel& b) {
    return a.rtype != b.rtype ? a.rtype < b.rtype : a.pos < b.pos;
  });
  return sel;
}

struct EmuOps {
  unsigned grid;
  zg_tuple* out;
  uint32_t* out_exp;
  uint64_t* info;  // [1] windows, [2] launches, [3] most tiles of a window
  int window(const PagePlan& p, unsigned long long block, uint32_t stride, uint32_t obj0, unsigned long long entries,
             uint32_t* obj1, unsigned long long* n) {
    unsigned long long h[2] = {0, 0};
    const uint32_t nres = p.sel[0].nres;
    zg_emu::launch([&](int) { page_window_kernel(p.row_ptr, block, stride, obj0, nres, entries, h); }, 0, 1, 32, 0);
    *obj1 = static_cast<uint32_t>(h[0]);
    *n = h[1];
    ++info[1];
    ++info[2];
    return 0;
  }
  int tiles(PagePlan& p, unsigned long long got, unsigned long long* total) {
    const uint64_t n_tiles = (uint64_t(p.obj1 - p.obj0) + 31) / 32;
    std::vector<unsigned long long> cnt(n_tiles + 1, 0), off(n_tiles + 1, 0);
    p.tile_count = cnt.data();
    p.tile_off = off.data();
    p.out = out + got;
    p.out_exp = out_exp + got;
    zg_emu::launch(page_count_kernel, p, grid, 64, 0);
    for (uint64_t t = 0; t < n_tiles; ++t) off[t + 1] = off[t] + cnt[t];  // cub::DeviceScan::ExclusiveSum
    zg_emu::launch(page_emit_kernel, p, grid, 64, 0);
    *total = off[n_tiles];
    info[2] += 2;
    info[3] = std::max<uint64_t>(info[3], n_tiles);
    return 0;
  }
};

}  // namespace

// Store::page: the first `want` matches after `after` (has_after == 0: from the start) and their expirations.
extern "C" uint64_t emu_page_host(void* h, const EmuFilter* x, uint32_t now, int has_after, const uint32_t* after,
                                  uint64_t want, zg_tuple* out, uint32_t* out_exp) {
  Emu* e = static_cast<Emu*>(h);
  const PageKey k{after[0], after[1], after[2], after[3]};
  std::vector<uint64_t> idx;
  e->st.page(to_filter(*x), now, has_after ? &k : nullptr, want, &idx);
  for (uint64_t i = 0; i < idx.size(); ++i) {
    out[i] = e->st.tuples[idx[i]];
    out_exp[i] = e->st.expires[idx[i]];
  }
  return idx.size();
}

// Device::page_filter over host memory: `out` takes `want` records (the subject shape: n_sel segments of `want`, merged
// back into the first `want`). info: [0] records, [1] windows, [2] launches, [3] most tiles of one window, [4] scanned.
// Returns 0, -1 (not published) or what page_walk returned.
extern "C" int emu_page_device(void* h, const EmuFilter* x, uint32_t now, int has_after, const uint32_t* after, uint64_t want,
                               uint32_t grid, zg_tuple* out, uint32_t* out_exp, uint64_t* info) {
  Emu* e = static_cast<Emu*>(h);
  if (!e->published) return -1;
  for (int i = 0; i < 5; ++i) info[i] = 0;
  const Store::Filter f = to_filter(*x);
  const Schema& sc = e->sc;
  if (f.impossible) return 0;
  const std::vector<FilterSel> sel = page_select(e, f);
  if (sel.empty()) return 0;
  const PageKey k{after[0], after[1], after[2], after[3]};
  const PageKey* from = has_after ? &k : nullptr;
  static const uint32_t zero = 0;
  auto ptr = [&](const std::vector<uint32_t>& v) { return v.empty() ? &zero : v.data(); };
  PagePlan p{};
  p.row_ptr = ptr(e->h.row_ptr);
  p.col = ptr(e->h.col);
  p.exp = sc.has_expiry ? ptr(e->h.exp) : nullptr;
  p.rrow_ptr = ptr(e->h.rrow_ptr);
  p.rcol = ptr(e->h.rcol);
  p.now = now;
  p.has_subj = f.has_subj;
  p.subj = f.has_subj ? f.subj : 0;
  if (!f.has_res && (f.has_subj || f.subj_wildcard)) {  // Device::filter_shape: kBySubject
    page_set_after(p, from);
    p.want = want;
    std::vector<zg_tuple> rec(sel.size() * want);
    std::vector<uint32_t> rec_exp(sel.size() * want), seg(sel.size(), 0);
    for (size_t at = 0; at < sel.size(); at += kMaxFilterSel) {
      p.n_sel = static_cast<uint32_t>(std::min<size_t>(kMaxFilterSel, sel.size() - at));
      std::copy(sel.begin() + at, sel.begin() + at + p.n_sel, p.sel);
      p.out = rec.data() + at * want;
      p.out_exp = rec_exp.data() + at * want;
      p.seg_count = seg.data() + at;
      zg_emu::launch(page_subject_kernel, p, std::min<uint32_t>(grid, p.n_sel), 32, 0);
      ++info[2];
    }
    std::vector<zg_tuple> t;
    std::vector<uint32_t> ex;
    page_merge(sel, seg.data(), rec.data(), rec_exp.data(), want, &t, &ex);
    for (uint32_t c : seg) info[4] += c;
    std::copy(t.begin(), t.end(), out);
    std::copy(ex.begin(), ex.end(), out_exp);
    info[0] = t.size();
    return 0;
  }
  EmuOps ops{grid, out, out_exp, info};
  unsigned long long got = 0;
  uint64_t scanned = 0;
  if (int rc = page_walk(ops, p, sel, f.has_res, f.res, from, want, &got, &scanned)) return rc;
  info[0] = got;
  info[4] = scanned;
  return 0;
}

// page_class_pos, for the test's restatement of the key
extern "C" int emu_page_class_pos(void* h, int rel, int stype, int srel) {
  return page_class_pos(static_cast<Emu*>(h)->sc, rel, static_cast<uint16_t>(stype), static_cast<uint16_t>(srel));
}

extern "C" int emu_page_slot_type(void* h, int slot) { return static_cast<Emu*>(h)->sc.slots[slot].type; }
