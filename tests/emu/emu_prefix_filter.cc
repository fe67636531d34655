// emu_prefix_filter.cc -- relationship filters by resource id prefix under the CPU SIMT emulator: the prefix scan
// (ingress.cuh prefix_match_kernel) over the store's own name arenas, then the filter and page kernels with bitmaps
// (filter.cuh, the kPrefix instantiations) and a prefix page's match lists (prefix_word_count_kernel,
// prefix_list_kernel, prefix_window_kernel) driven by page_walk. TEST INFRASTRUCTURE ONLY (built by
// tests/test_prefix_emulation.py into its own .so; never part of libzgpu.so).
//
// emu_page.cc (and through it emu_filter.cc, the emulator driver and the product's schema compiler and store) is
// compiled into this translation unit unchanged. Added here: Device::prefix_scan, Device::match_filter with a prefix
// and Device::page_filter's prefix path restated over host memory, and Store::match / Store::page with the prefix as
// the answers to compare with. Every buffer a kernel reads or writes -- the arenas, their record offsets, the prefix's
// bytes, the bitmaps, the match lists and their sums, the tile counts and the output -- ends at a PROT_NONE page and
// is sized exactly, so a read or write past its end faults.
#include "emu_page.cc"

// ingress.cuh's insert kernel claims 64-bit slots; cuda_emu.h has the 32-bit atomicCAS only.
static inline unsigned long long atomicCAS(unsigned long long* p, unsigned long long expected, unsigned long long desired) {
  __atomic_compare_exchange_n(p, &expected, desired, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
  return expected;
}

#include <sys/mman.h>
#include <unistd.h>

#include <memory>
#include <string>

#include "../../spicedb-kubeapi-proxy_b200/csrc/ingress.cuh"

namespace {

// `bytes` of zeroed memory whose last byte sits just before a PROT_NONE page.
struct Guarded {
  char* map = nullptr;
  size_t len = 0;
  void* p = nullptr;
  explicit Guarded(size_t bytes) {
    const size_t pg = static_cast<size_t>(sysconf(_SC_PAGESIZE));
    const size_t body = (bytes + pg - 1) / pg * pg + pg;
    map = static_cast<char*>(mmap(nullptr, body + pg, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0));
    if (map == MAP_FAILED) std::abort();
    if (mprotect(map + body, pg, PROT_NONE) != 0) std::abort();
    len = body + pg;
    p = map + body - bytes;
  }
  ~Guarded() { munmap(map, len); }
};

struct Arena {  // the device's guarded allocations of one call
  std::vector<std::unique_ptr<Guarded>> keep;
  template <class T>
  T* get(uint64_t n) {  // n >= 0 elements; n == 0 still gives a valid pointer to nothing
    keep.emplace_back(new Guarded(n * sizeof(T)));
    return static_cast<T*>(keep.back()->p);
  }
};

struct Bits {  // Device::prefix_scan's PrefixBits, and its counters
  std::vector<const uint32_t*> type;
  std::vector<uint32_t> n_ids;
  uint64_t names = 0, matched = 0, launches = 0;
};

// Device::prefix_scan over host memory: the types res_type may select, each bitmap covering the larger of the type's
// object capacity and its rows, filled by one prefix_match_kernel launch from the store's arenas.
void prefix_bits(Emu* e, Arena& a, int res_type, const std::string& prefix, unsigned grid, unsigned threads, Bits* b) {
  const Schema& sc = e->sc;
  const size_t nt = sc.types.size();
  b->type.assign(nt, nullptr);
  b->n_ids.assign(nt, 0);
  std::vector<char> want(nt, 0);
  for (size_t ri = 0; ri < sc.rel_slots.size() && ri < e->h.rels.size(); ++ri) {
    const int t = sc.slots[sc.rel_slots[ri]].type;
    if (res_type >= 0 && t != res_type) continue;
    want[t] = 1;
    b->n_ids[t] = std::max(b->n_ids[t], e->h.rels[ri].nres);
  }
  char* pfx = a.get<char>(prefix.size());
  std::memcpy(pfx, prefix.data(), prefix.size());
  unsigned long long matched = 0;
  PrefixPlan p{};
  p.prefix = reinterpret_cast<const uint8_t*>(pfx);
  p.len = prefix.size();
  p.matched = &matched;
  for (size_t t = 0; t < nt; ++t) {
    if (!want[t]) continue;
    if (t < e->h.n_objects.size()) b->n_ids[t] = std::max(b->n_ids[t], e->h.n_objects[t]);
    uint32_t* bits = a.get<uint32_t>((uint64_t(b->n_ids[t]) + 31) / 32);
    b->type[t] = bits;
    const std::vector<char>& ar = e->st.name_arena(static_cast<int>(t));
    if (ar.empty()) continue;
    std::vector<uint64_t> offs;
    for (uint64_t off = 0; off < ar.size();) {
      uint32_t len;
      std::memcpy(&len, ar.data() + off + 4, 4);
      offs.push_back(off);
      off += 8 + uint64_t(len);
    }
    char* arena = a.get<char>(ar.size());
    std::memcpy(arena, ar.data(), ar.size());
    unsigned long long* o = a.get<unsigned long long>(offs.size());
    std::copy(offs.begin(), offs.end(), o);
    PrefixType& x = p.type[p.n_types++];
    x.arena = reinterpret_cast<const uint8_t*>(arena);
    x.offs = o;
    x.n_recs = offs.size();
    x.bits = bits;
    x.n_ids = b->n_ids[t];
    b->names += offs.size();
  }
  if (p.n_types) {
    zg_emu::launch(prefix_match_kernel, p, grid, threads, 0);
    ++b->launches;
  }
  b->matched = matched;
}

Store::Filter prefix_filter(const EmuFilter* x, const char* prefix, uint64_t len) {
  Store::Filter f = to_filter(*x);
  f.prefix.assign(prefix, len);
  return f;
}

std::vector<const uint32_t*> class_bits(const Bits& b, const std::vector<FilterSel>& sel) {
  std::vector<const uint32_t*> out(sel.size());
  for (size_t k = 0; k < sel.size(); ++k) out[k] = b.type[sel[k].rtype];
  return out;
}

// Device::page_filter's Ops with a prefix: windows over the ascending list of a type's matched ids, tiles with bitmaps.
struct PrefixOps {
  Emu* e;
  Arena* a;
  const Bits* b;
  unsigned grid;
  zg_tuple* out;
  uint32_t* out_exp;
  uint64_t* info;  // [1] windows, [2] launches, [3] most tiles of a window, [5] list launches
  int list_type = -1;
  uint32_t m = 0;
  const uint32_t* ids = nullptr;
  const unsigned long long* csum = nullptr;
  void build_list(const PagePlan& p, unsigned long long block, uint32_t stride) {
    const int type = p.sel[0].rtype;
    const uint32_t n_ids = b->n_ids[type], words = (n_ids + 31) / 32;
    uint32_t* first = a->get<uint32_t>(uint64_t(words) + 1);
    const uint32_t* bits = b->type[type];
    zg_emu::launch([&](int) { prefix_word_count_kernel(bits, words, first); }, 0, grid, 64, 0);
    uint32_t run = 0;  // cub::DeviceScan::ExclusiveSum, in place
    for (uint64_t w = 0; w <= words; ++w) {
      const uint32_t c = first[w];
      first[w] = run;
      run += c;
    }
    m = first[words];
    uint32_t* list = a->get<uint32_t>(m);
    unsigned long long* ent = a->get<unsigned long long>(uint64_t(m) + 1);
    const uint32_t nres = p.sel[0].nres;
    const uint32_t* row_ptr = p.row_ptr;
    zg_emu::launch([&](int) { prefix_list_kernel(bits, words, first, row_ptr, block, stride, nres, list, ent); }, 0, grid, 64, 0);
    unsigned long long* sum = a->get<unsigned long long>(uint64_t(m) + 1);
    unsigned long long s = 0;
    for (uint64_t i = 0; i <= m; ++i) {
      sum[i] = s;
      s += ent[i];
    }
    ids = list;
    csum = sum;
    list_type = type;
    info[2] += 4;
    info[5] += 4;
  }
  int window(const PagePlan& p, unsigned long long block, uint32_t stride, uint32_t obj0, unsigned long long entries,
             uint32_t* obj1, unsigned long long* n) {
    if (list_type != p.sel[0].rtype) build_list(p, block, stride);
    unsigned long long* h = a->get<unsigned long long>(2);
    const uint32_t nres = p.sel[0].nres;
    zg_emu::launch([&](int) { prefix_window_kernel(ids, csum, m, obj0, nres, entries, h); }, 0, 1, 32, 0);
    *obj1 = static_cast<uint32_t>(h[0]);
    *n = h[1];
    ++info[1];
    ++info[2];
    ++info[5];
    return 0;
  }
  int tiles(PagePlan& p, unsigned long long got, unsigned long long* total) {
    const uint64_t n_tiles = (uint64_t(p.obj1 - p.obj0) + 31) / 32;
    unsigned long long* cnt = a->get<unsigned long long>(n_tiles + 1);
    unsigned long long* off = a->get<unsigned long long>(n_tiles + 1);
    p.tile_count = cnt;
    p.tile_off = off;
    p.out = out + got;
    p.out_exp = out_exp + got;
    zg_emu::launch(page_count_kernel<true>, p, grid, 64, 0);
    off[0] = 0;
    for (uint64_t t = 0; t < n_tiles; ++t) off[t + 1] = off[t] + cnt[t];
    zg_emu::launch(page_emit_kernel<true>, p, grid, 64, 0);
    *total = off[n_tiles];
    info[2] += 2;
    info[3] = std::max<uint64_t>(info[3], n_tiles);
    return 0;
  }
};

}  // namespace

extern "C" {

// Store::intern / Store::find: the names the filters match (the driver's loads name ids only).
uint32_t emu_prefix_intern(void* h, int type, const char* s, uint64_t len) {
  return static_cast<Emu*>(h)->st.intern(type, std::string(s, len));
}
uint32_t emu_prefix_find(void* h, int type, const char* s, uint64_t len) {
  return static_cast<Emu*>(h)->st.find(type, s, len);
}

// Device::prefix_scan alone: bits receives every selected type's bitmap back to back in type order (cap words).
// info: [0] names scanned, [1] ids matched, [2] launches. Returns the words written, or -1 when cap is too small.
long long emu_prefix_bits(void* h, int res_type, const char* prefix, uint64_t len, uint32_t grid, uint32_t* bits, uint64_t cap,
                          uint64_t* info) {
  Emu* e = static_cast<Emu*>(h);
  Arena a;
  Bits b;
  prefix_bits(e, a, res_type, std::string(prefix, len), grid, 64, &b);
  uint64_t w = 0;
  for (size_t t = 0; t < b.type.size(); ++t) {
    if (!b.type[t]) continue;
    const uint64_t n = (uint64_t(b.n_ids[t]) + 31) / 32;
    if (w + n > cap) return -1;
    std::copy(b.type[t], b.type[t] + n, bits + w);
    w += n;
  }
  info[0] = b.names;
  info[1] = b.matched;
  info[2] = b.launches;
  return static_cast<long long>(w);
}

// Store::match with the prefix.
uint64_t emu_prefix_match_host(void* h, const EmuFilter* x, const char* prefix, uint64_t len, uint32_t now, zg_tuple* out,
                               uint32_t* out_exp, uint64_t cap) {
  Emu* e = static_cast<Emu*>(h);
  std::vector<uint64_t> idx;
  e->st.match(prefix_filter(x, prefix, len), now, &idx);
  for (uint64_t i = 0; i < idx.size() && i < cap; ++i) {
    out[i] = e->st.tuples[idx[i]];
    out_exp[i] = e->st.expires[idx[i]];
  }
  return idx.size();
}

// Device::match_filter with a prefix: the bitmaps, the count launch, and the emit launch into an output of exactly the
// counted size. max_sel: classes per launch. info: [0] count, [1] emitted, [2] shape (1 subject, 2 scan), [3] launches,
// [4] ids matched. Returns 0, -1 (not published), -2 (a resource id with a prefix), -7 (cap too small).
int emu_prefix_match_device(void* h, const EmuFilter* x, const char* prefix, uint64_t len, uint32_t now, uint32_t grid,
                            uint32_t max_sel, zg_tuple* out, uint32_t* out_exp, uint64_t cap, uint64_t* info) {
  Emu* e = static_cast<Emu*>(h);
  if (!e->published) return -1;
  for (int i = 0; i < 5; ++i) info[i] = 0;
  const Store::Filter f = prefix_filter(x, prefix, len);
  if (f.has_res) return -2;
  if (f.impossible) return 0;
  const std::vector<FilterSel> sel = page_select(e, f);
  if (sel.empty()) return 0;
  Arena a;
  Bits b;
  prefix_bits(e, a, f.res_type, f.prefix, grid, 64, &b);
  info[3] += b.launches;
  info[4] = b.matched;
  const std::vector<const uint32_t*> bits = class_bits(b, sel);
  const int shape = (f.has_subj || f.subj_wildcard) ? 1 : 2;
  info[2] = static_cast<uint64_t>(shape);
  static const uint32_t zero = 0;
  auto ptr = [&](const std::vector<uint32_t>& v) { return v.empty() ? &zero : v.data(); };
  unsigned long long* count = a.get<unsigned long long>(1);
  const Schema& sc = e->sc;
  FilterPlan p{};
  p.row_ptr = ptr(e->h.row_ptr);
  p.col = ptr(e->h.col);
  p.exp = sc.has_expiry ? ptr(e->h.exp) : nullptr;
  p.rrow_ptr = ptr(e->h.rrow_ptr);
  p.rcol = ptr(e->h.rcol);
  p.has_subj = f.has_subj;
  p.subj = f.has_subj ? f.subj : 0;
  p.now = now;
  p.count = count;
  auto run = [&](bool em) {
    *count = 0;
    for (size_t at = 0; at < sel.size(); at += max_sel) {
      p.n_sel = static_cast<uint32_t>(std::min<size_t>(max_sel, sel.size() - at));
      std::copy(sel.begin() + at, sel.begin() + at + p.n_sel, p.sel);
      std::copy(bits.begin() + at, bits.begin() + at + p.n_sel, p.bits);
      if (shape == 1) {
        if (em) zg_emu::launch(filter_subject_kernel<true, true>, p, grid, 64, 0);
        else zg_emu::launch(filter_subject_kernel<false, true>, p, grid, 64, 0);
      } else {
        if (em) zg_emu::launch(filter_scan_kernel<true, true>, p, grid, 64, 0);
        else zg_emu::launch(filter_scan_kernel<false, true>, p, grid, 64, 0);
      }
      ++info[3];
    }
  };
  run(false);
  info[0] = *count;
  if (*count > cap) return -7;
  const uint64_t n = *count;
  p.out = a.get<zg_tuple>(n);
  p.out_exp = a.get<uint32_t>(n);
  p.cap = n;
  run(true);
  info[1] = *count;
  std::copy(p.out, p.out + n, out);
  std::copy(p.out_exp, p.out_exp + n, out_exp);
  return 0;
}

// Store::page with the prefix.
uint64_t emu_prefix_page_host(void* h, const EmuFilter* x, const char* prefix, uint64_t len, uint32_t now, int has_after,
                              const uint32_t* after, uint64_t want, zg_tuple* out, uint32_t* out_exp) {
  Emu* e = static_cast<Emu*>(h);
  const PageKey k{after[0], after[1], after[2], after[3]};
  std::vector<uint64_t> idx;
  e->st.page(prefix_filter(x, prefix, len), now, has_after ? &k : nullptr, want, &idx);
  for (uint64_t i = 0; i < idx.size(); ++i) {
    out[i] = e->st.tuples[idx[i]];
    out_exp[i] = e->st.expires[idx[i]];
  }
  return idx.size();
}

// Device::page_filter with a prefix over host memory. info: [0] records, [1] windows, [2] launches, [3] most tiles of
// one window, [4] scanned, [5] launches of the match lists and their windows. Returns 0, -1, -2 or page_walk's code.
int emu_prefix_page_device(void* h, const EmuFilter* x, const char* prefix, uint64_t len, uint32_t now, int has_after,
                           const uint32_t* after, uint64_t want, uint32_t grid, zg_tuple* out, uint32_t* out_exp, uint64_t* info) {
  Emu* e = static_cast<Emu*>(h);
  if (!e->published) return -1;
  for (int i = 0; i < 6; ++i) info[i] = 0;
  const Store::Filter f = prefix_filter(x, prefix, len);
  if (f.has_res) return -2;
  if (f.impossible) return 0;
  const std::vector<FilterSel> sel = page_select(e, f);
  if (sel.empty()) return 0;
  Arena a;
  Bits b;
  prefix_bits(e, a, f.res_type, f.prefix, grid, 64, &b);
  const std::vector<const uint32_t*> bits = class_bits(b, sel);
  const PageKey k{after[0], after[1], after[2], after[3]};
  const PageKey* from = has_after ? &k : nullptr;
  static const uint32_t zero = 0;
  auto ptr = [&](const std::vector<uint32_t>& v) { return v.empty() ? &zero : v.data(); };
  const Schema& sc = e->sc;
  PagePlan p{};
  p.row_ptr = ptr(e->h.row_ptr);
  p.col = ptr(e->h.col);
  p.exp = sc.has_expiry ? ptr(e->h.exp) : nullptr;
  p.rrow_ptr = ptr(e->h.rrow_ptr);
  p.rcol = ptr(e->h.rcol);
  p.now = now;
  p.has_subj = f.has_subj;
  p.subj = f.has_subj ? f.subj : 0;
  if (f.has_subj || f.subj_wildcard) {  // the subject shape: a segment of `want` per class, merged on the host
    page_set_after(p, from);
    p.want = want;
    zg_tuple* rec = a.get<zg_tuple>(sel.size() * want);
    uint32_t* rec_exp = a.get<uint32_t>(sel.size() * want);
    uint32_t* seg = a.get<uint32_t>(sel.size());
    for (size_t at = 0; at < sel.size(); at += kMaxFilterSel) {
      p.n_sel = static_cast<uint32_t>(std::min<size_t>(kMaxFilterSel, sel.size() - at));
      std::copy(sel.begin() + at, sel.begin() + at + p.n_sel, p.sel);
      std::copy(bits.begin() + at, bits.begin() + at + p.n_sel, p.bits);
      p.out = rec + at * want;
      p.out_exp = rec_exp + at * want;
      p.seg_count = seg + at;
      zg_emu::launch(page_subject_kernel<true>, p, std::min<uint32_t>(grid, p.n_sel), 32, 0);
      ++info[2];
    }
    std::vector<zg_tuple> t;
    std::vector<uint32_t> ex;
    page_merge(sel, seg, rec, rec_exp, want, &t, &ex);
    for (size_t i = 0; i < sel.size(); ++i) info[4] += seg[i];
    std::copy(t.begin(), t.end(), out);
    std::copy(ex.begin(), ex.end(), out_exp);
    info[0] = t.size();
    return 0;
  }
  zg_tuple* o = a.get<zg_tuple>(want);
  uint32_t* oe = a.get<uint32_t>(want);
  PrefixOps ops{e, &a, &b, grid, o, oe, info};
  unsigned long long got = 0;
  uint64_t scanned = 0;
  if (int rc = page_walk(ops, p, sel, false, 0, from, want, &got, &scanned, &bits)) return rc;
  std::copy(o, o + got, out);
  std::copy(oe, oe + got, out_exp);
  info[0] = got;
  info[4] = scanned;
  return 0;
}

}  // extern "C"
