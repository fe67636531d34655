// emu_import.cc -- zg_import_relationships' kernels (spicedb-kubeapi-proxy_b200/csrc/import.cuh) under the CPU SIMT
// emulator. TEST INFRASTRUCTURE ONLY (built by tests/emu/emu_import.py into its own .so; never part of libzgpu.so).
// The host side is the product's own schema compiler and store. The launch sequence of Device::import_check and
// Device::import_finish (device.cu) and the commit of capi.cu import_on_device are restated over host memory, with
// std::stable_sort standing in for the CUB radix sorts (both stable); the kernels run unchanged. The name mirror is
// built by the product's ingress_insert_kernel from the store's arena, and duplicates against the store are searched
// in Store::build()'s forward rows. One switch exists only here: the tag filter can be turned off, so that every probe
// of the mirror and of the new-name table compares bytes.
#define ZG_EMULATE 1
#include "cuda_emu.h"

static inline unsigned long long atomicCAS(unsigned long long* p, unsigned long long expected, unsigned long long desired) {
  __atomic_compare_exchange_n(p, &expected, desired, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
  return expected;
}
static inline unsigned long long atomicMin(unsigned long long* p, unsigned long long v) {
  unsigned long long cur = __atomic_load_n(p, __ATOMIC_SEQ_CST);
  while (v < cur && !__atomic_compare_exchange_n(p, &cur, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {
  }
  return cur;
}

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <numeric>
#include <string>

#include "../../spicedb-kubeapi-proxy_b200/csrc/import.cuh"
#include "../../spicedb-kubeapi-proxy_b200/csrc/store.h"

using namespace zg;

namespace {

struct EmuImport {
  Schema sc;
  Store store;
};

}  // namespace

extern "C" {

// One group as zg_import_group passes it (no expirations: they never reach the kernels).
struct EmuGroup {
  const char *res_type, *relation, *subj_type, *subj_rel;
  const char* res_ids;
  const uint32_t* res_off;
  const char* subj_ids;
  const uint32_t* subj_off;
  uint64_t n;
};

struct EmuImportOpts {
  uint64_t tag_mask;  // kIngressTagMask, or 0: no tag filter
  uint32_t grid, threads;
};

void* emu_imp_create(const char* schema, char* err, size_t cap) {
  auto* e = new EmuImport();
  const std::string m = e->sc.parse(schema);
  if (!m.empty()) {
    std::snprintf(err, cap, "%s", m.c_str());
    delete e;
    return nullptr;
  }
  e->store.reset(&e->sc);
  return e;
}
void emu_imp_destroy(void* h) { delete static_cast<EmuImport*>(h); }
int emu_imp_type_id(void* h, const char* name) { return static_cast<EmuImport*>(h)->sc.type_id(name); }
int emu_imp_slot_id(void* h, int type, const char* name) { return static_cast<EmuImport*>(h)->sc.slot_id(type, name); }

int emu_imp_intern(void* h, int type, const char* ids, const uint32_t* off, uint64_t n, uint32_t* out) {
  auto* e = static_cast<EmuImport*>(h);
  for (uint64_t i = 0; i < n; ++i) out[i] = e->store.intern(type, std::string(ids + off[i], off[i + 1] - off[i]));
  return ZG_OK;
}

int emu_imp_load(void* h, const zg_tuple* t, uint64_t n) {
  return static_cast<EmuImport*>(h)->store.load(t, nullptr, n).empty() ? ZG_OK : ZG_EINVAL;
}

// A type's name arena: the records [u32 id][u32 len][bytes]. Returns its size; copies it when it fits.
uint64_t emu_imp_arena(void* h, int type, char* buf, uint64_t cap) {
  const std::vector<char>& a = static_cast<EmuImport*>(h)->store.name_arena(type);
  if (buf && a.size() <= cap) std::memcpy(buf, a.data(), a.size());
  return a.size();
}

// Steps 1-5 of import.cuh over the groups (every literal field valid). *bad / *dup: the smallest call positions of a
// malformed id and of a duplicate (~0: none). When both are ~0 the new names are interned with the kernels' hashes and
// the tuples (call order, final ids) go to out and into the store. *n_new: the new names found.
int emu_imp_run(void* h, const EmuGroup* g, uint64_t ng, const EmuImportOpts* o, uint64_t* bad, uint64_t* dup,
                uint64_t* n_new, zg_tuple* out) {
  auto* e = static_cast<EmuImport*>(h);
  const Schema& sc = e->sc;
  Store& st = e->store;
  const size_t nt = sc.types.size();
  const bool locate = !st.tuples.empty();
  const HostSnapshot snap = locate ? st.build() : HostSnapshot();

  // stage the call as Device::import_check does
  std::vector<ImportGroupDev> gd(ng);
  std::vector<uint8_t> blob;
  std::vector<uint32_t> offs;
  uint64_t n = 0;
  for (uint64_t k = 0; k < ng; ++k) {
    ImportGroupDev& d = gd[k];
    const int rt = sc.type_id(g[k].res_type), sty = sc.type_id(g[k].subj_type);
    const int rel = rt < 0 ? -1 : sc.slot_id(rt, g[k].relation);
    const bool none = !g[k].subj_rel || !*g[k].subj_rel;
    const int sr = none || sty < 0 ? kNone : sc.slot_id(sty, g[k].subj_rel);
    if (rt < 0 || sty < 0 || rel < 0 || sr < 0) return ZG_EINVAL;
    d.item0 = n;
    d.n = g[k].n;
    d.res_blob = blob.size();
    blob.insert(blob.end(), g[k].res_ids, g[k].res_ids + g[k].res_off[g[k].n]);
    d.subj_blob = blob.size();
    blob.insert(blob.end(), g[k].subj_ids, g[k].subj_ids + g[k].subj_off[g[k].n]);
    d.off0 = offs.size();
    offs.insert(offs.end(), g[k].res_off, g[k].res_off + g[k].n + 1);
    offs.insert(offs.end(), g[k].subj_off, g[k].subj_off + g[k].n + 1);
    d.rtype = static_cast<uint32_t>(rt);
    d.stype = static_cast<uint32_t>(sty);
    d.rel = static_cast<uint32_t>(rel);
    d.srel = static_cast<uint32_t>(sr);
    d.pos_plain = static_cast<uint32_t>(page_class_pos(sc, rel, static_cast<uint16_t>(sty), static_cast<uint16_t>(sr)));
    d.pos_wild = static_cast<uint32_t>(page_class_pos(sc, rel, static_cast<uint16_t>(sty), kWildcard));
    d.k_plain = static_cast<uint32_t>(sc.class_of(rel, static_cast<uint16_t>(sty), static_cast<uint16_t>(sr)));
    d.k_wild = static_cast<uint32_t>(sc.class_of(rel, static_cast<uint16_t>(sty), kWildcard));
    if (locate) {
      const DRel& r = snap.rels[sc.slots[rel].rel_index];
      d.row_base = r.row_base;
      d.stride = r.stride;
      d.nres = r.nres;
    }
    n += g[k].n;
  }
  blob.resize(blob.size() + 8);
  *bad = *dup = kImportNone;
  *n_new = 0;
  if (!n) return ZG_OK;
  const ImportCall call{gd.data(), static_cast<uint32_t>(ng), blob.data(), offs.data(), n};

  // the name mirror: every record of the store's arena inserted by the product's kernel
  std::vector<std::vector<unsigned long long>> mslots(nt), moffs(nt);
  std::vector<IngressTable> tables(nt, IngressTable{nullptr, nullptr, 0});
  for (size_t t = 0; t < nt; ++t) {
    const std::vector<char>& ar = st.name_arena(static_cast<int>(t));
    for (uint64_t off = 0; off < ar.size();) {
      uint32_t len;
      std::memcpy(&len, ar.data() + off + 4, 4);
      moffs[t].push_back(off);
      off += 8 + uint64_t(len);
    }
    if (moffs[t].empty()) continue;
    uint64_t cap = 16;
    while (moffs[t].size() * 2 > cap) cap *= 2;
    mslots[t].assign(cap, 0);
    IngressInsertParams ip{};
    ip.arena = reinterpret_cast<const uint8_t*>(ar.data());
    ip.offs = moffs[t].data();
    ip.from = 0;
    ip.to = moffs[t].size();
    ip.slots = mslots[t].data();
    ip.mask = cap - 1;
    zg_emu::launch(ingress_insert_kernel, ip, o->grid, o->threads, 0);
    tables[t] = IngressTable{reinterpret_cast<const uint8_t*>(ar.data()), mslots[t].data(), cap - 1};
  }

  // 1. names
  const uint64_t occ = 2 * n;
  uint64_t cap = 64;
  while (cap < 2 * occ) cap *= 2;
  std::vector<unsigned long long> slots(cap, 0), first(cap, kImportNone), hash(cap, 0);
  std::vector<uint32_t> slot_type(cap, 0), occ_id(occ), occ_slot(occ);
  unsigned long long ctrl[4] = {kImportNone, kImportNone, 0, 0};
  ImportNamesParams np{};
  np.c = call;
  np.tables = tables.data();
  np.slots = slots.data();
  np.mask = cap - 1;
  np.first = first.data();
  np.hash = hash.data();
  np.slot_type = slot_type.data();
  np.occ_id = occ_id.data();
  np.occ_slot = occ_slot.data();
  np.bad = &ctrl[0];
  np.tag_mask = o->tag_mask;
  np.found = &ctrl[2];
  zg_emu::launch(import_names_kernel, np, o->grid, o->threads, 0);

  // 2. new names by (type, first occurrence), temporary ids
  std::vector<unsigned long long> keys(cap);
  std::vector<uint32_t> vals(cap);
  zg_emu::launch([&](int) { import_compact_kernel(slots.data(), cap, first.data(), slot_type.data(), keys.data(), vals.data(), &ctrl[3]); },
                 0, o->grid, o->threads, 0);
  const uint64_t nn = ctrl[3];
  std::vector<uint64_t> order(nn);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](uint64_t a, uint64_t b) { return keys[a] < keys[b]; });
  std::vector<unsigned long long> skeys(nn), out_hash(nn);
  std::vector<uint32_t> svals(nn), slot_tmp(cap, 0), extent(nt);
  for (uint64_t j = 0; j < nn; ++j) {
    skeys[j] = keys[order[j]];
    svals[j] = vals[order[j]];
  }
  std::vector<unsigned long long> start(nt, 0);
  std::vector<uint64_t> count(nt, 0);
  for (uint64_t j = nn; j-- > 0;) {
    start[skeys[j] >> 48] = j;
    ++count[skeys[j] >> 48];
  }
  for (size_t t = 0; t < nt; ++t) extent[t] = st.extent(static_cast<int>(t));
  zg_emu::launch([&](int) { import_rank_kernel(skeys.data(), svals.data(), nn, extent.data(), start.data(), hash.data(), slot_tmp.data(), out_hash.data()); },
                 0, o->grid, o->threads, 0);

  // 3. tuples and keys; the two stable passes of the sort by K
  std::vector<zg_tuple> tuples(n);
  std::vector<unsigned long long> hi(n), lo(n), hi2(n);
  std::vector<uint32_t> pos(n), pos2(n);
  std::vector<uint8_t> known(n);
  ImportAssembleParams ap{};
  ap.c = call;
  ap.occ_id = occ_id.data();
  ap.occ_slot = occ_slot.data();
  ap.slot_tmp = slot_tmp.data();
  ap.tuples = tuples.data();
  ap.key_hi = hi.data();
  ap.key_lo = lo.data();
  ap.vals = pos.data();
  ap.known = known.data();
  zg_emu::launch(import_assemble_kernel, ap, o->grid, o->threads, 0);
  pos2 = pos;
  std::stable_sort(pos2.begin(), pos2.end(), [&](uint32_t a, uint32_t b) { return lo[a] < lo[b]; });
  zg_emu::launch([&](int) { import_gather_kernel(hi.data(), pos2.data(), n, hi2.data()); }, 0, o->grid, o->threads, 0);
  {
    std::vector<uint64_t> idx(n);
    std::iota(idx.begin(), idx.end(), 0);
    std::stable_sort(idx.begin(), idx.end(), [&](uint64_t a, uint64_t b) { return hi2[a] < hi2[b]; });
    for (uint64_t j = 0; j < n; ++j) pos[j] = pos2[idx[j]];
  }

  // 4. duplicates
  zg_emu::launch([&](int) { import_adjacent_kernel(hi.data(), lo.data(), pos.data(), n, &ctrl[1]); }, 0, o->grid, o->threads, 0);
  if (locate) {
    ImportLocateParams lp{};
    lp.c = call;
    lp.tuples = tuples.data();
    lp.known = known.data();
    lp.row_ptr = snap.row_ptr.data();
    lp.col = snap.col.data();
    lp.owner_rank = 0;
    lp.owner_count = 1;
    lp.dup = &ctrl[1];
    zg_emu::launch(import_locate_kernel, lp, o->grid, o->threads, 0);
  }
  *bad = ctrl[0];
  *dup = ctrl[1];
  *n_new = nn;
  if (ctrl[0] != kImportNone || ctrl[1] != kImportNone) return ZG_OK;

  // 5. the ids the host hands out, the remap, and the commit
  std::vector<uint32_t> ids, next, rtype_of_rel(sc.slots.size());
  std::vector<unsigned long long> base(nt, 0);
  for (size_t t = 0; t < nt; ++t) {
    base[t] = ids.size();
    st.next_ids(static_cast<int>(t), count[t], &next);
    ids.insert(ids.end(), next.begin(), next.end());
  }
  for (size_t r = 0; r < sc.slots.size(); ++r) rtype_of_rel[r] = sc.slots[r].type;
  zg_emu::launch([&](int) { import_remap_kernel(tuples.data(), n, rtype_of_rel.data(), extent.data(), base.data(), ids.data()); },
                 0, o->grid, o->threads, 0);
  for (uint64_t j = 0; j < nn; ++j) {
    const uint64_t oc = skeys[j] & ((1ull << 48) - 1);
    const uint8_t* s;
    uint32_t len, type;
    import_occ(call, oc, &s, &len, &type);
    st.intern_new(static_cast<int>(type), reinterpret_cast<const char*>(s), len, out_hash[j]);
  }
  st.import(tuples.data(), nullptr, n);
  std::memcpy(out, tuples.data(), n * sizeof(zg_tuple));
  return ZG_OK;
}

}  // extern "C"
