// emu_ingress.cc -- device ingress (spicedb-kubeapi-proxy_b200/csrc/ingress.cuh) under the CPU SIMT emulator.
// TEST INFRASTRUCTURE ONLY (built by tests/emu/emu_ingress.py into its own .so; never part of libzgpu.so).
// The host side is the product's own schema compiler and store; the mirror's sync (device.cu Device::ingress_sync)
// and the literal resolution (capi.cu ingress_literals) are restated over host memory, and the insert and resolve
// kernels run unchanged. Two switches exist only here: the tag filter can be turned off (every probe compares bytes)
// and the initial table shrunk (long probe chains, many rebuilds).
#define ZG_EMULATE 1
#include "cuda_emu.h"

// The insert kernel claims 64-bit slots; cuda_emu.h has the 32-bit atomicCAS only.
static inline unsigned long long atomicCAS(unsigned long long* p, unsigned long long expected, unsigned long long desired) {
  __atomic_compare_exchange_n(p, &expected, desired, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
  return expected;
}

#include <sys/mman.h>
#include <unistd.h>

#include <cstdio>
#include <cstring>
#include <string>

#include "../../spicedb-kubeapi-proxy_b200/csrc/ingress.cuh"
#include "../../spicedb-kubeapi-proxy_b200/csrc/store.h"

using namespace zg;

namespace {

struct MirrorType {
  std::vector<char> arena;                 // the device arena: a byte-for-byte copy
  std::vector<unsigned long long> offs;    // record offsets
  std::vector<unsigned long long> slots;   // the table
  uint64_t bytes = 0, cap = 0;
};

struct EmuIngress {
  Schema sc;
  Store store;
  std::vector<MirrorType> types;
  uint64_t names = 0, sync_uploads = 0, rebuilds = 0, items = 0;
};

struct EmuIngressOpts {
  uint64_t tag_mask;   // kIngressTagMask, or 0: no tag filter
  uint64_t min_table;  // the product's 1024, or smaller
  uint32_t grid, threads;
};

void sync(EmuIngress* e, const EmuIngressOpts& o) {
  e->types.resize(e->store.n_types());
  bool uploaded = false;
  for (size_t t = 0; t < e->types.size(); ++t) {
    const std::vector<char>& ar = e->store.name_arena(static_cast<int>(t));
    MirrorType& y = e->types[t];
    if (ar.size() == y.bytes) continue;
    uploaded = true;
    const uint64_t n_old = y.offs.size();
    for (uint64_t off = y.bytes; off < ar.size();) {
      uint32_t len;
      std::memcpy(&len, ar.data() + off + 4, 4);
      y.offs.push_back(off);
      off += 8 + uint64_t(len);
    }
    const uint64_t n_all = y.offs.size();
    y.arena.assign(ar.begin(), ar.end());
    uint64_t cap = y.cap ? y.cap : o.min_table;
    while (n_all * 2 > cap) cap *= 2;
    uint64_t from = n_old;
    if (cap != y.cap) {
      y.slots.assign(cap, 0);
      if (y.cap) ++e->rebuilds;
      y.cap = cap;
      from = 0;
    }
    IngressInsertParams p{};
    p.arena = reinterpret_cast<const uint8_t*>(y.arena.data());
    p.offs = y.offs.data();
    p.from = from;
    p.to = n_all;
    p.slots = y.slots.data();
    p.mask = cap - 1;
    zg_emu::launch(ingress_insert_kernel, p, o.grid, o.threads, 0);
    y.bytes = ar.size();
    e->names += n_all - n_old;
  }
  if (uploaded) ++e->sync_uploads;
}

}  // namespace

extern "C" {

void* emu_ing_create(const char* schema, char* err, size_t cap) {
  auto* e = new EmuIngress();
  const std::string m = e->sc.parse(schema);
  if (!m.empty()) {
    std::snprintf(err, cap, "%s", m.c_str());
    delete e;
    return nullptr;
  }
  e->store.reset(&e->sc);
  return e;
}
void emu_ing_destroy(void* h) { delete static_cast<EmuIngress*>(h); }
int emu_ing_type_id(void* h, const char* name) { return static_cast<EmuIngress*>(h)->sc.type_id(name); }

// zg_intern_objects_packed, restated (the emulator's store is its own)
int emu_ing_intern(void* h, int type, const char* ids, const uint32_t* off, uint64_t n, uint32_t* out) {
  auto* e = static_cast<EmuIngress*>(h);
  if (type < 0 || type >= static_cast<int>(e->sc.types.size())) return ZG_EINVAL;
  for (uint64_t i = 0; i < n; ++i) {
    if (off[i] == off[i + 1]) {
      out[i] = ZG_NO_OBJECT;
      continue;
    }
    out[i] = e->store.intern(type, std::string(ids + off[i], off[i + 1] - off[i]));
  }
  return ZG_OK;
}

int emu_ing_load(void* h, const zg_tuple* t, uint64_t n) {
  return static_cast<EmuIngress*>(h)->store.load(t, nullptr, n).empty() ? ZG_OK : ZG_EINVAL;
}

// capi.cu ingress_literals + Device::ingress_resolve over host memory. subj_off == nullptr: subj_ids is the one
// subject, NUL-terminated.
int emu_ing_resolve(void* h, const char* res_type, const char* relation, const char* subj_type, const char* subj_rel,
                    const char* res_ids, const uint32_t* res_off, const char* subj_ids, const uint32_t* subj_off,
                    uint64_t n, zg_check* out, const EmuIngressOpts* o) {
  auto* e = static_cast<EmuIngress*>(h);
  if (n == 0) return ZG_OK;
  sync(e, *o);
  // the literal fields: resolve_check's rules
  const bool none_rel = !subj_rel || !*subj_rel || std::strcmp(subj_rel, "...") == 0;
  zg_check base{ZG_NO_OBJECT, ZG_NO_OBJECT - 1, kNone, 0, kNone, 0};
  const int rt = e->sc.type_id(res_type), st = e->sc.type_id(subj_type);
  bool ok = false;
  if (rt >= 0 && st >= 0) {
    const int perm = e->sc.slot_id(rt, relation);
    const int sr = none_rel ? 0 : e->sc.slot_id(st, subj_rel);
    if (perm >= 0 && sr >= 0) {
      base.srel = none_rel ? kNone : static_cast<uint16_t>(sr);
      base.stype = static_cast<uint16_t>(st);
      base.perm = static_cast<uint16_t>(perm);
      ok = true;
    }
  }
  auto table = [&](int t) {
    IngressTable x{nullptr, nullptr, 0};
    if (ok && t >= 0 && t < static_cast<int>(e->types.size()) && e->types[t].cap) {
      x.arena = reinterpret_cast<const uint8_t*>(e->types[t].arena.data());
      x.slots = e->types[t].slots.data();
      x.mask = e->types[t].cap - 1;
    }
    return x;
  };
  IngressResolveParams p{};
  p.rt = table(rt);
  p.st = table(st);
  p.res_ids = reinterpret_cast<const uint8_t*>(res_ids);
  p.res_off = res_off;
  p.subj_ids = reinterpret_cast<const uint8_t*>(subj_ids);
  p.subj_off = subj_off;
  if (!subj_off) {
    p.one_len = std::strlen(subj_ids);
    p.one_su = ok ? e->store.find(st, subj_ids, p.one_len) : ZG_NO_OBJECT;
  }
  p.ok = ok ? 1 : 0;
  p.same_type = rt == st ? 1 : 0;
  p.base = base;
  p.n = n;
  p.tag_mask = o->tag_mask;
  p.out = out;
  unsigned bad = 0;
  p.bad = &bad;
  zg_emu::launch(ingress_resolve_kernel, p, o->grid, o->threads, 0);
  e->items += n;
  return bad ? ZG_EINVAL : ZG_OK;
}

void emu_ing_counters(void* h, uint64_t* out) {
  auto* e = static_cast<EmuIngress*>(h);
  out[0] = e->names;
  out[1] = e->sync_uploads;
  out[2] = e->rebuilds;
  out[3] = e->items;
}

// `bytes` of memory whose last byte sits just before a PROT_NONE page: a read past the end faults.
void* emu_guarded_alloc(size_t bytes) {
  const size_t pg = static_cast<size_t>(sysconf(_SC_PAGESIZE));
  const size_t body = (bytes + pg - 1) / pg * pg;
  char* m = static_cast<char*>(mmap(nullptr, body + pg, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0));
  if (m == MAP_FAILED) return nullptr;
  if (mprotect(m + body, pg, PROT_NONE) != 0) return nullptr;
  return m + body - bytes;
}

}  // extern "C"
