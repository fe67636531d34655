// import.cuh -- zg_import_relationships on the device: resolve and deduplicate the names of an import, assemble its
// relationships and find the ones that are stored already or appear earlier in the call.
//
// The call's groups (one class each, packed like zg_check_bulk_packed) are staged as one blob of id bytes and one
// array of offsets. Every item has two name occurrences: o = 2 * item (the subject) and o = 2 * item + 1 (the
// resource), so occurrence order is first-appearance order: items in call order, the subject's name before the
// resource's. That is the order zg_write_relationships interns them in.
//
//   1. import_names_kernel: per occurrence, the id syntax check, the hash, a probe of the type's mirror (ingress.cuh);
//      a name the store does not have goes into a per-call table of new names, which keeps its first occurrence.
//   2. import_compact_kernel, a sort by (type, first occurrence) (CUB, in device.cu), import_rank_kernel: every new
//      name gets a temporary id, its type's id extent plus its rank, above every id the store has.
//   3. import_assemble_kernel: one zg_tuple per item and its page key K (PageKey); CUB sorts the keys.
//   4. import_adjacent_kernel (equal neighbours in K order) and import_locate_kernel (a binary search of the resident
//      forward row, as delta_locate_kernel does): the smallest call position of a duplicate.
//   5. import_remap_kernel: after the checks pass, the temporary ids become the real ones the host hands out.
// Steps 1-4 change nothing outside the call's scratch, so a failed import leaves the engine as it was.
#pragma once
#ifndef ZG_EMULATE  // tests/emu/: the same source under a CPU SIMT emulator (test infrastructure, never in libzgpu.so)
#include <cuda_runtime.h>
#endif
#include <cstdint>

#include "../../include/zgpu.h"
#include "ingress.cuh"
#include "schema.h"

namespace zg {

constexpr unsigned kImportThreads = 256;
constexpr uint32_t kImportMaxId = 1024;                  // longest object id (SpiceDB v1)
constexpr unsigned long long kImportNone = ~0ull;        // "no offender" / "no first occurrence"
constexpr uint32_t kImportNoSlot = 0xFFFFFFFFu;           // an occurrence whose name the store has

// One group of the call, as the kernels see it.
struct ImportGroupDev {
  unsigned long long item0;                // call position of its first item
  unsigned long long n;                    // its items
  unsigned long long res_blob, subj_blob;  // where its blobs start in the staged blob
  unsigned long long off0;                 // its res_off[0] in the staged offsets; subj_off follows at off0 + n + 1
  unsigned long long row_base;             // forward row table of its relation in the resident snapshot (DRel)
  uint32_t stride, nres;
  uint32_t rtype, stype;
  uint32_t rel, srel;                      // srel: that of a non-wildcard subject (kNone or a slot)
  uint32_t pos_plain, pos_wild;            // class positions in K (page_class_pos) of non-wildcard / wildcard items
  uint32_t k_plain, k_wild;                // class indexes within the relation (the forward row)
};

struct ImportCall {
  const ImportGroupDev* groups;
  uint32_t n_groups;
  const uint8_t* blob;
  const uint32_t* offs;
  unsigned long long n;  // items
};

__device__ __forceinline__ uint32_t import_group_of(const ImportCall& c, unsigned long long item) {
  uint32_t lo = 0, hi = c.n_groups;  // the last group whose item0 <= item
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) / 2;
    if (c.groups[mid].item0 <= item) lo = mid;
    else hi = mid;
  }
  return lo;
}

// The bytes, length and type of occurrence o.
__device__ __forceinline__ void import_occ(const ImportCall& c, unsigned long long o, const uint8_t** p, uint32_t* len,
                                           uint32_t* type) {
  const unsigned long long item = o >> 1;
  const ImportGroupDev& g = c.groups[import_group_of(c, item)];
  const unsigned long long j = item - g.item0;
  const bool res = o & 1;
  const uint32_t* off = c.offs + g.off0 + (res ? 0 : g.n + 1);
  const uint32_t b = off[j], e = off[j + 1];
  *p = c.blob + (res ? g.res_blob : g.subj_blob) + b;
  *len = e - b;
  *type = res ? g.rtype : g.stype;
}

__device__ __forceinline__ bool import_id_char(uint8_t ch) {
  return (ch >= 'a' && ch <= 'z') || (ch >= 'A' && ch <= 'Z') || (ch >= '0' && ch <= '9') || ch == '/' || ch == '_' ||
         ch == '|' || ch == '-' || ch == '=' || ch == '+';
}

// The per-call table of new names: u64 slots holding the top 24 bits of the name's hash mixed with its type (the
// tag) and `first occurrence claimed + 1`; power-of-two capacity of at least twice the occurrences, so it never fills.
__device__ __forceinline__ uint64_t import_slot_hash(uint64_t h, uint32_t type) {
  return h ^ ((uint64_t(type) + 1) * kHashMul);
}

struct ImportNamesParams {
  ImportCall c;
  const IngressTable* tables;       // per type: the mirror of the store's names (slots == nullptr: none)
  unsigned long long* slots;        // new-name table
  unsigned long long mask;          // its capacity - 1
  unsigned long long* first;        // per slot: the smallest occurrence of its name
  unsigned long long* hash;         // per slot: hash_bytes of its name
  uint32_t* slot_type;              // per slot: the name's type
  uint32_t* occ_id;                 // per occurrence: the store's id (ZG_NO_OBJECT: new, or the wildcard)
  uint32_t* occ_slot;               // per occurrence: its new-name slot, else kImportNoSlot
  unsigned long long* bad;          // the smallest call position with a malformed id
  unsigned long long tag_mask;      // kIngressTagMask; 0 makes every probe compare bytes (emulator tests)
  unsigned long long* found;        // occurrences the store had a name for
};

__global__ void __launch_bounds__(kImportThreads) import_names_kernel(const ImportNamesParams p) {
  const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
  unsigned long long found = 0;
  for (uint64_t o = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; o < 2 * p.c.n; o += stride) {
    const uint8_t* s;
    uint32_t len, type;
    import_occ(p.c, o, &s, &len, &type);
    p.occ_slot[o] = kImportNoSlot;
    p.occ_id[o] = ZG_NO_OBJECT;
    const bool is_res = o & 1;
    if (len == 1 && s[0] == '*') {  // the wildcard: a subject without a name, never a resource
      if (is_res) atomicMin(p.bad, static_cast<unsigned long long>(o >> 1));
      continue;
    }
    bool ok = len >= 1 && len <= kImportMaxId;
    for (uint32_t k = 0; ok && k < len; ++k) ok = import_id_char(s[k]);
    if (!ok) {
      atomicMin(p.bad, static_cast<unsigned long long>(o >> 1));
      continue;
    }
    const uint64_t h = ingress_hash(s, len);
    const uint32_t have = ingress_find(p.tables[type], s, len, h, p.tag_mask);
    if (have != ZG_NO_OBJECT) {
      p.occ_id[o] = have;
      ++found;
      continue;
    }
    const uint64_t hs = import_slot_hash(h, type);
    const unsigned long long mine = (hs & kIngressTagMask) | (o + 1);
    for (uint64_t i = hs & p.mask;; i = (i + 1) & p.mask) {
      unsigned long long v = p.slots[i];
      if (!v) {
        v = atomicCAS(&p.slots[i], 0ull, mine);
        if (!v) {  // claimed: the slot describes this name
          p.hash[i] = h;
          p.slot_type[i] = type;
          atomicMin(&p.first[i], static_cast<unsigned long long>(o));
          p.occ_slot[o] = static_cast<uint32_t>(i);
          break;
        }
      }
      if ((v ^ mine) & p.tag_mask) continue;
      const uint8_t* q;
      uint32_t qlen, qtype;
      import_occ(p.c, (v & kIngressOffMask) - 1, &q, &qlen, &qtype);
      if (qtype == type && qlen == len && ingress_equal(q, s, len)) {
        atomicMin(&p.first[i], static_cast<unsigned long long>(o));
        p.occ_slot[o] = static_cast<uint32_t>(i);
        break;
      }
    }
  }
  if (found) atomicAdd(p.found, found);
}

// Every claimed slot of the new-name table: key (type << 48 | first occurrence), value the slot, in no order.
__global__ void __launch_bounds__(kImportThreads) import_compact_kernel(const unsigned long long* slots, unsigned long long cap,
                                                                        const unsigned long long* first,
                                                                        const uint32_t* slot_type, unsigned long long* keys,
                                                                        uint32_t* vals, unsigned long long* count) {
  const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
  for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < cap; i += stride) {
    if (!slots[i]) continue;
    const unsigned long long at = atomicAdd(count, 1ull);
    keys[at] = (uint64_t(slot_type[i]) << 48) | first[i];
    vals[at] = static_cast<uint32_t>(i);
  }
}

// For the new names sorted by (type, first occurrence): the temporary id of each slot, its type's extent plus its
// rank within the type, and the names' hashes in that order (for the host's table).
__global__ void __launch_bounds__(kImportThreads) import_rank_kernel(const unsigned long long* keys, const uint32_t* vals,
                                                                     unsigned long long n_new, const uint32_t* extent,
                                                                     const unsigned long long* type_start,
                                                                     const unsigned long long* hash, uint32_t* slot_tmp,
                                                                     unsigned long long* out_hash) {
  const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
  for (uint64_t j = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; j < n_new; j += stride) {
    const uint32_t t = static_cast<uint32_t>(keys[j] >> 48);
    slot_tmp[vals[j]] = extent[t] + static_cast<uint32_t>(j - type_start[t]);
    out_hash[j] = hash[vals[j]];
  }
}

struct ImportAssembleParams {
  ImportCall c;
  const uint32_t* occ_id;
  const uint32_t* occ_slot;
  const uint32_t* slot_tmp;
  zg_tuple* tuples;              // per item, call order
  unsigned long long* key_hi;    // K: type << 32 | resource
  unsigned long long* key_lo;    // K: class position << 32 | subject (0 for the wildcard)
  uint32_t* vals;                // call position
  uint8_t* known;                // 1 when the store had both names: the only items the store can hold already
};

__global__ void __launch_bounds__(kImportThreads) import_assemble_kernel(const ImportAssembleParams p) {
  const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
  for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < p.c.n; i += stride) {
    const ImportGroupDev& g = p.c.groups[import_group_of(p.c, i)];
    const uint32_t so = p.occ_slot[2 * i], ro = p.occ_slot[2 * i + 1];
    const uint32_t res = ro == kImportNoSlot ? p.occ_id[2 * i + 1] : p.slot_tmp[ro];
    const uint32_t* off = p.c.offs + g.off0 + g.n + 1;
    const uint64_t j = i - g.item0;
    const bool wild = off[j + 1] - off[j] == 1 && p.c.blob[g.subj_blob + off[j]] == '*';
    zg_tuple t;
    t.res = res;
    t.rel = static_cast<uint16_t>(g.rel);
    t.stype = static_cast<uint16_t>(g.stype);
    t.flags = 0;
    t.srel = static_cast<uint16_t>(wild ? kWildcard : g.srel);
    t.subj = wild ? 0u : so == kImportNoSlot ? p.occ_id[2 * i] : p.slot_tmp[so];
    p.tuples[i] = t;
    p.key_hi[i] = (uint64_t(g.rtype) << 32) | res;
    p.key_lo[i] = (uint64_t(wild ? g.pos_wild : g.pos_plain) << 32) | t.subj;
    p.vals[i] = static_cast<uint32_t>(i);
    p.known[i] = ro == kImportNoSlot && (wild || so == kImportNoSlot);
  }
}

// The high words of K in the order `pos` lists the items (the first pass of the two-pass sort by K).
__global__ void __launch_bounds__(kImportThreads) import_gather_kernel(const unsigned long long* hi, const uint32_t* pos,
                                                                       unsigned long long n, unsigned long long* out) {
  const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
  for (uint64_t j = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; j < n; j += stride) out[j] = hi[pos[j]];
}

// pos: the call positions sorted stably by K (hi, lo: K by call position). An item whose key equals its
// predecessor's repeats an earlier item of the call.
__global__ void __launch_bounds__(kImportThreads) import_adjacent_kernel(const unsigned long long* hi, const unsigned long long* lo,
                                                                         const uint32_t* pos, unsigned long long n,
                                                                         unsigned long long* dup) {
  const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
  for (uint64_t j = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x + 1; j < n; j += stride) {
    const uint32_t a = pos[j - 1], b = pos[j];
    if (hi[a] == hi[b] && lo[a] == lo[b]) atomicMin(dup, static_cast<unsigned long long>(b));
  }
}

// Items whose names the store had, against the forward rows of the resident snapshot (every relationship of the store
// when it is current, expired ones not yet collected included). owner_count > 1: a shard of a sharded handle, which
// searches the items whose resource it owns.
struct ImportLocateParams {
  ImportCall c;
  const zg_tuple* tuples;
  const uint8_t* known;
  const uint32_t* row_ptr;
  const uint32_t* col;
  uint32_t owner_rank, owner_count;
  unsigned long long* dup;
};

__global__ void __launch_bounds__(kImportThreads) import_locate_kernel(const ImportLocateParams p) {
  const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
  for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < p.c.n; i += stride) {
    if (!p.known[i]) continue;
    const zg_tuple t = p.tuples[i];
    if (p.owner_count > 1 && t.res % p.owner_count != p.owner_rank) continue;
    const ImportGroupDev& g = p.c.groups[import_group_of(p.c, i)];
    if (t.res >= g.nres) continue;  // named after the last layout: no relationship has it
    const uint32_t k = t.srel == kWildcard ? g.k_wild : g.k_plain;
    const uint64_t row = g.row_base + uint64_t(t.res) * g.stride + k;
    uint32_t lo = p.row_ptr[row], hi = p.row_ptr[row + 1];
    while (lo < hi) {
      const uint32_t mid = lo + (hi - lo) / 2;
      if (p.col[mid] < t.subj) lo = mid + 1;
      else hi = mid;
    }
    if (lo < p.row_ptr[row + 1] && p.col[lo] == t.subj) atomicMin(p.dup, static_cast<unsigned long long>(i));
  }
}

// Temporary ids (>= the type's extent) to the ids the host hands out: ids[base[type] + tmp - extent[type]].
__global__ void __launch_bounds__(kImportThreads) import_remap_kernel(zg_tuple* tuples, unsigned long long n, const uint32_t* rtype_of_rel,
                                                                      const uint32_t* extent, const unsigned long long* base,
                                                                      const uint32_t* ids) {
  const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
  for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    zg_tuple t = tuples[i];
    const uint32_t rt = rtype_of_rel[t.rel];
    if (t.res >= extent[rt]) t.res = ids[base[rt] + t.res - extent[rt]];
    if (t.srel != kWildcard && t.subj >= extent[t.stype]) t.subj = ids[base[t.stype] + t.subj - extent[t.stype]];
    tuples[i] = t;
  }
}

}  // namespace zg
