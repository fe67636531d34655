// filter.cuh -- relationship filters (ReadRelationships, DeleteRelationships, write preconditions) answered from the
// resident CSR instead of a scan of the host store.
//
// The forward CSR is keyed by (resource, class) and the reverse CSR by (subject, class); a class fixes the relation,
// the subject type and the subject relation. So a filter selects a set of classes on the host (Device::match_filter)
// and the kernels below only walk rows of those classes. Three shapes, by what the filter names:
//   resource given            the row (resource, class) of every selected class; with a subject, a binary search in it
//   subject given, no resource  the subject's reverse row of every selected class
//   neither                   every row of the selected classes
// Every kernel counts its matches; the emitting instantiation also appends them as zg_tuple records (+ expirations).
// The host sizes the output from a count launch, so `cap` only guards: a record that does not fit is not written.
// No kernel reads past a row: an id at or beyond a table's object count matches nothing.
//
// filter_expired_kernel (zg_collect_expired) is the "neither" scan with another predicate: an entry matches when its
// expiration is set and at or before `now`, which it reads as the collection's `before`. Device::match_expired selects
// the classes that may carry an expiration (CF_EXPIRY) and no other.
#pragma once
#ifndef ZG_EMULATE  // tests/emu/: the same source under a CPU SIMT emulator (test infrastructure, never in libzgpu.so)
#include <cuda_runtime.h>
#endif
#include <cstdint>
#include <vector>

#include "../../include/zgpu.h"
#include "schema.h"

namespace zg {

constexpr int kMaxFilterSel = 64;  // selected classes per launch; a filter that selects more runs in several launches
constexpr unsigned kFilterThreads = 256;
constexpr unsigned kFilterFull = 0xFFFFFFFFu;

struct FilterSel {  // one selected (data relation, class)
  unsigned long long row_base;   // row_ptr index of (object 0, this class)
  unsigned long long rrow_base;  // rrow_ptr index of (subject 0, this class); a wildcard class has one row
  uint32_t nres, nsubj;          // objects / subjects the tables cover (nsubj = 1 for a wildcard class)
  uint32_t stride;               // forward row stride per object
  uint16_t rstride;              // reverse row stride per subject (0 for a wildcard class)
  uint16_t rel, stype, srel;     // what a record of this class says: relation slot, subject type, ZG_SREL_* or slot
  uint16_t pad;
};

struct FilterPlan {
  const uint32_t *row_ptr, *col, *exp, *rrow_ptr, *rcol;  // exp: nullptr when the schema has no expiration
  uint32_t n_sel;
  uint32_t has_subj;   // resource shape: only the entry `subj` of each row
  uint32_t res, subj;  // subj = 0 for the row of a wildcard class
  uint32_t now;        // 0: expired relationships match too
  zg_tuple* out;       // emit: cap records and their expirations
  uint32_t* out_exp;
  unsigned long long cap;
  unsigned long long* count;
  FilterSel sel[kMaxFilterSel];
};

__device__ __forceinline__ uint32_t filter_lower_bound(const uint32_t* a, uint32_t lo, uint32_t hi, uint32_t key) {
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (__ldg(a + mid) < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}
__device__ __forceinline__ bool filter_live(uint32_t expires, uint32_t now) { return now == 0 || expires == 0 || expires > now; }
__device__ __forceinline__ bool filter_expired(uint32_t expires, uint32_t before) { return expires != 0 && expires <= before; }

// Warp-collective: counts the lanes with `hit`, and (kEmit) appends their records behind one reservation.
template <bool kEmit>
__device__ __forceinline__ void filter_append(const FilterPlan& p, const FilterSel& s, bool hit, uint32_t res, uint32_t subj,
                                              uint32_t expires, unsigned lane) {
  const unsigned m = __ballot_sync(kFilterFull, hit);
  if (!m) return;
  unsigned long long at = 0;
  if (lane == 0) at = atomicAdd(p.count, static_cast<unsigned long long>(__popc(m)));
  if (!kEmit) return;
  at = __shfl_sync(kFilterFull, at, 0) + __popc(m & ((1u << lane) - 1u));
  if (hit && at < p.cap) {
    zg_tuple t;
    t.res = res;
    t.subj = s.srel == ZG_SREL_WILDCARD ? 0u : subj;
    t.rel = s.rel;
    t.stype = s.stype;
    t.srel = s.srel;
    t.flags = 0;
    p.out[at] = t;
    p.out_exp[at] = expires;
  }
}

// The entries [b, e) of the forward row of `res`, dealt out to the grid's warps 32 at a time. kExpired: the entries
// filter_expired selects instead of the live ones.
template <bool kEmit, bool kExpired = false>
__device__ __forceinline__ void filter_forward_row(const FilterPlan& p, const FilterSel& s, uint32_t res, uint32_t b, uint32_t e,
                                                   unsigned long long first, unsigned long long step, unsigned lane) {
  for (unsigned long long i0 = b + first; i0 < e; i0 += step) {
    const unsigned long long i = i0 + lane;
    bool hit = i < e;
    uint32_t subj = 0, ex = 0;
    if (hit) {
      subj = __ldg(p.col + i);
      if (p.exp) ex = __ldg(p.exp + i);
      hit = kExpired ? filter_expired(ex, p.now) : filter_live(ex, p.now);
    }
    filter_append<kEmit>(p, s, hit, res, subj, ex, lane);
  }
}

// Resource given. A long row (an organisation's members) is spread over every warp of the grid.
template <bool kEmit>
__global__ void __launch_bounds__(kFilterThreads) filter_resource_kernel(const FilterPlan p) {
  const unsigned lane = threadIdx.x & 31;
  const unsigned long long w = (blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x) >> 5;
  const unsigned long long n_warps = (static_cast<unsigned long long>(gridDim.x) * blockDim.x) >> 5;
  for (uint32_t k = 0; k < p.n_sel; ++k) {
    const FilterSel& s = p.sel[k];
    if (p.res >= s.nres) continue;
    const unsigned long long ri = s.row_base + static_cast<unsigned long long>(p.res) * s.stride;
    uint32_t b = __ldg(p.row_ptr + ri), e = __ldg(p.row_ptr + ri + 1);
    if (p.has_subj) {  // rows are sorted by subject id
      const uint32_t at = filter_lower_bound(p.col, b, e, p.subj);
      if (at < e && __ldg(p.col + at) == p.subj) b = at, e = at + 1;
      else e = b;
    }
    filter_forward_row<kEmit>(p, s, p.res, b, e, w * 32, n_warps * 32, lane);
  }
}

// Subject given, no resource: one relationship per entry of the subject's reverse row. The reverse CSR carries no
// expirations, so when they matter the entry is found again in the forward row of its resource.
template <bool kEmit>
__global__ void __launch_bounds__(kFilterThreads) filter_subject_kernel(const FilterPlan p) {
  const unsigned lane = threadIdx.x & 31;
  const unsigned long long w = (blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x) >> 5;
  const unsigned long long n_warps = (static_cast<unsigned long long>(gridDim.x) * blockDim.x) >> 5;
  const bool want_exp = p.exp && (kEmit || p.now);
  for (uint32_t k = 0; k < p.n_sel; ++k) {
    const FilterSel& s = p.sel[k];
    if (p.subj >= s.nsubj) continue;
    const unsigned long long ri = s.rrow_base + static_cast<unsigned long long>(p.subj) * s.rstride;
    const uint32_t b = __ldg(p.rrow_ptr + ri), e = __ldg(p.rrow_ptr + ri + 1);
    for (unsigned long long i0 = b + w * 32; i0 < e; i0 += n_warps * 32) {
      const unsigned long long i = i0 + lane;
      bool hit = i < e;
      uint32_t res = 0, ex = 0;
      if (hit) {
        res = __ldg(p.rcol + i);
        if (want_exp && res < s.nres) {
          const unsigned long long fi = s.row_base + static_cast<unsigned long long>(res) * s.stride;
          const uint32_t fb = __ldg(p.row_ptr + fi), fe = __ldg(p.row_ptr + fi + 1);
          const uint32_t at = filter_lower_bound(p.col, fb, fe, p.subj);
          if (at < fe && __ldg(p.col + at) == p.subj) ex = __ldg(p.exp + at);
        }
        hit = filter_live(ex, p.now);
      }
      filter_append<kEmit>(p, s, hit, res, p.subj, ex, lane);
    }
  }
}

// Neither: every row of the selected classes. A warp reads the offsets of 32 consecutive objects, one per lane, then
// works each non-empty row together. A count that does not depend on expirations needs the offsets only. kExpired:
// the entries filter_expired selects, which always depends on them. The plan is taken by value: inlined into the
// kernels it stays the kernel parameter, and filter_scan_kernel compiles to the SASS it had as a kernel of its own.
template <bool kEmit, bool kExpired>
__device__ __forceinline__ void filter_scan(const FilterPlan p) {
  const unsigned lane = threadIdx.x & 31;
  const unsigned long long w = (blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x) >> 5;
  const unsigned long long n_warps = (static_cast<unsigned long long>(gridDim.x) * blockDim.x) >> 5;
  const bool offsets_only = !kEmit && !kExpired && !(p.exp && p.now);
  for (uint32_t k = 0; k < p.n_sel; ++k) {
    const FilterSel& s = p.sel[k];
    for (unsigned long long obj0 = w * 32; obj0 < s.nres; obj0 += n_warps * 32) {
      const unsigned long long obj = obj0 + lane;
      uint32_t b = 0, e = 0;
      if (obj < s.nres) {
        const unsigned long long ri = s.row_base + obj * s.stride;
        b = __ldg(p.row_ptr + ri);
        e = __ldg(p.row_ptr + ri + 1);
      }
      if (offsets_only) {
        uint32_t sum = e - b;  // a 32-object group of one snapshot holds fewer than 2^32 entries
        for (int d = 16; d > 0; d >>= 1) sum += __shfl_xor_sync(kFilterFull, sum, d);
        if (lane == 0 && sum) atomicAdd(p.count, static_cast<unsigned long long>(sum));
        continue;
      }
      unsigned rows = __ballot_sync(kFilterFull, e > b);
      while (rows) {
        const int src = __ffs(rows) - 1;
        rows &= rows - 1;
        const uint32_t rb = __shfl_sync(kFilterFull, b, src), re = __shfl_sync(kFilterFull, e, src);
        filter_forward_row<kEmit, kExpired>(p, s, static_cast<uint32_t>(obj0 + src), rb, re, 0, 32, lane);
      }
    }
  }
}

template <bool kEmit>
__global__ void __launch_bounds__(kFilterThreads) filter_scan_kernel(const FilterPlan p) {
  filter_scan<kEmit, false>(p);
}

// Expired relationships of the selected classes: p.now is the collection's `before` (never 0).
template <bool kEmit>
__global__ void __launch_bounds__(kFilterThreads) filter_expired_kernel(const FilterPlan p) {
  filter_scan<kEmit, true>(p);
}

// ---- which ids the snapshot mentions (zg_retire_unused_names) ----
// An id of type T is mentioned when some relationship names it as its resource or as its subject. The forward rows of
// object o (every class of T's relations) sit together at fwd_base + o * fwd_stride, its reverse rows (every class T
// can be a subject of, wildcard classes aside) at rev_base + o * rev_stride (DESIGN §3), so "o has a non-empty row" is
// one difference of two offsets per direction. A warp covers 32 ids, one per lane, and its ballot is their bitmap
// word: every word is written once, with no atomics. Expired entries still mention their ids; wildcard rows mention
// none (their single reverse row lies outside every type's block, their forward entries name only the resource).
// Device::scan_mentions plans from the snapshot's layout (mention_types) and ORs the bitmaps of a sharded handle's
// shards; Store::mentioned builds the same bitmaps from the relationship list.
constexpr int kMaxMentionTypes = 64;  // types per launch; a schema with more runs several launches

struct MentionType {
  unsigned long long fwd_base;  // row_ptr index of (object 0, the type's first class)
  unsigned long long rev_base;  // rrow_ptr index of (object 0, the first class the type is a subject of)
  unsigned long long word0;     // the type's first word of `bits`
  uint32_t n_ids;               // the type's object capacity: bits cover ceil(n_ids / 32) words
  uint32_t fwd_stride;          // classes of the type's relations; 0: the type has none
  uint32_t rev_stride;          // classes the type is a subject of; 0: none
  uint32_t pad;
};

struct MentionPlan {
  const uint32_t *row_ptr, *rrow_ptr;
  uint32_t* bits;
  uint32_t n_types;
  MentionType type[kMaxMentionTypes];
};

__global__ void __launch_bounds__(kFilterThreads) mention_scan_kernel(const MentionPlan p) {
  const unsigned lane = threadIdx.x & 31;
  const unsigned long long w = (blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x) >> 5;
  const unsigned long long n_warps = (static_cast<unsigned long long>(gridDim.x) * blockDim.x) >> 5;
  for (uint32_t k = 0; k < p.n_types; ++k) {
    const MentionType& t = p.type[k];
    const unsigned long long words = (static_cast<unsigned long long>(t.n_ids) + 31) >> 5;
    for (unsigned long long wd = w; wd < words; wd += n_warps) {
      const unsigned long long o = wd * 32 + lane;
      bool hit = false;
      if (o < t.n_ids) {
        if (t.fwd_stride) {
          const unsigned long long r = t.fwd_base + o * t.fwd_stride;
          hit = __ldg(p.row_ptr + r + t.fwd_stride) != __ldg(p.row_ptr + r);
        }
        if (!hit && t.rev_stride) {
          const unsigned long long r = t.rev_base + o * t.rev_stride;
          hit = __ldg(p.rrow_ptr + r + t.rev_stride) != __ldg(p.rrow_ptr + r);
        }
      }
      const unsigned word = __ballot_sync(kFilterFull, hit);
      if (lane == 0) p.bits[t.word0 + wd] = word;
    }
  }
}

// The plan of every type of a snapshot's layout (its rels, cls and object capacities), bitmaps back to back in type
// order. Returns the words they take. A type's first relation starts its forward block (Store::layout hands out the
// rows of a type's relations in order), and its reverse block starts at the least rrow_base of its classes.
inline uint64_t mention_types(const Schema& sc, const std::vector<DRel>& rels, const std::vector<DCls>& cls,
                              const std::vector<uint32_t>& n_objects, std::vector<MentionType>* out) {
  out->assign(n_objects.size(), MentionType{});
  uint64_t words = 0;
  for (size_t t = 0; t < n_objects.size(); ++t) {
    MentionType& m = (*out)[t];
    m.n_ids = n_objects[t];
    m.word0 = words;
    words += (uint64_t(n_objects[t]) + 31) / 32;
    for (size_t ri = 0; ri < sc.rel_slots.size() && ri < rels.size(); ++ri)
      if (sc.slots[sc.rel_slots[ri]].type == static_cast<int>(t)) {
        m.fwd_base = rels[ri].row_base;
        m.fwd_stride = rels[ri].stride;
        break;
      }
    for (const DCls& c : cls)
      if (c.stype == t && c.sslot != kWildcard && (!m.rev_stride || c.rrow_base < m.rev_base)) {
        m.rev_base = c.rrow_base;
        m.rev_stride = c.rstride;
      }
  }
  return words;
}

}  // namespace zg
