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
#include <algorithm>
#include <cstdint>
#include <utility>
#include <vector>

#include "../../include/zgpu.h"
#include "schema.h"
#include "store.h"

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
  uint16_t pos;                  // pages: the class position, the class's index in its type's forward row block
  uint16_t rtype;                // pages: the resource type
};
static_assert(sizeof(FilterSel) == 40, "FilterSel is the plans' array element: two fields fill its tail padding");

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
  // kPrefix instantiations: per selected class, its resource type's bitmap of the ids whose name has the filter's
  // prefix (prefix_match_kernel). Last, so that the fields above keep their offsets.
  const uint32_t* bits[kMaxFilterSel];
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
// Bit `id` of a prefix bitmap covering `n` ids: the id's name has the prefix.
__device__ __forceinline__ bool filter_bit(const uint32_t* bits, uint32_t id, uint32_t n) {
  return id < n && (__ldg(bits + (id >> 5)) >> (id & 31) & 1u);
}
// The expiration of (res, subj) in class s, found in res's forward row (res < s.nres); 0 when absent.
__device__ __forceinline__ uint32_t filter_find_exp(const uint32_t* row_ptr, const uint32_t* col, const uint32_t* exp,
                                                    const FilterSel& s, uint32_t res, uint32_t subj) {
  const unsigned long long fi = s.row_base + static_cast<unsigned long long>(res) * s.stride;
  const uint32_t fb = __ldg(row_ptr + fi), fe = __ldg(row_ptr + fi + 1);
  const uint32_t at = filter_lower_bound(col, fb, fe, subj);
  return at < fe && __ldg(col + at) == subj ? __ldg(exp + at) : 0u;
}

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
template <bool kEmit, bool kPrefix = false>
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
      // kPrefix: an entry whose resource's bit is clear is dropped before its expiration is looked up. The two
      // branches are kept apart so that the unprefixed instantiations compile to the code they always had.
      if constexpr (kPrefix) {
        if (hit) {
          res = __ldg(p.rcol + i);
          hit = filter_bit(p.bits[k], res, s.nres);
          if (hit && want_exp) ex = filter_find_exp(p.row_ptr, p.col, p.exp, s, res, p.subj);
          hit = hit && filter_live(ex, p.now);
        }
      } else if (hit) {
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
// kPrefix: only the objects whose bit is set in the class's prefix bitmap. A warp's 32 objects are 32-aligned, so they
// are one bitmap word, read before any row offset: a word of unmatched objects costs that one load.
template <bool kEmit, bool kExpired, bool kPrefix = false>
__device__ __forceinline__ void filter_scan(const FilterPlan p) {
  const unsigned lane = threadIdx.x & 31;
  const unsigned long long w = (blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x) >> 5;
  const unsigned long long n_warps = (static_cast<unsigned long long>(gridDim.x) * blockDim.x) >> 5;
  const bool offsets_only = !kEmit && !kExpired && !(p.exp && p.now);
  for (uint32_t k = 0; k < p.n_sel; ++k) {
    const FilterSel& s = p.sel[k];
    for (unsigned long long obj0 = w * 32; obj0 < s.nres; obj0 += n_warps * 32) {
      uint32_t word = kFilterFull;
      if (kPrefix) {
        word = __ldg(p.bits[k] + (obj0 >> 5));
        if (!word) continue;
      }
      const unsigned long long obj = obj0 + lane;
      uint32_t b = 0, e = 0;
      if (obj < s.nres && (!kPrefix || (word >> lane & 1u))) {
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

template <bool kEmit, bool kPrefix = false>
__global__ void __launch_bounds__(kFilterThreads) filter_scan_kernel(const FilterPlan p) {
  filter_scan<kEmit, false, kPrefix>(p);
}

// Expired relationships of the selected classes: p.now is the collection's `before` (never 0).
template <bool kEmit>
__global__ void __launch_bounds__(kFilterThreads) filter_expired_kernel(const FilterPlan p) {
  filter_scan<kEmit, true>(p);
}

// ---- pages of a filter (zg_read_relationships_page, zg_delete_relationships_limited) ----
// A page is the first `want` (= limit + 1) live matches whose key K = (resource type, resource, class position,
// subject) follows the cursor's key, in K order. Within one resource type K is the physical order of `col`: row_ptr is
// object-major over every class of the type (DESIGN §3), and a row is sorted by subject. The host selects one type's
// classes, sorted by position, and walks windows of its objects:
//   page_window_kernel  from row_ptr alone, the least window end at which `entries` entries of the block follow
//   page_count_kernel   per tile (32 objects x the selected classes) its matches, stopping at `want`
//   (cub::DeviceScan)   exclusive offsets of the tile counts
//   page_emit_kernel    every tile that starts before `want` writes its matches at its offset, in K order
// The resource shape is the window of one object. The subject shape (page_subject_kernel) takes at most `want` live
// entries after the cursor from the subject's reverse row of every selected class; the host merges them into K order.
struct PagePlan {
  const uint32_t *row_ptr, *col, *exp, *rrow_ptr, *rcol;  // exp: nullptr when the schema has no expiration
  uint32_t n_sel;
  uint32_t has_subj, subj;  // resource shape: only the entry `subj` of each row; subject shape: the subject (0: "*")
  uint32_t now;             // 0: expired relationships match too
  uint32_t has_after;       // the start key: only entries with K > (after_type, after_res, after_pos, after_subj)
  uint32_t after_type, after_res, after_pos, after_subj;
  uint32_t obj0, obj1;      // the window [obj0, obj1) of the type's objects
  uint32_t pad;
  unsigned long long want;  // matches still wanted: a tile stops counting there, and nothing is written past it
  unsigned long long* tile_count;     // count: per tile (n_tiles + 1 entries, the last one 0)
  const unsigned long long* tile_off; // emit: their exclusive scan
  zg_tuple* out;                      // emit: `want` records and expirations; subject shape: n_sel segments of `want`
  uint32_t* out_exp;
  uint32_t* seg_count;                // subject shape: per selected class, the entries written to its segment
  FilterSel sel[kMaxFilterSel];
  const uint32_t* bits[kMaxFilterSel];  // kPrefix: as FilterPlan::bits
};

// The entries of (object o, class s) a page may return: past the start key when o is the cursor's object, and only
// `subj` with has_subj. o < s.nres.
__device__ __forceinline__ void page_row(const PagePlan& p, const FilterSel& s, uint32_t o, uint32_t* b, uint32_t* e) {
  const unsigned long long ri = s.row_base + static_cast<unsigned long long>(o) * s.stride;
  *b = __ldg(p.row_ptr + ri);
  *e = __ldg(p.row_ptr + ri + 1);
  if (p.has_after && o == p.after_res) {
    if (s.pos < p.after_pos || (s.pos == p.after_pos && p.after_subj == 0xFFFFFFFFu)) *e = *b;
    else if (s.pos == p.after_pos) *b = filter_lower_bound(p.col, *b, *e, p.after_subj + 1);
  }
  if (p.has_subj) {
    const uint32_t at = filter_lower_bound(p.col, *b, *e, p.subj);
    if (at < *e && __ldg(p.col + at) == p.subj) *b = at, *e = at + 1;
    else *e = *b;
  }
}

// One thread: the least obj1 in (obj0, nres] at which at least `entries` entries of the type's block follow obj0
// (nres when fewer do), and how many do. `block` = row_ptr index of (object 0, class position 0) of the type.
__global__ void page_window_kernel(const uint32_t* row_ptr, unsigned long long block, uint32_t stride, uint32_t obj0,
                                   uint32_t nres, unsigned long long entries, unsigned long long* out) {
  if (threadIdx.x | blockIdx.x) return;
  const uint32_t at0 = __ldg(row_ptr + block + static_cast<unsigned long long>(obj0) * stride);
  uint32_t lo = obj0 + 1, hi = nres;
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (__ldg(row_ptr + block + static_cast<unsigned long long>(mid) * stride) - at0 < entries) lo = mid + 1; else hi = mid;
  }
  out[0] = lo;
  out[1] = __ldg(row_ptr + block + static_cast<unsigned long long>(lo) * stride) - at0;
}

// Warp-collective walk of tile t: its matches in K order. kEmit: written from `base` on, never at or past p.want.
// Returns how many it found, counting stopping once `base` + that reaches p.want.
// kPrefix: only objects whose bit is set; the classes of a window share one resource type and so one bitmap, and a tile
// none of whose objects is set returns before it loads a row offset.
template <bool kEmit, bool kPrefix = false>
__device__ __forceinline__ unsigned long long page_tile(const PagePlan& p, unsigned long long t, unsigned long long base,
                                                        unsigned lane) {
  const unsigned long long o64 = p.obj0 + t * 32 + lane;
  bool mine = o64 < p.obj1;
  const uint32_t o = static_cast<uint32_t>(o64);
  if (kPrefix) {
    mine = mine && filter_bit(p.bits[0], o, p.sel[0].nres);
    if (!__ballot_sync(kFilterFull, mine)) return 0;
  }
  // the lane's object: does it have an entry the page may return, and how many (offsets only)
  unsigned long long n = 0;
  if (mine)
    for (uint32_t k = 0; k < p.n_sel; ++k) {
      if (o >= p.sel[k].nres) continue;
      uint32_t b, e;
      page_row(p, p.sel[k], o, &b, &e);
      n += e - b;
    }
  if (!kEmit && !(p.exp && p.now)) {  // without expirations a count needs the offsets only
    for (int d = 16; d > 0; d >>= 1) n += __shfl_xor_sync(kFilterFull, n, d);
    return n;
  }
  unsigned long long got = 0;
  unsigned objs = __ballot_sync(kFilterFull, n != 0);
  while (objs && base + got < p.want) {
    const int src = __ffs(objs) - 1;
    objs &= objs - 1;
    const uint32_t ob = static_cast<uint32_t>(p.obj0 + t * 32 + src);
    for (uint32_t k = 0; k < p.n_sel && base + got < p.want; ++k) {
      const FilterSel& s = p.sel[k];
      if (ob >= s.nres) continue;
      uint32_t b, e;
      page_row(p, s, ob, &b, &e);
      for (uint32_t i0 = b; i0 < e && base + got < p.want; i0 += 32) {
        const uint32_t i = i0 + lane;
        bool hit = i < e;
        uint32_t subj = 0, ex = 0;
        if (hit) {
          subj = __ldg(p.col + i);
          if (p.exp) ex = __ldg(p.exp + i);
          hit = filter_live(ex, p.now);
        }
        const unsigned m = __ballot_sync(kFilterFull, hit);
        const unsigned long long at = base + got + __popc(m & ((1u << lane) - 1u));
        if (kEmit && hit && at < p.want) {
          zg_tuple r;
          r.res = ob;
          r.subj = s.srel == ZG_SREL_WILDCARD ? 0u : subj;
          r.rel = s.rel;
          r.stype = s.stype;
          r.srel = s.srel;
          r.flags = 0;
          p.out[at] = r;
          p.out_exp[at] = ex;
        }
        got += __popc(m);
      }
    }
  }
  return got;
}

template <bool kPrefix = false>
__global__ void __launch_bounds__(kFilterThreads) page_count_kernel(const PagePlan p) {
  const unsigned lane = threadIdx.x & 31;
  const unsigned long long w = (blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x) >> 5;
  const unsigned long long n_warps = (static_cast<unsigned long long>(gridDim.x) * blockDim.x) >> 5;
  const unsigned long long tiles = (static_cast<unsigned long long>(p.obj1 - p.obj0) + 31) >> 5;
  for (unsigned long long t = w; t < tiles; t += n_warps) {
    const unsigned long long n = page_tile<false, kPrefix>(p, t, 0, lane);
    if (lane == 0) p.tile_count[t] = n;
  }
}

template <bool kPrefix = false>
__global__ void __launch_bounds__(kFilterThreads) page_emit_kernel(const PagePlan p) {
  const unsigned lane = threadIdx.x & 31;
  const unsigned long long w = (blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x) >> 5;
  const unsigned long long n_warps = (static_cast<unsigned long long>(gridDim.x) * blockDim.x) >> 5;
  const unsigned long long tiles = (static_cast<unsigned long long>(p.obj1 - p.obj0) + 31) >> 5;
  for (unsigned long long t = w; t < tiles; t += n_warps) {
    const unsigned long long base = __ldg(p.tile_off + t);
    if (base >= p.want) continue;  // tiles are in K order: every later one starts at or past it too
    if (__ldg(p.tile_count + t)) page_tile<true, kPrefix>(p, t, base, lane);
  }
}

// Subject given, no resource: one warp per selected class. Its reverse row is sorted by resource, and K orders by
// (type, resource, class position, subject) with the type, the position and the subject fixed for the row, so the
// entries after the cursor are a suffix of the row. The first `want` live ones go to the class's segment in order;
// expirations are found again in the forward row, as filter_subject_kernel does. kPrefix: only entries whose resource's
// bit is set in the class's bitmap.
template <bool kPrefix = false>
__global__ void __launch_bounds__(32) page_subject_kernel(const PagePlan p) {
  const unsigned lane = threadIdx.x & 31;
  for (uint32_t k = blockIdx.x; k < p.n_sel; k += gridDim.x) {
    const FilterSel& s = p.sel[k];
    unsigned long long got = 0;
    uint32_t start = 0;
    bool none = p.subj >= s.nsubj;
    if (p.has_after && !none) {
      if (s.rtype < p.after_type) none = true;
      else if (s.rtype == p.after_type) {  // (pos, subj) > (after_pos, after_subj): the cursor's resource is in
        const bool same_res_after = s.pos > p.after_pos || (s.pos == p.after_pos && p.subj > p.after_subj);
        if (same_res_after) start = p.after_res;
        else if (p.after_res == 0xFFFFFFFFu) none = true;
        else start = p.after_res + 1;
      }
    }
    if (!none) {
      const unsigned long long ri = s.rrow_base + static_cast<unsigned long long>(p.subj) * s.rstride;
      const uint32_t e = __ldg(p.rrow_ptr + ri + 1);
      const uint32_t b = filter_lower_bound(p.rcol, __ldg(p.rrow_ptr + ri), e, start);
      zg_tuple* out = p.out + k * p.want;
      uint32_t* out_exp = p.out_exp + k * p.want;
      for (uint32_t i0 = b; i0 < e && got < p.want; i0 += 32) {
        const uint32_t i = i0 + lane;
        bool hit = i < e;
        uint32_t res = 0, ex = 0;
        if constexpr (kPrefix) {  // as in filter_subject_kernel
          if (hit) {
            res = __ldg(p.rcol + i);
            hit = filter_bit(p.bits[k], res, s.nres);
            if (hit && p.exp) ex = filter_find_exp(p.row_ptr, p.col, p.exp, s, res, p.subj);
            hit = hit && filter_live(ex, p.now);
          }
        } else if (hit) {
          res = __ldg(p.rcol + i);
          if (p.exp && res < s.nres) {
            const unsigned long long fi = s.row_base + static_cast<unsigned long long>(res) * s.stride;
            const uint32_t fb = __ldg(p.row_ptr + fi), fe = __ldg(p.row_ptr + fi + 1);
            const uint32_t at = filter_lower_bound(p.col, fb, fe, p.subj);
            if (at < fe && __ldg(p.col + at) == p.subj) ex = __ldg(p.exp + at);
          }
          hit = filter_live(ex, p.now);
        }
        const unsigned m = __ballot_sync(kFilterFull, hit);
        const unsigned long long at = got + __popc(m & ((1u << lane) - 1u));
        if (hit && at < p.want) {
          zg_tuple r;
          r.res = res;
          r.subj = p.subj;
          r.rel = s.rel;
          r.stype = s.stype;
          r.srel = s.srel;
          r.flags = 0;
          out[at] = r;
          out_exp[at] = ex;
        }
        got += __popc(m);
      }
    }
    if (lane == 0) p.seg_count[k] = static_cast<uint32_t>(got < p.want ? got : p.want);
  }
}

// ---- the host side of a page: shared by Device::page_filter and the emulator's tests ----
inline void page_set_after(PagePlan& p, const PageKey* after) {
  p.has_after = after != nullptr;
  if (after) p.after_type = after->type, p.after_res = after->res, p.after_pos = after->pos, p.after_subj = after->subj;
}

// The scan and resource shapes: the classes `sel` (one plan's worth or fewer per type, sorted by type and position; a
// class's row_base - pos is its type's block) walked type by type, window by window, until `want` matches are found.
// Ops supplies the launches:
//   int window(const PagePlan&, block, stride, obj0, entries, *obj1, *n)   page_window_kernel, its answer copied back
//   int tiles(PagePlan&, got, *total)   count launch, scan and emit launch into the output from record `got` on, and
//                                       how many the window holds (the emit writes at most p.want of them)
// The first window of a type asks for `want - got` entries of the block; every window that comes up short (expired
// entries, classes not selected, the cursor's object) asks for at least twice as many as the one before it, more when
// its density of matches says the rest of the page needs more. *scanned: the entries of the block the windows
// covered. `bits` (optional, parallel to sel): the classes' prefix bitmaps, copied into p.bits with them. Returns 0 or
// what an op returned.
template <class Ops>
int page_walk(Ops& ops, PagePlan& p, const std::vector<FilterSel>& sel, bool by_resource, uint32_t res, const PageKey* after,
              unsigned long long want, unsigned long long* got, uint64_t* scanned,
              const std::vector<const uint32_t*>* bits = nullptr) {
  *got = 0;
  for (size_t g = 0; g < sel.size() && *got < want;) {
    size_t g1 = g;
    while (g1 < sel.size() && sel[g1].rtype == sel[g].rtype) ++g1;
    if (g1 - g > static_cast<size_t>(kMaxFilterSel)) return ZG_EINVAL;  // the caller pages such a type on the host
    const uint32_t type = sel[g].rtype, nres = sel[g].nres;
    p.n_sel = static_cast<uint32_t>(g1 - g);
    std::copy(sel.begin() + g, sel.begin() + g1, p.sel);
    if (bits) std::copy(bits->begin() + g, bits->begin() + g1, p.bits);
    g = g1;
    const bool at_cursor = after && after->type == type;
    if (after && type < after->type) continue;
    uint32_t obj = at_cursor ? after->res : 0, end = nres;
    if (by_resource) {
      if (at_cursor && res < after->res) continue;
      obj = res;
      end = res < nres ? res + 1 : res;
    }
    page_set_after(p, at_cursor ? after : nullptr);
    unsigned long long ask = want - *got;
    while (obj < end && *got < want) {
      uint32_t obj1 = end;
      unsigned long long n = 0;
      if (!by_resource)
        if (int rc = ops.window(p, p.sel[0].row_base - p.sel[0].pos, p.sel[0].stride, obj, ask, &obj1, &n)) return rc;
      p.obj0 = obj;
      p.obj1 = obj1;
      p.want = want - *got;
      unsigned long long total = 0;
      if (int rc = ops.tiles(p, *got, &total)) return rc;
      *scanned += by_resource ? total : n;
      *got += total < p.want ? total : p.want;
      obj = obj1;
      // the next window: at least twice this one, and as many entries as this window's density of matches says the
      // rest of the page needs, with a quarter more
      const unsigned long long left = want - *got;
      unsigned long long next = ask * 2;
      if (total && n / total < (1ull << 20)) next = std::max(next, left * (n / total + 1) + left / 4);
      ask = std::min(next, 1ull << 40);
    }
  }
  return 0;
}

// ---- selective pages of a prefix filter ----
// page_window_kernel sizes a window from row_ptr alone: with a prefix that matches few objects it would walk window
// after window of unmatched ones. A prefix page instead compacts a type's bitmap into the ascending list of its
// matched ids, with the exclusive sum of their entries in the type's block, and sizes windows over list positions:
//   prefix_word_count_kernel  per bitmap word, its set bits (then an exclusive scan gives each word's first position)
//   prefix_list_kernel        every matched id at its position, with its entries in the block
//   (exclusive scan of the entries)
//   prefix_window_kernel      the window from obj0 of at least `entries` entries of matched objects
// so the launches of a page depend on the matches it walks, never on the unmatched objects between them.
__global__ void __launch_bounds__(kFilterThreads) prefix_word_count_kernel(const uint32_t* bits, uint32_t words,
                                                                          uint32_t* count) {
  const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
  for (uint64_t w = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; w <= words; w += stride)
    count[w] = w < words ? __popc(__ldg(bits + w)) : 0u;
}

// ids[pos] = the matched id, ent[pos] = its entries in the block at (row_ptr + block, stride); ent[m] = 0.
__global__ void __launch_bounds__(kFilterThreads) prefix_list_kernel(const uint32_t* bits, uint32_t words, const uint32_t* first,
                                                                     const uint32_t* row_ptr, unsigned long long block,
                                                                     uint32_t stride, uint32_t nres, uint32_t* ids,
                                                                     unsigned long long* ent) {
  const uint64_t step = uint64_t(gridDim.x) * blockDim.x;
  for (uint64_t w = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; w <= words; w += step) {
    if (w == words) {
      ent[__ldg(first + words)] = 0;
      continue;
    }
    uint32_t word = __ldg(bits + w), pos = __ldg(first + w);
    while (word) {
      const uint32_t id = static_cast<uint32_t>(w * 32) + (__ffs(word) - 1);
      word &= word - 1;
      unsigned long long n = 0;
      if (id < nres) {
        const unsigned long long r = block + static_cast<unsigned long long>(id) * stride;
        n = __ldg(row_ptr + r + stride) - __ldg(row_ptr + r);
      }
      ids[pos] = id;
      ent[pos] = n;
      ++pos;
    }
  }
}

// One thread: from the first list position i whose id >= obj0, the least j in (i, m] at which the matched objects
// [i, j) hold at least `entries` entries (m when fewer do); out[0] = obj1 (ids[j], or nres at the list's end), out[1]
// = their entries. csum: the exclusive sum of the list's entries (m + 1 values).
__global__ void prefix_window_kernel(const uint32_t* ids, const unsigned long long* csum, uint32_t m, uint32_t obj0,
                                     uint32_t nres, unsigned long long entries, unsigned long long* out) {
  if (threadIdx.x | blockIdx.x) return;
  uint32_t i = filter_lower_bound(ids, 0, m, obj0);
  if (i == m) {
    out[0] = nres;
    out[1] = 0;
    return;
  }
  const unsigned long long at0 = __ldg(csum + i);
  uint32_t lo = i + 1, hi = m;
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (__ldg(csum + mid) - at0 < entries) lo = mid + 1; else hi = mid;
  }
  out[0] = lo < m ? __ldg(ids + lo) : nres;
  out[1] = __ldg(csum + lo) - at0;
}

// The subject shape: the segments of page_subject_kernel (seg_count[k] records of class sel[k] at rec + k * want),
// merged into K order and cut at `want`.
inline void page_merge(const std::vector<FilterSel>& sel, const uint32_t* seg_count, const zg_tuple* rec, const uint32_t* rec_exp,
                       unsigned long long want, std::vector<zg_tuple>* out, std::vector<uint32_t>* out_exp) {
  std::vector<std::pair<PageKey, uint64_t>> keys;
  for (size_t k = 0; k < sel.size(); ++k)
    for (uint64_t i = 0; i < seg_count[k]; ++i) {
      const zg_tuple& t = rec[k * want + i];
      keys.push_back({PageKey{sel[k].rtype, t.res, sel[k].pos, t.subj}, k * want + i});
    }
  const size_t n = static_cast<size_t>(std::min<unsigned long long>(want, keys.size()));
  std::partial_sort(keys.begin(), keys.begin() + n, keys.end(),
                    [](const auto& a, const auto& b) { return a.first < b.first; });
  for (size_t i = 0; i < n; ++i) {
    out->push_back(rec[keys[i].second]);
    out_exp->push_back(rec_exp[keys[i].second]);
  }
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
