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

#include "../../include/zgpu.h"

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

}  // namespace zg
