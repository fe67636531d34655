// delta.cuh -- kernels and host preparation of the incremental publish (see build.cu gpu_apply_delta).
// Kept apart from build.cu (which needs cub) so that tests/emu/ can run the same kernels on the CPU emulator.
#pragma once
#ifndef ZG_EMULATE
#include <cuda_runtime.h>
#ifndef ZG_BLOCK_SHARED_U32
#define ZG_BLOCK_SHARED_U32(name, n) __shared__ uint32_t name[n]
#endif
#endif

#include <algorithm>
#include <cstdint>
#include <string>
#include <unordered_map>
#include <vector>

#include "schema.h"
#include "store.h"

namespace zg {
// ---- incremental publish: merge a small sorted delta into the resident CSR ---------------------
//
// A WriteRelationships carries <= 1000 updates (pkg/spicedb/spicedb.go:34) against a store of up to 1e8
// relationships; rebuilding (two radix sorts of the whole store) costs 0.65 s there. Instead the delta is
// located in the old arrays (binary search inside the affected rows), the edge arrays are re-emitted in ONE
// streaming pass (a tile with no update inside is a constant-shift copy: HBM-bound, ~1.5 GB for 95 M
// relationships), and the row tables get the running count of inserts minus deletes added in place. No
// overlay for the check kernel to consult: readers always see one plain CSR.



struct DeltaDev {
  const unsigned long long* ins_key;
  const uint32_t* ins_val;
  const uint32_t* ins_exp;
  uint32_t* ins_pos;
  uint32_t n_ins;
  const unsigned long long* del_key;
  const uint32_t* del_val;
  uint32_t* del_pos;
  uint32_t n_del;
  const unsigned long long* tch_key;
  const uint32_t* tch_val;
  const uint32_t* tch_exp;
  uint32_t* tch_pos;
  uint32_t n_tch;
};

__device__ __forceinline__ uint32_t lower_bound_u32(const uint32_t* a, uint32_t lo, uint32_t hi, uint32_t key) {
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (a[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}
// #{i : a[i] <= x} and #{i : a[i] < x} over an ascending array
__device__ __forceinline__ uint32_t count_le(const uint32_t* a, uint32_t n, uint32_t x) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (a[mid] <= x) lo = mid + 1; else hi = mid;
  }
  return lo;
}
__device__ __forceinline__ uint32_t count_lt(const uint32_t* a, uint32_t n, uint32_t x) { return lower_bound_u32(a, 0, n, x); }
__device__ __forceinline__ uint32_t count_lt64(const unsigned long long* a, uint32_t n, unsigned long long x) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (a[mid] < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// position of every delta entry in the OLD edge array; bad[0] counts entries that contradict it
__global__ void delta_locate_kernel(const uint32_t* row_ptr, const uint32_t* col, DeltaDev d, uint32_t* bad) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t total = d.n_ins + d.n_del + d.n_tch;
  if (i >= total) return;
  unsigned long long key;
  uint32_t val;
  int kind;  // 0 insert, 1 delete, 2 touch
  if (i < d.n_ins) { key = d.ins_key[i]; val = d.ins_val[i]; kind = 0; }
  else if (i < d.n_ins + d.n_del) { key = d.del_key[i - d.n_ins]; val = d.del_val[i - d.n_ins]; kind = 1; }
  else { key = d.tch_key[i - d.n_ins - d.n_del]; val = d.tch_val[i - d.n_ins - d.n_del]; kind = 2; }
  const uint32_t lo = row_ptr[key], hi = row_ptr[key + 1];
  const uint32_t pos = lower_bound_u32(col, lo, hi, val);
  const bool present = pos < hi && col[pos] == val;
  if (present == (kind == 0)) atomicAdd(bad, 1u);
  if (kind == 0) d.ins_pos[i] = pos;
  else if (kind == 1) d.del_pos[i - d.n_ins] = pos;
  else d.tch_pos[i - d.n_ins - d.n_del] = pos;
}

constexpr int kMergeTile = 4096;  // old elements per block

// new[p + shift(p)] = old[p] for every surviving old element; shift(p) = #{inserts at or before p} -
// #{deletes before p}. A tile without an update inside moves by one constant.
__global__ void __launch_bounds__(256) delta_merge_kernel(const uint32_t* __restrict__ old_a, uint32_t* __restrict__ new_a,
                                                          const uint32_t* __restrict__ old_b, uint32_t* __restrict__ new_b,
                                                          uint32_t n_old, const uint32_t* ins_pos, uint32_t n_ins,
                                                          const uint32_t* del_pos, uint32_t n_del) {
  const uint32_t t0 = blockIdx.x * kMergeTile;
  if (t0 >= n_old) return;
  const uint32_t t1 = min(n_old, t0 + kMergeTile);
  ZG_BLOCK_SHARED_U32(sh, 4);
  if (threadIdx.x == 0) {
    sh[0] = count_le(ins_pos, n_ins, t0);
    sh[1] = count_le(ins_pos, n_ins, t1 - 1);
    sh[2] = count_lt(del_pos, n_del, t0);
    sh[3] = count_le(del_pos, n_del, t1 - 1);
  }
  __syncthreads();
  const uint32_t ci0 = sh[0], ci1 = sh[1], cd0 = sh[2], cd1 = sh[3];
  if (ci0 == ci1 && cd0 == cd1) {
    const uint32_t shift = ci0 - cd0;  // modular arithmetic: the sum below is exact
    for (uint32_t p = t0 + threadIdx.x; p < t1; p += blockDim.x) {
      new_a[p + shift] = old_a[p];
      if (old_b) new_b[p + shift] = old_b[p];
    }
    return;
  }
  for (uint32_t p = t0 + threadIdx.x; p < t1; p += blockDim.x) {
    const uint32_t cd = cd0 + count_lt(del_pos + cd0, cd1 - cd0, p);
    if (cd < n_del && del_pos[cd] == p) continue;  // deleted
    const uint32_t ci = ci0 + count_le(ins_pos + ci0, ci1 - ci0, p);
    new_a[p + ci - cd] = old_a[p];
    if (old_b) new_b[p + ci - cd] = old_b[p];
  }
}

__global__ void delta_insert_kernel(uint32_t* new_a, uint32_t* new_b, const uint32_t* ins_pos, const uint32_t* ins_val,
                                    const uint32_t* ins_exp, uint32_t n_ins, const uint32_t* del_pos, uint32_t n_del) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_ins) return;
  const uint32_t at = ins_pos[i] + i - count_lt(del_pos, n_del, ins_pos[i]);
  new_a[at] = ins_val[i];
  if (new_b) new_b[at] = ins_exp ? ins_exp[i] : 0u;
}

__global__ void delta_touch_kernel(uint32_t* new_exp, const uint32_t* tch_pos, const uint32_t* tch_exp, uint32_t n_tch,
                                   const uint32_t* ins_pos, uint32_t n_ins, const uint32_t* del_pos, uint32_t n_del) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_tch) return;
  const uint32_t p = tch_pos[i];
  new_exp[p + count_le(ins_pos, n_ins, p) - count_lt(del_pos, n_del, p)] = tch_exp[i];
}

// row_ptr[r] += #{insert keys < r} - #{delete keys < r}, for r in [first, pool]
__global__ void __launch_bounds__(256) delta_rows_kernel(uint32_t* row_ptr, unsigned long long first, unsigned long long pool,
                                                         const unsigned long long* ins_key, uint32_t n_ins,
                                                         const unsigned long long* del_key, uint32_t n_del) {
  const unsigned long long t0 = first + static_cast<unsigned long long>(blockIdx.x) * kMergeTile;
  if (t0 > pool) return;
  const unsigned long long t1 = min(pool + 1, t0 + kMergeTile);
  ZG_BLOCK_SHARED_U32(sh, 4);
  if (threadIdx.x == 0) {
    sh[0] = count_lt64(ins_key, n_ins, t0);
    sh[1] = count_lt64(ins_key, n_ins, t1 - 1);
    sh[2] = count_lt64(del_key, n_del, t0);
    sh[3] = count_lt64(del_key, n_del, t1 - 1);
  }
  __syncthreads();
  const uint32_t ci0 = sh[0], ci1 = sh[1], cd0 = sh[2], cd1 = sh[3];
  if (ci0 == ci1 && cd0 == cd1) {
    const uint32_t shift = ci0 - cd0;
    if (shift)
      for (unsigned long long r = t0 + threadIdx.x; r < t1; r += blockDim.x) row_ptr[r] += shift;
    return;
  }
  for (unsigned long long r = t0 + threadIdx.x; r < t1; r += blockDim.x)
    row_ptr[r] += (ci0 + count_lt64(ins_key + ci0, ci1 - ci0, r)) - (cd0 + count_lt64(del_key + cd0, cd1 - cd0, r));
}

struct HostDelta {
  std::vector<unsigned long long> ins_key, del_key, tch_key;
  std::vector<uint32_t> ins_val, ins_exp, del_val, tch_val, tch_exp;
};


// Net effect of the store's journal as sorted forward / reverse deltas (several applies may precede one publish).
// cls_delta: per-class change of the relationship count. Returns "", "relayout" (an object beyond the capacities
// of the resident layout) or an error. Owner filter (rank, count): only the entries whose resource id % count == rank
// (one shard of a sharded handle, Store::build).
inline std::string prepare_delta(const Store& store, const Schema& sc, const HostSnapshot& lay, HostDelta* f, HostDelta* r,
                                 std::vector<uint32_t>* cls_delta, uint32_t owner_rank = 0, uint32_t owner_count = 1) {
  struct Net {
    zg_tuple t;
    bool was, is;
    uint32_t exp;
  };
  std::unordered_map<Key, Net, KeyHash> net;
  net.reserve(store.journal.size() * 2);
  for (const auto& j : store.journal) {
    if (owner_count > 1 && j.t.res % owner_count != owner_rank) continue;
    const Key k = key_of(j.t);
    auto it = net.find(k);
    const bool now_is = j.kind != Store::kDeleted;
    if (it == net.end()) net.emplace(k, Net{j.t, j.kind != Store::kInserted, now_is, j.expires});
    else {
      it->second.is = now_is;
      it->second.exp = j.expires;
    }
  }
  struct Ent {
    unsigned long long key;
    uint32_t val, exp;
    int kind;
  };
  std::vector<Ent> fe, re;
  cls_delta->assign(lay.cls.size(), 0);
  for (const auto& kv : net) {
    const Net& n = kv.second;
    if (!n.was && !n.is) continue;
    const int kind = (!n.was && n.is) ? 0 : ((n.was && !n.is) ? 1 : 2);
    const zg_tuple& t = n.t;
    const int k = sc.class_of(t.rel, t.stype, t.srel);
    if (k < 0) return "journal holds a relationship the schema forbids";
    const DRel& rel = lay.rels[sc.slots[t.rel].rel_index];
    const DCls& c = lay.cls[rel.cls_begin + k];
    if (t.res >= rel.nres || (t.srel != kWildcard && t.subj >= c.nsubj)) return "relayout";
    const uint32_t subj = t.srel == kWildcard ? 0u : t.subj;
    fe.push_back(Ent{rel.row_base + static_cast<unsigned long long>(t.res) * rel.stride + k, subj, n.exp, kind});
    re.push_back(Ent{c.rrow_base + static_cast<unsigned long long>(subj) * c.rstride, t.res, n.exp, kind});
    if (kind == 0) ++(*cls_delta)[rel.cls_begin + k];
    if (kind == 1) --(*cls_delta)[rel.cls_begin + k];
  }
  auto split = [&](std::vector<Ent>& v, HostDelta& h, bool reverse) {
    std::sort(v.begin(), v.end(), [](const Ent& a, const Ent& b) { return a.key != b.key ? a.key < b.key : a.val < b.val; });
    for (const Ent& e : v) {
      if (e.kind == 0) { h.ins_key.push_back(e.key); h.ins_val.push_back(e.val); h.ins_exp.push_back(e.exp); }
      else if (e.kind == 1) { h.del_key.push_back(e.key); h.del_val.push_back(e.val); }
      else if (!reverse) { h.tch_key.push_back(e.key); h.tch_val.push_back(e.val); h.tch_exp.push_back(e.exp); }
    }
  };
  split(fe, *f, false);
  split(re, *r, true);
  return "";
}

}  // namespace zg
