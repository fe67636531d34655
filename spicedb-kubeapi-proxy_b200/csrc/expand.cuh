// expand.cuh -- ExpandPermissionTree: the subject tree of T:r#P built from the resident forward CSR, one arrow level
// per launch sequence (Device::expand).
//
// Every slot is lowered at schema load into a pre-order template (Schema::compute_expand_templates, XNode): the
// intermediate nodes, the relation leaves and the arrows one object contributes. A job is (request, parent node, rank,
// object, template root, depth); level 0 holds one job per request. Per level:
//   expand_count_kernel  one warp per (job, counted node): a relation leaf counts the live entries of the object's rows
//                        over the relation's classes, an arrow the live non-wildcard entries of the tupleset's rows,
//                        split into children with a target template (next-level jobs) and without (empty leaves)
//   a CUB exclusive sum  over [nodes | subjects | jobs] of every (job, counted node): every job's node block, every
//                        leaf's subject range, every arrow's child-job range and empty-leaf range
//   expand_emit_kernel   the same warps write the template's nodes, the leaf subjects, the empty leaves and the next
//                        level's jobs, each in row order (class order, then ascending id within a class)
// A child job deeper than ZG_MAX_DEPTH fails its request (ZG_EDEPTH) when it is emitted. The jobs of a failed request
// count nothing from the next level on, and its nodes are dropped when the call finishes.
#pragma once
#ifndef ZG_EMULATE
#include <cuda_runtime.h>
#endif
#include <cstdint>
#include <vector>

#include "../../include/zgpu.h"
#include "filter.cuh"
#include "schema.h"

namespace zg {

constexpr unsigned kExpandThreads = 256;
constexpr unsigned kExpandFull = 0xFFFFFFFFu;

struct XJob {
  uint32_t request, parent, rank, object;
  uint32_t tmpl;   // template root in XParams::nodes
  uint32_t depth;  // arrow hops from the request's root
};

struct XParams {
  const uint32_t *row_ptr, *col, *exp;  // exp: nullptr when the schema has no expiration
  const DRel* rels;
  const DCls* cls;
  const XNode* nodes;
  const uint32_t *tgts, *counted;
  uint32_t now;  // 0: expired relationships are live too
  uint32_t m;    // warps per job: the largest ncount of this level's templates, at least 1 (expand_warps)
  const XJob* jobs;
  unsigned long long n_jobs;
  uint32_t* failed;              // per request: 1 = ZG_EDEPTH
  unsigned long long* cnt;       // 3 n_jobs m + 1: nodes | subjects | next jobs per (job, counted node); then 0
  const unsigned long long* off; // their exclusive sum
  unsigned long long node_base, subj_base;  // nodes / subjects of the earlier levels
  zg_expand_node* out_nodes;
  zg_expand_subject* out_subj;
  XJob* next;
  unsigned long long* next_mask;  // bit c: a next-level job's template has c counted nodes (the next level's m)
};

// Warps per job of a level whose templates' counted-node counts are the set bits of mask.
inline uint32_t expand_warps(unsigned long long mask) {
  uint32_t m = 1;
  for (uint32_t c = 0; c < 64; ++c)
    if ((mask >> c) & 1ull) m = c > m ? c : m;
  return m;
}

__device__ __forceinline__ bool expand_live(const XParams& p, const DCls& c, uint32_t i) {
  return !(p.exp && (c.flags & CF_EXPIRY)) || filter_live(__ldg(p.exp + i), p.now);
}

// Live entries of the object's row of one class: from the offsets alone when the class cannot expire.
__device__ __forceinline__ uint32_t expand_row_count(const XParams& p, const DCls& c, uint32_t b, uint32_t e, unsigned lane) {
  if (!(p.exp && (c.flags & CF_EXPIRY))) return e - b;
  uint32_t n = 0;
  for (uint32_t i0 = b; i0 < e; i0 += 32) {
    const uint32_t i = i0 + lane;
    n += __popc(__ballot_sync(kExpandFull, i < e && filter_live(__ldg(p.exp + i), p.now)));
  }
  return n;
}

__device__ __forceinline__ void expand_row(const XParams& p, const DRel& r, uint32_t obj, uint32_t k, uint32_t* b, uint32_t* e) {
  *b = *e = 0;
  if (obj >= r.nres) return;  // never written (ZG_NO_OBJECT included): no rows
  const unsigned long long ri = r.row_base + static_cast<unsigned long long>(obj) * r.stride + k;
  *b = __ldg(p.row_ptr + ri);
  *e = __ldg(p.row_ptr + ri + 1);
}

__global__ void __launch_bounds__(kExpandThreads) expand_count_kernel(const XParams p) {
  const unsigned lane = threadIdx.x & 31;
  const unsigned long long n = p.n_jobs * p.m;
  const unsigned long long w = (blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x) >> 5;
  if (w >= n) return;
  const XJob job = p.jobs[w / p.m];
  const uint32_t k = static_cast<uint32_t>(w % p.m);
  const XNode root = p.nodes[job.tmpl];
  const bool alive = !p.failed[job.request];  // written by the emit launches only: one answer for every warp of a job
  unsigned long long nodes = alive && k == 0 ? root.size : 0, subj = 0, jobs = 0;
  if (alive && k < root.ncount) {
    const XNode x = p.nodes[job.tmpl + p.counted[root.counted + k]];
    const DRel r = p.rels[x.rel];
    for (uint32_t c = 0; c < r.ncls; ++c) {
      const DCls cl = p.cls[r.cls_begin + c];
      if (x.op == X_ARROW && cl.sslot == kWildcard) continue;
      uint32_t b, e;
      expand_row(p, r, job.object, c, &b, &e);
      const uint32_t live = expand_row_count(p, cl, b, e, lane);
      if (x.op == X_REL) subj += live;
      else if (p.tgts[x.tgt + c] != kNoTemplate) jobs += live;
      else nodes += live;
    }
  }
  if (lane == 0) {
    p.cnt[w] = nodes;
    p.cnt[n + w] = subj;
    p.cnt[2 * n + w] = jobs;
  }
}

__global__ void __launch_bounds__(kExpandThreads) expand_emit_kernel(const XParams p) {
  const unsigned lane = threadIdx.x & 31;
  const unsigned long long n = p.n_jobs * p.m;
  const unsigned long long w = (blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x) >> 5;
  if (w >= n) return;
  const unsigned long long j = w / p.m, w0 = j * p.m;
  const XJob job = p.jobs[j];
  const uint32_t k = static_cast<uint32_t>(w % p.m);
  if (p.cnt[w0] == 0) return;  // failed when it was counted
  const XNode root = p.nodes[job.tmpl];
  const unsigned long long base = p.node_base + p.off[w0];  // the job's template nodes, then its arrows' empty leaves
  if (k == 0 && lane < root.size) {
    const XNode x = p.nodes[job.tmpl + lane];
    zg_expand_node o;
    o.request = job.request;
    o.parent = lane == 0 ? job.parent : static_cast<uint32_t>(base + x.parent);
    o.rank = lane == 0 ? job.rank : x.rank;
    o.object = job.object;
    o.slot = x.slot;
    o.op = x.op == X_REL || x.op == X_NIL ? ZG_EXPAND_LEAF : x.op == X_ARROW ? ZG_EXPAND_UNION : x.op;
    o.n_subjects = 0;
    o.subjects = p.subj_base;
    if (x.op == X_REL) {
      const unsigned long long c = w0 + x.count;
      o.n_subjects = static_cast<uint32_t>(p.cnt[n + c]);
      o.subjects = p.subj_base + p.off[n + c] - p.off[n];
    }
    p.out_nodes[base + lane] = o;
  }
  if (k >= root.ncount) return;
  const uint32_t xi = p.counted[root.counted + k];
  const XNode x = p.nodes[job.tmpl + xi];
  const DRel r = p.rels[x.rel];
  const unsigned below = (1u << lane) - 1u;
  unsigned long long at_subj = p.subj_base + p.off[n + w] - p.off[n];
  unsigned long long at_job = p.off[2 * n + w] - p.off[2 * n];
  unsigned long long at_leaf = p.node_base + p.off[w] + (k == 0 ? root.size : 0);
  uint32_t rank = 0;
  for (uint32_t c = 0; c < r.ncls; ++c) {
    const DCls cl = p.cls[r.cls_begin + c];
    if (x.op == X_ARROW && cl.sslot == kWildcard) continue;
    const uint32_t target = x.op == X_ARROW ? p.tgts[x.tgt + c] : kNoTemplate;
    uint32_t b, e;
    expand_row(p, r, job.object, c, &b, &e);
    const uint32_t rank0 = rank;
    for (uint32_t i0 = b; i0 < e; i0 += 32) {
      const uint32_t i = i0 + lane;
      const bool live = i < e && expand_live(p, cl, i);
      const uint32_t id = live ? __ldg(p.col + i) : 0;
      const unsigned m = __ballot_sync(kExpandFull, live);
      const uint32_t before = __popc(m & below);
      if (live) {
        if (x.op == X_REL) {
          zg_expand_subject s;
          s.id = cl.sslot == kWildcard ? 0u : id;
          s.type = cl.stype;
          s.srel = cl.sslot;
          p.out_subj[at_subj + before] = s;
        } else if (target != kNoTemplate) {
          XJob c2;
          c2.request = job.request;
          c2.parent = static_cast<uint32_t>(base + xi);
          c2.rank = rank + before;
          c2.object = id;
          c2.tmpl = target;
          c2.depth = job.depth + 1;
          p.next[at_job + before] = c2;
          if (c2.depth > ZG_MAX_DEPTH) p.failed[job.request] = 1;
        } else {
          zg_expand_node o;
          o.request = job.request;
          o.parent = static_cast<uint32_t>(base + xi);
          o.rank = rank + before;
          o.object = job.object;
          o.slot = x.slot;
          o.op = ZG_EXPAND_LEAF;
          o.n_subjects = 0;
          o.subjects = p.subj_base;
          p.out_nodes[at_leaf + before] = o;
        }
      }
      const uint32_t got = __popc(m);
      rank += got;
      if (x.op == X_REL) at_subj += got;
      else if (target != kNoTemplate) at_job += got;
      else at_leaf += got;
    }
    if (lane == 0 && target != kNoTemplate && rank > rank0) atomicOr(p.next_mask, 1ull << p.nodes[target].ncount);
  }
}

// Drops the nodes and subjects of the failed requests (failed[request] != 0), remapping parents and subject ranges; a
// parent precedes its children, so one pass does it. Host code: the finish of Device::expand.
inline void expand_drop_failed(const std::vector<uint32_t>& failed, std::vector<zg_expand_node>* nodes,
                               std::vector<zg_expand_subject>* subjects) {
  std::vector<uint32_t> at(nodes->size(), UINT32_MAX);
  std::vector<zg_expand_node> kept;
  std::vector<zg_expand_subject> ksubj;
  for (size_t i = 0; i < nodes->size(); ++i) {
    zg_expand_node o = (*nodes)[i];
    if (failed[o.request]) continue;
    at[i] = static_cast<uint32_t>(kept.size());
    if (o.parent != UINT32_MAX) o.parent = at[o.parent];
    const uint64_t b = o.subjects;
    o.subjects = ksubj.size();
    ksubj.insert(ksubj.end(), subjects->begin() + b, subjects->begin() + b + o.n_subjects);
    kept.push_back(o);
  }
  nodes->swap(kept);
  subjects->swap(ksubj);
}

}  // namespace zg
