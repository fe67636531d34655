// kernels.cuh -- sm_90a CUDA kernels of the permission-check hot path.
//
// What this replaces in the reference: the per-item graph evaluation that
// CheckBulkPermissions / CheckPermission / LookupResources trigger inside the
// embedded SpiceDB (call sites pkg/authz/check.go:48, postfilter.go:134,
// watch.go:50, lookups.go:65; engine config pkg/spicedb/spicedb.go:25-56).
//
// Execution model (DESIGN.md "Kernels"):
//   * persistent grid, every SM (132 on an H100 SXM) x 4 CTAs x 8 warps; every WARP owns a private LIFO of edge
//     RANGES in shared memory (spilling to a per-warp HBM area) and pulls batches of 32
//     checks from a global counter;
//   * admission loads each subject's reverse rows (its direct memberships) into a small
//     per-check set in shared memory: direct probes become shared-memory compares, and a
//     range whose children could only match directly is resolved by searching the
//     memberships' short reverse rows instead of visiting the children (meet in the middle);
//   * one iteration pops ranges worth <= 32 edges, assigns one edge per lane (coalesced reads
//     of each CSR segment), and every lane visits its child node: two row offsets per
//     non-empty edge class, ballot/popc-compacted push of the userset and arrow ranges;
//   * found / error state is two warp-uniform 32-bit masks; a found check's remaining ranges
//     are dropped when popped (short circuit); long-running batches switch on a lossy memo of
//     (check, slot, object, depth) visits so DAG-shaped data stays polynomial;
//   * no tensor cores, no floating point: memory-latency / issue-bound integer traversal.
#pragma once
#ifndef ZG_EMULATE  // tests/emu/: the same source under a CPU SIMT emulator (test infrastructure, never in libzgpu.so)
#include <cuda_runtime.h>
#define ZG_DYNAMIC_SMEM(name) extern __shared__ __align__(16) uint8_t name[]
#ifndef ZG_BLOCK_SHARED_U32
#define ZG_BLOCK_SHARED_U32(name, n) __shared__ uint32_t name[n]
#endif
#endif

#include <cstdint>

#include "../../include/zgpu.h"
#include "closure_sig.cuh"
#include "schema.h"

namespace zg {

constexpr int kWarpsPerBlock = 8;
constexpr int kThreads = kWarpsPerBlock * 32;
#ifndef ZG_MIN_BLOCKS
#define ZG_MIN_BLOCKS 4
#endif
#ifndef ZG_STACK_CAP
#define ZG_STACK_CAP 64
#endif
#ifndef ZG_RSET_CAP
#define ZG_RSET_CAP 16
#endif
// Build-time tuning knobs (scripts/build_variant.sh). ZG_MIN_BLOCKS was A/B-measured on the H100: 4 beat 3 and 5 on
// cfg3 and cfg4 (DESIGN.md §6). ZG_PHASE_CLOCKS is an instrument, off in the library.
#ifndef ZG_PHASE_CLOCKS
#define ZG_PHASE_CLOCKS 0  // 1: every warp adds clock64() cycles per phase of a batch into KParams::events[3 .. 7]
                           // (admission, root visit, two-level meet, one-level meet, pop loop; zg_phase_clocks)
#endif
constexpr int kPhases = 5;
constexpr int kMinBlocks = ZG_MIN_BLOCKS;  // resident CTAs per SM the register budget is tuned for
constexpr int kStackCap = ZG_STACK_CAP;    // range items per warp in shared memory
constexpr int kRsetCap = ZG_RSET_CAP;      // reverse-row entries kept per check (subject's direct memberships), <= 31
constexpr int kStateWords = 5;             // per-lane query state parked in shared memory between leaf passes
constexpr int kMeetWords = 128;            // batch_l2's 128-bit filter of each lane's range (two 64-bit words per lane)
constexpr int kFCap = 64;                  // the largest range (children) the two-level meet answers
constexpr size_t kWarpSmem = kStackCap * sizeof(uint4) + ((kRsetCap + kStateWords) * 32 + kMeetWords) * sizeof(uint32_t);
constexpr unsigned kFull = 0xFFFFFFFFu;
constexpr uint16_t kJobDepthMask = 0x00FF;  // zg_check.flags of a raised sub-query: hop depth

// value bits of a (query, leaf) pair and of a sub-query
constexpr uint8_t kValT = 1, kValE = 2;

// Closure index of one two-level pair (DESIGN.md §4), built at publish (build.cu gpu_build_closure): for the
// kStepTargetL2 steps of class tgc, row u = col[row_ptr[u], row_ptr[u + 1]) lists, ascending and distinct, every object
// the subject u reaches through one of its memberships g: the union of g's reverse rows in class tgc. col is padded so
// that the aligned 16-byte block holding a row's last word lies inside the allocation. The entries are 16-bit when
// every object id of class tgc's resource type is below 65 536 in every pair of the snapshot, else 32-bit (width, in
// bytes); 16-bit rows are padded so that the aligned 32-byte sector holding a row's last entry lies inside it.
constexpr int kMaxClosure = 4;
#ifndef ZG_CLOSURE_BLOCKS
#define ZG_CLOSURE_BLOCKS 2
#endif
#ifndef ZG_CLOSURE_VERIFY
#define ZG_CLOSURE_VERIFY 8
#endif
constexpr int kClosureBlocks = ZG_CLOSURE_BLOCKS;  // 16-byte blocks in flight per lane per round of closure_meet
constexpr int kClosureVerify = ZG_CLOSURE_VERIFY;  // pending "maybe"s of a warp that trigger their searches
struct ClosureRef {
  const uint32_t* row_ptr;
  const void* col;  // entries of `width` bytes
  uint32_t nsubj;   // rows (subjects of the innermost direct class)
  uint16_t tgc;
  uint16_t width;   // 2 or 4; a kernel instantiated for one width reads only the indexes of that width
  // Signature of every row (closure_sig.cuh): sig_words 64-bit words per row, row u at sig[u * sig_words]. nullptr: none.
  const unsigned long long* sig;
  uint32_t sig_words;  // a power of two, 1 .. 32
  // Set table of every row (closure_sig.cuh table_bucket): row u's header at set_hdr[u], its buckets from
  // set_tab[header's first bucket]. nullptr: none.
  const unsigned long long* set_hdr;
  const unsigned long long* set_tab;
};
// check_kernel's MEET argument: no two-level step in the schema, or the width of the closure entries it reads, plus
// kMeetSig when the meet tests the range against the rows' signatures (sig_meet) instead of streaming the rows, or
// also kMeetSet when the signatures' "maybe"s are confirmed in the rows' set tables (16-bit indexes only)
constexpr int kMeetNone = 0, kMeet16 = 2, kMeet32 = 4, kMeetSig = 8, kMeetSet = 16;
constexpr int kMeetSig16 = kMeet16 | kMeetSig, kMeetSig32 = kMeet32 | kMeetSig, kMeetSet16 = kMeetSig16 | kMeetSet;
// Range records of a push step's class (closure_sig.cuh kRecSlots), read by flat_check_kernel. The record's address
// depends on obj alone, so it is loaded beside the subject's table header and signature line instead of after the
// range's offsets.
constexpr int kMaxFlatRecords = 4;
constexpr uint32_t kRecVecs = kRecSlots / 8;  // 16-byte loads per record
struct FlatRecordRef {
  const uint4* rec;  // nres records of kRecSlots 16-bit slots
  uint32_t nres;
  uint16_t gc;
};
template <int MEET> struct ClosureEntry { using type = uint32_t; };
template <> struct ClosureEntry<kMeet16> { using type = uint16_t; };
template <> struct ClosureEntry<kMeetSig16> { using type = uint16_t; };
template <> struct ClosureEntry<kMeetSet16> { using type = uint16_t; };

struct KParams {
  const uint32_t* row_ptr;
  const uint32_t* col;
  const uint32_t* exp;  // nullptr unless the schema uses expiration
  const uint32_t* rrow_ptr;  // reverse CSR (subject -> resources), rows interleaved per subject
  const uint32_t* rcol;
  int invert;  // answer direct probes from the subject's reverse rows when they are small
  const uint8_t* prog;
  uint32_t prog_bytes;
  const zg_check* queries;
  unsigned long long nq;
  uint32_t L;    // leaf stride of val (Snapshot::max_leaves)
  uint8_t* val;  // [nq * L] value bits per (query, leaf): what the fold of a multi-pass run reads (may be null)
  uint8_t* out;  // [nq] v1 codes (final_codes) or value bits (may be null)
  int final_codes;
  unsigned long long* next;  // batch counter (zeroed before launch)
  uint4* spill;              // per-warp spill areas
  uint32_t spill_cap;        // items per warp
  // sub-queries raised when an edge leads into a non-pure permission (or to another shard)
  zg_check* subq;
  uint32_t* subq_parent;  // q * L + leaf of the raising (query, leaf)
  unsigned long long* subq_count;
  unsigned long long subq_cap;
  uint32_t* flags;  // bit0: spill overflow, bit1: sub-query overflow, bit2: budget hit
  uint32_t now;
  uint32_t budget;
  int raw_items;  // queries are caller-supplied zg_check items: flags are ignored
  // Per-warp lossy memo of (job, slot, object, depth) child visits, switched on only for
  // batches that run long (DAG-shaped data multiplies paths; see DESIGN.md "Path memo").
  unsigned long long* memo;
  uint32_t memo_entries;  // per warp, power of two (0 = disabled)
  uint32_t memo_after;    // iterations before the memo is switched on for a batch
  // Object-hash sharded store (DESIGN.md 7): this device only holds the relationships whose
  // RESOURCE it owns (owner = object id % shard_count); an edge to an object of another shard
  // becomes a sub-query that is routed to its owner between passes.
  uint32_t shard_count;   // 0 / 1 = not sharded
  uint32_t shard_rank;
  unsigned long long* alg_bytes;  // COUNT variant only
  unsigned long long* events;     // [0] stack spills, [1] batches that switched the path memo on (cumulative),
                                  // [3 .. 7] phase cycles (ZG_PHASE_CLOCKS builds only)
  // Streamed admission: the queries are still being copied from the host while the kernel runs. *ready =
  // number of leading queries that have landed (a 8-byte copy enqueued after each chunk on the copy stream);
  // a warp waits until its batch is there. nullptr: everything is resident.
  const unsigned long long* ready;
  // LookupSubjects' second verification: every wildcard relationship is invisible (an ST_WILD step never matches),
  // so a subject that checks HAS is granted through its own relationships. Never set by the public check calls.
  int no_wildcards;
  // two-level steps whose pair has a closure index meet over it; the others keep batch_l2
  ClosureRef closure[kMaxClosure];
  uint32_t n_closure;
  // The residual pass after flat_check_kernel (check_kernel<..., RESIDUAL = true> only): the pass's i-th query is
  // queries[idx[i]], and the pass has *nq_dev queries (nq is only the grid's bound). flat_check_kernel writes both:
  // nq_dev[0] = this pass's residual, nq_dev[1] += it (a running total). nullptr: queries[i], nq.
  uint32_t* idx;
  unsigned long long* nq_dev;
  // flat_check_kernel only: the range records of the push steps' classes (a class without one reads the CSR)
  FlatRecordRef rec[kMaxFlatRecords];
  uint32_t n_rec;
};

// View of the program blob. Only the base pointer is kept in registers; table addresses are
// formed from the header offsets on use (sixteen live 64-bit pointers cost 32 registers).
struct Prog {
  const uint8_t* b;
  __device__ __forceinline__ const DHeader* hdr() const { return reinterpret_cast<const DHeader*>(b); }
#define ZG_TABLE(name, type, field) \
  __device__ __forceinline__ const type* name() const { return reinterpret_cast<const type*>(b + hdr()->field); }
  ZG_TABLE(slots, DSlot, off_slots)
  ZG_TABLE(units, DUnit, off_units)
  ZG_TABLE(cls, DCls, off_cls)
  ZG_TABLE(members, uint16_t, off_members)
  ZG_TABLE(trees, DTree, off_trees)
  ZG_TABLE(tree_ops, DTreeOp, off_tree_ops)
  ZG_TABLE(leaf_units, uint16_t, off_leaf_units)
  ZG_TABLE(type_inv, DTypeInv, off_type_inv)
  ZG_TABLE(inv_cls, uint16_t, off_inv_cls)
  ZG_TABLE(steps, DStep, off_steps)
  ZG_TABLE(type_rcls, DTypeInv, off_type_rcls)
  ZG_TABLE(rcls, uint16_t, off_rcls)
#undef ZG_TABLE
};

__device__ __forceinline__ Prog make_prog(const uint8_t* b) { return Prog{b}; }

// range item: x = begin, y = end (edge indices into col), z = meta, w unused
//   meta: bits 0-4 job slot, 5-10 depth of the children, 11 class has expiry,
//         16-31 slot the children are visited at
__device__ __forceinline__ uint32_t make_meta(uint32_t jslot, uint32_t depth, bool expiry, uint32_t tslot) {
  return jslot | (depth << 5) | (expiry ? (1u << 11) : 0u) | (tslot << 16);
}

template <bool COUNT>
struct WarpCtx {
  uint4* stack;
  uint4* spill;
  int top, spill_top;
  uint32_t spill_cap;
  unsigned found, err;  // warp-uniform, indexed by job slot
  unsigned raised;      // job slots that raised a sub-query in this leaf pass (their value is not final)
  uint32_t my_subj, my_ss;  // this lane's own query: subject id, stype<<16 | srel
  // Direction-optimised probes: rset[i * 32 + job] = resource id of every direct relationship
  // of the job's subject (its reverse rows), grouped by class (boundaries in my_cst), when
  // there are <= kRsetCap and some step of the job's permission may read them (SF_NO_RSET).
  uint32_t* rset;
  unsigned long long my_cst;  // class boundaries of this lane's own job (see cst_at)
  unsigned inv_mask;  // jobs that may meet in the middle: their reverse rows fit, or (cst bit kOverCap) only the
                      // two-level meets (closure_meet, batch_l2), which do not read the set
  unsigned long long bytes;
  unsigned long long* events;
  bool fatal;
  unsigned lane;
#if ZG_PHASE_CLOCKS
  long long ph[kPhases];  // warp-uniform cycles: admission, root visit, two-level meet, one-level meet, pop loop
#endif
};

template <bool COUNT>
__device__ __forceinline__ void spill_half(WarpCtx<COUNT>& c) {
  constexpr int H = kStackCap / 2;
  if (c.spill_top + H > static_cast<int>(c.spill_cap)) {
    c.fatal = true;
    c.top = 0;
    return;
  }
  for (int i = c.lane; i < H; i += 32) c.spill[c.spill_top + i] = c.stack[i];
  if (c.lane == 0) atomicAdd(c.events, 1ull);
  __syncwarp();
  int rest = c.top - H;  // <= H: read [H, top) and write [0, rest) never overlap
  uint4 t0, t1;
  int i0 = c.lane, i1 = c.lane + 32;
  if (i0 < rest) t0 = c.stack[H + i0];
  if (i1 < rest) t1 = c.stack[H + i1];
  __syncwarp();
  if (i0 < rest) c.stack[i0] = t0;
  if (i1 < rest) c.stack[i1] = t1;
  __syncwarp();
  c.spill_top += H;
  c.top = rest;
}

template <bool COUNT>
__device__ __forceinline__ void refill(WarpCtx<COUNT>& c) {
  constexpr int H = kStackCap / 2;
  int n = c.spill_top < H ? c.spill_top : H;
  for (int i = c.lane; i < n; i += 32) c.stack[i] = c.spill[c.spill_top - n + i];
  __syncwarp();
  c.spill_top -= n;
  c.top = n;
}

// Warp-collective push: lanes with want=true append their item in lane order.
template <bool COUNT>
__device__ __forceinline__ void push(WarpCtx<COUNT>& c, bool want, const uint4& item) {
  unsigned m = __ballot_sync(kFull, want);
  if (!m || c.fatal) return;
  int cnt = __popc(m);
  if (c.top + cnt > kStackCap) spill_half(c);
  if (c.fatal) return;
  if (want) c.stack[c.top + __popc(m & ((1u << c.lane) - 1u))] = item;
  c.top += cnt;
  __syncwarp();
}

// Binary search of the sorted segment arr[lo, hi) for key.
template <bool COUNT, class T>
__device__ __forceinline__ bool find_in(const T* __restrict__ arr, WarpCtx<COUNT>& c, uint32_t lo, uint32_t hi,
                                        uint32_t key, uint32_t* at = nullptr) {
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    const uint32_t v = __ldg(arr + mid);
    if (COUNT) c.bytes += sizeof(T);
    if (v == key) {
      if (at) *at = mid;
      return true;
    }
    if (v < key) lo = mid + 1; else hi = mid;
  }
  return false;
}

// Binary search of the sorted direct-subject segment col[lo, hi) for sid.
template <bool COUNT>
__device__ __forceinline__ bool probe(const KParams& p, WarpCtx<COUNT>& c, uint32_t lo, uint32_t hi, uint32_t sid,
                                      bool expiry) {
  uint32_t at = 0;
  if (!find_in(p.col, c, lo, hi, sid, &at)) return false;
  if (expiry) {
    const uint32_t e = __ldg(p.exp + at);
    if (COUNT) c.bytes += 4;
    return e == 0 || e > p.now;
  }
  return true;
}

// A probe step (ST_DIRECT / ST_WILD) answered from the forward rows: is sid a direct subject of obj in the step's class,
// or has obj a wildcard relationship of it, unexpired at p.now. visit's non-inverted probes and flat_check_kernel's.
// expiry: the step's class has CF_EXPIRY.
template <bool COUNT>
__device__ __forceinline__ bool probe_step(const KParams& p, WarpCtx<COUNT>& c, const DStep& st, uint32_t obj,
                                           uint32_t sid, bool expiry) {
  if (obj >= st.nres) return false;
  const unsigned long long ridx = st.row_base + static_cast<unsigned long long>(obj) * st.ncls;
  const uint32_t lo = __ldg(p.row_ptr + ridx), hi = __ldg(p.row_ptr + ridx + 1);
  if (COUNT) c.bytes += 8;
  if (hi <= lo) return false;
  if (st.kind == ST_DIRECT) return probe(p, c, lo, hi, sid, expiry);
  if (expiry) {  // ST_WILD
    const uint32_t e = __ldg(p.exp + lo);
    if (COUNT) c.bytes += 4;
    return e == 0 || e > p.now;
  }
  return true;
}

// Two independent binary searches advanced in lock step (two loads in flight per lane).
template <bool COUNT>
__device__ __forceinline__ void probe2(const uint32_t* __restrict__ arr, WarpCtx<COUNT>& c, uint32_t lo0, uint32_t hi0,
                                       uint32_t k0, uint32_t lo1, uint32_t hi1, uint32_t k1, bool& hit0, bool& hit1) {
  while (lo0 < hi0 || lo1 < hi1) {
    const bool a0 = lo0 < hi0, a1 = lo1 < hi1;
    const uint32_t m0 = lo0 + ((hi0 - lo0) >> 1), m1 = lo1 + ((hi1 - lo1) >> 1);
    uint32_t v0 = 0, v1 = 0;
    if (a0) v0 = __ldg(arr + m0);
    if (a1) v1 = __ldg(arr + m1);
    if (COUNT) c.bytes += 4u * (a0 + a1);
    if (a0) {
      if (v0 == k0) { hit0 = true; lo0 = hi0; }
      else if (v0 < k0) lo0 = m0 + 1; else hi0 = m0;
    }
    if (a1) {
      if (v1 == k1) { hit1 = true; lo1 = hi1; }
      else if (v1 < k1) lo1 = m1 + 1; else hi1 = m1;
    }
  }
}

// Do the sorted segments a[a0, a1) and b[b0, b1) share an element? Sizes within 4x of each other:
// two-pointer merge (one load per step); otherwise every element of the short one is searched in
// the long one.
template <bool COUNT, class B>
__device__ __forceinline__ bool intersects(const uint32_t* __restrict__ a, uint32_t a0, uint32_t a1,
                                           const B* __restrict__ b, uint32_t b0, uint32_t b1, WarpCtx<COUNT>& c) {
  const uint32_t na = a1 - a0, nb = b1 - b0;
  if (na == 0 || nb == 0) return false;
  if (na > 4u * nb) {
    for (uint32_t x = b0; x < b1; ++x) {
      const uint32_t k = __ldg(b + x);
      if (COUNT) c.bytes += sizeof(B);
      if (find_in(a, c, a0, a1, k)) return true;
    }
    return false;
  }
  if (nb > 4u * na) {
    for (uint32_t x = a0; x < a1; ++x) {
      const uint32_t k = __ldg(a + x);
      if (COUNT) c.bytes += 4;
      if (find_in(b, c, b0, b1, k)) return true;
    }
    return false;
  }
  uint32_t va = __ldg(a + a0), vb = __ldg(b + b0);
  if (COUNT) c.bytes += 4 + sizeof(B);
  for (;;) {
    if (va == vb) return true;
    if (va < vb) {
      if (++a0 == a1) return false;
      va = __ldg(a + a0);
      if (COUNT) c.bytes += 4;
    } else {
      if (++b0 == b1) return false;
      vb = __ldg(b + b0);
      if (COUNT) c.bytes += sizeof(B);
    }
  }
}

// Boundaries of a job's reverse-row set per invertible class of its subject type:
// 5 bits each (0..31), boundary i at bit 5*i; class i owns entries [b_i, b_{i+1}). Bit kOverCap: the subject has more
// memberships than the set holds (no boundary is valid; the two-level meet reads them from the subject's reverse rows).
constexpr uint32_t kOverCap = 63;
__device__ __forceinline__ uint32_t cst_at(unsigned long long cst, uint32_t i) {
  return static_cast<uint32_t>(cst >> (5u * i)) & 31u;
}
static_assert(kRsetCap <= 31, "class boundaries are 5-bit fields");

// Filter of batch_l2: two bits per object id in 128 (two 64-bit words). False-positive rate (1 - e^(-2n/128))^2 over
// a range of n children: 2 % at n = 10 (cfg3's mean), 12 % at n = 27 (its largest); only the search behind it answers.
__device__ __forceinline__ void l2_bits(uint32_t v, uint32_t& b1, uint32_t& b2) {
  const uint32_t hv = v * 0x9E3779B1u;
  b1 = hv >> 25;
  b2 = (hv >> 18) & 127u;
}
__device__ __forceinline__ bool l2_maybe(unsigned long long f0, unsigned long long f1, uint32_t v) {
  uint32_t b1, b2;
  l2_bits(v, b1, b2);
  return ((((b1 & 64u) ? f1 : f0) >> (b1 & 63u)) & (((b2 & 64u) ? f1 : f0) >> (b2 & 63u)) & 1ull) != 0;
}
// The filter of the range col[lo, hi), four independent loads in flight.
__device__ __forceinline__ void l2_filter(const uint32_t* __restrict__ col, uint32_t lo, uint32_t hi, unsigned long long& f0,
                                          unsigned long long& f1) {
  for (uint32_t x = lo; x < hi; x += 4) {
    uint32_t v[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = x + i < hi ? __ldg(col + x + i) : 0u;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (x + i >= hi) break;
      uint32_t b1, b2;
      l2_bits(v[i], b1, b2);
      if (b1 & 64u) f1 |= 1ull << (b1 & 63u); else f0 |= 1ull << (b1 & 63u);
      if (b2 & 64u) f1 |= 1ull << (b2 & 63u); else f0 |= 1ull << (b2 & 63u);
    }
  }
}
// Is v an element of the sorted range col[a, b)? (the filter said maybe)
template <bool COUNT, class T>
__device__ __forceinline__ bool l2_verify(const T* __restrict__ col, uint32_t a, uint32_t b, uint32_t v,
                                          unsigned long long& nb) {
  while (a < b) {
    const uint32_t mid = a + ((b - a) >> 1), t = __ldg(col + mid);
    if (COUNT) nb += sizeof(T);
    if (t == v) return true;
    if (t < v) a = mid + 1; else b = mid;
  }
  return false;
}

// Two-level meet, batched: every requesting lane of a visit round is served at once (per-lane meets ran with few of
// the 32 lanes active: row counts and early exits differ per check). Lane j wants "does some membership g of its
// subject (class tinv) list a child of its range col[lo, hi) in class tgc". Its memberships are rset entries [kb, ke) of its job, or -- for a subject with more memberships than the set
// holds -- the subject's own reverse row of class tinv. The (lane, membership) pairs of the whole warp are numbered
// with one scan and dealt out 32 at a time: every lane reads one pair's reverse row (all 32 rows in flight together)
// and tests its elements against the owner's 128-bit filter of the range; a "maybe" is verified by a binary search of
// the range, which lane j has just read. Pairs of a check that is already answered are skipped.
// k packs ke << 8 | kb (set entries) or 0x8000 | tinv (reverse row), and tgc << 16. Requesting lanes are those of
// checks not answered yet. Returns the job slots answered.
// Ranges are <= kFCap children (the caller keeps larger ones). Inlined: out of line, the call site spilled more of
// the traversal loop's registers (ptxas) and ran no faster on cfg3 (H100, DESIGN.md §6).
template <bool COUNT>
__device__ __forceinline__ unsigned batch_l2(const uint32_t* __restrict__ col, const uint32_t* __restrict__ rrow_ptr,
                                          const uint32_t* __restrict__ rcol, uint32_t* rset, uint32_t lane, bool want,
                                          uint32_t lo, uint32_t hi, uint32_t k, uint32_t jslot, uint32_t sid, uint32_t stype,
                                          unsigned long long* bytes) {
  ZG_DYNAMIC_SMEM(smem);
  const Prog pr = make_prog(smem);  // the program is staged at the start of shared memory
  unsigned long long nb = 0;
  unsigned long long f0 = 0, f1 = 0;
  uint32_t mb = 0, me = 0;
  if (want) {
    l2_filter(col, lo, hi, f0, f1);
    if (COUNT) nb += 4ull * (hi - lo);
    if (!(k & 0x8000u)) {
      mb = k & 31u;
      me = (k >> 8) & 31u;
    } else {
      const DCls scl = pr.cls()[pr.inv_cls()[pr.type_inv()[stype].begin + (k & 31u)]];
      if (!(scl.flags & CF_EMPTY) && sid < scl.nsubj) {
        const unsigned long long ri = scl.rrow_base + static_cast<unsigned long long>(sid) * scl.rstride;
        mb = __ldg(rrow_ptr + ri);
        me = __ldg(rrow_ptr + ri + 1);
        if (COUNT) nb += 8;
      }
    }
  }
  unsigned long long* const fw = reinterpret_cast<unsigned long long*>(rset + (kRsetCap + kStateWords) * 32);  // kMeetWords
  fw[lane] = f0;
  fw[32 + lane] = f1;
  const uint32_t cnt = me - mb;
  uint32_t incl = cnt;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t v = __shfl_up_sync(kFull, incl, d);
    if (static_cast<int>(lane) >= d) incl += v;
  }
  const uint32_t total = __shfl_sync(kFull, incl, 31);
  const uint32_t dm = mb - (incl - cnt);  // this lane's pair p is its membership p + dm
  const uint32_t pk = (k & 0xFFFF8000u) | jslot;
  __syncwarp();
  unsigned hits = 0;
  for (uint32_t base = 0; base < total; base += 32) {
    const uint32_t p = base + lane;
    int j = 0;  // owner lane of pair p: # lanes with incl <= p
#pragma unroll
    for (int step = 16; step >= 1; step >>= 1) {
      const int probe_lane = j + step - 1;
      const uint32_t v = __shfl_sync(kFull, incl, probe_lane & 31);
      if (probe_lane < 32 && v <= p) j += step;
    }
    const uint32_t jdm = __shfl_sync(kFull, dm, j), jpk = __shfl_sync(kFull, pk, j);
    const uint32_t jlo = __shfl_sync(kFull, lo, j), jhi = __shfl_sync(kFull, hi, j);
    const uint32_t js = jpk & 31u;
    bool hit = false;
    if (p < total && !((hits >> js) & 1u)) {
      const uint32_t r = p + jdm;
      uint32_t g;
      if (jpk & 0x8000u) {
        g = __ldg(rcol + r);
        if (COUNT) nb += 4;
      } else {
        g = rset[r * 32 + js];
      }
      const DCls cl = pr.cls()[jpk >> 16];
      if (g < cl.nsubj) {
        const unsigned long long ri = cl.rrow_base + static_cast<unsigned long long>(g) * cl.rstride;
        const uint32_t h = __ldg(rrow_ptr + ri + 1);
        uint32_t x = __ldg(rrow_ptr + ri);
        const unsigned long long g0 = fw[j], g1 = fw[32 + j];
        if (COUNT) nb += 8;
        for (; x < h && !hit; x += 4) {
          uint32_t v[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) v[i] = x + i < h ? __ldg(rcol + x + i) : 0u;
          if (COUNT) nb += 4ull * (h - x < 4u ? h - x : 4u);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            if (x + i >= h || hit || !l2_maybe(g0, g1, v[i])) continue;
            hit = l2_verify<COUNT>(col, jlo, jhi, v[i], nb);
          }
        }
      }
    }
    hits |= __reduce_or_sync(kFull, hit ? (1u << js) : 0u);
  }
  if (COUNT) *bytes += nb;
  return hits;
}

// Two-level meet over a closure index, batched like batch_l2: lane j wants "does its range col[lo, hi) list an element
// of its subject's closure row ccol[rb, re)" (rb < re). The rows of the requesting lanes are cut into aligned units --
// 16-byte blocks of 32-bit entries, kClosureBlocks per lane per round, or 32-byte sectors of 16-bit entries, one per
// lane per round (two 16-byte loads: the same registers in flight, four times the entries) -- numbered with one scan
// and dealt out 32 at a time, so neighbouring lanes read neighbouring units of a row and no load waits for another. Each
// entry of a unit that lies inside its row is tested against the owner's 128-bit filter of the range; a "maybe" is
// verified by a binary search of the range. Units of a check already answered are skipped. The COUNT variant counts
// sizeof(E) bytes per entry of a row streamed. fw: kMeetWords words of shared memory per warp. Returns the job slots
// answered.
template <bool COUNT, class E>
__device__ __forceinline__ unsigned closure_meet(const uint32_t* __restrict__ col, const E* ccol, unsigned long long* fw,
                                                 uint32_t lane, bool want, uint32_t lo, uint32_t hi, uint32_t rb, uint32_t re,
                                                 uint32_t jslot, unsigned long long* bytes) {
  constexpr bool kNarrow = sizeof(E) == 2;
  constexpr uint32_t kPer = kNarrow ? 16u : 4u;        // entries per unit
  constexpr int kVec = kNarrow ? 2 : 1;                // 16-byte loads per unit
  constexpr int kUnits = kNarrow ? 1 : kClosureBlocks;  // units per lane per round
  unsigned long long nb = 0;
  unsigned long long f0 = 0, f1 = 0;
  uint32_t b0 = 0, cnt = 0;
  if (want) {
    l2_filter(col, lo, hi, f0, f1);
    if (COUNT) nb += 4ull * (hi - lo);
    b0 = rb / kPer;
    cnt = (re - 1) / kPer + 1 - b0;
  }
  fw[lane] = f0;
  fw[32 + lane] = f1;
  uint32_t incl = cnt;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t v = __shfl_up_sync(kFull, incl, d);
    if (static_cast<int>(lane) >= d) incl += v;
  }
  const uint32_t total = __shfl_sync(kFull, incl, 31);
  const uint32_t db = b0 - (incl - cnt);  // this lane's unit p is unit p + db of ccol
  const unsigned long long cp = reinterpret_cast<unsigned long long>(ccol);
  __syncwarp();
  unsigned hits = 0;
  // This lane's pending "maybe": an entry the filter of owner pj let through, not verified yet (pj < 0: none). The
  // searches are deferred and run for the whole warp at once: verified one by one, nearly every round had a lane whose
  // search the warp waited for.
  int pj = -1;
  uint32_t pv = 0;
  for (uint32_t base = 0; base < total; base += 32u * kUnits) {
    uint4 q[kUnits][kVec];
    int jj[kUnits];  // owner lane of each unit loaded, -1: none
#pragma unroll
    for (int k = 0; k < kUnits; ++k) {
      const uint32_t p = base + 32u * k + lane;
      int j = 0;  // owner lane of unit p: # lanes with incl <= p
#pragma unroll
      for (int step = 16; step >= 1; step >>= 1) {
        const int probe_lane = j + step - 1;
        const uint32_t v = __shfl_sync(kFull, incl, probe_lane & 31);
        if (probe_lane < 32 && v <= p) j += step;
      }
      const uint32_t jdb = __shfl_sync(kFull, db, j & 31), js = __shfl_sync(kFull, jslot, j & 31);
      const uint4* const jcol = reinterpret_cast<const uint4*>(__shfl_sync(kFull, cp, j & 31));
      jj[k] = -1;
#pragma unroll
      for (int h = 0; h < kVec; ++h) q[k][h] = make_uint4(0, 0, 0, 0);
      if (p < total && !((hits >> js) & 1u)) {
        jj[k] = j;
        // all loads of the round in flight together (p + jdb wraps in 32 bits)
#pragma unroll
        for (int h = 0; h < kVec; ++h) q[k][h] = __ldg(jcol + (p + jdb) * kVec + h);
      }
    }
    unsigned mine = 0;  // job slots this lane answered in this round
#pragma unroll
    for (int k = 0; k < kUnits; ++k) {
      const int j = jj[k];
      const uint32_t src = j < 0 ? 0u : static_cast<uint32_t>(j);
      const uint32_t jdb = __shfl_sync(kFull, db, src), js = __shfl_sync(kFull, jslot, src);
      const uint32_t jrb = __shfl_sync(kFull, rb, src), jre = __shfl_sync(kFull, re, src);
      const uint32_t jlo = __shfl_sync(kFull, lo, src), jhi = __shfl_sync(kFull, hi, src);
      if (j < 0) continue;
      const uint32_t w0 = (base + 32u * k + lane + jdb) * kPer;
      if (COUNT) nb += sizeof(E) * static_cast<unsigned long long>(min(jre, w0 + kPer) - max(jrb, w0));
      const unsigned long long g0 = fw[j], g1 = fw[32 + j];
      if constexpr (!kNarrow) {
        const uint32_t v[4] = {q[k][0].x, q[k][0].y, q[k][0].z, q[k][0].w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          if (w0 + i < jrb || w0 + i >= jre || ((mine >> js) & 1u) || !l2_maybe(g0, g1, v[i])) continue;
          if (pj < 0) {
            pj = j;
            pv = v[i];
          } else if (l2_verify<COUNT>(col, jlo, jhi, v[i], nb)) {  // the slot is taken: verify this one now
            mine |= 1u << js;
          }
        }
      } else {
        // 16 entries, two per word (entry 2t in the low half of word t): the filter is tested on all of them first,
        // and only the "maybe"s inside the row reach the one search below (rare: ~2 % of the entries on cfg3)
        const uint32_t w[8] = {q[k][0].x, q[k][0].y, q[k][0].z, q[k][0].w, q[k][1].x, q[k][1].y, q[k][1].z, q[k][1].w};
        uint32_t m = 0;
#pragma unroll
        for (int i = 0; i < 16; ++i) m |= l2_maybe(g0, g1, (w[i >> 1] >> (16 * (i & 1))) & 0xFFFFu) ? 1u << i : 0u;
        const uint32_t first = jrb > w0 ? jrb - w0 : 0u, end = min(jre - w0, kPer);  // the row's entries of the sector
        m &= ((1u << end) - 1u) & ~((1u << first) - 1u);
        while (m && !((mine >> js) & 1u)) {
          const int i = __ffs(m) - 1;
          m &= m - 1;
          uint32_t wi = w[0];
#pragma unroll
          for (int t = 1; t < 8; ++t) wi = (i >> 1) == t ? w[t] : wi;
          const uint32_t v = (wi >> (16 * (i & 1))) & 0xFFFFu;
          if (pj < 0) {
            pj = j;
            pv = v;
          } else if (l2_verify<COUNT>(col, jlo, jhi, v, nb)) {  // the slot is taken: verify this one now
            mine |= 1u << js;
          }
        }
      }
    }
    const unsigned pend = __ballot_sync(kFull, pj >= 0);
    if (__popc(pend) >= kClosureVerify || (pend && base + 32u * kUnits >= total)) {
      const uint32_t src = pj < 0 ? 0u : static_cast<uint32_t>(pj);
      const uint32_t plo = __shfl_sync(kFull, lo, src), phi = __shfl_sync(kFull, hi, src);
      const uint32_t ps = __shfl_sync(kFull, jslot, src);
      if (pj >= 0 && !(((hits | mine) >> ps) & 1u) && l2_verify<COUNT>(col, plo, phi, pv, nb)) mine |= 1u << ps;
      pj = -1;
    }
    hits |= __reduce_or_sync(kFull, mine);
  }
  if (COUNT) *bytes += nb;
  return hits;
}

// Two-level meet over a closure index with signatures: lane j wants "does its range col[lo, hi) list an element of its
// subject's closure row ccol[rb, re)", whose signature (2^lg words) is at sig. The range is the small side (cfg3: ~10
// children against a row of ~80), so each lane tests its own range's children against the row's signature, 8 children
// per round with their loads in flight together, and only the "maybe"s are searched in the row. The searches of a round
// run for the whole warp at once (one lane's search per test would stall the warp once per test). The COUNT variant
// counts 4 bytes per child read, 8 per signature word and sizeof(E) per search probe. Returns the job slots answered.
// SET (the row has a set table, closure_sig.cuh): rb is the row's first bucket in tab, re its bucket count | seed << 24,
// and the "maybe"s of a round are confirmed by one exact lookup each, all in flight together, instead of searches: one
// dependent load per round instead of ~7 per "maybe", and no lane waits on another's search. 8 bytes per lookup.
constexpr uint32_t kSigTests = 8;  // children per round of a signature meet (4 spilled a little less in check_kernel
                                   // and ran no faster on cfg3: DESIGN.md §6)
// One round of a lane's signature meet: loads the children col[lo, lo + n) (n <= kSigTests) into v, all in flight
// together, then their signature words, and returns the mask of the children whose test said maybe. 12 bytes per child.
template <bool COUNT>
__device__ __forceinline__ unsigned sig_round(const uint32_t* __restrict__ col, uint32_t lo, uint32_t n,
                                              const unsigned long long* __restrict__ sig, uint32_t lg, uint32_t (&v)[kSigTests],
                                              unsigned long long& nb) {
#pragma unroll
  for (uint32_t i = 0; i < kSigTests; ++i) v[i] = i < n ? __ldg(col + lo + i) : 0u;
  unsigned long long w[kSigTests];
#pragma unroll
  for (uint32_t i = 0; i < kSigTests; ++i) w[i] = i < n ? __ldg(sig + sig_word(v[i], lg)) : 0ull;
  unsigned m = 0;
#pragma unroll
  for (uint32_t i = 0; i < kSigTests; ++i) {
    const unsigned long long b = sig_mask(v[i]);
    m |= (i < n && (w[i] & b) == b) ? 1u << i : 0u;
  }
  if (COUNT) nb += 12ull * n;
  return m;
}
// The "maybe"s m of a round confirmed in the row's set table (buckets tab[0, nbk), hashed under seed): one exact lookup
// each, all in flight together. True iff one of them is in the row. 8 bytes per lookup.
template <bool COUNT>
__device__ __forceinline__ bool table_round(const unsigned long long* __restrict__ tab, uint32_t nbk, uint32_t seed,
                                            unsigned m, const uint32_t (&v)[kSigTests], unsigned long long& nb) {
  unsigned long long w[kSigTests];
#pragma unroll
  for (uint32_t i = 0; i < kSigTests; ++i) w[i] = (m >> i) & 1u ? __ldg(tab + table_bucket(v[i], seed, nbk)) : ~0ull;
  bool h = false;
#pragma unroll
  for (uint32_t i = 0; i < kSigTests; ++i) h = h || (((m >> i) & 1u) && table_has(w[i], v[i]));
  if (COUNT) nb += 8ull * __popc(m);
  return h;
}

template <bool COUNT, bool SET = false, class E>
__device__ __forceinline__ unsigned sig_meet(const uint32_t* __restrict__ col, const E* __restrict__ ccol,
                                             const unsigned long long* __restrict__ sig, uint32_t lg, bool want, uint32_t lo,
                                             uint32_t hi, uint32_t rb, uint32_t re, uint32_t jslot,
                                             unsigned long long* bytes, const unsigned long long* __restrict__ tab = nullptr) {
  constexpr uint32_t kTests = kSigTests;
  unsigned long long nb = 0;
  unsigned hits = 0;
  bool more = want && lo < hi;
  while (__any_sync(kFull, more)) {
    uint32_t v[kTests];
    unsigned m = 0;  // the children of this round whose test said maybe
    if (more) {
      const uint32_t n = min(hi - lo, kTests);
      m = sig_round<COUNT>(col, lo, n, sig, lg, v, nb);
      lo += n;
      if constexpr (SET) m = table_round<COUNT>(tab + rb, re & 0xFFFFFFu, re >> 24, m, v, nb) ? 1u : 0u;  // (as a hit below)
    }
    bool hit = false;
    if constexpr (SET) {
      hit = m != 0;
      m = 0;
    }
    while (!SET && __any_sync(kFull, m != 0)) {
      if (m) {
        const uint32_t i = __ffs(m) - 1;
        m &= m - 1;
        uint32_t vi = v[0];
#pragma unroll
        for (uint32_t t = 1; t < kTests; ++t) vi = i == t ? v[t] : vi;
        if (l2_verify<COUNT>(ccol, rb, re, vi, nb)) {
          hit = true;
          m = 0;
        }
      }
    }
    hits |= __reduce_or_sync(kFull, hit ? 1u << jslot : 0u);
    more = more && lo < hi && !((hits >> jslot) & 1u);
  }
  if (COUNT) *bytes += nb;
  return hits;
}

// Warp-collective node visit: every lane may carry one (job slot, object, unit).
// Evaluates the unit's steps at the object: membership-of-itself test, direct and
// wildcard probes (from the subject's reverse-row set when the job is inverted, else a
// binary search of the row), and pushes the userset / arrow edge ranges. MEET = kMeetNone: the schema has no two-level
// step, and the two-level meet is left out (its code costs the traversal loop registers: cfg4, DESIGN.md §6); else the
// width of the closure entries the meet reads (kMeet16 / kMeet32: one closure_meet is inlined per instantiation;
// kMeetSig16 / kMeetSig32: sig_meet instead, for snapshots whose every built index has signatures; kMeetSet16:
// sig_meet confirming in set tables, for snapshots whose every built index has signatures and a set table).
template <bool COUNT, int MEET>
__device__ __forceinline__ void visit(const KParams& p, const Prog& pr, WarpCtx<COUNT>& c, bool active,
                                      uint32_t jslot, uint32_t obj, uint32_t unit, uint32_t depth) {
  const uint32_t sid = __shfl_sync(kFull, c.my_subj, jslot & 31);
  const uint32_t ss = __shfl_sync(kFull, c.my_ss, jslot & 31);
  const unsigned long long cst = __shfl_sync(kFull, c.my_cst, jslot & 31);
  const uint32_t stype = ss >> 16, srel = ss & 0xFFFFu;
  bool hit = false;
  int sb = 0, nprobe = 0, npush = 0;
#if ZG_PHASE_CLOCKS
  long long l1_cycles = 0;  // this lane's time in one-level meets (lanes of a warp run them side by side)
#endif
  if (active) {
    const DUnit u = pr.units()[unit];
    if (srel != kNone && sid == obj)
      for (int m = u.mem_begin; m < u.mem_end; ++m) hit = hit || pr.members()[m] == srel;
    if (!hit) {
      sb = u.step_begin;
      nprobe = u.push_begin - u.step_begin;
      npush = u.step_end - u.push_begin;
    }
  }
  // meets: the job may meet in the middle; inverted: its memberships are in the per-check set as well
  const bool meets = (c.inv_mask >> (jslot & 31)) & 1u, inverted = meets && !((cst >> kOverCap) & 1u);
  // ---- probes (DIRECT / WILD classes): every lane on its own, no warp collective involved. The steps of a unit
  // are ordered probes first (schema.cc); in round 1 every step, probe or not, went through the collective push.
  for (int i = 0; i < nprobe && !hit; ++i) {
    const DStep st = pr.steps()[sb + i];
    const bool expiry = (st.flags & CF_EXPIRY) != 0;
    const bool subject_fits = srel == kNone && stype == st.stype;
    if (!subject_fits || (st.kind == ST_WILD && p.no_wildcards)) continue;
    if (st.kind == ST_DIRECT && inverted && (st.flags & CF_INVERT)) {
      // direction-optimised probe: is obj among the subject's memberships of this class?
      const uint32_t kb = cst_at(cst, st.tinv), ke = cst_at(cst, st.tinv + 1u);
      for (uint32_t r = kb; r < ke; ++r)
        hit = hit || c.rset[r * 32 + (jslot & 31)] == obj;
    } else {
      hit = probe_step(p, c, st, obj, sid, expiry);
    }
  }
  if (hit) npush = 0;
  sb += nprobe;
  // ---- edge classes that may push a range (userset subjects, arrows): warp-collective
  const int maxsteps = __reduce_max_sync(kFull, npush);
  for (int i = 0; i < maxsteps; ++i) {
    using CE = typename ClosureEntry<MEET>::type;
    constexpr bool kSig = (MEET & kMeetSig) != 0, kSet = (MEET & kMeetSet) != 0;
    bool want = false, l2_want = false, cl_want = false;
    uint32_t l2_lo = 0, l2_hi = 0, l2_k = 0, cl_rb = 0, cl_re = 0, cl_lg = 0;
    const CE* cl_col = nullptr;
    const unsigned long long* cl_sig = nullptr;
    const unsigned long long* cl_tab = nullptr;  // kSet: the set table's buckets
    uint4 item = make_uint4(0, 0, 0, 0);
    if (i < npush && !hit) {
      const DStep st = pr.steps()[sb + i];
      const bool expiry = (st.flags & CF_EXPIRY) != 0;
      if (obj < st.nres) {
        const unsigned long long ridx = st.row_base + static_cast<unsigned long long>(obj) * st.ncls;
        const uint32_t lo = __ldg(p.row_ptr + ridx), hi = __ldg(p.row_ptr + ridx + 1);
        if (COUNT) c.bytes += 8;
        // A two-level step whose pair has a closure index reads the subject's row of it: its offsets depend on the
        // subject alone, so they are loaded together with the range's instead of after them.
        const CE* ccol = nullptr;
        uint32_t rb = 0, re = 0;
        bool crow_read = false;  // (counted where the offsets are used)
        if (MEET != kMeetNone && (st.flags & kStepTargetL2) && meets && depth + 2 <= ZG_MAX_DEPTH) {
          const uint32_t* crow = nullptr;
          uint32_t cn = 0;
#pragma unroll
          for (int k = 0; k < kMaxClosure; ++k)  // (by value: the address of a kernel parameter costs a local copy)
            if (k < static_cast<int>(p.n_closure) && p.closure[k].tgc == st.tgc && p.closure[k].width == sizeof(CE) &&
                (!kSig || p.closure[k].sig) && (!kSet || p.closure[k].set_hdr)) {
              crow = kSet ? reinterpret_cast<const uint32_t*>(p.closure[k].set_hdr) : p.closure[k].row_ptr;
              ccol = static_cast<const CE*>(p.closure[k].col);
              cn = p.closure[k].nsubj;
              if (kSig) {
                cl_sig = p.closure[k].sig;
                cl_lg = __ffs(p.closure[k].sig_words) - 1;
              }
              if (kSet) cl_tab = p.closure[k].set_tab;
            }
          if (crow && stype == st.tstype && sid < cn) {
            if (kSet) {  // rb: the row's first bucket, re: its bucket count | seed << 24 (closure_sig.cuh table_header)
              const unsigned long long h = __ldg(reinterpret_cast<const unsigned long long*>(crow) + sid);
              rb = static_cast<uint32_t>(h);
              re = static_cast<uint32_t>(h >> 32);
            } else {
              rb = __ldg(crow + sid);
              re = __ldg(crow + sid + 1);
            }
            crow_read = true;
            if (kSig) {
              cl_sig += static_cast<unsigned long long>(sid) << cl_lg;
              // The signature's line is wanted two dependent loads later (after the range's offsets and children):
              // fetched into L1 now, its tests hit there (cfg3 +0.5 %, H100, DESIGN.md §6; prefetching the row's
              // lines for the searches as well cost 18 %).
#ifndef ZG_EMULATE
              asm volatile("prefetch.global.L1 [%0];" ::"l"(cl_sig));
#endif
            }
          }
        }
        if (hi > lo) {
          if ((st.flags & kStepTargetLeaf) && inverted && !expiry && depth + 1 <= ZG_MAX_DEPTH) {
            // Children of this range can only be answered by "is the child one of the
            // subject's memberships of class tinv": meet in the middle. No membership (or a
            // child class for another subject type): nothing can match.
            const uint32_t kb = cst_at(cst, st.tinv), ke = stype == st.tstype ? cst_at(cst, st.tinv + 1u) : kb;
            if (ke - kb > hi - lo) {  // fewer children than memberships: visit the children
              want = true;
              item = make_uint4(lo, hi, make_meta(jslot, depth + 1, false, st.tslot), 0);
            } else {
              // For each membership key ask ITS reverse row (short, and shared by every range
              // of this check, so it stays in L1): "does this object list the key as a subject
              // of class gc". Two searches are advanced together for memory-level parallelism.
#if ZG_PHASE_CLOCKS
              const long long t1 = clock64();
#endif
              const DCls cl = pr.cls()[st.gc];
              for (uint32_t r = kb; r < ke && !hit; r += 2) {
                uint32_t l0 = 0, h0 = 0, l1 = 0, h1 = 0;
                const uint32_t m0 = c.rset[r * 32 + (jslot & 31)];
                const uint32_t m1 = r + 1 < ke ? c.rset[(r + 1) * 32 + (jslot & 31)] : 0xFFFFFFFFu;
                if (m0 < cl.nsubj) {
                  const unsigned long long ri = cl.rrow_base + static_cast<unsigned long long>(m0) * cl.rstride;
                  l0 = __ldg(p.rrow_ptr + ri);
                  h0 = __ldg(p.rrow_ptr + ri + 1);
                  if (COUNT) c.bytes += 8;
                }
                if (m1 < cl.nsubj) {
                  const unsigned long long ri = cl.rrow_base + static_cast<unsigned long long>(m1) * cl.rstride;
                  l1 = __ldg(p.rrow_ptr + ri);
                  h1 = __ldg(p.rrow_ptr + ri + 1);
                  if (COUNT) c.bytes += 8;
                }
                bool hit0 = false, hit1 = false;
                probe2(p.rcol, c, l0, h0, obj, l1, h1, obj, hit0, hit1);
                hit = hit0 || hit1;
              }
#if ZG_PHASE_CLOCKS
              l1_cycles += clock64() - t1;
#endif
            }
          } else if (MEET != kMeetNone && (st.flags & kStepTargetL2) && meets && depth + 2 <= ZG_MAX_DEPTH &&
                     (ccol || inverted || hi - lo <= static_cast<uint32_t>(kFCap))) {
            // Two levels at once (namespace -> team#member -> group#member -> user): a child t of this
            // range matches iff some membership g of the subject (class tinv) is a subject of t in the
            // children's single class tgc. The reverse row of g in that class lists exactly those t, in
            // ascending order like this range: the answer is "do the two sorted segments intersect",
            // once per membership. The children are never visited, nothing is pushed. A subject with more
            // memberships than the per-check set holds meets too: over a closure index whatever the range's
            // size (the index does not read the set), else through batch_l2, which reads them from its reverse
            // row; without an index, a range of more than kFCap children is walked.
            const uint32_t kb = cst_at(cst, st.tinv), ke = stype == st.tstype ? cst_at(cst, st.tinv + 1u) : kb;
            if (ccol) {
              // The pair has a closure index: the union of the memberships' reverse rows is the subject's row of it.
              // Ranges of up to kFCap children are handed to the whole warp below (closure_meet); a larger one is
              // intersected with the row by this lane.
              if (COUNT && crow_read) c.bytes += 8;
              if (kSig || hi - lo <= static_cast<uint32_t>(kFCap)) {  // (sig_meet's cost does not grow with the row)
                cl_want = kSet ? (re & 0xFFFFFFu) != 0 : re > rb;
                l2_lo = lo;
                l2_hi = hi;
                cl_rb = rb;
                cl_re = re;
                cl_col = ccol;
              } else {
                hit = intersects(p.col, lo, hi, ccol, rb, re, c);
              }
            } else if (hi - lo <= static_cast<uint32_t>(kFCap) && (inverted ? ke > kb : stype == st.tstype)) {
              // handed to the whole warp below (batch_l2)
              l2_want = true;
              l2_lo = lo;
              l2_hi = hi;
              l2_k = (inverted ? kb | (ke << 8) : 0x8000u | st.tinv) | (static_cast<uint32_t>(st.tgc) << 16);
            } else {
              // An inverted check whose range has more than kFCap children: this lane intersects the range with
              // each membership's reverse row on its own.
              const DCls cl = pr.cls()[st.tgc];
              for (uint32_t r = kb; r < ke && !hit; ++r) {
                const uint32_t g = c.rset[r * 32 + (jslot & 31)];
                if (g >= cl.nsubj) continue;
                const unsigned long long ri = cl.rrow_base + static_cast<unsigned long long>(g) * cl.rstride;
                const uint32_t l = __ldg(p.rrow_ptr + ri), h = __ldg(p.rrow_ptr + ri + 1);
                if (COUNT) c.bytes += 8;
                hit = intersects(p.col, lo, hi, p.rcol, l, h, c);
              }
            }
          } else {
            want = true;
            item = make_uint4(lo, hi, make_meta(jslot, depth + 1, expiry, st.tslot), 0);
          }
        }
      }
    }
    if (MEET != kMeetNone && __ballot_sync(kFull, l2_want)) {
#if ZG_PHASE_CLOCKS
      const long long t2 = clock64();
#endif
      unsigned long long cb = 0;
      c.found |= batch_l2<COUNT>(p.col, p.rrow_ptr, p.rcol, c.rset, c.lane, l2_want && !((c.found >> jslot) & 1u), l2_lo,
                                 l2_hi, l2_k, jslot & 31u, sid, stype, COUNT ? &cb : nullptr);
      if (COUNT) c.bytes += cb;
#if ZG_PHASE_CLOCKS
      c.ph[2] += clock64() - t2;
#endif
    }
    if (MEET != kMeetNone && __ballot_sync(kFull, cl_want)) {
#if ZG_PHASE_CLOCKS
      const long long t2 = clock64();
#endif
      unsigned long long cb = 0;
      if constexpr (kSet)
        c.found |= sig_meet<COUNT, true>(p.col, cl_col, cl_sig, cl_lg, cl_want && !((c.found >> jslot) & 1u), l2_lo, l2_hi,
                                         cl_rb, cl_re, jslot & 31u, COUNT ? &cb : nullptr, cl_tab);
      else if constexpr (kSig)
        c.found |= sig_meet<COUNT>(p.col, cl_col, cl_sig, cl_lg, cl_want && !((c.found >> jslot) & 1u), l2_lo, l2_hi, cl_rb,
                                   cl_re, jslot & 31u, COUNT ? &cb : nullptr);
      else
        c.found |= closure_meet<COUNT>(p.col, cl_col, reinterpret_cast<unsigned long long*>(c.rset + (kRsetCap + kStateWords) * 32),
                                       c.lane, cl_want && !((c.found >> jslot) & 1u), l2_lo, l2_hi, cl_rb, cl_re, jslot & 31u,
                                       COUNT ? &cb : nullptr);
      if (COUNT) c.bytes += cb;
#if ZG_PHASE_CLOCKS
      c.ph[2] += clock64() - t2;
#endif
    }
    push(c, want, item);
  }
  c.found |= __reduce_or_sync(kFull, hit ? (1u << jslot) : 0u);
#if ZG_PHASE_CLOCKS
  for (int d = 16; d >= 1; d >>= 1) l1_cycles = max(l1_cycles, __shfl_xor_sync(kFull, l1_cycles, d));
  c.ph[3] += l1_cycles;
#endif
}

__device__ __forceinline__ uint32_t kleene_or(uint32_t a, uint32_t b) {  // 0 F, 1 T, 2 E
  return (a == 1 || b == 1) ? 1u : ((a == 2 || b == 2) ? 2u : 0u);
}
__device__ __forceinline__ uint32_t kleene_and(uint32_t a, uint32_t b) {
  return (a == 0 || b == 0) ? 0u : ((a == 2 || b == 2) ? 2u : 1u);
}

// Postfix boolean program of a non-pure permission over its leaf values (2 bits per leaf in
// `vals`: 0 F, 1 T, 2 E). Kleene's E doubles as "not evaluated yet": the connectives are monotone,
// so a result that is not E cannot change whatever the missing leaves turn out to be.
__device__ __forceinline__ uint32_t eval_tree(const Prog& pr, const DTree& t, unsigned long long vals, bool trivial_self,
                                              uint32_t srel) {
  unsigned long long st = 0;  // 2-bit entries
  int sp = 0;
  for (int i = t.op_begin; i < t.op_end; ++i) {
    const DTreeOp o = pr.tree_ops()[i];
    if (o.kind == T_LEAF) {
      st |= ((vals >> (2u * o.arg)) & 3ull) << (2 * sp);
      ++sp;
    } else if (o.kind == T_TRIVIAL) {
      const unsigned long long v = (trivial_self && srel == o.arg) ? 1ull : 0ull;
      st |= v << (2 * sp);
      ++sp;
    } else {
      const uint32_t b = (st >> (2 * (sp - 1))) & 3u, a = (st >> (2 * (sp - 2))) & 3u;
      uint32_t v;
      if (o.kind == T_OR) v = kleene_or(a, b);
      else if (o.kind == T_AND) v = kleene_and(a, b);
      else v = kleene_and(a, b == 1 ? 0u : (b == 0 ? 1u : 2u));
      sp -= 2;
      st &= ~(0xFull << (2 * sp));
      st |= static_cast<unsigned long long>(v) << (2 * sp);
      ++sp;
    }
  }
  return static_cast<uint32_t>(st & 3u);
}

// Streamed admission: spin until `need` leading queries have landed. If the feed stopped (a failed copy) give
// up after seconds instead of hanging the device: the flag fails the host call, whatever is answered from
// there on is discarded.
__device__ __noinline__ void wait_ready(const unsigned long long* ready, unsigned long long need, uint32_t* flags) {
  const volatile unsigned long long* rd = ready;
  uint32_t spins = 0;
  while (*rd < need && spins < (1u << 23)) {
    __nanosleep(256);
    ++spins;
  }
  if (spins >= (1u << 23)) atomicOr(flags, 32u);
  // CTA-scope fence: orders the item loads after the poll without the L1 invalidate a device-scope fence
  // costs (the items are read with ld.global.cg, which does not use L1)
  __threadfence_block();
}

// Per-lane query state parked in shared memory while the warp traverses (kStateWords words):
//   0 resource object, 1 depth | leaves << 8 | is-tree << 15 | leaf_begin-or-unit << 16,
//   2 tree id, 3 / 4 leaf values (2 bits each)
// RESIDUAL: the residual pass of flat_check_kernel (KParams::idx / nq_dev; kMeetSet16, not streamed). Its own
// instantiation: the fields cost the plain kernel's traversal loop spills (DESIGN.md §4).
template <bool COUNT, bool STREAMED = false, int MEET = kMeet32, bool RESIDUAL = false>
__global__ void __launch_bounds__(kThreads, kMinBlocks) check_kernel(const KParams p) {
  static_assert(!RESIDUAL || (MEET == kMeetSet16 && !STREAMED), "the residual pass follows flat_check_kernel");
  constexpr bool kResidual = RESIDUAL;
  unsigned long long nq = p.nq;
  if (kResidual) {
#ifndef ZG_EMULATE
    cudaGridDependencySynchronize();  // launched as flat_check_kernel's programmatic dependent: wait for its residual
#endif
    nq = *p.nq_dev;
    if (nq == 0) return;
  }
  // the index in queries / out / val of the pass's i-th query
  auto qidx = [&](unsigned long long i) -> unsigned long long { return kResidual ? p.idx[i] : i; };
  ZG_DYNAMIC_SMEM(smem);
  for (uint32_t i = threadIdx.x; i < p.prog_bytes / 16; i += blockDim.x)
    reinterpret_cast<uint4*>(smem)[i] = reinterpret_cast<const uint4*>(p.prog)[i];
  __syncthreads();
  const Prog pr = make_prog(smem);
  const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  WarpCtx<COUNT> c;
  c.lane = lane;
  uint8_t* wsm = smem + p.prog_bytes + warp * kWarpSmem;
  c.stack = reinterpret_cast<uint4*>(wsm);
  c.rset = reinterpret_cast<uint32_t*>(wsm + kStackCap * sizeof(uint4));
  uint32_t* const state = c.rset + kRsetCap * 32 + lane;  // word k at state[k * 32]
  c.spill = p.spill + (static_cast<size_t>(blockIdx.x) * kWarpsPerBlock + warp) * p.spill_cap;
  c.spill_cap = p.spill_cap;
  c.bytes = 0;
  c.events = p.events;
  const uint32_t n_slots = pr.hdr()->n_slots, n_types = pr.hdr()->n_types;
  unsigned long long* const memo = p.memo + (static_cast<size_t>(blockIdx.x) * kWarpsPerBlock + warp) * p.memo_entries;
#if ZG_PHASE_CLOCKS
  for (int i = 0; i < kPhases; ++i) c.ph[i] = 0;
#endif

  for (;;) {
    unsigned long long base = 0;
    if (lane == 0) {
      base = atomicAdd(p.next, 32ull);
      // the copy engine is still feeding the queries: wait until this batch has landed
      if (STREAMED && base < nq) wait_ready(p.ready, base + 32 < nq ? base + 32 : nq, p.flags);
    }
    base = __shfl_sync(kFull, base, 0);
    if (base >= nq) break;
#if ZG_PHASE_CLOCKS
    const long long t_adm = clock64();
#endif
    const unsigned long long q = base + lane;
    const bool valid = q < nq;
    bool bad = false, expansive = false, no_rset = false;
    uint32_t nl = 0;
    c.my_subj = 0;
    c.my_ss = (0u << 16) | kNone;
    if (valid) {
      // ld.global.cg when the items are streamed in: nothing about them may come from a non-coherent cache
      const uint4 raw = STREAMED ? __ldcg(reinterpret_cast<const uint4*>(p.queries) + q)
                                 : __ldg(reinterpret_cast<const uint4*>(p.queries) + qidx(q));
      if (COUNT) c.bytes += 17;
      c.my_subj = raw.y;
      const uint32_t perm = raw.z & 0xFFFFu, stype = raw.z >> 16;
      const uint32_t srel = raw.w & 0xFFFFu, fl = p.raw_items ? 0u : raw.w >> 16;
      c.my_ss = (stype << 16) | srel;
      uint32_t w1 = fl & kJobDepthMask, tree = 0;
      if (stype >= n_types || (srel != kNone && (srel >= n_slots || pr.slots()[srel].type != stype))) bad = true;
      if (perm >= n_slots) {
        bad = true;
      } else {
        const DSlot s = pr.slots()[perm];
        no_rset = (s.flags & SF_NO_RSET) != 0;
        if (s.kind == SK_NONPURE) {
          const DTree t = pr.trees()[s.unit];
          tree = s.unit;
          nl = t.n_leaves;
          expansive = (t.flags & UF_EXPANSIVE) != 0;
          w1 |= (nl << 8) | (1u << 15) | (static_cast<uint32_t>(t.leaf_begin) << 16);
        } else {
          nl = 1;
          expansive = (pr.units()[s.unit].flags & UF_EXPANSIVE) != 0;
          w1 |= (1u << 8) | (static_cast<uint32_t>(s.unit) << 16);
        }
      }
      state[0] = raw.x;
      state[32] = w1;
      state[64] = tree;
      state[96] = 0xAAAAAAAAu;  // every leaf: E = not evaluated yet
      state[128] = 0xAAAAAAAAu;
    }
    // ---- direction-optimised probes: load the subject's reverse rows (its direct
    // memberships, class by class) when the check can fan out and they are few. Loaded once per
    // query: every leaf of a non-pure permission shares them.
    {
      bool inv = p.invert && valid && !bad && (c.my_ss & 0xFFFFu) == kNone && expansive;
      uint32_t rcnt = 0;
      unsigned long long cst = 0;
      int ib = 0, ncl = 0;
      if (inv) {
        const DTypeInv ti = pr.type_inv()[c.my_ss >> 16];
        ib = ti.begin;
        ncl = ti.end - ti.begin;
        if (ncl > kMaxInvClasses) {
          inv = false;
          ncl = 0;
        }
      }
      const bool meet = inv;  // stays when the memberships overflow the set: the two-level meet reads them itself
      if (no_rset) {
        // No step this check evaluates at the root reads the set: its probes are not invertible and its pushes
        // meet over a closure index (SF_NO_RSET). The check is admitted as one whose memberships overflow the set
        // (kOverCap), a state every reader of the set already handles without it: a direct probe searches the
        // forward row, the one-level meet is skipped (its range is visited), a two-level step with an index meets
        // over the subject's closure row whatever the range's size (visit), one without reads the memberships from
        // the subject's reverse row (batch_l2) or, past kFCap children, visits the range, and the children a step
        // pushes at the depth limit are visited like any other check's. Nothing is loaded.
        inv = false;
        ncl = 0;
      }
      const int maxcl = __reduce_max_sync(kFull, ncl);
      for (int i = 0; i < maxcl; ++i) {
        if (inv && i < ncl) {
          const uint32_t gc = pr.inv_cls()[ib + i];
          const DCls cl = pr.cls()[gc];
          if (!(cl.flags & CF_EMPTY) && c.my_subj < cl.nsubj) {
            const unsigned long long ri = cl.rrow_base + static_cast<unsigned long long>(c.my_subj) * cl.rstride;
            const uint32_t b = __ldg(p.rrow_ptr + ri);
            const uint32_t e = __ldg(p.rrow_ptr + ri + 1);
            if (COUNT) c.bytes += 8;
            if (rcnt + (e - b) > static_cast<uint32_t>(kRsetCap)) {
              inv = false;  // too many memberships: this check probes forward
            } else {
              for (uint32_t x = b; x < e; ++x) {
                c.rset[rcnt * 32 + lane] = __ldg(p.rcol + x);
                ++rcnt;
              }
              if (COUNT) c.bytes += 4ull * (e - b);
            }
          }
          cst |= static_cast<unsigned long long>(rcnt) << (5u * (i + 1));
        }
      }
      if (meet && !inv) cst |= 1ull << kOverCap;
      c.inv_mask = __ballot_sync(kFull, meet);
      c.my_cst = cst;
      __syncwarp();
    }
#if ZG_PHASE_CLOCKS
    c.ph[0] += clock64() - t_adm;
#endif
    c.fatal = false;
    bool undet = valid && !bad;
    uint32_t res = 2;  // invalid query -> error
    const int maxnl = __reduce_max_sync(kFull, undet ? static_cast<int>(nl) : 0);
    for (int l = 0; l < maxnl; ++l) {
      const bool act = undet && l < static_cast<int>(nl);
      const unsigned live_jobs = __ballot_sync(kFull, act);
      if (!live_jobs) continue;
      uint32_t obj = 0, unit = 0, depth = 0;
      if (act) {
        obj = state[0];
        const uint32_t w1 = state[32];
        depth = w1 & kJobDepthMask;
        unit = (w1 >> 15) & 1u ? pr.leaf_units()[(w1 >> 16) + l] : (w1 >> 16);
      }
      c.found = 0;
      c.err = 0;
      c.raised = 0;
      c.top = 0;
      c.spill_top = 0;

#if ZG_PHASE_CLOCKS
      long long t_ph = clock64(), meets = c.ph[2] + c.ph[3];  // root visit and pop loop exclude the meets inside them
#endif
      visit<COUNT, MEET>(p, pr, c, act, lane, obj, unit, depth);
#if ZG_PHASE_CLOCKS
      {
        const long long now = clock64(), m = c.ph[2] + c.ph[3];
        c.ph[1] += (now - t_ph) - (m - meets);
        t_ph = now;
        meets = m;
      }
#endif

      uint32_t iters = 0;
      bool use_memo = false;
      for (;;) {
        if (!c.fatal && c.top == 0) {
          if (c.spill_top == 0) break;
          refill(c);
        }
        if ((c.found & live_jobs) == live_jobs) break;  // every check already answered
        if (++iters > p.budget || c.fatal) {
          if (lane == 0) atomicOr(p.flags, c.fatal ? 1u : 4u);
          c.err |= live_jobs & ~c.found;
          break;
        }
        if (!use_memo && p.memo_entries && iters > p.memo_after) {
          // this batch is expanding far more than usual: path multiplicity. Remember child
          // visits from here on; an identical (job, slot, object, depth) visit is skipped.
          for (uint32_t i = lane; i < p.memo_entries; i += 32) memo[i] = 0ull;
          if (lane == 0) atomicAdd(p.events + 1, 1ull);
          __syncwarp();
          use_memo = true;
        }
        // ---- pop ranges worth <= 32 edges from the top of the stack
        const int n = c.top < 32 ? c.top : 32;
        uint4 it = make_uint4(0, 0, 0, 0);
        if (static_cast<int>(lane) < n) it = c.stack[c.top - 1 - lane];
        const bool dead = (c.found >> (it.z & 31)) & 1u;
        const uint32_t len = (static_cast<int>(lane) < n && !dead) ? it.y - it.x : 0u;
        uint32_t incl = len;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
          uint32_t v = __shfl_up_sync(kFull, incl, d);
          if (static_cast<int>(lane) >= d) incl += v;
        }
        const uint32_t excl = incl - len;
        const unsigned fullm = __ballot_sync(kFull, static_cast<int>(lane) < n && incl <= 32u);
        const int nfull = __popc(fullm);  // prefix of fully consumed items
        uint32_t total = __shfl_sync(kFull, incl, 31);
        if (total > 32u) total = 32u;
        __syncwarp();
        if (static_cast<int>(lane) == nfull && static_cast<int>(lane) < n)  // partially consumed item stays on top
          c.stack[c.top - 1 - lane].x = it.x + (32u - excl);
        c.top -= nfull;
        __syncwarp();
        // ---- lane k takes edge k: owner item j = #items with incl <= k
        int j = 0;
#pragma unroll
        for (int step = 16; step >= 1; step >>= 1) {
          const int probe_lane = j + step - 1;
          const uint32_t v = __shfl_sync(kFull, incl, probe_lane & 31);
          if (probe_lane < 32 && v <= lane) j += step;
        }
        const uint32_t jb = __shfl_sync(kFull, it.x, j & 31);
        const uint32_t jmeta = __shfl_sync(kFull, it.z, j & 31);
        const uint32_t jexcl = __shfl_sync(kFull, excl, j & 31);
        bool active = lane < total;
        const uint32_t jslot = jmeta & 31u, cdepth = (jmeta >> 5) & 63u, tslot = jmeta >> 16;
        uint32_t child = 0;
        const uint32_t sq_subj = __shfl_sync(kFull, c.my_subj, jslot);
        const uint32_t sq_ss = __shfl_sync(kFull, c.my_ss, jslot);
        if (active) {
          const uint32_t e = jb + (lane - jexcl);
          child = __ldg(p.col + e);
          if (COUNT) c.bytes += 4;
          if (jmeta & (1u << 11)) {
            const uint32_t ex = __ldg(p.exp + e);
            if (COUNT) c.bytes += 4;
            active = ex == 0 || ex > p.now;
          }
        }
        // the 51st hop is an error (pkg/spicedb/spicedb.go:33)
        const bool too_deep = active && cdepth > ZG_MAX_DEPTH;
        c.err |= __reduce_or_sync(kFull, too_deep ? (1u << jslot) : 0u);
        active = active && !too_deep;
        if (use_memo && active) {
          // exact key (a visit at another depth has another hop budget, so depth is part of it);
          // direct-mapped and lossy: a lost entry only costs a repeated visit
          const unsigned long long key = (1ull << 59) | (static_cast<unsigned long long>(jslot) << 54) |
                                         (static_cast<unsigned long long>(cdepth) << 48) |
                                         (static_cast<unsigned long long>(tslot) << 32) | child;
          unsigned long long hsh = key * 0x9E3779B97F4A7C15ull;
          const uint32_t at = static_cast<uint32_t>(hsh >> 40) & (p.memo_entries - 1u);
          if (memo[at] == key) active = false;
          else memo[at] = key;
        }
        uint32_t cunit = 0;
        bool raise = false;
        if (active) {
          const DSlot s = pr.slots()[tslot];
          const bool remote = p.shard_count > 1 && (child % p.shard_count) != p.shard_rank;
          if (s.kind == SK_NONPURE || remote) {
            // defer: Check(child#tslot @ S) becomes a sub-query of the next pass
            const unsigned long long at = atomicAdd(p.subq_count, 1ull);
            if (at < p.subq_cap) {
              zg_check sq;
              sq.res = child;
              sq.subj = sq_subj;
              sq.perm = static_cast<uint16_t>(tslot);
              sq.stype = static_cast<uint16_t>(sq_ss >> 16);
              sq.srel = static_cast<uint16_t>(sq_ss & 0xFFFFu);
              sq.flags = static_cast<uint16_t>(cdepth);
              p.subq[at] = sq;
              p.subq_parent[at] = static_cast<uint32_t>(qidx(base + jslot) * p.L + l);
            } else {
              atomicOr(p.flags, 2u);
            }
            raise = true;
            active = false;
          } else {
            cunit = s.unit;
          }
        }
        c.raised |= __reduce_or_sync(kFull, raise ? (1u << jslot) : 0u);
        visit<COUNT, MEET>(p, pr, c, active, jslot, child, cunit, cdepth);
      }
#if ZG_PHASE_CLOCKS
      c.ph[4] += (clock64() - t_ph) - (c.ph[2] + c.ph[3] - meets);
#endif

      if (act) {
        const bool t = (c.found >> lane) & 1u, e = (c.err >> lane) & 1u, r = (c.raised >> lane) & 1u;
        if (p.val) p.val[qidx(q) * p.L + l] = t ? kValT : (e ? kValE : 0);
        // a leaf that raised sub-queries is not final unless it is already true
        const uint32_t v = t ? 1u : ((e || r) ? 2u : 0u);
        const uint32_t w1 = state[32];
        if ((w1 >> 15) & 1u) {
          unsigned long long vals = (static_cast<unsigned long long>(state[128]) << 32) | state[96];
          vals = (vals & ~(3ull << (2 * l))) | (static_cast<unsigned long long>(v) << (2 * l));
          state[96] = static_cast<uint32_t>(vals);
          state[128] = static_cast<uint32_t>(vals >> 32);
          const uint32_t srel = c.my_ss & 0xFFFFu;
          res = eval_tree(pr, pr.trees()[state[64]], vals, c.my_subj == state[0], srel);
          if (res != 2u || l + 1 == static_cast<int>(nl)) undet = false;
        } else {
          res = v;
          undet = false;
        }
      }
    }
    if (valid && p.out) {
      const unsigned long long qi = qidx(q);
      if (p.final_codes) p.out[qi] = res == 1 ? ZG_HAS_PERMISSION : (res == 2 ? ZG_ITEM_ERROR : ZG_NO_PERMISSION);
      else p.out[qi] = res == 1 ? kValT : (res == 2 ? kValE : 0);
    }
    __syncwarp();
  }
  if (COUNT) {
    unsigned long long b = c.bytes;
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) b += __shfl_xor_sync(kFull, b, d);
    if (lane == 0 && b) atomicAdd(p.alg_bytes, b);
  }
#if ZG_PHASE_CLOCKS
  if (lane == 0)
    for (int i = 0; i < kPhases; ++i) atomicAdd(p.events + 3 + i, static_cast<unsigned long long>(c.ph[i]));
#endif
}

// ---- flat checks: a slot whose checks are direct probes and two-level meets only (SF_FLAT) -----------------------
//
// One check per thread, no shared memory, no warp-collective traversal: the program's records are read from global
// memory (a few hundred bytes, L1-resident). A check is answered here only when every step takes the branch
// check_kernel<kMeetSet16> takes for it: a valid item without a subject relation, of an SF_FLAT slot, with room for the
// two-level meet (hop depth + 2 <= ZG_MAX_DEPTH), and whose subject is of each meet step's type and has a row in its
// closure index. Every other item is appended to the residual list (KParams::idx, count in nq_dev) that check_kernel
// answers next. The answer is the same as check_kernel's, and so is the COUNT variant's byte count: the probes in step
// order until one hits, then per meet step 8 bytes for the range's offsets, 8 for the subject's table header when the
// range is not empty, and sig_meet's rounds (sig_round, table_round) until one finds the check.
#ifndef ZG_FLAT_MIN_BLOCKS
#define ZG_FLAT_MIN_BLOCKS 3
#endif
constexpr int kFlatThreads = 256;
// 3 CTAs (24 warps) per SM, 80 registers: a range record and eight children's signature words in flight per thread,
// no spills. Measured on cfg3 (H100 80GB HBM3, 700 W, DESIGN.md §6): 1.06x faster than 4 CTAs at 64 registers, which
// spill one word. Before the records, 4 CTAs at 64 registers were 1.19x faster than 6 at 40 and 1.35x than 8 at 32.
constexpr int kFlatMinBlocks = ZG_FLAT_MIN_BLOCKS;

// A program record read through the read-only cache (records of 8-byte multiples, 8-byte aligned in the blob).
template <class T>
__device__ __forceinline__ T ldg_rec(const T* r) {
  static_assert(sizeof(T) % 8 == 0, "8-byte words");
  union {
    unsigned long long w[sizeof(T) / 8];
    T t;
  } u;
#pragma unroll
  for (unsigned i = 0; i < sizeof(T) / 8; ++i) u.w[i] = __ldg(reinterpret_cast<const unsigned long long*>(r) + i);
  return u.t;
}

// The two-level meet of a range held inline in its record r (n <= kRecSlots - 1 children, slot j + 1 = child j): every
// child tested against the subject's signature, kSigTests at a time from L1, then the "maybe"s confirmed in the set
// table, kSigTests lookups in flight together. One dependent round trip (the buckets) after the record, where sig_meet's
// rounds take two per kSigTests children. The COUNT variant confirms every "maybe" and counts what those rounds read: 12
// bytes per child and 8 per "maybe", in rounds of kSigTests up to and including the first that holds a member.
template <bool COUNT>
__device__ __forceinline__ bool record_meet(const uint16_t* __restrict__ rs, const uint32_t (&r)[kRecSlots / 2], uint32_t n,
                                            const unsigned long long* __restrict__ sig, uint32_t lg,
                                            const unsigned long long* __restrict__ tab, uint32_t nbk, uint32_t seed,
                                            unsigned long long& nb) {
  unsigned maybe = 0;  // bit j: child j
#pragma unroll
  for (uint32_t c0 = 0; c0 < kRecSlots - 1; c0 += kSigTests) {
    if (c0 >= n) break;
    uint32_t v[kSigTests];
    unsigned long long w[kSigTests];
#pragma unroll
    for (uint32_t i = 0; i < kSigTests; ++i) {
      const uint32_t k = c0 + i + 1;
      v[i] = k < kRecSlots ? (r[k >> 1] >> (16 * (k & 1))) & 0xFFFFu : 0u;
      w[i] = c0 + i < n ? __ldg(sig + sig_word(v[i], lg)) : 0ull;
    }
#pragma unroll
    for (uint32_t i = 0; i < kSigTests; ++i) {
      const unsigned long long b = sig_mask(v[i]);
      maybe |= (c0 + i < n && (w[i] & b) == b) ? 1u << (c0 + i) : 0u;
    }
  }
  // The "maybe"s are read again from the record (an L1 hit: it was just loaded) rather than picked out of r, which would
  // keep r live and spill. A child is never 0xFFFF: it marks the unused lookups of a batch, whose bucket word 0 is empty.
  unsigned found = 0, todo = maybe;  // found: the confirmed children (COUNT), or 1 once one is
  while (todo && (COUNT || !found)) {
    uint32_t v[kSigTests], at[kSigTests];
#pragma unroll
    for (uint32_t t = 0; t < kSigTests; ++t) {
      const uint32_t a = todo ? __ffs(todo) - 1 : 32u;
      if (COUNT) at[t] = a;
      todo &= todo - 1;
      v[t] = a < 32 ? __ldg(rs + a + 1) : 0xFFFFu;
    }
    unsigned long long w[kSigTests];
#pragma unroll
    for (uint32_t t = 0; t < kSigTests; ++t) w[t] = v[t] != 0xFFFFu ? __ldg(tab + table_bucket(v[t], seed, nbk)) : 0ull;
#pragma unroll
    for (uint32_t t = 0; t < kSigTests; ++t) found |= table_has(w[t], v[t]) ? (COUNT ? 1u << at[t] : 1u) : 0u;
  }
  if (COUNT)
    for (uint32_t c0 = 0; c0 < n; c0 += kSigTests) {
      const uint32_t m = min(n - c0, kSigTests);
      const unsigned rm = ((1u << m) - 1u) << c0;
      nb += 12ull * m + 8ull * __popc(maybe & rm);
      if (found & rm) break;
    }
  return found != 0;
}

template <bool COUNT>
// (the COUNT variant is an instrument: it takes the registers it needs instead of the occupancy)
__global__ void __launch_bounds__(kFlatThreads, COUNT ? 1 : kFlatMinBlocks) flat_check_kernel(const KParams p) {
  const DHeader* const h = reinterpret_cast<const DHeader*>(p.prog);
  const DStep* const steps = reinterpret_cast<const DStep*>(p.prog + __ldg(&h->off_steps));
  const unsigned long long q = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  const unsigned lane = threadIdx.x & 31;
  const bool valid = q < p.nq;
  uint4 it = make_uint4(0, 0, 0, 0);
  if (valid) it = __ldg(reinterpret_cast<const uint4*>(p.queries) + q);
  const uint32_t obj = it.x, sid = it.y, perm = it.z & 0xFFFFu, stype = it.z >> 16;
  const uint32_t depth = p.raw_items ? 0u : (it.w >> 16) & kJobDepthMask;
  bool flat = valid && (it.w & 0xFFFFu) == kNone && perm < __ldg(&h->n_slots) && depth + 2 <= ZG_MAX_DEPTH;
  DUnit u{};
  if (flat) {
    const DSlot s = ldg_rec(reinterpret_cast<const DSlot*>(p.prog + __ldg(&h->off_slots)) + perm);
    flat = (s.flags & SF_FLAT) != 0;
    if (flat) u = ldg_rec(reinterpret_cast<const DUnit*>(p.prog + __ldg(&h->off_units)) + s.unit);
  }
  // the closure index of a meet step (by value from the parameters: their address costs a local copy)
  auto closure_of = [&](uint32_t tgc, uint32_t& nsubj, const unsigned long long*& hdr, const unsigned long long*& sig,
                        uint32_t& sig_words, const unsigned long long*& tab) {
#pragma unroll
    for (int k = 0; k < kMaxClosure; ++k)
      if (k < static_cast<int>(p.n_closure) && p.closure[k].tgc == tgc) {
        nsubj = p.closure[k].nsubj;
        hdr = p.closure[k].set_hdr;
        sig = p.closure[k].sig;
        sig_words = p.closure[k].sig_words;
        tab = p.closure[k].set_tab;
      }
  };
  for (int i = u.push_begin; flat && i < u.step_end; ++i) {
    const DStep st = ldg_rec(steps + i);
    uint32_t nsubj = 0, words = 0;
    const unsigned long long *hdr = nullptr, *sig = nullptr, *tab = nullptr;
    closure_of(st.tgc, nsubj, hdr, sig, words, tab);
    flat = stype == st.tstype && sid < nsubj && hdr && sig;
  }
  // The residual pass's batch and sub-query counters, which it reads only after this grid has finished
  // (cudaGridDependencySynchronize): cleared here instead of by a memset of their own.
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    *p.next = 0;
    *p.subq_count = 0;
  }
  // the rest goes to check_kernel: one atomic per warp
  const bool residual = valid && !flat;
  const unsigned rm = __ballot_sync(kFull, residual);
  if (rm) {
    const int leader = __ffs(rm) - 1;
    unsigned long long at = 0;
    if (static_cast<int>(lane) == leader) {
      at = atomicAdd(p.nq_dev, static_cast<unsigned long long>(__popc(rm)));
      atomicAdd(p.nq_dev + 1, static_cast<unsigned long long>(__popc(rm)));
    }
    at = __shfl_sync(kFull, at, leader);
    if (residual) p.idx[at + __popc(rm & ((1u << lane) - 1u))] = static_cast<uint32_t>(q);
  }
  WarpCtx<COUNT> c;  // (probe_step's byte count)
  c.bytes = 0;
  if (flat) {
    if (COUNT) c.bytes += 17;
    bool hit = false;
    // direct and wildcard probes, in step order (visit's non-inverted branch: an SF_FLAT slot has no CF_INVERT probe)
    for (int i = u.step_begin; i < u.push_begin && !hit; ++i) {
      const DStep st = ldg_rec(steps + i);
      if (stype != st.stype || (st.kind == ST_WILD && p.no_wildcards)) continue;
      hit = probe_step(p, c, st, obj, sid, (st.flags & CF_EXPIRY) != 0);
    }
    // two-level meets: the range's record (or its offsets), the subject's table header and signature line are loaded
    // together
    for (int i = u.push_begin; !hit && i < u.step_end; ++i) {
      const DStep st = ldg_rec(steps + i);
      if (obj >= st.nres) continue;
      uint32_t nsubj = 0, words = 0;
      const unsigned long long *hdr = nullptr, *sig = nullptr, *tab = nullptr;
      closure_of(st.tgc, nsubj, hdr, sig, words, tab);
      const uint4* rec = nullptr;
#pragma unroll
      for (int k = 0; k < kMaxFlatRecords; ++k)
        if (k < static_cast<int>(p.n_rec) && p.rec[k].gc == st.gc && obj < p.rec[k].nres) rec = p.rec[k].rec;
      uint32_t r[kRecSlots / 2];  // the record's slots, two per word
      if (rec)
#pragma unroll
        for (uint32_t k = 0; k < kRecVecs; ++k) {
          const uint4 x = __ldg(rec + static_cast<unsigned long long>(obj) * kRecVecs + k);
          r[4 * k] = x.x;
          r[4 * k + 1] = x.y;
          r[4 * k + 2] = x.z;
          r[4 * k + 3] = x.w;
        }
      const unsigned long long hw = __ldg(hdr + sid);
      const uint32_t lg = __ffs(words) - 1;
      sig += static_cast<unsigned long long>(sid) << lg;
#ifndef ZG_EMULATE
      asm volatile("prefetch.global.L1 [%0];" ::"l"(sig));
#endif
      if (COUNT) c.bytes += 8;
      const uint32_t nbk = static_cast<uint32_t>(hw >> 32) & 0xFFFFFFu, seed = static_cast<uint32_t>(hw >> 56);
      tab += static_cast<uint32_t>(hw);
      const uint32_t n = rec ? r[0] & 0xFFFFu : kRecLong;
      if (n != kRecLong) {
        if (n == 0) continue;
        if (COUNT) c.bytes += 8;
        if (nbk)
          hit = record_meet<COUNT>(reinterpret_cast<const uint16_t*>(rec + static_cast<unsigned long long>(obj) * kRecVecs),
                                   r, n, sig, lg, tab, nbk, seed, c.bytes);
      } else {  // no record, or a range too long for one: its offsets, then sig_meet's rounds
        const unsigned long long ridx = st.row_base + static_cast<unsigned long long>(obj) * st.ncls;
        uint32_t lo = __ldg(p.row_ptr + ridx);
        const uint32_t hi = __ldg(p.row_ptr + ridx + 1);
        if (hi <= lo) continue;
        if (COUNT) c.bytes += 8;
        while (nbk && lo < hi && !hit) {  // sig_meet's rounds, whose early exit the byte model follows
          uint32_t v[kSigTests];
          const uint32_t m = min(hi - lo, kSigTests);
          const unsigned mb = sig_round<COUNT>(p.col, lo, m, sig, lg, v, c.bytes);
          lo += m;
          hit = table_round<COUNT>(tab, nbk, seed, mb, v, c.bytes);
        }
      }
      // check_kernel still reads (and counts) the offsets and header of the steps after the one that finds the check
      if (COUNT && hit)
        for (int j = i + 1; j < u.step_end; ++j) {
          const DStep sj = ldg_rec(steps + j);
          if (obj >= sj.nres) continue;
          const unsigned long long rj = sj.row_base + static_cast<unsigned long long>(obj) * sj.ncls;
          c.bytes += __ldg(p.row_ptr + rj + 1) > __ldg(p.row_ptr + rj) ? 16 : 8;
        }
    }
    if (p.out) p.out[q] = p.final_codes ? (hit ? ZG_HAS_PERMISSION : ZG_NO_PERMISSION) : (hit ? kValT : 0);
    if (p.val) p.val[q * p.L] = hit ? kValT : 0;
  }
  if (COUNT) {
    unsigned long long b = c.bytes;
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) b += __shfl_xor_sync(kFull, b, d);
    if (lane == 0 && b) atomicAdd(p.alg_bytes, b);
  }
}

// ---- multi-pass runs: the boolean fold of a level whose queries raised sub-queries -------------

// Evaluates each query's boolean tree over its leaf values val[q * L + l] (the check kernel wrote
// them, the folds of deeper levels OR-ed the sub-query results in). out != null: write the v1 code
// (or the raw value bits) to out[q]; otherwise OR the value into the (query, leaf) of the previous
// level that raised this query.
__global__ void fold_kernel(const uint8_t* prog, const zg_check* queries, unsigned long long n, uint32_t L,
                            const uint8_t* val, uint8_t* out, const uint32_t* parent, uint8_t* parent_val, int raw_out) {
  const Prog pr = make_prog(prog);
  unsigned long long q = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  if (q >= n) return;
  const zg_check it = queries[q];
  uint32_t r = 2;  // invalid query -> error
  const bool ok = it.perm < pr.hdr()->n_slots && it.stype < pr.hdr()->n_types &&
                  (it.srel == kNone || (it.srel < pr.hdr()->n_slots && pr.slots()[it.srel].type == it.stype));
  if (ok) {
    const DSlot s = pr.slots()[it.perm];
    auto leafval = [&](uint32_t l) -> unsigned long long {
      const uint8_t v = val[q * L + l];
      return (v & kValT) ? 1ull : ((v & kValE) ? 2ull : 0ull);
    };
    if (s.kind != SK_NONPURE) {
      r = static_cast<uint32_t>(leafval(0));
    } else {
      const DTree t = pr.trees()[s.unit];
      unsigned long long vals = 0;
      for (uint32_t l = 0; l < t.n_leaves; ++l) vals |= leafval(l) << (2 * l);
      r = eval_tree(pr, t, vals, it.subj == it.res, it.srel);
    }
  }
  if (out) {
    if (raw_out) out[q] = r == 1 ? kValT : (r == 2 ? kValE : 0);  // value of a routed sub-query
    else out[q] = r == 1 ? ZG_HAS_PERMISSION : (r == 2 ? ZG_ITEM_ERROR : ZG_NO_PERMISSION);
  } else if (r) {
    const uint32_t pj = parent[q];
    const uint32_t bits = r == 1 ? kValT : kValE;
    atomicOr(reinterpret_cast<unsigned int*>(parent_val + (pj & ~3u)), bits << (8 * (pj & 3u)));
  }
}

// ---- sharded store: device-side routing of checks / raised sub-queries to their owners ---------------
//
// owner(item) = item.res % n_dest. Two passes of a counting sort: per-destination counts (shared-memory
// histogram, one atomic per block and destination), then a scatter that writes every item behind its
// destination's cursor together with its source index, so that the values coming back in ROUTED order can be
// folded into the (query, leaf) that raised them without un-permuting anything. The owner is a functor: the
// sharded LookupResources routes its answer keys home with the same two kernels (KeyHomeOwner below).
constexpr int kMaxRouteDest = 64;
struct ResOwner {
  __device__ __forceinline__ uint32_t operator()(const zg_check& it, uint32_t n_dest) const { return it.res % n_dest; }
};
template <class Item = zg_check, class Owner = ResOwner>
__global__ void __launch_bounds__(256) route_count_kernel(const Item* items, unsigned long long n, uint32_t n_dest,
                                                          unsigned long long* counts, Owner owner = Owner{}) {
  ZG_BLOCK_SHARED_U32(hist, kMaxRouteDest);
  for (uint32_t i = threadIdx.x; i < n_dest; i += blockDim.x) hist[i] = 0;
  __syncthreads();
  const unsigned long long stride = static_cast<unsigned long long>(gridDim.x) * blockDim.x;
  for (unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; i < n; i += stride)
    atomicAdd(&hist[owner(items[i], n_dest)], 1u);
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < n_dest; i += blockDim.x)
    if (hist[i]) atomicAdd(counts + i, static_cast<unsigned long long>(hist[i]));
}
// kSrc = false: nothing is folded back in routed order, src is not written (and may be null)
template <class Item = zg_check, class Owner = ResOwner, bool kSrc = true>
__global__ void __launch_bounds__(256) route_scatter_kernel(const Item* items, unsigned long long n, uint32_t n_dest,
                                                            unsigned long long* cursor, Item* routed, uint32_t* src,
                                                            Owner owner = Owner{}) {
  const unsigned long long stride = static_cast<unsigned long long>(gridDim.x) * blockDim.x;
  for (unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; i < n; i += stride) {
    const Item it = items[i];
    const unsigned long long at = atomicAdd(cursor + owner(it, n_dest), 1ull);
    routed[at] = it;
    if constexpr (kSrc) src[at] = static_cast<uint32_t>(i);
  }
}
// values of routed sub-queries (routed order) OR-ed into the (query, leaf) that raised sub-query src[i]
__global__ void or_children_src_kernel(const uint32_t* parent, const uint32_t* src, const uint8_t* child_val, unsigned long long n,
                                       uint8_t* parent_val) {
  unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const uint32_t bits = child_val[i] & (kValT | kValE);
  if (!bits) return;
  const uint32_t pj = parent[src[i]];
  atomicOr(reinterpret_cast<unsigned int*>(parent_val + (pj & ~3u)), bits << (8 * (pj & 3u)));
}
// out[src[i]] = val[i]: answers that came back in routed order, restored to the caller's order
__global__ void unroute_kernel(const uint32_t* src, const uint8_t* val, unsigned long long n, uint8_t* out) {
  unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  if (i < n) out[src[i]] = val[i];
}

// ---- sharded handle: the exchange through peer memory (device.h PeerTable, capi.cu run_sharded / run_sharded_lookup) --
//
// One process holds every shard, so a routed query is written straight into its owner's inbox, behind the part of
// every lower shard (t.base[d], from all shards' counts), and a value is read where its owner left it: no copy
// call, no staging, no reverse exchange. The table of the destinations' buffers (t.p[d]) is a kernel argument.

// The count and the scatter are written once over the item type and its owner: the check protocol's sub-queries
// (zg_check, ResOwner) here, LookupSubjects' walk entries (8 bytes, EntryOwner) in peer_entry_*_kernel below.
// route_count_kernel over the items a step wrote, their number read on the device (*n_dev, at most cap): the counts
// come back with the step's control words in the level's one round trip
template <class Item, class Owner>
__device__ __forceinline__ void peer_count_items(const Item* items, const unsigned long long* n_dev, unsigned long long cap,
                                                 uint32_t n_dest, unsigned long long* counts, Owner owner) {
  ZG_BLOCK_SHARED_U32(hist, kMaxRouteDest);
  for (uint32_t i = threadIdx.x; i < n_dest; i += blockDim.x) hist[i] = 0;
  __syncthreads();
  const unsigned long long n = min(*n_dev, cap);
  const unsigned long long stride = static_cast<unsigned long long>(gridDim.x) * blockDim.x;
  for (unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; i < n; i += stride)
    atomicAdd(&hist[owner(items[i], n_dest)], 1u);
  __syncthreads();
  for (uint32_t i = threadIdx.x; i < n_dest; i += blockDim.x)
    if (hist[i]) atomicAdd(counts + i, static_cast<unsigned long long>(hist[i]));
}
// route_scatter_kernel into the owners' inboxes: item i goes to t.p[d][t.base[d] + cursor[d]++] (d = its owner), and,
// with kPos, pos[i] = its index there, where the owner leaves its value
template <class Item, class Owner, bool kPos, class Table>
__device__ __forceinline__ void peer_scatter_items(const Item* items, unsigned long long n, uint32_t n_dest,
                                                   unsigned long long* cursor, const Table& t, uint32_t* pos, Owner owner) {
  const unsigned long long stride = static_cast<unsigned long long>(gridDim.x) * blockDim.x;
  for (unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; i < n; i += stride) {
    const Item it = items[i];
    const uint32_t d = owner(it, n_dest);
    const unsigned long long at = t.base[d] + atomicAdd(cursor + d, 1ull);
    static_cast<Item*>(t.p[d])[at] = it;
    if constexpr (kPos) pos[i] = static_cast<uint32_t>(at);
  }
}
// the sub-queries a pass raised, counted by owner
__global__ void __launch_bounds__(256) peer_count_kernel(const zg_check* items, const unsigned long long* n_dev,
                                                         unsigned long long cap, uint32_t n_dest, unsigned long long* counts) {
  peer_count_items(items, n_dev, cap, n_dest, counts, ResOwner{});
}
// ... and written into their owners' inboxes, with where each went (pos)
template <class Table>
__global__ void __launch_bounds__(256) peer_scatter_kernel(const zg_check* items, unsigned long long n, uint32_t n_dest,
                                                           unsigned long long* cursor, const Table t, uint32_t* pos) {
  peer_scatter_items<zg_check, ResOwner, true>(items, n, n_dest, cursor, t, pos, ResOwner{});
}
// or_children_src_kernel reading each child's value from its owner (t.p[d] = shard d's values of the next level)
template <class Table>
__global__ void peer_or_children_kernel(const zg_check* raised, const uint32_t* parent, const uint32_t* pos, unsigned long long n,
                                        uint32_t n_dest, const Table t, uint8_t* parent_val) {
  unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const uint32_t d = raised[i].res % n_dest;
  const uint32_t bits = static_cast<const uint8_t*>(t.p[d])[pos[i]] & (kValT | kValE);
  if (!bits) return;
  const uint32_t pj = parent[i];
  atomicOr(reinterpret_cast<unsigned int*>(parent_val + (pj & ~3u)), bits << (8 * (pj & 3u)));
}
// the callers' answers in their own order: out[i] = the level-0 code its owner computed (t.p[d] = shard d's codes)
template <class Table>
__global__ void peer_gather_kernel(const zg_check* items, const uint32_t* pos, unsigned long long n, uint32_t n_dest,
                                   const Table t, uint8_t* out) {
  unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  if (i < n) out[i] = static_cast<const uint8_t*>(t.p[items[i].res % n_dest])[pos[i]];
}
// LookupResources on the handle: a source shard's n 8-byte entries written to t.p[d] + t.base[d] for every d < n_dest,
// behind the parts of the lower shards. Every shard's new frontier entries to every shard (n_dest = S, the all-gather
// of a level), and every shard's answer keys to shard 0 (n_dest = 1).
template <class Table>
__global__ void __launch_bounds__(256) peer_put_kernel(const unsigned long long* src, unsigned long long n, uint32_t n_dest,
                                                       const Table t) {
  const unsigned long long stride = static_cast<unsigned long long>(gridDim.x) * blockDim.x;
  for (unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; i < n; i += stride) {
    const unsigned long long v = src[i];
    for (uint32_t d = 0; d < n_dest; ++d) static_cast<unsigned long long*>(t.p[d])[t.base[d] + i] = v;
  }
}

// ---- LookupResources: candidate generation by reverse BFS ----------------------------
//
// Every true result r of LookupResources(T, P, S) has a forward path r -> o1 -> ... -> ok
// where each o(i+1) is the subject object of a relationship on o(i) and S is a direct (or
// wildcard) subject on ok. Walking the reverse CSR from S therefore reaches a SUPERSET of
// the results (relation names, expiry and & / - are ignored here); the check kernel then
// verifies every candidate of type T, so the answer is exact for any schema.

struct RbfsParams {
  const uint32_t* rrow_ptr;
  const uint32_t* rcol;
  const uint8_t* prog;
  const unsigned long long* frontier;  // (type << 32 | object)
  unsigned long long n_in;
  unsigned long long* next;            // output frontier
  unsigned long long* next_count;
  unsigned long long next_cap;
  uint32_t* visited;                   // bitmap over all objects, bit = type_bit_base[type] + object
  const unsigned long long* type_bit_base;
  uint32_t want_type;                  // candidates of this type go to cand[]
  uint32_t* cand;
  unsigned long long* cand_count;
  unsigned long long cand_cap;
  uint32_t* flags;                     // bit 4: frontier / candidate overflow
  int wildcard_level;                  // level 0: also take the wildcard classes of the subject's type
};

// One warp per frontier object: for every class whose subjects have the object's type,
// read its reverse row (coalesced) and mark the resources.
__global__ void __launch_bounds__(256) rbfs_expand_kernel(const RbfsParams p) {
  const Prog pr = make_prog(p.prog);
  const unsigned lane = threadIdx.x & 31;
  const unsigned long long w = (blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x) >> 5;
  if (w >= p.n_in) return;
  const unsigned long long item = p.frontier[w];
  const uint32_t type = static_cast<uint32_t>(item >> 32), obj = static_cast<uint32_t>(item);
  const DTypeInv tc = pr.type_rcls()[type];
  for (int ci = tc.begin; ci < tc.end; ++ci) {
    const DCls cl = pr.cls()[pr.rcls()[ci]];
    if (cl.flags & CF_EMPTY) continue;
    uint32_t row = obj;
    if (cl.sslot == kWildcard) {
      if (!p.wildcard_level) continue;  // type:* only matches the original, relation-less subject
      row = 0;
    } else if (obj >= cl.nsubj) {
      continue;
    }
    const unsigned long long ri = cl.rrow_base + static_cast<unsigned long long>(row) * cl.rstride;
    const uint32_t b = __ldg(p.rrow_ptr + ri), e = __ldg(p.rrow_ptr + ri + 1);
    const unsigned long long bit_base = p.type_bit_base[cl.rtype];
    for (uint32_t i0 = b; i0 < e; i0 += 32) {
      const uint32_t i = i0 + lane;
      bool fresh = false;
      uint32_t r = 0;
      if (i < e) {
        r = __ldg(p.rcol + i);
        const unsigned long long bit = bit_base + r;
        const uint32_t mask = 1u << (bit & 31);
        fresh = !(atomicOr(p.visited + (bit >> 5), mask) & mask);
      }
      const unsigned fm = __ballot_sync(kFull, fresh);
      if (fm) {
        unsigned long long at = 0;
        if (lane == 0) at = atomicAdd(p.next_count, static_cast<unsigned long long>(__popc(fm)));
        at = __shfl_sync(kFull, at, 0) + __popc(fm & ((1u << lane) - 1u));
        if (fresh) {
          if (at < p.next_cap) p.next[at] = (static_cast<unsigned long long>(cl.rtype) << 32) | r;
          else atomicOr(p.flags, 16u);
        }
      }
      const bool is_cand = fresh && cl.rtype == p.want_type;
      const unsigned cm = __ballot_sync(kFull, is_cand);
      if (cm) {
        unsigned long long at = 0;
        if (lane == 0) at = atomicAdd(p.cand_count, static_cast<unsigned long long>(__popc(cm)));
        at = __shfl_sync(kFull, at, 0) + __popc(cm & ((1u << lane) - 1u));
        if (is_cand) {
          if (at < p.cand_cap) p.cand[at] = r;
          else atomicOr(p.flags, 16u);
        }
      }
    }
  }
}

// ---- batched LookupResources: K reverse walks in one frontier ---------------------------------
//
// The proxy runs one LookupResources per list request, concurrently (pkg/authz/responsefilterer.go:165,
// lookups.go:49-65). K of them share every launch: frontier entries carry the lookup they belong to,
// each lookup has its own visited bitmap slice, candidates are emitted directly as check items (the
// lookup's subject and permission filled in) with their owner beside them, and the level loop needs no
// host round trip: every level kernel reads its input count from device memory and an empty level is a
// no-op launch.
struct LookupParam {   // one per lookup of the batch
  uint32_t subj;
  uint16_t want_type, perm, stype, srel;
};
constexpr int kMaxLookupBatch = 64;
struct MrbfsParams {
  const uint32_t* rrow_ptr;
  const uint32_t* rcol;
  const uint8_t* prog;
  const LookupParam* lk;
  const unsigned long long* in;       // lookup << 48 | type << 32 | object
  unsigned long long* out;
  unsigned long long* counts;         // counts[level] = entries of `in`, counts[level + 1] = entries of `out`
  int level;
  unsigned long long cap;             // frontier capacity
  uint32_t* visited;                  // K slices of `words` u32
  unsigned long long words;
  const unsigned long long* type_bit_base;
  zg_check* cand;                     // candidate checks
  uint8_t* cand_owner;
  unsigned long long* cand_count;
  unsigned long long cand_cap;
  uint32_t* flags;                    // bit 4: frontier / candidate overflow
};

__global__ void __launch_bounds__(256) mrbfs_expand_kernel(const MrbfsParams p) {
  const unsigned long long n_in = p.counts[p.level];
  if (n_in == 0 || n_in > p.cap) return;
  const Prog pr = make_prog(p.prog);
  const unsigned lane = threadIdx.x & 31;
  const unsigned long long n_warps = (static_cast<unsigned long long>(gridDim.x) * blockDim.x) >> 5;
  for (unsigned long long w = (blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x) >> 5; w < n_in;
       w += n_warps) {
    const unsigned long long item = p.in[w];
    const uint32_t k = static_cast<uint32_t>(item >> 48), type = static_cast<uint32_t>(item >> 32) & 0xFFFFu,
                   obj = static_cast<uint32_t>(item);
    const LookupParam lk = p.lk[k];
    uint32_t* const vis = p.visited + k * p.words;
    const DTypeInv tc = pr.type_rcls()[type];
    for (int ci = tc.begin; ci < tc.end; ++ci) {
      const DCls cl = pr.cls()[pr.rcls()[ci]];
      if (cl.flags & CF_EMPTY) continue;
      uint32_t row = obj;
      if (cl.sslot == kWildcard) {
        if (p.level != 0 || lk.srel != kNone) continue;  // type:* only matches the original, relation-less subject
        row = 0;
      } else if (obj >= cl.nsubj) {
        continue;
      }
      const unsigned long long ri = cl.rrow_base + static_cast<unsigned long long>(row) * cl.rstride;
      const uint32_t b = __ldg(p.rrow_ptr + ri), e = __ldg(p.rrow_ptr + ri + 1);
      const unsigned long long bit_base = p.type_bit_base[cl.rtype];
      for (uint32_t i0 = b; i0 < e; i0 += 32) {
        const uint32_t i = i0 + lane;
        bool fresh = false;
        uint32_t r = 0;
        if (i < e) {
          r = __ldg(p.rcol + i);
          const unsigned long long bit = bit_base + r;
          const uint32_t mask = 1u << (bit & 31);
          fresh = !(atomicOr(vis + (bit >> 5), mask) & mask);
        }
        const unsigned fm = __ballot_sync(kFull, fresh);
        if (fm) {
          unsigned long long at = 0;
          if (lane == 0) at = atomicAdd(p.counts + p.level + 1, static_cast<unsigned long long>(__popc(fm)));
          at = __shfl_sync(kFull, at, 0) + __popc(fm & ((1u << lane) - 1u));
          if (fresh) {
            if (at < p.cap) p.out[at] = (static_cast<unsigned long long>(k) << 48) | (static_cast<unsigned long long>(cl.rtype) << 32) | r;
            else atomicOr(p.flags, 16u);
          }
        }
        const bool is_cand = fresh && cl.rtype == lk.want_type;
        const unsigned cm = __ballot_sync(kFull, is_cand);
        if (cm) {
          unsigned long long at = 0;
          if (lane == 0) at = atomicAdd(p.cand_count, static_cast<unsigned long long>(__popc(cm)));
          at = __shfl_sync(kFull, at, 0) + __popc(cm & ((1u << lane) - 1u));
          if (is_cand) {
            if (at < p.cand_cap) {
              zg_check q;
              q.res = r;
              q.subj = lk.subj;
              q.perm = lk.perm;
              q.stype = lk.stype;
              q.srel = lk.srel;
              q.flags = 0;
              p.cand[at] = q;
              p.cand_owner[at] = static_cast<uint8_t>(k);
            } else {
              atomicOr(p.flags, 16u);
            }
          }
        }
      }
    }
  }
}

// HAS candidates -> keys (owner << 32 | resource id), compacted; per-lookup result counts; lookups with an
// undecidable candidate (ITEM_ERROR) are flagged in err_mask. err_below: ITEM_ERROR candidates i < err_below become
// keys too, with bit kErrKeyBit set, so that the flag travels with the answers (sharded LookupResources sends them
// home; its self-membership candidates come after the walk's and, as on a replica, are left out when undecidable).
constexpr int kErrKeyBit = 38;  // just above the lookup index (< kMaxLookupBatch = 2^6) in the high word
__global__ void lookup_keys_kernel(const zg_check* cand, const uint8_t* owner, const uint8_t* codes, unsigned long long n,
                                   unsigned long long* keys, unsigned long long* n_keys, unsigned long long* per_lookup,
                                   unsigned long long* err_mask, unsigned long long err_below = 0) {
  unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  const bool in = i < n;
  const uint8_t code = in ? codes[i] : 0;
  const bool has = code == ZG_HAS_PERMISSION;
  const bool bad = in && code == ZG_ITEM_ERROR;
  if (bad) atomicOr(err_mask, 1ull << owner[i]);
  const bool emit = has || (bad && i < err_below);
  const unsigned m = __ballot_sync(kFull, emit);
  if (!m) return;
  const unsigned lane = threadIdx.x & 31;
  unsigned long long base = 0;
  if (lane == 0) base = atomicAdd(n_keys, static_cast<unsigned long long>(__popc(m)));
  base = __shfl_sync(kFull, base, 0);
  if (emit) {
    keys[base + __popc(m & ((1u << lane) - 1u))] = (static_cast<unsigned long long>(bad) << kErrKeyBit) |
                                                   (static_cast<unsigned long long>(owner[i]) << 32) | cand[i].res;
    if (has) atomicAdd(per_lookup + owner[i], 1ull);
  }
}
__global__ void low_words_kernel(const unsigned long long* keys, unsigned long long n, uint32_t* out) {
  unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  if (i < n) out[i] = static_cast<uint32_t>(keys[i]);
}

// LookupResources when the permission is a flat union of direct relations (the reference's
// own schema: `permission view = viewer + creator`, pkg/spicedb/bootstrap.yaml:13): the answer
// is the union of the subject's reverse rows of those classes. One warp copies them out.
struct FlatLookupClass {
  unsigned long long rrow_base;
  uint32_t nsubj;
  uint16_t stype;     // subject type the class accepts
  uint16_t wildcard;  // row 0 regardless of the subject id
  uint32_t rstride;   // reverse row stride per subject
  uint32_t pad;
};
__global__ void lookup_flat_kernel(const uint32_t* rrow_ptr, const uint32_t* rcol, const FlatLookupClass* cls, int ncls,
                                   uint32_t stype, uint32_t subj, uint32_t* out, unsigned long long cap,
                                   unsigned long long* count) {
  const unsigned lane = threadIdx.x & 31;
  unsigned long long w = 0;
  for (int c = 0; c < ncls; ++c) {
    if (cls[c].stype != stype) continue;  // relationships with another subject type cannot match
    const uint32_t row = cls[c].wildcard ? 0u : subj;
    if (row >= cls[c].nsubj) continue;
    const unsigned long long ri = cls[c].rrow_base + static_cast<unsigned long long>(row) * cls[c].rstride;
    const uint32_t b = rrow_ptr[ri], e = rrow_ptr[ri + 1];
    for (uint32_t i = b + lane; i < e; i += 32)
      if (w + (i - b) < cap) out[w + (i - b)] = rcol[i];
    w += e - b;
  }
  if (lane == 0) *count = w;
}

// ---- LookupResources helpers ---------------------------------------------------------

__global__ void lookup_fill_kernel(const uint32_t* cand, unsigned long long n, zg_check proto, zg_check* jobs) {
  unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  proto.res = cand[i];
  jobs[i] = proto;
}

// ids of candidates whose code is HAS, compacted with ballot + popc; order is
// restored by the caller (results are a set: pkg/authz/lookups.go:129).
__global__ void lookup_compact_kernel(const uint32_t* cand, const uint8_t* codes, unsigned long long n, uint32_t* out,
                                      unsigned long long cap, unsigned long long* count, uint32_t* flags) {
  unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  const bool has = i < n && codes[i] == ZG_HAS_PERMISSION;
  const bool bad = i < n && codes[i] == ZG_ITEM_ERROR;
  const unsigned m = __ballot_sync(kFull, has);
  if (__any_sync(kFull, bad) && (threadIdx.x & 31) == 0) atomicOr(flags, 8u);
  if (!m) return;
  unsigned long long base = 0;
  const unsigned lane = threadIdx.x & 31;
  if (lane == 0) base = atomicAdd(count, static_cast<unsigned long long>(__popc(m)));
  base = __shfl_sync(kFull, base, 0);
  if (has) {
    const unsigned long long at = base + __popc(m & ((1u << lane) - 1u));
    if (at < cap) out[at] = cand[i];
  }
}

// ---- pages of LookupResources (Device::lookup_page) -------------------------------------
//
// A page needs the answers in ascending id order after the cursor, up to the (limit + 1)-th one. The candidates after
// the cursor are selected and sorted once; then windows of the sorted candidates, from the front, are verified and
// scanned in order until limit + 1 answers are found or the candidates run out.

// Candidates with id > after (every candidate when !has_after) -> out (unordered), plus `self` (ZG_NO_OBJECT: none),
// the userset subject's own object, which the walk reaches only through stored edges. ctrl[0]: out's count; ctrl[1]
// = 1 when `self` is among the n candidates themselves (then its check failing fails the page, as it fails the
// unpaged call).
__global__ void lookup_select_kernel(const uint32_t* cand, unsigned long long n, uint32_t has_after, uint32_t after,
                                     uint32_t self, uint32_t* out, unsigned long long* ctrl) {
  const unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  const bool in = i < n + (self != ZG_NO_OBJECT ? 1 : 0);
  const uint32_t id = !in ? 0u : i < n ? cand[i] : self;
  if (in && i < n && id == self) ctrl[1] = 1;
  const bool keep = in && (!has_after || id > after);
  const unsigned m = __ballot_sync(kFull, keep);
  if (!m) return;
  const unsigned lane = threadIdx.x & 31;
  unsigned long long base = 0;
  if (lane == 0) base = atomicAdd(ctrl, static_cast<unsigned long long>(__popc(m)));
  base = __shfl_sync(kFull, base, 0);
  if (keep) out[base + __popc(m & ((1u << lane) - 1u))] = id;
}

// *at = the first index of ids[0, n) (ascending) whose id > after: the exhaustive list needs no selection.
__global__ void lookup_bound_kernel(const uint32_t* ids, unsigned long long n, uint32_t after, unsigned long long* at) {
  unsigned long long lo = 0, hi = n;
  while (lo < hi) {
    const unsigned long long mid = (lo + hi) / 2;
    if (ids[mid] <= after) lo = mid + 1;
    else hi = mid;
  }
  *at = lo;
}

// One window ids[0, n) of the sorted candidates, in id order, with their codes (nullptr: every candidate is an answer,
// the flat path). An id equal to its predecessor (ids[-1] too when has_prev) is a repeat and counts once. ctrl[0]
// holds the answers found by the earlier windows; the window's answers take ranks from there, and those of rank <
// want go to out[rank]. ctrl[1] = 1 when a candidate whose check ended in ZG_ITEM_ERROR lies at or before the answer
// of rank want - 1 (anywhere in the window when the window does not reach that rank): that answer decides the page,
// so an undecidable candidate before it fails the page. `quiet`: the self candidate when the walk did not reach it;
// like the unpaged call, its failed check leaves it out without failing. One block scans tile after tile and stops
// at the deciding answer.
constexpr unsigned kWindowThreads = 1024;
__global__ void __launch_bounds__(kWindowThreads) lookup_window_kernel(const uint32_t* ids, unsigned long long n,
                                                                      uint32_t has_prev, const uint8_t* codes,
                                                                      uint32_t quiet, unsigned long long want,
                                                                      uint32_t* out, unsigned long long* ctrl) {
  ZG_BLOCK_SHARED_U32(sh, 34);  // [0, 32) the warps' offsets in the tile, [32] the tile's answers, [33] the deciding thread
  const unsigned t = threadIdx.x, lane = t & 31, wid = t >> 5;
  unsigned long long found = ctrl[0];  // the same in every thread
  for (unsigned long long base = 0; base < n; base += kWindowThreads) {
    const unsigned long long i = base + t;
    bool has = false, bad = false;
    uint32_t id = 0;
    if (i < n) {
      id = ids[i];
      const bool dup = i > 0 ? ids[i - 1] == id : has_prev && ids[-1] == id;
      const uint8_t c = codes ? codes[i] : static_cast<uint8_t>(ZG_HAS_PERMISSION);
      has = !dup && c == ZG_HAS_PERMISSION;
      bad = !dup && c == ZG_ITEM_ERROR && id != quiet;
    }
    const unsigned m = __ballot_sync(kFull, has);
    if (lane == 0) sh[wid] = __popc(m);
    __syncthreads();
    if (wid == 0) {  // exclusive prefix of the warps' counts, the tile's total, no deciding thread yet
      const unsigned v = sh[lane];
      unsigned x = v;
      for (unsigned d = 1; d < 32; d <<= 1) {
        const unsigned y = __shfl_up_sync(kFull, x, d);
        if (lane >= d) x += y;
      }
      sh[lane] = x - v;
      if (lane == 31) {
        sh[32] = x;
        sh[33] = ~0u;
      }
    }
    __syncthreads();
    const unsigned long long rank = found + sh[wid] + __popc(m & ((1u << lane) - 1u));
    if (has && rank < want) out[rank] = id;
    if (has && rank == want - 1) sh[33] = t;
    __syncthreads();
    if (bad && t <= sh[33]) ctrl[1] = 1;
    found += sh[32];
    if (found >= want) break;  // uniform: the page is decided in this tile
  }
  if (t == 0) ctrl[0] = found < want ? found : want;
}

// ---- LookupResources on the object-hash sharded store (dist.DeviceShardedLookup) ------------------------------
//
// Shard k holds the reverse rows of the relationships whose resource it owns, so every object it discovers with
// mrbfs_expand_kernel is its own: each rank keeps its own visited slices, each object enters the replicated frontier
// once, and candidates start on their owner. The kernels below complete the candidates, send the verified ones
// home and split them per lookup there.

// Answer keys (lookup << 32 | id, kErrKeyBit for an undecidable candidate) go to the rank that asked the lookup.
struct KeyHomeOwner {
  const uint8_t* home;  // per lookup of the round
  __device__ __forceinline__ uint32_t operator()(unsigned long long key, uint32_t) const {
    return home[(key >> 32) & (kMaxLookupBatch - 1)];
  }
};

// A userset subject T:x#r of a lookup of type T whose object x this shard owns; bit: x's bit in the lookup's visited
// slice, ~0 when x is no object of this shard (the walk cannot have reached it).
struct SelfCand {
  uint32_t k, pad;
  unsigned long long bit;
};
// x becomes a candidate of its own lookup unless the walk (or the exhaustive fill) already made it one
__global__ void lookup_self_kernel(const LookupParam* lk, const SelfCand* self, uint32_t n_self, const uint32_t* visited,
                                   unsigned long long words, zg_check* cand, uint8_t* cand_owner, unsigned long long* cand_count) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_self) return;
  const SelfCand s = self[i];
  if (s.bit != ~0ull && ((visited[s.k * words + (s.bit >> 5)] >> (s.bit & 31)) & 1u)) return;
  const LookupParam l = lk[s.k];
  zg_check q;
  q.res = l.subj;
  q.subj = l.subj;
  q.perm = l.perm;
  q.stype = l.stype;
  q.srel = l.srel;
  q.flags = 0;
  const unsigned long long at = atomicAdd(cand_count, 1ull);
  cand[at] = q;
  cand_owner[at] = static_cast<uint8_t>(s.k);
}

// Exhaustive candidates of lookup k (its walk overflowed): every resource of its type this shard owns, marked in
// the lookup's visited slice (cleared by the caller) so that lookup_self_kernel does not add one of them twice.
__global__ void lookup_fill_owned_kernel(const uint32_t* res, unsigned long long n, LookupParam l, uint32_t k, uint32_t* vis,
                                         unsigned long long bit_base, zg_check* cand, uint8_t* cand_owner) {
  const unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const uint32_t r = res[i];
  zg_check q;
  q.res = r;
  q.subj = l.subj;
  q.perm = l.perm;
  q.stype = l.stype;
  q.srel = l.srel;
  q.flags = 0;
  cand[i] = q;
  cand_owner[i] = static_cast<uint8_t>(k);
  const unsigned long long bit = bit_base + r;
  atomicOr(vis + (bit >> 5), 1u << (bit & 31));
}

// Keys that arrived home, sorted: the answers in (lookup, id) order, then the error keys. ids[i] = id of answer i;
// lookup k's answers are ids[first[k] .. end[k]) (both left 0 for a lookup without answers); err_mask: lookups with
// an undecidable candidate.
__global__ void lookup_split_kernel(const unsigned long long* keys, unsigned long long n, uint32_t* ids,
                                    unsigned long long* first, unsigned long long* end, unsigned long long* err_mask) {
  const unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const unsigned long long key = keys[i];
  const uint32_t k = static_cast<uint32_t>(key >> 32) & (kMaxLookupBatch - 1);
  if ((key >> kErrKeyBit) & 1ull) {
    atomicOr(err_mask, 1ull << k);
    return;
  }
  ids[i] = static_cast<uint32_t>(key);
  const unsigned long long run = key >> 32;  // lookup and error bit: a run of answers ends at either change
  if (i == 0 || (keys[i - 1] >> 32) != run) first[k] = i;
  if (i + 1 == n || (keys[i + 1] >> 32) != run) end[k] = i + 1;
}

// ---- LookupSubjects: forward walk from the resource (the mirror of mrbfs_expand_kernel) -------------------
//
// Every subject s with Check(T:r#P @ ST:s[#SR]) = HAS is the subject of a relationship on some object the
// evaluation of P visits, or is one of those objects itself (userset self-membership). Walking the forward CSR
// from r over the edge classes P's evaluation can read (FwalkParams::mask, Schema::fwd_mask) therefore reaches a
// SUPERSET of the answer (expiry and & / - are ignored), and one check launch verifies it. Wildcard classes
// are not walked: they name no subject, the wildcard probe item covers them.
struct FwalkParams {
  const uint32_t* row_ptr;
  const uint32_t* col;
  const FwdClass* fwd;                 // fwd[type_off[t], type_off[t + 1]): edge classes of the relations of type t
  const uint32_t* type_off;
  const uint32_t* mask;                // bit gc: class gc is read by the permission's evaluation
  unsigned long long* in;              // type << 32 | object
  unsigned long long* out;
  unsigned long long* counts;          // counts[level] = entries of `in`, counts[level + 1] = entries of `out`
  int level;
  unsigned long long cap;              // frontier capacity
  uint32_t* visited;                   // bitmap over all objects, bit = type_bit_base[type] + object
  const unsigned long long* type_bit_base;
  zg_check proto;                      // res, perm, stype, srel of the lookup; subj is set per candidate
  zg_check* cand;
  unsigned long long* cand_count;
  unsigned long long cand_cap;
  uint32_t* flags;                     // bit 4: frontier / candidate overflow
};

// Level 0 of the walk and the two items every lookup verifies: [0] the wildcard probe (a never-written subject:
// it stands for every subject outside the candidates), [1] the resource itself when it has the subject type.
__global__ void fwalk_seed_kernel(const FwalkParams p, uint32_t res_type) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const unsigned long long bit = p.type_bit_base[res_type] + p.proto.res;
  p.visited[bit >> 5] |= 1u << (bit & 31);
  p.in[0] = (static_cast<unsigned long long>(res_type) << 32) | p.proto.res;
  p.counts[0] = 1;
  zg_check q = p.proto;
  q.subj = ZG_NO_OBJECT - 1;
  p.cand[0] = q;
  unsigned long long n = 1;
  if (res_type == p.proto.stype) {
    q.subj = p.proto.res;
    p.cand[n++] = q;
  }
  *p.cand_count = n;
}

// One warp per frontier object: for every masked class of the object's type, read its forward row (coalesced)
// and mark the subjects. Reads its input count from device memory: the level loop needs no host round trip.
__global__ void __launch_bounds__(256) fwalk_expand_kernel(const FwalkParams p) {
  const unsigned long long n_in = p.counts[p.level];
  if (n_in == 0 || n_in > p.cap) return;
  const unsigned lane = threadIdx.x & 31;
  const unsigned long long n_warps = (static_cast<unsigned long long>(gridDim.x) * blockDim.x) >> 5;
  for (unsigned long long w = (blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x) >> 5; w < n_in;
       w += n_warps) {
    const unsigned long long item = p.in[w];
    const uint32_t type = static_cast<uint32_t>(item >> 32), obj = static_cast<uint32_t>(item);
    for (uint32_t ci = p.type_off[type]; ci < p.type_off[type + 1]; ++ci) {
      const FwdClass fc = p.fwd[ci];
      if (!((p.mask[fc.gc >> 5] >> (fc.gc & 31)) & 1u) || obj >= fc.nres) continue;
      const unsigned long long ri = fc.row_base + static_cast<unsigned long long>(obj) * fc.ncls;
      const uint32_t b = __ldg(p.row_ptr + ri), e = __ldg(p.row_ptr + ri + 1);
      const unsigned long long bit_base = p.type_bit_base[fc.stype];
      for (uint32_t i0 = b; i0 < e; i0 += 32) {
        const uint32_t i = i0 + lane;
        bool fresh = false;
        uint32_t s = 0;
        if (i < e) {
          s = __ldg(p.col + i);
          const unsigned long long bit = bit_base + s;
          const uint32_t m = 1u << (bit & 31);
          fresh = !(atomicOr(p.visited + (bit >> 5), m) & m);
        }
        const unsigned fm = __ballot_sync(kFull, fresh);
        if (fm) {
          unsigned long long at = 0;
          if (lane == 0) at = atomicAdd(p.counts + p.level + 1, static_cast<unsigned long long>(__popc(fm)));
          at = __shfl_sync(kFull, at, 0) + __popc(fm & ((1u << lane) - 1u));
          if (fresh) {
            if (at < p.cap) p.out[at] = (static_cast<unsigned long long>(fc.stype) << 32) | s;
            else atomicOr(p.flags, 16u);
          }
        }
        const bool is_cand = fresh && fc.stype == p.proto.stype;
        const unsigned cm = __ballot_sync(kFull, is_cand);
        if (cm) {
          unsigned long long at = 0;
          if (lane == 0) at = atomicAdd(p.cand_count, static_cast<unsigned long long>(__popc(cm)));
          at = __shfl_sync(kFull, at, 0) + __popc(cm & ((1u << lane) - 1u));
          if (is_cand) {
            if (at < p.cand_cap) {
              zg_check q = p.proto;
              q.subj = s;
              p.cand[at] = q;
            } else {
              atomicOr(p.flags, 16u);
            }
          }
        }
      }
    }
  }
}

// Walk overflow (or ZGPU_NO_RBFS): every object of the subject type is a candidate, behind the probe item.
__global__ void ls_fill_kernel(zg_check proto, unsigned long long n, zg_check* jobs) {
  const unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  if (i > n) return;
  proto.subj = i == 0 ? ZG_NO_OBJECT - 1 : static_cast<uint32_t>(i - 1);
  jobs[i] = proto;
}

// Verified candidates [1, n) (item 0 is the probe): HAS subjects go to has_ids and has_items (the input of the
// no-wildcards pass), NO subjects to no_ids; an undecidable candidate sets flags bit 3. counts: [0] HAS, [1] NO.
__global__ void ls_split_kernel(const zg_check* items, const uint8_t* codes, unsigned long long n, uint32_t* has_ids,
                                zg_check* has_items, uint32_t* no_ids, unsigned long long* counts, uint32_t* flags) {
  const unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x + 1;
  const uint8_t code = i < n ? codes[i] : 0;
  const bool has = code == ZG_HAS_PERMISSION, no = code == ZG_NO_PERMISSION;
  const unsigned lane = threadIdx.x & 31;
  if (__any_sync(kFull, code == ZG_ITEM_ERROR) && lane == 0) atomicOr(flags, 8u);
  const unsigned hm = __ballot_sync(kFull, has), nm = __ballot_sync(kFull, no);
  unsigned long long hb = 0, nb = 0;
  if (lane == 0 && hm) hb = atomicAdd(counts, static_cast<unsigned long long>(__popc(hm)));
  if (lane == 0 && nm) nb = atomicAdd(counts + 1, static_cast<unsigned long long>(__popc(nm)));
  hb = __shfl_sync(kFull, hb, 0);
  nb = __shfl_sync(kFull, nb, 0);
  const unsigned below = (1u << lane) - 1u;
  if (has) {
    const unsigned long long at = hb + __popc(hm & below);
    has_ids[at] = items[i].subj;
    has_items[at] = items[i];
  } else if (no) {
    no_ids[nb + __popc(nm & below)] = items[i].subj;
  }
}

// ---- LookupSubjects on the object-hash sharded store (dist.DeviceShardedLookup.lookup_subjects) ---------------
//
// Shard k holds the forward rows of the objects it owns, but the subjects in those rows can be owned by any shard.
// So the walk routes what it discovers to the owner, and the owner deduplicates: every rank keeps a visited slice
// per lookup, in which the bit of an object it owns means "admitted" (it entered this rank's frontier once), and
// the bit of an object it does not own means "already sent for this lookup". An object enters the frontier of its
// owner at the first level any rank discovers it, which is the level a replica's fwalk_expand_kernel reaches it:
// the admitted objects, and so the candidates, are the replica's.
struct SubjectsParam {  // one per lookup of the round
  uint32_t res;
  uint16_t res_type, perm, stype, srel;
};
struct SsWalkParams {
  const uint32_t* row_ptr;
  const uint32_t* col;
  const FwdClass* fwd;                 // as FwalkParams
  const uint32_t* type_off;
  const uint32_t* mask;                // Schema::fwd_mask: mask_words words per permission slot
  uint32_t mask_words;
  uint32_t shard_rank, shard_count;
  const SubjectsParam* lk;
  const unsigned long long* in;        // lookup << 48 | type << 32 | object
  unsigned long long n_in;
  unsigned long long* out;             // expand: the outbox; admit: the next frontier
  unsigned long long* out_count;
  unsigned long long cap;              // entries of `out`
  uint32_t* visited;                   // K slices of `words` u32, bit = type_bit_base[type] + object
  unsigned long long words;
  const unsigned long long* type_bit_base;
  zg_check* cand;                      // admit: candidate checks of this rank
  uint8_t* cand_owner;
  unsigned long long* cand_count;
  unsigned long long cand_cap;
  uint32_t* flags;                     // bit 4: outbox / frontier / candidate overflow
};

// One warp per frontier object (all owned by this rank), the classes of its type that the lookup's permission
// reads, as fwalk_expand_kernel. A subject is put in the outbox unless this rank already admitted it (owned) or
// already sent it (not owned) for this lookup; the owner's admission decides whether it is new.
__global__ void __launch_bounds__(256) ss_expand_kernel(const SsWalkParams p) {
  const unsigned lane = threadIdx.x & 31;
  const unsigned long long n_warps = (static_cast<unsigned long long>(gridDim.x) * blockDim.x) >> 5;
  for (unsigned long long w = (blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x) >> 5; w < p.n_in;
       w += n_warps) {
    const unsigned long long item = p.in[w];
    const uint32_t k = static_cast<uint32_t>(item >> 48), type = static_cast<uint32_t>(item >> 32) & 0xFFFFu,
                   obj = static_cast<uint32_t>(item);
    const uint32_t* const mask = p.mask + static_cast<size_t>(p.lk[k].perm) * p.mask_words;
    uint32_t* const vis = p.visited + k * p.words;
    for (uint32_t ci = p.type_off[type]; ci < p.type_off[type + 1]; ++ci) {
      const FwdClass fc = p.fwd[ci];
      if (!((mask[fc.gc >> 5] >> (fc.gc & 31)) & 1u) || obj >= fc.nres) continue;
      const unsigned long long ri = fc.row_base + static_cast<unsigned long long>(obj) * fc.ncls;
      const uint32_t b = __ldg(p.row_ptr + ri), e = __ldg(p.row_ptr + ri + 1);
      const unsigned long long bit_base = p.type_bit_base[fc.stype];
      for (uint32_t i0 = b; i0 < e; i0 += 32) {
        const uint32_t i = i0 + lane;
        bool fresh = false;
        uint32_t s = 0;
        if (i < e) {
          s = __ldg(p.col + i);
          const unsigned long long bit = bit_base + s;
          const uint32_t m = 1u << (bit & 31);
          // owned bits are only set by ss_admit_kernel, never while this kernel runs
          fresh = s % p.shard_count == p.shard_rank ? !(vis[bit >> 5] & m) : !(atomicOr(vis + (bit >> 5), m) & m);
        }
        const unsigned fm = __ballot_sync(kFull, fresh);
        if (fm) {
          unsigned long long at = 0;
          if (lane == 0) at = atomicAdd(p.out_count, static_cast<unsigned long long>(__popc(fm)));
          at = __shfl_sync(kFull, at, 0) + __popc(fm & ((1u << lane) - 1u));
          if (fresh) {
            if (at < p.cap) p.out[at] = (item & (0xFFFFull << 48)) | (static_cast<unsigned long long>(fc.stype) << 32) | s;
            else atomicOr(p.flags, 16u);
          }
        }
      }
    }
  }
}

// Outbox entries are routed to the owner of their object
struct EntryOwner {
  __device__ __forceinline__ uint32_t operator()(unsigned long long entry, uint32_t n_dest) const {
    return static_cast<uint32_t>(entry) % n_dest;
  }
};

// LookupSubjects on the sharded handle (capi.cu run_sharded_subjects): a level's outbox (ss_expand_kernel's entries,
// their number read on the device) counted by owner, then written straight into the owners' inboxes behind the parts
// of the lower shards. Nothing comes back per entry, so no position is kept.
__global__ void __launch_bounds__(256) peer_entry_count_kernel(const unsigned long long* entries, const unsigned long long* n_dev,
                                                               unsigned long long cap, uint32_t n_dest, unsigned long long* counts) {
  peer_count_items(entries, n_dev, cap, n_dest, counts, EntryOwner{});
}
template <class Table>
__global__ void __launch_bounds__(256) peer_entry_scatter_kernel(const unsigned long long* entries, unsigned long long n,
                                                                 uint32_t n_dest, unsigned long long* cursor, const Table t) {
  peer_scatter_items<unsigned long long, EntryOwner, false>(entries, n, n_dest, cursor, t, nullptr, EntryOwner{});
}

// Admission at the owner, one thread per arrived entry: a test-and-set of the object's bit in the lookup's slice.
// A fresh entry joins the next frontier; a fresh object of the lookup's subject type is also a candidate
// {res, object, perm, stype, srel}. The round's level-0 seeds (each resource, on its owner) are admitted the same way.
__global__ void ss_admit_kernel(const SsWalkParams p) {
  const unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  const unsigned lane = threadIdx.x & 31;
  bool fresh = false, is_cand = false;
  unsigned long long item = 0;
  SubjectsParam l{};
  if (i < p.n_in) {
    item = p.in[i];
    const uint32_t k = static_cast<uint32_t>(item >> 48), type = static_cast<uint32_t>(item >> 32) & 0xFFFFu;
    const unsigned long long bit = p.type_bit_base[type] + static_cast<uint32_t>(item);
    const uint32_t m = 1u << (bit & 31);
    fresh = !(atomicOr(p.visited + k * p.words + (bit >> 5), m) & m);
    l = p.lk[k];
    is_cand = fresh && type == l.stype;
  }
  const unsigned fm = __ballot_sync(kFull, fresh), cm = __ballot_sync(kFull, is_cand);
  const unsigned below = (1u << lane) - 1u;
  unsigned long long fb = 0, cb = 0;
  if (lane == 0 && fm) fb = atomicAdd(p.out_count, static_cast<unsigned long long>(__popc(fm)));
  if (lane == 0 && cm) cb = atomicAdd(p.cand_count, static_cast<unsigned long long>(__popc(cm)));
  fb = __shfl_sync(kFull, fb, 0) + __popc(fm & below);
  cb = __shfl_sync(kFull, cb, 0) + __popc(cm & below);
  if (fresh) {
    if (fb < p.cap) p.out[fb] = item;
    else atomicOr(p.flags, 16u);
  }
  if (is_cand) {
    if (cb < p.cand_cap) {
      zg_check q;
      q.res = l.res;
      q.subj = static_cast<uint32_t>(item);
      q.perm = l.perm;
      q.stype = l.stype;
      q.srel = l.srel;
      q.flags = 0;
      p.cand[cb] = q;
      p.cand_owner[cb] = static_cast<uint8_t>(item >> 48);
    } else {
      atomicOr(p.flags, 16u);
    }
  }
}

// Exhaustive candidates of lookup k (its walk overflowed): the n ids of the subject type this rank owns,
// rank, rank + shard_count, ...
__global__ void ss_fill_owned_kernel(SubjectsParam l, uint32_t k, unsigned long long n, uint32_t shard_rank, uint32_t shard_count,
                                     zg_check* cand, uint8_t* cand_owner) {
  const unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  zg_check q;
  q.res = l.res;
  q.subj = static_cast<uint32_t>(shard_rank + i * shard_count);
  q.perm = l.perm;
  q.stype = l.stype;
  q.srel = l.srel;
  q.flags = 0;
  cand[i] = q;
  cand_owner[i] = static_cast<uint8_t>(k);
}

// First verification of this rank's candidates: failed bit k: the probe or a candidate of lookup k is undecidable
// (the lookup is ZG_EDEPTH); granted bit k: lookup k's probe checks HAS without a subject relation (the wildcard
// grants the permission). Only the owner of the resource holds the probe (subject ZG_NO_OBJECT - 1).
__global__ void ss_verdict_kernel(const zg_check* cand, const uint8_t* owner, const uint8_t* codes, unsigned long long n,
                                  unsigned long long* granted, unsigned long long* failed) {
  const unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const uint8_t code = codes[i];
  if (code == ZG_ITEM_ERROR) atomicOr(failed, 1ull << owner[i]);
  else if (code == ZG_HAS_PERMISSION && cand[i].subj == ZG_NO_OBJECT - 1 && cand[i].srel == kNone)
    atomicOr(granted, 1ull << owner[i]);
}

// Answer keys (excluded << kExclKeyBit | lookup << 32 | id; KeyHomeOwner sends them home) of the verified candidates
// other than the probes, for the lookups that did not fail: a HAS candidate is listed, unless its lookup is granted,
// in which case it goes to the no-wildcards verification (nw, nw_owner); a NO candidate of a granted lookup whose
// wildcard entry is asked for is excluded. After that verification the same kernel runs over its items with
// granted = failed = 0: its HAS subjects are listed.
constexpr int kExclKeyBit = 38;  // just above the lookup index: a lookup's listed ids sort before every excluded one
__global__ void ss_keys_kernel(const zg_check* cand, const uint8_t* owner, const uint8_t* codes, unsigned long long n,
                               unsigned long long granted, unsigned long long failed, unsigned long long include,
                               unsigned long long* keys, unsigned long long* n_keys, zg_check* nw, uint8_t* nw_owner,
                               unsigned long long* n_nw) {
  const unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  const unsigned lane = threadIdx.x & 31;
  bool listed = false, excl = false, again = false;
  uint32_t k = 0, subj = 0;
  if (i < n) {
    k = owner[i];
    subj = cand[i].subj;
    const uint8_t code = codes[i];
    const bool live = subj != ZG_NO_OBJECT - 1 && !((failed >> k) & 1ull), g = (granted >> k) & 1ull;
    listed = live && code == ZG_HAS_PERMISSION && !g;
    again = live && code == ZG_HAS_PERMISSION && g;
    excl = live && code == ZG_NO_PERMISSION && g && ((include >> k) & 1ull);
  }
  const bool key = listed || excl;
  const unsigned km = __ballot_sync(kFull, key), am = __ballot_sync(kFull, again);
  const unsigned below = (1u << lane) - 1u;
  unsigned long long kb = 0, ab = 0;
  if (lane == 0 && km) kb = atomicAdd(n_keys, static_cast<unsigned long long>(__popc(km)));
  if (lane == 0 && am) ab = atomicAdd(n_nw, static_cast<unsigned long long>(__popc(am)));
  kb = __shfl_sync(kFull, kb, 0) + __popc(km & below);
  ab = __shfl_sync(kFull, ab, 0) + __popc(am & below);
  if (key)
    keys[kb] = (static_cast<unsigned long long>(excl) << kExclKeyBit) | (static_cast<unsigned long long>(k) << 32) | subj;
  if (again) {
    nw[ab] = cand[i];
    nw_owner[ab] = static_cast<uint8_t>(k);
  }
}

// Keys that arrived home, sorted: run r = key >> 32 (lookup k's listed ids: r = k; its excluded ids:
// r = 64 + k) is ids[first[r] .. end[r]), both left 0 for an empty run.
__global__ void ss_split_kernel(const unsigned long long* keys, unsigned long long n, uint32_t* ids, unsigned long long* first,
                                unsigned long long* end) {
  const unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const unsigned long long key = keys[i], run = key >> 32;
  ids[i] = static_cast<uint32_t>(key);
  if (i == 0 || (keys[i - 1] >> 32) != run) first[run] = i;
  if (i + 1 == n || (keys[i + 1] >> 32) != run) end[run] = i + 1;
}

}  // namespace zg
