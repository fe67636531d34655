// ingress.cuh -- packed check ids resolved on the device against a mirror of the interned names.
//
// The host interns every object name of a type into an arena of records [u32 id][u32 len][bytes] (store.h TypeObjs)
// and finds them through an open-addressing table. The device keeps, per type, a byte-for-byte copy of that arena
// (record offsets mean the same on both sides), the offsets of its records, and a table of its own: u64 slots
// holding the top 24 bits of the name's hash (the tag) and `record offset + 1` (0 = empty), power-of-two capacity,
// load <= 1/2. A probe compares the tag first, so most probes that miss never touch the arena. device.cu
// (Device::ingress_sync) keeps the mirror in step with the store; the kernels below are all it runs.
//
// Ids are read in place from the caller's blob. They start at any byte alignment, and a thread never reads outside
// its id's range [off[i], off[i+1]): whole aligned 8-byte words where they lie inside the range, single bytes at the
// two ragged ends (WordStream).
#pragma once
#ifndef ZG_EMULATE  // tests/emu/: the same source under a CPU SIMT emulator (test infrastructure, never in libzgpu.so)
#include <cuda_runtime.h>
#endif
#include <cstdint>

#include "../../include/zgpu.h"
#include "hash_bytes.h"

namespace zg {

constexpr uint64_t kIngressOffMask = (1ull << 40) - 1;      // slot bits 0..39: record offset + 1
constexpr uint64_t kIngressTagMask = ~kIngressOffMask;      // slot bits 40..63: top 24 bits of the hash
constexpr unsigned kIngressThreads = 256;

// The bytes [s, s + n) as little-endian 64-bit words, word j = bytes 8j .. 8j + 7, zero past n. Reads only bytes
// inside the range: an aligned 8-byte window is loaded whole when it lies inside, byte by byte where it straddles
// an end; an unaligned word is the funnel of two windows.
struct WordStream {
  uintptr_t s, e, a;  // range [s, e); a = s rounded down to 8
  unsigned sh;        // s - a, in bits
  uint64_t cur;       // window at a + 8k (sh != 0 only)
  uint64_t k = 0;

  __device__ __forceinline__ WordStream(const uint8_t* p, uint64_t n)
      : s(reinterpret_cast<uintptr_t>(p)), e(reinterpret_cast<uintptr_t>(p) + n), a(s & ~uintptr_t(7)),
        sh(static_cast<unsigned>(s - a) * 8), cur(0) {
    if (sh) cur = window(0);
  }
  __device__ __forceinline__ uint64_t window(uint64_t w) const {
    const uintptr_t lo = a + 8 * w;
    if (lo >= s && lo + 8 <= e) return *reinterpret_cast<const uint64_t*>(lo);
    uint64_t v = 0;
    const uintptr_t b = lo < s ? s : lo, t = lo + 8 < e ? lo + 8 : e;
    for (uintptr_t q = b; q < t; ++q) v |= uint64_t(*reinterpret_cast<const uint8_t*>(q)) << (8 * (q - lo));
    return v;
  }
  __device__ __forceinline__ uint64_t next() {
    if (!sh) return window(k++);
    const uint64_t nx = window(++k);
    const uint64_t w = (cur >> sh) | (nx << (64 - sh));
    cur = nx;
    return w;
  }
};

__device__ __forceinline__ uint64_t ingress_hash(const uint8_t* p, uint64_t n) {
  WordStream ws(p, n);
  return hash_words(static_cast<size_t>(n), [&](size_t) { return ws.next(); });
}

__device__ __forceinline__ bool ingress_equal(const uint8_t* x, const uint8_t* y, uint64_t n) {
  WordStream a(x, n), b(y, n);
  for (uint64_t j = 0; j < (n + 7) / 8; ++j)
    if (a.next() != b.next()) return false;
  return true;
}

// One type's mirror, as the kernels see it. slots == nullptr: the type has no interned name.
struct IngressTable {
  const uint8_t* arena;
  const unsigned long long* slots;
  unsigned long long mask;  // capacity - 1
};

// Store::find on the device: the id of the name [p, p + n), or ZG_NO_OBJECT.
__device__ __forceinline__ uint32_t ingress_find(const IngressTable& t, const uint8_t* p, uint64_t n, uint64_t h,
                                                 uint64_t tag_mask) {
  if (!t.slots) return ZG_NO_OBJECT;
  for (uint64_t i = h & t.mask;; i = (i + 1) & t.mask) {
    const uint64_t v = t.slots[i];
    if (!v) return ZG_NO_OBJECT;
    if ((v ^ h) & tag_mask) continue;
    const uint8_t* rec = t.arena + ((v & kIngressOffMask) - 1);
    const uint64_t hdr = WordStream(rec, 8).next();  // [u32 id][u32 len], records are not aligned
    if ((hdr >> 32) == n && ingress_equal(rec + 8, p, n)) return static_cast<uint32_t>(hdr);
  }
}

// Inserts records offs[from .. to) of one type's arena into its table (atomicCAS on the slots: names are unique,
// so every record claims exactly one empty slot).
struct IngressInsertParams {
  const uint8_t* arena;
  const unsigned long long* offs;
  unsigned long long from, to;
  unsigned long long* slots;
  unsigned long long mask;
};

__global__ void __launch_bounds__(kIngressThreads) ingress_insert_kernel(const IngressInsertParams p) {
  const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
  for (uint64_t k = p.from + uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; k < p.to; k += stride) {
    const uint64_t off = p.offs[k];
    const uint8_t* rec = p.arena + off;
    const uint64_t len = WordStream(rec, 8).next() >> 32;
    const uint64_t h = ingress_hash(rec + 8, len);
    const unsigned long long v = (h & kIngressTagMask) | (off + 1);
    for (uint64_t i = h & p.mask;; i = (i + 1) & p.mask)
      if (atomicCAS(&p.slots[i], 0ull, v) == 0ull) break;
  }
}

// zg_resolve_checks_packed on the device. The literal fields were resolved once on the host (base, ok, and the one
// subject's id when every item has the same subject); per item the kernel finds the resource and the subject.
struct IngressResolveParams {
  IngressTable rt, st;
  const uint8_t* res_ids;
  const uint32_t* res_off;     // n + 1
  const uint8_t* subj_ids;     // per-item subjects, or the one subject's bytes (subj_off == nullptr)
  const uint32_t* subj_off;    // n + 1, or nullptr
  unsigned long long one_len;  // length of the one subject
  uint32_t one_su;             // its id (host-resolved), ZG_NO_OBJECT when never written
  int ok;                      // the literal fields resolved: else every item is `base` (ZG_ITEM_ERROR)
  int same_type;               // resource type == subject type (the self-membership rule)
  zg_check base;
  unsigned long long n;
  unsigned long long tag_mask;  // kIngressTagMask; 0 makes every probe compare bytes (emulator tests)
  zg_check* out;
  unsigned* bad;  // set when an offset decreases
};

__global__ void __launch_bounds__(kIngressThreads) ingress_resolve_kernel(const IngressResolveParams p) {
  const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
  for (uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < p.n; i += stride) {
    zg_check c = p.base;
    const uint32_t rb = p.res_off[i], re = p.res_off[i + 1];
    uint32_t sb = 0, se = 0;
    if (p.subj_off) {
      sb = p.subj_off[i];
      se = p.subj_off[i + 1];
    }
    if (re < rb || se < sb) {
      atomicOr(p.bad, 1u);
      p.out[i] = c;
      continue;
    }
    if (p.ok) {
      const uint8_t* rid = p.res_ids + rb;
      const uint64_t rl = re - rb;
      const uint32_t res = ingress_find(p.rt, rid, rl, ingress_hash(rid, rl), p.tag_mask);
      const uint8_t* sid = p.subj_off ? p.subj_ids + sb : p.subj_ids;
      const uint64_t sl = p.subj_off ? se - sb : p.one_len;
      uint32_t su = p.subj_off ? ingress_find(p.st, sid, sl, ingress_hash(sid, sl), p.tag_mask) : p.one_su;
      // two never-written names that are the same object must still compare equal
      if (su == ZG_NO_OBJECT)
        su = (res == ZG_NO_OBJECT && p.same_type && rl == sl && ingress_equal(rid, sid, rl)) ? ZG_NO_OBJECT
                                                                                             : ZG_NO_OBJECT - 1;
      c.res = res;
      c.subj = su;
    }
    p.out[i] = c;
  }
}

// ---- resource id prefixes (optional_resource_id_prefix) ----
// The ids of a type whose interned name starts with a prefix, read from the type's mirror: every record [u32 id][u32
// len][bytes] whose name is at least as long as the prefix and whose first bytes equal it sets bit `id` of the type's
// bitmap (n_ids bits: the snapshot's object capacity; an id at or past it is interned after the snapshot and no
// relationship of the snapshot names it). The comparison (ingress_equal) reads the name through a WordStream of the
// prefix's length, so no read leaves the record; names shorter than the prefix are never read. One launch covers every selected type.
constexpr int kMaxPrefixTypes = 64;  // types per launch; a schema with more runs several launches

struct PrefixType {
  const uint8_t* arena;
  const unsigned long long* offs;  // record offsets
  unsigned long long n_recs;
  uint32_t* bits;                  // ceil(n_ids / 32) words, zeroed by the host
  uint32_t n_ids;
  uint32_t pad;
};

struct PrefixPlan {
  const uint8_t* prefix;    // device bytes, 8-byte aligned
  unsigned long long len;   // 1 .. 1024
  unsigned long long* matched;  // += records that set a bit
  uint32_t n_types;
  uint32_t pad;
  PrefixType type[kMaxPrefixTypes];
};

__global__ void __launch_bounds__(kIngressThreads) prefix_match_kernel(const PrefixPlan p) {
  const uint64_t stride = uint64_t(gridDim.x) * blockDim.x;
  unsigned long long found = 0;
  for (uint32_t k = 0; k < p.n_types; ++k) {
    const PrefixType& t = p.type[k];
    for (uint64_t r = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; r < t.n_recs; r += stride) {
      const uint8_t* rec = t.arena + t.offs[r];
      const uint64_t hdr = WordStream(rec, 8).next();  // records are not aligned
      const uint32_t id = static_cast<uint32_t>(hdr);
      if ((hdr >> 32) < p.len || id >= t.n_ids || !ingress_equal(rec + 8, p.prefix, p.len)) continue;
      atomicOr(t.bits + (id >> 5), 1u << (id & 31));
      ++found;
    }
  }
  for (int d = 16; d > 0; d >>= 1) found += __shfl_xor_sync(0xFFFFFFFFu, found, d);
  if ((threadIdx.x & 31) == 0 && found) atomicAdd(p.matched, found);
}

}  // namespace zg
