// build.cu -- builds the CSR snapshot ON THE GPU from the raw relationship list.
//
// What it replaces: the reference's embedded SpiceDB keeps relationships in an
// in-memory datastore that every write updates (pkg/spicedb/spicedb.go:50); here a write
// republishes the snapshot, so build time is write-visibility latency
// (pkg/authz/distributedtx/activity.go:54-76 expects the write to be readable on return).
//
// Pipeline (all on one stream; cub radix sorts + scans, HBM-bound streaming passes):
//   1. key kernel: relationship -> row index (type_base + object * stride + class), subject
//   2. stable radix sort by subject, then stable radix sort by row index
//      => ordered by (row, subject), equal keys in load order (TOUCH: the last one wins)
//   3. flag the last entry of every (row, subject) run, exclusive scan, compact
//      => col / exp;   histogram of rows + inclusive scan => row_ptr
//   4. reverse CSR: one more stable radix sort of (class rrow_base + subject * rstride) keys; the
//      entries are already in ascending resource order within a class; histogram + scan
//   5. per type: objects that own >= 1 relationship (cub::DeviceSelect over row_ptr)
// The host builder (store.cc) produces identical arrays; ZGPU_VERIFY_BUILD=1 compares them.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <algorithm>
#include <cstring>
#include <unordered_map>

#include "delta.cuh"
#include "device.h"
#include "closure_sig.cuh"

namespace zg {

namespace {

struct BSlot {  // per relation slot
  unsigned long long row_base;
  uint32_t stride;
  uint16_t ncls;
  uint16_t cls_begin;
};

#define BCUDA(expr)                                                              \
  do {                                                                           \
    cudaError_t _e = (expr);                                                     \
    if (_e != cudaSuccess) return std::string(#expr) + ": " + cudaGetErrorString(_e); \
  } while (0)


// dead_key = pool: tombstoned relationships, and those another shard owns (res % own_count != own_rank), sort after
// every real row
__global__ void key_kernel(const zg_tuple* t, unsigned long long n, const BSlot* slots, const DCls* cls,
                           unsigned long long dead_key, uint32_t own_rank, uint32_t own_count, unsigned long long* rowkey,
                           uint32_t* subj, uint32_t* idx) {
  unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const zg_tuple x = t[i];
  idx[i] = static_cast<uint32_t>(i);
  subj[i] = x.srel == kWildcard ? 0u : x.subj;
  unsigned long long key = dead_key;
  if (!(x.flags & 1) && (own_count < 2 || x.res % own_count == own_rank)) {
    const BSlot s = slots[x.rel];
    for (uint32_t k = 0; k < s.ncls; ++k) {
      const DCls c = cls[s.cls_begin + k];
      if (c.stype == x.stype && c.sslot == x.srel) {
        key = s.row_base + static_cast<unsigned long long>(x.res) * s.stride + k;
        break;
      }
    }
  }
  rowkey[i] = key;
}

__global__ void gather_u64_kernel(const unsigned long long* src, const uint32_t* idx, unsigned long long n,
                                  unsigned long long* dst) {
  unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  if (i < n) dst[i] = src[idx[i]];
}

// last entry of each (row, subject) run among live entries
__global__ void flag_kernel(const unsigned long long* rowkey, const uint32_t* idx, const uint32_t* subj_by_tuple,
                            unsigned long long n, unsigned long long dead_key, uint32_t* flag) {
  unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = rowkey[i];
  uint32_t f = 0;
  if (k != dead_key) {
    f = 1;
    if (i + 1 < n && rowkey[i + 1] == k && subj_by_tuple[idx[i + 1]] == subj_by_tuple[idx[i]]) f = 0;
  }
  flag[i] = f;
}

// compact unique entries; count rows and classes; emit reverse keys
__global__ void emit_kernel(const unsigned long long* rowkey, const uint32_t* idx, const uint32_t* flag,
                            const uint32_t* pos, unsigned long long n, const zg_tuple* t, const uint32_t* expires,
                            const BSlot* slots, const DCls* cls, uint32_t* col, uint32_t* exp, uint32_t* row_cnt,
                            uint32_t* cls_cnt, unsigned long long* rkey, uint32_t* rres, uint32_t* rrow_cnt) {
  unsigned long long i = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  if (i >= n || !flag[i]) return;
  const uint32_t p = pos[i], ti = idx[i];
  const zg_tuple x = t[ti];
  const uint32_t s = x.srel == kWildcard ? 0u : x.subj;
  col[p] = s;
  if (exp) exp[p] = expires[ti];
  const unsigned long long row = rowkey[i];
  atomicAdd(row_cnt + row + 1, 1u);
  const BSlot bs = slots[x.rel];
  const uint32_t gc = bs.cls_begin + static_cast<uint32_t>((row - bs.row_base) % bs.stride);
  atomicAdd(cls_cnt + gc, 1u);
  const unsigned long long rk = cls[gc].rrow_base + static_cast<unsigned long long>(s) * cls[gc].rstride;
  rkey[p] = rk;
  rres[p] = x.res;
  atomicAdd(rrow_cnt + rk + 1, 1u);
}

__global__ void owner_flag_kernel(const uint32_t* row_ptr, unsigned long long type_base, uint32_t stride, uint32_t n_obj,
                                  uint8_t* flag) {
  uint32_t o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= n_obj) return;
  flag[o] = stride && row_ptr[type_base + static_cast<unsigned long long>(o + 1) * stride] >
                          row_ptr[type_base + static_cast<unsigned long long>(o) * stride];
}

int bits_for(unsigned long long max_value) {
  int b = 1;
  while (b < 64 && (max_value >> b)) ++b;
  return b;
}

// ---- closure index of a two-level pair (a = innermost direct class, b = userset class tgc) ----
// row u = the union of rrow(g, b) over g in rrow(u, a); the reverse rows are read from the resident snapshot

__device__ __forceinline__ void rrow_of(const uint32_t* rrow_ptr, const DCls& c, uint32_t s, uint32_t* lo, uint32_t* hi) {
  const unsigned long long ri = c.rrow_base + static_cast<unsigned long long>(s) * c.rstride;
  *lo = rrow_ptr[ri];
  *hi = rrow_ptr[ri + 1];
}

// cnt[u + 1] = sum of |rrow(g, b)| over the memberships g of u; *rels += relationships of class a (and of class b for
// the subjects g < b.nsubj, counted by the threads u < b.nsubj)
__global__ void closure_count_kernel(const uint32_t* rrow_ptr, const uint32_t* rcol, DCls a, DCls b, uint32_t n,
                                     unsigned long long* cnt, unsigned long long* rels) {
  const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long sum = 0, own = 0;
  if (u < n) {
    uint32_t lo = 0, hi = 0;
    if (u < a.nsubj) rrow_of(rrow_ptr, a, u, &lo, &hi);
    own = hi - lo;
    for (uint32_t x = lo; x < hi; ++x) {
      const uint32_t g = rcol[x];
      if (g >= b.nsubj) continue;
      uint32_t l = 0, h = 0;
      rrow_of(rrow_ptr, b, g, &l, &h);
      sum += h - l;
    }
    cnt[u + 1] = sum;
    if (u < b.nsubj) {
      uint32_t l = 0, h = 0;
      rrow_of(rrow_ptr, b, u, &l, &h);
      own += h - l;
    }
  }
  for (int d = 16; d >= 1; d >>= 1) own += __shfl_xor_sync(0xFFFFFFFFu, own, d);
  if ((threadIdx.x & 31) == 0 && own) atomicAdd(rels, own);
}

__global__ void closure_fill_kernel(const uint32_t* rrow_ptr, const uint32_t* rcol, DCls a, DCls b, uint32_t n,
                                    const unsigned long long* off, uint32_t* out) {
  const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= n || u >= a.nsubj) return;
  unsigned long long at = off[u];
  uint32_t lo, hi;
  rrow_of(rrow_ptr, a, u, &lo, &hi);
  for (uint32_t x = lo; x < hi; ++x) {
    const uint32_t g = rcol[x];
    if (g >= b.nsubj) continue;
    uint32_t l, h;
    rrow_of(rrow_ptr, b, g, &l, &h);
    for (uint32_t y = l; y < h; ++y) out[at++] = rcol[y];
  }
}

// distinct entries of each sorted row: counted into ucnt[u + 1] (out == nullptr), or written to out[row_ptr[u] ..] at
// the index's width (T = uint16_t: every entry is below 65 536)
template <class T>
__global__ void closure_unique_kernel(const uint32_t* sorted, const unsigned long long* off, uint32_t n, uint32_t* ucnt,
                                      const uint32_t* row_ptr, T* out) {
  const uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= n) return;
  const unsigned long long lo = off[u], hi = off[u + 1];
  uint32_t k = 0, at = out ? row_ptr[u] : 0u;
  for (unsigned long long x = lo; x < hi; ++x) {
    if (x > lo && sorted[x] == sorted[x - 1]) continue;
    if (out) out[at + k] = static_cast<T>(sorted[x]);
    ++k;
  }
  if (!out) ucnt[u + 1] = k;
}

// Signature of every closure row, one warp per row: lane w owns word w of the row's 2^lg, and every lane tests every
// entry of the row (32 read at a time, then broadcast) for its word, so no word is written by two lanes.
template <class E>
__global__ void closure_sig_kernel(const uint32_t* row_ptr, const E* col, uint32_t n, uint32_t lg, unsigned long long* sig) {
  const uint32_t lane = threadIdx.x & 31u;
  const unsigned long long u = (static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (u >= n) return;  // warp-uniform
  const uint32_t lo = row_ptr[u], hi = row_ptr[u + 1];
  unsigned long long w = 0;
  for (uint32_t b = lo; b < hi; b += 32) {
    const uint32_t mine = b + lane < hi ? static_cast<uint32_t>(col[b + lane]) : 0u;
    const uint32_t cnt = min(32u, hi - b);
    for (uint32_t j = 0; j < cnt; ++j) {
      const uint32_t v = __shfl_sync(0xFFFFFFFFu, mine, j);
      if (sig_word(v, lg) == lane) w |= sig_mask(v);
    }
  }
  if (lane < (1u << lg)) sig[(u << lg) + lane] = w;
}

// Set table of every 16-bit closure row (closure_sig.cuh), one warp per row, in two launches over the same placement:
// the row's entries are dealt 32 at a time, lanes with the same bucket find each other (__match_any_sync), and each
// takes the bucket's next slot in entry order from a per-warp histogram in shared memory, so a bucket holds its entries
// ascending. Choose (tab == nullptr): tries bucket counts from table_first_nb on, growing by table_grow_nb, `seeds` seeds
// each, until no bucket gets more than kTableSlots entries; writes the row's bucket count into cnt[u + 1] and nb / seed into
// hdr[u], or sets *failed when the row needs more than kTableMaxBuckets buckets. Fill: cnt holds the rows' first
// buckets; writes the entries into tab (all 0xFFFF before) and completes hdr[u].
constexpr unsigned kTableWarps = 4;
__global__ void __launch_bounds__(kTableWarps * 32)
    closure_table_kernel(const uint32_t* row_ptr, const uint16_t* col, uint32_t n, uint32_t seeds,
                         unsigned long long* cnt, unsigned long long* hdr, uint16_t* tab, uint32_t* failed) {
  __shared__ uint32_t hist_words[kTableWarps][kTableMaxBuckets / 4];
  const uint32_t lane = threadIdx.x & 31u, below = (1u << lane) - 1u;
  const unsigned long long u = (static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  if (u >= n) return;  // warp-uniform
  uint32_t* hw = hist_words[threadIdx.x >> 5];
  uint8_t* hist = reinterpret_cast<uint8_t*>(hw);
  const uint32_t lo = row_ptr[u], hi = row_ptr[u + 1];
  // places the row into nb buckets under `seed`: false as soon as a bucket would get a fifth entry; writes the entries
  // to out when it is given (counts stay below 4 + 32, so a byte holds them)
  auto place = [&](uint32_t nb, uint32_t seed, uint16_t* out) -> bool {
    for (uint32_t i = lane; i < (nb + 3) / 4; i += 32) hw[i] = 0;
    __syncwarp();
    for (uint32_t b = lo; b < hi; b += 32) {
      const bool mine = b + lane < hi;
      const uint32_t v = mine ? col[b + lane] : 0u;
      const uint32_t k = mine ? table_bucket(v, seed, nb) : ~0u;
      const unsigned peers = __match_any_sync(0xFFFFFFFFu, k);
      const uint32_t base = mine ? hist[k] : 0u, slot = base + __popc(peers & below);
      __syncwarp();
      if (mine && !(peers & below)) hist[k] = static_cast<uint8_t>(base + __popc(peers));
      __syncwarp();
      if (__any_sync(0xFFFFFFFFu, mine && slot >= kTableSlots)) return false;
      if (out && mine) out[static_cast<unsigned long long>(k) * kTableSlots + slot] = static_cast<uint16_t>(v);
    }
    return true;
  };
  if (!tab) {
    uint32_t nb = table_first_nb(hi - lo), seed = 0;
    bool ok = hi == lo;
    while (!ok && nb <= kTableMaxBuckets) {
      for (seed = 0; seed < seeds; ++seed)
        if ((ok = place(nb, seed, nullptr))) break;
      if (!ok) nb = table_grow_nb(nb);
    }
    if (!ok) {
      if (lane == 0) atomicExch(failed, 1u);
      return;
    }
    if (lane == 0) {
      cnt[u + 1] = nb;
      hdr[u] = table_header(0, nb, seed);
    }
  } else {
    const unsigned long long h = hdr[u], off = cnt[u];
    const uint32_t nb = static_cast<uint32_t>(h >> 32) & 0xFFFFFFu, seed = static_cast<uint32_t>(h >> 56);
    place(nb, seed, tab + off * kTableSlots);
    if (lane == 0) hdr[u] = table_header(static_cast<uint32_t>(off), nb, seed);
  }
}

// Range records of one class (closure_sig.cuh kRecSlots): one thread per 16-bit slot, so that a warp writes two
// records whole. Counts the rows longer than a record holds in *n_long.
__global__ void flat_record_kernel(const uint32_t* row_ptr, const uint32_t* col, unsigned long long row_base, uint32_t ncls,
                                   uint32_t nres, uint16_t* rec, unsigned long long* n_long) {
  const unsigned long long t = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x;
  if (t >= static_cast<unsigned long long>(nres) * kRecSlots) return;
  const uint32_t obj = static_cast<uint32_t>(t / kRecSlots), k = static_cast<uint32_t>(t % kRecSlots);
  const unsigned long long row = row_base + static_cast<unsigned long long>(obj) * ncls;
  const uint32_t lo = row_ptr[row], n = row_ptr[row + 1] - lo;
  const bool inline_row = n < kRecSlots;
  uint32_t v = kRecLong;
  if (k == 0) v = inline_row ? n : kRecLong;
  else if (inline_row && k <= n) v = col[lo + k - 1];
  rec[t] = static_cast<uint16_t>(v);
  if (k == 0 && !inline_row) atomicAdd(n_long, 1ull);
}

}  // namespace

std::string gpu_build_closure(const Snapshot& s, const DCls& a, const DCls& b, uint64_t cap, Snapshot::Closure* c,
                              cudaStream_t st) {
  c->built = false;
  c->entries = 0;
  c->nsubj = a.nsubj;
  const uint32_t n = std::max(a.nsubj, b.nsubj);  // threads of the count pass (it also sums class b's relationships)
  if (a.nsubj == 0) return "";
  DevBuf d_off, d_keys[2], d_tmp, d_rels;
  struct Release {
    std::vector<DevBuf*> v;
    ~Release() {
      for (DevBuf* x : v) x->release();
    }
  } rel{{&d_off, &d_keys[0], &d_keys[1], &d_tmp, &d_rels}};
  if (!d_off.ensure((size_t(n) + 1) * 8) || !d_rels.ensure(16)) return "out of device memory (closure index)";
  BCUDA(cudaMemsetAsync(d_off.p, 0, (size_t(n) + 1) * 8, st));
  BCUDA(cudaMemsetAsync(d_rels.p, 0, 8, st));
  const unsigned blk = 256, grid = (n + blk - 1) / blk;
  const uint32_t* rp = s.rrow_ptr.as<uint32_t>();
  const uint32_t* rc = s.rcol.as<uint32_t>();
  closure_count_kernel<<<grid, blk, 0, st>>>(rp, rc, a, b, n, d_off.as<unsigned long long>(), d_rels.as<unsigned long long>());
  unsigned long long* off = d_off.as<unsigned long long>();
  size_t tb = 0;
  cub::DeviceScan::InclusiveSum(nullptr, tb, off, off, a.nsubj + 1, st);
  if (!d_tmp.ensure(tb + 256)) return "out of device memory (closure index)";
  tb = d_tmp.cap;
  BCUDA(cub::DeviceScan::InclusiveSum(d_tmp.p, tb, off, off, a.nsubj + 1, st));
  unsigned long long hb[2] = {0, 0};
  BCUDA(cudaMemcpyAsync(&hb[0], off + a.nsubj, 8, cudaMemcpyDeviceToHost, st));
  BCUDA(cudaMemcpyAsync(&hb[1], d_rels.p, 8, cudaMemcpyDeviceToHost, st));
  BCUDA(cudaStreamSynchronize(st));
  const uint64_t total = hb[0], rels = hb[1];
  // Size budget, checked on the exact count before anything is allocated: the entries before duplicates are removed
  // (sorted twice) must stay within kClosureRatio x the relationships of the two classes, a quarter of the free device
  // memory (two 32-bit sort buffers and the index at its width per entry), and what one cub sort takes (2^31 keys).
  // `cap` (ZGPU_CLOSURE_CAP) replaces the ratio.
  size_t free_b = 0, total_b = 0;
  BCUDA(cudaMemGetInfo(&free_b, &total_b));
  const uint64_t limit =
      std::min<uint64_t>({cap != ~0ull ? cap : kClosureRatio * rels, free_b / 4 / (8 + c->width), (1ull << 31) - 1});
  if (total > limit) {  // no index: the pair's steps keep batch_l2
    c->row_ptr.release();
    c->col.release();
    return "";
  }
  if (total) {
    if (!d_keys[0].ensure(total * 4) || !d_keys[1].ensure(total * 4)) return "out of device memory (closure index)";
    closure_fill_kernel<<<(a.nsubj + blk - 1) / blk, blk, 0, st>>>(rp, rc, a, b, a.nsubj, off, d_keys[0].as<uint32_t>());
    size_t sb = 0;
    cub::DeviceSegmentedSort::SortKeys(nullptr, sb, d_keys[0].as<uint32_t>(), d_keys[1].as<uint32_t>(), static_cast<int>(total),
                                       static_cast<int>(a.nsubj), off, off + 1, st);
    if (!d_tmp.ensure(sb + 256)) return "out of device memory (closure sort scratch)";
    sb = d_tmp.cap;
    BCUDA(cub::DeviceSegmentedSort::SortKeys(d_tmp.p, sb, d_keys[0].as<uint32_t>(), d_keys[1].as<uint32_t>(),
                                             static_cast<int>(total), static_cast<int>(a.nsubj), off, off + 1, st));
  }
  if (!c->row_ptr.ensure((size_t(a.nsubj) + 1) * 4)) return "out of device memory (closure index)";
  uint32_t* crow = c->row_ptr.as<uint32_t>();
  BCUDA(cudaMemsetAsync(crow, 0, (size_t(a.nsubj) + 1) * 4, st));
  const unsigned ug = (a.nsubj + blk - 1) / blk;
  if (total) closure_unique_kernel<uint32_t><<<ug, blk, 0, st>>>(d_keys[1].as<uint32_t>(), off, a.nsubj, crow, nullptr, nullptr);
  tb = 0;
  cub::DeviceScan::InclusiveSum(nullptr, tb, crow, crow, a.nsubj + 1, st);
  if (!d_tmp.ensure(tb + 256)) return "out of device memory (closure index)";
  tb = d_tmp.cap;
  BCUDA(cub::DeviceScan::InclusiveSum(d_tmp.p, tb, crow, crow, a.nsubj + 1, st));
  uint32_t nu = 0;
  BCUDA(cudaMemcpyAsync(&nu, crow + a.nsubj, 4, cudaMemcpyDeviceToHost, st));
  BCUDA(cudaStreamSynchronize(st));
  // + 4 words, or + 16 16-bit entries: the aligned 16-byte block (32-byte sector) that holds a row's last entry ends
  // inside the allocation
  const size_t col_bytes = (size_t(nu) + (c->width == 2 ? 16 : 4)) * c->width;
  if (!c->col.ensure(col_bytes)) return "out of device memory (closure index)";
  BCUDA(cudaMemsetAsync(c->col.p, 0, col_bytes, st));
  if (total && c->width == 2)
    closure_unique_kernel<<<ug, blk, 0, st>>>(d_keys[1].as<uint32_t>(), off, a.nsubj, nullptr, crow, c->col.as<uint16_t>());
  else if (total)
    closure_unique_kernel<<<ug, blk, 0, st>>>(d_keys[1].as<uint32_t>(), off, a.nsubj, nullptr, crow, c->col.as<uint32_t>());
  BCUDA(cudaStreamSynchronize(st));
  BCUDA(cudaGetLastError());
  c->entries = nu;
  c->built = true;
  return "";
}

std::string gpu_build_closure_sig(Snapshot::Closure* c, uint32_t words, cudaStream_t st) {
  c->sig_words = 0;
  if (!c->built || words == 0) {
    c->sig.release();
    return "";
  }
  if (words == ~0u) {
    words = 1;
    while (words < 32 && 64ull * words * c->nsubj < 12ull * c->entries) words <<= 1;
  } else {
    words = 1u << (31 - __builtin_clz(std::min(words, 32u)));  // a power of two, at most 32
  }
  const uint32_t lg = static_cast<uint32_t>(__builtin_ctz(words));
  const size_t bytes = (size_t(c->nsubj) << lg) * 8;
  size_t free_b = 0, total_b = 0;
  BCUDA(cudaMemGetInfo(&free_b, &total_b));
  if (bytes > (free_b + c->sig.cap) / 4) {  // (counting the pair's old signature buffer as free: it is reused)
    c->sig.release();
    return "";
  }
  if (!c->sig.ensure(bytes ? bytes : 8)) return "out of device memory (closure signatures)";
  if (c->nsubj) {
    const unsigned blk = 256;
    const unsigned long long grid = (static_cast<unsigned long long>(c->nsubj) * 32 + blk - 1) / blk;
    if (c->width == 2)
      closure_sig_kernel<<<grid, blk, 0, st>>>(c->row_ptr.as<uint32_t>(), c->col.as<uint16_t>(), c->nsubj, lg,
                                               c->sig.as<unsigned long long>());
    else
      closure_sig_kernel<<<grid, blk, 0, st>>>(c->row_ptr.as<uint32_t>(), c->col.as<uint32_t>(), c->nsubj, lg,
                                               c->sig.as<unsigned long long>());
    BCUDA(cudaGetLastError());
  }
  BCUDA(cudaStreamSynchronize(st));
  c->sig_words = words;
  return "";
}

std::string gpu_build_closure_table(Snapshot::Closure* c, uint32_t seeds, cudaStream_t st) {
  c->set_built = false;
  c->set_buckets = 0;
  auto none = [c]() {
    c->set_hdr.release();
    c->set_tab.release();
    return std::string();
  };
  if (!c->built || c->width != 2 || c->nsubj == 0 || seeds == 0) return none();
  seeds = std::min(seeds, 256u);  // (8 bits of the header)
  const size_t n = c->nsubj;
  DevBuf d_cnt, d_tmp, d_failed;
  struct Release {
    std::vector<DevBuf*> v;
    ~Release() {
      for (DevBuf* x : v) x->release();
    }
  } rel{{&d_cnt, &d_tmp, &d_failed}};
  if (!c->set_hdr.ensure(n * 8) || !d_cnt.ensure((n + 1) * 8) || !d_failed.ensure(4))
    return "out of device memory (closure set table)";
  unsigned long long* cnt = d_cnt.as<unsigned long long>();
  BCUDA(cudaMemsetAsync(cnt, 0, (n + 1) * 8, st));
  BCUDA(cudaMemsetAsync(d_failed.p, 0, 4, st));
  const unsigned blk = kTableWarps * 32;
  const unsigned long long grid = (static_cast<unsigned long long>(n) * 32 + blk - 1) / blk;
  const uint32_t* rp = c->row_ptr.as<uint32_t>();
  const uint16_t* col = c->col.as<uint16_t>();
  closure_table_kernel<<<grid, blk, 0, st>>>(rp, col, c->nsubj, seeds, cnt, c->set_hdr.as<unsigned long long>(), nullptr,
                                             d_failed.as<uint32_t>());
  BCUDA(cudaGetLastError());
  size_t tb = 0;
  cub::DeviceScan::InclusiveSum(nullptr, tb, cnt, cnt, n + 1, st);
  if (!d_tmp.ensure(tb + 256)) return "out of device memory (closure set table)";
  tb = d_tmp.cap;
  BCUDA(cub::DeviceScan::InclusiveSum(d_tmp.p, tb, cnt, cnt, n + 1, st));
  unsigned long long total = 0;
  uint32_t failed = 0;
  BCUDA(cudaMemcpyAsync(&total, cnt + n, 8, cudaMemcpyDeviceToHost, st));
  BCUDA(cudaMemcpyAsync(&failed, d_failed.p, 4, cudaMemcpyDeviceToHost, st));
  BCUDA(cudaStreamSynchronize(st));
  // a row that needs more buckets than the build takes, or a first bucket past 32 bits: no table
  if (failed || total >= (1ull << 32)) return none();
  const size_t bytes = size_t(total) * 8;
  size_t free_b = 0, total_b = 0;
  BCUDA(cudaMemGetInfo(&free_b, &total_b));
  if (bytes + n * 8 > (free_b + c->set_tab.cap + c->set_hdr.cap) / 4) return none();  // (the pair's old buffers are reused)
  if (!c->set_tab.ensure(bytes ? bytes : 8)) return "out of device memory (closure set table)";
  BCUDA(cudaMemsetAsync(c->set_tab.p, 0xFF, bytes ? bytes : 8, st));
  closure_table_kernel<<<grid, blk, 0, st>>>(rp, col, c->nsubj, seeds, cnt, c->set_hdr.as<unsigned long long>(),
                                             c->set_tab.as<uint16_t>(), d_failed.as<uint32_t>());
  BCUDA(cudaGetLastError());
  BCUDA(cudaStreamSynchronize(st));
  c->set_buckets = total;
  c->set_built = true;
  return "";
}

std::string gpu_build_flat_records(const Snapshot& s, Snapshot::FlatRecords* r, cudaStream_t st) {
  r->built = false;
  r->long_rows = 0;
  const size_t bytes = size_t(r->nres) * kRecSlots * 2;
  size_t free_b = 0, total_b = 0;
  BCUDA(cudaMemGetInfo(&free_b, &total_b));
  if (bytes > (free_b + r->rec.cap) / 4) {  // (counting the class's old records as free: they are reused)
    r->rec.release();
    return "";
  }
  DevBuf d_long;
  if (!r->rec.ensure(bytes ? bytes : 16) || !d_long.ensure(8)) {
    d_long.release();
    return "out of device memory (range records)";
  }
  unsigned long long n_long = 0;
  cudaError_t ce = cudaMemsetAsync(d_long.p, 0, 8, st);
  if (ce == cudaSuccess && bytes) {
    const unsigned blk = 256;
    const unsigned long long grid = (static_cast<unsigned long long>(r->nres) * kRecSlots + blk - 1) / blk;
    flat_record_kernel<<<grid, blk, 0, st>>>(s.row_ptr.as<uint32_t>(), s.col.as<uint32_t>(), r->row_base, r->ncls,
                                              r->nres, r->rec.as<uint16_t>(), d_long.as<unsigned long long>());
    ce = cudaGetLastError();
  }
  if (ce == cudaSuccess) ce = cudaMemcpyAsync(&n_long, d_long.p, 8, cudaMemcpyDeviceToHost, st);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
  d_long.release();
  if (ce != cudaSuccess) return std::string("range records: ") + cudaGetErrorString(ce);
  r->long_rows = n_long;
  r->built = true;
  return "";
}

std::string sort_u32(const uint32_t* d_in, uint32_t* d_out, uint64_t n, cudaStream_t st) {
  static thread_local DevBuf tmp;  // grow-only scratch per calling thread
  size_t bytes = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, bytes, d_in, d_out, n, 0, 32, st);
  if (!tmp.ensure(bytes + 256)) return "out of device memory (sort scratch)";
  bytes = tmp.cap;
  BCUDA(cub::DeviceRadixSort::SortKeys(tmp.p, bytes, d_in, d_out, n, 0, 32, st));
  return "";
}

std::string sort_u64(const unsigned long long* d_in, unsigned long long* d_out, uint64_t n, int end_bit, cudaStream_t st) {
  static thread_local DevBuf tmp;
  size_t bytes = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, bytes, d_in, d_out, n, 0, end_bit, st);
  if (!tmp.ensure(bytes + 256)) return "out of device memory (sort scratch)";
  bytes = tmp.cap;
  BCUDA(cub::DeviceRadixSort::SortKeys(tmp.p, bytes, d_in, d_out, n, 0, end_bit, st));
  return "";
}

// per type: objects that are the resource of >= 1 relationship (ascending ids), from the forward row table
std::string gpu_resource_lists(Snapshot* s, cudaStream_t st) {
  const size_t nt = s->n_objects.size();
  const unsigned blk = 256;
  s->resources.resize(nt);
  s->n_resources.assign(nt, 0);
  DevBuf d_of, d_num, d_tmp;
  struct Release {
    std::vector<DevBuf*> v;
    ~Release() {
      for (DevBuf* b : v) b->release();
    }
  } rel2{{&d_of, &d_num, &d_tmp}};
  if (!d_num.ensure(16)) return "out of device memory";
  for (size_t t = 0; t < nt; ++t) {
    const uint32_t no = s->n_objects[t];
    if (!s->resources[t].ensure(std::max<size_t>(size_t(no) * 4, 16))) return "out of device memory (resource lists)";
    if (!no || !s->type_ncls[t]) continue;
    if (!d_of.ensure(no)) return "out of device memory";
    owner_flag_kernel<<<(no + blk - 1) / blk, blk, 0, st>>>(s->row_ptr.as<uint32_t>(), s->type_base[t], s->type_ncls[t], no,
                                                            d_of.as<uint8_t>());
    size_t tb = 0;
    thrust::counting_iterator<uint32_t> ids(0);
    cub::DeviceSelect::Flagged(nullptr, tb, ids, d_of.as<uint8_t>(), s->resources[t].as<uint32_t>(), d_num.as<uint32_t>(), no, st);
    if (!d_tmp.ensure(tb + 256)) return "out of device memory (select scratch)";
    tb = d_tmp.cap;
    BCUDA(cub::DeviceSelect::Flagged(d_tmp.p, tb, ids, d_of.as<uint8_t>(), s->resources[t].as<uint32_t>(),
                                     d_num.as<uint32_t>(), no, st));
    uint32_t cnt = 0;
    BCUDA(cudaMemcpyAsync(&cnt, d_num.p, 4, cudaMemcpyDeviceToHost, st));
    BCUDA(cudaStreamSynchronize(st));
    s->n_resources[t] = cnt;
  }
  s->resources_stale = false;
  return "";
}

// Fills `s` (row_ptr, col, exp, rrow_ptr, rcol, resources) from the store's relationship list.
// `lay` comes from Store::layout(); on return lay->cls has CF_EMPTY cleared for non-empty classes.
std::string gpu_build_snapshot(const Store& store, const Schema& sc, HostSnapshot* lay, cudaStream_t st, Snapshot* s,
                               uint32_t owner_rank, uint32_t owner_count) {
  const uint64_t n = store.tuples.size();
  if (n >= 0xFFFFFFF0ull) return "more than 2^32 relationships in one snapshot";
  const uint64_t pool = lay->pool, rpool = lay->rpool;
  const bool with_exp = sc.has_expiry;

  std::vector<BSlot> bslots(sc.slots.size(), BSlot{0, 0, 0, 0});
  for (size_t i = 0; i < sc.rel_slots.size(); ++i) {
    const DRel& r = lay->rels[i];
    bslots[sc.rel_slots[i]] = BSlot{r.row_base, r.stride, r.ncls, r.cls_begin};
  }
  DevBuf d_t, d_e, d_slots, d_cls, d_key[2], d_idx[2], d_subj[2], d_flag, d_pos, d_tmp, d_rkey[2], d_rres[2], d_clscnt;
  struct Release {
    std::vector<DevBuf*> v;
    ~Release() {
      for (DevBuf* b : v) b->release();
    }
  } rel{{&d_t, &d_e, &d_slots, &d_cls, &d_key[0], &d_key[1], &d_idx[0], &d_idx[1], &d_subj[0], &d_subj[1], &d_flag,
         &d_pos, &d_tmp, &d_rkey[0], &d_rkey[1], &d_rres[0], &d_rres[1], &d_clscnt}};
  auto need = [&](DevBuf& b, size_t bytes) { return b.ensure(bytes ? bytes : 16); };
  const size_t nn = n ? n : 1;
  if (!need(d_t, nn * sizeof(zg_tuple)) || !need(d_slots, bslots.size() * sizeof(BSlot)) ||
      !need(d_cls, lay->cls.size() * sizeof(DCls)) || !need(d_key[0], nn * 8) || !need(d_key[1], nn * 8) ||
      !need(d_idx[0], nn * 4) || !need(d_idx[1], nn * 4) || !need(d_subj[0], nn * 4) || !need(d_subj[1], nn * 4) ||
      !need(d_flag, nn * 4) || !need(d_pos, nn * 4) || !need(d_clscnt, (lay->cls.size() + 1) * 4) ||
      (with_exp && !need(d_e, nn * 4)))
    return "out of device memory (snapshot build)";
  BCUDA(cudaMemcpyAsync(d_t.p, store.tuples.data(), n * sizeof(zg_tuple), cudaMemcpyHostToDevice, st));
  if (with_exp) BCUDA(cudaMemcpyAsync(d_e.p, store.expires.data(), n * 4, cudaMemcpyHostToDevice, st));
  BCUDA(cudaMemcpyAsync(d_slots.p, bslots.data(), bslots.size() * sizeof(BSlot), cudaMemcpyHostToDevice, st));
  BCUDA(cudaMemcpyAsync(d_cls.p, lay->cls.data(), lay->cls.size() * sizeof(DCls), cudaMemcpyHostToDevice, st));
  BCUDA(cudaMemsetAsync(d_clscnt.p, 0, (lay->cls.size() + 1) * 4, st));

  if (!s->row_ptr.ensure((pool + 1) * 4) || !s->rrow_ptr.ensure((rpool + 1) * 4))
    return "out of device memory (row tables)";
  BCUDA(cudaMemsetAsync(s->row_ptr.p, 0, (pool + 1) * 4, st));
  BCUDA(cudaMemsetAsync(s->rrow_ptr.p, 0, (rpool + 1) * 4, st));

  const unsigned blk = 256;
  const unsigned grid = static_cast<unsigned>((nn + blk - 1) / blk);
  uint64_t n_unique = 0;
  if (n) {
    const int kbits = bits_for(pool);  // keys are < pool, tombstones == pool
    key_kernel<<<grid, blk, 0, st>>>(d_t.as<zg_tuple>(), n, d_slots.as<BSlot>(), d_cls.as<DCls>(), pool, owner_rank,
                                     owner_count, d_key[0].as<unsigned long long>(), d_subj[0].as<uint32_t>(), d_idx[0].as<uint32_t>());
    // pass A: stable sort of tuple indices by subject
    size_t tmp_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, d_subj[0].as<uint32_t>(), d_subj[1].as<uint32_t>(),
                                    d_idx[0].as<uint32_t>(), d_idx[1].as<uint32_t>(), n, 0, 32, st);
    size_t tmp2 = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tmp2, d_key[0].as<unsigned long long>(), d_key[1].as<unsigned long long>(),
                                    d_idx[0].as<uint32_t>(), d_idx[1].as<uint32_t>(), n, 0, kbits, st);
    size_t tmp3 = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tmp3, d_flag.as<uint32_t>(), d_pos.as<uint32_t>(), n, st);
    size_t tmp4 = 0, tmp5 = 0;
    cub::DeviceScan::InclusiveSum(nullptr, tmp4, s->row_ptr.as<uint32_t>(), s->row_ptr.as<uint32_t>(), pool + 1, st);
    cub::DeviceScan::InclusiveSum(nullptr, tmp5, s->rrow_ptr.as<uint32_t>(), s->rrow_ptr.as<uint32_t>(), rpool + 1, st);
    tmp_bytes = std::max({tmp_bytes, tmp2, tmp3, tmp4, tmp5}) + 256;
    if (!d_tmp.ensure(tmp_bytes)) return "out of device memory (sort scratch)";
    BCUDA(cub::DeviceRadixSort::SortPairs(d_tmp.p, tmp_bytes, d_subj[0].as<uint32_t>(), d_subj[1].as<uint32_t>(),
                                          d_idx[0].as<uint32_t>(), d_idx[1].as<uint32_t>(), n, 0, 32, st));
    // pass B: stable sort by row index (dead relationships sort last)
    gather_u64_kernel<<<grid, blk, 0, st>>>(d_key[0].as<unsigned long long>(), d_idx[1].as<uint32_t>(), n,
                                            d_key[1].as<unsigned long long>());
    BCUDA(cub::DeviceRadixSort::SortPairs(d_tmp.p, tmp_bytes, d_key[1].as<unsigned long long>(),
                                          d_key[0].as<unsigned long long>(), d_idx[1].as<uint32_t>(),
                                          d_idx[0].as<uint32_t>(), n, 0, kbits, st));
    // now d_key[0] = sorted row keys, d_idx[0] = tuple indices in (row, subject, load order);
    // d_subj[0] still holds the subject per tuple index (sort inputs are left intact)
    flag_kernel<<<grid, blk, 0, st>>>(d_key[0].as<unsigned long long>(), d_idx[0].as<uint32_t>(), d_subj[0].as<uint32_t>(), n,
                                      pool, d_flag.as<uint32_t>());
    BCUDA(cub::DeviceScan::ExclusiveSum(d_tmp.p, tmp_bytes, d_flag.as<uint32_t>(), d_pos.as<uint32_t>(), n, st));
    uint32_t last_pos = 0, last_flag = 0;
    BCUDA(cudaMemcpyAsync(&last_pos, d_pos.as<uint32_t>() + (n - 1), 4, cudaMemcpyDeviceToHost, st));
    BCUDA(cudaMemcpyAsync(&last_flag, d_flag.as<uint32_t>() + (n - 1), 4, cudaMemcpyDeviceToHost, st));
    BCUDA(cudaStreamSynchronize(st));
    n_unique = static_cast<uint64_t>(last_pos) + last_flag;
  }
  const size_t nu = n_unique ? n_unique : 1;
  // + 64: the check kernel streams rows with aligned 128-bit loads, which may read (and ignore) up to 12 bytes past a row
  // edge arrays of a large store get the growth headroom of the incremental publish from the start (see below)
  const size_t edge_bytes = static_cast<size_t>(nu) * 4 + 64,
               edge_cap = nu >= (1u << 20) ? edge_bytes + edge_bytes / 32 + (4u << 20) : edge_bytes;
  if (!s->col.ensure(edge_cap) || !s->rcol.ensure(edge_cap) || (with_exp && !s->exp.ensure(edge_cap)) ||
      !d_rkey[0].ensure(nu * 8) || !d_rkey[1].ensure(nu * 8) || !d_rres[0].ensure(nu * 4) || !d_rres[1].ensure(nu * 4))
    return "out of device memory (edge arrays)";
  if (n) {
    emit_kernel<<<grid, blk, 0, st>>>(d_key[0].as<unsigned long long>(), d_idx[0].as<uint32_t>(), d_flag.as<uint32_t>(),
                                      d_pos.as<uint32_t>(), n, d_t.as<zg_tuple>(), with_exp ? d_e.as<uint32_t>() : nullptr,
                                      d_slots.as<BSlot>(), d_cls.as<DCls>(), s->col.as<uint32_t>(),
                                      with_exp ? s->exp.as<uint32_t>() : nullptr, s->row_ptr.as<uint32_t>(),
                                      d_clscnt.as<uint32_t>(), d_rkey[0].as<unsigned long long>(), d_rres[0].as<uint32_t>(),
                                      s->rrow_ptr.as<uint32_t>());
    size_t tb = d_tmp.cap;
    BCUDA(cub::DeviceScan::InclusiveSum(d_tmp.p, tb, s->row_ptr.as<uint32_t>(), s->row_ptr.as<uint32_t>(), pool + 1, st));
    tb = d_tmp.cap;
    BCUDA(cub::DeviceScan::InclusiveSum(d_tmp.p, tb, s->rrow_ptr.as<uint32_t>(), s->rrow_ptr.as<uint32_t>(), rpool + 1, st));
  }
  if (n_unique) {
    // reverse CSR: entries are in (type, object, class) order, i.e. ascending resource within a
    // class; a stable sort by (class reverse base + subject) finishes the job
    size_t tb = 0;
    const int rbits = bits_for(rpool);
    cub::DeviceRadixSort::SortPairs(nullptr, tb, d_rkey[0].as<unsigned long long>(), d_rkey[1].as<unsigned long long>(),
                                    d_rres[0].as<uint32_t>(), s->rcol.as<uint32_t>(), n_unique, 0, rbits, st);
    if (!d_tmp.ensure(tb + 256)) return "out of device memory (sort scratch)";
    tb = d_tmp.cap;
    BCUDA(cub::DeviceRadixSort::SortPairs(d_tmp.p, tb, d_rkey[0].as<unsigned long long>(),
                                          d_rkey[1].as<unsigned long long>(), d_rres[0].as<uint32_t>(),
                                          s->rcol.as<uint32_t>(), n_unique, 0, rbits, st));
  }
  // classes that hold at least one relationship
  std::vector<uint32_t> cls_cnt(lay->cls.size() + 1, 0);
  BCUDA(cudaMemcpyAsync(cls_cnt.data(), d_clscnt.p, cls_cnt.size() * 4, cudaMemcpyDeviceToHost, st));
  BCUDA(cudaStreamSynchronize(st));
  for (size_t c = 0; c < lay->cls.size(); ++c)
    if (cls_cnt[c]) lay->cls[c].flags &= static_cast<uint16_t>(~CF_EMPTY);

  s->cls_count.assign(cls_cnt.begin(), cls_cnt.end() - 1);
  s->type_base = lay->type_base;
  s->type_ncls = lay->type_ncls;
  s->n_objects = lay->n_objects;
  s->delta_ok = true;
  if (nu >= (1u << 20)) {
    // The alternates of the incremental publish (merge_direction), with its headroom, come with the snapshot: the first
    // write after a bulk load must not pay for three store-sized allocations (hundreds of ms where cudaMalloc is slow).
    // That write still builds the host relationship index (Store::ensure_index), which a bulk load leaves stale.
    // Best effort: a failure here is met again, and reported, by the write that needs them.
    const size_t need = static_cast<size_t>(nu) * 4 + 64, roomy = need + need / 32 + (4u << 20);
    s->col_alt.ensure(roomy);
    s->rcol_alt.ensure(roomy);
    if (with_exp) s->exp_alt.ensure(roomy);
    cudaGetLastError();
  }
  {
    std::string rerr = gpu_resource_lists(s, st);
    if (!rerr.empty()) return rerr;
  }
  BCUDA(cudaGetLastError());
  lay->n_tuples = n_unique;
  s->n_tuples = n_unique;
  s->bytes += (pool + 1) * 4 + (rpool + 1) * 4 + n_unique * (with_exp ? 12 : 8);
  return "";
}


namespace {

// one direction (forward or reverse) of the merge
std::string merge_direction(const HostDelta& h, bool with_exp, DevBuf& row_ptr, uint64_t pool, DevBuf& edges, DevBuf& exp,
                            DevBuf& edges_alt, DevBuf& exp_alt, uint64_t n_old, cudaStream_t st, DevBuf& scratch,
                            uint32_t* d_bad) {
  const uint32_t ni = static_cast<uint32_t>(h.ins_key.size()), nd = static_cast<uint32_t>(h.del_key.size()),
                 nt = with_exp ? static_cast<uint32_t>(h.tch_key.size()) : 0u;
  const uint64_t n_new = n_old + ni - nd;
  if (n_new >= 0xFFFFFFF0ull) return "more than 2^32 relationships in one snapshot";
  // scratch layout (u64 keys first, then u32 arrays)
  const size_t keys = size_t(ni) + nd + nt;
  const size_t bytes = keys * 8 + (size_t(ni) * 3 + size_t(nd) * 2 + size_t(nt) * 3) * 4 + 64;
  if (!scratch.ensure(bytes)) return "out of device memory (delta scratch)";
  uint8_t* base = scratch.as<uint8_t>();
  auto* d_ins_key = reinterpret_cast<unsigned long long*>(base);
  auto* d_del_key = d_ins_key + ni;
  auto* d_tch_key = d_del_key + nd;
  auto* u32p = reinterpret_cast<uint32_t*>(d_tch_key + nt);
  uint32_t* d_ins_val = u32p; u32p += ni;
  uint32_t* d_ins_exp = u32p; u32p += ni;
  uint32_t* d_ins_pos = u32p; u32p += ni;
  uint32_t* d_del_val = u32p; u32p += nd;
  uint32_t* d_del_pos = u32p; u32p += nd;
  uint32_t* d_tch_val = u32p; u32p += nt;
  uint32_t* d_tch_exp = u32p; u32p += nt;
  uint32_t* d_tch_pos = u32p; u32p += nt;
  auto up = [&](void* dst, const void* src, size_t b) -> cudaError_t {
    return b ? cudaMemcpyAsync(dst, src, b, cudaMemcpyHostToDevice, st) : cudaSuccess;
  };
  BCUDA(up(d_ins_key, h.ins_key.data(), size_t(ni) * 8));
  BCUDA(up(d_del_key, h.del_key.data(), size_t(nd) * 8));
  BCUDA(up(d_ins_val, h.ins_val.data(), size_t(ni) * 4));
  BCUDA(up(d_del_val, h.del_val.data(), size_t(nd) * 4));
  if (with_exp) {
    BCUDA(up(d_ins_exp, h.ins_exp.data(), size_t(ni) * 4));
    BCUDA(up(d_tch_key, h.tch_key.data(), size_t(nt) * 8));
    BCUDA(up(d_tch_val, h.tch_val.data(), size_t(nt) * 4));
    BCUDA(up(d_tch_exp, h.tch_exp.data(), size_t(nt) * 4));
  }
  DeltaDev d{d_ins_key, d_ins_val, with_exp ? d_ins_exp : nullptr, d_ins_pos, ni, d_del_key, d_del_val, d_del_pos, nd,
             d_tch_key, d_tch_val, d_tch_exp, d_tch_pos, nt};
  const unsigned blk = 256;
  if (keys) delta_locate_kernel<<<static_cast<unsigned>((keys + blk - 1) / blk), blk, 0, st>>>(row_ptr.as<uint32_t>(),
                                                                                             edges.as<uint32_t>(), d, d_bad);
  if (ni || nd) {
    // headroom when the alternate has to grow (3 % + 4 MB): without it every write that adds edges re-allocates a
    // store-sized buffer, and a cudaMalloc / cudaFree of 400 MB can cost 100 ms
    const size_t need = std::max<uint64_t>(n_new, 1) * 4 + 64, roomy = need + need / 32 + (4u << 20);
    if (!edges_alt.ensure(edges_alt.cap < need ? roomy : need) || (with_exp && !exp_alt.ensure(exp_alt.cap < need ? roomy : need)))
      return "out of device memory (edge arrays)";
    if (n_old)
      delta_merge_kernel<<<static_cast<unsigned>((n_old + kMergeTile - 1) / kMergeTile), 256, 0, st>>>(
          edges.as<uint32_t>(), edges_alt.as<uint32_t>(), with_exp ? exp.as<uint32_t>() : nullptr,
          with_exp ? exp_alt.as<uint32_t>() : nullptr, static_cast<uint32_t>(n_old), d_ins_pos, ni, d_del_pos, nd);
    if (ni)
      delta_insert_kernel<<<(ni + blk - 1) / blk, blk, 0, st>>>(edges_alt.as<uint32_t>(), with_exp ? exp_alt.as<uint32_t>() : nullptr,
                                                              d_ins_pos, d_ins_val, with_exp ? d_ins_exp : nullptr, ni, d_del_pos, nd);
    if (nt)
      delta_touch_kernel<<<(nt + blk - 1) / blk, blk, 0, st>>>(exp_alt.as<uint32_t>(), d_tch_pos, d_tch_exp, nt, d_ins_pos, ni,
                                                             d_del_pos, nd);
    unsigned long long first = pool;
    if (ni) first = std::min<unsigned long long>(first, h.ins_key.front());
    if (nd) first = std::min<unsigned long long>(first, h.del_key.front());
    ++first;  // row_ptr[key] itself (the start of the first touched row) does not move
    if (first <= pool)
      delta_rows_kernel<<<static_cast<unsigned>((pool + 1 - first + kMergeTile - 1) / kMergeTile), 256, 0, st>>>(
          row_ptr.as<uint32_t>(), first, pool, d_ins_key, ni, d_del_key, nd);
    std::swap(edges, edges_alt);
    if (with_exp) std::swap(exp, exp_alt);
  } else if (nt) {
    // expirations only: patch in place (positions do not move)
    delta_touch_kernel<<<(nt + blk - 1) / blk, blk, 0, st>>>(exp.as<uint32_t>(), d_tch_pos, d_tch_exp, nt, d_ins_pos, 0, d_del_pos, 0);
  }
  BCUDA(cudaGetLastError());
  return "";
}

}  // namespace

std::string gpu_apply_delta(const Store& store, const Schema& sc, const HostSnapshot& lay, cudaStream_t st, Snapshot* s,
                            std::vector<uint32_t>* cls_delta, uint32_t owner_rank, uint32_t owner_count) {
  const bool with_exp = sc.has_expiry;
  HostDelta f, r;
  {
    std::string perr = prepare_delta(store, sc, lay, &f, &r, cls_delta, owner_rank, owner_count);
    if (!perr.empty()) return perr;
  }
  if (f.ins_key.empty() && f.del_key.empty() && f.tch_key.empty()) return "";
  static thread_local DevBuf scratch_f, scratch_r, bad;
  if (!bad.ensure(16)) return "out of device memory";
  BCUDA(cudaMemsetAsync(bad.p, 0, 16, st));
  const uint64_t n_old = s->n_tuples;
  DevBuf none1, none2;
  std::string err = merge_direction(f, with_exp, s->row_ptr, lay.pool, s->col, s->exp, s->col_alt, s->exp_alt, n_old, st,
                                    scratch_f, bad.as<uint32_t>());
  if (!err.empty()) return err;
  err = merge_direction(r, false, s->rrow_ptr, lay.rpool, s->rcol, none1, s->rcol_alt, none2, n_old, st, scratch_r,
                        bad.as<uint32_t>() + 1);
  if (!err.empty()) return err;
  uint32_t hb[2] = {0, 0};
  BCUDA(cudaMemcpyAsync(hb, bad.p, 8, cudaMemcpyDeviceToHost, st));
  BCUDA(cudaStreamSynchronize(st));
  if (hb[0] || hb[1]) return "corrupt";  // the resident snapshot disagrees with the store: rebuild it
  s->n_tuples = n_old + f.ins_key.size() - f.del_key.size();
  return "";
}

}  // namespace zg
