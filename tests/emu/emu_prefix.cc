// emu_prefix.cc -- the resource id prefix scan (spicedb-kubeapi-proxy_b200/csrc/ingress.cuh prefix_match_kernel) under
// the CPU SIMT emulator. TEST INFRASTRUCTURE ONLY (built by tests/test_prefix_emulation.py into its own .so; never part
// of libzgpu.so). The caller hands in one type's arena as the device mirror holds it (records [u32 id][u32 len][bytes]
// back to back) with its record offsets; the arena's last byte sits just before a PROT_NONE page, so a read past the
// last record faults.
#define ZG_EMULATE 1
#include "cuda_emu.h"

// ingress.cuh's insert kernel claims 64-bit slots; cuda_emu.h has the 32-bit atomicCAS only.
static inline unsigned long long atomicCAS(unsigned long long* p, unsigned long long expected, unsigned long long desired) {
  __atomic_compare_exchange_n(p, &expected, desired, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
  return expected;
}

#include <sys/mman.h>
#include <unistd.h>

#include <cstring>
#include <vector>

#include "../../spicedb-kubeapi-proxy_b200/csrc/ingress.cuh"

using namespace zg;

extern "C" {

// Runs the kernel over the arena (copied so that it ends at a guard page: the caller varies its records' alignment by
// its length) and the prefix. bits: ceil(n_ids / 32) words, zeroed here. Returns the kernel's match count, or -1 when
// the guard page is unavailable.
long long emu_prefix_scan(const char* arena, uint64_t bytes, const uint64_t* offs, uint64_t n_recs, uint32_t n_ids,
                          const char* prefix, uint64_t len, uint32_t* bits, unsigned grid, unsigned threads) {
  const size_t pg = static_cast<size_t>(sysconf(_SC_PAGESIZE));
  const size_t body = (bytes + pg - 1) / pg * pg + pg;
  char* m = static_cast<char*>(mmap(nullptr, body + pg, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0));
  if (m == MAP_FAILED) return -1;
  if (mprotect(m + body, pg, PROT_NONE) != 0) return -1;
  char* a = m + body - bytes;
  std::memcpy(a, arena, bytes);
  std::vector<uint64_t> pfx((len + 7) / 8 + 1, 0);
  std::memcpy(pfx.data(), prefix, len);
  std::vector<unsigned long long> o(offs, offs + n_recs);
  std::memset(bits, 0, ((uint64_t(n_ids) + 31) / 32) * 4);
  unsigned long long matched = 0;
  PrefixPlan p{};
  p.prefix = reinterpret_cast<const uint8_t*>(pfx.data());
  p.len = len;
  p.matched = &matched;
  p.n_types = 1;
  p.type[0].arena = reinterpret_cast<const uint8_t*>(a);
  p.type[0].offs = o.data();
  p.type[0].n_recs = n_recs;
  p.type[0].bits = bits;
  p.type[0].n_ids = n_ids;
  zg_emu::launch(prefix_match_kernel, p, grid, threads, 0);
  munmap(m, body + pg);
  return static_cast<long long>(matched);
}

}  // extern "C"
