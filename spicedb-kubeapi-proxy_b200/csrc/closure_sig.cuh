// closure_sig.cuh -- the signature and the set table of a closure row: what build.cu writes at publish and kernels.cuh
// sig_meet reads.
#pragma once
#include <cstdint>

namespace zg {

// Signature of a closure row (built at publish, build.cu): a blocked Bloom filter of 2^lg 64-bit words. Entry v sets
// three bits of one word: h = v * 0x9E3779B1, word h >> (32 - lg), bits h[0:6), h[6:12), h[12:18). A test is one 8-byte
// load and one AND; it says "maybe" for every entry of the row.
__host__ __device__ __forceinline__ uint32_t sig_word(uint32_t v, uint32_t lg) {
  const uint32_t h = v * 0x9E3779B1u;
  return lg ? h >> (32u - lg) : 0u;
}
__host__ __device__ __forceinline__ unsigned long long sig_mask(uint32_t v) {
  const uint32_t h = v * 0x9E3779B1u;
  return (1ull << (h & 63u)) | (1ull << ((h >> 6) & 63u)) | (1ull << ((h >> 12) & 63u));
}

// Hashed copy of a 16-bit closure row (the set table, built at publish when the target type holds fewer than 65 536
// objects, so that no entry is 0xFFFF): nb 8-byte buckets of four 16-bit slots, entry v in bucket
// table_bucket(v, seed, nb), each bucket's entries ascending from slot 0 and its empty slots 0xFFFF. nb and the seed
// are chosen per row so that no bucket gets more than four entries (build.cu closure_table_kernel), which makes a
// lookup exact: v is in the row iff a slot of its bucket holds v (sig_meet confirms its "maybe"s this way). The row's
// header is one 64-bit word: its first bucket (32 bits), nb (24 bits) and the seed (8 bits).
constexpr uint32_t kTableSlots = 4;
constexpr uint32_t kTableSeeds = 32;          // seeds tried per bucket count before the count grows by about 1/8
constexpr uint32_t kTableMaxBuckets = 8192;   // buckets of the largest row the build takes (its per-warp histogram)
__host__ __device__ __forceinline__ uint32_t table_hash(uint32_t v, uint32_t seed) {
  uint32_t h = (v + seed * 0x9E3779B9u) * 0x85EBCA6Bu;
  h ^= h >> 15;
  h *= 0x2C1B3C6Du;
  return h ^ (h >> 12);
}
__host__ __device__ __forceinline__ uint32_t table_bucket(uint32_t v, uint32_t seed, uint32_t nb) {
  const uint64_t p = static_cast<uint64_t>(table_hash(v, seed)) * nb;  // (the multiply-high: nb need not be a power of two)
  return static_cast<uint32_t>(p >> 32);
}
// the first bucket count tried for a row of len entries (mean occupancy 2), and the next after a failed seed budget
__host__ __device__ __forceinline__ uint32_t table_first_nb(uint32_t len) { return (len + 1) / 2; }
__host__ __device__ __forceinline__ uint32_t table_grow_nb(uint32_t nb) { return nb + (nb + 7) / 8; }
__host__ __device__ __forceinline__ unsigned long long table_header(uint32_t off, uint32_t nb, uint32_t seed) {
  return off | (static_cast<unsigned long long>(nb) << 32) | (static_cast<unsigned long long>(seed) << 56);
}
// Does the bucket word w hold v (v < 0xFFFF)? (a 16-bit lane of w ^ v x 0x0001000100010001 is zero)
__host__ __device__ __forceinline__ bool table_has(unsigned long long w, uint32_t v) {
  const unsigned long long x = w ^ (static_cast<unsigned long long>(v) * 0x0001000100010001ull);
  return ((x - 0x0001000100010001ull) & ~x & 0x8000800080008000ull) != 0;
}

// Range record of one object in one edge class (build.cu gpu_build_flat_records; kernels.cuh flat_check_kernel): the
// object's range col[row_ptr[row], row_ptr[row + 1]) copied into a fixed-stride record of kRecSlots 16-bit slots at
// rec + obj * kRecSlots. Slot 0 holds the range's length n, slots 1 .. n its children in CSR order, the rest 0xFFFF. A
// range longer than kRecSlots - 1 has kRecLong in slot 0 and is read from the CSR. The children are objects of a meet's
// target type, which has fewer than 65 536 objects wherever set tables exist.
#ifndef ZG_FLAT_RECORD_SLOTS
#define ZG_FLAT_RECORD_SLOTS 32  // 64-byte records (32-byte records, 15 inline children: 16)
#endif
constexpr uint32_t kRecSlots = ZG_FLAT_RECORD_SLOTS;
constexpr uint32_t kRecLong = 0xFFFFu;
static_assert(kRecSlots == 16 || kRecSlots == 32, "records of 32 or 64 bytes");

}  // namespace zg
