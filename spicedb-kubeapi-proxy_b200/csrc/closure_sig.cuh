// closure_sig.cuh -- the signature of a closure row: what build.cu writes at publish and kernels.cuh sig_meet tests.
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

}  // namespace zg
