// hash_bytes.h -- the hash of an object id's bytes, shared by the host interning tables (store.cc), the device
// mirror of those tables (ingress.cuh) and the CPU SIMT emulator: one definition, so a name hashes to the same slot
// on every side.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstring>

#if defined(__CUDACC__) || defined(ZG_EMULATE)
#define ZG_HD __host__ __device__
#else
#define ZG_HD
#endif

namespace zg {

constexpr uint64_t kHashSeed = 0x9E3779B97F4A7C15ull;
constexpr uint64_t kHashMul = 0xD6E8FEB86659FD93ull;

// Hash of n bytes given as little-endian 64-bit words: `word(j)` returns bytes [8j, 8j + 8) of the id, the bytes at
// or past n reading as zero. The host reads the words with memcpy, the device from its own word reader.
template <class Word>
ZG_HD inline uint64_t hash_words(size_t n, Word word) {
  uint64_t h = kHashSeed ^ (n * kHashMul);
  const size_t nw = (n + 7) / 8;
  for (size_t j = 0; j < nw; ++j) {
    h = (h ^ word(j)) * kHashMul;
    h ^= h >> 32;
  }
  h *= kHashSeed;
  return h ^ (h >> 29);
}

// Host form over a byte pointer (store.cc, little-endian hosts).
inline uint64_t hash_bytes(const char* s, size_t n) {
  return hash_words(n, [s, n](size_t j) {
    uint64_t w = 0;
    const size_t off = j * 8;
    if (n - off >= 8) std::memcpy(&w, s + off, 8);
    else std::memcpy(&w, s + off, n - off);
    return w;
  });
}

}  // namespace zg
