// text_hash.cuh -- simeon's string hash and word-character rule, shared by the text encoder (simeon_encode.cu) and the BM25
// index (bm25.cu), on the host and on the device.
#pragma once
#include <stdint.h>

namespace yb {

// splitmix64_mix (simeon include/simeon/hasher.hpp:12-16)
__host__ __device__ __forceinline__ uint64_t sm64_mix(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
}

// the first state of splitmix64_hash for a seed
__host__ __device__ __forceinline__ uint64_t gram_hash_h0(uint64_t seed) { return sm64_mix(seed ^ 0x9E3779B97F4A7C15ULL); }

// ASCII lowercase (std::tolower in the "C" locale)
__host__ __device__ __forceinline__ uint8_t ascii_lower(uint8_t c) { return (c >= 'A' && c <= 'Z') ? (uint8_t)(c | 0x20) : c; }

// splitmix64_hash of k bytes at p (simeon src/hasher.cpp:33-47); h0 = gram_hash_h0(seed).  FOLD hashes the ASCII-lowercased
// bytes, as Bm25Index hashes its words and their n-grams (bm25.cpp:19-41).
template <bool FOLD = false>
__host__ __device__ __forceinline__ uint64_t gram_hash(const uint8_t* __restrict__ p, uint64_t k, uint64_t h0) {
    uint64_t h = h0;
    uint64_t i = 0;
    while (i + 8 <= k) {
        uint64_t chunk = 0;
#pragma unroll
        for (int b = 0; b < 8; ++b) chunk |= (uint64_t)(FOLD ? ascii_lower(p[i + b]) : p[i + b]) << (8 * b);
        h = sm64_mix(h ^ chunk);
        i += 8;
    }
    if (i < k) {
        uint64_t tail = 0;
        for (uint64_t j = 0; i + j < k; ++j) tail |= (uint64_t)(FOLD ? ascii_lower(p[i + j]) : p[i + j]) << (8 * j);
        tail ^= (uint64_t)(k - i) << 56;
        h = sm64_mix(h ^ tail);
    }
    return sm64_mix(h ^ k);
}

// std::isalnum in the "C" locale, or '_' (simeon src/tokenizer.cpp:13-15, src/bm25.cpp:103-105): bytes >= 0x80 separate words
__host__ __device__ __forceinline__ bool is_word_char(uint8_t c) {
    return (c >= '0' && c <= '9') || (c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z') || c == '_';
}

}  // namespace yb
