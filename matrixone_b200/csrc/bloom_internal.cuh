// bloom_internal.cuh -- the device side of the runtime bloom filter (bloom.cu) shared with its other readers (filtered search).
#pragma once
#include "common.cuh"
#include "xxh3_128.cuh"
#include "../../include/mo_b200_bloom.h"

namespace mob {

// device mirror of bf's bitmap, created and uploaded on first use (bloom.cu).  will_write marks the device copy as newer than the
// host bytes.  Returns nullptr (error set) on failure.
uint64_t *bloom_mirror(ThreadCtx &t, const bloomfilter_t *bf, bool will_write);

__device__ __forceinline__ xxh3::Hash128 bloom_key_hash(const uint8_t *p, size_t len, uint64_t seed) {
    // bloom_calculate_hash, bloom.c:43-66: narrow integers are widened so that equal values of different widths share their hash
    switch (len) {
    case 1: return xxh3::hash_u64((uint64_t)(int64_t)(int8_t)p[0], seed);
    case 2: return xxh3::hash_u64((uint64_t)(int64_t)(int16_t)((uint16_t)p[0] | ((uint16_t)p[1] << 8)), seed);
    case 4: return xxh3::hash_u64((uint64_t)(int64_t)(int32_t)xxh3::rd32(p), seed);
    case 8: return xxh3::hash_u64(xxh3::rd64(p), seed);
    default: return xxh3::hash_bytes(p, len, seed);
    }
}

// bloomfilter_test of one hashed key: all k positions (h.lo + i h.hi) & (nbits - 1) set
__device__ __forceinline__ bool bloom_test_hash(const uint64_t *__restrict__ bits, uint64_t nbits, uint32_t k, xxh3::Hash128 h) {
    bool all = true;   // (issuing all k probes before looking at any was measured: 6 % slower -- the early exit saves more sectors than the overlap gains)
    for (uint32_t j = 0; j < k && all; j++) {
        const uint64_t pos = (h.lo + (uint64_t)j * h.hi) & (nbits - 1);
        all = (__ldg(&bits[pos >> 6]) >> (pos & 63)) & 1ull;
    }
    return all;
}

}  // namespace mob
