// keytable.cuh -- the open-addressing table of 8-byte keys behind GROUP_IDS (colops.cu), the plan's CTA and global group tables (plan.cu),
// the join map (join.cu) and bloom test_and_add's scratch table (bloom.cu); and, at the end, the same slots over byte-string keys (STR_GROUP_IDS,
// STR_JOIN_FIND).
//
// A table of mask + 1 slots (a power of two) owns mask + 2 key slots.  A key starts at slot mix64(key) & mask and probes linearly, wrapping
// from the last slot to slot 0.  A slot is empty while it holds kEmptyKey (all ones), so a table is initialised by filling its key array with
// 0xff bytes.  A real key of all ones cannot live in a probe slot: it owns slot mask + 1, which holds all ones from initialisation, so
// inserting or finding it neither probes nor writes.  A table without that extra slot must keep the all-ones key away from it.
#pragma once
#include <stdint.h>
#include "xxh3_128.cuh"

namespace mob {

constexpr uint64_t kEmptyKey = 0xffffffffffffffffull;
constexpr uint64_t kNoSlot = 0xffffffffffffffffull;   // kt_insert_from: every slot holds another key

__device__ __forceinline__ uint64_t mix64(uint64_t x) {   // the murmur3 64-bit finalizer
    x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
    return x;
}

// the slot where key is or now is, probing from slot s (not the all-ones key); kNoSlot once all mask + 1 slots hold other keys
template <typename Slot>
__device__ __forceinline__ Slot kt_insert_from(uint64_t *keys, Slot mask, uint64_t key, Slot s) {
    for (Slot probes = 0; probes <= mask; probes++) {
        uint64_t cur = keys[s];
        if (cur == key) return s;
        if (cur == kEmptyKey) {
            cur = atomicCAS((unsigned long long *)&keys[s], (unsigned long long)kEmptyKey, (unsigned long long)key);
            if (cur == kEmptyKey || cur == key) return s;
        }
        s = (s + 1) & mask;
    }
    return (Slot)kNoSlot;
}

// slot = the key's slot, claimed if the key is new, and true; false once all mask + 1 slots hold other keys.  Slot is uint64_t, or unsigned
// for a table that small (the CTA table in shared memory: 32-bit slot arithmetic keeps its probe loop short).
template <typename Slot>
__device__ __forceinline__ bool kt_insert(uint64_t *keys, Slot mask, uint64_t key, Slot &slot) {
    if (key == kEmptyKey) { slot = mask + 1; return true; }
    slot = kt_insert_from(keys, mask, key, (Slot)mix64(key) & mask);
    return slot != (Slot)kNoSlot;
}

// slot = the key's slot and true, or false when the key is absent; never writes.  Stops at the first empty slot: the table must have one.
__device__ __forceinline__ bool kt_find(const uint64_t *keys, uint64_t mask, uint64_t key, uint64_t &slot) {
    if (key == kEmptyKey) { slot = mask + 1; return true; }
    for (uint64_t s = mix64(key) & mask;; s = (s + 1) & mask) {
        const uint64_t cur = keys[s];
        if (cur == key) { slot = s; return true; }
        if (cur == kEmptyKey) return false;
    }
}

// *first = min(*first, row).  The value only decreases, so a stale read can only be larger than the truth and skipping the atomic when it is
// already <= row is safe: after the first few rows of a group almost every row skips it.
__device__ __forceinline__ void first_row_min(unsigned long long *first, unsigned long long row) {
    if (*((volatile unsigned long long *)first) > row) atomicMin(first, row);
}

// ---- byte-string keys (STR_GROUP_IDS in colops.cu, STR_JOIN_FIND in join.cu) ----------------------------------------------------------------
// The same slots hold one word per key: (32-bit hash tag << 32) | virtual row, the row that owns the key's bytes.  Rows stay below 2^31, so no
// such word is kEmptyKey.  A key starts at slot hash & mask; where the tags match the two byte strings are compared, so keys are equal exactly
// when their bytes are.  The hash is XXH3 (xxh3_128.cuh), low 64 bits; hash_mask is all ones except under MoB200_SetTuning("strkey_hash_bits").
struct ByteKey { const uint8_t *p; uint64_t n; };

// virtual row v < nexist: key bytes [toff[v], toff[v + 1]) of tbytes (an existing group), else [koff[i], koff[i + 1]) of kbytes, i = v - nexist
struct StrKeys {
    const uint8_t *tbytes; const uint64_t *toff; const uint8_t *kbytes; const uint64_t *koff; uint64_t nexist;
    __device__ __forceinline__ ByteKey at(uint64_t v) const {
        if (v < nexist) return ByteKey{tbytes + toff[v], toff[v + 1] - toff[v]};
        const uint64_t i = v - nexist;
        return ByteKey{kbytes + koff[i], koff[i + 1] - koff[i]};
    }
};

__device__ __forceinline__ bool bytes_equal(ByteKey a, ByteKey b) {
    if (a.n != b.n) return false;
    for (uint64_t j = 0; j < a.n; j++) if (a.p[j] != b.p[j]) return false;
    return true;
}

__device__ __forceinline__ uint64_t str_hash(ByteKey k, uint64_t hash_mask) { return xxh3::hash_bytes(k.p, k.n, 0).lo & hash_mask; }
__device__ __forceinline__ uint64_t str_word(uint64_t h, uint64_t v) { return ((h >> 32) << 32) | v; }

// the slot of the key whose word is `word` (hash h), claimed if no slot holds an equal key; same(row) compares the key with that row's key.
// kNoSlot once all mask + 1 slots hold other keys.
template <class Same>
__device__ __forceinline__ uint64_t kt_insert_str(uint64_t *slots, uint64_t mask, uint64_t h, uint64_t word, Same same) {
    uint64_t s = h & mask;
    for (uint64_t probes = 0; probes <= mask; probes++) {
        uint64_t cur = slots[s];
        if (cur == kEmptyKey) {
            cur = atomicCAS((unsigned long long *)&slots[s], (unsigned long long)kEmptyKey, (unsigned long long)word);
            if (cur == kEmptyKey) return s;
        }
        if ((cur >> 32) == (word >> 32) && same((uint32_t)cur)) return s;
        s = (s + 1) & mask;
    }
    return kNoSlot;
}

// the row that owns the key (hash h) and true, or false when the key is absent; never writes.  The table must have an empty slot.
template <class Same>
__device__ __forceinline__ bool kt_find_str(const uint64_t *slots, uint64_t mask, uint64_t h, Same same, uint32_t &row) {
    for (uint64_t s = h & mask;; s = (s + 1) & mask) {
        const uint64_t cur = slots[s];
        if (cur == kEmptyKey) return false;
        if ((cur >> 32) == (h >> 32) && same((uint32_t)cur)) { row = (uint32_t)cur; return true; }
    }
}

}  // namespace mob
