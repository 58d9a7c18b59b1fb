// hash_table.cuh — the open-addressed hash table rule shared by the aggregate's group table and pair sets
// (aggregate.cu) and the join's build table (join.cu): the empty-slot marker, the hash, the capacity and the
// probe sequence.  One definition, so that every table places and finds a 64-bit key the same way.
#pragma once
#include <algorithm>

#include "common.cuh"

namespace dfgpu {

// The marker of an empty slot.  The one key that equals it is kept in a separate slot (slot cap) by every table.
constexpr unsigned long long EMPTY_KEY = ~0ull;

__device__ __forceinline__ unsigned long long mix64(unsigned long long x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdull;
  x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull;
  x ^= x >> 33;
  return x;
}

// Capacity and probe sequence of the group table and of the COUNT(DISTINCT) pair sets: cap slots (a power of two), a
// hash's home slot is its TOP log2(cap) bits, and probing steps linearly, wrapping at cap.  The host fills both fields
// (set_cap); every kernel that places or looks up a key goes through home() and next().
struct ProbeRule {
  long long cap;
  int hshift;  // 64 - log2(cap)
  __host__ void set_cap(long long c) {
    int lg = 0;
    while ((1ll << lg) < c) lg++;
    cap = c;
    hshift = 64 - lg;
  }
  __device__ __forceinline__ unsigned long long home(unsigned long long hash) const { return hshift >= 64 ? 0ull : hash >> hshift; }
  __device__ __forceinline__ unsigned long long next(unsigned long long slot) const { return (slot + 1ull) & ((unsigned long long)cap - 1ull); }
};

inline long long next_pow2(long long x) {
  long long p = 1;
  while (p < x) p <<= 1;
  return p;
}

// Sizing policy of every table: a table for n entries has at least min_cap slots and at least twice n, rounded up to a
// power of two.
inline long long table_cap(long long n, long long min_cap) { return std::max(min_cap, next_pow2(2 * n)); }

}  // namespace dfgpu
