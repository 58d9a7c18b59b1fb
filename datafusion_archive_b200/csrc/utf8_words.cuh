// utf8_words.cuh — device reads of Utf8 bytes shared by the predicate kernels (utf8_predicate.cu), the string hash of
// GROUP BY keys (utf8_gather.cu) and the join's Utf8 keys (join.cu).
#pragma once
#include "common.cuh"

namespace dfgpu {

__device__ __forceinline__ unsigned fsr(unsigned lo, unsigned hi, int bits) { return __funnelshift_r(lo, hi, bits); }

// 16 bytes of a string, starting at byte q of a 16-byte aligned buffer, as four little-endian words.  `avail` >= 1 bytes
// from q belong to the string: the next aligned word is read only when those bytes reach into it.
__device__ __forceinline__ uint4 load16(const unsigned char* base, long long q, int avail) {
  const uint4* w = reinterpret_cast<const uint4*>(base + (q & ~15ll));
  const int sh = int(q & 15);
  const uint4 lo = __ldg(w);
  if (sh == 0) return lo;
  const uint4 hi = sh + min(avail, 16) > 16 ? __ldg(w + 1) : make_uint4(0u, 0u, 0u, 0u);
  const int b = (sh & 3) * 8;
  switch (sh >> 2) {
    case 0: return make_uint4(fsr(lo.x, lo.y, b), fsr(lo.y, lo.z, b), fsr(lo.z, lo.w, b), fsr(lo.w, hi.x, b));
    case 1: return make_uint4(fsr(lo.y, lo.z, b), fsr(lo.z, lo.w, b), fsr(lo.w, hi.x, b), fsr(hi.x, hi.y, b));
    case 2: return make_uint4(fsr(lo.z, lo.w, b), fsr(lo.w, hi.x, b), fsr(hi.x, hi.y, b), fsr(hi.y, hi.z, b));
    default: return make_uint4(fsr(lo.w, hi.x, b), fsr(hi.x, hi.y, b), fsr(hi.y, hi.z, b), fsr(hi.z, hi.w, b));
  }
}

// 64-bit FNV-1a over bytes [b, e), finalised with a 64-bit mixer: the hash of a Utf8 GROUP BY key and of a Utf8 join
// key part.  It reads byte by byte, so it does not depend on where the string starts.
__device__ __forceinline__ unsigned long long utf8_hash_bytes(const unsigned char* __restrict__ bytes, int b, int e) {
  unsigned long long h = 0xcbf29ce484222325ull;
  for (; b < e; b++) { h ^= bytes[b]; h *= 0x100000001b3ull; }
  h ^= h >> 32; h *= 0xd6e8feb86659fd93ull; h ^= h >> 32;
  return h;
}

}  // namespace dfgpu
