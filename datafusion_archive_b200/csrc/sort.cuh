// sort.cuh — the stable LSD radix sort of u32 row ids shared by dfgpu_sort (sort.cu) and dfgpu_window (window.cu): the
// order-preserving key encoding (KeySrc, sort_key), the sort passes (Sorter, make_sorter) and the dense ranks of a Utf8
// column (utf8_rank).  sort.cu describes the passes.  Everything is in an anonymous namespace: each translation unit that
// includes it has its own copy of the kernels.
#pragma once
#include <algorithm>

#include "scan.cuh"

namespace dfgpu {
namespace {

constexpr int SORT_THREADS = 256;
constexpr int SORT_CHUNKS = 16;  // 256-row chunks per tile
constexpr int SORT_TILE = SORT_THREADS * SORT_CHUNKS;
constexpr int SORT_WARPS = SORT_THREADS / 32;

// What one sort key reads for row r
enum : int {
  KS_FIXED = 0,  // a numeric column of `dtype`
  KS_NULL = 1,   // the null bit of `valid`: null 0, valid 1 (null below every value)
  KS_WORD = 2,   // Utf8: bytes [8 * word, 8 * word + 8) as a big-endian word, zero-padded past the end
  KS_LEN = 3,    // Utf8: min(bytes left from byte 8 * word, 9)
  KS_RANK = 4    // the u32 at `vals`[r]
};
struct KeySrc {
  int kind;
  int dtype;
  int desc;
  int word;
  const void* vals;
  const unsigned char* valid;  // null: no nulls
  const int* off;
  const unsigned char* bytes;
};

__device__ __forceinline__ bool bit_at(const unsigned char* b, unsigned r) { return (b[r >> 3] >> (r & 7)) & 1; }

// key(r), order-preserving: integers by value, floats by the MIN / MAX accumulators' encoding (-0.0 below +0.0) with
// every NaN as the largest word, after +inf.  A null row (KS_FIXED / KS_RANK) encodes as 0; a null Utf8 as ''.
__device__ __forceinline__ unsigned long long sort_key(const KeySrc& s, unsigned r) {
  const bool valid = !s.valid || bit_at(s.valid, r);
  unsigned long long e = 0, ones = ~0ull;
  switch (s.kind) {
    case KS_NULL:
      e = valid ? 1ull : 0ull;
      ones = 0xffull;
      break;
    case KS_WORD:
    case KS_LEN: {
      const int b0 = valid ? s.off[r] : 0, len = valid ? s.off[r + 1] - b0 : 0, at = 8 * s.word;
      if (s.kind == KS_LEN) {
        e = (unsigned long long)min(max(len - at, 0), 9);
        ones = 0xffull;
      } else {
        for (int k = 0; k < 8; k++) e = (e << 8) | (at + k < len ? s.bytes[b0 + at + k] : 0u);
      }
      break;
    }
    case KS_RANK:
      e = valid ? ((const unsigned*)s.vals)[r] : 0u;
      ones = 0xffffffffull;
      break;
    default:
      if (valid) {
        switch (s.dtype) {
          case DFGPU_INT8: e = ((const unsigned char*)s.vals)[r] ^ 0x80u; break;
          case DFGPU_UINT8: e = ((const unsigned char*)s.vals)[r]; break;
          case DFGPU_INT16: e = ((const unsigned short*)s.vals)[r] ^ 0x8000u; break;
          case DFGPU_UINT16: e = ((const unsigned short*)s.vals)[r]; break;
          case DFGPU_INT32: e = ((const unsigned*)s.vals)[r] ^ 0x80000000u; break;
          case DFGPU_UINT32: e = ((const unsigned*)s.vals)[r]; break;
          case DFGPU_INT64: e = ((const unsigned long long*)s.vals)[r] ^ 0x8000000000000000ull; break;
          case DFGPU_FLOAT32: {
            const unsigned b = ((const unsigned*)s.vals)[r];
            e = (b & 0x7fffffffu) > 0x7f800000u ? 0xffffffffu : ((b >> 31) ? ~b : (b ^ 0x80000000u));
            break;
          }
          case DFGPU_FLOAT64: {
            const unsigned long long b = ((const unsigned long long*)s.vals)[r];
            e = (b & 0x7fffffffffffffffull) > 0x7ff0000000000000ull ? ~0ull : ((b >> 63) ? ~b : (b ^ 0x8000000000000000ull));
            break;
          }
          default: e = ((const unsigned long long*)s.vals)[r]; break;  // UInt64
        }
      }
      switch (s.dtype) {
        case DFGPU_INT8: case DFGPU_UINT8: ones = 0xffull; break;
        case DFGPU_INT16: case DFGPU_UINT16: ones = 0xffffull; break;
        case DFGPU_INT32: case DFGPU_UINT32: case DFGPU_FLOAT32: ones = 0xffffffffull; break;
        default: break;
      }
  }
  return s.desc ? (~e & ones) : e;
}

__global__ void __launch_bounds__(SORT_THREADS) k_sort_iota(long long n, unsigned* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) out[i] = (unsigned)i;
}

// keys[i] = key(perm[i]); or_and[0] |= every key, or_and[1] &= every key
template <class K>
__global__ void __launch_bounds__(SORT_THREADS) k_sort_encode(KeySrc s, const unsigned* __restrict__ perm, long long m, K* __restrict__ keys,
                                                             unsigned long long* __restrict__ or_and) {
  unsigned long long o = 0, a = ~0ull;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (long long)gridDim.x * blockDim.x) {
    const K e = (K)sort_key(s, perm[i]);
    keys[i] = e;
    o |= e;
    a &= e;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    o |= __shfl_xor_sync(0xffffffffu, o, d);
    a &= __shfl_xor_sync(0xffffffffu, a, d);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicOr(or_and, o);
    atomicAnd(or_and + 1, a);
  }
}

// counts[d * ntiles + t] = the rows of tile t whose digit (key >> shift) & 255 is d; the lanes of a warp with one digit
// add once
template <class K>
__global__ void __launch_bounds__(SORT_THREADS) k_sort_count(const K* __restrict__ keys, long long m, int shift, long long ntiles,
                                                            unsigned* __restrict__ counts) {
  __shared__ unsigned s_hist[256];
  const int lane = threadIdx.x & 31;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    s_hist[threadIdx.x] = 0;
    __syncthreads();
#pragma unroll 1
    for (int c = 0; c < SORT_CHUNKS; c++) {
      const long long i = tile * SORT_TILE + c * SORT_THREADS + threadIdx.x;
      const unsigned d = i < m ? (unsigned)((keys[i] >> shift) & 255u) : 256u;
      const unsigned peers = __match_any_sync(0xffffffffu, d);
      if (d < 256u && lane == __ffs(peers) - 1) atomicAdd(&s_hist[d], (unsigned)__popc(peers));
    }
    __syncthreads();
    counts[(long long)threadIdx.x * ntiles + tile] = s_hist[threadIdx.x];
    __syncthreads();
  }
}

// Stable scatter of one pass: offs[d * ntiles + t] (the scanned counts) is where tile t's rows of digit d start.  Each
// 256-row chunk is placed after the chunks before it; within a chunk, warp w's rows of digit d after those of warps < w,
// and a warp's rows in lane order.
template <class K>
__global__ void __launch_bounds__(SORT_THREADS) k_sort_scatter(const K* __restrict__ kin, const unsigned* __restrict__ pin, long long m, int shift,
                                                              long long ntiles, const unsigned* __restrict__ offs, K* __restrict__ kout,
                                                              unsigned* __restrict__ pout) {
  __shared__ unsigned s_base[256];
  __shared__ unsigned s_warp[SORT_WARPS][256];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned below = (1u << lane) - 1u;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    s_base[threadIdx.x] = offs[(long long)threadIdx.x * ntiles + tile];
    for (int w = 0; w < SORT_WARPS; w++) s_warp[w][threadIdx.x] = 0;
    __syncthreads();
#pragma unroll 1
    for (int c = 0; c < SORT_CHUNKS; c++) {
      const long long i = tile * SORT_TILE + c * SORT_THREADS + threadIdx.x;
      K k = 0;
      unsigned p = 0, d = 256u;
      if (i < m) {
        k = kin[i];
        p = pin[i];
        d = (unsigned)((k >> shift) & 255u);
      }
      const unsigned peers = __match_any_sync(0xffffffffu, d);
      if (d < 256u && lane == __ffs(peers) - 1) s_warp[warp][d] = (unsigned)__popc(peers);
      __syncthreads();
      unsigned run = s_base[threadIdx.x];  // digit threadIdx.x: each warp's start in this chunk
      for (int w = 0; w < SORT_WARPS; w++) {
        const unsigned x = s_warp[w][threadIdx.x];
        s_warp[w][threadIdx.x] = run;
        run += x;
      }
      s_base[threadIdx.x] = run;
      __syncthreads();
      if (d < 256u) {
        const unsigned pos = s_warp[warp][d] + (unsigned)__popc(peers & below);
        kout[pos] = k;
        pout[pos] = p;
      }
      __syncthreads();
      for (int w = 0; w < SORT_WARPS; w++) s_warp[w][threadIdx.x] = 0;
      __syncthreads();
    }
  }
}

// Utf8 ranks, after round `word` has sorted perm by (segment, word, length term): flags[i] = 1 where position i starts a
// new tie segment; *more = 1 when a tied row has bytes left past this word
__global__ void __launch_bounds__(SORT_THREADS) k_sort_seg_flags(KeySrc w, KeySrc l, const unsigned* __restrict__ seg, const unsigned* __restrict__ perm,
                                                                long long m, unsigned* __restrict__ flags, unsigned long long* __restrict__ more) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (long long)gridDim.x * blockDim.x) {
    const unsigned r = perm[i];
    const unsigned long long len = sort_key(l, r);
    unsigned f = 1;
    if (i > 0) {
      const unsigned q = perm[i - 1];
      f = seg[r] != seg[q] || sort_key(w, r) != sort_key(w, q) || len != sort_key(l, q);
    }
    flags[i] = f;
    if (!f && len == 9) *more = 1;
  }
}

// seg[perm[i]] = the segment of position i: the inclusive scan of the flags, less one
__global__ void __launch_bounds__(SORT_THREADS) k_sort_seg_write(const unsigned* __restrict__ perm, long long m, const unsigned* __restrict__ flags,
                                                                const unsigned* __restrict__ excl, unsigned* __restrict__ seg) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (long long)gridDim.x * blockDim.x)
    seg[perm[i]] = excl[i] + flags[i] - 1u;
}


// A permutation of m row ids being sorted key by key: perm[cur] is the current order.  The key and count buffers are
// shared by every sort that runs one after the other.
struct Sorter {
  dfgpu_ctx* ctx;
  long long m, ntiles;
  unsigned* perm[2];
  int cur;
  void* keys[2];              // m words of up to 8 bytes each
  unsigned* counts;           // 256 * ntiles + 1
  unsigned long long* or_and;  // 2 words

  // sort perm[cur] stably by `s`, a key of sizeof(K) bytes
  template <class K>
  void by(const KeySrc& s) {
    const unsigned long long init[2] = {0ull, ~0ull};
    DF_CUDA(cudaMemcpyAsync(or_and, init, sizeof(init), cudaMemcpyHostToDevice, ctx->stream));
    K* kin = (K*)keys[0];
    K* kout = (K*)keys[1];
    launch(ctx, "k_sort_encode", k_sort_encode<K>, grid_for(ctx, m, SORT_THREADS, 16), SORT_THREADS, PROFILED, s, (const unsigned*)perm[cur], m, kin,
           or_and);
    unsigned long long h[2];
    read_words(ctx, or_and, sizeof(h), h);  // also orders `init` before its stack frame goes
    const unsigned long long varying = h[0] ^ h[1];
    const int grid = grid_for(ctx, m, SORT_TILE, 8);
    for (int d = 0; d < int(sizeof(K)); d++) {
      if (((varying >> (8 * d)) & 255u) == 0) continue;  // the same digit in every row: the pass would not move a row
      launch(ctx, "k_sort_count", k_sort_count<K>, grid, SORT_THREADS, PROFILED, (const K*)kin, m, 8 * d, ntiles, counts);
      scan_exclusive<unsigned, unsigned>(ctx, counts, counts, 256 * ntiles, true);
      launch(ctx, "k_sort_scatter", k_sort_scatter<K>, grid, SORT_THREADS, PROFILED, (const K*)kin, (const unsigned*)perm[cur], m, 8 * d, ntiles,
             (const unsigned*)counts, kout, perm[cur ^ 1]);
      std::swap(kin, kout);
      cur ^= 1;
    }
  }
  void by_width(int w, const KeySrc& s) {
    switch (w) {
      case 1: by<unsigned char>(s); break;
      case 2: by<unsigned short>(s); break;
      case 4: by<unsigned>(s); break;
      default: by<unsigned long long>(s); break;
    }
  }
};

Sorter make_sorter(dfgpu_ctx* ctx, long long m, DevBufs& scratch) {
  Sorter S{};
  S.ctx = ctx;
  S.m = m;
  S.ntiles = (m + SORT_TILE - 1) / SORT_TILE;
  for (int i = 0; i < 2; i++) {
    S.perm[i] = scratch.alloc<unsigned>(size_t(std::max(1ll, m)) * 4);
    S.keys[i] = scratch.alloc<void>(size_t(std::max(1ll, m)) * 8);
  }
  S.counts = scratch.alloc<unsigned>(size_t(256 * S.ntiles + 1) * 4);
  S.or_and = scratch.alloc<unsigned long long>(16);
  return S;
}

// The dense rank of each kept row's string (rows[0..m) of column c, nulls as ''), in Utf8 order: equal strings share a
// rank.  MSD rounds over 8-byte words: round j sorts the rows by (tie segment, word j, bytes left from byte 8j capped
// at 9) and splits the segments where that differs; the length term puts 'a' before 'a\0', whose padded words are
// equal.  It stops when no two rows tie or no tied row has bytes left.  rank has a word for each of the n input rows.
void utf8_rank(Sorter& L, const DevColumn& c, const unsigned char* valid, long long n, DevBufs& scratch, unsigned* rank) {
  dfgpu_ctx* ctx = L.ctx;
  const long long m = L.m;
  Sorter S = L;  // the key and count buffers are shared; the permutation is this sort's own
  S.perm[0] = scratch.alloc<unsigned>(size_t(m) * 4);
  S.perm[1] = scratch.alloc<unsigned>(size_t(m) * 4);
  S.cur = 0;
  DF_CUDA(cudaMemcpyAsync(S.perm[0], L.perm[L.cur], size_t(m) * 4, cudaMemcpyDeviceToDevice, ctx->stream));
  DF_CUDA(cudaMemsetAsync(rank, 0, size_t(n) * 4, ctx->stream));  // segment 0 for every kept row
  unsigned* flags = scratch.alloc<unsigned>(size_t(m) * 4);
  unsigned* excl = scratch.alloc<unsigned>(size_t(m + 1) * 4);
  unsigned long long* more = scratch.alloc<unsigned long long>(8);
  const int grid = grid_for(ctx, m, SORT_THREADS, 16);
  for (int j = 0;; j++) {
    const KeySrc w{KS_WORD, DFGPU_UTF8, 0, j, nullptr, valid, c.offsets, (const unsigned char*)c.values};
    KeySrc l = w;
    l.kind = KS_LEN;
    const KeySrc seg{KS_RANK, DFGPU_UINT32, 0, 0, rank, nullptr, nullptr, nullptr};
    S.by<unsigned char>(l);
    S.by<unsigned long long>(w);
    if (j > 0) S.by<unsigned>(seg);
    DF_CUDA(cudaMemsetAsync(more, 0, 8, ctx->stream));
    launch(ctx, "k_sort_seg_flags", k_sort_seg_flags, grid, SORT_THREADS, PROFILED, w, l, (const unsigned*)rank, (const unsigned*)S.perm[S.cur], m,
           flags, more);
    const unsigned long long segments = scan_exclusive<unsigned, unsigned>(ctx, flags, excl, m, true);
    launch(ctx, "k_sort_seg_write", k_sort_seg_write, grid, SORT_THREADS, PROFILED, (const unsigned*)S.perm[S.cur], m, (const unsigned*)flags,
           (const unsigned*)excl, rank);
    if (segments == (unsigned long long)m || read_word(ctx, more) == 0) return;
  }
}


}  // namespace
}  // namespace dfgpu
