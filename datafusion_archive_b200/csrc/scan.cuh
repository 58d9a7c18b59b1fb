// scan.cuh — exclusive prefix sum of a device array: out[i] = in[0] + ... + in[i - 1] and out[n] = the total, summed in
// 64 bits.  Three launches: one CTA scans each 2048-element tile and writes the tile's total, one 1024-thread CTA scans
// the tile totals, and each tile adds its offset.  `in` and `out` may be the same array: every thread reads its elements
// before it writes them, and no thread touches another's.
#pragma once
#include <algorithm>

#include "common.cuh"

namespace dfgpu {
namespace {

constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 8;
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

template <class In, class Out>
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_tiles(const In* in, long long n, Out* out, unsigned long long* sums) {
  __shared__ unsigned long long s_warp[SCAN_THREADS / 32];
  const long long base = (long long)blockIdx.x * SCAN_TILE + (long long)threadIdx.x * SCAN_ITEMS;
  unsigned long long v[SCAN_ITEMS];
  unsigned long long run = 0;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; i++) {
    v[i] = run;  // exclusive within the thread
    run += base + i < n ? (unsigned long long)in[base + i] : 0ull;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long incl = run;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long x = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += x;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  unsigned long long excl = incl - run;
  for (int w = 0; w < warp; w++) excl += s_warp[w];
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; i++)
    if (base + i < n) out[base + i] = Out(v[i] + excl);  // tile-local; k_scan_add finishes it
  if (threadIdx.x == SCAN_THREADS - 1) sums[blockIdx.x] = excl + run;
}

// one CTA: exclusive scan of the nb tile totals in place; their total goes to sums[nb]
__global__ void __launch_bounds__(1024) k_scan_totals(unsigned long long* sums, long long nb) {
  __shared__ unsigned long long s_part[1024];
  const long long per = (nb + 1023) / 1024, lo = (long long)threadIdx.x * per, hi = min(nb, lo + per);
  unsigned long long acc = 0;
  for (long long b = lo; b < hi; b++) acc += sums[b];
  s_part[threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long run = 0;
    for (int i = 0; i < 1024; i++) {
      const unsigned long long x = s_part[i];
      s_part[i] = run;
      run += x;
    }
    sums[nb] = run;
  }
  __syncthreads();
  unsigned long long run = s_part[threadIdx.x];
  for (long long b = lo; b < hi; b++) {
    const unsigned long long x = sums[b];
    sums[b] = run;
    run += x;
  }
}

template <class Out>
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_add(Out* out, long long n, const unsigned long long* sums) {
  const unsigned long long add = sums[blockIdx.x];
  const long long base = (long long)blockIdx.x * SCAN_TILE;
  for (int i = threadIdx.x; i < SCAN_TILE; i += SCAN_THREADS)
    if (base + i < n) out[base + i] = Out(out[base + i] + add);
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) out[n] = Out(sums[gridDim.x]);
}

template <class T>
struct ScanType;
template <>
struct ScanType<int> {
  static constexpr const char* name = "i32";
};
template <>
struct ScanType<unsigned> {
  static constexpr const char* name = "u32";
};
template <>
struct ScanType<unsigned long long> {
  static constexpr const char* name = "u64";
};

// out[0..n] = the exclusive scan of in[0..n) with out[n] = the total, which is returned in 64 bits.  Synchronises the
// stream.
template <class In, class Out>
unsigned long long scan_exclusive(dfgpu_ctx* ctx, const In* in, Out* out, long long n, bool profiled) {
  static const std::string tiles = std::string("k_scan_tiles<") + ScanType<In>::name + ", " + ScanType<Out>::name + ">";
  static const std::string add = std::string("k_scan_add<") + ScanType<Out>::name + ">";
  const long long nb = std::max(1ll, (n + SCAN_TILE - 1) / SCAN_TILE);
  unsigned long long* sums = (unsigned long long*)ctx->alloc(size_t(nb + 1) * 8);
  const LaunchOpts opts{0, profiled};
  launch(ctx, tiles.c_str(), k_scan_tiles<In, Out>, int(nb), SCAN_THREADS, opts, in, n, out, sums);
  launch(ctx, "k_scan_totals", k_scan_totals, 1, 1024, opts, sums, nb);
  launch(ctx, add.c_str(), k_scan_add<Out>, int(nb), SCAN_THREADS, opts, out, n, (const unsigned long long*)sums);
  const unsigned long long total = read_word(ctx, sums + nb);
  ctx->free(sums);
  return total;
}

}  // namespace
}  // namespace dfgpu
