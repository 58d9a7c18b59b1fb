// gather.cuh — the row selection and column gathers shared by the join (join.cu) and the sort (sort.cu); the kernels and
// their host launchers live in gather.cu.
//
// Selection: the rows are cut into tiles of MARK_TILE; a mark kernel (mark_tiles) writes each tile's MARK_TILE / 32 pass
// bits as 32-bit mask words (warp w of the CTA writes words i * 8 + w, one __ballot_sync each) and its pass count; the
// counts are scanned into tile offsets; select_rows (k_join_select) writes the passing row numbers of each tile, in row
// order, at its offset.
// Gathers: gather_column copies one column by a u32 row-index list, keeping its dtype and validity: k_join_gather<T> (1,
// 2, 4, 8 bytes), k_join_gather_bits (validity and Boolean values), and gather_utf8 (utf8_gather.cu) for Utf8 columns.
#pragma once
#include "common.cuh"

namespace dfgpu {

constexpr int SEL_THREADS = 256;  // threads per CTA of the mark, select and gather kernels
constexpr int MARK_TILE = 2048;
constexpr int MARK_WORDS = MARK_TILE / 32;
constexpr int WARP_WORDS = MARK_WORDS / (SEL_THREADS / 32);  // mask words per warp and tile: 8

template <class Pass>
__device__ __forceinline__ void mark_tiles(long long n, unsigned* __restrict__ mask, unsigned* __restrict__ tile_cnt, Pass pass) {
  __shared__ unsigned s_cnt[SEL_THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long ntiles = (n + MARK_TILE - 1) / MARK_TILE;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    unsigned c = 0;
#pragma unroll 1
    for (int i = 0; i < MARK_TILE / SEL_THREADS; i++) {
      const long long r = tile * MARK_TILE + i * SEL_THREADS + threadIdx.x;
      const unsigned w = __ballot_sync(0xffffffffu, r < n && pass(r));
      c += (unsigned)__popc(w);
      if (lane == 0) mask[r >> 5] = w;
    }
    if (lane == 0) s_cnt[warp] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned total = 0;
      for (int w = 0; w < SEL_THREADS / 32; w++) total += s_cnt[w];
      tile_cnt[tile] = total;
    }
    __syncthreads();
  }
}

// The passing row numbers of the `ntiles` tiles of `mask`, in row order: tile t's at out[tile_off[t]..].  `grid` is the
// mark kernel's.
void select_rows(dfgpu_ctx* ctx, int grid, const unsigned* mask, long long ntiles, const unsigned long long* tile_off, unsigned* out);

// Gather one column by a row-index list.  `idx64` is filled on first use (Utf8 columns take 64-bit indices).
void gather_column(dfgpu_ctx* ctx, const DevColumn& src, const unsigned* idx, long long n, DevBufs& scratch, unsigned long long*& idx64,
                   unsigned long long* d_nulls, DevColumn* out);

}  // namespace dfgpu
