// gather.cu — see gather.cuh.
#include <algorithm>

#include "gather.cuh"

namespace dfgpu {

void gather_utf8(dfgpu_ctx* ctx, const DevColumn& src, const unsigned long long* d_idx, long long nsel, DevColumn* out);

// One tile per CTA iteration: each warp takes 8 of the tile's mask words; a prefix over the words' popcounts (within the
// warp, then over the warps) places each word's rows, and the lanes of a word write its set bits' row numbers together.
__global__ void __launch_bounds__(SEL_THREADS) k_join_select(const unsigned* __restrict__ mask, long long ntiles,
                                                            const unsigned long long* __restrict__ tile_off, unsigned* __restrict__ out) {
  __shared__ unsigned s_warp[SEL_THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned below = (1u << lane) - 1u;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long w0 = tile * MARK_WORDS + warp * WARP_WORDS;
    const unsigned word = lane < WARP_WORDS ? mask[w0 + lane] : 0u;
    const unsigned c = (unsigned)__popc(word);
    unsigned incl = c;
#pragma unroll
    for (int o = 1; o < WARP_WORDS; o <<= 1) {
      const unsigned x = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += x;
    }
    if (lane == WARP_WORDS - 1) s_warp[warp] = incl;
    __syncthreads();
    unsigned before = 0;
    for (int w = 0; w < warp; w++) before += s_warp[w];
    const unsigned long long at = tile_off[tile] + before;
#pragma unroll
    for (int j = 0; j < WARP_WORDS; j++) {
      const unsigned wj = __shfl_sync(0xffffffffu, word, j), ej = __shfl_sync(0xffffffffu, incl - c, j);
      if ((wj >> lane) & 1u) out[at + ej + (unsigned)__popc(wj & below)] = (unsigned)((w0 + j) * 32 + lane);
    }
    __syncthreads();
  }
}

template <class T>
__global__ void __launch_bounds__(SEL_THREADS) k_join_gather(const T* __restrict__ src, const unsigned* __restrict__ idx, long long n, T* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) out[i] = src[idx[i]];
}
// bit i of the output = bit idx[i] of src, written as whole 32-bit words; `zeros` (may be null) counts the zero bits
__global__ void __launch_bounds__(SEL_THREADS) k_join_gather_bits(const unsigned char* __restrict__ src, const unsigned* __restrict__ idx, long long n,
                                                                 unsigned* __restrict__ out, unsigned long long* __restrict__ zeros) {
  const long long padded = (n + 31) & ~31ll;
  unsigned long long z = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < padded; i += (long long)gridDim.x * blockDim.x) {
    bool bit = false;
    if (i < n) {
      const unsigned j = idx[i];
      bit = (src[j >> 3] >> (j & 7)) & 1;
    }
    const unsigned w = __ballot_sync(0xffffffffu, bit);
    if ((threadIdx.x & 31) == 0) {
      out[i >> 5] = w;
      const long long valid = min(32ll, n - i);
      z += (unsigned long long)(valid - __popc(w));
    }
  }
  if (zeros && z) atomicAdd(zeros, z);
}
__global__ void __launch_bounds__(SEL_THREADS) k_join_widen(const unsigned* __restrict__ idx, long long n, unsigned long long* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) out[i] = idx[i];
}

void select_rows(dfgpu_ctx* ctx, int grid, const unsigned* mask, long long ntiles, const unsigned long long* tile_off, unsigned* out) {
  launch(ctx, "k_join_select", k_join_select, grid, SEL_THREADS, PROFILED, mask, ntiles, tile_off, out);
}

void gather_column(dfgpu_ctx* ctx, const DevColumn& src, const unsigned* idx, long long n, DevBufs& scratch, unsigned long long*& idx64,
                   unsigned long long* d_nulls, DevColumn* out) {
  out->dtype = src.dtype;
  const int grid = grid_for(ctx, n, SEL_THREADS, 16);
  if (src.dtype == DFGPU_UTF8) {
    if (!idx64) {
      idx64 = scratch.alloc<unsigned long long>(size_t(std::max(1ll, n)) * sizeof(unsigned long long));
      if (n > 0) launch(ctx, "k_join_widen", k_join_widen, grid, SEL_THREADS, PROFILED, idx, n, idx64);
    }
    gather_utf8(ctx, src, idx64, n, out);
  } else if (src.dtype == DFGPU_BOOL) {
    out->values_bytes = size_t((n + 31) / 32) * 4 + 4;
    out->values = ctx->alloc(out->values_bytes);
    if (n > 0)
      launch(ctx, "k_join_gather_bits", k_join_gather_bits, grid, SEL_THREADS, PROFILED, (const unsigned char*)src.values, idx, n, (unsigned*)out->values,
             (unsigned long long*)nullptr);
    out->values_bytes = size_t(n + 7) / 8;
  } else {
    const int w = dtype_width(src.dtype);
    out->values_bytes = size_t(std::max(1ll, n)) * size_t(w);
    out->values = ctx->alloc(out->values_bytes);
    if (n > 0) {
      switch (w) {
        case 1: launch(ctx, "k_join_gather<1>", k_join_gather<unsigned char>, grid, SEL_THREADS, PROFILED, (const unsigned char*)src.values, idx, n, (unsigned char*)out->values); break;
        case 2: launch(ctx, "k_join_gather<2>", k_join_gather<unsigned short>, grid, SEL_THREADS, PROFILED, (const unsigned short*)src.values, idx, n, (unsigned short*)out->values); break;
        case 4: launch(ctx, "k_join_gather<4>", k_join_gather<unsigned>, grid, SEL_THREADS, PROFILED, (const unsigned*)src.values, idx, n, (unsigned*)out->values); break;
        default: launch(ctx, "k_join_gather<8>", k_join_gather<unsigned long long>, grid, SEL_THREADS, PROFILED, (const unsigned long long*)src.values, idx, n, (unsigned long long*)out->values); break;
      }
    }
  }
  if (src.null_count > 0 && src.validity && n > 0) {
    out->validity = (uint8_t*)ctx->alloc(size_t((n + 31) / 32) * 4);
    DF_CUDA(cudaMemsetAsync(d_nulls, 0, 8, ctx->stream));
    launch(ctx, "k_join_gather_bits", k_join_gather_bits, grid, SEL_THREADS, PROFILED, (const unsigned char*)src.validity, idx, n, (unsigned*)out->validity, d_nulls);
    set_null_count(ctx, *out, (int64_t)read_word(ctx, d_nulls));
  }
}

}  // namespace dfgpu
