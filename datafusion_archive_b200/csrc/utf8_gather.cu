// utf8_gather.cu — order-preserving gather of a Utf8 (arrow 0.12 BinaryArray: i32 offsets + bytes)
// column by a list of selected row numbers.  Replaces the Utf8 arm of `fn filter`
// (src/execution/filter.rs:93-103: per-row String allocation + BinaryArray::from(Vec<&str>)).
// The row numbers come out of the fused filter kernel as one more projected column (V_PUSH_ROWID).
#include "utf8_words.cuh"

namespace dfgpu {

constexpr int SC_THREADS = 256;
constexpr int SC_ITEMS = 16;
constexpr int SC_TILE = SC_THREADS * SC_ITEMS;

// A gather index addresses (source, row): source = idx >> UTF8_SRC_SHIFT.  The filter path has one
// source (the batch's column); Utf8 GROUP BY keys gather representatives from every batch seen.
__device__ __forceinline__ const Utf8Source& src_of(const Utf8Source* srcs, unsigned long long idx, long long* row) {
  *row = (long long)(idx & ((1ull << UTF8_SRC_SHIFT) - 1ull));
  return srcs[idx >> UTF8_SRC_SHIFT];
}

// lengths of the selected strings, written to out[i + 1] (out[0] = 0 is set by the host)
__global__ void k_utf8_lengths(const unsigned long long* __restrict__ idx, const Utf8Source* __restrict__ srcs, long long n, int* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    long long r;
    const Utf8Source& s = src_of(srcs, idx[i], &r);
    out[i + 1] = s.off[r + 1] - s.off[r];
  }
}

// in-place inclusive scan, three launches: per-block scan + block totals, scan of totals, add-back
__global__ void __launch_bounds__(SC_THREADS) k_scan_block(int* __restrict__ a, long long n, long long* __restrict__ sums) {
  __shared__ long long s_warp[SC_THREADS / 32];
  const long long base = (long long)blockIdx.x * SC_TILE + (long long)threadIdx.x * SC_ITEMS;
  long long v[SC_ITEMS];
  long long run = 0;
#pragma unroll
  for (int k = 0; k < SC_ITEMS; k++) {
    v[k] = base + k < n ? (long long)a[base + k] : 0;
    run += v[k];
    v[k] = run;
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long incl = run;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  long long wbase = 0;
  for (int w = 0; w < warp; w++) wbase += s_warp[w];
  const long long excl = wbase + incl - run;
#pragma unroll
  for (int k = 0; k < SC_ITEMS; k++)
    if (base + k < n) a[base + k] = (int)(v[k] + excl);  // block-local; the add-back finishes it
  if (threadIdx.x == SC_THREADS - 1) sums[blockIdx.x] = excl + run;
}
__global__ void k_scan_sums(long long* sums, long long nblocks) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    long long run = 0;
    for (long long b = 0; b < nblocks; b++) {
      run += sums[b];
      sums[b] = run;
    }
  }
}
__global__ void __launch_bounds__(SC_THREADS) k_scan_add(int* __restrict__ a, long long n, const long long* __restrict__ sums) {
  if (blockIdx.x == 0) return;
  const long long add = sums[blockIdx.x - 1];
  const long long base = (long long)blockIdx.x * SC_TILE;
  for (int k = threadIdx.x; k < SC_TILE; k += SC_THREADS)
    if (base + k < n) a[base + k] = (int)((long long)a[base + k] + add);
}

// one warp per selected row: copy its bytes
__global__ void k_utf8_copy(const unsigned long long* __restrict__ idx, const Utf8Source* __restrict__ srcs, long long n,
                            const int* __restrict__ new_off, unsigned char* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long i = warp0; i < n; i += nwarps) {
    long long r;
    const Utf8Source& sc = src_of(srcs, idx[i], &r);
    const int s = sc.off[r], len = sc.off[r + 1] - s, d = new_off[i];
    for (int b = lane; b < len; b += 32) out[d + b] = sc.bytes[s + b];
  }
}

// 64-bit FNV-1a over each string, finalised with a 64-bit mixer: the GROUP BY key of a Utf8 column
__global__ void k_utf8_hash(const int* __restrict__ off, const unsigned char* __restrict__ bytes, long long n, unsigned long long* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int e = off[i + 1];
    out[i] = utf8_hash_bytes(bytes, off[i], e);
  }
}

void gather_utf8_multi(dfgpu_ctx* ctx, const Utf8Source* d_srcs, const unsigned long long* d_idx, long long nsel, DevColumn* out);

// gather `src` (Utf8) by `d_idx[0..nsel)` into `out`.  Synchronises the stream (byte count).
void gather_utf8(dfgpu_ctx* ctx, const DevColumn& src, const unsigned long long* d_idx, long long nsel, DevColumn* out) {
  Utf8Source h{src.offsets, (const unsigned char*)src.values};
  Utf8Source* d = (Utf8Source*)ctx->alloc(sizeof(Utf8Source));
  DF_CUDA(cudaMemcpyAsync(d, &h, sizeof(h), cudaMemcpyHostToDevice, ctx->stream));
  DF_CUDA(cudaStreamSynchronize(ctx->stream));  // `h` is a stack object
  gather_utf8_multi(ctx, d, d_idx, nsel, out);
  ctx->free(d);
}

// offsets[i] -= lo: a batch that is a slice of a longer Utf8 column uploads only its own bytes [lo, hi)
__global__ void k_rebase_offsets(int* __restrict__ off, long long n, int lo) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) off[i] -= lo;
}
void rebase_offsets(dfgpu_ctx* ctx, int* d_off, long long n, int lo) {
  if (n <= 0 || lo == 0) return;
  long long g = (n + 255) / 256;
  if (g > 4096) g = 4096;
  k_rebase_offsets<<<(unsigned)g, 256, 0, ctx->stream>>>(d_off, n, lo);
  DF_CUDA(cudaGetLastError());
  ctx->launches++;
}

// dst[i] = src[i] + add: splices one rank's offsets array into the concatenated Utf8 column of the regroup merge
__global__ void k_shift_copy_i32(int* __restrict__ dst, const int* __restrict__ src, long long n, int add) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) dst[i] = src[i] + add;
}
void shift_copy_i32(dfgpu_ctx* ctx, int* dst, const int* src, long long n, int add) {
  if (n <= 0) return;
  long long g = (n + 255) / 256;
  if (g > 4096) g = 4096;
  k_shift_copy_i32<<<(unsigned)g, 256, 0, ctx->stream>>>(dst, src, n, add);
  DF_CUDA(cudaGetLastError());
  ctx->launches++;
}

void utf8_hash(dfgpu_ctx* ctx, const DevColumn& src, long long n, unsigned long long* d_out) {
  if (n <= 0) return;
  const int grid = (int)std::min<long long>((n + 255) / 256, (long long)ctx->sm_count * 16);
  k_utf8_hash<<<grid, 256, 0, ctx->stream>>>(src.offsets, (const unsigned char*)src.values, n, d_out);
  DF_CUDA(cudaGetLastError());
  ctx->launches++;
}

// offsets[1..n] hold n string lengths: turn them into the end offsets (offsets[0] = 0 is the caller's) and return the
// total, which must fit the i32 offsets.  Synchronises the stream.
long long scan_utf8_lengths(dfgpu_ctx* ctx, int* offsets, long long n) {
  const long long nblocks = (n + SC_TILE - 1) / SC_TILE;
  long long* sums = (long long*)ctx->alloc(size_t(nblocks) * 8);
  k_scan_block<<<(unsigned)nblocks, SC_THREADS, 0, ctx->stream>>>(offsets + 1, n, sums);
  DF_CUDA(cudaGetLastError());
  k_scan_sums<<<1, 32, 0, ctx->stream>>>(sums, nblocks);
  DF_CUDA(cudaGetLastError());
  k_scan_add<<<(unsigned)nblocks, SC_THREADS, 0, ctx->stream>>>(offsets + 1, n, sums);
  DF_CUDA(cudaGetLastError());
  ctx->launches += 3;
  DF_CUDA(cudaMemcpyAsync(ctx->h_scratch + 24, sums + (nblocks - 1), 8, cudaMemcpyDeviceToHost, ctx->stream));
  DF_CUDA(cudaStreamSynchronize(ctx->stream));
  ctx->free(sums);
  const long long total = (long long)ctx->h_scratch[24];
  if (total >= (1ll << 31)) fail(DFGPU_ERR_NOT_IMPLEMENTED, "Utf8 output larger than 2 GiB (i32 offsets)");
  return total;
}

void gather_utf8_multi(dfgpu_ctx* ctx, const Utf8Source* d_srcs, const unsigned long long* d_idx, long long nsel, DevColumn* out) {
  out->dtype = DFGPU_UTF8;
  out->offsets = (int32_t*)ctx->alloc(size_t(nsel + 1) * 4);
  DF_CUDA(cudaMemsetAsync(out->offsets, 0, 4, ctx->stream));
  long long total = 0;
  if (nsel > 0) {
    const int grid = (int)std::min<long long>((nsel + 255) / 256, (long long)ctx->sm_count * 8);
    k_utf8_lengths<<<grid, 256, 0, ctx->stream>>>(d_idx, d_srcs, nsel, out->offsets);
    DF_CUDA(cudaGetLastError());
    ctx->launches++;
    total = scan_utf8_lengths(ctx, out->offsets, nsel);
  }
  out->values_bytes = size_t(total);
  out->values = ctx->alloc(std::max<size_t>(16, (size_t(total) + 15) & ~size_t(15)));  // whole 16-byte words
  if (total > 0) {
    const int grid = (int)std::min<long long>((nsel * 32 + 255) / 256, (long long)ctx->sm_count * 16);
    k_utf8_copy<<<grid, 256, 0, ctx->stream>>>(d_idx, d_srcs, nsel, out->offsets, (unsigned char*)out->values);
    DF_CUDA(cudaGetLastError());
    ctx->launches++;
  }
}

}  // namespace dfgpu
