// utf8_gather.cu — order-preserving gather of a Utf8 (arrow 0.12 BinaryArray: i32 offsets + bytes)
// column by a list of selected row numbers.  Replaces the Utf8 arm of `fn filter`
// (src/execution/filter.rs:93-103: per-row String allocation + BinaryArray::from(Vec<&str>)).
// The row numbers come out of the fused filter kernel as one more projected column (V_PUSH_ROWID).
#include "scan.cuh"
#include "utf8_words.cuh"

namespace dfgpu {

// A gather index addresses (source, row): source = idx >> UTF8_SRC_SHIFT.  The filter path has one
// source (the batch's column); Utf8 GROUP BY keys gather representatives from every batch seen.
__device__ __forceinline__ const Utf8Source& src_of(const Utf8Source* srcs, unsigned long long idx, long long* row) {
  *row = (long long)(idx & ((1ull << UTF8_SRC_SHIFT) - 1ull));
  return srcs[idx >> UTF8_SRC_SHIFT];
}

// lengths of the selected strings, written to out[i]
__global__ void k_utf8_lengths(const unsigned long long* __restrict__ idx, const Utf8Source* __restrict__ srcs, long long n, int* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    long long r;
    const Utf8Source& s = src_of(srcs, idx[i], &r);
    out[i] = s.off[r + 1] - s.off[r];
  }
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
  launch(ctx, "k_rebase_offsets", k_rebase_offsets, grid_for(ctx, n, 256, 16), 256, {}, d_off, n, lo);
}

// dst[i] = src[i] + add: splices one rank's offsets array into the concatenated Utf8 column of the regroup merge
__global__ void k_shift_copy_i32(int* __restrict__ dst, const int* __restrict__ src, long long n, int add) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) dst[i] = src[i] + add;
}
void shift_copy_i32(dfgpu_ctx* ctx, int* dst, const int* src, long long n, int add) {
  if (n <= 0) return;
  launch(ctx, "k_shift_copy_i32", k_shift_copy_i32, grid_for(ctx, n, 256, 16), 256, {}, dst, src, n, add);
}

void utf8_hash(dfgpu_ctx* ctx, const DevColumn& src, long long n, unsigned long long* d_out) {
  if (n <= 0) return;
  launch(ctx, "k_utf8_hash", k_utf8_hash, grid_for(ctx, n, 256, 16), 256, {}, (const int*)src.offsets, (const unsigned char*)src.values, n, d_out);
}

// offsets[0..n) hold n string lengths: they become the n + 1 offsets of the strings laid end to end.  Returns the total,
// which must fit the i32 offsets.  Synchronises the stream.
long long lengths_to_offsets(dfgpu_ctx* ctx, int* offsets, long long n) {
  const unsigned long long total = scan_exclusive<int, int>(ctx, offsets, offsets, n, false);
  if (total >= (1ull << 31)) fail(DFGPU_ERR_NOT_IMPLEMENTED, "Utf8 output larger than 2 GiB (i32 offsets)");
  return (long long)total;
}

void gather_utf8_multi(dfgpu_ctx* ctx, const Utf8Source* d_srcs, const unsigned long long* d_idx, long long nsel, DevColumn* out) {
  out->dtype = DFGPU_UTF8;
  out->offsets = (int32_t*)ctx->alloc(size_t(nsel + 1) * 4);
  long long total = 0;
  if (nsel > 0) {
    launch(ctx, "k_utf8_lengths", k_utf8_lengths, grid_for(ctx, nsel, 256, 8), 256, {}, d_idx, d_srcs, nsel, out->offsets);
    total = lengths_to_offsets(ctx, out->offsets, nsel);
  } else {
    DF_CUDA(cudaMemsetAsync(out->offsets, 0, 4, ctx->stream));
  }
  out->values_bytes = size_t(total);
  out->values = ctx->alloc(std::max<size_t>(16, (size_t(total) + 15) & ~size_t(15)));  // whole 16-byte words
  if (total > 0)
    launch(ctx, "k_utf8_copy", k_utf8_copy, grid_for(ctx, nsel * 32, 256, 16), 256, {}, d_idx, d_srcs, nsel, (const int*)out->offsets,
           (unsigned char*)out->values);
}

}  // namespace dfgpu
