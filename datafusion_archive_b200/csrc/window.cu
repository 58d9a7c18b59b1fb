// window.cu — dfgpu_window: window functions over one specification (PARTITION BY keys, ORDER BY keys), one output column
// per function, in the input's row order; include/dfgpu.h documents the semantics.
//
// The rows are ordered by the partition keys and then the ORDER BY keys with the stable radix sort of sort.cuh (the
// permutation stays the identity, k_sort_iota, without keys).  After the sort:
//   k_win_flags     per sorted position i, pflag[i] = 1 where a partition starts (a partition key's encoding, value
//                   word or null bit, differs from position i - 1) and gflag[i] = 1 where a peer group starts (pflag,
//                   or an ORDER BY key differs); Utf8 keys compare by their dense rank
//   scan_exclusive  of both flag arrays: the partition and peer-group number of every position
//   k_win_bounds    pid[i] and gid[i], the first position of every partition and peer group, and inv[perm[i]] = i
//   per aggregate   a segmented inclusive scan of the argument in sorted order that restarts at every partition start,
//                   with a (value, valid count) carry: k_win_tile_reduce (each 2048-position tile's segmented total),
//                   k_win_carry (one CTA scans the tile totals into each tile's carry-in) and k_win_tile_scan (each
//                   tile rescans from its carry-in and stores the running value at the last position of each peer
//                   group, gval[g] / gcnt[g]).  The association of every float sum is fixed by n alone, so a float
//                   SUM / AVG gives the same bits on every run.
//   k_win_out       per output row r: i = inv[r]; the ranks are subtractions of first positions, an aggregate is its
//                   peer group's value (the RANGE frame through the last peer; without ORDER BY the partition total)
// With a communicator attached, every rank first all-gathers the key and argument columns in rank order, computes the
// window over the whole input and keeps its own rows.
#include <memory>
#include <type_traits>

#include "sort.cuh"

namespace dfgpu {

void shift_copy_i32(dfgpu_ctx* ctx, int* dst, const int* src, long long n, int add);  // utf8_gather.cu

namespace {

constexpr int WIN_THREADS = 256;
constexpr int WIN_ITEMS = 8;
constexpr int WIN_TILE = WIN_THREADS * WIN_ITEMS;
constexpr int WIN_CARRY_THREADS = 1024;

__global__ void __launch_bounds__(SORT_THREADS) k_win_flags(const KeySrc* __restrict__ keys, int nkeys, int npart, const unsigned* __restrict__ perm,
                                                           long long n, unsigned* __restrict__ pflag, unsigned* __restrict__ gflag) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    unsigned p = 1, g = 1;
    if (i > 0) {
      const unsigned r = perm[i], q = perm[i - 1];
      p = 0;
      g = 0;
      for (int k = 0; k < nkeys && !p; k++) {
        const KeySrc s = keys[k];
        if (sort_key(s, r) != sort_key(s, q)) {
          g = 1;
          if (k < npart) p = 1;
        }
      }
    }
    pflag[i] = p;
    gflag[i] = g;
  }
}

// pid / gid hold the exclusive scans of the flags on entry and the partition / peer-group number of each position on exit
__global__ void __launch_bounds__(SORT_THREADS) k_win_bounds(const unsigned* __restrict__ perm, long long n, const unsigned* __restrict__ pflag,
                                                            const unsigned* __restrict__ gflag, unsigned* __restrict__ pid, unsigned* __restrict__ gid,
                                                            unsigned* __restrict__ pfirst, unsigned* __restrict__ gfirst, unsigned* __restrict__ inv) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const unsigned pf = pflag[i], gf = gflag[i];
    const unsigned p = pid[i] + pf - 1u, g = gid[i] + gf - 1u;
    pid[i] = p;
    gid[i] = g;
    if (pf) pfirst[p] = (unsigned)i;
    if (gf) gfirst[g] = (unsigned)i;
    inv[perm[i]] = (unsigned)i;
  }
}

// ---- the segmented scan --------------------------------------------------------------------------------------------
// Operators on the scanned value: integer SUM wraps in 64 bits (the output keeps the low bits of its width), float SUM
// adds in the argument's precision (AVG in f64), MIN / MAX compare order-preserving words (sort_key's encoding: -0.0
// below +0.0; a NaN is the largest word for MIN and 0, below every number, for MAX, so it is skipped unless every value
// is NaN).  COUNT scans the integer SUM operator over zeros and keeps only the count.
struct OpSumU64 {
  using T = unsigned long long;
  static __device__ __forceinline__ T id() { return 0ull; }
  static __device__ __forceinline__ T op(T a, T b) { return a + b; }
};
struct OpMin {
  using T = unsigned long long;
  static __device__ __forceinline__ T id() { return ~0ull; }
  static __device__ __forceinline__ T op(T a, T b) { return b < a ? b : a; }
};
struct OpMax {
  using T = unsigned long long;
  static __device__ __forceinline__ T id() { return 0ull; }
  static __device__ __forceinline__ T op(T a, T b) { return b > a ? b : a; }
};
struct OpSumF32 {
  using T = float;
  static __device__ __forceinline__ T id() { return 0.0f; }
  static __device__ __forceinline__ T op(T a, T b) { return __fadd_rn(a, b); }
};
struct OpSumF64 {
  using T = double;
  static __device__ __forceinline__ T id() { return 0.0; }
  static __device__ __forceinline__ T op(T a, T b) { return __dadd_rn(a, b); }
};

// What a function reads of its argument: values of `dtype`, `valid` null when there is no null
struct WinArg {
  const void* vals;
  const unsigned char* valid;
  int dtype;
  int func;
};

__device__ __forceinline__ double arg_f64(const WinArg& a, unsigned r) {
  switch (a.dtype) {
    case DFGPU_INT8: return (double)((const signed char*)a.vals)[r];
    case DFGPU_UINT8: return (double)((const unsigned char*)a.vals)[r];
    case DFGPU_INT16: return (double)((const short*)a.vals)[r];
    case DFGPU_UINT16: return (double)((const unsigned short*)a.vals)[r];
    case DFGPU_INT32: return (double)((const int*)a.vals)[r];
    case DFGPU_UINT32: return (double)((const unsigned*)a.vals)[r];
    case DFGPU_INT64: return (double)((const long long*)a.vals)[r];
    case DFGPU_UINT64: return (double)((const unsigned long long*)a.vals)[r];
    case DFGPU_FLOAT32: return (double)((const float*)a.vals)[r];
    default: return ((const double*)a.vals)[r];
  }
}

// integers widened to 64 bits (signed ones sign-extended), for the wrapping SUM
__device__ __forceinline__ unsigned long long arg_u64(const WinArg& a, unsigned r) {
  switch (a.dtype) {
    case DFGPU_INT8: return (unsigned long long)(long long)((const signed char*)a.vals)[r];
    case DFGPU_UINT8: return ((const unsigned char*)a.vals)[r];
    case DFGPU_INT16: return (unsigned long long)(long long)((const short*)a.vals)[r];
    case DFGPU_UINT16: return ((const unsigned short*)a.vals)[r];
    case DFGPU_INT32: return (unsigned long long)(long long)((const int*)a.vals)[r];
    case DFGPU_UINT32: return ((const unsigned*)a.vals)[r];
    default: return ((const unsigned long long*)a.vals)[r];
  }
}

template <class T>
__device__ __forceinline__ T arg_value(const WinArg& a, unsigned r);
template <>
__device__ __forceinline__ unsigned long long arg_value<unsigned long long>(const WinArg& a, unsigned r) {
  if (a.func == DFGPU_AGG_SUM) return arg_u64(a, r);
  if (a.func == DFGPU_AGG_COUNT) return 0ull;
  const KeySrc s{KS_FIXED, a.dtype, 0, 0, a.vals, nullptr, nullptr, nullptr};
  const unsigned long long e = sort_key(s, r);
  const unsigned long long nan = a.dtype == DFGPU_FLOAT32 ? 0xffffffffull : ~0ull;
  return a.func == DFGPU_AGG_MAX && (a.dtype == DFGPU_FLOAT32 || a.dtype == DFGPU_FLOAT64) && e == nan ? 0ull : e;
}
template <>
__device__ __forceinline__ float arg_value<float>(const WinArg& a, unsigned r) {
  return ((const float*)a.vals)[r];
}
template <>
__device__ __forceinline__ double arg_value<double>(const WinArg& a, unsigned r) {
  return arg_f64(a, r);
}

template <class T>
struct Seg {
  T v;
  unsigned c;  // valid values
  unsigned f;  // a partition starts in the span
};

template <class Op>
__device__ __forceinline__ Seg<typename Op::T> seg_id() {
  return Seg<typename Op::T>{Op::id(), 0u, 0u};
}
// a's span followed by b's
template <class Op>
__device__ __forceinline__ Seg<typename Op::T> seg_op(const Seg<typename Op::T>& a, const Seg<typename Op::T>& b) {
  return b.f ? b : Seg<typename Op::T>{Op::op(a.v, b.v), a.c + b.c, a.f};
}

// sorted position i as a one-element span
template <class Op>
__device__ __forceinline__ Seg<typename Op::T> seg_at(const WinArg& a, const unsigned* __restrict__ perm, const unsigned* __restrict__ pflag,
                                                      long long i) {
  using T = typename Op::T;
  const unsigned r = perm[i];
  const bool ok = !a.valid || bit_at(a.valid, r);
  return Seg<T>{ok ? arg_value<T>(a, r) : Op::id(), ok ? 1u : 0u, pflag[i]};
}

template <class T>
__device__ __forceinline__ T shfl_up(T x, int o) {
  return __shfl_up_sync(0xffffffffu, x, o);
}

// The block's exclusive scan of x (in thread order) and its total, in a fixed association
template <class Op>
__device__ __forceinline__ void block_scan(Seg<typename Op::T> x, Seg<typename Op::T>& excl, Seg<typename Op::T>& total) {
  using S = Seg<typename Op::T>;
  __shared__ S s_warp[WIN_THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  S incl = x;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const S y{shfl_up(incl.v, o), shfl_up(incl.c, o), shfl_up(incl.f, o)};
    if (lane >= o) incl = seg_op<Op>(y, incl);
  }
  S le{shfl_up(incl.v, 1), shfl_up(incl.c, 1), shfl_up(incl.f, 1)};
  if (lane == 0) le = seg_id<Op>();
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  S pre = seg_id<Op>();
  total = seg_id<Op>();
#pragma unroll
  for (int w = 0; w < WIN_THREADS / 32; w++) {
    if (w < warp) pre = seg_op<Op>(pre, s_warp[w]);
    total = seg_op<Op>(total, s_warp[w]);
  }
  excl = seg_op<Op>(pre, le);
}

template <class Op>
__global__ void __launch_bounds__(WIN_THREADS) k_win_tile_reduce(WinArg a, const unsigned* __restrict__ perm, const unsigned* __restrict__ pflag,
                                                                long long n, Seg<typename Op::T>* __restrict__ tiles) {
  using S = Seg<typename Op::T>;
  const long long base = (long long)blockIdx.x * WIN_TILE + (long long)threadIdx.x * WIN_ITEMS;
  S x = seg_id<Op>();
#pragma unroll
  for (int j = 0; j < WIN_ITEMS; j++)
    if (base + j < n) x = seg_op<Op>(x, seg_at<Op>(a, perm, pflag, base + j));
  S excl, total;
  block_scan<Op>(x, excl, total);
  if (threadIdx.x == 0) tiles[blockIdx.x] = total;
}

// one CTA: tiles[t] becomes the exclusive segmented scan of the tile totals, the carry into tile t
template <class Op>
__global__ void __launch_bounds__(WIN_CARRY_THREADS) k_win_carry(Seg<typename Op::T>* tiles, long long nt) {
  using S = Seg<typename Op::T>;
  __shared__ S s_part[WIN_CARRY_THREADS];
  const long long per = (nt + WIN_CARRY_THREADS - 1) / WIN_CARRY_THREADS, lo = (long long)threadIdx.x * per, hi = min(nt, lo + per);
  S acc = seg_id<Op>();
  for (long long t = lo; t < hi; t++) acc = seg_op<Op>(acc, tiles[t]);
  s_part[threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    S run = seg_id<Op>();
    for (int i = 0; i < WIN_CARRY_THREADS; i++) {
      const S x = s_part[i];
      s_part[i] = run;
      run = seg_op<Op>(run, x);
    }
  }
  __syncthreads();
  S run = s_part[threadIdx.x];
  for (long long t = lo; t < hi; t++) {
    const S x = tiles[t];
    tiles[t] = run;
    run = seg_op<Op>(run, x);
  }
}

// the running value at the last position of each peer group: gval[g], gcnt[g]
template <class Op>
__global__ void __launch_bounds__(WIN_THREADS) k_win_tile_scan(WinArg a, const unsigned* __restrict__ perm, const unsigned* __restrict__ pflag,
                                                              const unsigned* __restrict__ gflag, const unsigned* __restrict__ gid, long long n,
                                                              const Seg<typename Op::T>* __restrict__ carry, typename Op::T* __restrict__ gval,
                                                              unsigned* __restrict__ gcnt) {
  using S = Seg<typename Op::T>;
  const long long base = (long long)blockIdx.x * WIN_TILE + (long long)threadIdx.x * WIN_ITEMS;
  S e[WIN_ITEMS];
  S x = seg_id<Op>();
#pragma unroll
  for (int j = 0; j < WIN_ITEMS; j++) {
    e[j] = base + j < n ? seg_at<Op>(a, perm, pflag, base + j) : seg_id<Op>();
    x = seg_op<Op>(x, e[j]);
  }
  S excl, total;
  block_scan<Op>(x, excl, total);
  S run = seg_op<Op>(carry[blockIdx.x], excl);
#pragma unroll
  for (int j = 0; j < WIN_ITEMS; j++) {
    const long long i = base + j;
    if (i < n) {
      run = seg_op<Op>(run, e[j]);
      if (i == n - 1 || gflag[i + 1]) {
        gval[gid[i]] = run.v;
        gcnt[gid[i]] = run.c;
      }
    }
  }
}

// ---- the output --------------------------------------------------------------------------------------------------
// What k_win_out writes for a function
struct WinOut {
  int func;
  int dtype;      // of the argument (of the output for the ranks and COUNT)
  void* out;      // cnt values of the output dtype
  unsigned* valid;  // cnt bits, or null: every row valid
};

__device__ __forceinline__ void store(void* out, long long j, int width, unsigned long long bits) {
  switch (width) {
    case 1: ((unsigned char*)out)[j] = (unsigned char)bits; break;
    case 2: ((unsigned short*)out)[j] = (unsigned short)bits; break;
    case 4: ((unsigned*)out)[j] = (unsigned)bits; break;
    default: ((unsigned long long*)out)[j] = bits; break;
  }
}

// the value of an order-preserving MIN / MAX word (arg_value's encoding)
__device__ __forceinline__ unsigned long long decode(int dtype, unsigned long long e) {
  switch (dtype) {
    case DFGPU_INT8: return e ^ 0x80u;
    case DFGPU_INT16: return e ^ 0x8000u;
    case DFGPU_INT32: return e ^ 0x80000000u;
    case DFGPU_INT64: return e ^ 0x8000000000000000ull;
    case DFGPU_FLOAT32:
      if (e == 0 || e == 0xffffffffull) return 0x7fc00000u;
      return (e >> 31) ? (e ^ 0x80000000u) : (~e & 0xffffffffull);
    case DFGPU_FLOAT64:
      if (e == 0 || e == ~0ull) return 0x7ff8000000000000ull;
      return (e >> 63) ? (e ^ 0x8000000000000000ull) : ~e;
    default: return e;
  }
}

// rows [lo, lo + cnt) of the input order; output row j = r - lo
template <class T>
__global__ void __launch_bounds__(SORT_THREADS) k_win_out(WinOut o, long long lo, long long cnt, const unsigned* __restrict__ inv,
                                                         const unsigned* __restrict__ pid, const unsigned* __restrict__ gid,
                                                         const unsigned* __restrict__ pfirst, const unsigned* __restrict__ gfirst,
                                                         const T* __restrict__ gval, const unsigned* __restrict__ gcnt, unsigned long long* __restrict__ nulls) {
  const long long padded = (cnt + 31) / 32 * 32;
  unsigned z = 0;
  for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < padded; j += (long long)gridDim.x * blockDim.x) {
    bool ok = false;
    if (j < cnt) {
      const unsigned i = inv[lo + j], g = gid[i];
      ok = true;
      switch (o.func) {
        case DFGPU_WIN_ROW_NUMBER: store(o.out, j, 8, (unsigned long long)(i - pfirst[pid[i]]) + 1ull); break;
        case DFGPU_WIN_RANK: store(o.out, j, 8, (unsigned long long)(gfirst[g] - pfirst[pid[i]]) + 1ull); break;
        case DFGPU_WIN_DENSE_RANK: store(o.out, j, 8, (unsigned long long)(g - gid[pfirst[pid[i]]]) + 1ull); break;
        case DFGPU_AGG_COUNT: store(o.out, j, 8, (unsigned long long)gcnt[g]); break;
        default: {
          const unsigned c = gcnt[g];
          ok = c > 0;
          const T v = ok ? gval[g] : T(0);
          if constexpr (sizeof(T) == 8 && T(-1) > T(0)) {  // unsigned long long: integer SUM, MIN, MAX
            const int width = o.dtype == DFGPU_INT8 || o.dtype == DFGPU_UINT8     ? 1
                              : o.dtype == DFGPU_INT16 || o.dtype == DFGPU_UINT16 ? 2
                              : o.dtype == DFGPU_INT32 || o.dtype == DFGPU_UINT32 || o.dtype == DFGPU_FLOAT32 ? 4
                                                                                                              : 8;
            store(o.out, j, width, !ok ? 0ull : o.func == DFGPU_AGG_SUM ? v : decode(o.dtype, v));
          } else if (o.func == DFGPU_AGG_AVG) {
            ((double*)o.out)[j] = ok ? __ddiv_rn((double)v, (double)c) : 0.0;
          } else {
            ((T*)o.out)[j] = v;
          }
        }
      }
    }
    if (o.valid) {
      const unsigned m = __ballot_sync(0xffffffffu, ok);
      const unsigned in = __ballot_sync(0xffffffffu, j < cnt);
      if ((threadIdx.x & 31) == 0) {
        o.valid[j >> 5] = m;
        z += __popc(in & ~m);
      }
    }
  }
  if (nulls && z) atomicAdd(nulls, (unsigned long long)z);
}

// the validity of n rows as one byte per row (valid null: all valid)
__global__ void __launch_bounds__(SORT_THREADS) k_win_unpack(const unsigned char* __restrict__ valid, long long n, unsigned char* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = !valid || bit_at(valid, (unsigned)i);
}

// one byte per row -> bits, one warp per output word
__global__ void __launch_bounds__(SORT_THREADS) k_win_pack(const unsigned char* __restrict__ bytes, long long n, unsigned* __restrict__ words) {
  const long long padded = (n + 31) / 32 * 32;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < padded; i += (long long)gridDim.x * blockDim.x) {
    const unsigned m = __ballot_sync(0xffffffffu, i < n && bytes[i] != 0);
    if ((threadIdx.x & 31) == 0) words[i >> 5] = m;
  }
}

bool is_rank_fn(int f) { return f == DFGPU_WIN_ROW_NUMBER || f == DFGPU_WIN_RANK || f == DFGPU_WIN_DENSE_RANK; }

// All ranks' rows of `cols` (this rank's are n rows), in rank order, into `g`; *lo = the first global row of this rank.
void gather_ranks(dfgpu_ctx* ctx, long long n, const std::vector<const DevColumn*>& cols, dfgpu_batch& g, long long* lo) {
  const int W = ctx->world, me = ctx->rank, nc = int(cols.size());
  const int NH = 1 + 2 * nc;  // rows, then per column: nulls, Utf8 bytes
  DevBufs tmp(ctx);
  unsigned long long* d_h = tmp.alloc(size_t(NH) * 8 * size_t(W + 1));
  std::vector<unsigned long long> h(size_t(NH), 0), all(size_t(NH) * size_t(W));
  h[0] = (unsigned long long)n;
  for (int c = 0; c < nc; c++) {
    h[size_t(1 + 2 * c)] = (unsigned long long)cols[size_t(c)]->null_count;
    h[size_t(2 + 2 * c)] = cols[size_t(c)]->dtype == DFGPU_UTF8 ? (unsigned long long)cols[size_t(c)]->values_bytes : 0ull;
  }
  DF_CUDA(cudaMemcpyAsync(d_h, h.data(), h.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
  comm_allgather_u64(ctx, d_h, d_h + NH, size_t(NH));
  DF_CUDA(cudaMemcpyAsync(all.data(), d_h + NH, all.size() * 8, cudaMemcpyDeviceToHost, ctx->stream));
  DF_CUDA(cudaStreamSynchronize(ctx->stream));
  long long N = 0;
  std::vector<long long> base(size_t(W), 0), rows(size_t(W), 0);
  for (int r = 0; r < W; r++) {
    base[size_t(r)] = N;
    rows[size_t(r)] = (long long)all[size_t(r) * NH];
    N += rows[size_t(r)];
  }
  *lo = base[size_t(me)];
  g.ctx = ctx;
  g.nrows = N;
  if (N >= (1ll << 32)) fail(DFGPU_ERR_NOT_IMPLEMENTED, "window input of 2^32 rows or more");  // every rank refuses alike
  std::vector<size_t> off(static_cast<size_t>(W)), cnt(static_cast<size_t>(W));
  for (int c = 0; c < nc; c++) {
    const DevColumn& lc = *cols[size_t(c)];
    DevColumn gc;
    gc.dtype = lc.dtype;
    if (lc.dtype == DFGPU_UTF8) {
      size_t total = 0;
      std::vector<size_t> bbase(static_cast<size_t>(W));
      for (int r = 0; r < W; r++) {
        bbase[size_t(r)] = off[size_t(r)] = total;
        cnt[size_t(r)] = size_t(all[size_t(r) * NH + 2 + 2 * size_t(c)]);
        total += cnt[size_t(r)];
      }
      if (total >= (1ull << 31)) fail(DFGPU_ERR_NOT_IMPLEMENTED, "window over 2 GiB or more of Utf8 key bytes");
      gc.values_bytes = total;
      gc.values = ctx->alloc(total ? total : 1);
      comm_allgather_bytes_v(ctx, lc.values, gc.values, off.data(), cnt.data());
      int* raw = tmp.alloc<int>(size_t(N + W) * 4);  // every rank's rows + 1 offsets, then rebased
      for (int r = 0; r < W; r++) {
        off[size_t(r)] = size_t(base[size_t(r)] + r) * 4;
        cnt[size_t(r)] = size_t(rows[size_t(r)] + 1) * 4;
      }
      comm_allgather_bytes_v(ctx, lc.offsets, raw, off.data(), cnt.data());
      gc.offsets = (int32_t*)ctx->alloc(size_t(N + 1) * 4);
      for (int r = 0; r < W; r++)
        if (rows[size_t(r)]) shift_copy_i32(ctx, gc.offsets + base[size_t(r)], raw + base[size_t(r)] + r, rows[size_t(r)], int(bbase[size_t(r)]));
      const int last = int(total);
      DF_CUDA(cudaMemcpyAsync(gc.offsets + N, &last, 4, cudaMemcpyHostToDevice, ctx->stream));
      DF_CUDA(cudaStreamSynchronize(ctx->stream));  // `last` is a stack variable
    } else {
      const size_t w = size_t(dtype_width(lc.dtype));
      for (int r = 0; r < W; r++) {
        off[size_t(r)] = size_t(base[size_t(r)]) * w;
        cnt[size_t(r)] = size_t(rows[size_t(r)]) * w;
      }
      gc.values_bytes = size_t(N) * w;
      gc.values = ctx->alloc(gc.values_bytes ? gc.values_bytes : 8);
      comm_allgather_bytes_v(ctx, lc.values, gc.values, off.data(), cnt.data());
    }
    long long nulls = 0;
    for (int r = 0; r < W; r++) nulls += (long long)all[size_t(r) * NH + 1 + 2 * size_t(c)];
    if (nulls > 0) {  // as bytes: the ranks' bitmaps do not start on byte boundaries of the whole
      unsigned char* mine = tmp.alloc<unsigned char>(size_t(std::max(1ll, n)));
      unsigned char* every = tmp.alloc<unsigned char>(size_t(std::max(1ll, N)));
      if (n > 0)
        launch(ctx, "k_win_unpack", k_win_unpack, grid_for(ctx, n, SORT_THREADS, 16), SORT_THREADS, {},
               (const unsigned char*)(lc.null_count > 0 ? lc.validity : nullptr), n, mine);
      for (int r = 0; r < W; r++) {
        off[size_t(r)] = size_t(base[size_t(r)]);
        cnt[size_t(r)] = size_t(rows[size_t(r)]);
      }
      comm_allgather_bytes_v(ctx, mine, every, off.data(), cnt.data());
      gc.validity = (uint8_t*)ctx->alloc(size_t((N + 31) / 32) * 4);
      launch(ctx, "k_win_pack", k_win_pack, grid_for(ctx, (N + 31) / 32 * 32, SORT_THREADS, 8), SORT_THREADS, {}, (const unsigned char*)every, N,
             (unsigned*)gc.validity);
      gc.null_count = nulls;
    }
    g.cols.push_back(gc);
  }
  DF_CUDA(cudaStreamSynchronize(ctx->stream));  // the scratch above goes back to the pool
}

struct WinFn {
  int func;
  const DevColumn* arg;  // null for the ranks
  int out_dtype;
};

// The segmented scan of one aggregate: gval / gcnt of every peer group
template <class Op>
void seg_scan(dfgpu_ctx* ctx, const WinArg& a, const unsigned* perm, const unsigned* pflag, const unsigned* gflag, const unsigned* gid, long long n,
              DevBufs& scratch, typename Op::T* gval, unsigned* gcnt) {
  using S = Seg<typename Op::T>;
  const long long nt = (n + WIN_TILE - 1) / WIN_TILE;
  S* tiles = scratch.alloc<S>(size_t(nt) * sizeof(S));
  launch(ctx, "k_win_tile_reduce", k_win_tile_reduce<Op>, int(nt), WIN_THREADS, PROFILED, a, perm, pflag, n, tiles);
  launch(ctx, "k_win_carry", k_win_carry<Op>, 1, WIN_CARRY_THREADS, PROFILED, tiles, nt);
  launch(ctx, "k_win_tile_scan", k_win_tile_scan<Op>, int(nt), WIN_THREADS, PROFILED, a, perm, pflag, gflag, gid, n, (const S*)tiles, gval, gcnt);
}

// The window over the n rows of the key and argument columns; the result holds rows [lo, lo + cnt)
void window(dfgpu_ctx* ctx, long long n, const std::vector<const DevColumn*>& part, const std::vector<const DevColumn*>& order,
            const std::vector<int>& desc, const std::vector<WinFn>& fns, long long lo, long long cnt, dfgpu_result* res) {
  DevBufs scratch(ctx);
  for (const WinFn& f : fns) {
    res->cols.emplace_back();
    DevColumn& c = res->cols.back();
    c.dtype = f.out_dtype;
    c.values_bytes = size_t(cnt) * size_t(dtype_width(f.out_dtype));
    c.values = ctx->alloc(std::max<size_t>(8, c.values_bytes));
  }
  if (n == 0) return;
  // 1. the permutation: the last key first, the ORDER BY keys descending where asked, the partition keys ascending
  Sorter S = make_sorter(ctx, n, scratch);
  S.cur = 0;
  launch(ctx, "k_sort_iota", k_sort_iota, grid_for(ctx, n, SORT_THREADS, 16), SORT_THREADS, PROFILED, n, S.perm[0]);
  std::vector<const DevColumn*> keys = part;
  keys.insert(keys.end(), order.begin(), order.end());
  std::vector<unsigned*> ranks(keys.size(), nullptr);
  for (size_t k = 0; k < keys.size(); k++)
    if (keys[k]->dtype == DFGPU_UTF8 && n > 1) {
      ranks[k] = scratch.alloc<unsigned>(size_t(n) * 4);
      utf8_rank(S, *keys[k], keys[k]->null_count > 0 ? keys[k]->validity : nullptr, n, scratch, ranks[k]);
    }
  std::vector<KeySrc> srcs;  // for the boundary flags: each key's word, then its null bit
  int npart = 0;
  for (size_t k = 0; k < keys.size(); k++) {
    const DevColumn& c = *keys[k];
    const unsigned char* valid = c.null_count > 0 ? c.validity : nullptr;
    if (c.dtype == DFGPU_UTF8) srcs.push_back(KeySrc{KS_RANK, DFGPU_UINT32, 0, 0, ranks[k], valid, nullptr, nullptr});
    else srcs.push_back(KeySrc{KS_FIXED, c.dtype, 0, 0, c.values, valid, nullptr, nullptr});
    if (valid) srcs.push_back(KeySrc{KS_NULL, 0, 0, 0, nullptr, valid, nullptr, nullptr});
    if (k + 1 == part.size()) npart = int(srcs.size());
  }
  if (n > 1) {
    for (size_t k = keys.size(); k-- > 0;) {
      const int d = k >= part.size() && desc[k - part.size()] ? 1 : 0;
      const DevColumn& c = *keys[k];
      const unsigned char* valid = c.null_count > 0 ? c.validity : nullptr;
      if (c.dtype == DFGPU_UTF8) S.by<unsigned>(KeySrc{KS_RANK, DFGPU_UINT32, d, 0, ranks[k], valid, nullptr, nullptr});
      else S.by_width(dtype_width(c.dtype), KeySrc{KS_FIXED, c.dtype, d, 0, c.values, valid, nullptr, nullptr});
      if (valid) S.by<unsigned char>(KeySrc{KS_NULL, 0, d, 0, nullptr, valid, nullptr, nullptr});
    }
  }
  const unsigned* perm = S.perm[S.cur];
  // 2. boundaries, partition and peer-group numbers, first positions and the inverse permutation
  KeySrc* d_srcs = scratch.alloc<KeySrc>(std::max<size_t>(1, srcs.size()) * sizeof(KeySrc));
  if (!srcs.empty()) DF_CUDA(cudaMemcpyAsync(d_srcs, srcs.data(), srcs.size() * sizeof(KeySrc), cudaMemcpyHostToDevice, ctx->stream));
  unsigned* pflag = scratch.alloc<unsigned>(size_t(n) * 4);
  unsigned* gflag = scratch.alloc<unsigned>(size_t(n) * 4);
  unsigned* pid = scratch.alloc<unsigned>(size_t(n + 1) * 4);
  unsigned* gid = scratch.alloc<unsigned>(size_t(n + 1) * 4);
  unsigned* inv = scratch.alloc<unsigned>(size_t(n) * 4);
  const int grid = grid_for(ctx, n, SORT_THREADS, 16);
  launch(ctx, "k_win_flags", k_win_flags, grid, SORT_THREADS, PROFILED, (const KeySrc*)d_srcs, int(srcs.size()), npart, perm, n, pflag, gflag);
  const unsigned long long np = scan_exclusive<unsigned, unsigned>(ctx, pflag, pid, n, true);
  const unsigned long long ng = scan_exclusive<unsigned, unsigned>(ctx, gflag, gid, n, true);
  unsigned* pfirst = scratch.alloc<unsigned>(size_t(np) * 4);
  unsigned* gfirst = scratch.alloc<unsigned>(size_t(ng) * 4);
  launch(ctx, "k_win_bounds", k_win_bounds, grid, SORT_THREADS, PROFILED, perm, n, (const unsigned*)pflag, (const unsigned*)gflag, pid, gid, pfirst, gfirst,
         inv);
  // 3. each function
  unsigned long long* d_nulls = scratch.alloc<unsigned long long>(8 * fns.size());
  DF_CUDA(cudaMemsetAsync(d_nulls, 0, 8 * fns.size(), ctx->stream));
  unsigned* gcnt = scratch.alloc<unsigned>(size_t(ng) * 4);
  void* gval = scratch.alloc<void>(size_t(ng) * 8);
  const int ogrid = grid_for(ctx, (cnt + 31) / 32 * 32, SORT_THREADS, 16);
  for (size_t k = 0; k < fns.size(); k++) {
    const WinFn& f = fns[k];
    DevColumn& c = res->cols[k];
    const bool nullable = !is_rank_fn(f.func) && f.func != DFGPU_AGG_COUNT;
    if (nullable && cnt > 0) c.validity = (uint8_t*)ctx->alloc(size_t((cnt + 31) / 32) * 4);
    const WinOut o{f.func, is_rank_fn(f.func) ? DFGPU_UINT64 : f.arg->dtype, c.values, (unsigned*)c.validity};
    WinArg a{nullptr, nullptr, 0, f.func};
    if (f.arg) a = WinArg{f.arg->values, f.arg->null_count > 0 ? f.arg->validity : nullptr, f.arg->dtype, f.func};
    auto out = [&](auto* vals) {
      using T = std::remove_pointer_t<decltype(vals)>;
      if (cnt > 0)
        launch(ctx, "k_win_out", k_win_out<T>, ogrid, SORT_THREADS, PROFILED, o, lo, cnt, (const unsigned*)inv, (const unsigned*)pid, (const unsigned*)gid,
               (const unsigned*)pfirst, (const unsigned*)gfirst, (const T*)vals, (const unsigned*)gcnt, d_nulls + k);
    };
    if (is_rank_fn(f.func)) {
      out((unsigned long long*)gval);
    } else if (f.func == DFGPU_AGG_MIN) {
      seg_scan<OpMin>(ctx, a, perm, pflag, gflag, gid, n, scratch, (unsigned long long*)gval, gcnt);
      out((unsigned long long*)gval);
    } else if (f.func == DFGPU_AGG_MAX) {
      seg_scan<OpMax>(ctx, a, perm, pflag, gflag, gid, n, scratch, (unsigned long long*)gval, gcnt);
      out((unsigned long long*)gval);
    } else if (f.func == DFGPU_AGG_AVG || (f.func == DFGPU_AGG_SUM && f.arg->dtype == DFGPU_FLOAT64)) {
      seg_scan<OpSumF64>(ctx, a, perm, pflag, gflag, gid, n, scratch, (double*)gval, gcnt);
      out((double*)gval);
    } else if (f.func == DFGPU_AGG_SUM && f.arg->dtype == DFGPU_FLOAT32) {
      seg_scan<OpSumF32>(ctx, a, perm, pflag, gflag, gid, n, scratch, (float*)gval, gcnt);
      out((float*)gval);
    } else {  // integer SUM, COUNT
      seg_scan<OpSumU64>(ctx, a, perm, pflag, gflag, gid, n, scratch, (unsigned long long*)gval, gcnt);
      out((unsigned long long*)gval);
    }
  }
  std::vector<unsigned long long> nulls(fns.size());
  DF_CUDA(cudaMemcpyAsync(nulls.data(), d_nulls, 8 * fns.size(), cudaMemcpyDeviceToHost, ctx->stream));
  DF_CUDA(cudaStreamSynchronize(ctx->stream));
  for (size_t k = 0; k < fns.size(); k++) set_null_count(ctx, res->cols[k], int64_t(nulls[k]));
}

}  // namespace
}  // namespace dfgpu

using namespace dfgpu;

extern "C" int dfgpu_window(dfgpu_ctx* ctx, const dfgpu_batch* in, const dfgpu_insn* const* part, const int* part_len, int npart,
                            const dfgpu_insn* const* order, const int* order_len, const int32_t* desc, int norder, const dfgpu_agg* fns, int nfns,
                            dfgpu_result** out) {
  return guarded([&] {
    if (!ctx || !in || !out || npart < 0 || norder < 0 || nfns < 0 || (npart > 0 && (!part || !part_len)) ||
        (norder > 0 && (!order || !order_len)) || (nfns > 0 && !fns))
      fail(DFGPU_ERR_GENERAL, "dfgpu_window: null argument");
    ctx->use();
    const long long n = in->nrows;
    if (ctx->world <= 1 && n >= (1ll << 32)) fail(DFGPU_ERR_NOT_IMPLEMENTED, "window input of 2^32 rows or more");
    std::vector<int32_t> col_dtypes;
    for (const DevColumn& c : in->cols) col_dtypes.push_back(c.dtype);
    // a program's column: a plain column in place, anything else evaluated as a projection (as dfgpu_sort does)
    std::vector<std::unique_ptr<dfgpu_result, int (*)(dfgpu_result*)>> evaluated;
    auto column = [&](const dfgpu_insn* p, int len, int32_t* dt) -> const DevColumn* {
      const int rc = dfgpu_check_program(col_dtypes.empty() ? nullptr : col_dtypes.data(), int(col_dtypes.size()), p, len, dt);
      if (rc != DFGPU_OK) fail(rc, dfgpu_last_error());
      if (len == 1 && p[0].op == DFGPU_OP_COL) return &in->cols[size_t(p[0].col)];
      dfgpu_result* r = nullptr;
      const int rc2 = dfgpu_filter_project(ctx, in, nullptr, 0, &p, &len, 1, &r);
      if (rc2 != DFGPU_OK) fail(rc2, dfgpu_last_error());
      evaluated.emplace_back(r, dfgpu_result_free);
      resolve(r);
      return &r->cols[0];
    };
    std::vector<const DevColumn*> pcols, ocols;
    std::vector<int> d;
    for (int i = 0; i < npart; i++) {
      int32_t dt = 0;
      pcols.push_back(column(part[i], part_len[i], &dt));
      if (dt == DFGPU_BOOL) fail(DFGPU_ERR_NOT_IMPLEMENTED, "PARTITION BY a Boolean key is not supported");
    }
    for (int i = 0; i < norder; i++) {
      int32_t dt = 0;
      ocols.push_back(column(order[i], order_len[i], &dt));
      if (dt == DFGPU_BOOL) fail(DFGPU_ERR_NOT_IMPLEMENTED, "ORDER BY a Boolean key is not supported");
      d.push_back(desc && desc[i] ? 1 : 0);
    }
    std::vector<WinFn> wf;
    for (int k = 0; k < nfns; k++) {
      const dfgpu_agg& f = fns[k];
      WinFn w{f.func, nullptr, 0};
      int want = DFGPU_UINT64;
      if (f.func == DFGPU_AGG_COUNT_DISTINCT) fail(DFGPU_ERR_NOT_IMPLEMENTED, "COUNT(DISTINCT x) OVER (..) is not supported");
      if (!is_rank_fn(f.func)) {
        if (f.func < DFGPU_AGG_MIN || f.func > DFGPU_AGG_AVG) fail(DFGPU_ERR_GENERAL, "Unsupported window function '" + std::to_string(f.func) + "'");
        if (f.arg_len < 1 || !f.arg) fail(DFGPU_ERR_GENERAL, "dfgpu_window: null argument");
        int32_t dt = 0;
        w.arg = column(f.arg, f.arg_len, &dt);
        if (!is_numeric(dt)) fail(DFGPU_ERR_EXECUTION, std::string("Unsupported data type for aggregate: ") + dtype_name(dt));
        want = f.func == DFGPU_AGG_COUNT ? DFGPU_UINT64 : f.func == DFGPU_AGG_AVG ? DFGPU_FLOAT64 : dt;
      }
      w.out_dtype = f.out_dtype ? f.out_dtype : want;
      if (w.out_dtype != want) fail(DFGPU_ERR_EXECUTION, "unexpected type when creating array from aggregate map");
      wf.push_back(w);
    }
    auto res = std::make_unique<dfgpu_result>();
    res->ctx = ctx;
    res->nrows = n;
    if (ctx->world > 1) {
      // the columns the specification reads, from every rank in rank order
      std::vector<const DevColumn*> used;
      auto index = [&](const DevColumn* c) {
        for (size_t i = 0; i < used.size(); i++)
          if (used[i] == c) return i;
        used.push_back(c);
        return used.size() - 1;
      };
      std::vector<size_t> pi, oi, ai;
      for (auto* c : pcols) pi.push_back(index(c));
      for (auto* c : ocols) oi.push_back(index(c));
      for (auto& w : wf) ai.push_back(w.arg ? index(w.arg) : 0);
      dfgpu_batch g;
      long long lo = 0;
      gather_ranks(ctx, n, used, g, &lo);
      for (size_t i = 0; i < pcols.size(); i++) pcols[i] = &g.cols[pi[i]];
      for (size_t i = 0; i < ocols.size(); i++) ocols[i] = &g.cols[oi[i]];
      for (size_t k = 0; k < wf.size(); k++)
        if (wf[k].arg) wf[k].arg = &g.cols[ai[k]];
      window(ctx, g.nrows, pcols, ocols, d, wf, lo, n, res.get());
    } else {
      window(ctx, n, pcols, ocols, d, wf, 0, n, res.get());
    }
    *out = res.release();
  });
}
