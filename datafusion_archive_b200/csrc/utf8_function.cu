// utf8_function.cu — Utf8 functions: upper, lower, trim, ltrim, rtrim, substr, length / char_length, octet_length.
//
// ProgramBuilder::add reduces every maximal nest of DFGPU_OP_UTF8_FN over one Utf8 column to a Utf8View: the byte range
// steps (trim, substr) in order, then one ASCII case map, or a length (expr_compile.cu).  Each step maps a string's byte
// range [b, e) to a sub-range, and the case maps keep both the length and the character boundaries, so a nest of any
// depth is one pass over each string.  Evaluation:
//   - k_utf8_view_len, one thread per row, resolves [b, e) and writes the Int64 result (length, octet_length), or the
//     output length and b.  octet_length of a bare column reads the offsets only.
//   - The lengths become offsets by the Utf8 gather's scan (lengths_to_offsets, utf8_gather.cu).
//   - k_utf8_view_copy, one warp per row like k_utf8_copy, copies [b, e) with the case map applied.  A view that only
//     changes the case of every row of a column without nulls takes the source's offsets, rebased to 0, and skips the
//     length pass and the scan.
// Both kernels take an optional list of row numbers: filter/project evaluates a Utf8 projection over the rows its WHERE
// selected, so the projection's cost follows the selectivity.  The views that predicates, aggregates and keys read are
// evaluated over every row of the batch before the scan (ProgramBuilder::eval_utf8_predicates).
//
// A Utf8 result has i32 offsets from 0, its bytes allocated in whole 16-byte words (the string predicates read aligned
// 16-byte words) and the source's validity; a null row has length 0.  The per-row range code is __host__ __device__:
// dfgpu_utf8_fn_host runs it on one string on the host.
#include <climits>

#include "expr_vm.cuh"

namespace dfgpu {

long long lengths_to_offsets(dfgpu_ctx* ctx, int* offsets, long long n);
void shift_copy_i32(dfgpu_ctx* ctx, int* dst, const int* src, long long n, int add);

namespace {

constexpr int UF_THREADS = 256;

__host__ __device__ __forceinline__ bool is_cont(unsigned char c) { return (c & 0xC0) == 0x80; }

__host__ __device__ __forceinline__ unsigned char map_case(unsigned char c, int m) {
  if (m == DFGPU_UTF8FN_UPPER && c >= 'a' && c <= 'z') return (unsigned char)(c - 32);
  if (m == DFGPU_UTF8FN_LOWER && c >= 'A' && c <= 'Z') return (unsigned char)(c + 32);
  return c;
}

// Apply the view's range steps to the byte range [*pb, *pe) of one string; s(i) is byte i of the buffer.  Each step
// sees its input as a string of its own: its first byte starts a character whatever it is, as LIKE's `_` counts.
template <class Get>
__host__ __device__ void view_range(const Get& s, const Utf8ViewSpec& v, int* pb, int* pe) {
  int b = *pb, e = *pe;
  for (int k = 0; k < v.nsteps; k++) {
    const Utf8Step& st = v.step[k];
    if (st.op == DFGPU_UTF8FN_SUBSTR) {
      // characters at positions [start, start + count) clipped to [1, n]; the sum saturates; count < 0: to the end
      const long long lo = st.start > 1 ? st.start : 1;
      const long long hi = st.count < 0 || st.start > LLONG_MAX - st.count ? LLONG_MAX : st.start + st.count;
      if (hi <= lo) {
        e = b;
        continue;
      }
      long long skip = lo - 1, take = hi - lo;
      int q = b;
      for (; skip > 0 && q < e; skip--) {
        q++;
        while (q < e && is_cont(s(q))) q++;
      }
      int r = q;
      for (; take > 0 && r < e; take--) {
        r++;
        while (r < e && is_cont(s(r))) r++;
      }
      b = q;
      e = r;
    } else {
      if (st.op != DFGPU_UTF8FN_RTRIM)
        while (b < e && s(b) == ' ') b++;
      if (st.op != DFGPU_UTF8FN_LTRIM)
        while (e > b && s(e - 1) == ' ') e--;
    }
  }
  *pb = b;
  *pe = e;
}

// Characters of [b, e): the first byte and every later byte that is not 10xxxxxx
template <class Get>
long long count_chars(const Get& s, int b, int e) {
  long long n = 0;
  for (int q = b; q < e; q++) n += (q == b || !is_cont(s(q))) ? 1 : 0;
  return n;
}

// The same count on the device, four bytes at a time: aligned 32-bit words of a buffer allocated in whole 16-byte words
__device__ __forceinline__ int count_chars_words(const unsigned char* base, int b, int e) {
  if (e <= b) return 0;
  int n = is_cont(__ldg(base + b)) ? 1 : 0;  // a leading continuation byte still starts a character
  for (int q = b & ~3; q < e; q += 4) {
    const unsigned w = __ldg(reinterpret_cast<const unsigned*>(base + q));
    unsigned lead = (~w | (w << 1)) & 0x80808080u;  // bit 7 of each byte: not 10xxxxxx
    if (q < b) lead &= 0xffffffffu << (8 * (b - q));
    if (q + 4 > e) lead &= 0xffffffffu >> (8 * (q + 4 - e));
    n += __popc(lead);
  }
  return n;
}

struct DevBytes {
  const unsigned char* p;
  __device__ __forceinline__ unsigned char operator()(int i) const { return __ldg(p + i); }
};

struct ViewParams {
  const int* off;                  // source offsets
  const unsigned char* bytes;      // source bytes, 16-byte aligned, in whole 16-byte words
  const unsigned char* valid;      // source validity, or null
  const unsigned long long* rows;  // the rows to evaluate, or null: rows 0 .. n-1
  long long n;
  long long* out_int;              // Int64 result per row, or null
  int* out_len;                    // else: the length of row i at out_len[i] ...
  int* begin;                      // ... and its first source byte at begin[i]
  Utf8ViewSpec spec;
};

__global__ void __launch_bounds__(UF_THREADS) k_utf8_view_len(const __grid_constant__ ViewParams p) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += (long long)gridDim.x * blockDim.x) {
    const long long row = p.rows ? (long long)__ldg(p.rows + i) : i;
    int b = 0, e = 0;  // a null row: length 0
    if (!p.valid || ((__ldg(p.valid + (row >> 3)) >> (row & 7)) & 1u)) {
      b = __ldg(p.off + row);
      e = __ldg(p.off + row + 1);
      view_range(DevBytes{p.bytes}, p.spec, &b, &e);
    }
    if (p.out_int) {
      p.out_int[i] = p.spec.result == DFGPU_UTF8FN_OCTET_LENGTH ? e - b : count_chars_words(p.bytes, b, e);
    } else {
      p.out_len[i] = e - b;
      p.begin[i] = b;
    }
  }
}

struct CopyParams {
  const unsigned char* bytes;  // source bytes
  const int* begin;            // first source byte of each output row, or null: src_off[i]
  const int* src_off;
  const int* out_off;
  long long n;
  unsigned char* out;
  int case_map;
};

// one warp per row: copy its range with the case map applied
__global__ void __launch_bounds__(UF_THREADS) k_utf8_view_copy(const __grid_constant__ CopyParams p) {
  const int lane = threadIdx.x & 31;
  const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long i = warp0; i < p.n; i += nwarps) {
    const int s = p.begin ? __ldg(p.begin + i) : __ldg(p.src_off + i);
    const int d = __ldg(p.out_off + i), len = __ldg(p.out_off + i + 1) - d;
    for (int k = lane; k < len; k += 32) p.out[d + k] = map_case(__ldg(p.bytes + s + k), p.case_map);
  }
}

// Evaluate `spec` over rows[0..n) of `src` (rows 0..n-1 when `rows` is null): the Int64 results into out_int, or else the
// Utf8 column into *out (offsets and bytes allocated here; validity is the caller's)
void eval_view(dfgpu_ctx* ctx, const DevColumn& src, const Utf8ViewSpec& spec, const unsigned long long* rows, long long n,
               DevColumn* out, long long* out_int) {
  if (reinterpret_cast<uintptr_t>(src.values) & 15) fail(DFGPU_ERR_INTERNAL, "Utf8 byte buffer not 16-byte aligned");
  ViewParams p;
  memset(&p, 0, sizeof(p));
  p.off = src.offsets;
  p.bytes = (const unsigned char*)src.values;
  p.valid = src.null_count > 0 ? src.validity : nullptr;
  p.rows = rows;
  p.n = n;
  p.spec = spec;
  if (out_int) {
    p.out_int = out_int;
    if (n > 0) launch(ctx, "k_utf8_view_len", k_utf8_view_len, grid_for(ctx, n, UF_THREADS, 16), UF_THREADS, PROFILED, p);
    return;
  }
  out->dtype = DFGPU_UTF8;
  out->offsets = (int32_t*)ctx->alloc(size_t(n + 1) * 4);
  long long total = 0;
  int* begin = nullptr;
  DevBufs scratch(ctx);
  if (n > 0 && spec.nsteps == 0 && !rows && !p.valid) {
    // only the case changes: the source's ranges, rebased to 0
    int lo, hi;
    read_words(ctx, src.offsets, 4, &lo);
    read_words(ctx, src.offsets + n, 4, &hi);
    shift_copy_i32(ctx, out->offsets, src.offsets, n + 1, -lo);
    total = (long long)hi - lo;
  } else if (n > 0) {
    begin = scratch.alloc<int>(size_t(n) * 4);
    p.out_len = out->offsets;
    p.begin = begin;
    launch(ctx, "k_utf8_view_len", k_utf8_view_len, grid_for(ctx, n, UF_THREADS, 16), UF_THREADS, PROFILED, p);
    total = lengths_to_offsets(ctx, out->offsets, n);  // refuses more than 2 GiB
  } else {
    DF_CUDA(cudaMemsetAsync(out->offsets, 0, 4, ctx->stream));
  }
  out->values_bytes = size_t(total);
  out->values = ctx->alloc(std::max<size_t>(16, (size_t(total) + 15) & ~size_t(15)));  // whole 16-byte words
  if (total > 0) {
    CopyParams c;
    c.bytes = p.bytes;
    c.begin = begin;
    c.src_off = src.offsets;
    c.out_off = out->offsets;
    c.n = n;
    c.out = (unsigned char*)out->values;
    c.case_map = spec.case_map;
    launch(ctx, "k_utf8_view_copy", k_utf8_view_copy, grid_for(ctx, n * 32, UF_THREADS, 16), UF_THREADS, PROFILED, c);
  }
}

}  // namespace

void ProgramBuilder::eval_utf8_views(dfgpu_ctx* ctx) {
  const long long n = batch_->nrows;
  for (Utf8View& v : utf8_views_) {
    if (v.projection) continue;  // filter/project evaluates it over the selected rows
    const DevColumn& src = batch_->cols[size_t(v.src)];
    if (v.spec.result) {
      long long* d = (long long*)ctx->alloc(size_t(n > 0 ? n : 1) * 8);
      owned_.push_back(d);
      synth_[size_t(v.synth)].ptr = d;
      eval_view(ctx, src, v.spec, nullptr, n, nullptr, d);
      continue;
    }
    eval_view(ctx, src, v.spec, nullptr, n, &v.out, nullptr);
    owned_.push_back(v.out.offsets);
    owned_.push_back(v.out.values);
    v.out.validity = src.validity;
    v.out.null_count = src.null_count;
    if (v.synth >= 0) synth_[size_t(v.synth)].ptr = v.out.values;
  }
}

void ProgramBuilder::eval_utf8_view_rows(dfgpu_ctx* ctx, int v, const unsigned long long* rows, long long n, DevColumn* out) const {
  const Utf8View& uv = utf8_views_[size_t(v)];
  eval_view(ctx, batch_->cols[size_t(uv.src)], uv.spec, rows, n, out, nullptr);
}

}  // namespace dfgpu

using namespace dfgpu;

extern "C" int dfgpu_utf8_fn_host(const char* s, int64_t s_len, const dfgpu_insn* prog, int prog_len, char* out, int64_t* out_len,
                                  int64_t* out_int, int32_t* out_dtype) {
  return guarded([&] {
    if (s_len < 0 || (!s && s_len > 0) || !prog || prog_len <= 0 || (!out && s_len > 0) || !out_len || !out_int || !out_dtype)
      fail(DFGPU_ERR_GENERAL, "dfgpu_utf8_fn_host: bad argument");
    if (s_len > INT32_MAX) fail(DFGPU_ERR_NOT_IMPLEMENTED, "dfgpu_utf8_fn_host: too long");
    dfgpu_batch schema_only;  // ctx == nullptr: owns nothing
    DevColumn c;
    c.dtype = DFGPU_UTF8;
    schema_only.cols.push_back(c);
    ProgramBuilder pb(&schema_only);
    int view = -1;
    pb.add(prog, prog_len, "expression", &view);
    if (view < 0) {  // an Int64 result: the program is the view's synthetic column alone
      if (pb.utf8_views().size() != 1 || pb.nprogs() != 1 || pb.prog(0).code.size() != 1)
        fail(DFGPU_ERR_GENERAL, "dfgpu_utf8_fn_host: the program is not one Utf8 function nest over column 0");
      view = 0;
    }
    const Utf8ViewSpec& spec = pb.utf8_views()[size_t(view)].spec;
    auto get = [&](int i) { return (unsigned char)s[i]; };
    int b = 0, e = int(s_len);
    view_range(get, spec, &b, &e);
    *out_len = 0;
    *out_int = 0;
    if (spec.result) {
      *out_dtype = DFGPU_INT64;
      *out_int = spec.result == DFGPU_UTF8FN_OCTET_LENGTH ? e - b : count_chars(get, b, e);
    } else {
      *out_dtype = DFGPU_UTF8;
      for (int i = b; i < e; i++) out[i - b] = (char)map_case((unsigned char)s[i], spec.case_map);
      *out_len = e - b;
    }
  });
}
