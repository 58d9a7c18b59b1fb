// utf8_predicate.cu — Utf8 comparisons and LIKE / NOT LIKE, evaluated before an operator's scan.
//
// ProgramBuilder::add recognises every maximal Utf8 comparison or LIKE of a program and turns it into a Boolean
// synthetic column (expr_compile.cu).  ProgramBuilder::eval_utf8_predicates, called once per batch by every operator,
// fills those columns here: one thread per row, a warp per 32 consecutive rows whose results are ballotted into one
// 32-bit word of an LSB-first bitmap without nulls.  The scan kernels read the bitmap like any Boolean column, so none
// of them contains string code.
//
// String bytes are read in aligned 16-byte words and shifted into place with funnel shifts; a read never leaves the
// aligned words that contain the row's bytes, and every Utf8 byte buffer is allocated in whole 16-byte words
// (dfgpu_batch_upload), so a string that ends at the buffer's end is read safely.  The literal (or LIKE segment) is
// copied to the device once per call and staged in shared memory by each CTA, zero-padded to whole 16-byte words.
#include "expr_vm.cuh"
#include "utf8_words.cuh"

namespace dfgpu {

namespace {

constexpr int UP_THREADS = 256;

// LIKE pattern classes; the kernel is specialised by class
enum LikeClass { LIKE_EXACT = 0, LIKE_PREFIX = 1, LIKE_SUFFIX = 2, LIKE_CONTAINS = 3, LIKE_GENERAL = 4 };
const char* const kLikeClassName[] = {"exact", "prefix", "suffix", "contains", "general"};

// A compiled LIKE pattern: the class and the bytes the matcher needs — the one literal segment for exact / prefix /
// suffix / contains, else the whole pattern.
struct LikePattern {
  int cls;
  std::string lit;
};

// Split on '%': no '_' and at most a leading and a trailing run of '%' around one segment gives one of the four
// literal classes; everything else is general.  A pattern of '%' only is the prefix ''.
LikePattern compile_like(const std::string& p) {
  if (p.find('_') == std::string::npos) {
    size_t a = 0, b = 0;
    while (a < p.size() && p[a] == '%') a++;
    if (a == p.size()) return {p.empty() ? LIKE_EXACT : LIKE_PREFIX, std::string()};
    while (p[p.size() - 1 - b] == '%') b++;
    const std::string core = p.substr(a, p.size() - a - b);
    if (core.find('%') == std::string::npos) {
      if (a == 0 && b == 0) return {LIKE_EXACT, core};
      if (a == 0) return {LIKE_PREFIX, core};
      if (b == 0) return {LIKE_SUFFIX, core};
      return {LIKE_CONTAINS, core};
    }
  }
  return {LIKE_GENERAL, p};
}

// The general matcher, shared by the kernel and dfgpu_utf8_like_host.  `s(i)` is byte i of the string (n bytes).
// A segment item '_' takes one byte and the continuation bytes (10xxxxxx) after it; any other byte matches itself.
// Returns the end of the segment pat[i, j) matched at string position q, or -1.
template <class Get>
__host__ __device__ __forceinline__ int match_seg(const Get& s, int n, int q, const unsigned char* pat, int i, int j) {
  for (int k = i; k < j; k++) {
    if (q >= n) return -1;
    if (pat[k] == '_') {
      q++;
      while (q < n && (s(q) & 0xC0) == 0x80) q++;
    } else {
      if (s(q) != pat[k]) return -1;
      q++;
    }
  }
  return q;
}

// The first segment is anchored at the start, the last at the end; each middle segment is matched at its leftmost
// position.  A segment's end does not decrease as its start moves right and '%' is the only variable-length wildcard,
// so the leftmost match (the earliest end) never loses a match that a later one would find.
template <class Get>
__host__ __device__ bool like_general(const Get& s, int n, const unsigned char* pat, int m) {
  int first = 0;
  while (first < m && pat[first] != '%') first++;
  if (first == m) return match_seg(s, n, 0, pat, 0, m) == n;
  int pos = match_seg(s, n, 0, pat, 0, first);
  if (pos < 0) return false;
  int last = m;
  while (pat[last - 1] != '%') last--;  // the last segment is pat[last, m)
  for (int i = first + 1; i < last;) {
    int j = i;
    while (pat[j] != '%') j++;
    if (j > i) {
      int e = -1;
      for (int q = pos; q < n && e < 0; q++) e = match_seg(s, n, q, pat, i, j);
      if (e < 0) return false;
      pos = e;
    }
    i = j + 1;
  }
  if (last == m) return true;
  for (int q = pos; q <= n; q++)
    if (match_seg(s, n, q, pat, last, m) == n) return true;
  return false;
}

struct Utf8PredParams {
  const int* aoff;             // rebased i32 offsets of the left column
  const unsigned char* abytes; // its bytes, 16-byte aligned, allocated in whole 16-byte words
  const unsigned char* avalid; // LSB-first validity or null
  const int* boff;             // right column (column against column), else null
  const unsigned char* bbytes;
  const unsigned char* bvalid;
  const unsigned char* lit;    // device copy of the literal / LIKE segment / general pattern
  int lit_len;
  int op;                      // DFGPU_OP_EQ .. DFGPU_OP_GE; LIKE, NOT_LIKE: (not) equal / (not) matched, false on a null
  long long n;
  unsigned* out;               // ceil(n / 32) words
};

__device__ __forceinline__ bool valid_bit(const unsigned char* v, long long row) {
  return !v || ((__ldg(v + (row >> 3)) >> (row & 7)) & 1u);
}

// A string in global memory: `len` bytes from byte `start` of `base`
struct GStr {
  const unsigned char* base;
  long long start;
  int len;
  __device__ __forceinline__ uint4 get16(int i) const { return load16(base, start + i, len - i); }
  __device__ __forceinline__ unsigned char operator()(int i) const { return __ldg(base + start + i); }
};
// The literal, staged in shared memory (16-byte aligned, zero-padded); read at multiples of 16 only
struct SLit {
  const unsigned char* s;
  __device__ __forceinline__ uint4 get16(int i) const { return *reinterpret_cast<const uint4*>(s + i); }
};

// Byte difference (x - y) at the first of the first k (1..16) bytes where x and y differ, else 0
__device__ __forceinline__ int diff_word(unsigned x, unsigned y, int k) {
  const unsigned m = k >= 4 ? 0xffffffffu : (1u << (8 * k)) - 1u;
  const unsigned d = (x ^ y) & m;
  if (!d) return 0;
  const int b = (__ffs(int(d)) - 1) & ~7;
  return int((x >> b) & 0xffu) - int((y >> b) & 0xffu);
}
__device__ __forceinline__ int diff16(uint4 x, uint4 y, int k) {
  int d = diff_word(x.x, y.x, k);
  if (d || k <= 4) return d;
  d = diff_word(x.y, y.y, k - 4);
  if (d || k <= 8) return d;
  d = diff_word(x.z, y.z, k - 8);
  if (d || k <= 12) return d;
  return diff_word(x.w, y.w, k - 12);
}

// Byte-wise comparison of the first k bytes of a and b, up to the first difference: < 0, 0, > 0
template <class A, class B>
__device__ __forceinline__ int compare_prefix(const A& a, const B& b, int k) {
  for (int i = 0; i < k; i += 16) {
    const int d = diff16(a.get16(i), b.get16(i), min(16, k - i));
    if (d) return d;
  }
  return 0;
}

__device__ __forceinline__ bool apply_cmp(int op, int c) {
  switch (op) {
    case DFGPU_OP_EQ: case DFGPU_OP_LIKE: return c == 0;
    case DFGPU_OP_NE: case DFGPU_OP_NOT_LIKE: return c != 0;
    case DFGPU_OP_LT: return c < 0;
    case DFGPU_OP_LE: return c <= 0;
    case DFGPU_OP_GT: return c > 0;
    default: return c >= 0;
  }
}

// Stage the literal in shared memory, zero-padded to whole 16-byte words
__device__ __forceinline__ void stage_literal(unsigned char* s_lit, const Utf8PredParams& p) {
  const int padded = (p.lit_len + 15) & ~15;
  for (int i = threadIdx.x; i < padded; i += blockDim.x) s_lit[i] = i < p.lit_len ? p.lit[i] : 0;
  __syncthreads();
}

// Runs `eval(row)` for every row, a warp per 32 consecutive rows, and stores the warp's ballot as one bitmap word
template <class F>
__device__ __forceinline__ void for_each_word(const Utf8PredParams& p, const F& eval) {
  const int lane = threadIdx.x & 31;
  const long long nwords = (p.n + 31) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < nwords; w += nwarps) {
    const long long row = (w << 5) + lane;
    const bool r = row < p.n && eval(row);
    const unsigned bits = __ballot_sync(0xffffffffu, r);
    if (lane == 0) p.out[w] = bits;
  }
}

// x op y.  ORDER = false: = / <> (and an exact LIKE), decided on the lengths alone wherever they differ;
// ORDER = true: < <= > >=.  RCOL: y is a second column, else the literal.
template <bool ORDER, bool RCOL>
__global__ void __launch_bounds__(UP_THREADS) k_utf8_cmp(const __grid_constant__ Utf8PredParams p) {
  __shared__ __align__(16) unsigned char s_lit[RCOL ? 16 : DFGPU_UTF8_LITERAL_MAX];
  if (!RCOL) stage_literal(s_lit, p);
  const bool like = p.op == DFGPU_OP_LIKE || p.op == DFGPU_OP_NOT_LIKE;
  for_each_word(p, [&](long long row) {
    const bool va = valid_bit(p.avalid, row), vb = !RCOL || valid_bit(p.bvalid, row);
    int c;
    if (!va || !vb) {
      if (like) return false;  // a null satisfies neither LIKE nor NOT LIKE
      c = int(va) - int(vb);   // null equals null and orders below every string
    } else {
      const int a0 = __ldg(p.aoff + row), la = __ldg(p.aoff + row + 1) - a0;
      const GStr a{p.abytes, a0, la};
      int lb;
      if (RCOL) {
        const int b0 = __ldg(p.boff + row);
        lb = __ldg(p.boff + row + 1) - b0;
        const GStr b{p.bbytes, b0, lb};
        if (!ORDER) c = la != lb ? 1 : compare_prefix(a, b, la);
        else c = compare_prefix(a, b, min(la, lb));
      } else {
        lb = p.lit_len;
        const SLit b{s_lit};
        if (!ORDER) c = la != lb ? 1 : compare_prefix(a, b, la);
        else c = compare_prefix(a, b, min(la, lb));
      }
      if (ORDER && c == 0) c = la - lb;  // a proper prefix orders first
    }
    return apply_cmp(p.op, c);
  });
}

// x LIKE p / x NOT LIKE p (p.op) for the pattern classes other than exact
template <int CLASS>
__global__ void __launch_bounds__(UP_THREADS) k_utf8_like(const __grid_constant__ Utf8PredParams p) {
  __shared__ __align__(16) unsigned char s_lit[DFGPU_UTF8_LITERAL_MAX];
  stage_literal(s_lit, p);
  const bool neg = p.op == DFGPU_OP_NOT_LIKE;
  for_each_word(p, [&](long long row) {
    if (!valid_bit(p.avalid, row)) return false;  // a null satisfies neither LIKE nor NOT LIKE
    const int a0 = __ldg(p.aoff + row), la = __ldg(p.aoff + row + 1) - a0;
    const int m = p.lit_len;
    const SLit l{s_lit};
    bool hit;
    if (CLASS == LIKE_PREFIX) {
      hit = la >= m && compare_prefix(GStr{p.abytes, a0, la}, l, m) == 0;
    } else if (CLASS == LIKE_SUFFIX) {
      hit = la >= m && compare_prefix(GStr{p.abytes, (long long)a0 + la - m, m}, l, m) == 0;
    } else if (CLASS == LIKE_CONTAINS) {
      hit = m == 0;
      for (int q = 0; q + m <= la && !hit && m > 0; q++) hit = compare_prefix(GStr{p.abytes, (long long)a0 + q, la - q}, l, m) == 0;
    } else {
      hit = like_general(GStr{p.abytes, a0, la}, la, s_lit, m);
    }
    return hit != neg;
  });
}

const char* cmp_name(int op) {
  switch (op) {
    case DFGPU_OP_LT: return "lt";
    case DFGPU_OP_LE: return "le";
    case DFGPU_OP_GT: return "gt";
    default: return "ge";
  }
}

}  // namespace

ProgramBuilder::~ProgramBuilder() {
  for (void* q : owned_) ctx_->free(q);
}

void ProgramBuilder::eval_utf8_predicates(dfgpu_ctx* ctx) {
  utf8_evaluated_ = true;
  ctx_ = ctx;
  const long long n = batch_->nrows;
  eval_utf8_views(ctx);  // a predicate may read a view
  for (const Utf8Pred& sp : utf8_preds_) {
    const size_t words = size_t((n + 31) / 32);
    unsigned* bits = (unsigned*)ctx->alloc((words ? words : 1) * 4);
    owned_.push_back(bits);
    synth_[size_t(sp.synth)].ptr = bits;
    if (n == 0) continue;
    const bool like = sp.op == DFGPU_OP_LIKE || sp.op == DFGPU_OP_NOT_LIKE;
    const LikePattern lp = like ? compile_like(sp.lit) : LikePattern{LIKE_EXACT, sp.lit};
    Utf8PredParams p;
    memset(&p, 0, sizeof(p));
    auto bind = [&](int ref, const int** off, const unsigned char** bytes, const unsigned char** valid) {
      const DevColumn& c = ref >= 0 ? batch_->cols[size_t(ref)] : utf8_views_[size_t(-2 - ref)].out;
      if (reinterpret_cast<uintptr_t>(c.values) & 15) fail(DFGPU_ERR_INTERNAL, "Utf8 byte buffer not 16-byte aligned");
      *off = c.offsets;
      *bytes = (const unsigned char*)c.values;
      *valid = c.null_count > 0 ? c.validity : nullptr;
    };
    bind(sp.a, &p.aoff, &p.abytes, &p.avalid);
    const bool rcol = sp.b != -1;
    if (rcol) bind(sp.b, &p.boff, &p.bbytes, &p.bvalid);
    p.op = sp.op;
    p.n = n;
    p.out = bits;
    if (!rcol) {
      p.lit_len = int(lp.lit.size());
      unsigned char* d = (unsigned char*)ctx->alloc(lp.lit.size() + 16);
      owned_.push_back(d);
      if (!lp.lit.empty()) DF_CUDA(cudaMemcpyAsync(d, lp.lit.data(), lp.lit.size(), cudaMemcpyHostToDevice, ctx->stream));
      p.lit = d;
    }
    const int grid = grid_for(ctx, n, UP_THREADS, 16);
    if (like && lp.cls != LIKE_EXACT) {
      const std::string name = std::string("k_utf8_like<") + kLikeClassName[lp.cls] + ">";
      switch (lp.cls) {
        case LIKE_PREFIX: launch(ctx, name.c_str(), k_utf8_like<LIKE_PREFIX>, grid, UP_THREADS, PROFILED, p); break;
        case LIKE_SUFFIX: launch(ctx, name.c_str(), k_utf8_like<LIKE_SUFFIX>, grid, UP_THREADS, PROFILED, p); break;
        case LIKE_CONTAINS: launch(ctx, name.c_str(), k_utf8_like<LIKE_CONTAINS>, grid, UP_THREADS, PROFILED, p); break;
        default: launch(ctx, name.c_str(), k_utf8_like<LIKE_GENERAL>, grid, UP_THREADS, PROFILED, p); break;
      }
    } else if (like || sp.op == DFGPU_OP_EQ || sp.op == DFGPU_OP_NE) {
      const std::string name = std::string("k_utf8_cmp<eq, ") + (rcol ? "col>" : "lit>");
      if (rcol) launch(ctx, name.c_str(), k_utf8_cmp<false, true>, grid, UP_THREADS, PROFILED, p);
      else launch(ctx, name.c_str(), k_utf8_cmp<false, false>, grid, UP_THREADS, PROFILED, p);
    } else {
      const std::string name = std::string("k_utf8_cmp<") + cmp_name(sp.op) + ", " + (rcol ? "col>" : "lit>");
      if (rcol) launch(ctx, name.c_str(), k_utf8_cmp<true, true>, grid, UP_THREADS, PROFILED, p);
      else launch(ctx, name.c_str(), k_utf8_cmp<true, false>, grid, UP_THREADS, PROFILED, p);
    }
  }
}

}  // namespace dfgpu

using namespace dfgpu;

extern "C" int dfgpu_utf8_like_host(const char* s, int64_t s_len, const char* pattern, int64_t pattern_len, int32_t* match, int32_t* pattern_class) {
  return guarded([&] {
    if (s_len < 0 || pattern_len < 0 || (!s && s_len > 0) || (!pattern && pattern_len > 0) || !match || !pattern_class)
      fail(DFGPU_ERR_GENERAL, "dfgpu_utf8_like_host: bad argument");
    if (pattern_len > DFGPU_UTF8_LITERAL_MAX || s_len > INT32_MAX) fail(DFGPU_ERR_NOT_IMPLEMENTED, "dfgpu_utf8_like_host: too long");
    const std::string str(s ? s : "", size_t(s_len));
    const LikePattern lp = compile_like(std::string(pattern ? pattern : "", size_t(pattern_len)));
    bool hit;
    switch (lp.cls) {
      case LIKE_EXACT: hit = str == lp.lit; break;
      case LIKE_PREFIX: hit = str.compare(0, lp.lit.size(), lp.lit) == 0 && str.size() >= lp.lit.size(); break;
      case LIKE_SUFFIX: hit = str.size() >= lp.lit.size() && str.compare(str.size() - lp.lit.size(), lp.lit.size(), lp.lit) == 0; break;
      case LIKE_CONTAINS: hit = str.find(lp.lit) != std::string::npos; break;
      default: {
        auto get = [&](int i) { return (unsigned char)str[size_t(i)]; };
        hit = like_general(get, int(str.size()), reinterpret_cast<const unsigned char*>(lp.lit.data()), int(lp.lit.size()));
      }
    }
    *match = hit ? 1 : 0;
    *pattern_class = lp.cls;
  });
}
