// expr_vm.cuh — the expression "compiler" and its device-side evaluator.
//
// The reference compiles an `Expr` tree into nested closures, one temporary Arrow array per node
// and one N-row literal array per literal (src/execution/expression.rs:283-505, 226-243).  Here the
// postfix program from the C ABI is type-checked on the host, lowered to a tiny register-stack
// bytecode whose right-hand leaf operands (literals, columns) are folded into the consuming
// instruction, and interpreted INSIDE the scan kernels, R rows per thread at a time, with the
// operand stack held in registers.  All control flow of the interpreter is warp-uniform (every
// thread runs the same program), so it costs a few scalar instructions per op per R rows; no
// intermediate array is ever written to HBM.
#pragma once
#include "common.cuh"

namespace dfgpu {

enum MType : uint8_t { MT_NONE = 0, MT_F64 = 1, MT_F32 = 2, MT_I = 3, MT_U = 4, MT_BOOL = 5 };
enum VOp : uint8_t {
  V_PUSH_COL = 0, V_PUSH_IMM, V_PUSH_ROWID /* global row number (gather index of variable-width columns) */, V_CAST,
  V_ADD, V_SUB, V_MUL, V_DIV,
  V_EQ, V_NE, V_LT, V_LE, V_GT, V_GE,
  V_AND, V_OR,
  V_RSUB, V_RDIV,  // operands exchanged (emitted for stack-mode instructions only, see expr_compile.cu)
  // scalar functions (DFGPU_OP_FN), Float64 only, `aux` = DFGPU_FN_* code: V_FN applies a one-argument function to the
  // accumulator like V_CAST, V_FN2 / V_RFN2 a two-argument one in any RhsMode (V_RFN2: operands exchanged)
  V_FN, V_FN2, V_RFN2,
  // CASE (DFGPU_OP_CASE), lowered as a fold backward from the ELSE (expr_compile.cu).  Stack operands only, the
  // accumulator holding the THEN value v, the entry below it the condition c:
  //   V_SEL   pops c and the fold so far e below it: c ? v : e
  //   V_SEL0  (the last WHEN of a CASE without ELSE) pops c: c ? v : null
  // A condition is taken when it is true and valid.
  V_SEL, V_SEL0
};
// The interpreter kernels' DEPTH template argument is the register-stack depth (1, 2, 4 or 8), kFnDepth for a program set
// that contains V_FN* (has_fn below): depth 8 with the scalar functions compiled in, or kCaseDepth for a set that contains
// V_SEL* (has_case): the extended interpreter, depth 8 with the scalar functions, CASE, validity tracking and per-entry
// error bits.  Only those instantiations contain that code, so the kernels that run other queries keep theirs: CASE's
// bookkeeping costs a function-only query nothing.
constexpr int kFnDepth = 9;
constexpr int kCaseDepth = 10;
inline std::string depth_arg(int depth) {
  return depth == kFnDepth ? "kFnDepth" : depth == kCaseDepth ? "kCaseDepth" : std::to_string(depth);
}
enum RhsMode : uint8_t { RHS_STACK = 0, RHS_IMM = 1, RHS_COL = 2 };

struct __align__(16) DevInsn {   // 16 bytes, lives in kernel parameter (constant) space
  uint8_t op;      // VOp
  uint8_t mode;    // RhsMode for binary ops
  uint8_t mtype;   // machine type of the operands (CAST: of the source)
  uint8_t dtype;   // Arrow dtype of the operands (int width for wrap-around); CAST: target dtype
  int16_t slot;    // column slot for PUSH_COL / RHS_COL
  int16_t aux;     // CAST: source dtype; V_FN*: DFGPU_FN_* code
  unsigned long long imm;  // PUSH_IMM / RHS_IMM payload (raw bits, already widened)
};

constexpr int kMaxInsn = 96;
constexpr int kMaxProgs = 24;
constexpr int kMaxCols = 12;

struct ColRef {
  const void* ptr;
  const unsigned char* validity;  // LSB-first bitmap re-based to row 0, or null when the column has no nulls
  int dtype;
  int _pad;
};

struct ProgramSet {
  DevInsn insn[kMaxInsn];
  ColRef cols[kMaxCols];
  uint8_t start[kMaxProgs + 1];
  uint8_t out_dtype[kMaxProgs];
  int nprog;
  int ncols;
  int max_depth;
  int f64_only;  // every operand Float64/Boolean and no CAST: the lean evaluator applies
  int has_nulls; // some referenced column carries a validity bitmap, or some program's result can be a CASE-made null
                 // (CompiledProgram::makes_nulls): kernels use the NULLS evaluator
  uint8_t nullable[kMaxProgs];  // program result can be null (arrow 0.12 array_ops semantics)
};
// Some program of the set calls a scalar function or has a CASE (V_FN*, V_SEL*): its kernels run with DEPTH = kFnDepth,
// or kCaseDepth when has_case.  Read from the code rather than stored, so that the kernel parameter blocks keep their
// layout.
inline bool has_fn(const ProgramSet& ps) {
  for (int pc = 0; pc < ps.start[ps.nprog]; pc++)
    if (ps.insn[pc].op >= V_FN) return true;
  return false;
}
inline bool has_case(const ProgramSet& ps) {
  for (int pc = 0; pc < ps.start[ps.nprog]; pc++)
    if (ps.insn[pc].op >= V_SEL) return true;
  return false;
}
// Some program of the set divides: the only instruction whose kernels can raise an error (DivideByZero, for integers and
// floats alike).  A set without one cannot fail once its kernel is launched.
inline bool has_div(const ProgramSet& ps) {
  for (int pc = 0; pc < ps.start[ps.nprog]; pc++)
    if (ps.insn[pc].op == V_DIV || ps.insn[pc].op == V_RDIV) return true;
  return false;
}

// Interpreter-free shapes.  ProgramBuilder::add recognises them; the operators pass them to kernels that evaluate them
// with straight-line code (same arithmetic as the interpreter, no decode in the inner loop).
// One leaf: a column copy, or one operation whose left operand is a column and whose right operand is a column or an
// immediate, both of one 4- or 8-byte numeric dtype.
struct Leaf {
  int kind;       // 0 = none (use the interpreter), 1 = copy column a, 2 = a op column b, 3 = a op imm
  int op;         // VOp
  int a, b;       // column slots (b: kind 2 only, else 0)
  int dtype;      // Arrow dtype of the operands (of the column, for a copy: any fixed width)
  uint8_t mtype;  // machine type of the operands
  uint8_t conn;   // in a chain: joins the running result with this leaf, 0 = AND, 1 = OR
  unsigned long long imm;  // kind 3: raw bits, widened like DevInsn::imm
};
// Up to 4 comparison leaves evaluated left to right: term[0] [conn term[1] [conn term[2] [conn term[3]]]]
struct LeafChain {
  int nterms;  // 0 = not a chain
  Leaf term[4];
};
static_assert(sizeof(Leaf) == 32 && sizeof(LeafChain) == 136, "FPParams and AggParams carry chains and leaves: keep them compact");

// ---- host side ----------------------------------------------------------------------------
struct CompiledProgram {
  std::vector<DevInsn> code;
  bool nullable = false;
  bool makes_nulls = false;  // nullable, and has a CASE without ELSE: can be null even where every input column is valid
  int out_dtype = 0;
  int max_depth = 0;
  Leaf leaf{};        // kind 1: the program is exactly one column; 2 / 3: one + - * / (no integer division, no
                      // arithmetic on integers narrower than 64 bits); else kind 0
  LeafChain chain{};  // nterms > 0: the program is a chain of comparisons joined by AND / OR
};

// A Utf8 comparison or LIKE that ProgramBuilder::add recognised.  It is evaluated before the operator's scan, into a
// bit-packed Boolean column without nulls (utf8_predicate.cu), and the program reads that column as synthetic column
// `synth`.  No string code runs inside the scan kernels.
struct Utf8Pred {
  int op;           // DFGPU_OP_EQ .. DFGPU_OP_GE (a literal on the left already mirrored), DFGPU_OP_LIKE, DFGPU_OP_NOT_LIKE
  int a, b;         // operands: a batch column c >= 0, or Utf8 view v as -2 - v; b == -1: a op lit
  std::string lit;  // the literal, or the LIKE pattern (a copy: the program's bytes are borrowed)
  int synth;        // synthetic column index
};

// A nest of Utf8 functions (DFGPU_OP_UTF8_FN) over one Utf8 column, reduced to one view of each string: the range steps
// in order, innermost first, then the outermost case map.  The ASCII case maps keep the length and the character
// boundaries, so they commute with every range step.  utf8_function.cu evaluates it.
constexpr int kMaxUtf8Steps = 16;
struct Utf8Step {
  int op;           // DFGPU_UTF8FN_TRIM / _LTRIM / _RTRIM / _SUBSTR (SUBSTR_FROM is SUBSTR with count -1)
  long long start;  // SUBSTR: 1-based first character
  long long count;  // SUBSTR: characters; -1: to the end
};
struct Utf8ViewSpec {
  int nsteps;
  int case_map;     // 0 none, DFGPU_UTF8FN_UPPER, DFGPU_UTF8FN_LOWER
  int result;       // 0: the Utf8 string; DFGPU_UTF8FN_LENGTH / _OCTET_LENGTH: its length as Int64
  Utf8Step step[kMaxUtf8Steps];
};
struct Utf8View {
  int src;            // batch column (Utf8)
  Utf8ViewSpec spec;
  int synth;          // synthetic column the programs read (Int64 results, a Utf8 program result), else -1
  bool projection;    // a Utf8 projection: filter/project evaluates it over the selected rows, not before the scan
  DevColumn out;      // Utf8 result of eval_utf8_predicates (offsets from 0, bytes in whole 16-byte words)
};

class ProgramBuilder {
 public:
  explicit ProgramBuilder(const dfgpu_batch* batch) : batch_(batch) {}
  ProgramBuilder(const ProgramBuilder&) = delete;
  ProgramBuilder& operator=(const ProgramBuilder&) = delete;
  ~ProgramBuilder();  // returns the predicate bitmaps and view columns to the ctx pool
  // Type-check + lower one postfix program; appends to the set and returns its index.  With `utf8_view`, a program whose
  // value is a Utf8 function nest is not appended: it is recorded as a projection view, *utf8_view receives its index
  // and -1 is returned (else *utf8_view = -1).
  int add(const dfgpu_insn* p, int n, const char* what, int* utf8_view = nullptr);
  // Program yielding the global row number (UInt64): the gather index for variable-width columns.
  int add_rowid();
  // Program yielding `bias + global row number` (UInt64).
  int add_rowid_plus(unsigned long long bias);
  // Program that just reads a device array which is not a column of the batch (e.g. key hashes).
  int add_synthetic_column(const void* dptr, int dtype);
  int out_dtype(int prog) const { return progs_[size_t(prog)].out_dtype; }
  const CompiledProgram& prog(int i) const { return progs_[size_t(i)]; }
  int nprogs() const { return int(progs_.size()); }
  // Finalise into the POD passed to kernels.
  void finish(ProgramSet* out) const;
  int slot_of_column(int col);
  // Evaluate the recognised Utf8 predicates over the batch on ctx->stream and point their synthetic columns at the
  // bitmaps (utf8_predicate.cu).  Every operator calls it once per batch, after the last add() and before finish().
  // The Utf8 function views are evaluated first (utf8_function.cu), the predicates after, so a predicate may read a view.
  void eval_utf8_predicates(dfgpu_ctx* ctx);
  const std::vector<Utf8Pred>& utf8_preds() const { return utf8_preds_; }
  const std::vector<Utf8View>& utf8_views() const { return utf8_views_; }
  // Evaluate projection view `v` over the rows `rows[0..n)` of the batch (all n rows when `rows` is null) into *out,
  // a column the caller owns (utf8_function.cu).
  void eval_utf8_view_rows(dfgpu_ctx* ctx, int v, const unsigned long long* rows, long long n, DevColumn* out) const;

 private:
  int new_synth(const void* dptr, int dtype, int src = -1);  // a synthetic column slot; returns the synthetic index
  bool synth_nullable(int k) const;
  void eval_utf8_views(dfgpu_ctx* ctx);  // every view but the projections, before the predicates (utf8_function.cu)
  const dfgpu_batch* batch_;
  std::vector<Utf8Pred> utf8_preds_;
  std::vector<Utf8View> utf8_views_;
  bool utf8_evaluated_ = false;
  dfgpu_ctx* ctx_ = nullptr;  // of owned_
  std::vector<void*> owned_;  // device bitmaps and literals of utf8_preds_, columns of utf8_views_
  std::vector<CompiledProgram> progs_;
  std::vector<int> slots_;  // slot -> batch column index, or -1 - k for synthetic column k
  // src >= 0: the synthetic column is null where batch column `src` is (a Utf8 function's result)
  struct Synth { const void* ptr; int dtype; int src; };
  std::vector<Synth> synth_;
};

MType mtype_of(int dtype);

#ifdef __CUDACC__
// ---- device side ---------------------------------------------------------------------------
__device__ __forceinline__ double u2d(unsigned long long x) { return __longlong_as_double((long long)x); }
__device__ __forceinline__ unsigned long long d2u(double x) { return (unsigned long long)__double_as_longlong(x); }
__device__ __forceinline__ float u2f(unsigned long long x) { return __uint_as_float((unsigned)x); }
__device__ __forceinline__ unsigned long long f2u(float x) { return (unsigned long long)__float_as_uint(x); }

// wrap a 64-bit integer result to the width of `dtype` (Rust release-mode wrapping arithmetic)
__device__ __forceinline__ unsigned long long norm_int(unsigned long long x, int dtype) {
  switch (dtype) {
    case DFGPU_INT8: return (unsigned long long)(long long)(signed char)x;
    case DFGPU_INT16: return (unsigned long long)(long long)(short)x;
    case DFGPU_INT32: return (unsigned long long)(long long)(int)x;
    case DFGPU_UINT8: return x & 0xffull;
    case DFGPU_UINT16: return x & 0xffffull;
    case DFGPU_UINT32: return x & 0xffffffffull;
    default: return x;
  }
}

// load element `row` of a column, widened to the 64-bit machine representation
__device__ __forceinline__ unsigned long long load_elem(const void* p, int dtype, long long row) {
  switch (dtype) {
    case DFGPU_FLOAT64: case DFGPU_INT64: case DFGPU_UINT64: return __ldg((const unsigned long long*)p + row);
    case DFGPU_FLOAT32: case DFGPU_UINT32: return (unsigned long long)__ldg((const unsigned*)p + row);
    case DFGPU_INT32: return (unsigned long long)(long long)__ldg((const int*)p + row);
    case DFGPU_INT16: return (unsigned long long)(long long)__ldg((const short*)p + row);
    case DFGPU_UINT16: return (unsigned long long)__ldg((const unsigned short*)p + row);
    case DFGPU_INT8: return (unsigned long long)(long long)__ldg((const signed char*)p + row);
    case DFGPU_UINT8: return (unsigned long long)__ldg((const unsigned char*)p + row);
    case DFGPU_BOOL:  // BooleanArray values: bit-packed, LSB first (boolean_ops! operands, expression.rs:212-224)
      return (unsigned long long)((__ldg((const unsigned char*)p + (row >> 3)) >> (row & 7)) & 1u);
    default: return 0;
  }
}

// same, through a generic pointer (shared-memory staged tiles)
__device__ __forceinline__ unsigned long long load_elem_generic(const void* p, int dtype, int idx) {
  switch (dtype) {
    case DFGPU_FLOAT64: case DFGPU_INT64: case DFGPU_UINT64: return ((const unsigned long long*)p)[idx];
    case DFGPU_FLOAT32: case DFGPU_UINT32: return (unsigned long long)((const unsigned*)p)[idx];
    case DFGPU_INT32: return (unsigned long long)(long long)((const int*)p)[idx];
    case DFGPU_INT16: return (unsigned long long)(long long)((const short*)p)[idx];
    case DFGPU_UINT16: return (unsigned long long)((const unsigned short*)p)[idx];
    case DFGPU_INT8: return (unsigned long long)(long long)((const signed char*)p)[idx];
    case DFGPU_UINT8: return (unsigned long long)((const unsigned char*)p)[idx];
    default: return 0;
  }
}

// Operand sources for the evaluator.  GlobalRows: R arbitrary row indices straight from HBM
// (-1 = past the end).  StagedTile: rows lrow0 + r*32 of a tile staged in shared memory, columns
// laid out back to back at col_off[slot]; validity comes from `valid` (bit r).
// 64-bit read-only load with an L2 eviction policy (createpolicy.fractional.L2::evict_first for
// columns that are streamed exactly once)
__device__ __forceinline__ unsigned long long ld_stream_u64(const unsigned long long* p, unsigned long long policy) {
  unsigned long long v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.b64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(policy));
  return v;
}
__device__ __forceinline__ unsigned long long l2_evict_first_policy() {
  unsigned long long pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}

template <int R>
struct GlobalRows {
  long long rows[R];
  unsigned valid;
  unsigned long long l2_policy = 0;  // createpolicy word for the 64-bit column loads; 0 = default caching
  __device__ __forceinline__ unsigned long long load(const ProgramSet& ps, int slot, int r) const {
    return rows[r] >= 0 ? load_elem(ps.cols[slot].ptr, ps.cols[slot].dtype, rows[r]) : 0ull;
  }
  // all R rows of a column: the dtype dispatch is warp-uniform and paid once, not per row
  __device__ __forceinline__ void load_rows(const ProgramSet& ps, int slot, unsigned long long (&out)[R]) const {
    const void* base = ps.cols[slot].ptr;
    switch (ps.cols[slot].dtype) {
      case DFGPU_FLOAT64: case DFGPU_INT64: case DFGPU_UINT64:
        if (l2_policy) {  // streamed once: do not let the input push a hash table out of L2
#pragma unroll
          for (int r = 0; r < R; r++) out[r] = rows[r] >= 0 ? ld_stream_u64((const unsigned long long*)base + rows[r], l2_policy) : 0ull;
        } else {
#pragma unroll
          for (int r = 0; r < R; r++) out[r] = rows[r] >= 0 ? __ldg((const unsigned long long*)base + rows[r]) : 0ull;
        }
        break;
      case DFGPU_FLOAT32: case DFGPU_UINT32:
#pragma unroll
        for (int r = 0; r < R; r++) out[r] = rows[r] >= 0 ? (unsigned long long)__ldg((const unsigned*)base + rows[r]) : 0ull;
        break;
      case DFGPU_INT32:
#pragma unroll
        for (int r = 0; r < R; r++) out[r] = rows[r] >= 0 ? (unsigned long long)(long long)__ldg((const int*)base + rows[r]) : 0ull;
        break;
      default:
#pragma unroll
        for (int r = 0; r < R; r++) out[r] = load(ps, slot, r);
        break;
    }
  }
  __device__ __forceinline__ unsigned long long rowid(int r) const { return (unsigned long long)rows[r]; }
  // bit r = row r of this thread is non-null in column `slot`
  __device__ __forceinline__ unsigned col_valid(const ProgramSet& ps, int slot) const {
    const unsigned char* vb = ps.cols[slot].validity;
    if (!vb) return (1u << R) - 1u;
    unsigned m = 0;
#pragma unroll
    for (int r = 0; r < R; r++)
      if (rows[r] >= 0 && ((vb[rows[r] >> 3] >> (rows[r] & 7)) & 1)) m |= 1u << r;
    return m;
  }
};
template <int R>
struct StagedTile {
  const unsigned char* stage;
  const int* col_off;
  int lrow0;
  unsigned valid;
  long long row0;  // global row number of (tile, lrow0)
  __device__ __forceinline__ unsigned long long load(const ProgramSet& ps, int slot, int r) const {
    return load_elem_generic(stage + col_off[slot], ps.cols[slot].dtype, lrow0 + r * 32);
  }
  // all R rows of a staged column: the dtype dispatch is warp-uniform and paid once, not per row
  __device__ __forceinline__ void load_rows(const ProgramSet& ps, int slot, unsigned long long (&out)[R]) const {
    const unsigned char* base = stage + col_off[slot];
    switch (ps.cols[slot].dtype) {
      case DFGPU_FLOAT64: case DFGPU_INT64: case DFGPU_UINT64: {
        const unsigned long long* p = (const unsigned long long*)base + lrow0;
#pragma unroll
        for (int r = 0; r < R; r++) out[r] = p[r * 32];
        break;
      }
      case DFGPU_FLOAT32: case DFGPU_UINT32: {
        const unsigned* p = (const unsigned*)base + lrow0;
#pragma unroll
        for (int r = 0; r < R; r++) out[r] = (unsigned long long)p[r * 32];
        break;
      }
      case DFGPU_INT32: {
        const int* p = (const int*)base + lrow0;
#pragma unroll
        for (int r = 0; r < R; r++) out[r] = (unsigned long long)(long long)p[r * 32];
        break;
      }
      default:
#pragma unroll
        for (int r = 0; r < R; r++) out[r] = load(ps, slot, r);
        break;
    }
  }
  __device__ __forceinline__ unsigned long long rowid(int r) const { return (unsigned long long)(row0 + r * 32); }
  __device__ __forceinline__ unsigned col_valid(const ProgramSet&, int) const { return (1u << R) - 1u; }  // staged path is null-free
};

__device__ __forceinline__ void store_elem(void* p, int dtype, long long idx, unsigned long long v) {
  switch (dtype) {
    case DFGPU_FLOAT64: case DFGPU_INT64: case DFGPU_UINT64: ((unsigned long long*)p)[idx] = v; break;
    case DFGPU_FLOAT32: case DFGPU_UINT32: case DFGPU_INT32: ((unsigned*)p)[idx] = (unsigned)v; break;
    case DFGPU_INT16: case DFGPU_UINT16: ((unsigned short*)p)[idx] = (unsigned short)v; break;
    case DFGPU_INT8: case DFGPU_UINT8: ((unsigned char*)p)[idx] = (unsigned char)v; break;
    default: break;
  }
}

__device__ __forceinline__ int dtype_width_dev(int dtype) {
  switch (dtype) {
    case DFGPU_INT8: case DFGPU_UINT8: return 1;
    case DFGPU_INT16: case DFGPU_UINT16: return 2;
    case DFGPU_INT32: case DFGPU_UINT32: case DFGPU_FLOAT32: return 4;
    default: return 8;
  }
}

// Rust `as` (saturating float->int, NaN -> 0; wrapping int->int; nearest int->float)
__device__ __forceinline__ unsigned long long cast_value(unsigned long long v, int src_mt, int src_dt, int dst_dt) {
  // to floats
  if (dst_dt == DFGPU_FLOAT64) {
    switch (src_mt) {
      case MT_F64: return v;
      case MT_F32: return d2u((double)u2f(v));
      case MT_I: return d2u((double)(long long)v);
      default: return d2u((double)v);
    }
  }
  if (dst_dt == DFGPU_FLOAT32) {
    switch (src_mt) {
      case MT_F64: return f2u((float)u2d(v));
      case MT_F32: return v;
      case MT_I: return f2u((float)(long long)v);
      default: return f2u((float)v);
    }
  }
  // to integers
  if (src_mt == MT_F64 || src_mt == MT_F32) {
    double x = src_mt == MT_F64 ? u2d(v) : (double)u2f(v);
    if (x != x) return 0;
    double lo, hi;
    switch (dst_dt) {
      case DFGPU_INT8: lo = -128.0; hi = 127.0; break;
      case DFGPU_INT16: lo = -32768.0; hi = 32767.0; break;
      case DFGPU_INT32: lo = -2147483648.0; hi = 2147483647.0; break;
      case DFGPU_INT64: lo = -9223372036854775808.0; hi = 9223372036854775807.0; break;
      case DFGPU_UINT8: lo = 0.0; hi = 255.0; break;
      case DFGPU_UINT16: lo = 0.0; hi = 65535.0; break;
      case DFGPU_UINT32: lo = 0.0; hi = 4294967295.0; break;
      default: lo = 0.0; hi = 18446744073709551615.0; break;
    }
    if (dst_dt == DFGPU_UINT64) {
      if (x <= lo) return 0;
      if (x >= hi) return ~0ull;
      return (unsigned long long)x;
    }
    if (dst_dt == DFGPU_INT64) {
      if (x <= lo) return 0x8000000000000000ull;
      if (x >= hi) return 0x7fffffffffffffffull;
      return (unsigned long long)(long long)x;
    }
    if (x <= lo) x = lo;
    if (x >= hi) x = hi;
    return norm_int((unsigned long long)(long long)x, dst_dt);
  }
  return norm_int(v, dst_dt);  // int -> int: truncate / extend (value already sign/zero extended)
}

// Built-in scalar function `fn` (DFGPU_FN_*) of x (and y), each the Rust f64 method of the same name.  Out of line, so the
// code of the transcendentals, and the slow argument reduction of sin / cos / tan, is there once per module rather than
// once per row at every call site.
static __device__ __noinline__ double scalar_fn(int fn, double x, double y) {
  switch (fn) {
    case DFGPU_FN_SQRT: return sqrt(x);
    case DFGPU_FN_ABS: return u2d(d2u(x) & 0x7fffffffffffffffull);  // clears the sign bit, NaN payloads included
    case DFGPU_FN_FLOOR: return floor(x);
    case DFGPU_FN_CEIL: return ceil(x);
    case DFGPU_FN_TRUNC: return trunc(x);
    case DFGPU_FN_ROUND: {  // half away from zero; x - trunc(x) is exact, so 0.49999999999999994 stays 0
      const double t = trunc(x);
      return fabs(x - t) >= 0.5 ? t + copysign(1.0, x) : t;
    }
    case DFGPU_FN_SIGNUM: return x != x ? x : copysign(1.0, x);  // by the sign bit: signum(-0.0) = -1.0
    case DFGPU_FN_EXP: return exp(x);
    case DFGPU_FN_LN: return log(x);
    case DFGPU_FN_LOG2: return log2(x);
    case DFGPU_FN_LOG10: return log10(x);
    case DFGPU_FN_SIN: return sin(x);
    case DFGPU_FN_COS: return cos(x);
    case DFGPU_FN_TAN: return tan(x);
    case DFGPU_FN_ASIN: return asin(x);
    case DFGPU_FN_ACOS: return acos(x);
    case DFGPU_FN_ATAN: return atan(x);
    case DFGPU_FN_POWER: return pow(x, y);
    default: return atan2(x, y);  // DFGPU_FN_ATAN2; the compiler accepts no other code
  }
}

// Evaluate program `prog` of `ps` for the R rows described by `src` (GlobalRows / StagedTile).
// Returns the value stack top in out[]; bit r of the return value is set when valid row r divided
// by zero.  With F64ONLY every operand is Float64/Boolean (checked on the host): the machine-type
// dispatch disappears and only the warp-uniform opcode switch is left.
//
// NULLS: arrow 0.12 array_ops null semantics (restated from the crate; call sites expression.rs:127,216):
// arithmetic and And/Or yield null when either side is null — the builder's append_null stores the
// type's default, so the VALUE of a null result is 0 / false, which is what FilterRelation's
// `filter.value(i)` (filter.rs:86) and update_accumulators' `z.value(row)` (aggregate.rs:561-601) read;
// comparisons never yield null: nulls are ordered (lt/lt_eq: null on the left -> true; gt/gt_eq: null
// on the right -> true; eq: both null).  `out_valid` receives the validity bits of the result.
//
// The extended interpreter (DEPTH == kCaseDepth) always tracks validity, so that the nulls a CASE without ELSE makes reach
// the result; without NULLS it reads every column as valid (the input bitmaps are dropped, as under a WHERE).  It also
// evaluates CASE lazily: each stack entry carries the DivideByZero bits of its rows (badmask for the accumulator, spille
// for the spilled entries), an operation ORs its operands' bits and a select keeps err(c) | (taken ? err(v) : err(e)).
// The result's bits are the top entry's.  For a program without CASE that is the OR over every operation, which is
// what the other instantiations compute in badmask directly.
template <int DEPTH, int R, bool F64ONLY, bool NULLS, class Src>
__device__ __forceinline__ unsigned eval_program_n(const ProgramSet& ps, int prog, const Src& src,
                                                   unsigned long long (&out)[R], unsigned& out_valid) {
  // Accumulator machine: the top of the operand stack lives in `out` (registers, statically indexed);
  // deeper entries are spilled to a small per-thread array indexed by the run-time depth (local memory,
  // L1 resident).  A push therefore costs R stores instead of shifting the whole register stack, and a
  // stack-mode instruction R loads (its operands were exchanged at lowering so that the accumulator is
  // always the left input).
  constexpr unsigned ALL = (1u << R) - 1u;
  constexpr bool FN = DEPTH >= kFnDepth;   // the scalar-function cases are compiled in
  constexpr bool CS = DEPTH == kCaseDepth; // and the CASE cases, with their bookkeeping
  constexpr bool TV = NULLS || CS;         // validity is tracked
  constexpr int D = FN ? 8 : DEPTH;
  constexpr int SPILL = D > 1 ? D - 1 : 1;
  unsigned long long spill[SPILL][R];
  unsigned spillv[SPILL];
  unsigned spille[SPILL];  // CS: DivideByZero bits of the spilled entries
  unsigned accv = ALL;
  int depth = 0;
#pragma unroll
  for (int r = 0; r < R; r++) out[r] = 0;
  unsigned badmask = 0;
  const int begin = ps.start[prog], end = ps.start[prog + 1];
  for (int pc = begin; pc < end; ++pc) {
    // one 16-byte constant-bank read per instruction
    const uint4 raw = *reinterpret_cast<const uint4*>(&ps.insn[pc]);
    const int op = raw.x & 0xff;
    const int mode = (raw.x >> 8) & 0xff;
    const int mt = (raw.x >> 16) & 0xff;
    const int dt = (raw.x >> 24) & 0xff;
    const int slot = (int)(short)(raw.y & 0xffff);
    const unsigned long long imm = ((unsigned long long)raw.w << 32) | raw.z;
    if constexpr (CS) {  // discarded in every other instantiation, which therefore keeps its code
      if (op >= V_SEL) {
        // pop the condition c (the entry below the accumulator v) and, for V_SEL, the fold e below it
        depth--;
        const int dc = depth - 1 < SPILL ? depth - 1 : SPILL - 1;
        unsigned taken = 0;
#pragma unroll
        for (int r = 0; r < R; r++) taken |= (unsigned)(spill[dc][r] & 1ull) << r;
        taken &= spillv[dc];  // a null condition is not taken
        const unsigned errc = spille[dc];
        if (op == V_SEL) {
          depth--;
          const int de = depth - 1 < SPILL ? depth - 1 : SPILL - 1;
#pragma unroll
          for (int r = 0; r < R; r++)
            if (!((taken >> r) & 1u)) out[r] = spill[de][r];
          accv = (accv & taken) | (spillv[de] & ~taken);
          badmask = errc | (badmask & taken) | (spille[de] & ~taken);
        } else {
#pragma unroll
          for (int r = 0; r < R; r++)
            if (!((taken >> r) & 1u)) out[r] = 0ull;
          accv &= taken;
          badmask = errc | (badmask & taken);
        }
        continue;
      }
    }
    if constexpr (FN) {
      if (op >= V_FN) {
        // scalar function: Float64 in, Float64 out; a row is null where an argument is, with value 0 (like arithmetic)
        const int fn = (int)(short)(raw.y >> 16);
        unsigned valid = accv;
        if (op == V_FN) {  // one argument: the accumulator
#pragma unroll
          for (int r = 0; r < R; r++) out[r] = d2u(scalar_fn(fn, u2d(out[r]), 0.0));
        } else {  // two arguments, right one as in the binary ops below; V_RFN2: the accumulator is the right argument
          unsigned long long y[R];
          if (mode == RHS_IMM) {
#pragma unroll
            for (int r = 0; r < R; r++) y[r] = imm;
          } else if (mode == RHS_COL) {
            src.load_rows(ps, slot, y);
            if (NULLS) valid &= src.col_valid(ps, slot);
          } else {
            depth--;
            const int d = depth - 1 >= 0 ? (depth - 1 < SPILL ? depth - 1 : SPILL - 1) : 0;
#pragma unroll
            for (int r = 0; r < R; r++) y[r] = spill[d][r];
            if (TV) valid &= spillv[d];
            if constexpr (CS) badmask |= spille[d];
          }
          const bool swap = op == V_RFN2;
#pragma unroll
          for (int r = 0; r < R; r++) out[r] = d2u(scalar_fn(fn, u2d(swap ? y[r] : out[r]), u2d(swap ? out[r] : y[r])));
        }
        if (TV) {
#pragma unroll
          for (int r = 0; r < R; r++)
            if (!((valid >> r) & 1u)) out[r] = 0ull;
          accv = valid;
        }
        continue;
      }
    }
    if (op <= V_PUSH_ROWID) {
      if (D > 1 && depth > 0) {  // spill the current top
        const int d = depth - 1 < SPILL ? depth - 1 : SPILL - 1;
#pragma unroll
        for (int r = 0; r < R; r++) spill[d][r] = out[r];
        if (TV) spillv[d] = accv;
        if constexpr (CS) spille[d] = badmask;
      }
      depth++;
      if constexpr (CS) badmask = 0;
      if (TV) accv = NULLS && op == V_PUSH_COL ? src.col_valid(ps, slot) : ALL;
      if (op == V_PUSH_IMM) {
#pragma unroll
        for (int r = 0; r < R; r++) out[r] = imm;
      } else if (op == V_PUSH_ROWID) {
#pragma unroll
        for (int r = 0; r < R; r++) out[r] = src.rowid(r);
      } else {
        src.load_rows(ps, slot, out);
      }
    } else if (op == V_CAST) {
      const int src_dt = (int)(short)(raw.y >> 16);
#pragma unroll
      for (int r = 0; r < R; r++) out[r] = cast_value(out[r], mt, src_dt, dt);
      if (TV) {
#pragma unroll
        for (int r = 0; r < R; r++)
          if (!((accv >> r) & 1u)) out[r] = 0ull;
      }
    } else {
      unsigned long long y[R];
      unsigned vb = ALL;
      const unsigned va = accv;
      if (mode == RHS_IMM) {
#pragma unroll
        for (int r = 0; r < R; r++) y[r] = imm;
      } else if (mode == RHS_COL) {
        src.load_rows(ps, slot, y);
        if (NULLS) vb = src.col_valid(ps, slot);
      } else {
        // pop the entry below the top (the instruction's left operand before the exchange)
        depth--;
        const int d = depth - 1 >= 0 ? (depth - 1 < SPILL ? depth - 1 : SPILL - 1) : 0;
#pragma unroll
        for (int r = 0; r < R; r++) y[r] = spill[d][r];
        if (TV) vb = spillv[d];
        if constexpr (CS) badmask |= spille[d];
      }
      const unsigned both = va & vb;
      // The (machine type, op) dispatch is hoisted out of the per-row loop: it is warp-uniform and
      // paid once per R rows.  A zero divisor sets the row's bit in badmask (arrow 0.12
      // array_ops::divide returns ArrowError::DivideByZero for ints and floats alike).
#define DF_ROWS(EXPR) _Pragma("unroll") for (int r = 0; r < R; r++) { const unsigned long long a = out[r], b = y[r]; (void)a; (void)b; out[r] = (EXPR); }
#define DF_DIVCHK(WHICH, COND) _Pragma("unroll") for (int r = 0; r < R; r++) { const unsigned long long z = WHICH[r]; if ((COND) && (!TV || ((both >> r) & 1u))) badmask |= 1u << r; }
      switch (F64ONLY ? (op == V_AND || op == V_OR ? (int)MT_BOOL : (int)MT_F64) : mt) {
        case MT_F64:
          switch (op) {
            case V_ADD: DF_ROWS(d2u(u2d(a) + u2d(b))) break;
            case V_SUB: DF_ROWS(d2u(u2d(a) - u2d(b))) break;
            case V_RSUB: DF_ROWS(d2u(u2d(b) - u2d(a))) break;
            case V_MUL: DF_ROWS(d2u(u2d(a) * u2d(b))) break;
            case V_DIV: DF_DIVCHK(y, u2d(z) == 0.0) DF_ROWS(d2u(u2d(a) / u2d(b))) break;
            case V_RDIV: DF_DIVCHK(out, u2d(z) == 0.0) DF_ROWS(d2u(u2d(b) / u2d(a))) break;
            case V_EQ: DF_ROWS((unsigned long long)(u2d(a) == u2d(b))) break;
            case V_NE: DF_ROWS((unsigned long long)(u2d(a) != u2d(b))) break;
            case V_LT: DF_ROWS((unsigned long long)(u2d(a) < u2d(b))) break;
            case V_LE: DF_ROWS((unsigned long long)(u2d(a) <= u2d(b))) break;
            case V_GT: DF_ROWS((unsigned long long)(u2d(a) > u2d(b))) break;
            default: DF_ROWS((unsigned long long)(u2d(a) >= u2d(b))) break;
          }
          break;
        case MT_F32:
          switch (op) {
            case V_ADD: DF_ROWS(f2u(u2f(a) + u2f(b))) break;
            case V_SUB: DF_ROWS(f2u(u2f(a) - u2f(b))) break;
            case V_RSUB: DF_ROWS(f2u(u2f(b) - u2f(a))) break;
            case V_MUL: DF_ROWS(f2u(u2f(a) * u2f(b))) break;
            case V_DIV: DF_DIVCHK(y, u2f(z) == 0.0f) DF_ROWS(f2u(u2f(a) / u2f(b))) break;
            case V_RDIV: DF_DIVCHK(out, u2f(z) == 0.0f) DF_ROWS(f2u(u2f(b) / u2f(a))) break;
            case V_EQ: DF_ROWS((unsigned long long)(u2f(a) == u2f(b))) break;
            case V_NE: DF_ROWS((unsigned long long)(u2f(a) != u2f(b))) break;
            case V_LT: DF_ROWS((unsigned long long)(u2f(a) < u2f(b))) break;
            case V_LE: DF_ROWS((unsigned long long)(u2f(a) <= u2f(b))) break;
            case V_GT: DF_ROWS((unsigned long long)(u2f(a) > u2f(b))) break;
            default: DF_ROWS((unsigned long long)(u2f(a) >= u2f(b))) break;
          }
          break;
        case MT_I:
#define DF_SDIV(N, D) ((D) == 0ull ? 0ull : ((long long)(D) == -1ll ? norm_int(0ull - (N), dt) : norm_int((unsigned long long)((long long)(N) / (long long)(D)), dt)))
          switch (op) {
            case V_ADD: DF_ROWS(norm_int(a + b, dt)) break;
            case V_SUB: DF_ROWS(norm_int(a - b, dt)) break;
            case V_RSUB: DF_ROWS(norm_int(b - a, dt)) break;
            case V_MUL: DF_ROWS(norm_int(a * b, dt)) break;
            case V_DIV: DF_DIVCHK(y, z == 0ull) DF_ROWS(DF_SDIV(a, b)) break;
            case V_RDIV: DF_DIVCHK(out, z == 0ull) DF_ROWS(DF_SDIV(b, a)) break;
            case V_EQ: DF_ROWS((unsigned long long)(a == b)) break;
            case V_NE: DF_ROWS((unsigned long long)(a != b)) break;
            case V_LT: DF_ROWS((unsigned long long)((long long)a < (long long)b)) break;
            case V_LE: DF_ROWS((unsigned long long)((long long)a <= (long long)b)) break;
            case V_GT: DF_ROWS((unsigned long long)((long long)a > (long long)b)) break;
            default: DF_ROWS((unsigned long long)((long long)a >= (long long)b)) break;
          }
#undef DF_SDIV
          break;
        case MT_U:
          switch (op) {
            case V_ADD: DF_ROWS(norm_int(a + b, dt)) break;
            case V_SUB: DF_ROWS(norm_int(a - b, dt)) break;
            case V_RSUB: DF_ROWS(norm_int(b - a, dt)) break;
            case V_MUL: DF_ROWS(norm_int(a * b, dt)) break;
            case V_DIV: DF_DIVCHK(y, z == 0ull) DF_ROWS(b == 0ull ? 0ull : a / b) break;
            case V_RDIV: DF_DIVCHK(out, z == 0ull) DF_ROWS(a == 0ull ? 0ull : b / a) break;
            case V_EQ: DF_ROWS((unsigned long long)(a == b)) break;
            case V_NE: DF_ROWS((unsigned long long)(a != b)) break;
            case V_LT: DF_ROWS((unsigned long long)(a < b)) break;
            case V_LE: DF_ROWS((unsigned long long)(a <= b)) break;
            case V_GT: DF_ROWS((unsigned long long)(a > b)) break;
            default: DF_ROWS((unsigned long long)(a >= b)) break;
          }
          break;
        default:  // MT_BOOL
          switch (op) {
            case V_AND: DF_ROWS(a & b) break;
            case V_OR: DF_ROWS(a | b) break;
            case V_EQ: DF_ROWS((unsigned long long)(a == b)) break;
            default: DF_ROWS((unsigned long long)(a != b)) break;
          }
          break;
      }
#undef DF_ROWS
#undef DF_DIVCHK
      if (TV) {
        if (op >= V_EQ && op <= V_GE) {
          // comparisons: never null; a null operand is ordered, not propagated (a = accumulator = the
          // left input of the instruction as emitted, b = y = its right input)
#pragma unroll
          for (int r = 0; r < R; r++) {
            if (!((both >> r) & 1u)) {
              const bool ln = !((va >> r) & 1u), rn = !((vb >> r) & 1u);
              bool v;
              switch (op) {
                case V_EQ: v = ln && rn; break;
                case V_NE: v = !(ln && rn); break;
                case V_LT: case V_LE: v = ln; break;
                default: v = rn; break;
              }
              out[r] = v ? 1ull : 0ull;
            }
          }
          accv = ALL;
        } else {
          // arithmetic, And, Or: null if either side is null; append_null stores the default value
#pragma unroll
          for (int r = 0; r < R; r++)
            if (!((both >> r) & 1u)) out[r] = 0ull;
          accv = both;
        }
      }
    }
  }
  out_valid = TV ? accv : ALL;
  return badmask & src.valid;
}

template <int DEPTH, int R, bool F64ONLY, class Src>
__device__ __forceinline__ unsigned eval_program(const ProgramSet& ps, int prog, const Src& src,
                                                 unsigned long long (&out)[R]) {
  unsigned ov;
  return eval_program_n<DEPTH, R, F64ONLY, false>(ps, prog, src, out, ov);
}
#endif  // __CUDACC__

}  // namespace dfgpu
