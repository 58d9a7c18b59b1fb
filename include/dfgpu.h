/*
 * dfgpu.h — C ABI of the H100-native (sm_90a) engine for DataFusion 0.6.0's Arrow-batch hot path.
 *
 * This is the drop-in boundary.  The reference (andygrove/datafusion-archive, Rust) has no FFI; its
 * operator "plugin API" is the `Relation` trait plus the `Expr`/`LogicalPlan` IR.  Each entry point
 * below names the reference interface it replaces (file:line relative to the reference root).
 * A Rust `extern "C"` block binding these symbols, and the `impl Relation for Gpu*Relation` that
 * calls them, is shown in INTEGRATION.md.
 *
 * Conventions
 *   - Every function returns 0 on success, a DFGPU_ERR_* code otherwise; the message is available
 *     from dfgpu_last_error() (thread-local, valid until the next call on the same thread).
 *     The shim maps codes onto `ExecutionError` variants (src/execution/error.rs:51-60).
 *   - No CPU fallback exists anywhere behind this ABI: an unsupported dtype / operator returns
 *     DFGPU_ERR_NOT_IMPLEMENTED; a missing GPU returns DFGPU_ERR_CUDA.
 *   - Input buffers are BORROWED for the duration of a call (Arrow `ArrayData` views: values
 *     pointer, length, offset, optional LSB-first validity bitmap).  Outputs are copied into
 *     caller-allocated buffers after a shape query — no cross-allocator frees.
 *   - One host thread per dfgpu_ctx (the reference is `Rc<RefCell<..>>`, i.e. !Send:
 *     src/execution/context.rs:34).  One ctx drives one GPU; multi-GPU = one process (or ctx) per
 *     GPU with row-range partitioning, joined by dfgpu_comm_init() for the partial-aggregate merge.
 */
#ifndef DFGPU_H
#define DFGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DFGPU_ABI_VERSION 2

/* ---- error codes (→ ExecutionError variants, src/execution/error.rs:51-60) ---- */
enum {
  DFGPU_OK = 0,
  DFGPU_ERR_GENERAL = 1,         /* ExecutionError::General          */
  DFGPU_ERR_EXECUTION = 2,       /* ExecutionError::ExecutionError   */
  DFGPU_ERR_NOT_IMPLEMENTED = 3, /* ExecutionError::NotImplemented   */
  DFGPU_ERR_INVALID_COLUMN = 4,  /* ExecutionError::InvalidColumn    */
  DFGPU_ERR_INTERNAL = 5,        /* ExecutionError::InternalError    */
  DFGPU_ERR_ARROW = 6,           /* ExecutionError::ArrowError (e.g. DivideByZero, length mismatch) */
  DFGPU_ERR_CUDA = 7,            /* device / driver / NCCL failure   */
  DFGPU_ERR_OOM = 8
};

/* ---- Arrow data types on the path (arrow::datatypes::DataType) ---- */
enum {
  DFGPU_BOOL = 1, /* bit-packed, LSB first */
  DFGPU_INT8 = 2,
  DFGPU_INT16 = 3,
  DFGPU_INT32 = 4,
  DFGPU_INT64 = 5,
  DFGPU_UINT8 = 6,
  DFGPU_UINT16 = 7,
  DFGPU_UINT32 = 8,
  DFGPU_UINT64 = 9,
  DFGPU_FLOAT32 = 10,
  DFGPU_FLOAT64 = 11,
  DFGPU_UTF8 = 12 /* arrow 0.12 BinaryArray: i32 offsets (len+1) + u8 data */
};

/* Borrowed view of one Arrow array (arrow `ArrayData`): element i lives at values[(offset+i)],
 * validity bit i at validity[(offset+i)>>3] >> ((offset+i)&7) & 1 (1 = valid, NULL = all valid).
 * For DFGPU_UTF8 `values` is the byte buffer and `offsets` the i32 offsets buffer. */
typedef struct dfgpu_col {
  int32_t dtype;
  int32_t _pad;
  int64_t len;
  int64_t offset;
  const void* values;
  const uint8_t* validity;
  const int32_t* offsets;
  int64_t values_bytes; /* UTF8 only: size of the byte buffer; 0 otherwise */
} dfgpu_col;

/* ---- expression programs ----
 * An `Expr` tree (src/logicalplan.rs:136-167) is lowered to a postfix program of dfgpu_insn.
 * This replaces the closure tree built by compile_scalar_expr (src/execution/expression.rs:283-505).
 * `dtype` is the column type for COL, the literal type for LIT, the TARGET type for CAST (`col`
 * then carries the source type) and, advisory, the left operand type for binary ops: the engine
 * re-infers operand types itself and rejects mixed-type operands the way the reference does
 * (ExecutionError "math_ops" / "comparison_ops": expression.rs:166,207).  */
enum {
  DFGPU_OP_COL = 1,  /* Expr::Column(col)                         expression.rs:311-315 */
  DFGPU_OP_LIT = 2,  /* Expr::Literal(ScalarValue)                expression.rs:226-243 */
  DFGPU_OP_CAST = 3, /* Expr::Cast{expr,data_type}                expression.rs:246-280,316-378 */
  DFGPU_OP_LIT_UTF8 = 4, /* Expr::Literal(ScalarValue::Utf8): `lit.str` = address of the bytes, `col` = byte length (>= 0;
                            0 = ''), `dtype` = DFGPU_UTF8.  The bytes are borrowed for the call; a program the library keeps
                            past the call (dfgpu_aggregate_create / _set_predicate) owns a copy.  A negative length or a
                            null address with a nonzero length is DFGPU_ERR_GENERAL "malformed expression program".
                            DFGPU_OP_LIT with dtype DFGPU_UTF8 stays "No support for literal type Utf8".  Additive. */
  DFGPU_OP_ADD = 10, /* Operator::Plus     → array_ops::add       expression.rs:466 */
  DFGPU_OP_SUB = 11, /* Operator::Minus    → array_ops::subtract  expression.rs:473 */
  DFGPU_OP_MUL = 12, /* Operator::Multiply → array_ops::multiply  expression.rs:480 */
  DFGPU_OP_DIV = 13, /* Operator::Divide   → array_ops::divide    expression.rs:487 */
  /* + - * /: both operands of one dtype, which is the result's.  Integers wrap at the operand width (Rust release
     semantics), `/` truncates toward zero and MIN / -1 = MIN.  Floats are IEEE, each result rounded once to nearest
     (no FTZ, no fused multiply-add).  A zero divisor of any type, -0.0 included, is DFGPU_ERR_ARROW "DivideByZero",
     raised only for a row that survives the WHERE (a WHERE reads every row); without a WHERE a null row does not
     raise it, while under a WHERE a surviving row's null slot is divided like any other value. */
  DFGPU_OP_EQ = 20,  /* array_ops::eq      expression.rs:410 */
  DFGPU_OP_NE = 21,  /* array_ops::neq     expression.rs:417 */
  DFGPU_OP_LT = 22,  /* array_ops::lt      expression.rs:424 */
  DFGPU_OP_LE = 23,  /* array_ops::lt_eq   expression.rs:431 */
  DFGPU_OP_GT = 24,  /* array_ops::gt      expression.rs:438 */
  DFGPU_OP_GE = 25,  /* array_ops::gt_eq   expression.rs:445 */
  DFGPU_OP_LIKE = 26,     /* Operator::Like    (sqlparser.rs / logicalplan.rs Operator), postfix `x p`; see Utf8 predicates */
  DFGPU_OP_NOT_LIKE = 27, /* Operator::NotLike */
  DFGPU_OP_AND = 30, /* array_ops::and     expression.rs:452 */
  DFGPU_OP_OR = 31,  /* array_ops::or      expression.rs:459 */
  DFGPU_OP_FN = 40,  /* Expr::ScalarFunction{name,args,return_type} logicalplan.rs:156-160: `col` = DFGPU_FN_* code,
                        `dtype` = Float64; the arguments come first, in order.  Additive: libraries older than it
                        reject it with "operator: 40". */
  DFGPU_OP_UTF8_FN = 41, /* Expr::ScalarFunction of a Utf8 function: `col` = DFGPU_UTF8FN_* code, `dtype` = the result
                           type (DFGPU_UTF8, or DFGPU_INT64 for LENGTH / OCTET_LENGTH).  The arguments come first: the
                           Utf8 operand (a column or another DFGPU_OP_UTF8_FN), then the function's DFGPU_OP_LIT Int64
                           values.  See "Utf8 functions" below.  Additive. */
  DFGPU_OP_CASE = 42 /* CASE WHEN c1 THEN v1 [WHEN c2 THEN v2 ..] [ELSE e] END: the operands come first, in the order
                        c1 v1 .. cn vn [e]; `col` = the number of operands, 2n, or 2n + 1 with an ELSE; `dtype` = the result
                        type.  See "CASE" below.  Additive: libraries older than it reject it with "operator: 42". */
};

/* CASE (DFGPU_OP_CASE).
 *   - Choice: the value of the first WHEN whose condition is true; a false or null condition is not taken.  When no WHEN
 *     is taken, the ELSE value; without ELSE, null (with value 0 under the null, like every null an expression makes).
 *     The result has the validity of the branch chosen.
 *   - Laziness: a row raises DivideByZero only from the conditions up to and including the first true one and from the
 *     value chosen; a branch not taken or a condition after the one taken never raises, in nested CASEs too.  The rule
 *     of DFGPU_OP_DIV applies on top: only a row that survives the WHERE raises.
 *   - Nulls: a CASE-made null is a null wherever a result can carry one, under a WHERE too (a projection then has a
 *     validity bitmap, while the input columns' bitmaps are still dropped).  COUNT, AVG, COUNT(DISTINCT) and a reduction
 *     without GROUP BY skip it; GROUP BY SUM / MIN / MAX and GROUP BY keys read its value 0.
 *   - Types: every condition is Boolean (DFGPU_ERR_EXECUTION "CASE WHEN condition did not evaluate to boolean"); every
 *     THEN / ELSE operand has one numeric or Boolean dtype, the result type (DFGPU_ERR_EXECUTION "CASE branch types
 *     differ: Int64 and Float64"); a Utf8 result is DFGPU_ERR_NOT_IMPLEMENTED "CASE with a Utf8 result".  Utf8
 *     predicates are conditions like any other.  An operand count below 2 or above the operands present, or a `dtype`
 *     other than the result type, is DFGPU_ERR_GENERAL "malformed expression program".
 *   - A CASE may appear wherever a numeric or Boolean expression may; its operands are any expressions, CASE included. */

/* Built-in scalar functions (DFGPU_OP_FN).  The reference declares Expr::ScalarFunction and plans it
 * (sqlplanner.rs:343-365: every argument cast to the declared type) but never executes it
 * (context.rs:255-257 unimplemented!()).  Every function takes Float64 arguments and returns Float64; a
 * caller of this ABI inserts the CASTs, as the planner does.  Each value follows the Rust f64 method named
 * beside it, since a reference UDF is a Rust closure; a row is null where an argument is null.  No
 * function raises an error: domain errors give NaN or +-inf. */
enum {
  DFGPU_FN_SQRT = 1,   /* f64::sqrt   */
  DFGPU_FN_ABS = 2,    /* f64::abs    */
  DFGPU_FN_FLOOR = 3,  /* f64::floor  */
  DFGPU_FN_CEIL = 4,   /* f64::ceil   */
  DFGPU_FN_TRUNC = 5,  /* f64::trunc  */
  DFGPU_FN_ROUND = 6,  /* f64::round: half away from zero */
  DFGPU_FN_SIGNUM = 7, /* f64::signum: +-1.0 by the sign bit, NaN for NaN */
  DFGPU_FN_EXP = 8,    /* f64::exp    */
  DFGPU_FN_LN = 9,     /* f64::ln     */
  DFGPU_FN_LOG2 = 10,  /* f64::log2   */
  DFGPU_FN_LOG10 = 11, /* f64::log10  */
  DFGPU_FN_SIN = 12,   /* f64::sin    */
  DFGPU_FN_COS = 13,   /* f64::cos    */
  DFGPU_FN_TAN = 14,   /* f64::tan    */
  DFGPU_FN_ASIN = 15,  /* f64::asin   */
  DFGPU_FN_ACOS = 16,  /* f64::acos   */
  DFGPU_FN_ATAN = 17,  /* f64::atan   */
  DFGPU_FN_POWER = 18, /* f64::powf(x, y), two arguments */
  DFGPU_FN_ATAN2 = 19  /* f64::atan2(y, x), two arguments */
};

/* Utf8 predicates (the reference plans them but executes neither: comparison_ops! has no Utf8 arm,
 * expression.rs:171-209, and literals other than numbers are refused, :306-309).
 *   - DFGPU_OP_EQ .. DFGPU_OP_GE between two Utf8 operands: a column against a DFGPU_OP_LIT_UTF8 literal (on either
 *     side) or against another Utf8 column.  Byte-wise lexicographic order, a proper prefix first (Rust's [u8] Ord;
 *     for valid UTF-8 this is code-point order).  The bytes are never validated.  Nulls as for every numeric
 *     comparison: null equals null, null orders below every string including '', and the result has no nulls.
 *   - DFGPU_OP_LIKE / DFGPU_OP_NOT_LIKE: `x` a Utf8 column, `p` a Utf8 literal.  `%` matches any run of characters
 *     (possibly empty), `_` exactly one; a character is one UTF-8 code point: a byte that is not 10xxxxxx starts one.
 *     Case-sensitive, no escape character (`\` is an ordinary byte).  A null `x` satisfies neither LIKE nor NOT LIKE;
 *     the result has no nulls.
 *   - They may appear wherever a Boolean may: WHERE, a Boolean projection, the aggregate's fused WHERE, under AND / OR.
 *   - Refused: a non-literal pattern and literal against literal (DFGPU_ERR_NOT_IMPLEMENTED); non-Utf8 LIKE operands
 *     (DFGPU_ERR_EXECUTION naming the operator); Utf8 against a number ("comparison_ops"); a Utf8 literal anywhere
 *     else (DFGPU_ERR_EXECUTION "No support for literal type Utf8(..)"); a literal or pattern longer than
 *     DFGPU_UTF8_LITERAL_MAX bytes (DFGPU_ERR_NOT_IMPLEMENTED). */
#define DFGPU_UTF8_LITERAL_MAX 4096

/* Utf8 functions (DFGPU_OP_UTF8_FN).  PostgreSQL's, under the C locale, defined for any bytes (never validated).  A
 * character is one UTF-8 code point as LIKE's `_` counts them: the first byte of a string and every later byte that is
 * not 10xxxxxx start one.  A null argument gives a null; a Utf8 result keeps the source's validity, with length 0 on
 * null rows.  Any nesting over one Utf8 column is allowed, e.g. upper(trim(substr(s, 2))), length(lower(s)).
 *   - Utf8 results may be projected, and compared or LIKE-matched wherever Utf8 predicates may appear.  Int64 results
 *     may appear wherever an Int64 column may, aggregate arguments and GROUP BY keys included.
 *   - Refused: a Utf8 result as a GROUP BY key ("Utf8 GROUP BY keys must be plain columns") or aggregate argument (as for
 *     a Utf8 column); a Utf8 literal argument (DFGPU_ERR_NOT_IMPLEMENTED); a non-Utf8 argument (DFGPU_ERR_EXECUTION
 *     "function 'upper' takes a Utf8 argument, not Int32"); a start or count that is not a DFGPU_OP_LIT Int64
 *     (DFGPU_ERR_NOT_IMPLEMENTED); a negative count (DFGPU_ERR_EXECUTION "negative substring length not allowed"). */
enum {
  DFGPU_UTF8FN_UPPER = 1,        /* ASCII a-z -> A-Z, every other byte unchanged (no Unicode case mapping) */
  DFGPU_UTF8FN_LOWER = 2,        /* ASCII A-Z -> a-z, every other byte unchanged */
  DFGPU_UTF8FN_TRIM = 3,         /* remove spaces (0x20 only) at both ends */
  DFGPU_UTF8FN_LTRIM = 4,        /* ... at the start */
  DFGPU_UTF8FN_RTRIM = 5,        /* ... at the end */
  DFGPU_UTF8FN_SUBSTR_FROM = 6,  /* substr(s, start): the characters from position `start` (1-based) on */
  DFGPU_UTF8FN_SUBSTR = 7,       /* substr(s, start, count): positions [start, start + count) clipped to [1, n];
                                    start may be <= 0 or past the end; the sum saturates */
  DFGPU_UTF8FN_LENGTH = 8,       /* number of characters, Int64 (SQL length / char_length) */
  DFGPU_UTF8FN_OCTET_LENGTH = 9  /* number of bytes, Int64 */
};

typedef struct dfgpu_insn {
  int32_t op;
  int32_t col;   /* COL: column index; CAST: source dtype; LIT_UTF8: byte length */
  int32_t dtype; /* see above */
  int32_t _pad;
  union {
    double f64;
    int64_t i64;
    uint64_t u64;
    float f32;
    const char* str; /* LIT_UTF8: address of the literal's bytes */
  } lit;
} dfgpu_insn;

/* ---- aggregates (src/execution/expression.rs:32-39 AggregateType) ----
 * DFGPU_AGG_COUNT_DISTINCT is AggregateType::CountDistinct (expression.rs:32-39), which the reference
 * declares but never produces or executes (COUNT(DISTINCT) is a ROADMAP.md 0.6.x item): the number of
 * distinct non-null argument values per group.  Additive: libraries older than it reject code 5 with
 * "Unsupported aggregate function".
 * DFGPU_AGG_AVG is AggregateType::Avg, likewise declared but never executed by the reference: the mean of
 * the non-null argument values as Float64 (sum in f64 / count, one IEEE division), null when there are
 * none.  Additive like code 5. */
enum {
  DFGPU_AGG_MIN = 1,
  DFGPU_AGG_MAX = 2,
  DFGPU_AGG_SUM = 3,
  DFGPU_AGG_COUNT = 4,
  DFGPU_AGG_COUNT_DISTINCT = 5,
  DFGPU_AGG_AVG = 6
};

/* One aggregate expression: func(arg).  `arg` is a postfix program (exactly one argument, as
 * compile_expr asserts: expression.rs:91).  `out_dtype` is Expr::AggregateFunction.return_type
 * (arg type for MIN/MAX/SUM, UInt64 for COUNT and COUNT(DISTINCT): src/sqlplanner.rs:320-341;
 * Float64 for AVG).  0 = the default for the function. */
typedef struct dfgpu_agg {
  int32_t func;
  int32_t arg_len;
  const dfgpu_insn* arg;
  int32_t out_dtype;
  int32_t _pad;
} dfgpu_agg;

typedef struct dfgpu_ctx dfgpu_ctx;       /* one GPU + stream + memory pool                  */
typedef struct dfgpu_batch dfgpu_batch;   /* device-resident RecordBatch (columns in HBM)    */
typedef struct dfgpu_result dfgpu_result; /* device-resident output batch                    */
typedef struct dfgpu_aggstate dfgpu_aggstate; /* device hash table / accumulators of one AggregateRelation */

/* ---- library / context ---- */
int dfgpu_abi_version(void);
const char* dfgpu_last_error(void);
/* Replaces nothing in the reference (it has no device); called once from ExecutionContext::new
 * (src/execution/context.rs:38).  `device` is the CUDA ordinal this ctx owns. */
int dfgpu_init(int device, dfgpu_ctx** out);
int dfgpu_shutdown(dfgpu_ctx* ctx);
int dfgpu_device_count(int* out);
/* Block until all work queued on the ctx stream is complete. */
int dfgpu_sync(dfgpu_ctx* ctx);
/* Pinned host memory for Arrow buffers (so uploads/downloads are single DMA transfers). */
int dfgpu_host_alloc(size_t bytes, void** out);
int dfgpu_host_free(void* p);
/* Device timing on the ctx stream (CUDA events): start / stop→milliseconds. */
int dfgpu_timer_start(dfgpu_ctx* ctx);
int dfgpu_timer_stop(dfgpu_ctx* ctx, float* ms);
/* Write `bytes` (> L2) of scratch to evict L2 between timed iterations. */
int dfgpu_flush_l2(dfgpu_ctx* ctx);
/* Counters: number of engine kernels launched on this ctx since init. */
int dfgpu_kernel_launches(const dfgpu_ctx* ctx, int64_t* out);
/* Per-kernel device timing of the dominant (scan) kernels: CUDA events recorded on the ctx stream
 * immediately around each launch of the filter/project, hash-aggregate and reduce kernels.
 * enable(1) starts a fresh accumulation; get() synchronises and returns the summed kernel time and
 * the number of timed launches since enable. */
int dfgpu_profile_enable(dfgpu_ctx* ctx, int on);
int dfgpu_profile_get(dfgpu_ctx* ctx, double* kernel_ms, int64_t* launches);

/* ---- batches: the RecordBatch handed to Relation::next's consumer (src/execution/relation.rs:27-32) ---- */
/* Copy the Arrow buffers of one RecordBatch into HBM (one cudaMemcpyAsync per buffer; pageable
 * memory is staged through a pinned ring).  All columns must have the same `len`. */
int dfgpu_batch_upload(dfgpu_ctx* ctx, const dfgpu_col* cols, int ncols, dfgpu_batch** out);
int dfgpu_batch_rows(const dfgpu_batch* b, int64_t* nrows);
int dfgpu_batch_free(dfgpu_batch* b);

/* ---- compile_scalar_expr's checks alone (src/execution/expression.rs:283-505) ----
 * Type-check one expression program against a schema (`col_dtypes[i]` = dtype of column i) exactly as
 * dfgpu_filter_project / dfgpu_aggregate_update would before launching anything, without touching a
 * GPU: identical operand dtypes ("math_ops" / "comparison_ops"), Boolean operands for AND / OR, the CAST
 * rules, Float64 arguments and the arity of DFGPU_OP_FN, column indices.  `out_dtype` receives the result
 * type.  Usable on a machine with no device. */
int dfgpu_check_program(const int32_t* col_dtypes, int ncols, const dfgpu_insn* prog, int prog_len, int32_t* out_dtype);
/* The LIKE matcher alone, on the host, for one string: compiles `pattern` exactly as the operators do and matches
 * `s` with the matcher of the pattern's class.  *match = 1 / 0; *pattern_class = 0 exact, 1 prefix `abc%`, 2 suffix
 * `%abc`, 3 contains `%abc%`, 4 general.  Usable on a machine with no device. */
int dfgpu_utf8_like_host(const char* s, int64_t s_len, const char* pattern, int64_t pattern_len, int32_t* match, int32_t* pattern_class);
/* One Utf8 function nest alone, on the host, for one string: `prog` is a DFGPU_OP_UTF8_FN program over column 0 (Utf8),
 * compiled and evaluated by the same per-row code as the kernels.  *out_dtype receives DFGPU_UTF8 or DFGPU_INT64.  A
 * Utf8 result is written to out[0 .. *out_len) (`out` holds at least s_len bytes: no result is longer than its source),
 * an Int64 result to *out_int.  Usable on a machine with no device. */
int dfgpu_utf8_fn_host(const char* s, int64_t s_len, const dfgpu_insn* prog, int prog_len, char* out, int64_t* out_len,
                       int64_t* out_int, int32_t* out_dtype);

/* ---- FilterRelation + ProjectRelation fused (src/execution/filter.rs:46-110,
 *      src/execution/projection.rs:46-66, wiring at src/execution/context.rs:126-161) ----
 * pred_len == 0: no WHERE clause.  nproj == 0: emit every input column (what FilterRelation alone
 * does: filter.rs:55-57).  Output rows keep input order (filter.rs:86-90).  A projection whose type is
 * Boolean (a comparison or AND / OR: expression.rs:212-224,236-290) comes back as a DFGPU_BOOL column,
 * bit-packed LSB first like arrow's BooleanArray; dfgpu_result_col_bytes reports (nrows + 7) / 8.
 * Stream-ordered calls: a query with a WHERE clause whose referenced columns have no nulls, whose outputs are all
 * numeric (no Boolean, no Utf8) and which divides nowhere returns once its work is queued, before the kernel has
 * finished.  Every other call returns finished, and reports DivideByZero itself.  The accessors below
 * (dfgpu_result_shape, _col_bytes, _col_nulls, _copy_col, _col_device_ptr, _col_host_ptr) wait for the kernel
 * before they answer; dfgpu_result_col_dtype and dfgpu_result_free never wait.  dfgpu_shutdown waits for every
 * call still running, and the shape of a result that outlives its ctx stays readable. */
int dfgpu_filter_project(dfgpu_ctx* ctx, const dfgpu_batch* batch, const dfgpu_insn* pred, int pred_len,
                         const dfgpu_insn* const* proj, const int* proj_len, int nproj, dfgpu_result** out);

/* Same operator, host buffers in, host buffers out, for one big RecordBatch: the batch is cut into
 * row-range chunks and upload (H2D), kernel and download (D2H) of successive chunks overlap on three
 * streams; only the referenced columns cross PCIe.  This is what GpuFilterProjectRelation::next calls
 * for large batches.  The result's columns live in pinned host memory owned by the library
 * (dfgpu_result_col_host_ptr for zero-copy, dfgpu_result_copy_col to copy out).
 * Input buffers should be pinned (dfgpu_host_alloc) for the copies to be asynchronous.
 * Batches whose referenced columns include Utf8, Boolean or nullable columns are not chunk-pipelined: the
 * referenced columns are uploaded whole, the resident operator runs, and the result stays in device memory
 * (dfgpu_result_on_host tells which; dfgpu_result_copy_col works for both). */
int dfgpu_filter_project_host(dfgpu_ctx* ctx, const dfgpu_col* cols, int ncols, const dfgpu_insn* pred, int pred_len,
                              const dfgpu_insn* const* proj, const int* proj_len, int nproj, int64_t chunk_rows /*0 = default*/,
                              dfgpu_result** out);

/* ---- AggregateRelation (src/execution/aggregate.rs:38-61, 615-631, 703-952) ----
 * create → update once per input batch (the `while let Some(batch)` loops at aggregate.rs:707,796)
 * → finish (materialise group columns then aggregate columns: aggregate.rs:890-949; with a
 * communicator attached this is also where the partial-aggregate merge happens).
 * nkeys == 0: no GROUP BY (aggregate.rs:703-785).  Keys are postfix programs (group_expr are
 * compiled scalar exprs: context.rs:171-175); integer and Utf8 types only (aggregate.rs:63-76). */
int dfgpu_aggregate_create(dfgpu_ctx* ctx, const dfgpu_insn* const* keys, const int* key_len, int nkeys,
                           const dfgpu_agg* aggs, int naggs, int64_t expected_groups /*0 = unknown*/,
                           dfgpu_aggstate** out);
/* FilterRelation fused under the aggregate: the wiring `Aggregate{input: Selection{expr, ..}}` that
 * ExecutionContext::execute builds for `SELECT .. WHERE .. GROUP BY ..` (src/execution/context.rs:126-139,
 * 162-192; src/sqlplanner.rs:93-96).  The predicate (a Boolean postfix program over the SAME input columns,
 * else "Filter expression did not evaluate to boolean": filter.rs:62-67) is evaluated inside the scan
 * kernel before the probe: one pass over the input, no intermediate batch.  Must be called before the
 * first dfgpu_aggregate_update; pred_len == 0 removes it. */
int dfgpu_aggregate_set_predicate(dfgpu_aggstate* st, const dfgpu_insn* pred, int pred_len);
int dfgpu_aggregate_update(dfgpu_aggstate* st, const dfgpu_batch* batch);
/* Same as update for one big HOST RecordBatch (the `while let Some(batch)` body with the upload inside): the
 * batch is cut into row-range chunks, every H2D copy is queued up front on a copy stream and the scan of
 * chunk c waits only for chunk c's copies, so PCIe and the kernel overlap.  Input buffers should be pinned
 * (dfgpu_host_alloc).  Nullable / Utf8 / small batches take the plain upload path inside. */
int dfgpu_aggregate_update_host(dfgpu_aggstate* st, const dfgpu_col* cols, int ncols, int64_t chunk_rows /*0 = default*/);
int dfgpu_aggregate_finish(dfgpu_aggstate* st, dfgpu_result** out);
int dfgpu_aggregate_free(dfgpu_aggstate* st);

/* ---- inner, semi and anti equi-join on integer and Utf8 keys ----
 * The reference has no join: its planner plans none and its `Relation` trait (src/execution/relation.rs:27-32) has
 * no join relation; "JOIN support (hash join ...)" is the headline of its next milestone (ROADMAP.md, 0.7.0).  These
 * entry points are what a GpuHashJoinRelation implementing that trait calls: build once over the right input, then
 * probe once per batch of the left input.
 *   - A pair (probe row p, build row b) is output when every key is non-null on both sides and the keys are equal.
 *     Null keys never match (SQL join semantics; unlike DFGPU_OP_EQ, under which a null equals a null).
 *   - Output rows keep probe-row order; the order of one probe row's matches is unspecified.
 *   - Keys are postfix programs, 1 to 4 of them, each of any of the 8 integer types or Utf8.  The integer parts'
 *     widths sum to at most 64 bits (Utf8 parts do not count); they are packed as GROUP BY keys are (the last integer
 *     part in the low bits; a single one keeps its sign- or zero-extended 64-bit value).  Utf8 parts compare byte for
 *     byte ('a' is not 'a ', '' equals ''; no collation, trimming or UTF-8 validation), and keys that share a hash
 *     never match unless equal.  A key program that is not a plain column is evaluated exactly as a projection
 *     (a CAST(UInt32 AS Int32) wraps; lower(s) and substr(s, 1, 3) are Utf8 keys).  Probe key i must have the type of
 *     build key i (DFGPU_ERR_EXECUTION "JOIN key types differ: Utf8 and Int64").  Float and Boolean keys and integer
 *     parts wider than 64 bits are DFGPU_ERR_NOT_IMPLEMENTED naming the types; a key raising DivideByZero is
 *     DFGPU_ERR_ARROW.
 *   - Output columns keep their dtype and validity: fixed-width, Boolean (bit-packed) and Utf8.
 *   - A build side of 2^32 rows or more, a probe batch of 2^32 rows or more and a probe batch producing 2^32 or more
 *     output rows are DFGPU_ERR_NOT_IMPLEMENTED. */
typedef struct dfgpu_join dfgpu_join; /* the build side's hash table and its kept columns */
enum { DFGPU_JOIN_SEMI = 1, DFGPU_JOIN_ANTI = 2, DFGPU_JOIN_ANTI_NULL_AWARE = 3 }; /* dfgpu_join_semi kinds */
/* Build the table over `build` (borrowed for the call only).  The join keeps its own device copy of the columns
 * `keep_cols` (build-batch column numbers) and of its Utf8 key columns, so the caller may free the batch afterwards.
 * DFGPU_JOIN_TAG_BITS (1 to 64, default 64) cuts a Utf8 key's hash tag for tests of the collision handling. */
int dfgpu_join_build(dfgpu_ctx* ctx, const dfgpu_batch* build, const dfgpu_insn* const* keys, const int* key_len, int nkeys,
                     const int* keep_cols, int n_keep, dfgpu_join** out);
/* Probe with one batch: the result is the `probe_cols` of `probe` followed by the `build_cols` of the build batch
 * (its column numbering; each must be among `keep_cols`, else DFGPU_ERR_GENERAL), one row per matching pair. */
int dfgpu_join_probe(dfgpu_join* j, const dfgpu_batch* probe, const dfgpu_insn* const* keys, const int* key_len, int nkeys,
                     const int* probe_cols, int n_probe_cols, const int* build_cols, int n_build_cols, dfgpu_result** out);
/* Semi and anti join with one probe batch: the `probe_cols` of the probe rows that pass, in probe-row order, each
 * probe row at most once.  `kind`:
 *   DFGPU_JOIN_SEMI             a row passes when every key part is non-null and some build row has an equal key
 *                               (SQL `x IN (SELECT y ..)`, `EXISTS (.. WHERE u.a = t.a ..)`)
 *   DFGPU_JOIN_ANTI             a row passes when no build row has an equal key; a row with a null key part passes
 *                               (SQL `NOT EXISTS`)
 *   DFGPU_JOIN_ANTI_NULL_AWARE  exactly one key (else DFGPU_ERR_GENERAL).  An empty build side: every row passes.
 *                               A build row with a null key: no row passes (no kernel runs).  Otherwise a row passes
 *                               when its key is non-null and no build row has an equal key (SQL `x NOT IN (SELECT y ..)`
 *                               under three-valued logic, unknown read as false)
 * Keys, key types and their refusals and the 2^32-row probe limit are those of dfgpu_join_probe.  A join built for
 * semi / anti probes needs no kept columns (n_keep = 0). */
int dfgpu_join_semi(dfgpu_join* j, const dfgpu_batch* probe, const dfgpu_insn* const* keys, const int* key_len, int nkeys, int kind,
                    const int* probe_cols, int n_probe_cols, dfgpu_result** out);
int dfgpu_join_free(dfgpu_join* j);

/* ---- ORDER BY / LIMIT / HAVING over a device result ----
 * The reference plans LogicalPlan::Sort and LogicalPlan::Limit (src/sqlplanner.rs) but its ExecutionContext::execute
 * leaves both unimplemented!() (src/execution/context.rs:113,194).  dfgpu_sort is what a Sort / Limit relation calls:
 *   - Keep: the rows where `keep` (a Boolean postfix program over `in`) is true; a null or false row is dropped.
 *     keep_len 0 keeps every row.  A program that is not Boolean is DFGPU_ERR_EXECUTION.
 *   - Order: the kept rows, stably ordered by keys[0], then keys[1], ..; desc[i] != 0 orders key i descending (`desc`
 *     may be NULL: all ascending).  Rows equal on every key keep their input order.  Integers order by value; floats
 *     by the MIN / MAX accumulators' order (-0.0 before +0.0, every NaN equal and after +inf); Utf8 byte-wise
 *     lexicographically, a proper prefix first, as Utf8 `<`.  A null is below every value: first ascending, last
 *     descending.  A Boolean key is DFGPU_ERR_NOT_IMPLEMENTED.  nkeys 0 keeps the input order.
 *   - Limit: the first `limit` rows of that order (limit < 0: all of them).
 *   - Output: every column of `in`, with its dtype, validity and null count.  Key and keep programs that are not a
 *     plain column are evaluated first exactly as a projection without a WHERE (dfgpu_filter_project).
 *   - An input of 2^32 rows or more is DFGPU_ERR_NOT_IMPLEMENTED.
 * The library knows nothing of GROUP BY: a caller wanting a total order over an aggregate's result appends its group
 * key columns as the last, ascending keys. */
int dfgpu_sort(dfgpu_ctx* ctx, const dfgpu_batch* in, const dfgpu_insn* keep, int keep_len, const dfgpu_insn* const* keys, const int* key_len,
               const int32_t* desc, int nkeys, int64_t limit, dfgpu_result** out);
/* A batch that views the columns of a device result without copying them (an aggregate's result goes into dfgpu_sort
 * without a download and upload).  Free the view with dfgpu_batch_free before freeing the result.  A host-resident
 * result is DFGPU_ERR_GENERAL. */
int dfgpu_result_as_batch(const dfgpu_result* r, dfgpu_batch** out);

/* ---- window functions: f(args) OVER (PARTITION BY .. ORDER BY ..) ----
 * The reference has no window functions.  dfgpu_window evaluates the functions of one window specification:
 *   - Order: rows are ordered by the partition keys `part` (ascending), then by the ORDER BY keys `order` (desc[i] != 0:
 *     descending; `desc` may be NULL), under dfgpu_sort's rules: nulls first ascending, -0.0 before +0.0, every NaN after
 *     +inf, Utf8 byte-wise.  Rows that tie keep their input order.  A Boolean key is DFGPU_ERR_NOT_IMPLEMENTED.
 *   - Partition: rows whose partition keys have equal sort encodings (two nulls share one, all NaNs share one, -0.0 and
 *     +0.0 do not).  npart 0: the whole input is one partition.  Peers: rows of one partition equal on every ORDER BY key.
 *   - Frame: with ORDER BY, the partition's rows through the row's last peer (RANGE BETWEEN UNBOUNDED PRECEDING AND
 *     CURRENT ROW); without, the whole partition.
 *   - Functions (`fns[k].func`, result column k): DFGPU_WIN_ROW_NUMBER (1 + the row's position in its partition),
 *     DFGPU_WIN_RANK (1 + the rows of the partition before the row's first peer), DFGPU_WIN_DENSE_RANK (1 + the peer groups
 *     before the row's), all UInt64 with `arg` unused; DFGPU_AGG_COUNT (UInt64, the valid values of the frame) and
 *     DFGPU_AGG_SUM / MIN / MAX (the argument's type) / AVG (Float64) over the valid values of the frame, with the
 *     aggregates' value rules (integer SUM wraps at its width; MIN / MAX with -0.0 < +0.0, NaN skipped unless every value
 *     is NaN).  A frame without a valid value is null, except for COUNT (0).  Float SUM / AVG add in an order fixed by
 *     the input alone, so they give the same bits on every run and on any number of ranks.  DFGPU_AGG_COUNT_DISTINCT
 *     is DFGPU_ERR_NOT_IMPLEMENTED; a non-numeric argument and `out_dtype` are refused as dfgpu_aggregate_create does.
 *   - Output: one column per function, one row per input row, in `in`'s row order.  Key and argument programs that are
 *     not a plain column are evaluated first exactly as a projection without a WHERE (dfgpu_filter_project).
 *   - An input of 2^32 rows or more is DFGPU_ERR_NOT_IMPLEMENTED.
 * With a communicator attached the specification runs over the rank-ordered concatenation of every rank's `in` (each
 * rank all-gathers the key and argument columns), and the result holds this rank's rows only.  Every rank must call it,
 * a rank without rows with an empty batch of the same columns. */
enum { DFGPU_WIN_ROW_NUMBER = 16, DFGPU_WIN_RANK = 17, DFGPU_WIN_DENSE_RANK = 18 };
int dfgpu_window(dfgpu_ctx* ctx, const dfgpu_batch* in, const dfgpu_insn* const* part, const int* part_len, int npart,
                 const dfgpu_insn* const* order, const int* order_len, const int32_t* desc, int norder,
                 const dfgpu_agg* fns, int nfns, dfgpu_result** out);

/* ---- results ---- */
int dfgpu_result_shape(const dfgpu_result* r, int64_t* nrows, int* ncols);
int dfgpu_result_col_dtype(const dfgpu_result* r, int i, int32_t* dtype);
/* Utf8 columns: number of data bytes (offsets buffer has nrows+1 entries). */
int dfgpu_result_col_bytes(const dfgpu_result* r, int i, int64_t* nbytes);
/* null_count of column i (aggregate outputs can be null: aggregate.rs:641-643). */
int dfgpu_result_col_nulls(const dfgpu_result* r, int i, int64_t* null_count);
/* Copy column i to host.  dst_values: nrows*width bytes (Utf8: nbytes); dst_validity: ceil(nrows/8)
 * bytes or NULL; dst_offsets: (nrows+1) i32 for Utf8, else NULL. */
int dfgpu_result_copy_col(const dfgpu_result* r, int i, void* dst_values, uint8_t* dst_validity, int32_t* dst_offsets);
/* 1 when the result's columns live in pinned host memory (the chunk-pipelined dfgpu_filter_project_host), else 0. */
int dfgpu_result_on_host(const dfgpu_result* r, int* on_host);
/* Host pointer of column i's values (host-resident results only). */
int dfgpu_result_col_host_ptr(const dfgpu_result* r, int i, const void** hptr);
/* Device pointer of column i's values (for zero-copy consumers on the same GPU). */
int dfgpu_result_col_device_ptr(const dfgpu_result* r, int i, const void** dptr);
int dfgpu_result_free(dfgpu_result* r);

/* ---- multi-GPU: row-range partitioned batches, one ctx (process) per GPU ----
 * The reference has no distribution (ROADMAP.md:36-51 is roadmap only).  A communicator makes
 * dfgpu_aggregate_finish merge the per-rank partial aggregates (NCCL over NVLink/NVSwitch) so that
 * every rank returns the global result.  `nccl_unique_id` is the 128-byte ncclUniqueId created by
 * dfgpu_comm_unique_id on rank 0 and distributed by the host application. */
int dfgpu_comm_unique_id(uint8_t out_id[128]);
int dfgpu_comm_init(dfgpu_ctx* ctx, int rank, int world, const uint8_t nccl_unique_id[128]);
int dfgpu_comm_destroy(dfgpu_ctx* ctx);
/* Number of ranks of the attached communicator (1 = none). */
int dfgpu_comm_world(const dfgpu_ctx* ctx, int64_t* world);

#ifdef __cplusplus
}
#endif
#endif /* DFGPU_H */
