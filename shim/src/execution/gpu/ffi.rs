//! `extern "C"` declarations of include/dfgpu.h (ABI version 2) and the mapping of its status codes onto
//! `ExecutionError` (src/execution/error.rs:51-60).
#![allow(non_camel_case_types)]
use std::ffi::CStr;
use std::os::raw::{c_char, c_int, c_void};

use super::super::error::{ExecutionError, Result};

#[repr(C)] pub struct dfgpu_ctx { _p: [u8; 0] }
#[repr(C)] pub struct dfgpu_batch { _p: [u8; 0] }
#[repr(C)] pub struct dfgpu_result { _p: [u8; 0] }
#[repr(C)] pub struct dfgpu_aggstate { _p: [u8; 0] }
#[repr(C)] pub struct dfgpu_join { _p: [u8; 0] }

// dfgpu dtype codes (arrow::datatypes::DataType)
pub const DT_BOOL: i32 = 1;
pub const DT_INT8: i32 = 2;
pub const DT_INT16: i32 = 3;
pub const DT_INT32: i32 = 4;
pub const DT_INT64: i32 = 5;
pub const DT_UINT8: i32 = 6;
pub const DT_UINT16: i32 = 7;
pub const DT_UINT32: i32 = 8;
pub const DT_UINT64: i32 = 9;
pub const DT_FLOAT32: i32 = 10;
pub const DT_FLOAT64: i32 = 11;
pub const DT_UTF8: i32 = 12;

// expression opcodes
pub const OP_COL: i32 = 1;
pub const OP_LIT: i32 = 2;
pub const OP_CAST: i32 = 3;
/// Expr::Literal(ScalarValue::Utf8): `lit` = address of the bytes (borrowed for the call), `col` = byte length.
pub const OP_LIT_UTF8: i32 = 4;
pub const OP_ADD: i32 = 10;
pub const OP_SUB: i32 = 11;
pub const OP_MUL: i32 = 12;
pub const OP_DIV: i32 = 13;
pub const OP_EQ: i32 = 20;
pub const OP_NE: i32 = 21;
pub const OP_LT: i32 = 22;
pub const OP_LE: i32 = 23;
pub const OP_GT: i32 = 24;
pub const OP_GE: i32 = 25;
/// Operator::Like / NotLike: `x p`, x a Utf8 column, p a Utf8 literal
pub const OP_LIKE: i32 = 26;
pub const OP_NOT_LIKE: i32 = 27;
pub const OP_AND: i32 = 30;
pub const OP_OR: i32 = 31;
/// Expr::ScalarFunction of a built-in function: `col` = FN_* code, `dtype` = Float64, arguments first.
pub const OP_FN: i32 = 40;

// built-in scalar functions (DFGPU_FN_*): Float64 arguments, Float64 result, each the Rust f64 method of the same name
pub const FN_SQRT: i32 = 1;
pub const FN_ABS: i32 = 2;
pub const FN_FLOOR: i32 = 3;
pub const FN_CEIL: i32 = 4;
pub const FN_TRUNC: i32 = 5;
pub const FN_ROUND: i32 = 6;
pub const FN_SIGNUM: i32 = 7;
pub const FN_EXP: i32 = 8;
pub const FN_LN: i32 = 9;
pub const FN_LOG2: i32 = 10;
pub const FN_LOG10: i32 = 11;
pub const FN_SIN: i32 = 12;
pub const FN_COS: i32 = 13;
pub const FN_TAN: i32 = 14;
pub const FN_ASIN: i32 = 15;
pub const FN_ACOS: i32 = 16;
pub const FN_ATAN: i32 = 17;
pub const FN_POWER: i32 = 18;
pub const FN_ATAN2: i32 = 19;
/// Expr::ScalarFunction of a Utf8 function: `col` = UTF8FN_* code, `dtype` = Utf8 or Int64 (length / octet_length);
/// the Utf8 operand (a column or another OP_UTF8_FN) first, then the function's OP_LIT Int64 arguments.
pub const OP_UTF8_FN: i32 = 41;

// Utf8 functions (DFGPU_UTF8FN_*): ASCII case maps, space trims, substr by 1-based characters, lengths
pub const UTF8FN_UPPER: i32 = 1;
pub const UTF8FN_LOWER: i32 = 2;
pub const UTF8FN_TRIM: i32 = 3;
pub const UTF8FN_LTRIM: i32 = 4;
pub const UTF8FN_RTRIM: i32 = 5;
pub const UTF8FN_SUBSTR_FROM: i32 = 6;
pub const UTF8FN_SUBSTR: i32 = 7;
pub const UTF8FN_LENGTH: i32 = 8;
pub const UTF8FN_OCTET_LENGTH: i32 = 9;

// aggregate functions (src/execution/expression.rs:32-39 AggregateType)
pub const AGG_MIN: i32 = 1;
pub const AGG_MAX: i32 = 2;
pub const AGG_SUM: i32 = 3;
pub const AGG_COUNT: i32 = 4;
/// AggregateType::CountDistinct; the reference's parser (sqlparser 0.2.1) cannot express it, so the shim only
/// carries the constant.
pub const AGG_COUNT_DISTINCT: i32 = 5;
/// AggregateType::Avg: the mean of the non-null values as Float64, null when there are none.
pub const AGG_AVG: i32 = 6;

/// Borrowed view of one Arrow array (dfgpu_col).
#[repr(C)]
pub struct dfgpu_col {
    pub dtype: i32,
    pub _pad: i32,
    pub len: i64,
    pub offset: i64,
    pub values: *const c_void,
    pub validity: *const u8,
    pub offsets: *const i32,
    pub values_bytes: i64,
}

/// One postfix instruction of an expression program (dfgpu_insn; `lit` carries f64 / i64 / u64 / f32 bits, or for
/// OP_LIT_UTF8 the address of the literal's bytes, which the caller keeps alive for the call).
#[repr(C)]
#[derive(Clone, Copy)]
pub struct dfgpu_insn {
    pub op: i32,
    pub col: i32,
    pub dtype: i32,
    pub _pad: i32,
    pub lit: u64,
}

#[repr(C)]
pub struct dfgpu_agg {
    pub func: i32,
    pub arg_len: i32,
    pub arg: *const dfgpu_insn,
    pub out_dtype: i32,
    pub _pad: i32,
}

extern "C" {
    pub fn dfgpu_abi_version() -> c_int;
    pub fn dfgpu_last_error() -> *const c_char;
    pub fn dfgpu_init(device: c_int, out: *mut *mut dfgpu_ctx) -> c_int;
    pub fn dfgpu_shutdown(ctx: *mut dfgpu_ctx) -> c_int;
    pub fn dfgpu_host_alloc(bytes: usize, out: *mut *mut c_void) -> c_int;
    pub fn dfgpu_host_free(p: *mut c_void) -> c_int;
    pub fn dfgpu_batch_upload(ctx: *mut dfgpu_ctx, cols: *const dfgpu_col, ncols: c_int, out: *mut *mut dfgpu_batch) -> c_int;
    pub fn dfgpu_batch_free(b: *mut dfgpu_batch) -> c_int;
    pub fn dfgpu_filter_project(
        ctx: *mut dfgpu_ctx, batch: *const dfgpu_batch, pred: *const dfgpu_insn, pred_len: c_int,
        proj: *const *const dfgpu_insn, proj_len: *const c_int, nproj: c_int, out: *mut *mut dfgpu_result,
    ) -> c_int;
    /// host buffers in, pinned host buffers out, chunk-pipelined H2D | kernel | D2H (large batches)
    pub fn dfgpu_filter_project_host(
        ctx: *mut dfgpu_ctx, cols: *const dfgpu_col, ncols: c_int, pred: *const dfgpu_insn, pred_len: c_int,
        proj: *const *const dfgpu_insn, proj_len: *const c_int, nproj: c_int, chunk_rows: i64, out: *mut *mut dfgpu_result,
    ) -> c_int;
    pub fn dfgpu_aggregate_create(
        ctx: *mut dfgpu_ctx, keys: *const *const dfgpu_insn, key_len: *const c_int, nkeys: c_int,
        aggs: *const dfgpu_agg, naggs: c_int, expected_groups: i64, out: *mut *mut dfgpu_aggstate,
    ) -> c_int;
    /// the WHERE clause of a Selection directly under the Aggregate, fused into the scan kernel
    pub fn dfgpu_aggregate_set_predicate(st: *mut dfgpu_aggstate, pred: *const dfgpu_insn, pred_len: c_int) -> c_int;
    pub fn dfgpu_aggregate_update(st: *mut dfgpu_aggstate, batch: *const dfgpu_batch) -> c_int;
    /// one big host RecordBatch: chunked H2D overlapped with the scan
    pub fn dfgpu_aggregate_update_host(st: *mut dfgpu_aggstate, cols: *const dfgpu_col, ncols: c_int, chunk_rows: i64) -> c_int;
    pub fn dfgpu_aggregate_finish(st: *mut dfgpu_aggstate, out: *mut *mut dfgpu_result) -> c_int;
    pub fn dfgpu_aggregate_free(st: *mut dfgpu_aggstate) -> c_int;
    /// inner equi-join on integer keys (ROADMAP.md 0.7.0 "JOIN support"; no reference relation): build over the right
    /// input once, keeping a device copy of `keep_cols`
    pub fn dfgpu_join_build(
        ctx: *mut dfgpu_ctx, build: *const dfgpu_batch, keys: *const *const dfgpu_insn, key_len: *const c_int, nkeys: c_int,
        keep_cols: *const c_int, n_keep: c_int, out: *mut *mut dfgpu_join,
    ) -> c_int;
    /// one probe batch: its `probe_cols`, then the kept `build_cols`, one row per matching pair
    pub fn dfgpu_join_probe(
        j: *mut dfgpu_join, probe: *const dfgpu_batch, keys: *const *const dfgpu_insn, key_len: *const c_int, nkeys: c_int,
        probe_cols: *const c_int, n_probe_cols: c_int, build_cols: *const c_int, n_build_cols: c_int, out: *mut *mut dfgpu_result,
    ) -> c_int;
    /// semi / anti join (kind: DFGPU_JOIN_SEMI, _ANTI, _ANTI_NULL_AWARE = 1, 2, 3): the `probe_cols` of the passing
    /// probe rows, in probe order
    pub fn dfgpu_join_semi(
        j: *mut dfgpu_join, probe: *const dfgpu_batch, keys: *const *const dfgpu_insn, key_len: *const c_int, nkeys: c_int, kind: c_int,
        probe_cols: *const c_int, n_probe_cols: c_int, out: *mut *mut dfgpu_result,
    ) -> c_int;
    pub fn dfgpu_join_free(j: *mut dfgpu_join) -> c_int;
    /// Sort / Limit over a device result (LogicalPlan::Sort / Limit, unimplemented!() at context.rs:113,194): keep the
    /// rows where `keep` is true, order them stably by the keys (desc[i] != 0: descending), return the first `limit`
    /// (< 0: all)
    pub fn dfgpu_sort(
        ctx: *mut dfgpu_ctx, input: *const dfgpu_batch, keep: *const dfgpu_insn, keep_len: c_int, keys: *const *const dfgpu_insn,
        key_len: *const c_int, desc: *const i32, nkeys: c_int, limit: i64, out: *mut *mut dfgpu_result,
    ) -> c_int;
    /// window functions of one specification (no reference counterpart): rows partitioned by `part`, ordered by `order`
    /// (desc[i] != 0: descending); one result column per `fns` entry (func = DFGPU_WIN_* or DFGPU_AGG_*), in input row
    /// order; with a communicator, over every rank's rows in rank order, returning this rank's rows
    pub fn dfgpu_window(
        ctx: *mut dfgpu_ctx, input: *const dfgpu_batch, part: *const *const dfgpu_insn, part_len: *const c_int, npart: c_int,
        order: *const *const dfgpu_insn, order_len: *const c_int, desc: *const i32, norder: c_int, fns: *const dfgpu_agg, nfns: c_int,
        out: *mut *mut dfgpu_result,
    ) -> c_int;
    /// a batch viewing a device result's columns (free it before the result)
    pub fn dfgpu_result_as_batch(r: *const dfgpu_result, out: *mut *mut dfgpu_batch) -> c_int;
    pub fn dfgpu_result_shape(r: *const dfgpu_result, nrows: *mut i64, ncols: *mut c_int) -> c_int;
    pub fn dfgpu_result_col_dtype(r: *const dfgpu_result, i: c_int, dtype: *mut i32) -> c_int;
    pub fn dfgpu_result_col_bytes(r: *const dfgpu_result, i: c_int, nbytes: *mut i64) -> c_int;
    pub fn dfgpu_result_col_nulls(r: *const dfgpu_result, i: c_int, nulls: *mut i64) -> c_int;
    pub fn dfgpu_result_copy_col(r: *const dfgpu_result, i: c_int, dst_values: *mut c_void, dst_validity: *mut u8, dst_offsets: *mut i32) -> c_int;
    pub fn dfgpu_result_on_host(r: *const dfgpu_result, on_host: *mut c_int) -> c_int;
    pub fn dfgpu_result_col_host_ptr(r: *const dfgpu_result, i: c_int, hptr: *mut *const c_void) -> c_int;
    pub fn dfgpu_result_free(r: *mut dfgpu_result) -> c_int;
    pub fn dfgpu_comm_unique_id(out_id: *mut u8) -> c_int;
    pub fn dfgpu_comm_init(ctx: *mut dfgpu_ctx, rank: c_int, world: c_int, id: *const u8) -> c_int;
    pub fn dfgpu_comm_destroy(ctx: *mut dfgpu_ctx) -> c_int;
    /// number of ranks of the attached communicator (1 without one): a rank whose input is empty still has to join
    /// the merge of dfgpu_aggregate_finish (GpuAggregateRelation::next)
    pub fn dfgpu_comm_world(ctx: *const dfgpu_ctx, world: *mut i64) -> c_int;
    // ---- the rest of include/dfgpu.h (diagnostics, timing, zero-copy consumers), declared for completeness ----
    pub fn dfgpu_device_count(out: *mut c_int) -> c_int;
    pub fn dfgpu_sync(ctx: *mut dfgpu_ctx) -> c_int;
    pub fn dfgpu_timer_start(ctx: *mut dfgpu_ctx) -> c_int;
    pub fn dfgpu_timer_stop(ctx: *mut dfgpu_ctx, ms: *mut f32) -> c_int;
    pub fn dfgpu_flush_l2(ctx: *mut dfgpu_ctx) -> c_int;
    pub fn dfgpu_kernel_launches(ctx: *const dfgpu_ctx, out: *mut i64) -> c_int;
    pub fn dfgpu_profile_enable(ctx: *mut dfgpu_ctx, on: c_int) -> c_int;
    pub fn dfgpu_profile_get(ctx: *mut dfgpu_ctx, kernel_ms: *mut f64, launches: *mut i64) -> c_int;
    pub fn dfgpu_batch_rows(b: *const dfgpu_batch, nrows: *mut i64) -> c_int;
    /// type check of one expression program without a device (the checks compile_scalar_expr makes: expression.rs:136-290)
    pub fn dfgpu_check_program(col_dtypes: *const i32, ncols: c_int, prog: *const dfgpu_insn, prog_len: c_int, out_dtype: *mut i32) -> c_int;
    /// the LIKE pattern compiler and matcher on the host, for one string
    pub fn dfgpu_utf8_like_host(s: *const c_char, s_len: i64, pattern: *const c_char, pattern_len: i64, is_match: *mut i32, pattern_class: *mut i32) -> c_int;
    /// one Utf8 function nest over column 0 on the host, for one string
    pub fn dfgpu_utf8_fn_host(s: *const c_char, s_len: i64, prog: *const dfgpu_insn, prog_len: c_int, out: *mut c_char, out_len: *mut i64,
                              out_int: *mut i64, out_dtype: *mut i32) -> c_int;
    pub fn dfgpu_result_col_device_ptr(r: *const dfgpu_result, i: c_int, dptr: *mut *const c_void) -> c_int;
}

/// nonzero status -> ExecutionError (src/execution/error.rs:51-60)
pub fn check(rc: c_int) -> Result<()> {
    if rc == 0 {
        return Ok(());
    }
    let msg = unsafe { CStr::from_ptr(dfgpu_last_error()) }.to_string_lossy().into_owned();
    Err(match rc {
        1 => ExecutionError::General(msg),
        3 => ExecutionError::NotImplemented(msg),
        4 => ExecutionError::InvalidColumn(msg),
        5 => ExecutionError::InternalError(msg),
        // 2 EXECUTION, 6 ARROW (DivideByZero, length mismatch), 7 CUDA, 8 OOM
        _ => ExecutionError::ExecutionError(msg),
    })
}
