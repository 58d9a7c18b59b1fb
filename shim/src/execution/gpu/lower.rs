//! `Expr` -> postfix expression program of the C ABI.  Replaces compile_scalar_expr
//! (src/execution/expression.rs:283-505): instead of a closure tree the expression is flattened; type
//! checking (identical operand dtypes, Boolean operands for And / Or, the Cast rules) happens inside the
//! library with the reference's error strings.
use arrow::datatypes::{DataType, Schema};

use super::super::error::{ExecutionError, Result};
use super::super::super::logicalplan::{Expr, Operator, ScalarValue};
use super::ffi::*;

pub fn dtype_code(dt: &DataType) -> Result<i32> {
    Ok(match dt {
        DataType::Boolean => DT_BOOL,
        DataType::Int8 => DT_INT8,
        DataType::Int16 => DT_INT16,
        DataType::Int32 => DT_INT32,
        DataType::Int64 => DT_INT64,
        DataType::UInt8 => DT_UINT8,
        DataType::UInt16 => DT_UINT16,
        DataType::UInt32 => DT_UINT32,
        DataType::UInt64 => DT_UINT64,
        DataType::Float32 => DT_FLOAT32,
        DataType::Float64 => DT_FLOAT64,
        DataType::Utf8 => DT_UTF8,
        other => return Err(ExecutionError::NotImplemented(format!("data type {:?} on the GPU path", other))),
    })
}

fn insn(op: i32, col: i32, dtype: i32, lit: u64) -> dfgpu_insn {
    dfgpu_insn { op, col, dtype, _pad: 0, lit }
}

/// (dtype code, raw bits) of a literal — Expr::Literal(ScalarValue), expression.rs:289-310
fn literal(v: &ScalarValue) -> Result<(i32, u64)> {
    Ok(match v {
        ScalarValue::Int8(x) => (DT_INT8, *x as i64 as u64),
        ScalarValue::Int16(x) => (DT_INT16, *x as i64 as u64),
        ScalarValue::Int32(x) => (DT_INT32, *x as i64 as u64),
        ScalarValue::Int64(x) => (DT_INT64, *x as u64),
        ScalarValue::UInt8(x) => (DT_UINT8, *x as u64),
        ScalarValue::UInt16(x) => (DT_UINT16, *x as u64),
        ScalarValue::UInt32(x) => (DT_UINT32, *x as u64),
        ScalarValue::UInt64(x) => (DT_UINT64, *x),
        ScalarValue::Float32(x) => (DT_FLOAT32, x.to_bits() as u64),
        ScalarValue::Float64(x) => (DT_FLOAT64, x.to_bits()),
        other => return Err(ExecutionError::ExecutionError(format!("No support for literal type {:?}", other))),
    })
}

fn op_code(op: &Operator) -> Result<i32> {
    Ok(match op {
        Operator::Eq => OP_EQ,
        Operator::NotEq => OP_NE,
        Operator::Lt => OP_LT,
        Operator::LtEq => OP_LE,
        Operator::Gt => OP_GT,
        Operator::GtEq => OP_GE,
        Operator::And => OP_AND,
        Operator::Or => OP_OR,
        Operator::Plus => OP_ADD,
        Operator::Minus => OP_SUB,
        Operator::Multiply => OP_MUL,
        Operator::Divide => OP_DIV,
        Operator::Like => OP_LIKE,
        Operator::NotLike => OP_NOT_LIKE,
        other => return Err(ExecutionError::ExecutionError(format!("operator: {:?}", other))), // expression.rs:494-497
    })
}

/// The built-in scalar functions: (name, FN_* code, arity).  Names match in any letter case.
pub const BUILTIN_FUNCTIONS: &[(&str, i32, usize)] = &[
    ("sqrt", FN_SQRT, 1), ("abs", FN_ABS, 1), ("floor", FN_FLOOR, 1), ("ceil", FN_CEIL, 1), ("trunc", FN_TRUNC, 1),
    ("round", FN_ROUND, 1), ("signum", FN_SIGNUM, 1), ("exp", FN_EXP, 1), ("ln", FN_LN, 1), ("log2", FN_LOG2, 1),
    ("log10", FN_LOG10, 1), ("sin", FN_SIN, 1), ("cos", FN_COS, 1), ("tan", FN_TAN, 1), ("asin", FN_ASIN, 1),
    ("acos", FN_ACOS, 1), ("atan", FN_ATAN, 1), ("power", FN_POWER, 2), ("atan2", FN_ATAN2, 2),
];

/// (FN_* code, arity) of a built-in function
pub fn builtin_function(name: &str) -> Option<(i32, usize)> {
    BUILTIN_FUNCTIONS.iter().find(|f| f.0.eq_ignore_ascii_case(name)).map(|f| (f.1, f.2))
}

/// The Utf8 functions: (name, UTF8FN_* code, minimum and maximum arity, result dtype).  substr with two arguments is
/// UTF8FN_SUBSTR_FROM.
pub const UTF8_FUNCTIONS: &[(&str, i32, usize, usize, i32)] = &[
    ("upper", UTF8FN_UPPER, 1, 1, DT_UTF8), ("lower", UTF8FN_LOWER, 1, 1, DT_UTF8), ("trim", UTF8FN_TRIM, 1, 1, DT_UTF8),
    ("ltrim", UTF8FN_LTRIM, 1, 1, DT_UTF8), ("rtrim", UTF8FN_RTRIM, 1, 1, DT_UTF8), ("substr", UTF8FN_SUBSTR, 2, 3, DT_UTF8),
    ("length", UTF8FN_LENGTH, 1, 1, DT_INT64), ("char_length", UTF8FN_LENGTH, 1, 1, DT_INT64),
    ("octet_length", UTF8FN_OCTET_LENGTH, 1, 1, DT_INT64),
];

/// `remap[i]` = index of input column i among the columns actually uploaded (pruned to the referenced ones).
pub fn lower(e: &Expr, schema: &Schema, remap: &[Option<usize>], out: &mut Vec<dfgpu_insn>) -> Result<()> {
    match e {
        Expr::Column(i) => {
            let at = remap.get(*i).and_then(|x| *x).ok_or_else(|| ExecutionError::InvalidColumn(format!("column index {} out of range", i)))?;
            out.push(insn(OP_COL, at as i32, dtype_code(schema.field(*i).data_type())?, 0));
        }
        // a Utf8 literal: `lit` = address of the bytes, `col` = their length.  The plan's ScalarValue outlives the call,
        // and the engine copies the bytes of any program it keeps (dfgpu_aggregate_create / _set_predicate).
        Expr::Literal(ScalarValue::Utf8(s)) => {
            if s.len() > i32::MAX as usize {
                return Err(ExecutionError::NotImplemented("Utf8 literal longer than 2^31 bytes".to_string()));
            }
            out.push(insn(OP_LIT_UTF8, s.len() as i32, DT_UTF8, s.as_ptr() as usize as u64));
        }
        Expr::Literal(v) => {
            let (dt, bits) = literal(v)?;
            out.push(insn(OP_LIT, 0, dt, bits));
        }
        Expr::Cast { expr, data_type } => {
            lower(expr, schema, remap, out)?;
            let src = expr.get_type(schema);
            out.push(insn(OP_CAST, dtype_code(&src)?, dtype_code(data_type)?, 0)); // col carries the source dtype
        }
        Expr::BinaryExpr { left, op, right } => {
            lower(left, schema, remap, out)?;
            lower(right, schema, remap, out)?;
            out.push(insn(op_code(op)?, 0, dtype_code(&left.get_type(schema)).unwrap_or(0), 0));
        }
        Expr::ScalarFunction { name, args, .. } if UTF8_FUNCTIONS.iter().any(|f| f.0.eq_ignore_ascii_case(name)) => {
            let &(_, code, min, max, dt) = UTF8_FUNCTIONS.iter().find(|f| f.0.eq_ignore_ascii_case(name)).unwrap();
            if args.len() < min || args.len() > max {
                return Err(ExecutionError::ExecutionError(format!("function '{}' takes {} to {} argument(s), got {}", name, min, max, args.len())));
            }
            for a in args {
                lower(a, schema, remap, out)?;
            }
            let code = if code == UTF8FN_SUBSTR && args.len() == 2 { UTF8FN_SUBSTR_FROM } else { code };
            out.push(insn(OP_UTF8_FN, code, dt, 0));
        }
        Expr::ScalarFunction { name, args, .. } => {
            let (code, arity) = builtin_function(name).ok_or_else(|| ExecutionError::General(format!("Invalid function '{}'", name)))?;
            if args.len() != arity {
                // the planner rejects extra arguments but not missing ones
                return Err(ExecutionError::ExecutionError(format!("function '{}' takes {} argument(s), got {}", name, arity, args.len())));
            }
            for a in args {
                lower(a, schema, remap, out)?;
            }
            out.push(insn(OP_FN, code, DT_FLOAT64, 0));
        }
        other => return Err(ExecutionError::ExecutionError(format!("expression {:?}", other))), // expression.rs:500-503
    }
    Ok(())
}

/// Columns an expression reads (collect_expr, src/sqlplanner.rs:435-458).
pub fn collect_columns(e: &Expr, acc: &mut Vec<usize>) {
    match e {
        Expr::Column(i) => {
            if !acc.contains(i) {
                acc.push(*i)
            }
        }
        Expr::BinaryExpr { left, right, .. } => {
            collect_columns(left, acc);
            collect_columns(right, acc);
        }
        Expr::Cast { expr, .. } | Expr::IsNull(expr) | Expr::IsNotNull(expr) => collect_columns(expr, acc),
        Expr::Sort { expr, .. } => collect_columns(expr, acc),
        Expr::AggregateFunction { args, .. } | Expr::ScalarFunction { args, .. } => args.iter().for_each(|a| collect_columns(a, acc)),
        Expr::Literal(_) => {}
    }
}
