// logicalplan.h — C++ mirror of the reference's logical IR and Arrow-side value types
// (src/logicalplan.rs: Operator :67-84, ScalarValue :96-111, Expr :136-167, LogicalPlan :311-348,
// get_supertype :446, can_coerce_from :556).  The reference is Rust; no toolchain for it exists in
// this image, so the host layer above the C ABI is C++ with the same names, argument meaning and
// error behaviour.  Debug formatting reproduces Rust's `{:?}` output so the reference's plan-text
// tests (src/sqlplanner.rs:547-707) can be replayed verbatim.
#pragma once
#include <cstdint>
#include <memory>
#include <set>
#include <string>
#include <vector>

#include "../../../include/dfgpu.h"

namespace dfhost {

// ---- errors: ExecutionError (src/execution/error.rs:48-60) ----------------------------------------
struct ExecutionError {
  int code;  // DFGPU_ERR_*
  std::string msg;
};
[[noreturn]] inline void fail(int code, const std::string& m) { throw ExecutionError{code, m}; }

// ---- arrow::datatypes ---------------------------------------------------------------------------
using DataType = int;  // DFGPU_BOOL .. DFGPU_UTF8
const char* datatype_debug(DataType dt);
int datatype_width(DataType dt);

struct Field {
  std::string name;
  DataType data_type = 0;
  bool nullable = false;
  std::string qualifier = {};  // the table (or its alias) a scanned column belongs to; `q.c` resolves by it.  Not printed.
};
struct Schema {
  std::vector<Field> fields;
  std::string to_string() const;
};
using SchemaRef = std::shared_ptr<Schema>;

// ---- ScalarValue ---------------------------------------------------------------------------------
struct ScalarValue {
  DataType dtype = 0;  // 0 = Null
  union { int64_t i; uint64_t u; double d; float f; bool b; } v{};
  std::string s;  // Utf8
  static ScalarValue Int64(int64_t x) { ScalarValue r; r.dtype = DFGPU_INT64; r.v.i = x; return r; }
  static ScalarValue Float64(double x) { ScalarValue r; r.dtype = DFGPU_FLOAT64; r.v.d = x; return r; }
  static ScalarValue Utf8(const std::string& x) { ScalarValue r; r.dtype = DFGPU_UTF8; r.s = x; return r; }
  DataType get_datatype() const { return dtype; }
  std::string debug() const;
};
std::string rust_debug_f64(double x);

// ---- Operator ------------------------------------------------------------------------------------
enum class Operator { Eq, NotEq, Lt, LtEq, Gt, GtEq, Plus, Minus, Multiply, Divide, Modulus, And, Or, Not, Like, NotLike };
const char* operator_debug(Operator op);

// ---- Expr ----------------------------------------------------------------------------------------
struct Expr;
using ExprRef = std::shared_ptr<const Expr>;
struct Expr {
  // Case: args = c1 v1 .. cn vn [e], every v and e of one type (the planner casts them), as DFGPU_OP_CASE takes them
  // WindowFunction: name(args) OVER (PARTITION BY partition_by ORDER BY order_by), order_by being Sort exprs; data_type is
  // the result type
  enum Kind { Column, Literal, BinaryExpr, IsNotNull, IsNull, Cast, Sort, ScalarFunction, AggregateFunction, Case, WindowFunction } kind = Column;
  size_t index = 0;         // Column
  ScalarValue value;        // Literal
  ExprRef left, right;      // BinaryExpr; `left` is also the operand of IsNull/IsNotNull/Cast/Sort
  Operator op = Operator::Eq;
  DataType data_type = 0;   // Cast target / function return type
  bool asc = true;          // Sort
  std::string name;         // functions
  std::vector<ExprRef> args;
  bool distinct = false;    // AggregateFunction: COUNT(DISTINCT ..)
  std::vector<ExprRef> partition_by, order_by;  // WindowFunction

  static ExprRef column(size_t i);
  static ExprRef literal(const ScalarValue& v);
  static ExprRef binary(ExprRef l, Operator op, ExprRef r);
  static ExprRef cast(ExprRef e, DataType dt);
  static ExprRef aggregate(const std::string& name, std::vector<ExprRef> args, DataType rt, bool distinct = false);
  static ExprRef scalar_fn(const std::string& name, std::vector<ExprRef> args, DataType rt);
  static ExprRef sort(ExprRef e, bool asc);
  static ExprRef is_null(ExprRef e, bool negated);
  static ExprRef case_when(std::vector<ExprRef> args);
  static ExprRef window(const std::string& name, std::vector<ExprRef> args, std::vector<ExprRef> partition_by, std::vector<ExprRef> order_by,
                        DataType rt);

  DataType get_type(const Schema& schema) const;             // logicalplan.rs:170-198
  ExprRef cast_to(DataType t, const Schema& schema) const;   // logicalplan.rs:200-215
  std::string debug() const;                                 // logicalplan.rs:266-307
};

// ---- LogicalPlan -----------------------------------------------------------------------------------
struct LogicalPlan;
using PlanRef = std::shared_ptr<const LogicalPlan>;
struct LogicalPlan {
  // Join (no reference counterpart: ROADMAP.md 0.7.0): inner equi-join of `input` (left, probe side) and `right` (build
  // side, one TableScan) on on_keys (left expr, right expr), both over the joined schema = left fields ++ right
  // fields.  Chains are left-deep.
  // A semi / anti join (join_kind) keeps the rows of `input` that have a match in `right` (Semi), that have none (Anti),
  // or that have none under NOT IN's three-valued logic (AntiNullAware, one key); its schema is `input`'s, and `right`
  // is a Projection whose columns are the build keys.  The right keys of on_keys are numbered over the left fields
  // followed by `right`'s, as for an inner join.
  // Window (no reference counterpart): the rows of `input` with one more column per window_expr (Expr::WindowFunction over
  // `input`'s schema); its schema is input's fields followed by one field per window call, named by the function.
  enum Kind { Limit, Projection, Selection, Aggregate, Sort, TableScan, EmptyRelation, Join, Window } kind = EmptyRelation;
  enum class JoinKind { Inner, Semi, Anti, AntiNullAware } join_kind = JoinKind::Inner;  // Join
  size_t limit = 0;
  std::vector<ExprRef> expr;        // Projection / Sort exprs; Selection: expr[0]
  std::vector<ExprRef> group_expr;  // Aggregate
  std::vector<ExprRef> aggr_expr;   // Aggregate
  std::vector<ExprRef> window_expr;  // Window
  PlanRef input;
  PlanRef right;                                    // Join
  std::vector<std::pair<ExprRef, ExprRef>> on_keys;  // Join
  SchemaRef schema_;
  std::string schema_name, table_name;
  bool has_projection = false;
  std::vector<size_t> projection;

  const SchemaRef& schema() const;  // logicalplan.rs:352-362
  std::string debug() const;        // logicalplan.rs:365-442
};

// The column indices an expression reads (collect_expr, sqlplanner.rs:435-458), added to `acc`.
void collect_columns(const Expr& e, std::set<size_t>& acc);

// Whether an expression holds a window function call
bool contains_window(const Expr& e);

// The same expression with every column index lowered by `by` (a key over a joined schema -> over its right input).
ExprRef shift_columns(const ExprRef& e, size_t by);

// ---- type coercion lattice -------------------------------------------------------------------------
bool get_supertype(DataType l, DataType r, DataType* out);  // logicalplan.rs:446-554
bool can_coerce_from(DataType left, DataType other);        // logicalplan.rs:556-605

}  // namespace dfhost
