// logicalplan.cpp — see logicalplan.h.
#include "logicalplan.h"

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace dfhost {

const char* datatype_debug(DataType dt) {
  switch (dt) {
    case DFGPU_BOOL: return "Boolean";
    case DFGPU_INT8: return "Int8";
    case DFGPU_INT16: return "Int16";
    case DFGPU_INT32: return "Int32";
    case DFGPU_INT64: return "Int64";
    case DFGPU_UINT8: return "UInt8";
    case DFGPU_UINT16: return "UInt16";
    case DFGPU_UINT32: return "UInt32";
    case DFGPU_UINT64: return "UInt64";
    case DFGPU_FLOAT32: return "Float32";
    case DFGPU_FLOAT64: return "Float64";
    case DFGPU_UTF8: return "Utf8";
  }
  return "Null";
}

int datatype_width(DataType dt) {
  switch (dt) {
    case DFGPU_INT8: case DFGPU_UINT8: return 1;
    case DFGPU_INT16: case DFGPU_UINT16: return 2;
    case DFGPU_INT32: case DFGPU_UINT32: case DFGPU_FLOAT32: return 4;
    case DFGPU_INT64: case DFGPU_UINT64: case DFGPU_FLOAT64: return 8;
  }
  return 0;
}

std::string Schema::to_string() const {
  std::string s;
  for (size_t i = 0; i < fields.size(); i++) {
    if (i) s += ", ";
    s += fields[i].name + ": " + datatype_debug(fields[i].data_type);
  }
  return s;
}

// Rust `{:?}` of f64: shortest digits that round-trip; plain decimal with a mandatory fractional
// part for 1e-5 <= |x| < 1e16, exponent form otherwise.
std::string rust_debug_f64(double x) {
  if (std::isnan(x)) return "NaN";
  if (std::isinf(x)) return x < 0 ? "-inf" : "inf";
  if (x == 0) return std::signbit(x) ? "-0.0" : "0.0";
  char buf[64];
  int prec = 1;
  for (; prec <= 17; prec++) {
    snprintf(buf, sizeof buf, "%.*e", prec - 1, x);
    if (strtod(buf, nullptr) == x) break;
  }
  // buf = d.ddddde[+-]XX
  std::string m(buf);
  size_t epos = m.find('e');
  int exp10 = atoi(m.c_str() + epos + 1);
  std::string digits;
  bool neg = false;
  for (size_t i = 0; i < epos; i++) {
    if (m[i] == '-') neg = true;
    else if (m[i] != '.') digits += m[i];
  }
  std::string out = neg ? "-" : "";
  if (exp10 >= 16 || exp10 < -5) {
    out += digits.substr(0, 1);
    if (digits.size() > 1) out += "." + digits.substr(1);
    out += "e" + std::to_string(exp10);
    return out;
  }
  if (exp10 >= 0) {
    std::string ip = digits.substr(0, std::min(digits.size(), size_t(exp10 + 1)));
    while (int(ip.size()) < exp10 + 1) ip += '0';
    std::string fp = digits.size() > size_t(exp10 + 1) ? digits.substr(size_t(exp10 + 1)) : "0";
    return out + ip + "." + fp;
  }
  return out + "0." + std::string(size_t(-exp10 - 1), '0') + digits;
}

static std::string rust_debug_f32(float x) {
  if (std::isnan(x)) return "NaN";
  if (std::isinf(x)) return x < 0 ? "-inf" : "inf";
  char buf[64];
  for (int prec = 1; prec <= 9; prec++) {
    snprintf(buf, sizeof buf, "%.*g", prec, double(x));
    if (strtof(buf, nullptr) == x) break;
  }
  std::string s(buf);
  if (s.find('.') == std::string::npos && s.find('e') == std::string::npos) s += ".0";
  return s;
}

static std::string rust_debug_str(const std::string& s) {
  std::string o = "\"";
  for (char c : s) {
    if (c == '"' || c == '\\') { o += '\\'; o += c; }
    else if (c == '\n') o += "\\n";
    else if (c == '\t') o += "\\t";
    else o += c;
  }
  return o + "\"";
}

std::string ScalarValue::debug() const {  // #[derive(Debug)] on ScalarValue
  switch (dtype) {
    case DFGPU_BOOL: return std::string("Boolean(") + (v.b ? "true" : "false") + ")";
    case DFGPU_FLOAT32: return "Float32(" + rust_debug_f32(v.f) + ")";
    case DFGPU_FLOAT64: return "Float64(" + rust_debug_f64(v.d) + ")";
    case DFGPU_INT8: case DFGPU_INT16: case DFGPU_INT32: case DFGPU_INT64:
      return std::string(datatype_debug(dtype)) + "(" + std::to_string(v.i) + ")";
    case DFGPU_UINT8: case DFGPU_UINT16: case DFGPU_UINT32: case DFGPU_UINT64:
      return std::string(datatype_debug(dtype)) + "(" + std::to_string(v.u) + ")";
    case DFGPU_UTF8: return "Utf8(" + rust_debug_str(s) + ")";
  }
  return "Null";
}

const char* operator_debug(Operator op) {
  switch (op) {
    case Operator::Eq: return "Eq"; case Operator::NotEq: return "NotEq"; case Operator::Lt: return "Lt";
    case Operator::LtEq: return "LtEq"; case Operator::Gt: return "Gt"; case Operator::GtEq: return "GtEq";
    case Operator::Plus: return "Plus"; case Operator::Minus: return "Minus"; case Operator::Multiply: return "Multiply";
    case Operator::Divide: return "Divide"; case Operator::Modulus: return "Modulus"; case Operator::And: return "And";
    case Operator::Or: return "Or"; case Operator::Not: return "Not"; case Operator::Like: return "Like";
    case Operator::NotLike: return "NotLike";
  }
  return "?";
}

// ---- Expr ------------------------------------------------------------------------------------------
ExprRef Expr::column(size_t i) { auto e = std::make_shared<Expr>(); e->kind = Column; e->index = i; return e; }
ExprRef Expr::literal(const ScalarValue& v) { auto e = std::make_shared<Expr>(); e->kind = Literal; e->value = v; return e; }
ExprRef Expr::binary(ExprRef l, Operator op, ExprRef r) {
  auto e = std::make_shared<Expr>(); e->kind = BinaryExpr; e->left = std::move(l); e->op = op; e->right = std::move(r); return e;
}
ExprRef Expr::cast(ExprRef x, DataType dt) { auto e = std::make_shared<Expr>(); e->kind = Cast; e->left = std::move(x); e->data_type = dt; return e; }
ExprRef Expr::aggregate(const std::string& name, std::vector<ExprRef> args, DataType rt, bool distinct) {
  auto e = std::make_shared<Expr>(); e->kind = AggregateFunction; e->name = name; e->args = std::move(args); e->data_type = rt; e->distinct = distinct; return e;
}
ExprRef Expr::scalar_fn(const std::string& name, std::vector<ExprRef> args, DataType rt) {
  auto e = std::make_shared<Expr>(); e->kind = ScalarFunction; e->name = name; e->args = std::move(args); e->data_type = rt; return e;
}
ExprRef Expr::sort(ExprRef x, bool asc) { auto e = std::make_shared<Expr>(); e->kind = Sort; e->left = std::move(x); e->asc = asc; return e; }
ExprRef Expr::case_when(std::vector<ExprRef> args) { auto e = std::make_shared<Expr>(); e->kind = Case; e->args = std::move(args); return e; }
ExprRef Expr::window(const std::string& name, std::vector<ExprRef> args, std::vector<ExprRef> partition_by, std::vector<ExprRef> order_by, DataType rt) {
  auto e = std::make_shared<Expr>(); e->kind = WindowFunction; e->name = name; e->args = std::move(args); e->partition_by = std::move(partition_by);
  e->order_by = std::move(order_by); e->data_type = rt; return e;
}
ExprRef Expr::is_null(ExprRef x, bool negated) {
  auto e = std::make_shared<Expr>(); e->kind = negated ? IsNotNull : IsNull; e->left = std::move(x); return e;
}

DataType Expr::get_type(const Schema& schema) const {
  switch (kind) {
    case Column:
      if (index >= schema.fields.size()) fail(DFGPU_ERR_INVALID_COLUMN, "column index out of range");
      return schema.fields[index].data_type;
    case Literal:
      if (value.dtype == 0) fail(DFGPU_ERR_NOT_IMPLEMENTED, "ScalarValue::Null has no data type (reference: unimplemented!())");
      return value.get_datatype();
    case Cast: case ScalarFunction: case AggregateFunction: case WindowFunction: return data_type;
    case IsNull: case IsNotNull: return DFGPU_BOOL;
    case Sort: return left->get_type(schema);
    case Case: return args[1]->get_type(schema);
    case BinaryExpr:
      switch (op) {
        case Operator::Eq: case Operator::NotEq: case Operator::Lt: case Operator::LtEq: case Operator::Gt: case Operator::GtEq:
        case Operator::And: case Operator::Or:
          return DFGPU_BOOL;
        default: {
          DataType out;
          if (get_supertype(left->get_type(schema), right->get_type(schema), &out)) return out;
          return DFGPU_UTF8;  // unwrap_or(DataType::Utf8) //TODO ??? (logicalplan.rs:192)
        }
      }
  }
  return 0;
}

ExprRef Expr::cast_to(DataType t, const Schema& schema) const {
  DataType this_type = get_type(schema);
  if (this_type == t) return std::make_shared<Expr>(*this);
  if (can_coerce_from(t, this_type)) {
    if (kind == Case) {  // cast the THEN / ELSE values instead: the engine casts columns and literals, not expressions
      std::vector<ExprRef> a = args;
      auto recast = [&](ExprRef& v) {
        // a value the planner already widened (CAST(#3 AS Int64)) is widened from its source in one step: the same
        // value, since every coercion is exact or rounds once, and a CAST the engine can run
        const bool widened = v->kind == Cast && (v->left->kind == Column || v->left->kind == Literal) &&
                             can_coerce_from(v->data_type, v->left->get_type(schema));
        v = (widened ? v->left : v)->cast_to(t, schema);
      };
      for (size_t k = 1; k < a.size(); k += 2) recast(a[k]);
      if (a.size() % 2) recast(a.back());
      return Expr::case_when(std::move(a));
    }
    return Expr::cast(std::make_shared<Expr>(*this), t);
  }
  fail(DFGPU_ERR_GENERAL, std::string("Cannot automatically convert ") + datatype_debug(this_type) + " to " + datatype_debug(t));
}

std::string Expr::debug() const {
  switch (kind) {
    case Column: return "#" + std::to_string(index);
    case Literal: return value.debug();
    case Cast: return "CAST(" + left->debug() + " AS " + datatype_debug(data_type) + ")";
    case IsNull: return left->debug() + " IS NULL";
    case IsNotNull: return left->debug() + " IS NOT NULL";
    case BinaryExpr: return left->debug() + " " + operator_debug(op) + " " + right->debug();
    case Sort: return left->debug() + (asc ? " ASC" : " DESC");
    case Case: {
      std::string s = "CASE";
      for (size_t i = 0; i + 1 < args.size(); i += 2) s += " WHEN " + args[i]->debug() + " THEN " + args[i + 1]->debug();
      if (args.size() % 2) s += " ELSE " + args.back()->debug();
      return s + " END";
    }
    case ScalarFunction: case AggregateFunction: case WindowFunction: {
      std::string s = name + (distinct ? "(DISTINCT " : "(");
      for (size_t i = 0; i < args.size(); i++) {
        if (i) s += ", ";
        s += args[i]->debug();
      }
      s += ")";
      if (kind != WindowFunction) return s;
      s += " OVER (";
      for (size_t i = 0; i < partition_by.size(); i++) s += (i ? ", " : "PARTITION BY ") + partition_by[i]->debug();
      for (size_t i = 0; i < order_by.size(); i++) s += (i ? ", " : partition_by.empty() ? "ORDER BY " : " ORDER BY ") + order_by[i]->debug();
      return s + ")";
    }
  }
  return "?";
}

void collect_columns(const Expr& e, std::set<size_t>& acc) {
  switch (e.kind) {
    case Expr::Column: acc.insert(e.index); break;
    case Expr::BinaryExpr: collect_columns(*e.left, acc); collect_columns(*e.right, acc); break;
    case Expr::Cast: case Expr::IsNull: case Expr::IsNotNull: case Expr::Sort: collect_columns(*e.left, acc); break;
    case Expr::ScalarFunction: case Expr::AggregateFunction: case Expr::Case:
      for (auto& a : e.args) collect_columns(*a, acc);
      break;
    case Expr::WindowFunction:
      for (auto& a : e.args) collect_columns(*a, acc);
      for (auto& a : e.partition_by) collect_columns(*a, acc);
      for (auto& a : e.order_by) collect_columns(*a, acc);
      break;
    default: break;
  }
}

bool contains_window(const Expr& e) {
  if (e.kind == Expr::WindowFunction) return true;
  if ((e.left && contains_window(*e.left)) || (e.right && contains_window(*e.right))) return true;
  for (auto& a : e.args)
    if (contains_window(*a)) return true;
  return false;
}

ExprRef shift_columns(const ExprRef& e, size_t by) {
  auto c = std::make_shared<Expr>(*e);
  if (c->kind == Expr::Column) c->index -= by;
  if (c->left) c->left = shift_columns(c->left, by);
  if (c->right) c->right = shift_columns(c->right, by);
  for (auto& a : c->args) a = shift_columns(a, by);
  for (auto& a : c->partition_by) a = shift_columns(a, by);
  for (auto& a : c->order_by) a = shift_columns(a, by);
  return c;
}

// ---- LogicalPlan -------------------------------------------------------------------------------------
const SchemaRef& LogicalPlan::schema() const {
  if (kind == Selection) return input->schema();
  return schema_;
}

static std::string exprs_debug(const std::vector<ExprRef>& v) {
  std::string s;
  for (size_t i = 0; i < v.size(); i++) {
    if (i) s += ", ";
    s += v[i]->debug();
  }
  return s;
}

static void fmt_with_indent(const LogicalPlan& p, std::string& f, int indent) {
  if (indent > 0) {
    f += "\n";
    for (int i = 0; i < indent; i++) f += "  ";
  }
  switch (p.kind) {
    case LogicalPlan::EmptyRelation: f += "EmptyRelation"; break;
    case LogicalPlan::TableScan: {
      f += "TableScan: " + p.table_name + " projection=";
      if (!p.has_projection) f += "None";
      else {
        f += "Some([";
        for (size_t i = 0; i < p.projection.size(); i++) f += (i ? ", " : "") + std::to_string(p.projection[i]);
        f += "])";
      }
      break;
    }
    case LogicalPlan::Projection:
      f += "Projection: " + exprs_debug(p.expr);
      fmt_with_indent(*p.input, f, indent + 1);
      break;
    case LogicalPlan::Selection:
      f += "Selection: " + p.expr[0]->debug();
      fmt_with_indent(*p.input, f, indent + 1);
      break;
    case LogicalPlan::Aggregate:
      f += "Aggregate: groupBy=[[" + exprs_debug(p.group_expr) + "]], aggr=[[" + exprs_debug(p.aggr_expr) + "]]";
      fmt_with_indent(*p.input, f, indent + 1);
      break;
    case LogicalPlan::Sort:
      f += "Sort: " + exprs_debug(p.expr);
      fmt_with_indent(*p.input, f, indent + 1);
      break;
    case LogicalPlan::Limit:
      f += "Limit: " + std::to_string(p.limit);
      fmt_with_indent(*p.input, f, indent + 1);
      break;
    case LogicalPlan::Window:
      f += "Window: windowExpr=[[" + exprs_debug(p.window_expr) + "]]";
      fmt_with_indent(*p.input, f, indent + 1);
      break;
    case LogicalPlan::Join:
      f += p.join_kind == LogicalPlan::JoinKind::Inner ? "Join"
           : p.join_kind == LogicalPlan::JoinKind::Semi ? "SemiJoin"
           : p.join_kind == LogicalPlan::JoinKind::Anti ? "AntiJoin"
                                                        : "AntiJoin (null-aware)";
      f += ": on=[";
      for (size_t i = 0; i < p.on_keys.size(); i++)
        f += (i ? ", " : "") + p.on_keys[i].first->debug() + " Eq " + p.on_keys[i].second->debug();
      f += "]";
      fmt_with_indent(*p.input, f, indent + 1);
      fmt_with_indent(*p.right, f, indent + 1);
      break;
  }
}

std::string LogicalPlan::debug() const {
  std::string f;
  fmt_with_indent(*this, f, 0);
  return f;
}

// ---- coercion ----------------------------------------------------------------------------------------
static bool is_sint(DataType t) { return t >= DFGPU_INT8 && t <= DFGPU_INT64; }
static bool is_uint(DataType t) { return t >= DFGPU_UINT8 && t <= DFGPU_UINT64; }
static bool is_flt(DataType t) { return t == DFGPU_FLOAT32 || t == DFGPU_FLOAT64; }

// The reference spells this lattice out pair by pair (logicalplan.rs:456-553, tried in both operand
// orders); the same function in closed form:
//   same signedness        -> the wider type
//   signed x unsigned      -> the signed type, if it is at least as wide as the unsigned one
//   any integer x float    -> the float type
//   Float32 x Float64      -> Float64;  Utf8 x Utf8 -> Utf8;  Boolean x Boolean -> Boolean
bool get_supertype(DataType l, DataType r, DataType* out) {
  if (l == r && (is_sint(l) || is_uint(l) || is_flt(l) || l == DFGPU_UTF8 || l == DFGPU_BOOL)) { *out = l; return true; }
  const bool li = is_sint(l) || is_uint(l), ri = is_sint(r) || is_uint(r);
  if (li && ri) {
    const int wl = datatype_width(l), wr = datatype_width(r);
    if (is_sint(l) == is_sint(r)) { *out = wl >= wr ? l : r; return true; }
    const DataType s = is_sint(l) ? l : r, u = is_sint(l) ? r : l;
    if (datatype_width(s) >= datatype_width(u)) { *out = s; return true; }
    return false;
  }
  if (li && is_flt(r)) { *out = r; return true; }
  if (ri && is_flt(l)) { *out = l; return true; }
  if (is_flt(l) && is_flt(r)) { *out = DFGPU_FLOAT64; return true; }
  return false;
}

bool can_coerce_from(DataType left, DataType other) {
  if (is_sint(left)) return is_sint(other) && datatype_width(other) <= datatype_width(left);
  if (is_uint(left)) return is_uint(other) && datatype_width(other) <= datatype_width(left);
  if (left == DFGPU_FLOAT32) return is_sint(other) || is_uint(other) || other == DFGPU_FLOAT32;
  if (left == DFGPU_FLOAT64) return is_sint(other) || is_uint(other) || is_flt(other);
  return false;
}

}  // namespace dfhost
