// execution.cpp — see execution.h.
#include "execution.h"
#include <cerrno>
#include <cctype>
#include <cstdint>

#include <cstring>
#include <set>

namespace dfhost {

namespace {
[[noreturn]] void gpu_fail(int rc) { fail(rc, dfgpu_last_error()); }
#define GPU_CHECK(expr)          \
  do {                           \
    int _rc = (expr);            \
    if (_rc != 0) gpu_fail(_rc); \
  } while (0)
}  // namespace

dfgpu_col Array::view() const {
  dfgpu_col c;
  memset(&c, 0, sizeof(c));
  c.dtype = data_type;
  c.len = len;
  c.offset = offset;
  c.values = values;
  c.validity = null_count > 0 ? validity : nullptr;
  c.offsets = offsets;
  c.values_bytes = values_bytes;
  return c;
}

// ---- CSV -----------------------------------------------------------------------------------------
CsvDataSource::CsvDataSource(const std::string& filename, SchemaRef schema, size_t batch_size)
    : schema_(std::move(schema)), file_(filename), batch_size_(batch_size ? batch_size : 1024) {
  if (!file_.is_open()) fail(DFGPU_ERR_GENERAL, "IoError: cannot open " + filename);
}

static std::vector<std::string> split_csv_line(const std::string& line) {
  std::vector<std::string> out;
  std::string cur;
  bool inq = false;
  for (size_t i = 0; i < line.size(); i++) {
    char c = line[i];
    if (inq) {
      if (c == '"') {
        if (i + 1 < line.size() && line[i + 1] == '"') { cur += '"'; i++; }
        else inq = false;
      } else cur += c;
    } else if (c == '"') inq = true;
    else if (c == ',') { out.push_back(cur); cur.clear(); }
    else if (c == '\r') {}
    else cur += c;
  }
  out.push_back(cur);
  return out;
}

static bool parse_signed(const std::string& s, long long lo, long long hi, long long* out) {
  if (s.empty() || isspace((unsigned char)s[0])) return false;
  char* end = nullptr;
  errno = 0;
  const long long v = strtoll(s.c_str(), &end, 10);
  if (end == s.c_str() || *end || errno == ERANGE || v < lo || v > hi) return false;
  *out = v;
  return true;
}
static bool parse_unsigned(const std::string& s, unsigned long long hi, unsigned long long* out) {
  if (s.empty() || isspace((unsigned char)s[0]) || s[0] == '-') return false;
  char* end = nullptr;
  errno = 0;
  const unsigned long long v = strtoull(s.c_str(), &end, 10);
  if (end == s.c_str() || *end || errno == ERANGE || v > hi) return false;
  *out = v;
  return true;
}

template <class T>
static void push_val(Array& a, T v) {
  size_t n = a.own_values.size();
  a.own_values.resize(n + sizeof(T));
  memcpy(a.own_values.data() + n, &v, sizeof(T));
}

std::optional<RecordBatch> CsvDataSource::next() {
  std::string line;
  if (!header_skipped_) {
    header_skipped_ = true;
    std::getline(file_, line);  // has_headers = true, unconditionally (datasource.rs:41)
    line_no_++;
  }
  RecordBatch b;
  b.schema = schema_;
  for (auto& f : schema_->fields) {
    auto a = std::make_shared<Array>();
    a->data_type = f.data_type;
    if (f.data_type == DFGPU_UTF8) a->own_offsets.push_back(0);
    b.columns.push_back(a);
  }
  size_t rows = 0;
  auto set_bit = [](std::vector<uint8_t>& bits, size_t i, bool v) {
    if (bits.size() < i / 8 + 1) bits.resize(i / 8 + 1, 0);
    if (v) bits[i / 8] |= uint8_t(1u << (i % 8));
  };
  while (rows < batch_size_ && std::getline(file_, line)) {
    line_no_++;
    if (line.empty()) continue;
    auto fields = split_csv_line(line);
    if (fields.size() < schema_->fields.size())
      fail(DFGPU_ERR_ARROW, "ParseError(\"line " + std::to_string(line_no_) + " has too few columns\")");
    for (size_t c = 0; c < schema_->fields.size(); c++) {
      Array& a = *b.columns[c];
      const std::string& s = fields[c];
      char* end = nullptr;
      // arrow 0.12 csv reader: an empty field of a primitive column is a null (append_null); an empty
      // Utf8 field is the empty string; anything unparsable is a ParseError.  Restated from the
      // published reader, unpinned: the reference's tests read no file with empty fields
      // (test/data/null_test.csv is not referenced by any test).
      const bool primitive = a.data_type != DFGPU_UTF8;
      if (primitive && s.empty()) {
        set_bit(a.own_validity, rows, false);
        a.null_count++;
        if (a.data_type == DFGPU_BOOL) set_bit(a.own_values, rows, false);
        else a.own_values.resize(a.own_values.size() + size_t(datatype_width(a.data_type)), 0);
        continue;
      }
      if (primitive) set_bit(a.own_validity, rows, true);
      switch (a.data_type) {
        case DFGPU_UTF8:
          a.own_values.insert(a.own_values.end(), s.begin(), s.end());
          a.own_offsets.push_back(int32_t(a.own_values.size()));
          break;
        case DFGPU_BOOL:  // Rust str::parse::<bool>: exactly "true" / "false"
          if (s != "true" && s != "false") goto bad;
          set_bit(a.own_values, rows, s == "true");
          break;
        case DFGPU_FLOAT64: { if (isspace((unsigned char)s[0])) goto bad; double v = strtod(s.c_str(), &end); if (end == s.c_str() || *end) goto bad; push_val(a, v); break; }
        case DFGPU_FLOAT32: { if (isspace((unsigned char)s[0])) goto bad; float v = strtof(s.c_str(), &end); if (end == s.c_str() || *end) goto bad; push_val(a, v); break; }
        // integers: Rust's str::parse rejects white space, trailing characters and values outside the type
        case DFGPU_INT8: { long long v; if (!parse_signed(s, -128, 127, &v)) goto bad; push_val(a, int8_t(v)); break; }
        case DFGPU_INT16: { long long v; if (!parse_signed(s, -32768, 32767, &v)) goto bad; push_val(a, int16_t(v)); break; }
        case DFGPU_INT32: { long long v; if (!parse_signed(s, INT32_MIN, INT32_MAX, &v)) goto bad; push_val(a, int32_t(v)); break; }
        case DFGPU_INT64: { long long v; if (!parse_signed(s, INT64_MIN, INT64_MAX, &v)) goto bad; push_val(a, int64_t(v)); break; }
        case DFGPU_UINT8: { unsigned long long v; if (!parse_unsigned(s, 0xffull, &v)) goto bad; push_val(a, uint8_t(v)); break; }
        case DFGPU_UINT16: { unsigned long long v; if (!parse_unsigned(s, 0xffffull, &v)) goto bad; push_val(a, uint16_t(v)); break; }
        case DFGPU_UINT32: { unsigned long long v; if (!parse_unsigned(s, 0xffffffffull, &v)) goto bad; push_val(a, uint32_t(v)); break; }
        case DFGPU_UINT64: { unsigned long long v; if (!parse_unsigned(s, ~0ull, &v)) goto bad; push_val(a, uint64_t(v)); break; }
        default: fail(DFGPU_ERR_NOT_IMPLEMENTED, std::string("CSV column type ") + datatype_debug(a.data_type));
      }
      continue;
    bad:
      fail(DFGPU_ERR_ARROW, "ParseError(\"Error while parsing value " + s + " at line " + std::to_string(line_no_) + "\")");
    }
    rows++;
  }
  if (rows == 0) return std::nullopt;
  for (auto& a : b.columns) {
    a->len = int64_t(rows);
    if (a->data_type == DFGPU_BOOL) a->own_values.resize((rows + 7) / 8, 0);
    a->values = a->own_values.data();
    a->values_bytes = int64_t(a->own_values.size());
    if (a->data_type == DFGPU_UTF8) a->offsets = a->own_offsets.data();
    if (a->null_count > 0) {
      a->own_validity.resize((rows + 7) / 8, 0);
      a->validity = a->own_validity.data();
    } else {
      a->own_validity.clear();
    }
  }
  b.num_rows = int64_t(rows);
  return b;
}

// ---- memory source ----------------------------------------------------------------------------------
MemoryDataSource::MemoryDataSource(SchemaRef schema, std::vector<ArrayRef> cols, size_t batch_size)
    : schema_(std::move(schema)), cols_(std::move(cols)) {
  nrows_ = cols_.empty() ? 0 : cols_[0]->len;
  for (auto& c : cols_)
    if (c->len != nrows_) fail(DFGPU_ERR_GENERAL, "all columns of a table must have the same length");
  batch_size_ = batch_size ? int64_t(batch_size) : (nrows_ > 0 ? nrows_ : 1);
}

std::optional<RecordBatch> MemoryDataSource::next() {
  if (pos_ >= nrows_) return std::nullopt;
  const int64_t n = std::min(batch_size_, nrows_ - pos_);
  RecordBatch b;
  b.schema = schema_;
  b.num_rows = n;
  for (auto& c : cols_) {
    auto s = std::make_shared<Array>(*c);  // shares the borrowed pointers
    s->offset = c->offset + pos_;
    s->len = n;
    b.columns.push_back(s);
  }
  pos_ += n;
  return b;
}

// ---- built-in scalar functions ---------------------------------------------------------------------------
const std::vector<BuiltinFunction>& builtin_functions() {
  static const std::vector<BuiltinFunction> table = {
      {"sqrt", DFGPU_OP_FN, DFGPU_FN_SQRT, 1, 1, {DFGPU_FLOAT64}, DFGPU_FLOAT64},  {"abs", DFGPU_OP_FN, DFGPU_FN_ABS, 1, 1, {DFGPU_FLOAT64}, DFGPU_FLOAT64},
      {"floor", DFGPU_OP_FN, DFGPU_FN_FLOOR, 1, 1, {DFGPU_FLOAT64}, DFGPU_FLOAT64},  {"ceil", DFGPU_OP_FN, DFGPU_FN_CEIL, 1, 1, {DFGPU_FLOAT64}, DFGPU_FLOAT64},
      {"trunc", DFGPU_OP_FN, DFGPU_FN_TRUNC, 1, 1, {DFGPU_FLOAT64}, DFGPU_FLOAT64},  {"round", DFGPU_OP_FN, DFGPU_FN_ROUND, 1, 1, {DFGPU_FLOAT64}, DFGPU_FLOAT64},
      {"signum", DFGPU_OP_FN, DFGPU_FN_SIGNUM, 1, 1, {DFGPU_FLOAT64}, DFGPU_FLOAT64},  {"exp", DFGPU_OP_FN, DFGPU_FN_EXP, 1, 1, {DFGPU_FLOAT64}, DFGPU_FLOAT64},
      {"ln", DFGPU_OP_FN, DFGPU_FN_LN, 1, 1, {DFGPU_FLOAT64}, DFGPU_FLOAT64},  {"log2", DFGPU_OP_FN, DFGPU_FN_LOG2, 1, 1, {DFGPU_FLOAT64}, DFGPU_FLOAT64},
      {"log10", DFGPU_OP_FN, DFGPU_FN_LOG10, 1, 1, {DFGPU_FLOAT64}, DFGPU_FLOAT64},  {"sin", DFGPU_OP_FN, DFGPU_FN_SIN, 1, 1, {DFGPU_FLOAT64}, DFGPU_FLOAT64},
      {"cos", DFGPU_OP_FN, DFGPU_FN_COS, 1, 1, {DFGPU_FLOAT64}, DFGPU_FLOAT64},  {"tan", DFGPU_OP_FN, DFGPU_FN_TAN, 1, 1, {DFGPU_FLOAT64}, DFGPU_FLOAT64},
      {"asin", DFGPU_OP_FN, DFGPU_FN_ASIN, 1, 1, {DFGPU_FLOAT64}, DFGPU_FLOAT64},  {"acos", DFGPU_OP_FN, DFGPU_FN_ACOS, 1, 1, {DFGPU_FLOAT64}, DFGPU_FLOAT64},
      {"atan", DFGPU_OP_FN, DFGPU_FN_ATAN, 1, 1, {DFGPU_FLOAT64}, DFGPU_FLOAT64},  {"power", DFGPU_OP_FN, DFGPU_FN_POWER, 2, 2, {DFGPU_FLOAT64, DFGPU_FLOAT64}, DFGPU_FLOAT64},
      {"atan2", DFGPU_OP_FN, DFGPU_FN_ATAN2, 2, 2, {DFGPU_FLOAT64, DFGPU_FLOAT64}, DFGPU_FLOAT64},
      // Utf8 functions (DFGPU_OP_UTF8_FN); substr(s, start) is DFGPU_UTF8FN_SUBSTR_FROM
      {"upper", DFGPU_OP_UTF8_FN, DFGPU_UTF8FN_UPPER, 1, 1, {DFGPU_UTF8}, DFGPU_UTF8},
      {"lower", DFGPU_OP_UTF8_FN, DFGPU_UTF8FN_LOWER, 1, 1, {DFGPU_UTF8}, DFGPU_UTF8},
      {"trim", DFGPU_OP_UTF8_FN, DFGPU_UTF8FN_TRIM, 1, 1, {DFGPU_UTF8}, DFGPU_UTF8},
      {"ltrim", DFGPU_OP_UTF8_FN, DFGPU_UTF8FN_LTRIM, 1, 1, {DFGPU_UTF8}, DFGPU_UTF8},
      {"rtrim", DFGPU_OP_UTF8_FN, DFGPU_UTF8FN_RTRIM, 1, 1, {DFGPU_UTF8}, DFGPU_UTF8},
      {"substr", DFGPU_OP_UTF8_FN, DFGPU_UTF8FN_SUBSTR, 2, 3, {DFGPU_UTF8, DFGPU_INT64, DFGPU_INT64}, DFGPU_UTF8},
      {"length", DFGPU_OP_UTF8_FN, DFGPU_UTF8FN_LENGTH, 1, 1, {DFGPU_UTF8}, DFGPU_INT64},
      {"char_length", DFGPU_OP_UTF8_FN, DFGPU_UTF8FN_LENGTH, 1, 1, {DFGPU_UTF8}, DFGPU_INT64},
      {"octet_length", DFGPU_OP_UTF8_FN, DFGPU_UTF8FN_OCTET_LENGTH, 1, 1, {DFGPU_UTF8}, DFGPU_INT64},
  };
  return table;
}

const BuiltinFunction* find_builtin_function(const std::string& name) {
  std::string n = name;
  for (auto& c : n) c = char(tolower((unsigned char)c));
  for (const auto& f : builtin_functions())
    if (n == f.name) return &f;
  return nullptr;
}

std::shared_ptr<FunctionMeta> builtin_function_meta(const std::string& name) {
  const BuiltinFunction* f = find_builtin_function(name);
  if (!f) return nullptr;
  auto fm = std::make_shared<FunctionMeta>();
  fm->name = f->name;
  for (int i = 0; i < f->arity; i++) fm->args.push_back(Field{"n", f->arg_types[i], false});
  fm->return_type = f->return_type;
  return fm;
}

// ---- Expr -> postfix program of the C ABI -------------------------------------------------------------
namespace {

void lower(const Expr& e, const Schema& schema, const std::map<size_t, int>& remap, std::vector<dfgpu_insn>& out) {
  dfgpu_insn in;
  memset(&in, 0, sizeof(in));
  switch (e.kind) {
    case Expr::Column: {
      auto it = remap.find(e.index);
      if (it == remap.end()) fail(DFGPU_ERR_INVALID_COLUMN, "column index out of range");
      in.op = DFGPU_OP_COL;
      in.col = it->second;
      in.dtype = schema.fields[e.index].data_type;
      out.push_back(in);
      return;
    }
    case Expr::Literal: {
      const ScalarValue& v = e.value;
      if (v.dtype == DFGPU_UTF8) {  // an operand of a Utf8 comparison or LIKE; the engine refuses it anywhere else
        in.op = DFGPU_OP_LIT_UTF8;
        in.dtype = DFGPU_UTF8;
        in.col = int(v.s.size());
        in.lit.str = v.s.data();  // the plan's ScalarValue outlives the call
        out.push_back(in);
        return;
      }
      if (!(v.dtype >= DFGPU_INT8 && v.dtype <= DFGPU_FLOAT64))
        fail(DFGPU_ERR_EXECUTION, "No support for literal type " + v.debug());  // expression.rs:306-309
      in.op = DFGPU_OP_LIT;
      in.dtype = v.dtype;
      if (v.dtype == DFGPU_FLOAT64) in.lit.f64 = v.v.d;
      else if (v.dtype == DFGPU_FLOAT32) { in.lit.u64 = 0; in.lit.f32 = v.v.f; }
      else in.lit.u64 = v.v.u;
      out.push_back(in);
      return;
    }
    case Expr::Cast:
      lower(*e.left, schema, remap, out);
      in.op = DFGPU_OP_CAST;
      in.dtype = e.data_type;
      in.col = e.left->kind == Expr::Literal ? e.left->value.dtype : (e.left->kind == Expr::Column ? schema.fields[e.left->index].data_type : 0);
      out.push_back(in);
      return;
    case Expr::BinaryExpr: {
      lower(*e.left, schema, remap, out);
      lower(*e.right, schema, remap, out);
      switch (e.op) {
        case Operator::Eq: in.op = DFGPU_OP_EQ; break;
        case Operator::NotEq: in.op = DFGPU_OP_NE; break;
        case Operator::Lt: in.op = DFGPU_OP_LT; break;
        case Operator::LtEq: in.op = DFGPU_OP_LE; break;
        case Operator::Gt: in.op = DFGPU_OP_GT; break;
        case Operator::GtEq: in.op = DFGPU_OP_GE; break;
        case Operator::And: in.op = DFGPU_OP_AND; break;
        case Operator::Or: in.op = DFGPU_OP_OR; break;
        case Operator::Plus: in.op = DFGPU_OP_ADD; break;
        case Operator::Minus: in.op = DFGPU_OP_SUB; break;
        case Operator::Multiply: in.op = DFGPU_OP_MUL; break;
        case Operator::Divide: in.op = DFGPU_OP_DIV; break;
        case Operator::Like: in.op = DFGPU_OP_LIKE; break;
        case Operator::NotLike: in.op = DFGPU_OP_NOT_LIKE; break;
        default: fail(DFGPU_ERR_EXECUTION, std::string("operator: ") + operator_debug(e.op));  // expression.rs:494-497
      }
      out.push_back(in);
      return;
    }
    case Expr::ScalarFunction: {
      const BuiltinFunction* f = find_builtin_function(e.name);
      if (!f) fail(DFGPU_ERR_GENERAL, "Invalid function '" + e.name + "'");
      // the planner rejects extra arguments but not missing ones
      if (e.args.size() < size_t(f->min_arity) || e.args.size() > size_t(f->arity))
        fail(DFGPU_ERR_EXECUTION, "function '" + e.name + "' takes " +
                                      (f->min_arity < f->arity ? std::to_string(f->min_arity) + " or " : std::string()) + std::to_string(f->arity) +
                                      (f->arity == 1 ? " argument" : " arguments") + ", got " + std::to_string(e.args.size()));
      for (auto& a : e.args) lower(*a, schema, remap, out);
      in.op = f->op;
      in.col = f->code == DFGPU_UTF8FN_SUBSTR && e.args.size() == 2 ? DFGPU_UTF8FN_SUBSTR_FROM : f->code;
      in.dtype = f->return_type;
      out.push_back(in);
      return;
    }
    case Expr::Case:
      for (auto& a : e.args) lower(*a, schema, remap, out);
      in.op = DFGPU_OP_CASE;
      in.col = int(e.args.size());
      in.dtype = e.get_type(schema);
      out.push_back(in);
      return;
    default: fail(DFGPU_ERR_EXECUTION, "expression " + e.debug());  // expression.rs:500-503
  }
}

// Rust `{}` (Display) of a number, as literal_array! names its closure (expression.rs:230)
std::string display_number(const ScalarValue& v) {
  switch (v.dtype) {
    case DFGPU_FLOAT64: { std::string s = rust_debug_f64(v.v.d); if (s.size() > 2 && s.compare(s.size() - 2, 2, ".0") == 0) s.resize(s.size() - 2); return s; }
    case DFGPU_FLOAT32: { std::string s = rust_debug_f64(double(v.v.f)); if (s.size() > 2 && s.compare(s.size() - 2, 2, ".0") == 0) s.resize(s.size() - 2); return s; }
    case DFGPU_INT8: case DFGPU_INT16: case DFGPU_INT32: case DFGPU_INT64: return std::to_string(v.v.i);
    default: return std::to_string(v.v.u);
  }
}

struct Pruned {
  std::map<size_t, int> remap;       // input column index -> uploaded column index
  std::vector<size_t> cols;          // uploaded column -> input column index
};

Pruned prune(const std::vector<ExprRef>& exprs, size_t ncols, bool all) {
  std::set<size_t> acc;
  if (all) for (size_t i = 0; i < ncols; i++) acc.insert(i);
  for (auto& e : exprs) if (e) collect_columns(*e, acc);
  Pruned p;
  for (size_t c : acc) {
    if (c >= ncols) fail(DFGPU_ERR_INVALID_COLUMN, "column index out of range");
    p.remap[c] = int(p.cols.size());
    p.cols.push_back(c);
  }
  return p;
}

struct BatchGuard {
  dfgpu_batch* b = nullptr;
  ~BatchGuard() { if (b) dfgpu_batch_free(b); }
};
struct ResultGuard {
  dfgpu_result* r = nullptr;
  ~ResultGuard() { if (r) dfgpu_result_free(r); }
};

dfgpu_batch* upload(dfgpu_ctx* gpu, const RecordBatch& batch, const Pruned& p) {
  std::vector<dfgpu_col> cols;
  for (size_t c : p.cols) cols.push_back(batch.columns[c]->view());
  if (cols.empty()) {
    // a query that references no column still needs the row count: upload a 1-byte-per-row dummy? no —
    // carry the row count through an empty Int8 column view of the first input column's length
    fail(DFGPU_ERR_NOT_IMPLEMENTED, "queries that reference no column");
  }
  dfgpu_batch* out = nullptr;
  GPU_CHECK(dfgpu_batch_upload(gpu, cols.data(), int(cols.size()), &out));
  return out;
}

// `schema`'s columns of `r`: its first schema->fields.size() columns, or all of them when it has no fields
RecordBatch download(dfgpu_result* r, SchemaRef schema) {
  RecordBatch out;
  out.schema = std::move(schema);
  int64_t nrows = 0;
  int ncols = 0;
  GPU_CHECK(dfgpu_result_shape(r, &nrows, &ncols));
  if (out.schema && !out.schema->fields.empty()) ncols = std::min(ncols, int(out.schema->fields.size()));
  out.num_rows = nrows;
  for (int i = 0; i < ncols; i++) {
    auto a = std::make_shared<Array>();
    int32_t dt = 0;
    int64_t nulls = 0, nbytes = 0;
    GPU_CHECK(dfgpu_result_col_dtype(r, i, &dt));
    GPU_CHECK(dfgpu_result_col_nulls(r, i, &nulls));
    GPU_CHECK(dfgpu_result_col_bytes(r, i, &nbytes));
    a->data_type = dt;
    a->len = nrows;
    a->null_count = nulls;
    a->own_values.resize(size_t(nbytes > 0 ? nbytes : 1));
    if (nulls > 0) a->own_validity.resize(size_t((nrows + 7) / 8));
    if (dt == DFGPU_UTF8) a->own_offsets.resize(size_t(nrows + 1));
    GPU_CHECK(dfgpu_result_copy_col(r, i, a->own_values.data(), nulls > 0 ? a->own_validity.data() : nullptr,
                                    dt == DFGPU_UTF8 ? a->own_offsets.data() : nullptr));
    a->values = a->own_values.data();
    a->values_bytes = nbytes;
    a->validity = nulls > 0 ? a->own_validity.data() : nullptr;
    a->offsets = dt == DFGPU_UTF8 ? a->own_offsets.data() : nullptr;
    out.columns.push_back(a);
  }
  return out;
}

}  // namespace

std::string runtime_expr_name(const Expr& e, const Schema& s) {
  switch (e.kind) {
    case Expr::Column: return e.index < s.fields.size() ? s.fields[e.index].name : "?";
    case Expr::Literal: return display_number(e.value);
    case Expr::Cast: return e.left->kind == Expr::Column ? runtime_expr_name(*e.left, s) : "lit";
    case Expr::BinaryExpr: return e.left->debug() + " " + operator_debug(e.op) + " " + e.right->debug();
    case Expr::AggregateFunction: case Expr::ScalarFunction: return e.name;
    default: return e.debug();
  }
}

// ---- GPU relations ---------------------------------------------------------------------------------------
GpuFilterProjectRelation::GpuFilterProjectRelation(dfgpu_ctx* gpu, RelationRef input, ExprRef predicate, std::vector<ExprRef> proj, SchemaRef schema)
    : gpu_(gpu), input_(std::move(input)), predicate_(std::move(predicate)), proj_(std::move(proj)), schema_(std::move(schema)) {}

std::optional<RecordBatch> GpuFilterProjectRelation::next() {
  auto batch = input_->next();
  if (!batch) return std::nullopt;
  // proj_ empty: FilterRelation alone gathers every input column (filter.rs:55-57).
  std::vector<ExprRef> exprs = proj_;
  if (exprs.empty())
    for (size_t c = 0; c < batch->columns.size(); c++) exprs.push_back(Expr::column(c));
  // One kernel pass takes a bounded number of distinct columns and expressions (kMaxCols / kMaxProgs of
  // expr_vm.cuh), so a wide select list is evaluated in several passes over groups of expressions; every pass
  // evaluates the same predicate and therefore keeps the same rows in the same order.
  constexpr size_t kCols = 12, kProgs = 23;
  std::set<size_t> pcols;
  if (predicate_) collect_columns(*predicate_, pcols);
  std::vector<std::vector<size_t>> groups(1);
  std::set<size_t> used = pcols;
  for (size_t i = 0; i < exprs.size(); i++) {
    std::set<size_t> with = used;
    collect_columns(*exprs[i], with);
    if (!groups.back().empty() && (with.size() > kCols || groups.back().size() >= kProgs)) {
      groups.emplace_back();
      with = pcols;
      collect_columns(*exprs[i], with);
    }
    used = with;
    groups.back().push_back(i);
  }
  if (groups.size() == 1) return process(*batch, exprs, schema_);
  RecordBatch out;
  out.schema = schema_;
  for (auto& g : groups) {
    std::vector<ExprRef> part_exprs;
    auto sub = std::make_shared<Schema>();
    for (size_t i : g) {
      part_exprs.push_back(exprs[i]);
      sub->fields.push_back(schema_->fields[i]);
    }
    RecordBatch part = process(*batch, part_exprs, sub);
    out.num_rows = part.num_rows;
    for (auto& col : part.columns) out.columns.push_back(col);
  }
  return out;
}

RecordBatch GpuFilterProjectRelation::process(const RecordBatch& in_batch, const std::vector<ExprRef>& proj, const SchemaRef& out_schema) {
  const RecordBatch* batch = &in_batch;
  const Schema& in_schema = *input_->schema();
  std::vector<ExprRef> all = proj;
  all.push_back(predicate_);
  Pruned pr = prune(all, batch->columns.size(), false);
  std::vector<dfgpu_insn> pred;
  if (predicate_) lower(*predicate_, in_schema, pr.remap, pred);
  std::vector<std::vector<dfgpu_insn>> progs;
  for (auto& e : proj) {
    progs.emplace_back();
    lower(*e, in_schema, pr.remap, progs.back());
  }
  std::vector<const dfgpu_insn*> pp;
  std::vector<int> pl;
  for (auto& p : progs) { pp.push_back(p.data()); pl.push_back(int(p.size())); }
  // Large batches: host buffers straight in.  The library overlaps upload, kernel and download by row-range chunk
  // when it can and returns pinned host columns, wrapped zero-copy here (the pinned block lives as long as the
  // RecordBatch); otherwise it runs the resident operator on the whole batch and the result is in device memory.
  if (batch->num_rows >= (4ll << 20)) {
    std::vector<dfgpu_col> cols;
    for (size_t c : pr.cols) cols.push_back(batch->columns[c]->view());
    if (cols.empty()) fail(DFGPU_ERR_NOT_IMPLEMENTED, "queries that reference no column");
    ResultGuard r;
    GPU_CHECK(dfgpu_filter_project_host(gpu_, cols.data(), int(cols.size()), pred.data(), int(pred.size()), pp.data(), pl.data(), int(pp.size()), 0, &r.r));
    int on_host = 0;
    GPU_CHECK(dfgpu_result_on_host(r.r, &on_host));
    if (!on_host) return download(r.r, out_schema);
    dfgpu_result* raw = r.r;
    r.r = nullptr;
    std::shared_ptr<void> owner(raw, [](void* p) { dfgpu_result_free(static_cast<dfgpu_result*>(p)); });
    RecordBatch out;
    out.schema = out_schema;
    int64_t nrows = 0;
    int ncols = 0;
    GPU_CHECK(dfgpu_result_shape(raw, &nrows, &ncols));
    out.num_rows = nrows;
    for (int i = 0; i < ncols; i++) {
      auto a = std::make_shared<Array>();
      int32_t dt = 0;
      const void* hp = nullptr;
      GPU_CHECK(dfgpu_result_col_dtype(raw, i, &dt));
      GPU_CHECK(dfgpu_result_col_host_ptr(raw, i, &hp));
      a->data_type = dt;
      a->len = nrows;
      a->values = hp;
      a->values_bytes = nrows * datatype_width(dt);
      a->owner = owner;
      out.columns.push_back(a);
    }
    return out;
  }
  BatchGuard b;
  b.b = upload(gpu_, *batch, pr);
  ResultGuard r;
  GPU_CHECK(dfgpu_filter_project(gpu_, b.b, pred.data(), int(pred.size()), pp.data(), pl.data(), int(pp.size()), &r.r));
  return download(r.r, out_schema);
}

// ---- join -------------------------------------------------------------------------------------------------
namespace {

void set_bit(std::vector<uint8_t>& bits, int64_t i, bool v) {
  if (v) bits[size_t(i >> 3)] |= uint8_t(1u << (i & 7));
}
bool get_bit(const uint8_t* bits, int64_t i) { return (bits[i >> 3] >> (i & 7)) & 1; }

// One owned array holding column `c` of every batch, in order (Utf8 offsets rebased, bitmaps re-packed).
ArrayRef concat_column(const std::vector<RecordBatch>& batches, size_t c, DataType dt) {
  auto out = std::make_shared<Array>();
  out->data_type = dt;
  int64_t n = 0, nulls = 0;
  for (auto& b : batches) {
    n += b.columns[c]->len;
    nulls += b.columns[c]->null_count;
  }
  out->len = n;
  out->null_count = nulls;
  if (nulls > 0) out->own_validity.assign(size_t((n + 7) / 8), 0);
  const int w = datatype_width(dt);
  if (dt == DFGPU_BOOL) out->own_values.assign(size_t((n + 7) / 8), 0);
  else if (w > 0) out->own_values.resize(size_t(n) * size_t(w));
  if (dt == DFGPU_UTF8) out->own_offsets.assign(1, 0);
  int64_t row = 0;
  for (auto& b : batches) {
    const Array& a = *b.columns[c];
    for (int64_t r = 0; r < a.len && nulls > 0; r++)
      set_bit(out->own_validity, row + r, a.null_count == 0 || !a.validity || get_bit(a.validity, a.offset + r));
    if (dt == DFGPU_BOOL) {
      for (int64_t r = 0; r < a.len; r++) set_bit(out->own_values, row + r, get_bit(static_cast<const uint8_t*>(a.values), a.offset + r));
    } else if (w > 0) {
      if (a.len > 0) memcpy(out->own_values.data() + size_t(row) * size_t(w), static_cast<const uint8_t*>(a.values) + size_t(a.offset) * size_t(w), size_t(a.len) * size_t(w));
    } else if (dt == DFGPU_UTF8) {
      const int32_t lo = a.offsets[a.offset], base = out->own_offsets.back();
      if (int64_t(base) + a.offsets[a.offset + a.len] - lo >= (int64_t(1) << 31)) fail(DFGPU_ERR_NOT_IMPLEMENTED, "JOIN build column of more than 2 GiB of Utf8");
      const uint8_t* bytes = static_cast<const uint8_t*>(a.values);
      out->own_values.insert(out->own_values.end(), bytes + lo, bytes + a.offsets[a.offset + a.len]);
      for (int64_t r = 1; r <= a.len; r++) out->own_offsets.push_back(base + (a.offsets[a.offset + r] - lo));
    }
    row += a.len;
  }
  out->values = out->own_values.data();
  out->values_bytes = int64_t(out->own_values.size());
  out->validity = nulls > 0 ? out->own_validity.data() : nullptr;
  out->offsets = dt == DFGPU_UTF8 ? out->own_offsets.data() : nullptr;
  return out;
}

std::vector<ExprRef> column_exprs(const std::vector<size_t>& cols) {
  std::vector<ExprRef> v;
  for (size_t c : cols) v.push_back(Expr::column(c));
  return v;
}

struct Programs {
  std::vector<std::vector<dfgpu_insn>> progs;
  std::vector<const dfgpu_insn*> ptr;
  std::vector<int> len;
  Programs(const std::vector<ExprRef>& exprs, const Schema& schema, const Pruned& pr) : progs(exprs.size()) {
    for (size_t i = 0; i < exprs.size(); i++) {
      lower(*exprs[i], schema, pr.remap, progs[i]);
      ptr.push_back(progs[i].data());
      len.push_back(int(progs[i].size()));
    }
  }
};

}  // namespace

GpuHashJoinRelation::GpuHashJoinRelation(dfgpu_ctx* gpu, SchemaRef schema, RelationRef left, RelationRef right, std::vector<ExprRef> left_keys,
                                         std::vector<ExprRef> right_keys, std::vector<size_t> left_cols, std::vector<size_t> right_cols,
                                         LogicalPlan::JoinKind kind)
    : gpu_(gpu), schema_(std::move(schema)), left_(std::move(left)), right_(std::move(right)), left_keys_(std::move(left_keys)),
      right_keys_(std::move(right_keys)), left_cols_(std::move(left_cols)), right_cols_(std::move(right_cols)), kind_(kind) {}

GpuHashJoinRelation::~GpuHashJoinRelation() { release(); }

void GpuHashJoinRelation::release() {
  if (join_) dfgpu_join_free(join_);
  join_ = nullptr;
  released_ = true;
}

void GpuHashJoinRelation::build() {
  std::vector<RecordBatch> batches;
  while (auto b = right_->next()) batches.push_back(std::move(*b));
  const Schema& rs = *right_->schema();
  std::vector<ExprRef> all = right_keys_;
  for (auto& e : column_exprs(right_cols_)) all.push_back(e);
  Pruned pr = prune(all, rs.fields.size(), false);
  RecordBatch whole;  // the referenced columns of every batch, concatenated (the build table is built once)
  whole.columns.resize(rs.fields.size());
  for (size_t c : pr.cols) whole.columns[c] = concat_column(batches, c, rs.fields[c].data_type);
  BatchGuard b;
  b.b = upload(gpu_, whole, pr);
  batches.clear();
  Programs keys(right_keys_, rs, pr);
  std::vector<int> keep;
  for (size_t c : right_cols_) keep.push_back(pr.remap.at(c));
  GPU_CHECK(dfgpu_join_build(gpu_, b.b, keys.ptr.data(), keys.len.data(), int(keys.ptr.size()), keep.data(), int(keep.size()), &join_));
  build_out_ = keep;
}

std::optional<RecordBatch> GpuHashJoinRelation::next() {
  if (released_) return std::nullopt;
  if (!join_) build();
  auto batch = left_->next();
  if (!batch) {  // probe side exhausted: the table is not needed any more
    release();
    return std::nullopt;
  }
  const Schema& ls = *left_->schema();
  std::vector<ExprRef> all = left_keys_;
  for (auto& e : column_exprs(left_cols_)) all.push_back(e);
  Pruned pr = prune(all, batch->columns.size(), false);
  BatchGuard b;
  b.b = upload(gpu_, *batch, pr);
  Programs keys(left_keys_, ls, pr);
  std::vector<int> probe_cols;
  for (size_t c : left_cols_) probe_cols.push_back(pr.remap.at(c));
  ResultGuard r;
  if (kind_ == LogicalPlan::JoinKind::Inner) {
    GPU_CHECK(dfgpu_join_probe(join_, b.b, keys.ptr.data(), keys.len.data(), int(keys.ptr.size()), probe_cols.data(), int(probe_cols.size()),
                               build_out_.data(), int(build_out_.size()), &r.r));
  } else {
    const int kind = kind_ == LogicalPlan::JoinKind::Semi ? DFGPU_JOIN_SEMI : kind_ == LogicalPlan::JoinKind::Anti ? DFGPU_JOIN_ANTI : DFGPU_JOIN_ANTI_NULL_AWARE;
    GPU_CHECK(dfgpu_join_semi(join_, b.b, keys.ptr.data(), keys.len.data(), int(keys.ptr.size()), kind, probe_cols.data(), int(probe_cols.size()), &r.r));
  }
  RecordBatch got = download(r.r, schema_);
  RecordBatch out;
  out.schema = schema_;
  out.num_rows = got.num_rows;
  for (auto& f : schema_->fields) {  // placeholders: dtype and length only
    auto a = std::make_shared<Array>();
    a->data_type = f.data_type;
    a->len = got.num_rows;
    out.columns.push_back(a);
  }
  const size_t nl = ls.fields.size();
  for (size_t i = 0; i < left_cols_.size(); i++) out.columns[left_cols_[i]] = got.columns[i];
  for (size_t i = 0; i < right_cols_.size(); i++) out.columns[nl + right_cols_[i]] = got.columns[left_cols_.size() + i];
  return out;
}

GpuWindowRelation::GpuWindowRelation(dfgpu_ctx* gpu, SchemaRef schema, RelationRef input, std::vector<size_t> cols, bool projected,
                                     std::vector<ExprRef> window_expr)
    : gpu_(gpu), schema_(std::move(schema)), input_(std::move(input)), cols_(std::move(cols)), projected_(projected), window_expr_(std::move(window_expr)) {}

std::optional<RecordBatch> GpuWindowRelation::next() {
  if (done_) return std::nullopt;
  done_ = true;
  std::vector<RecordBatch> batches;
  while (auto b = input_->next()) batches.push_back(std::move(*b));
  const size_t nin = schema_->fields.size() - window_expr_.size();
  RecordBatch whole;  // the window's input: the columns in cols_, concatenated; placeholders elsewhere
  whole.schema = schema_;
  for (auto& b : batches) whole.num_rows += b.num_rows;
  for (size_t c = 0; c < nin; c++) {
    auto a = std::make_shared<Array>();
    a->data_type = schema_->fields[c].data_type;
    a->len = whole.num_rows;
    whole.columns.push_back(a);
  }
  for (size_t k = 0; k < cols_.size(); k++)
    whole.columns[cols_[k]] = concat_column(batches, projected_ ? k : cols_[k], schema_->fields[cols_[k]].data_type);
  batches.clear();
  int64_t world = 1;
  dfgpu_comm_world(gpu_, &world);
  if (whole.num_rows == 0 && world == 1) return std::nullopt;
  // the columns every call reads, uploaded once
  std::vector<ExprRef> all;
  for (auto& w : window_expr_) all.push_back(w);
  Pruned pr = prune(all, nin, false);
  if (pr.cols.empty()) {  // only ranks over no key: any column carries the row count
    pr.remap[cols_[0]] = 0;
    pr.cols.push_back(cols_[0]);
  }
  const Schema& in_schema = *schema_;
  BatchGuard b;
  b.b = upload(gpu_, whole, pr);
  std::vector<ArrayRef> out(window_expr_.size());
  std::vector<bool> done(window_expr_.size(), false);
  for (size_t i = 0; i < window_expr_.size(); i++) {
    if (done[i]) continue;
    // every call of this OVER specification
    const Expr& w = *window_expr_[i];
    auto spec = [](const Expr& e) {
      std::string s;
      for (auto& p : e.partition_by) s += p->debug() + ",";
      s += "|";
      for (auto& o : e.order_by) s += o->debug() + ",";
      return s;
    };
    std::vector<size_t> calls;
    for (size_t j = i; j < window_expr_.size(); j++)
      if (!done[j] && spec(*window_expr_[j]) == spec(w)) calls.push_back(j);
    std::vector<ExprRef> okeys;
    std::vector<int32_t> desc;
    for (auto& o : w.order_by) {
      okeys.push_back(o->left);
      desc.push_back(o->asc ? 0 : 1);
    }
    const Programs part(w.partition_by, in_schema, pr), order(okeys, in_schema, pr);
    std::vector<std::vector<dfgpu_insn>> args(calls.size());
    std::vector<dfgpu_agg> fns(calls.size());
    for (size_t k = 0; k < calls.size(); k++) {
      const Expr& e = *window_expr_[calls[k]];
      std::string n = e.name;
      for (auto& c : n) c = char(tolower((unsigned char)c));
      int f = n == "row_number" ? DFGPU_WIN_ROW_NUMBER : n == "rank" ? DFGPU_WIN_RANK : n == "dense_rank" ? DFGPU_WIN_DENSE_RANK : 0;
      if (!f) f = n == "min" ? DFGPU_AGG_MIN : n == "max" ? DFGPU_AGG_MAX : n == "sum" ? DFGPU_AGG_SUM : n == "count" ? DFGPU_AGG_COUNT : DFGPU_AGG_AVG;
      if (!e.args.empty()) lower(*e.args[0], in_schema, pr.remap, args[k]);
      memset(&fns[k], 0, sizeof(dfgpu_agg));
      fns[k].func = f;
      fns[k].arg = args[k].empty() ? nullptr : args[k].data();
      fns[k].arg_len = int(args[k].size());
      fns[k].out_dtype = e.data_type;
    }
    ResultGuard r;
    GPU_CHECK(dfgpu_window(gpu_, b.b, part.ptr.data(), part.len.data(), int(part.ptr.size()), order.ptr.data(), order.len.data(), desc.data(),
                           int(order.ptr.size()), fns.data(), int(fns.size()), &r.r));
    RecordBatch got = download(r.r, nullptr);
    for (size_t k = 0; k < calls.size(); k++) {
      out[calls[k]] = got.columns[k];
      done[calls[k]] = true;
    }
  }
  if (whole.num_rows == 0) return std::nullopt;  // this rank had no rows: it joined the exchange only
  for (auto& a : out) whole.columns.push_back(a);
  return whole;
}

const std::vector<RecordBatch>& SharedScan::batches() {
  if (!drained_) {
    while (auto b = ds_->next()) batches_.push_back(std::move(*b));
    drained_ = true;
  }
  return batches_;
}

std::optional<RecordBatch> SharedScanRelation::next() {
  const auto& all = scan_->batches();
  if (pos_ >= all.size()) return std::nullopt;
  return all[pos_++];
}

GpuAggregateRelation::GpuAggregateRelation(dfgpu_ctx* gpu, SchemaRef schema, RelationRef input, std::vector<ExprRef> group_expr,
                                           std::vector<ExprRef> aggr_expr, ExprRef predicate, std::optional<ResultStage> stage)
    : gpu_(gpu), schema_(std::move(schema)), input_(std::move(input)), group_expr_(std::move(group_expr)), aggr_expr_(std::move(aggr_expr)),
      predicate_(std::move(predicate)), stage_(std::move(stage)) {}

RecordBatch GpuAggregateRelation::finish(dfgpu_aggstate* st) {
  ResultGuard r;
  GPU_CHECK(dfgpu_aggregate_finish(st, &r.r));
  if (!stage_) return download(r.r, schema_);
  // every rank holds the same global result, so each sorts it alike and no collective is needed
  const Schema& as = *stage_->aggregate_schema;
  BatchGuard view;  // freed before the result it views
  GPU_CHECK(dfgpu_result_as_batch(r.r, &view.b));
  const Pruned cols = prune({}, as.fields.size(), true);
  std::vector<dfgpu_insn> keep;
  if (stage_->keep) lower(*stage_->keep, as, cols.remap, keep);
  std::vector<ExprRef> keys;
  std::vector<int32_t> desc;
  for (auto& s : stage_->sort) {
    keys.push_back(s->left);
    desc.push_back(s->asc ? 0 : 1);
  }
  if (stage_->ordered)
    for (size_t k = 0; k < group_expr_.size(); k++) {
      keys.push_back(Expr::column(k));
      desc.push_back(0);
    }
  const Programs kp(keys, as, cols);
  ResultGuard sorted;
  GPU_CHECK(dfgpu_sort(gpu_, view.b, keep.data(), int(keep.size()), kp.ptr.data(), kp.len.data(), desc.data(), int(keys.size()), stage_->limit,
                       &sorted.r));
  return download(sorted.r, schema_);
}

std::optional<RecordBatch> ShardRelation::next() {
  auto batch = input_->next();
  if (!batch) return std::nullopt;
  const int64_t n = batch->num_rows, per = (n + world_ - 1) / world_;
  const int64_t lo = std::min<int64_t>(n, int64_t(rank_) * per), hi = std::min<int64_t>(n, lo + per);
  RecordBatch out;
  out.schema = batch->schema;
  out.num_rows = hi - lo;
  for (auto& c : batch->columns) {
    auto s = std::make_shared<Array>(*c);  // shares the buffers
    s->offset = c->offset + lo;
    s->len = hi - lo;
    if (c->null_count > 0 && c->validity) {
      int64_t nulls = 0;
      for (int64_t r = 0; r < s->len; r++) nulls += !((c->validity[(s->offset + r) >> 3] >> ((s->offset + r) & 7)) & 1);
      s->null_count = nulls;
    }
    if (!c->own_values.empty()) { s->values = s->own_values.data(); }
    if (!c->own_validity.empty()) { s->validity = s->own_validity.data(); }
    if (!c->own_offsets.empty()) { s->offsets = s->own_offsets.data(); }
    out.columns.push_back(s);
  }
  return out;
}

std::optional<RecordBatch> GpuAggregateRelation::next() {
  if (end_of_results_) return std::nullopt;  // aggregate.rs:616-619
  end_of_results_ = true;
  const Schema& in_schema = *input_->schema();
  std::vector<ExprRef> all = group_expr_;
  std::vector<int> funcs;
  for (auto& a : aggr_expr_) {
    if (a->kind != Expr::AggregateFunction) fail(DFGPU_ERR_GENERAL, "Invalid aggregate expression");
    if (a->args.size() != 1) fail(DFGPU_ERR_INTERNAL, "aggregate functions take exactly one argument (reference: assert_eq! at expression.rs:91)");
    std::string n = a->name;
    for (auto& c : n) c = char(tolower((unsigned char)c));
    int f = n == "min" ? DFGPU_AGG_MIN : n == "max" ? DFGPU_AGG_MAX : n == "sum" ? DFGPU_AGG_SUM : n == "count" ? DFGPU_AGG_COUNT : 0;
    if (n == "avg") f = DFGPU_AGG_AVG;
    if (a->distinct) f = f == DFGPU_AGG_COUNT ? DFGPU_AGG_COUNT_DISTINCT : 0;
    if (!f) fail(DFGPU_ERR_GENERAL, "Unsupported aggregate function '" + a->name + "'");  // expression.rs:103-106
    funcs.push_back(f);
    all.push_back(a->args[0]);
  }
  if (predicate_) all.push_back(predicate_);
  dfgpu_aggstate* st = nullptr;
  struct StGuard { dfgpu_aggstate** s; ~StGuard() { if (*s) dfgpu_aggregate_free(*s); } } sg{&st};
  std::optional<Pruned> pr;
  while (auto batch = input_->next()) {
    if (!pr) {
      pr = prune(all, batch->columns.size(), false);
      std::vector<std::vector<dfgpu_insn>> kp(group_expr_.size()), ap(aggr_expr_.size());
      std::vector<const dfgpu_insn*> kptr;
      std::vector<int> klen;
      for (size_t k = 0; k < group_expr_.size(); k++) {
        lower(*group_expr_[k], in_schema, pr->remap, kp[k]);
        kptr.push_back(kp[k].data());
        klen.push_back(int(kp[k].size()));
      }
      std::vector<dfgpu_agg> aggs(aggr_expr_.size());
      for (size_t a = 0; a < aggr_expr_.size(); a++) {
        lower(*aggr_expr_[a]->args[0], in_schema, pr->remap, ap[a]);
        aggs[a].func = funcs[a];
        aggs[a].arg = ap[a].data();
        aggs[a].arg_len = int(ap[a].size());
        aggs[a].out_dtype = aggr_expr_[a]->data_type;
        aggs[a]._pad = 0;
      }
      GPU_CHECK(dfgpu_aggregate_create(gpu_, kptr.data(), klen.data(), int(kptr.size()), aggs.data(), int(aggs.size()), 0, &st));
      if (predicate_) {  // Aggregate{input: Selection}: the WHERE clause runs inside the scan kernel
        std::vector<dfgpu_insn> pred;
        lower(*predicate_, in_schema, pr->remap, pred);
        GPU_CHECK(dfgpu_aggregate_set_predicate(st, pred.data(), int(pred.size())));
      }
    }
    // host buffers straight in: large batches are uploaded in chunks that overlap with the scan
    std::vector<dfgpu_col> cols;
    for (size_t c : pr->cols) cols.push_back(batch->columns[c]->view());
    if (cols.empty()) fail(DFGPU_ERR_NOT_IMPLEMENTED, "queries that reference no column");
    GPU_CHECK(dfgpu_aggregate_update_host(st, cols.data(), int(cols.size()), 0));
  }
  if (!st) {
    // empty input: no GROUP BY -> one row of nulls; GROUP BY -> empty batch (with a communicator attached the
    // rank still has to join the exchange: an empty aggregate state does that)
    int64_t world = 1;
    dfgpu_comm_world(gpu_, &world);
    if (!group_expr_.empty() && world > 1) {
      const Schema& isch = in_schema;
      std::vector<ExprRef> ex = group_expr_;
      for (auto& a : aggr_expr_) ex.push_back(a->args[0]);
      Pruned p0 = prune(ex, isch.fields.size(), false);
      std::vector<std::vector<dfgpu_insn>> kp(group_expr_.size()), ap(aggr_expr_.size());
      std::vector<const dfgpu_insn*> kptr;
      std::vector<int> klen;
      for (size_t k = 0; k < group_expr_.size(); k++) {
        lower(*group_expr_[k], isch, p0.remap, kp[k]);
        kptr.push_back(kp[k].data());
        klen.push_back(int(kp[k].size()));
      }
      std::vector<dfgpu_agg> aggs(aggr_expr_.size());
      for (size_t a = 0; a < aggr_expr_.size(); a++) {
        lower(*aggr_expr_[a]->args[0], isch, p0.remap, ap[a]);
        aggs[a].func = funcs[a];
        aggs[a].arg = ap[a].data();
        aggs[a].arg_len = int(ap[a].size());
        aggs[a].out_dtype = aggr_expr_[a]->data_type;
        aggs[a]._pad = 0;
      }
      GPU_CHECK(dfgpu_aggregate_create(gpu_, kptr.data(), klen.data(), int(kptr.size()), aggs.data(), int(aggs.size()), 0, &st));
      return finish(st);
    }
    if (!group_expr_.empty()) {
      RecordBatch out;
      out.schema = schema_;
      return out;
    }
    std::vector<std::vector<dfgpu_insn>> ap(aggr_expr_.size());
    std::vector<dfgpu_agg> aggs(aggr_expr_.size());
    for (size_t a = 0; a < aggr_expr_.size(); a++) {
      dfgpu_insn in;
      memset(&in, 0, sizeof(in));
      in.op = DFGPU_OP_COL;
      ap[a].push_back(in);
      aggs[a].func = funcs[a];
      aggs[a].arg = ap[a].data();
      aggs[a].arg_len = 1;
      aggs[a].out_dtype = aggr_expr_[a]->data_type;
      aggs[a]._pad = 0;
    }
    GPU_CHECK(dfgpu_aggregate_create(gpu_, nullptr, nullptr, 0, aggs.data(), int(aggs.size()), 0, &st));
  }
  return finish(st);
}

// ---- ExecutionContext ----------------------------------------------------------------------------------
namespace {
struct ContextSchemaProvider : SchemaProvider {  // context.rs:244-258
  std::shared_ptr<std::map<std::string, DataSourceRef>> datasources;
  SchemaRef get_table_meta(const std::string& name) const override {
    auto it = datasources->find(name);
    return it == datasources->end() ? nullptr : it->second->schema();
  }
  // the built-in catalogue; the reference has unimplemented!() here (context.rs:255-257)
  std::shared_ptr<FunctionMeta> get_function_meta(const std::string& name) const override { return builtin_function_meta(name); }
};
}  // namespace

ExecutionContext::ExecutionContext(int device) : datasources_(std::make_shared<std::map<std::string, DataSourceRef>>()) {
  GPU_CHECK(dfgpu_init(device, &gpu_));
}
ExecutionContext::~ExecutionContext() {
  for (auto& w : joins_)
    if (auto j = w.lock()) j->release();
  if (gpu_) dfgpu_shutdown(gpu_);
}

void ExecutionContext::set_partition(int rank, int world, const uint8_t* nccl_unique_id) {
  GPU_CHECK(dfgpu_comm_init(gpu_, rank, world, nccl_unique_id));
  rank_ = rank;
  world_ = world;
}

void ExecutionContext::register_datasource(const std::string& name, DataSourceRef ds) { (*datasources_)[name] = std::move(ds); }

PlanRef ExecutionContext::plan(const std::string& sql) {
  ASTRef ast = parse_sql(sql);
  auto sp = std::make_shared<ContextSchemaProvider>();
  sp->datasources = datasources_;
  return SqlToRel(sp).sql_to_rel(ast);
}

RelationRef ExecutionContext::sql(const std::string& sql) { return execute(plan(sql)); }

namespace {
// The Aggregate under the result stage `top` of an aggregate query (Projection? Limit? Sort? Selection? over it, at
// least one of them), with the stage in *st; null when `top` is not one
const LogicalPlan* aggregate_under(const LogicalPlan& top, GpuAggregateRelation::ResultStage* st) {
  const LogicalPlan* p = &top;
  if (p->kind == LogicalPlan::Projection) p = p->input.get();
  if (p->kind == LogicalPlan::Limit) {
    st->limit = int64_t(p->limit);
    st->ordered = true;
    p = p->input.get();
  }
  if (p->kind == LogicalPlan::Sort) {
    st->sort = p->expr;
    st->ordered = true;
    p = p->input.get();
  }
  if (p->kind == LogicalPlan::Selection) {
    st->keep = p->expr[0];
    p = p->input.get();
  }
  if (p == &top || p->kind != LogicalPlan::Aggregate) return nullptr;
  st->aggregate_schema = p->schema();
  return p;
}

void count_scans(const LogicalPlan& p, std::map<std::string, int>& n) {
  if (p.kind == LogicalPlan::TableScan) n[p.table_name]++;
  if (p.input) count_scans(*p.input, n);
  if (p.right) count_scans(*p.right, n);
}
}  // namespace

RelationRef ExecutionContext::execute(const PlanRef& plan) {
  // a table the plan scans more than once is drained once and replayed to each scan; a table scanned once is read as is
  std::map<std::string, int> scans;
  count_scans(*plan, scans);
  shared_.clear();
  for (auto& [name, n] : scans) {
    auto it = datasources_->find(name);
    if (n > 1 && it != datasources_->end()) shared_[name] = std::make_shared<SharedScan>(it->second);
  }
  RelationRef r = execute_node(plan, nullptr, true);
  shared_.clear();
  return r;
}

RelationRef ExecutionContext::execute_node(const PlanRef& plan, const std::set<size_t>* needed, bool shard) {
  if (verbose) printf("Logical plan: %s\n", plan->debug().c_str());
  GpuAggregateRelation::ResultStage stage;
  const LogicalPlan* agg = aggregate_under(*plan, &stage);
  if (agg || plan->kind == LogicalPlan::Aggregate) {  // context.rs:162-192 -> AggregateRelation
    // Aggregate{input: Selection{expr, input}} (what `SELECT .. WHERE .. GROUP BY ..` plans to,
    // sqlplanner.rs:93-96): the reference stacks FilterRelation under AggregateRelation; here the predicate is
    // handed to the aggregate's scan kernel and only the columns it, the keys and the arguments read are uploaded
    std::optional<GpuAggregateRelation::ResultStage> result_stage;
    if (agg) result_stage = stage;
    else agg = plan.get();
    ExprRef pred;
    PlanRef src = agg->input;
    if (src->kind == LogicalPlan::Selection) {
      pred = src->expr[0];
      src = src->input;
    }
    std::set<size_t> used;
    for (auto& e : agg->group_expr) collect_columns(*e, used);
    for (auto& e : agg->aggr_expr) collect_columns(*e, used);
    if (pred) collect_columns(*pred, used);
    RelationRef input_rel = execute_node(src, &used, shard);
    return std::make_shared<GpuAggregateRelation>(gpu_, plan->schema(), input_rel, agg->group_expr, agg->aggr_expr, pred, result_stage);
  }
  switch (plan->kind) {
    case LogicalPlan::TableScan: {
      auto it = datasources_->find(plan->table_name);
      if (it == datasources_->end()) fail(DFGPU_ERR_GENERAL, "No table registered as '" + plan->table_name + "'");
      auto sh = shared_.find(plan->table_name);
      RelationRef scan;
      if (sh != shared_.end()) scan = std::make_shared<SharedScanRelation>(sh->second);
      else scan = std::make_shared<DataSourceRelation>(it->second);
      if (world_ > 1 && shard) return std::make_shared<ShardRelation>(scan, rank_, world_);  // this rank's row range of every batch
      return scan;
    }
    case LogicalPlan::Join: {
      // Broadcast join across ranks: the probe (left) side keeps the sharding of its leftmost table, the build (right)
      // side is the whole table on every rank, so every output pair is produced by exactly one rank.  A semi / anti join
      // (a subquery: its plan is the build side) decides each probe row on exactly one rank; its schema is the left
      // schema, so it has no right columns.
      const size_t nl = plan->input->schema()->fields.size(), n = plan->schema()->fields.size();
      std::vector<size_t> lcols, rcols;
      for (size_t c = 0; c < n; c++)
        if (!needed || needed->count(c)) (c < nl ? lcols : rcols).push_back(c < nl ? c : c - nl);
      std::vector<ExprRef> lkeys, rkeys;
      std::set<size_t> lneed(lcols.begin(), lcols.end());
      for (auto& k : plan->on_keys) {
        lkeys.push_back(k.first);
        rkeys.push_back(shift_columns(k.second, nl));
        collect_columns(*k.first, lneed);
      }
      RelationRef l = execute_node(plan->input, &lneed, shard);
      RelationRef r = execute_node(plan->right, nullptr, false);
      auto j = std::make_shared<GpuHashJoinRelation>(gpu_, plan->schema(), l, r, lkeys, rkeys, lcols, rcols, plan->join_kind);
      joins_.push_back(j);
      return j;
    }
    case LogicalPlan::Selection: {  // context.rs:126-139 -> FilterRelation
      // FilterRelation alone passes every input column on, so every column is needed (nullptr): a Join below then
      // materialises all its columns and leaves no placeholder.  (The planner fuses a Selection into the Projection or
      // Aggregate above it, which prune instead.)
      RelationRef input_rel = execute_node(plan->input, nullptr, shard);
      return std::make_shared<GpuFilterProjectRelation>(gpu_, input_rel, plan->expr[0], std::vector<ExprRef>{}, input_rel->schema());
    }
    case LogicalPlan::Projection: {  // context.rs:140-161 -> ProjectRelation (fused with a Selection below it)
      ExprRef pred;
      PlanRef src = plan->input;
      if (src->kind == LogicalPlan::Selection) {
        pred = src->expr[0];
        src = src->input;
      }
      std::set<size_t> used;
      for (auto& e : plan->expr) collect_columns(*e, used);
      if (pred) collect_columns(*pred, used);
      RelationRef input_rel = execute_node(src, &used, shard);
      const Schema& in_schema = *input_rel->schema();
      auto schema = std::make_shared<Schema>();
      for (auto& e : plan->expr)  // projection.rs:52-57: (name, type, nullable = true)
        schema->fields.push_back(Field{runtime_expr_name(*e, in_schema), e->get_type(in_schema), true});
      return std::make_shared<GpuFilterProjectRelation>(gpu_, input_rel, pred, plan->expr, schema);
    }
    case LogicalPlan::Window: {
      // the window sees exactly what `SELECT <the columns it and the plan above read> FROM .. WHERE ..` returns: a
      // Selection under it runs as a filter / project of those columns
      ExprRef pred;
      PlanRef src = plan->input;
      if (src->kind == LogicalPlan::Selection) {
        pred = src->expr[0];
        src = src->input;
      }
      const size_t nin = src->schema()->fields.size();
      std::set<size_t> cols;
      for (size_t c = 0; c < nin; c++)
        if (!needed || needed->count(c)) cols.insert(c);
      for (auto& w : plan->window_expr) collect_columns(*w, cols);
      if (cols.empty() && nin > 0) cols.insert(0);  // the row count
      std::set<size_t> used = cols;
      if (pred) collect_columns(*pred, used);
      RelationRef input_rel = execute_node(src, &used, shard);
      std::vector<size_t> colv(cols.begin(), cols.end());
      if (pred) {
        auto schema = std::make_shared<Schema>();
        for (size_t c : colv) schema->fields.push_back(src->schema()->fields[c]);
        input_rel = std::make_shared<GpuFilterProjectRelation>(gpu_, input_rel, pred, column_exprs(colv), schema);
      }
      return std::make_shared<GpuWindowRelation>(gpu_, plan->schema(), input_rel, colv, pred != nullptr, plan->window_expr);
    }
    default:
      fail(DFGPU_ERR_NOT_IMPLEMENTED, "Limit / Sort / EmptyRelation plans are not executable (reference: unimplemented!() at context.rs:194)");
  }
}

}  // namespace dfhost
