// expr_compile.cu — host half of the expression VM: type-check a postfix program the way
// compile_scalar_expr would (src/execution/expression.rs:283-505), fold right-hand leaves into the
// consuming instruction, and emit the device bytecode of expr_vm.cuh.
#include <climits>
#include <memory>

#include "expr_vm.cuh"

namespace dfgpu {

MType mtype_of(int dt) {
  switch (dt) {
    case DFGPU_FLOAT64: return MT_F64;
    case DFGPU_FLOAT32: return MT_F32;
    case DFGPU_BOOL: return MT_BOOL;
    case DFGPU_INT8: case DFGPU_INT16: case DFGPU_INT32: case DFGPU_INT64: return MT_I;
    case DFGPU_UINT8: case DFGPU_UINT16: case DFGPU_UINT32: case DFGPU_UINT64: return MT_U;
  }
  return MT_NONE;
}

namespace {

struct Node {
  enum Kind { COL, LIT, CAST, BIN, FN, UFN, CASE } kind = COL;
  int col = 0;               // COL: batch column, or -1 - k for synthetic column k (a recognised Utf8 predicate or
                             // function); kViewCol for a Utf8 view that no program reads
  int view = -1;             // COL of a Utf8 view: its index
  int dtype = 0;             // result dtype
  unsigned long long imm = 0;  // LIT payload, widened to the machine representation; UFN: start
  long long count = 0;       // UFN: count
  int op = 0;                // DFGPU_OP_* for BIN, DFGPU_FN_* for FN, DFGPU_UTF8FN_* for UFN
  std::string str;           // LIT of dtype Utf8: the bytes
  std::unique_ptr<Node> l, r;  // FN: the arguments (r: second argument of a two-argument function, else null); UFN: l
  std::vector<std::unique_ptr<Node>> args;  // CASE: c1 v1 .. cn vn [e]
};
constexpr int kViewCol = INT_MIN;

bool is_utf8_lit(const Node* nd) { return nd->kind == Node::LIT && nd->dtype == DFGPU_UTF8; }

// A Utf8 literal is an operand of a Utf8 comparison or LIKE only; anywhere else it keeps the reference's error
// (expression.rs:306-309), spelled like ScalarValue's Debug
void refuse_utf8_literal(const Node* nd) {
  if (!nd || !is_utf8_lit(nd)) return;
  std::string d = "Utf8(\"";
  for (char ch : nd->str) {
    if (ch == '"' || ch == '\\') d += '\\';
    d += ch;
  }
  fail(DFGPU_ERR_EXECUTION, "No support for literal type " + d + "\")");
}

const char* op_debug_name(int op) {
  switch (op) {
    case DFGPU_OP_ADD: return "Plus"; case DFGPU_OP_SUB: return "Minus"; case DFGPU_OP_MUL: return "Multiply";
    case DFGPU_OP_DIV: return "Divide"; case DFGPU_OP_EQ: return "Eq"; case DFGPU_OP_NE: return "NotEq";
    case DFGPU_OP_LT: return "Lt"; case DFGPU_OP_LE: return "LtEq"; case DFGPU_OP_GT: return "Gt";
    case DFGPU_OP_GE: return "GtEq"; case DFGPU_OP_AND: return "And"; case DFGPU_OP_OR: return "Or";
  }
  return "?";
}

unsigned long long widen_literal(const dfgpu_insn& in) {
  switch (in.dtype) {
    case DFGPU_FLOAT64: case DFGPU_INT64: case DFGPU_UINT64: return in.lit.u64;
    case DFGPU_FLOAT32: { uint32_t b; memcpy(&b, &in.lit.f32, 4); return b; }
    case DFGPU_INT32: return (unsigned long long)(long long)(int32_t)in.lit.i64;
    case DFGPU_INT16: return (unsigned long long)(long long)(int16_t)in.lit.i64;
    case DFGPU_INT8: return (unsigned long long)(long long)(int8_t)in.lit.i64;
    case DFGPU_UINT32: return in.lit.u64 & 0xffffffffull;
    case DFGPU_UINT16: return in.lit.u64 & 0xffffull;
    case DFGPU_UINT8: return in.lit.u64 & 0xffull;
  }
  return 0;
}

// DFGPU_FN_* code -> name, nullptr for an unknown code; arity of a known code
const char* fn_name(int code) {
  static const char* const names[] = {nullptr, "sqrt", "abs", "floor", "ceil", "trunc", "round", "signum", "exp", "ln", "log2",
                                      "log10", "sin", "cos", "tan", "asin", "acos", "atan", "power", "atan2"};
  return code >= 1 && code <= DFGPU_FN_ATAN2 ? names[code] : nullptr;
}
int fn_arity(int code) { return code == DFGPU_FN_POWER || code == DFGPU_FN_ATAN2 ? 2 : 1; }

// DFGPU_UTF8FN_* code -> SQL name, nullptr for an unknown code; the number of Int64 literal arguments after the string
const char* utf8_fn_name(int code) {
  static const char* const names[] = {nullptr, "upper", "lower", "trim", "ltrim", "rtrim", "substr", "substr", "length", "octet_length"};
  return code >= 1 && code <= DFGPU_UTF8FN_OCTET_LENGTH ? names[code] : nullptr;
}
int utf8_fn_nlits(int code) { return code == DFGPU_UTF8FN_SUBSTR ? 2 : code == DFGPU_UTF8FN_SUBSTR_FROM ? 1 : 0; }

VOp vop_of(int op) {
  switch (op) {
    case DFGPU_OP_ADD: return V_ADD; case DFGPU_OP_SUB: return V_SUB; case DFGPU_OP_MUL: return V_MUL;
    case DFGPU_OP_DIV: return V_DIV; case DFGPU_OP_EQ: return V_EQ; case DFGPU_OP_NE: return V_NE;
    case DFGPU_OP_LT: return V_LT; case DFGPU_OP_LE: return V_LE; case DFGPU_OP_GT: return V_GT;
    case DFGPU_OP_GE: return V_GE; case DFGPU_OP_AND: return V_AND; default: return V_OR;
  }
}

// COL op COL | COL op LIT over 4- or 8-byte numeric operands (the type check gave both sides one dtype), else kind 0.
// Called after lowering: every column already has its slot.
Leaf leaf_of(ProgramBuilder* pb, const Node* nd) {
  Leaf f;
  memset(&f, 0, sizeof(f));
  if (nd->kind != Node::BIN || nd->l->kind != Node::COL || (nd->r->kind != Node::COL && nd->r->kind != Node::LIT)) return f;
  const int dt = nd->l->dtype;
  if (!is_numeric4or8(dt) || nd->r->dtype != dt) return f;
  const bool rcol = nd->r->kind == Node::COL;
  f.kind = rcol ? 2 : 3;
  f.op = vop_of(nd->op);
  f.a = pb->slot_of_column(nd->l->col);
  f.b = rcol ? pb->slot_of_column(nd->r->col) : 0;
  f.dtype = dt;
  f.mtype = mtype_of(dt);
  f.imm = rcol ? 0 : nd->r->imm;
  return f;
}

// Appends the comparison leaves of a left-deep AND / OR chain to *c; false when `nd` is not one of at most 4 terms.
bool chain_of(ProgramBuilder* pb, const Node* nd, LeafChain* c) {
  const Node* leaf = nd;
  int conn = 0;
  if (nd->kind == Node::BIN && (nd->op == DFGPU_OP_AND || nd->op == DFGPU_OP_OR)) {
    if (!chain_of(pb, nd->l.get(), c)) return false;
    leaf = nd->r.get();
    conn = nd->op == DFGPU_OP_OR ? 1 : 0;
  }
  const Leaf t = leaf_of(pb, leaf);
  if (c->nterms == 4 || !t.kind || t.op < V_EQ || t.op > V_GE) return false;
  c->term[c->nterms] = t;
  c->term[c->nterms++].conn = uint8_t(conn);
  return true;
}

}  // namespace

int ProgramBuilder::slot_of_column(int col) {
  for (size_t i = 0; i < slots_.size(); i++)
    if (slots_[i] == col) return int(i);
  if (int(slots_.size()) >= kMaxCols)
    fail(DFGPU_ERR_NOT_IMPLEMENTED, "expression set references more than " + std::to_string(kMaxCols) + " distinct columns");
  slots_.push_back(col);
  return int(slots_.size()) - 1;
}

int ProgramBuilder::add(const dfgpu_insn* p, int n, const char* what, int* utf8_view) {
  if (utf8_view) *utf8_view = -1;
  if (n <= 0 || !p) fail(DFGPU_ERR_GENERAL, std::string("empty expression program for ") + what);
  // A maximal nest of Utf8 functions becomes one Utf8View when something other than a Utf8 function consumes it: an
  // Int64 result is a synthetic column, a Utf8 one a COL node naming the view (read by Utf8 predicates only)
  auto lower_view = [&](std::unique_ptr<Node>& x) {
    if (!x || x->kind != Node::UFN) return;
    std::vector<const Node*> nest;  // outermost first
    const Node* q = x.get();
    for (; q->kind == Node::UFN; q = q->l.get()) nest.push_back(q);
    Utf8View v;
    memset(&v.spec, 0, sizeof(v.spec));
    v.src = q->col;
    v.synth = -1;
    v.projection = false;
    for (auto it = nest.rbegin(); it != nest.rend(); ++it) {
      const int code = (*it)->op;
      if (code == DFGPU_UTF8FN_UPPER || code == DFGPU_UTF8FN_LOWER) {
        v.spec.case_map = code;  // the outermost one wins
      } else if (code == DFGPU_UTF8FN_LENGTH || code == DFGPU_UTF8FN_OCTET_LENGTH) {
        v.spec.result = code;  // Int64: always the outermost function
      } else {
        if (v.spec.nsteps == kMaxUtf8Steps)
          fail(DFGPU_ERR_NOT_IMPLEMENTED, "more than " + std::to_string(kMaxUtf8Steps) + " nested trim / substr calls");
        Utf8Step& s = v.spec.step[v.spec.nsteps++];
        s.op = code == DFGPU_UTF8FN_SUBSTR_FROM ? DFGPU_UTF8FN_SUBSTR : code;
        s.start = (long long)(*it)->imm;
        s.count = code == DFGPU_UTF8FN_SUBSTR_FROM ? -1 : (*it)->count;
      }
    }
    const int dtype = x->dtype;
    utf8_views_.push_back(v);
    x = std::make_unique<Node>();
    x->kind = Node::COL;
    x->dtype = dtype;
    x->view = int(utf8_views_.size()) - 1;
    if (dtype == DFGPU_INT64) {
      utf8_views_.back().synth = new_synth(nullptr, DFGPU_INT64, v.src);
      x->col = -1 - utf8_views_.back().synth;
    } else {
      x->col = kViewCol;
    }
  };
  // 1. postfix -> tree, with the reference's type rules
  std::vector<std::unique_ptr<Node>> st;
  for (int i = 0; i < n; i++) {
    auto nd = std::make_unique<Node>();
    const dfgpu_insn& in = p[i];
    switch (in.op) {
      case DFGPU_OP_COL: {  // Expr::Column (expression.rs:311-315)
        if (in.col < 0 || size_t(in.col) >= batch_->cols.size())
          fail(DFGPU_ERR_INVALID_COLUMN, "column index " + std::to_string(in.col) + " out of range");
        nd->kind = Node::COL;
        nd->col = in.col;
        nd->dtype = batch_->cols[size_t(in.col)].dtype;
        break;
      }
      case DFGPU_OP_LIT: {  // Expr::Literal (expression.rs:289-310)
        if (!is_numeric(in.dtype))
          fail(DFGPU_ERR_EXECUTION, std::string("No support for literal type ") + dtype_name(in.dtype));
        nd->kind = Node::LIT;
        nd->dtype = in.dtype;
        nd->imm = widen_literal(in);
        break;
      }
      case DFGPU_OP_LIT_UTF8: {  // Expr::Literal(ScalarValue::Utf8): the bytes are copied, the program's are borrowed
        if (in.dtype != DFGPU_UTF8 || in.col < 0 || (!in.lit.str && in.col > 0)) fail(DFGPU_ERR_GENERAL, "malformed expression program");
        if (in.col > DFGPU_UTF8_LITERAL_MAX)
          fail(DFGPU_ERR_NOT_IMPLEMENTED, "Utf8 literal of " + std::to_string(in.col) + " bytes (at most " + std::to_string(DFGPU_UTF8_LITERAL_MAX) + ")");
        nd->kind = Node::LIT;
        nd->dtype = DFGPU_UTF8;
        nd->str.assign(in.lit.str ? in.lit.str : "", size_t(in.col));
        break;
      }
      case DFGPU_OP_CAST: {  // Expr::Cast (expression.rs:316-378)
        if (st.empty()) fail(DFGPU_ERR_GENERAL, "malformed expression program");
        auto inner = std::move(st.back());
        st.pop_back();
        lower_view(inner);
        refuse_utf8_literal(inner.get());
        if (inner->kind == Node::LIT) {
          // only Literal Int64 -> Float64 exists in the reference (expression.rs:345-373)
          if (inner->dtype != DFGPU_INT64)
            fail(DFGPU_ERR_NOT_IMPLEMENTED, std::string("CAST from ") + dtype_name(inner->dtype) + " to " + dtype_name(in.dtype));
          if (in.dtype != DFGPU_FLOAT64)
            fail(DFGPU_ERR_NOT_IMPLEMENTED, std::string("CAST from Int64 to ") + dtype_name(in.dtype));
          double d = double((long long)inner->imm);
          nd->kind = Node::LIT;
          nd->dtype = DFGPU_FLOAT64;
          memcpy(&nd->imm, &d, 8);
        } else if (inner->kind == Node::COL) {
          // The reference casts columns to Int16/Int32 only and panics otherwise
          // (cast_column_outer!, expression.rs:272-280).  Any numeric -> numeric cast is done here
          // (needed for the planner's own CAST(#i AS Int64) output, sqlplanner.rs:581); the result
          // type reported is the TARGET type (the reference reports the source: expression.rs:324).
          if (!is_numeric(inner->dtype) || !is_numeric(in.dtype))
            fail(DFGPU_ERR_NOT_IMPLEMENTED, std::string("CAST column from ") + dtype_name(inner->dtype) + " to " + dtype_name(in.dtype));
          nd->kind = Node::CAST;
          nd->dtype = in.dtype;
          nd->l = std::move(inner);
        } else {
          fail(DFGPU_ERR_GENERAL, "CAST not implemented for expression");  // expression.rs:374-377
        }
        break;
      }
      case DFGPU_OP_FN: {  // Expr::ScalarFunction (logicalplan.rs:156-160), which the reference plans but never executes
        const char* name = fn_name(in.col);
        if (!name) fail(DFGPU_ERR_EXECUTION, "unknown scalar function code " + std::to_string(in.col));
        const int arity = fn_arity(in.col);
        if (int(st.size()) < arity)
          fail(DFGPU_ERR_EXECUTION, std::string("function '") + name + "' takes " + std::to_string(arity) + (arity == 1 ? " argument" : " arguments"));
        nd->kind = Node::FN;
        nd->op = in.col;
        nd->dtype = DFGPU_FLOAT64;
        if (arity == 2) {
          nd->r = std::move(st.back());
          st.pop_back();
        }
        nd->l = std::move(st.back());
        st.pop_back();
        lower_view(nd->l);
        lower_view(nd->r);
        refuse_utf8_literal(nd->l.get());
        refuse_utf8_literal(nd->r.get());
        // monomorphic over Float64: the caller casts, as the planner does (sqlplanner.rs:343-365)
        for (const Node* a : {nd->l.get(), nd->r.get()})
          if (a && a->dtype != DFGPU_FLOAT64)
            fail(DFGPU_ERR_EXECUTION, std::string("function '") + name + "' takes Float64 arguments, not " + dtype_name(a->dtype));
        break;
      }
      case DFGPU_OP_UTF8_FN: {  // Expr::ScalarFunction of a Utf8 function (see "Utf8 functions" in dfgpu.h)
        const char* name = utf8_fn_name(in.col);
        if (!name) fail(DFGPU_ERR_EXECUTION, "unknown Utf8 function code " + std::to_string(in.col));
        const int nlits = utf8_fn_nlits(in.col);
        const bool is_len = in.col == DFGPU_UTF8FN_LENGTH || in.col == DFGPU_UTF8FN_OCTET_LENGTH;
        if (in.dtype != (is_len ? DFGPU_INT64 : DFGPU_UTF8)) fail(DFGPU_ERR_GENERAL, "malformed expression program");
        if (int(st.size()) < 1 + nlits)
          fail(DFGPU_ERR_EXECUTION, std::string("function '") + name + "' takes " + std::to_string(1 + nlits) + (nlits ? " arguments" : " argument"));
        long long arg[2] = {0, 0};
        for (int k = nlits - 1; k >= 0; k--) {
          const auto& a = st.back();
          if (a->kind != Node::LIT || a->dtype != DFGPU_INT64)
            fail(DFGPU_ERR_NOT_IMPLEMENTED, std::string("function '") + name + "': start and count must be Int64 literals");
          arg[k] = (long long)a->imm;
          st.pop_back();
        }
        nd->kind = Node::UFN;
        nd->op = in.col;
        nd->dtype = in.dtype;
        nd->l = std::move(st.back());
        st.pop_back();
        if (is_utf8_lit(nd->l.get())) fail(DFGPU_ERR_NOT_IMPLEMENTED, std::string("function '") + name + "' over a Utf8 literal");
        if (nd->l->dtype != DFGPU_UTF8 || (nd->l->kind != Node::COL && nd->l->kind != Node::UFN))
          fail(DFGPU_ERR_EXECUTION, std::string("function '") + name + "' takes a Utf8 argument, not " + dtype_name(nd->l->dtype));
        if (nlits == 2 && arg[1] < 0) fail(DFGPU_ERR_EXECUTION, "negative substring length not allowed");
        nd->imm = (unsigned long long)arg[0];
        nd->count = arg[1];
        break;
      }
      case DFGPU_OP_CASE: {  // CASE WHEN c1 THEN v1 .. [ELSE e] END: `col` operands c1 v1 .. cn vn [e], `dtype` the result type
        if (in.col < 2 || in.col > int(st.size())) fail(DFGPU_ERR_GENERAL, "malformed expression program");
        nd->kind = Node::CASE;
        for (auto it = st.end() - in.col; it != st.end(); ++it) nd->args.push_back(std::move(*it));
        st.resize(st.size() - size_t(in.col));
        int rt = 0;
        for (size_t k = 0; k < nd->args.size(); k++) {
          lower_view(nd->args[k]);
          const Node* a = nd->args[k].get();
          if (k % 2 == 0 && k + 1 < nd->args.size()) {
            if (a->dtype != DFGPU_BOOL) fail(DFGPU_ERR_EXECUTION, "CASE WHEN condition did not evaluate to boolean");
            continue;
          }
          if (a->dtype == DFGPU_UTF8) fail(DFGPU_ERR_NOT_IMPLEMENTED, "CASE with a Utf8 result");
          if (rt && a->dtype != rt)
            fail(DFGPU_ERR_EXECUTION, std::string("CASE branch types differ: ") + dtype_name(rt) + " and " + dtype_name(a->dtype));
          rt = a->dtype;
        }
        if (in.dtype != rt) fail(DFGPU_ERR_GENERAL, "malformed expression program");
        nd->dtype = rt;
        break;
      }
      default: {
        int op = in.op;
        bool is_math = op >= DFGPU_OP_ADD && op <= DFGPU_OP_DIV;
        bool is_cmp = op >= DFGPU_OP_EQ && op <= DFGPU_OP_GE;
        bool is_bool = op == DFGPU_OP_AND || op == DFGPU_OP_OR;
        const bool is_like = op == DFGPU_OP_LIKE || op == DFGPU_OP_NOT_LIKE;
        if (!is_math && !is_cmp && !is_bool && !is_like) fail(DFGPU_ERR_EXECUTION, "operator: " + std::to_string(op));
        if (st.size() < 2) fail(DFGPU_ERR_GENERAL, "malformed expression program");
        nd->kind = Node::BIN;
        nd->op = op;
        nd->r = std::move(st.back());
        st.pop_back();
        nd->l = std::move(st.back());
        st.pop_back();
        lower_view(nd->l);
        lower_view(nd->r);
        int lt = nd->l->dtype, rt = nd->r->dtype;
        if (!is_cmp && !is_like) {
          refuse_utf8_literal(nd->l.get());
          refuse_utf8_literal(nd->r.get());
        }
        // A maximal Utf8 comparison or LIKE (Utf8 operands are columns or literals: nothing else yields Utf8) becomes a
        // Boolean synthetic column, filled by eval_utf8_predicates before the scan
        if (is_like || (is_cmp && lt == DFGPU_UTF8 && rt == DFGPU_UTF8)) {
          const char* name = op == DFGPU_OP_LIKE ? "Like" : op == DFGPU_OP_NOT_LIKE ? "NotLike" : op_debug_name(op);
          if (lt != DFGPU_UTF8 || rt != DFGPU_UTF8)
            fail(DFGPU_ERR_EXECUTION, std::string(name) + ": operands must be Utf8, not " + dtype_name(lt) + " and " + dtype_name(rt));
          const bool llit = nd->l->kind == Node::LIT, rlit = nd->r->kind == Node::LIT;
          if (llit && rlit) fail(DFGPU_ERR_NOT_IMPLEMENTED, std::string(name) + " between two Utf8 literals");
          if (is_like && !rlit) fail(DFGPU_ERR_NOT_IMPLEMENTED, std::string(name) + " with a pattern that is not a literal");
          Utf8Pred sp;
          sp.op = op;
          if (llit) {  // 'lit' op x  ==  x op' 'lit'
            sp.op = op == DFGPU_OP_LT ? DFGPU_OP_GT : op == DFGPU_OP_LE ? DFGPU_OP_GE : op == DFGPU_OP_GT ? DFGPU_OP_LT : op == DFGPU_OP_GE ? DFGPU_OP_LE : op;
            std::swap(nd->l, nd->r);
          }
          auto ref = [](const Node* x) { return x->view >= 0 ? -2 - x->view : x->col; };
          sp.a = ref(nd->l.get());
          sp.b = nd->r->kind == Node::COL ? ref(nd->r.get()) : -1;
          if (sp.b < 0) sp.lit = nd->r->str;
          sp.synth = new_synth(nullptr, DFGPU_BOOL);
          utf8_preds_.push_back(std::move(sp));
          nd = std::make_unique<Node>();
          nd->kind = Node::COL;
          nd->col = -1 - utf8_preds_.back().synth;
          nd->dtype = DFGPU_BOOL;
          break;
        }
        if (is_bool) {
          if (lt != DFGPU_BOOL || rt != DFGPU_BOOL)
            fail(DFGPU_ERR_INTERNAL, "boolean_ops: operand is not a BooleanArray (the reference panics here: expression.rs:217-221)");
          nd->dtype = DFGPU_BOOL;
        } else {
          if (lt != rt || !is_numeric(lt)) fail(DFGPU_ERR_EXECUTION, is_cmp ? "comparison_ops" : "math_ops");
          nd->dtype = is_cmp ? DFGPU_BOOL : lt;
        }
        break;
      }
    }
    st.push_back(std::move(nd));
  }
  if (st.size() != 1) fail(DFGPU_ERR_GENERAL, "malformed expression program");
  refuse_utf8_literal(st[0].get());
  lower_view(st[0]);
  if (st[0]->kind == Node::COL && st[0]->col == kViewCol) {  // the program's value is a Utf8 function nest
    Utf8View& v = utf8_views_[size_t(st[0]->view)];
    if (utf8_view) {
      v.projection = true;
      *utf8_view = st[0]->view;
      return -1;
    }
    v.synth = new_synth(nullptr, DFGPU_UTF8, v.src);  // typed as Utf8; every operator refuses a Utf8 program value
    st[0]->col = -1 - v.synth;
  }

  // 2. tree -> bytecode with right-hand leaf folding; track the live register-stack depth
  CompiledProgram cp;
  {
    // can the result be null?  (columns with nulls propagate through arithmetic / And / Or / Cast;
    // comparisons never produce nulls)
    struct N {
      const dfgpu_batch* b;
      const ProgramBuilder* pb;
      bool go(const Node* nd) const {
        switch (nd->kind) {
          case Node::COL:
            if (nd->col == kViewCol) return false;  // read by a Utf8 predicate only, whose result is never null
            return nd->col >= 0 ? b->cols[size_t(nd->col)].null_count > 0 : pb->synth_nullable(-1 - nd->col);
          case Node::LIT: return false;
          case Node::CAST: return go(nd->l.get());
          case Node::FN: return go(nd->l.get()) || (nd->r && go(nd->r.get()));  // like arithmetic
          case Node::CASE: {  // the chosen branch's validity; null when no WHEN is taken and there is no ELSE
            const size_t n = nd->args.size();
            if (n % 2 == 0) return true;
            for (size_t k = 1; k < n; k += 2)
              if (go(nd->args[k].get())) return true;
            return go(nd->args[n - 1].get());
          }
          default: {
            const bool cmp = nd->op >= DFGPU_OP_EQ && nd->op <= DFGPU_OP_GE;
            return !cmp && (go(nd->l.get()) || go(nd->r.get()));
          }
        }
      }
    } nn{batch_, this};
    cp.nullable = nn.go(st[0].get());
  }
  int depth = 0;
  struct Emit {
    ProgramBuilder* pb;
    CompiledProgram* cp;
    int* depth;
    void bump(int d) {
      *depth += d;
      if (*depth > cp->max_depth) cp->max_depth = *depth;
    }
    void go(const Node* nd) {
      DevInsn di;
      memset(&di, 0, sizeof(di));
      switch (nd->kind) {
        case Node::COL:
          di.op = V_PUSH_COL;
          di.slot = int16_t(pb->slot_of_column(nd->col));
          di.dtype = uint8_t(nd->dtype);
          di.mtype = mtype_of(nd->dtype);
          cp->code.push_back(di);
          bump(1);
          break;
        case Node::LIT:
          di.op = V_PUSH_IMM;
          di.imm = nd->imm;
          di.dtype = uint8_t(nd->dtype);
          di.mtype = mtype_of(nd->dtype);
          cp->code.push_back(di);
          bump(1);
          break;
        case Node::CAST:
          go(nd->l.get());
          di.op = V_CAST;
          di.dtype = uint8_t(nd->dtype);
          di.aux = int16_t(nd->l->dtype);
          di.mtype = mtype_of(nd->l->dtype);
          cp->code.push_back(di);
          break;
        case Node::CASE: {
          // a fold backward from the ELSE: e, then cn vn SEL, .., c1 v1 SEL, so that the stack holds at most the fold, one
          // condition and the operand being evaluated, whatever the number of WHENs.  Without ELSE the last WHEN is SEL0.
          const size_t n = nd->args.size();
          const bool has_else = n % 2 == 1;
          if (has_else) go(nd->args[n - 1].get());
          for (size_t k = (n & ~size_t(1)); k >= 2; k -= 2) {
            go(nd->args[k - 2].get());
            go(nd->args[k - 1].get());
            const bool sel0 = !has_else && k == (n & ~size_t(1));
            di.op = sel0 ? V_SEL0 : V_SEL;
            di.dtype = uint8_t(nd->dtype);
            di.mtype = mtype_of(nd->dtype);
            cp->code.push_back(di);
            bump(sel0 ? -1 : -2);
          }
          break;
        }
        case Node::FN:
          if (!nd->r) {  // one argument: applied to the accumulator, like CAST
            go(nd->l.get());
            di.op = V_FN;
            di.dtype = DFGPU_FLOAT64;
            di.mtype = MT_F64;
            di.aux = int16_t(nd->op);
            cp->code.push_back(di);
            break;
          }
          [[fallthrough]];
        case Node::BIN:
          go(nd->l.get());
          if (nd->kind == Node::FN) {
            di.op = V_FN2;
            di.aux = int16_t(nd->op);
          } else {
            di.op = vop_of(nd->op);
          }
          di.dtype = uint8_t(nd->l->dtype);
          di.mtype = mtype_of(nd->l->dtype);
          if (nd->r->kind == Node::LIT) {
            di.mode = RHS_IMM;
            di.imm = nd->r->imm;
          } else if (nd->r->kind == Node::COL) {
            di.mode = RHS_COL;
            di.slot = int16_t(pb->slot_of_column(nd->r->col));
          } else {
            go(nd->r.get());
            di.mode = RHS_STACK;
            // The evaluator keeps the TOP of the stack (here: the right operand) in its accumulator and
            // pops the operand below it as the second input, so a stack-mode instruction is emitted with
            // its operands exchanged: reverse subtract / divide / function, mirrored comparisons.
            switch (di.op) {
              case V_SUB: di.op = V_RSUB; break;
              case V_DIV: di.op = V_RDIV; break;
              case V_FN2: di.op = V_RFN2; break;
              case V_LT: di.op = V_GT; break;
              case V_LE: di.op = V_GE; break;
              case V_GT: di.op = V_LT; break;
              case V_GE: di.op = V_LE; break;
              default: break;
            }
            bump(-1);
          }
          cp->code.push_back(di);
          break;
      }
    }
  } em{this, &cp, &depth};
  em.go(st[0].get());
  cp.out_dtype = st[0]->dtype;
  for (const DevInsn& di : cp.code) cp.makes_nulls = cp.makes_nulls || (cp.nullable && di.op == V_SEL0);

  // 3. interpreter-free shapes
  const Node* root = st[0].get();
  if (root->kind == Node::COL) {
    cp.leaf.kind = 1;
    cp.leaf.a = cp.code[0].slot;
    cp.leaf.dtype = root->dtype;
    cp.leaf.mtype = mtype_of(root->dtype);
  } else {
    const Leaf f = leaf_of(this, root);
    const bool arith = f.op >= V_ADD && f.op <= V_DIV;
    if (f.kind && arith && (is_float(f.dtype) || (is_numeric8(f.dtype) && f.op != V_DIV))) cp.leaf = f;
  }
  if (!chain_of(this, root, &cp.chain)) cp.chain = LeafChain{};
  progs_.push_back(std::move(cp));
  return int(progs_.size()) - 1;
}

int ProgramBuilder::add_rowid() {
  CompiledProgram cp;
  DevInsn di;
  memset(&di, 0, sizeof(di));
  di.op = V_PUSH_ROWID;
  di.dtype = DFGPU_UINT64;
  di.mtype = MT_U;
  cp.code.push_back(di);
  cp.out_dtype = DFGPU_UINT64;
  cp.max_depth = 1;
  progs_.push_back(std::move(cp));
  return int(progs_.size()) - 1;
}

int ProgramBuilder::add_rowid_plus(unsigned long long bias) {
  CompiledProgram cp;
  DevInsn di;
  memset(&di, 0, sizeof(di));
  di.op = V_PUSH_ROWID;
  di.dtype = DFGPU_UINT64;
  di.mtype = MT_U;
  cp.code.push_back(di);
  memset(&di, 0, sizeof(di));
  di.op = V_ADD;
  di.mode = RHS_IMM;
  di.dtype = DFGPU_UINT64;
  di.mtype = MT_U;
  di.imm = bias;
  cp.code.push_back(di);
  cp.out_dtype = DFGPU_UINT64;
  cp.max_depth = 1;
  progs_.push_back(std::move(cp));
  return int(progs_.size()) - 1;
}

int ProgramBuilder::new_synth(const void* dptr, int dtype, int src) {
  if (int(slots_.size()) >= kMaxCols) fail(DFGPU_ERR_NOT_IMPLEMENTED, "too many distinct columns");
  synth_.push_back(Synth{dptr, dtype, src});
  slots_.push_back(-int(synth_.size()));  // -1 - k
  return int(synth_.size()) - 1;
}

// A Utf8 predicate's bitmap is never null; a Utf8 function's result is null where its source column is
bool ProgramBuilder::synth_nullable(int k) const {
  const int src = synth_[size_t(k)].src;
  return src >= 0 && batch_->cols[size_t(src)].null_count > 0;
}

int ProgramBuilder::add_synthetic_column(const void* dptr, int dtype) {
  new_synth(dptr, dtype);
  CompiledProgram cp;
  DevInsn di;
  memset(&di, 0, sizeof(di));
  di.op = V_PUSH_COL;
  di.slot = int16_t(slots_.size() - 1);
  di.dtype = uint8_t(dtype);
  di.mtype = mtype_of(dtype);
  cp.code.push_back(di);
  cp.out_dtype = dtype;
  cp.max_depth = 1;
  progs_.push_back(std::move(cp));
  return int(progs_.size()) - 1;
}

void ProgramBuilder::finish(ProgramSet* out) const {
  memset(out, 0, sizeof(*out));
  if ((!utf8_preds_.empty() || !utf8_views_.empty()) && !utf8_evaluated_ && batch_->ctx)
    fail(DFGPU_ERR_INTERNAL, "Utf8 predicates not evaluated before the scan");
  if (int(progs_.size()) > kMaxProgs)
    fail(DFGPU_ERR_NOT_IMPLEMENTED, "more than " + std::to_string(kMaxProgs) + " expressions in one operator");
  int pc = 0, maxd = 1;
  for (size_t i = 0; i < progs_.size(); i++) {
    out->start[i] = uint8_t(pc);
    if (pc + int(progs_[i].code.size()) > kMaxInsn)
      fail(DFGPU_ERR_NOT_IMPLEMENTED, "expression programs exceed " + std::to_string(kMaxInsn) + " instructions");
    for (const auto& di : progs_[i].code) out->insn[pc++] = di;
    out->out_dtype[i] = uint8_t(progs_[i].out_dtype);
    out->nullable[i] = progs_[i].nullable ? 1 : 0;
    if (progs_[i].makes_nulls) out->has_nulls = 1;  // a CASE without ELSE can make a null from any input
    if (progs_[i].max_depth > maxd) maxd = progs_[i].max_depth;
  }
  out->f64_only = 1;
  for (int i = 0; i < pc; i++) {
    const DevInsn& di = out->insn[i];
    if (di.op == V_CAST || !(di.mtype == MT_F64 || di.mtype == MT_BOOL)) out->f64_only = 0;
  }
  out->start[progs_.size()] = uint8_t(pc);
  out->nprog = int(progs_.size());
  out->ncols = int(slots_.size());
  out->max_depth = maxd;
  for (size_t s = 0; s < slots_.size(); s++) {
    if (slots_[s] < 0) {
      const int k = -1 - slots_[s];
      const Synth& sy = synth_[size_t(k)];
      out->cols[s].ptr = sy.ptr;
      out->cols[s].validity = synth_nullable(k) ? batch_->cols[size_t(sy.src)].validity : nullptr;
      if (out->cols[s].validity) out->has_nulls = 1;
      out->cols[s].dtype = sy.dtype;
      continue;
    }
    const DevColumn& c = batch_->cols[size_t(slots_[s])];
    out->cols[s].ptr = c.values;
    out->cols[s].validity = c.null_count > 0 ? c.validity : nullptr;
    if (c.null_count > 0) out->has_nulls = 1;
    out->cols[s].dtype = c.dtype;
  }
}

}  // namespace dfgpu
