// sqlplanner.cpp — see sqlplanner.h.  Rule-for-rule mirror of SqlToRel::sql_to_rel / sql_to_rex:
// literal typing (Long -> Int64, Double -> Float64), get_supertype + cast_to on both operands of
// every binary expression, aggregate detection by scanning the SELECT list, COUNT(1)/COUNT(*) ->
// COUNT(#0), output = group exprs ++ aggregate exprs.
#include "sqlplanner.h"

#include <algorithm>
#include <cctype>

namespace dfhost {

static std::string lower(std::string s) {
  for (auto& c : s) c = char(tolower((unsigned char)c));
  return s;
}

DataType convert_data_type(const ASTNode& n) {
  switch (n.sql_type) {
    case SQLType::Boolean: return DFGPU_BOOL;
    case SQLType::SmallInt: return DFGPU_INT16;
    case SQLType::Int: return DFGPU_INT32;
    case SQLType::BigInt: return DFGPU_INT64;
    case SQLType::Float: case SQLType::Real: case SQLType::Double: return DFGPU_FLOAT64;
    case SQLType::Char: case SQLType::Varchar: return DFGPU_UTF8;
    default: fail(DFGPU_ERR_NOT_IMPLEMENTED, "Unsupported SQL type " + n.id);
  }
}

Field expr_to_field(const Expr& e, const Schema& input_schema) {
  switch (e.kind) {
    case Expr::Column:
      if (e.index >= input_schema.fields.size()) fail(DFGPU_ERR_INVALID_COLUMN, "column index out of range");
      return input_schema.fields[e.index];
    case Expr::Literal: return Field{"lit", e.value.get_datatype(), true};
    case Expr::ScalarFunction: case Expr::AggregateFunction: case Expr::WindowFunction: return Field{e.name, e.data_type, true};
    case Expr::Cast: return Field{"cast", e.data_type, true};
    case Expr::Case: return Field{"case", e.get_type(input_schema), true};
    case Expr::BinaryExpr: {
      DataType st;
      if (!get_supertype(e.left->get_type(input_schema), e.right->get_type(input_schema), &st))
        fail(DFGPU_ERR_INTERNAL, "no common supertype (reference: unwrap() panic at sqlplanner.rs:422)");
      return Field{"binary_expr", st, true};
    }
    default: fail(DFGPU_ERR_NOT_IMPLEMENTED, "Cannot determine schema type for expression " + e.debug());
  }
}

std::vector<Field> exprlist_to_fields(const std::vector<ExprRef>& expr, const Schema& input_schema) {
  std::vector<Field> out;
  for (auto& e : expr) out.push_back(expr_to_field(*e, input_schema));
  return out;
}

namespace {
void refuse_windows(const ASTNode& select);
ExprRef over_window(const ExprRef& e, size_t ninput, std::vector<ExprRef>& calls);
}  // namespace

PlanRef SqlToRel::sql_to_rel(const ASTRef& sql) const {
  switch (sql->kind) {
    case ASTNode::SQLSelect: {
      refuse_windows(*sql);
      // parse the input relation so we have access to the row type
      PlanRef input;
      ExprRef residual;  // the ON terms of the joins that are not keys
      if (sql->relation) input = plan_from(*sql, &residual);
      else {
        auto e = std::make_shared<LogicalPlan>();
        e->kind = LogicalPlan::EmptyRelation;
        e->schema_ = std::make_shared<Schema>();
        input = e;
      }
      const SchemaRef input_schema = input->schema();  // semi / anti joins of the WHERE clause keep it

      // selection first
      PlanRef selection_plan;
      ExprRef where = sql->selection ? plan_where(sql->selection, *input_schema, &input) : nullptr;
      if (where || residual) {  // the join residual first, then the WHERE clause
        ExprRef pred = residual;
        if (where) pred = pred ? Expr::binary(pred, Operator::And, where) : where;
        auto s = std::make_shared<LogicalPlan>();
        s->kind = LogicalPlan::Selection;
        s->expr.push_back(pred);
        s->input = input;
        selection_plan = s;
      }

      std::vector<ExprRef> expr;
      for (auto& e : sql->projection) expr.push_back(sql_to_rex(e, *input_schema));

      // collect aggregate expressions
      std::vector<ExprRef> aggr_expr;
      for (auto& e : expr)
        if (e->kind == Expr::AggregateFunction) aggr_expr.push_back(e);
      const bool windowed = std::any_of(expr.begin(), expr.end(), [](const ExprRef& e) { return contains_window(*e); });
      if (windowed && (!aggr_expr.empty() || sql->has_group_by))
        fail(DFGPU_ERR_NOT_IMPLEMENTED, "window functions are not supported in an aggregate query");

      if (!aggr_expr.empty()) {
        PlanRef aggregate_input = selection_plan ? selection_plan : input;
        std::vector<ExprRef> group_expr;
        if (sql->has_group_by)
          for (auto& e : sql->group_by) group_expr.push_back(sql_to_rex(e, *input_schema));
        std::vector<ExprRef> all_fields = group_expr;
        for (auto& x : aggr_expr) all_fields.push_back(x);
        auto aggr_schema = std::make_shared<Schema>();
        aggr_schema->fields = exprlist_to_fields(all_fields, *input_schema);
        auto a = std::make_shared<LogicalPlan>();
        a->kind = LogicalPlan::Aggregate;
        a->input = aggregate_input;
        a->group_expr = group_expr;
        a->aggr_expr = aggr_expr;
        a->schema_ = aggr_schema;
        if (sql->having || sql->has_order_by || sql->limit) return plan_aggregate_result(*sql, a, expr, *input_schema);
        return a;
      }

      PlanRef projection_input = selection_plan ? selection_plan : input;
      const Schema* projection_input_schema = input_schema.get();
      if (windowed) {  // Projection <- Window <- [Selection] <- input: each window call becomes a column of the Window
        auto w = std::make_shared<LogicalPlan>();
        w->kind = LogicalPlan::Window;
        w->input = projection_input;
        for (auto& e : expr) e = over_window(e, input_schema->fields.size(), w->window_expr);
        w->schema_ = std::make_shared<Schema>(*input_schema);
        for (auto& x : w->window_expr) w->schema_->fields.push_back(expr_to_field(*x, *input_schema));
        projection_input = w;
        projection_input_schema = w->schema_.get();
      }
      auto projection_schema = std::make_shared<Schema>();
      projection_schema->fields = exprlist_to_fields(expr, *projection_input_schema);
      auto proj = std::make_shared<LogicalPlan>();
      proj->kind = LogicalPlan::Projection;
      proj->expr = expr;
      proj->input = projection_input;
      proj->schema_ = projection_schema;

      if (sql->having) fail(DFGPU_ERR_GENERAL, "HAVING is not implemented yet");

      PlanRef order_by_plan = proj;
      if (sql->has_order_by) {
        auto s = std::make_shared<LogicalPlan>();
        s->kind = LogicalPlan::Sort;
        for (auto& o : sql->order_by) s->expr.push_back(Expr::sort(sql_to_rex(o.expr, *proj->schema()), o.asc));
        s->input = proj;
        s->schema_ = proj->schema();
        order_by_plan = s;
      }
      if (sql->limit) {
        if (sql->limit->kind != ASTNode::SQLLong) fail(DFGPU_ERR_GENERAL, "LIMIT parameter is not a number");
        auto l = std::make_shared<LogicalPlan>();
        l->kind = LogicalPlan::Limit;
        l->limit = size_t(sql->limit->lval);
        l->schema_ = order_by_plan->schema();
        l->input = order_by_plan;
        return l;
      }
      return order_by_plan;
    }
    case ASTNode::SQLIdentifier: {
      SchemaRef schema = schema_provider_->get_table_meta(sql->id);
      if (!schema) fail(DFGPU_ERR_GENERAL, "no schema found for table " + sql->id);
      auto t = std::make_shared<LogicalPlan>();
      t->kind = LogicalPlan::TableScan;
      t->schema_name = "default";
      t->table_name = sql->id;
      auto qualified = std::make_shared<Schema>(*schema);  // each field knows its table, for `q.c`
      for (auto& f : qualified->fields) f.qualifier = sql->qualifier.empty() ? sql->id : sql->qualifier;
      t->schema_ = qualified;
      return t;
    }
    default: fail(DFGPU_ERR_EXECUTION, "sql_to_rel does not support this relation: " + sql->debug());
  }
}

namespace {
// 1: every column of `e` is below `split` (at least one); 2: every one at or above it; 0: otherwise
int side_of(const Expr& e, size_t split) {
  std::set<size_t> cols;
  collect_columns(e, cols);
  if (cols.empty()) return 0;
  bool l = false, r = false;
  for (size_t c : cols) (c < split ? l : r) = true;
  return l && r ? 0 : (l ? 1 : 2);
}
void ast_and_terms(const ASTRef& e, std::vector<ASTRef>& out) {
  if (e->kind == ASTNode::SQLBinaryExpr && e->op == SQLOperator::And) {
    ast_and_terms(e->left, out);
    ast_and_terms(e->right, out);
  } else {
    out.push_back(e);
  }
}
bool is_subquery_term(const ASTNode& e) { return e.kind == ASTNode::SQLInSubquery || e.kind == ASTNode::SQLExists; }
bool contains_aggregate(const ASTRef& e) {
  if (!e) return false;
  if (e->kind == ASTNode::SQLFunction) {
    const std::string l = lower(e->id);
    if (l == "min" || l == "max" || l == "sum" || l == "avg" || l == "count") return true;
  }
  for (auto& a : e->args)
    if (contains_aggregate(a)) return true;
  return contains_aggregate(e->left) || contains_aggregate(e->right);
}
void and_terms(const ExprRef& e, std::vector<ExprRef>& out) {
  if (e->kind == Expr::BinaryExpr && e->op == Operator::And) {
    and_terms(e->left, out);
    and_terms(e->right, out);
  } else {
    out.push_back(e);
  }
}
// Whether an AST holds a window call, subqueries included
bool ast_has_window(const ASTRef& e) {
  if (!e) return false;
  if (e->kind == ASTNode::SQLFunction && e->over) return true;
  for (auto* v : {&e->args, &e->partition_by, &e->projection, &e->group_by})
    for (auto& a : *v)
      if (ast_has_window(a)) return true;
  for (auto& o : e->window_order)
    if (ast_has_window(o.expr)) return true;
  for (auto& o : e->order_by)
    if (ast_has_window(o.expr)) return true;
  for (auto& j : e->joins)
    if (ast_has_window(j.on)) return true;
  return ast_has_window(e->left) || ast_has_window(e->right) || ast_has_window(e->subquery) || ast_has_window(e->selection) ||
         ast_has_window(e->having);
}
// A window call is allowed in the SELECT list of a non-aggregate query only
void refuse_windows(const ASTNode& select) {
  auto refuse = [](const char* where) { fail(DFGPU_ERR_GENERAL, std::string("window functions are not allowed in ") + where); };
  for (auto& j : select.joins)
    if (ast_has_window(j.on)) refuse("ON");
  if (select.selection) {
    std::vector<ASTRef> terms;
    ast_and_terms(select.selection, terms);
    for (auto& t : terms)
      if (is_subquery_term(*t) && ast_has_window(t->subquery)) refuse("an IN / EXISTS subquery");
    if (ast_has_window(select.selection)) refuse("WHERE");
  }
  for (auto& g : select.group_by)
    if (ast_has_window(g)) refuse("GROUP BY");
  if (ast_has_window(select.having)) refuse("HAVING");
}
// `e` over the Window's output: each window call becomes the column of the equal call (equal plan text) in `calls`,
// appended when there is none
ExprRef over_window(const ExprRef& e, size_t ninput, std::vector<ExprRef>& calls) {
  if (e->kind == Expr::WindowFunction) {
    const std::string d = e->debug();
    size_t i = 0;
    while (i < calls.size() && calls[i]->debug() != d) i++;
    if (i == calls.size()) calls.push_back(e);
    return Expr::column(ninput + i);
  }
  if (!contains_window(*e)) return e;
  auto c = std::make_shared<Expr>(*e);
  if (c->left) c->left = over_window(c->left, ninput, calls);
  if (c->right) c->right = over_window(c->right, ninput, calls);
  for (auto& a : c->args) a = over_window(a, ninput, calls);
  return c;
}
}  // namespace

namespace {
// `e` (over the aggregate's input) over the aggregate's output: a subtree equal to a GROUP BY expression (equal plan
// text) becomes that column, an aggregate call the column of the equal aggregate, appended to `aggr` (hidden) when
// there is none.  A column of the input left over is an error.
ExprRef over_aggregate(const ExprRef& e, const std::vector<ExprRef>& group, std::vector<ExprRef>& aggr, const Schema& input) {
  const std::string d = e->debug();
  for (size_t k = 0; k < group.size(); k++)
    if (group[k]->debug() == d) return Expr::column(k);
  if (e->kind == Expr::AggregateFunction) {
    size_t i = 0;
    while (i < aggr.size() && aggr[i]->debug() != d) i++;
    if (i == aggr.size()) aggr.push_back(e);
    return Expr::column(group.size() + i);
  }
  if (e->kind == Expr::Column)
    fail(DFGPU_ERR_GENERAL, "Column '" + input.fields[e->index].name + "' must appear in the GROUP BY clause or be used in an aggregate function");
  auto c = std::make_shared<Expr>(*e);
  if (c->left) c->left = over_aggregate(c->left, group, aggr, input);
  if (c->right) c->right = over_aggregate(c->right, group, aggr, input);
  for (auto& a : c->args) a = over_aggregate(a, group, aggr, input);
  return c;
}
}  // namespace

// Aggregate -> Selection (HAVING) -> Sort -> Limit -> Projection (only when HAVING or ORDER BY added hidden aggregates,
// to drop them).  HAVING and the ORDER BY keys are planned over the input like the SELECT list, then rewritten over the
// aggregate's output; an integer literal k in ORDER BY is the k-th SELECT-list item.
PlanRef SqlToRel::plan_aggregate_result(const ASTNode& select, std::shared_ptr<LogicalPlan> a, const std::vector<ExprRef>& select_exprs,
                                        const Schema& input_schema) const {
  const size_t visible = a->group_expr.size() + a->aggr_expr.size();
  std::vector<ExprRef> aggr = a->aggr_expr;
  ExprRef having;
  if (select.having) having = over_aggregate(sql_to_rex(select.having, input_schema), a->group_expr, aggr, input_schema);
  std::vector<ExprRef> sort;
  for (auto& o : select.order_by) {
    ExprRef e;
    if (o.expr->kind == ASTNode::SQLLong) {
      const long long k = o.expr->lval;
      if (k < 1 || size_t(k) > select_exprs.size()) fail(DFGPU_ERR_GENERAL, "ORDER BY position " + std::to_string(k) + " is not in select list");
      e = select_exprs[size_t(k - 1)];
    } else {
      e = sql_to_rex(o.expr, input_schema);
    }
    sort.push_back(Expr::sort(over_aggregate(e, a->group_expr, aggr, input_schema), o.asc));
  }
  std::vector<ExprRef> all_fields = a->group_expr;
  for (auto& x : aggr) all_fields.push_back(x);
  auto schema = std::make_shared<Schema>();
  schema->fields = exprlist_to_fields(all_fields, input_schema);
  a->aggr_expr = aggr;
  a->schema_ = schema;
  if (having && having->get_type(*schema) != DFGPU_BOOL) fail(DFGPU_ERR_GENERAL, "HAVING expression did not evaluate to boolean");
  for (auto& s : sort)
    if (s->get_type(*schema) == DFGPU_BOOL) fail(DFGPU_ERR_NOT_IMPLEMENTED, "ORDER BY a Boolean expression is not supported: " + s->left->debug());
  PlanRef plan = a;
  if (having) {
    auto s = std::make_shared<LogicalPlan>();
    s->kind = LogicalPlan::Selection;
    s->expr.push_back(having);
    s->input = plan;
    plan = s;
  }
  if (!sort.empty()) {
    auto s = std::make_shared<LogicalPlan>();
    s->kind = LogicalPlan::Sort;
    s->expr = sort;
    s->input = plan;
    s->schema_ = schema;
    plan = s;
  }
  if (select.limit) {
    if (select.limit->kind != ASTNode::SQLLong) fail(DFGPU_ERR_GENERAL, "LIMIT parameter is not a number");
    auto l = std::make_shared<LogicalPlan>();
    l->kind = LogicalPlan::Limit;
    l->limit = size_t(select.limit->lval);
    l->schema_ = schema;
    l->input = plan;
    plan = l;
  }
  if (aggr.size() + a->group_expr.size() > visible) {
    auto proj = std::make_shared<LogicalPlan>();
    proj->kind = LogicalPlan::Projection;
    for (size_t i = 0; i < visible; i++) proj->expr.push_back(Expr::column(i));
    proj->input = plan;
    proj->schema_ = std::make_shared<Schema>();
    proj->schema_->fields.assign(schema->fields.begin(), schema->fields.begin() + long(visible));
    plan = proj;
  }
  return plan;
}

// FROM table_ref { JOIN table_ref ON expr }: a left-deep chain of Join nodes.  Each ON clause is planned like a WHERE
// clause over the joined schema; its top-level AND terms `l Eq r` with l over the left input only and r over the right
// input only (or the reverse) are the keys, every other term is returned in *residual (AND-ed, in order) for the
// Selection above the joins.
PlanRef SqlToRel::plan_from(const ASTNode& select, ExprRef* residual) const {
  PlanRef plan = sql_to_rel(select.relation);
  std::vector<std::string> names{select.relation->qualifier.empty() ? select.relation->id : select.relation->qualifier};
  for (const JoinClause& jc : select.joins) {
    PlanRef right = sql_to_rel(jc.relation);
    const std::string q = jc.relation->qualifier.empty() ? jc.relation->id : jc.relation->qualifier;
    if (std::find(names.begin(), names.end(), q) != names.end())
      fail(DFGPU_ERR_GENERAL, "Table '" + q + "' appears more than once in FROM: give each occurrence an alias");
    names.push_back(q);
    auto schema = std::make_shared<Schema>(*plan->schema());
    const size_t split = schema->fields.size();
    for (auto& f : right->schema()->fields) schema->fields.push_back(f);
    ExprRef on = sql_to_rex(jc.on, *schema);
    if (on->get_type(*schema) != DFGPU_BOOL) fail(DFGPU_ERR_GENERAL, "JOIN ON expression did not evaluate to boolean");
    std::vector<ExprRef> terms;
    and_terms(on, terms);
    auto j = std::make_shared<LogicalPlan>();
    j->kind = LogicalPlan::Join;
    j->input = plan;
    j->right = right;
    j->schema_ = schema;
    for (auto& t : terms) {
      if (t->kind == Expr::BinaryExpr && t->op == Operator::Eq) {
        const int l = side_of(*t->left, split), r = side_of(*t->right, split);
        if (l == 1 && r == 2) { j->on_keys.emplace_back(t->left, t->right); continue; }
        if (l == 2 && r == 1) { j->on_keys.emplace_back(t->right, t->left); continue; }
      }
      *residual = *residual ? Expr::binary(*residual, Operator::And, t) : t;
    }
    if (j->on_keys.empty()) fail(DFGPU_ERR_NOT_IMPLEMENTED, "JOIN needs at least one equality between the two inputs");
    plan = j;
  }
  return plan;
}

// The WHERE clause of a SELECT over *input: each top-level AND term that is an IN / EXISTS subquery becomes a semi or
// anti join above *input, in order; the other terms are returned AND-ed, in order (null if there are none).
ExprRef SqlToRel::plan_where(const ASTRef& where, const Schema& schema, PlanRef* input) const {
  std::vector<ASTRef> terms;
  ast_and_terms(where, terms);
  if (std::none_of(terms.begin(), terms.end(), [](const ASTRef& t) { return is_subquery_term(*t); })) return sql_to_rex(where, schema);
  ExprRef pred;
  for (auto& t : terms) {
    if (is_subquery_term(*t)) {
      *input = plan_subquery(*t, *input, {});
      continue;
    }
    ExprRef e = sql_to_rex(t, schema);
    pred = pred ? Expr::binary(pred, Operator::And, e) : e;
  }
  return pred;
}

// `term` ([NOT] IN / [NOT] EXISTS) as a semi / anti join of `left` (the query's FROM plan) and the subquery.  The probe
// keys are the IN operand and the outer side of each correlated equality, the build keys the subquery's column and the
// inner sides; the subquery's other WHERE terms (over its own columns) and its ON residual are the build side's
// Selection, under the Projection of the build keys.
PlanRef SqlToRel::plan_subquery(const ASTNode& term, PlanRef left, const std::vector<SchemaRef>& far) const {
  const ASTNode& q = *term.subquery;
  const bool in = term.kind == ASTNode::SQLInSubquery;
  const std::string form = std::string(term.negated ? "NOT " : "") + (in ? "IN" : "EXISTS");
  if (q.has_group_by || q.having || q.has_order_by || q.limit)
    fail(DFGPU_ERR_NOT_IMPLEMENTED, "GROUP BY, HAVING, ORDER BY and LIMIT are not supported in an " + form + " subquery");
  for (auto& e : q.projection)
    if (contains_aggregate(e)) fail(DFGPU_ERR_NOT_IMPLEMENTED, "aggregates are not supported in an " + form + " subquery");
  if (!q.relation) fail(DFGPU_ERR_NOT_IMPLEMENTED, "an " + form + " subquery needs a FROM clause");
  if (in && q.projection.size() != 1) fail(DFGPU_ERR_GENERAL, "IN subquery must return exactly one column");
  ExprRef pred;
  PlanRef sub = plan_from(q, &pred);
  const SchemaRef sub_schema = sub->schema(), outer_schema = left->schema();
  const size_t ns = sub_schema->fields.size(), nl = outer_schema->fields.size();
  Schema both = *sub_schema;  // the subquery's fields, then the outer query's
  for (auto& f : outer_schema->fields) both.fields.push_back(f);
  const Scope scope{ns, far};
  std::vector<ExprRef> probe, build;
  if (in) {
    const Scope outer_scope{nl, far};
    ExprRef x = rex(term.left, *outer_schema, &outer_scope);
    ExprRef y = rex(q.projection[0], both, &scope);
    std::set<size_t> ycols;
    collect_columns(*y, ycols);
    if (!ycols.empty() && *ycols.rbegin() >= ns) fail(DFGPU_ERR_NOT_IMPLEMENTED, "the column of an IN subquery must be over the subquery's own tables");
    const DataType xt = x->get_type(*outer_schema), yt = y->get_type(*sub_schema);
    DataType st;
    if (!get_supertype(xt, yt, &st))
      fail(DFGPU_ERR_GENERAL, std::string("No common supertype found for binary operator Eq with input types ") + datatype_debug(xt) + " and " +
                                  datatype_debug(yt));
    probe.push_back(x->cast_to(st, *outer_schema));
    build.push_back(y->cast_to(st, *sub_schema));
  }
  if (q.selection) {
    std::vector<SchemaRef> far_in{outer_schema};  // a nested subquery's far scopes
    far_in.insert(far_in.end(), far.begin(), far.end());
    std::vector<ASTRef> terms;
    ast_and_terms(q.selection, terms);
    for (auto& t : terms) {
      if (is_subquery_term(*t)) {
        sub = plan_subquery(*t, sub, far_in);
        continue;
      }
      ExprRef e = rex(t, both, &scope);
      std::set<size_t> cols;
      collect_columns(*e, cols);
      if (cols.empty() || *cols.rbegin() < ns) {  // over the subquery's columns only
        pred = pred ? Expr::binary(pred, Operator::And, e) : e;
        continue;
      }
      if (*cols.begin() >= ns) fail(DFGPU_ERR_NOT_IMPLEMENTED, "a subquery WHERE term over outer columns only is not supported");
      if (e->kind == Expr::BinaryExpr && e->op == Operator::Eq) {
        const int l = side_of(*e->left, ns), r = side_of(*e->right, ns);
        if (l == 1 && r == 2) {
          build.push_back(e->left);
          probe.push_back(shift_columns(e->right, ns));
          continue;
        }
        if (l == 2 && r == 1) {
          build.push_back(e->right);
          probe.push_back(shift_columns(e->left, ns));
          continue;
        }
      }
      fail(DFGPU_ERR_NOT_IMPLEMENTED, "a correlated subquery term must be an equality between an inner and an outer expression");
    }
  }
  if (in && term.negated && probe.size() > 1) fail(DFGPU_ERR_NOT_IMPLEMENTED, "correlated NOT IN subqueries are not supported");
  if (!in && probe.empty()) fail(DFGPU_ERR_NOT_IMPLEMENTED, form + " subquery without a correlated equality is not supported");
  if (pred) {
    auto s = std::make_shared<LogicalPlan>();
    s->kind = LogicalPlan::Selection;
    s->expr.push_back(pred);
    s->input = sub;
    sub = s;
  }
  auto proj = std::make_shared<LogicalPlan>();
  proj->kind = LogicalPlan::Projection;
  proj->expr = build;
  proj->input = sub;
  proj->schema_ = std::make_shared<Schema>();
  proj->schema_->fields = exprlist_to_fields(build, *sub_schema);
  auto j = std::make_shared<LogicalPlan>();
  j->kind = LogicalPlan::Join;
  j->join_kind = !term.negated ? LogicalPlan::JoinKind::Semi : in ? LogicalPlan::JoinKind::AntiNullAware : LogicalPlan::JoinKind::Anti;
  j->input = left;
  j->right = proj;
  j->schema_ = outer_schema;
  for (size_t i = 0; i < probe.size(); i++) j->on_keys.emplace_back(probe[i], Expr::column(nl + i));
  return j;
}

ExprRef SqlToRel::sql_to_rex(const ASTRef& sql, const Schema& schema) const { return rex(sql, schema, nullptr); }

// l op r with both operands cast to their supertype (sqlplanner.rs:402-414)
ExprRef SqlToRel::coerced_binary(const ExprRef& l, Operator op, const ExprRef& r, const Schema& schema) {
  DataType lt = l->get_type(schema), rt = r->get_type(schema), st;
  if (!get_supertype(lt, rt, &st))
    fail(DFGPU_ERR_GENERAL, std::string("No common supertype found for binary operator ") + operator_debug(op) + " with input types " +
                                datatype_debug(lt) + " and " + datatype_debug(rt));
  return Expr::binary(l->cast_to(st, schema), op, r->cast_to(st, schema));
}

ExprRef SqlToRel::rex(const ASTRef& sql, const Schema& schema, const Scope* scope) const {
  switch (sql->kind) {
    case ASTNode::SQLLong: return Expr::literal(ScalarValue::Int64(sql->lval));
    case ASTNode::SQLDouble: return Expr::literal(ScalarValue::Float64(sql->dval));
    case ASTNode::SQLString: return Expr::literal(ScalarValue::Utf8(sql->id));
    case ASTNode::SQLIdentifier: {
      // `q.c`: the field of that table (or alias) and name.  `c`: the first field of that name, unless fields of that
      // name come from more than one table.  In a subquery the fields of its own tables are searched first.
      auto find = [&](const Schema& sch, size_t lo, size_t hi) {
        long long found = -1;
        for (size_t i = lo; i < hi; i++) {
          const Field& f = sch.fields[i];
          if (f.name != sql->id || (!sql->qualifier.empty() && f.qualifier != sql->qualifier)) continue;
          if (found < 0) found = (long long)i;
          else if (sch.fields[size_t(found)].qualifier != f.qualifier)
            fail(DFGPU_ERR_GENERAL, "Ambiguous reference to column '" + sql->id + "'");
        }
        return found;
      };
      const size_t n = schema.fields.size(), inner = scope ? std::min(scope->inner, n) : n;
      long long found = find(schema, 0, inner);
      if (found < 0 && inner < n) found = find(schema, inner, n);
      if (found >= 0) return Expr::column(size_t(found));
      if (scope)
        for (auto& s : scope->far)
          if (find(*s, 0, s->fields.size()) >= 0)
            fail(DFGPU_ERR_NOT_IMPLEMENTED, "a subquery may only reference the query just outside it, not '" + sql->id +
                                                "' of a query further out (correlation that skips a level)");
      fail(DFGPU_ERR_EXECUTION, "Invalid identifier '" + (sql->qualifier.empty() ? "" : sql->qualifier + ".") + sql->id + "' for schema " +
                                    schema.to_string());
    }
    case ASTNode::SQLInSubquery:
    case ASTNode::SQLExists:
      fail(DFGPU_ERR_NOT_IMPLEMENTED, "IN / EXISTS subqueries are supported only as AND terms of WHERE");
    case ASTNode::SQLWildcard:
      fail(DFGPU_ERR_NOT_IMPLEMENTED, "SQL wildcard operator is not supported in projection - please use explicit column names");
    case ASTNode::SQLCast: return Expr::cast(rex(sql->left, schema, scope), convert_data_type(*sql));
    case ASTNode::SQLIsNull: return Expr::is_null(rex(sql->left, schema, scope), false);
    case ASTNode::SQLIsNotNull: return Expr::is_null(rex(sql->left, schema, scope), true);
    case ASTNode::SQLBinaryExpr: {
      Operator op;
      switch (sql->op) {
        case SQLOperator::Gt: op = Operator::Gt; break;
        case SQLOperator::GtEq: op = Operator::GtEq; break;
        case SQLOperator::Lt: op = Operator::Lt; break;
        case SQLOperator::LtEq: op = Operator::LtEq; break;
        case SQLOperator::Eq: op = Operator::Eq; break;
        case SQLOperator::NotEq: op = Operator::NotEq; break;
        case SQLOperator::Plus: op = Operator::Plus; break;
        case SQLOperator::Minus: op = Operator::Minus; break;
        case SQLOperator::Multiply: op = Operator::Multiply; break;
        case SQLOperator::Divide: op = Operator::Divide; break;
        case SQLOperator::Modulus: op = Operator::Modulus; break;
        case SQLOperator::And: op = Operator::And; break;
        case SQLOperator::Or: op = Operator::Or; break;
        case SQLOperator::Not: op = Operator::Not; break;
        case SQLOperator::Like: op = Operator::Like; break;
        default: op = Operator::NotLike; break;
      }
      return coerced_binary(rex(sql->left, schema, scope), op, rex(sql->right, schema, scope), schema);
    }
    case ASTNode::SQLCase: {
      // the simple form CASE x WHEN a THEN .. is the searched form with conditions x Eq a; the THEN / ELSE values are cast
      // to their supertype, as the operands of a binary operator are
      ExprRef x = sql->left ? rex(sql->left, schema, scope) : nullptr;
      std::vector<ExprRef> args;
      for (size_t i = 0; i < sql->args.size(); i++) {
        ExprRef a = rex(sql->args[i], schema, scope);
        args.push_back(x && i % 2 == 0 ? coerced_binary(x, Operator::Eq, a, schema) : a);
      }
      if (sql->right) args.push_back(rex(sql->right, schema, scope));
      std::vector<size_t> vals;  // the THEN values, then the ELSE
      for (size_t i = 1; i < args.size(); i += 2) vals.push_back(i);
      if (args.size() % 2) vals.push_back(args.size() - 1);
      DataType st = args[1]->get_type(schema);
      for (size_t k : vals) {
        const DataType t = args[k]->get_type(schema), prev = st;
        if (!get_supertype(prev, t, &st))
          fail(DFGPU_ERR_GENERAL, std::string("No common supertype found for CASE with input types ") + datatype_debug(prev) + " and " +
                                      datatype_debug(t));
      }
      for (size_t k : vals) args[k] = args[k]->cast_to(st, schema);
      return Expr::case_when(std::move(args));
    }
    case ASTNode::SQLFunction: {
      const std::string lid = lower(sql->id);
      if (sql->over) {
        std::vector<ExprRef> args, part, order;
        DataType rt = DFGPU_UINT64;
        if (lid == "row_number" || lid == "rank" || lid == "dense_rank") {
          if (!sql->args.empty()) fail(DFGPU_ERR_GENERAL, sql->id + "() takes no arguments");
        } else if (lid == "min" || lid == "max" || lid == "sum" || lid == "avg" || lid == "count") {
          if (sql->distinct) fail(DFGPU_ERR_NOT_IMPLEMENTED, "COUNT(DISTINCT x) OVER (..) is not supported");
          if (sql->args.size() != 1) fail(DFGPU_ERR_GENERAL, sql->id + "() OVER (..) takes exactly one argument");
          const ASTRef& a = sql->args[0];
          // COUNT(1) / COUNT(*) -> COUNT(first_column), as for the aggregate
          if (lid == "count" && ((a->kind == ASTNode::SQLLong && a->lval == 1) || a->kind == ASTNode::SQLWildcard)) args.push_back(Expr::column(0));
          else args.push_back(rex(a, schema, scope));
          rt = lid == "count" ? DFGPU_UINT64 : lid == "avg" ? DFGPU_FLOAT64 : args[0]->get_type(schema);
        } else {
          fail(DFGPU_ERR_GENERAL, "Invalid function '" + sql->id + "'");
        }
        for (auto& p : sql->partition_by) part.push_back(rex(p, schema, scope));
        for (auto& o : sql->window_order) order.push_back(Expr::sort(rex(o.expr, schema, scope), o.asc));
        for (auto* v : {&args, &part, &order})
          for (auto& x : *v)
            if (contains_window(*x)) fail(DFGPU_ERR_GENERAL, "window functions cannot be nested");
        for (auto* v : {&part, &order})
          for (auto& x : *v)
            if (x->get_type(schema) == DFGPU_BOOL)
              fail(DFGPU_ERR_NOT_IMPLEMENTED, std::string(v == &part ? "PARTITION BY" : "ORDER BY") + " a Boolean key is not supported");
        return Expr::window(sql->id, args, part, order, rt);
      }
      for (auto& a : sql->args)
        if ((lid == "min" || lid == "max" || lid == "sum" || lid == "avg" || lid == "count") && ast_has_window(a))
          fail(DFGPU_ERR_GENERAL, "window functions are not allowed in an aggregate argument");
      if (lid == "min" || lid == "max" || lid == "sum" || lid == "avg") {
        std::vector<ExprRef> rex_args;
        for (auto& a : sql->args) rex_args.push_back(rex(a, schema, scope));
        if (rex_args.empty()) fail(DFGPU_ERR_INTERNAL, "aggregate function without arguments (reference: index panic at sqlplanner.rs:320)");
        // return type is same as the argument type for MIN / MAX / SUM; AVG is Float64 (the reference types it as
        // its argument too, but never executes it)
        if (lid == "avg") return Expr::aggregate(sql->id, rex_args, DFGPU_FLOAT64);
        return Expr::aggregate(sql->id, rex_args, rex_args[0]->get_type(schema));
      }
      if (lid == "count" && sql->distinct) {
        std::vector<ExprRef> rex_args;
        for (auto& a : sql->args) rex_args.push_back(rex(a, schema, scope));
        if (rex_args.size() != 1) fail(DFGPU_ERR_GENERAL, "COUNT(DISTINCT) takes exactly one argument");
        return Expr::aggregate(sql->id, rex_args, DFGPU_UINT64, true);
      }
      if (lid == "count") {
        std::vector<ExprRef> rex_args;
        for (auto& a : sql->args) {
          // COUNT(1) / COUNT(*) -> COUNT(first_column)
          if ((a->kind == ASTNode::SQLLong && a->lval == 1) || a->kind == ASTNode::SQLWildcard) rex_args.push_back(Expr::column(0));
          else rex_args.push_back(rex(a, schema, scope));
        }
        return Expr::aggregate(sql->id, rex_args, DFGPU_UINT64);
      }
      auto fm = schema_provider_->get_function_meta(sql->id);
      if (!fm) fail(DFGPU_ERR_GENERAL, "Invalid function '" + sql->id + "'");
      std::vector<ExprRef> safe_args;
      for (size_t i = 0; i < sql->args.size(); i++) {
        ExprRef a = rex(sql->args[i], schema, scope);
        if (i >= fm->args.size()) fail(DFGPU_ERR_INTERNAL, "too many function arguments (reference: index panic at sqlplanner.rs:356)");
        safe_args.push_back(a->cast_to(fm->args[i].data_type, schema));
      }
      return Expr::scalar_fn(sql->id, safe_args, fm->return_type);
    }
    default: fail(DFGPU_ERR_GENERAL, "Unsupported ast node " + sql->debug() + " in sqltorel");
  }
}

}  // namespace dfhost
