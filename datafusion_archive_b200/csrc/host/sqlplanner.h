// sqlplanner.h — SQL AST -> LogicalPlan, mirroring SqlToRel (src/sqlplanner.rs:28-375).
#pragma once
#include <functional>

#include "logicalplan.h"
#include "sqlparser.h"

namespace dfhost {

struct FunctionMeta {  // src/logicalplan.rs:30-64
  std::string name;
  std::vector<Field> args;
  DataType return_type = 0;
};

struct SchemaProvider {  // trait SchemaProvider, src/sqlplanner.rs:28-31
  virtual ~SchemaProvider() {}
  virtual SchemaRef get_table_meta(const std::string& name) const = 0;
  virtual std::shared_ptr<FunctionMeta> get_function_meta(const std::string& name) const = 0;
};

class SqlToRel {
 public:
  explicit SqlToRel(std::shared_ptr<SchemaProvider> sp) : schema_provider_(std::move(sp)) {}
  PlanRef sql_to_rel(const ASTRef& sql) const;                     // sqlplanner.rs:46-209
  ExprRef sql_to_rex(const ASTRef& sql, const Schema& schema) const;  // sqlplanner.rs:212-375
 private:
  PlanRef plan_from(const ASTNode& select, ExprRef* residual) const;  // FROM with joins (no reference counterpart)
  // IN / EXISTS subqueries (no reference counterpart).  A subquery's expressions are planned over its own fields
  // followed by the fields of the query just outside it: `inner` is the number of its own, and a name resolves in the
  // innermost scope that has it.  `far` are the schemas of the queries further out, which it may not reference.
  struct Scope {
    size_t inner;
    std::vector<SchemaRef> far;
  };
  ExprRef rex(const ASTRef& sql, const Schema& schema, const Scope* scope) const;
  static ExprRef coerced_binary(const ExprRef& l, Operator op, const ExprRef& r, const Schema& schema);
  ExprRef plan_where(const ASTRef& where, const Schema& schema, PlanRef* input) const;
  PlanRef plan_subquery(const ASTNode& term, PlanRef left, const std::vector<SchemaRef>& far) const;
  // HAVING, ORDER BY and LIMIT of an aggregate query over its Aggregate (no reference counterpart: sqlplanner.rs:112)
  PlanRef plan_aggregate_result(const ASTNode& select, std::shared_ptr<LogicalPlan> aggregate, const std::vector<ExprRef>& select_exprs,
                                const Schema& input_schema) const;
  std::shared_ptr<SchemaProvider> schema_provider_;
};

DataType convert_data_type(const ASTNode& cast_node);              // sqlplanner.rs:379-394
Field expr_to_field(const Expr& e, const Schema& input_schema);    // sqlplanner.rs:396-428
std::vector<Field> exprlist_to_fields(const std::vector<ExprRef>& expr, const Schema& input_schema);

}  // namespace dfhost
