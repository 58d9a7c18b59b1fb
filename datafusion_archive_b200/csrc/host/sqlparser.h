// sqlparser.h — SQL subset front-end.  The reference delegates parsing to crate sqlparser 0.2.1
// (Cargo.toml:34, wrapped by src/dfparser.rs:74); that crate is not in the reference repository, so this
// is a restatement of the grammar subset the planner consumes (src/sqlplanner.rs:46-375): one
// SELECT [list] [FROM ident] [WHERE e] [GROUP BY e,..] [HAVING e] [ORDER BY e [ASC|DESC],..] [LIMIT n].  Beyond it, FROM
// takes inner joins (the reference has none; its ROADMAP.md 0.7.0 plans them):
//   from      := table_ref { [INNER] JOIN table_ref ON expr }
//   table_ref := name [ [AS] alias ]
//   column    := name | qualifier '.' name        -- qualifier = the alias if given, else the table name
// and WHERE takes subqueries (planned as semi / anti joins, only as top-level AND terms):
//   expr [NOT] IN ( select )  |  [NOT] EXISTS ( select )
// and a function call takes a window (no reserved word is added: OVER is read only right after a call's closing
// parenthesis when `(` follows, PARTITION BY only inside that parenthesis):
//   name ( args ) OVER ( [PARTITION BY expr, ..] [ORDER BY expr [ASC|DESC], ..] )
#pragma once
#include <memory>
#include <string>
#include <vector>

namespace dfhost {

enum class SQLOperator { Plus, Minus, Multiply, Divide, Modulus, Gt, Lt, GtEq, LtEq, Eq, NotEq, And, Or, Not, Like, NotLike };
enum class SQLType { Boolean, SmallInt, Int, BigInt, Float, Real, Double, Char, Varchar, Other };

struct ASTNode;
using ASTRef = std::shared_ptr<ASTNode>;
struct OrderByExpr { ASTRef expr; bool asc = true; };
struct JoinClause { ASTRef relation; ASTRef on; };  // INNER JOIN relation ON on

struct ASTNode {
  enum Kind { SQLIdentifier, SQLWildcard, SQLLong, SQLDouble, SQLString, SQLBinaryExpr, SQLCast, SQLIsNull, SQLIsNotNull, SQLFunction, SQLSelect,
              SQLInSubquery, SQLExists, SQLCase } kind = SQLIdentifier;
  std::string id;       // identifier / function name / string literal / unknown type name
  std::string qualifier;  // SQLIdentifier: `q` of a column `q.c`; of a table after FROM / JOIN: its alias, or empty
  long long lval = 0;   // SQLLong
  double dval = 0;      // SQLDouble
  ASTRef left, right;   // binary; `left` = operand of cast / is-null
  // SQLCase: `left` = the operand of the simple form CASE x WHEN .. (else null), `args` = WHEN / THEN pairs, `right` = ELSE
  // (or null)
  SQLOperator op = SQLOperator::Eq;
  SQLType sql_type = SQLType::Other;
  std::vector<ASTRef> args;
  bool distinct = false;  // SQLFunction: COUNT(DISTINCT expr)
  // SQLFunction with a window: f(..) OVER (PARTITION BY `partition_by` ORDER BY `window_order`)
  bool over = false;
  std::vector<ASTRef> partition_by;
  std::vector<OrderByExpr> window_order;
  // SQLInSubquery: `left` [NOT] IN (`subquery`); SQLExists: [NOT] EXISTS (`subquery`)
  ASTRef subquery;
  bool negated = false;
  // SQLSelect
  std::vector<ASTRef> projection;
  ASTRef relation, selection, having, limit;
  bool has_group_by = false, has_order_by = false;
  std::vector<ASTRef> group_by;
  std::vector<OrderByExpr> order_by;
  std::vector<JoinClause> joins;  // after `relation`, left-deep
  std::string debug() const;
};

// Throws ExecutionError{DFGPU_ERR_GENERAL (ParserError), ...} on malformed input.
ASTRef parse_sql(const std::string& sql);

}  // namespace dfhost
