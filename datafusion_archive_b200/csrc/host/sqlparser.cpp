// sqlparser.cpp — tokenizer + precedence-climbing parser (see sqlparser.h).
#include "sqlparser.h"

#include <cctype>
#include <cerrno>
#include <cstdlib>

#include "logicalplan.h"

namespace dfhost {
namespace {

struct Token {
  enum Kind { End, Ident, Number, String, Sym } kind = End;
  std::string text;
};

std::string upper(std::string s) {
  for (auto& c : s) c = char(toupper((unsigned char)c));
  return s;
}

[[noreturn]] void perr(const std::string& m) { fail(DFGPU_ERR_GENERAL, "ParserError(\"" + m + "\")"); }

std::vector<Token> tokenize(const std::string& s) {
  std::vector<Token> out;
  size_t i = 0;
  while (i < s.size()) {
    char c = s[i];
    if (isspace((unsigned char)c)) { i++; continue; }
    Token t;
    if (isalpha((unsigned char)c) || c == '_') {
      size_t j = i;
      while (j < s.size() && (isalnum((unsigned char)s[j]) || s[j] == '_')) j++;
      t.kind = Token::Ident; t.text = s.substr(i, j - i); i = j;
    } else if (isdigit((unsigned char)c)) {
      size_t j = i;
      while (j < s.size() && (isdigit((unsigned char)s[j]) || s[j] == '.')) j++;
      t.kind = Token::Number; t.text = s.substr(i, j - i); i = j;
    } else if (c == '\'') {
      size_t j = i + 1;
      std::string v;
      while (j < s.size() && s[j] != '\'') v += s[j++];
      if (j >= s.size()) perr("Unterminated string literal");
      t.kind = Token::String; t.text = v; i = j + 1;
    } else if (c == '"') {  // delimited identifier
      size_t j = i + 1;
      std::string v;
      while (j < s.size() && s[j] != '"') v += s[j++];
      if (j >= s.size()) perr("Unterminated identifier");
      t.kind = Token::Ident; t.text = v; i = j + 1;
    } else {
      t.kind = Token::Sym;
      if ((c == '<' && i + 1 < s.size() && (s[i + 1] == '=' || s[i + 1] == '>')) || (c == '>' && i + 1 < s.size() && s[i + 1] == '=') ||
          (c == '!' && i + 1 < s.size() && s[i + 1] == '=')) {
        t.text = s.substr(i, 2); i += 2;
      } else if (c == '.' && !out.empty() && out.back().kind == Token::Ident && i + 1 < s.size() &&
                 (isalpha((unsigned char)s[i + 1]) || s[i + 1] == '_' || s[i + 1] == '"')) {  // qualifier.name
        t.text = "."; i++;
      } else if (std::string("=<>+-*/%(),;").find(c) != std::string::npos) {
        t.text = std::string(1, c); i++;
      } else {
        perr(std::string("Unexpected character '") + c + "'");
      }
    }
    out.push_back(t);
  }
  out.push_back(Token{});
  return out;
}

struct Parser {
  std::vector<Token> toks;
  size_t pos = 0;
  const Token& peek() const { return toks[pos]; }
  Token next() { return toks[pos == toks.size() - 1 ? pos : pos++]; }
  bool is_kw(const char* kw) const { return peek().kind == Token::Ident && upper(peek().text) == kw; }
  bool accept_kw(const char* kw) { if (is_kw(kw)) { pos++; return true; } return false; }
  bool accept_sym(const char* s) { if (peek().kind == Token::Sym && peek().text == s) { pos++; return true; } return false; }
  void expect_sym(const char* s) { if (!accept_sym(s)) perr(std::string("Expected ") + s + ", found: " + peek().text); }
  void expect_kw(const char* s) { if (!accept_kw(s)) perr(std::string("Expected ") + s + ", found: " + peek().text); }

  static bool reserved(const std::string& u) {
    static const char* kws[] = {"SELECT", "FROM", "WHERE", "GROUP", "BY", "HAVING", "ORDER", "LIMIT", "AND", "OR", "NOT", "AS", "ASC", "DESC", "IS", "NULL", "LIKE", "CAST",
                                 // joins: reserved so that `FROM a LEFT JOIN b` cannot read LEFT as an alias of a
                                 "JOIN", "INNER", "ON", "LEFT", "RIGHT", "FULL", "OUTER", "CROSS", "NATURAL", "USING",
                                 "CASE", "WHEN", "THEN", "ELSE", "END"};
    for (auto k : kws) if (u == k) return true;
    return false;
  }

  int next_precedence() const {
    const Token& t = peek();
    if (t.kind == Token::Ident) {
      std::string u = upper(t.text);
      if (u == "OR") return 5;
      if (u == "AND") return 10;
      if (u == "NOT") return 15;
      if (u == "IS") return 17;
      if (u == "LIKE" || u == "IN") return 20;
      return 0;
    }
    if (t.kind == Token::Sym) {
      const std::string& s = t.text;
      if (s == "=" || s == "<" || s == "<=" || s == ">" || s == ">=" || s == "!=" || s == "<>") return 20;
      if (s == "+" || s == "-") return 30;
      if (s == "*" || s == "/" || s == "%") return 40;
    }
    return 0;
  }

  // The parser, the planner and the plan printer recurse over the expression tree: bound its depth and
  // size so that hostile input ends in a ParserError instead of a stack overflow (the reference's
  // recursive-descent parser would abort the process).
  static constexpr int kMaxExprDepth = 400, kMaxExprNodes = 4000;
  int depth_ = 0, nodes_ = 0;

  ASTRef parse_expr(int precedence = 0) {
    struct Depth {
      int& d;
      explicit Depth(int& x) : d(x) { ++d; }
      ~Depth() { --d; }
    } guard(depth_);
    if (depth_ > kMaxExprDepth) perr("expression nested too deeply");
    ASTRef expr = parse_prefix();
    for (;;) {
      int np = next_precedence();
      if (precedence >= np) break;
      if (++nodes_ > kMaxExprNodes) perr("expression too large");
      expr = parse_infix(expr, np);
    }
    return expr;
  }

  SQLType parse_type(std::string* name) {
    Token t = next();
    if (t.kind != Token::Ident) perr("Expected a data type name");
    std::string u = upper(t.text);
    *name = u;
    SQLType ty = SQLType::Other;
    if (u == "BOOLEAN") ty = SQLType::Boolean;
    else if (u == "SMALLINT") ty = SQLType::SmallInt;
    else if (u == "INT" || u == "INTEGER") ty = SQLType::Int;
    else if (u == "BIGINT") ty = SQLType::BigInt;
    else if (u == "FLOAT") ty = SQLType::Float;
    else if (u == "REAL") ty = SQLType::Real;
    else if (u == "DOUBLE") ty = SQLType::Double;
    else if (u == "CHAR") ty = SQLType::Char;
    else if (u == "VARCHAR") ty = SQLType::Varchar;
    if (accept_sym("(")) {  // precision / length
      while (!accept_sym(")")) { if (peek().kind == Token::End) perr("Expected )"); next(); }
    }
    return ty;
  }

  ASTRef parse_prefix() {
    Token t = next();
    auto n = std::make_shared<ASTNode>();
    switch (t.kind) {
      case Token::Number:
        if (t.text.find('.') != std::string::npos) { n->kind = ASTNode::SQLDouble; n->dval = strtod(t.text.c_str(), nullptr); }
        else {
          // digits beyond i64 are refused, not saturated: `-9223372036854775808` is the prefix `-` applied to
          // 9223372036854775808, which does not fit, so INT64_MIN is written `-9223372036854775807 - 1`
          errno = 0;
          n->kind = ASTNode::SQLLong;
          n->lval = strtoll(t.text.c_str(), nullptr, 10);
          if (errno == ERANGE) perr("Could not parse '" + t.text + "' as i64: number too large to fit in target type");
        }
        return n;
      case Token::String: n->kind = ASTNode::SQLString; n->id = t.text; return n;
      case Token::Sym:
        if (t.text == "*") { n->kind = ASTNode::SQLWildcard; return n; }
        if (t.text == "(") { ASTRef e = parse_expr(); expect_sym(")"); return e; }
        if (t.text == "-" && peek().kind == Token::Number) {  // negative literal
          ASTRef v = parse_prefix();
          v->lval = -v->lval; v->dval = -v->dval;
          return v;
        }
        perr("Prefix parser expected a keyword but found " + t.text);
      case Token::Ident: {
        std::string u = upper(t.text);
        if (u == "SELECT") { pos--; return parse_select(); }
        // EXISTS (SELECT ..) and NOT EXISTS (SELECT ..); EXISTS followed by anything else is an identifier or function
        const bool not_exists = u == "NOT" && is_kw("EXISTS") && subquery_at(pos + 1);
        if (not_exists || (u == "EXISTS" && subquery_at(pos))) {
          if (not_exists) pos++;
          n->kind = ASTNode::SQLExists;
          n->negated = not_exists;
          n->subquery = parse_subquery();
          return n;
        }
        if (u == "CASE") {  // CASE [x] WHEN c THEN v [WHEN ..] [ELSE e] END
          n->kind = ASTNode::SQLCase;
          if (!is_kw("WHEN") && !is_kw("END")) n->left = parse_expr();
          while (accept_kw("WHEN")) {
            n->args.push_back(parse_expr());
            expect_kw("THEN");
            n->args.push_back(parse_expr());
          }
          if (n->args.empty()) perr("Expected WHEN after CASE, found: " + peek().text);
          if (accept_kw("ELSE")) n->right = parse_expr();
          expect_kw("END");
          return n;
        }
        if (u == "WHEN" || u == "THEN" || u == "ELSE" || u == "END") perr("Expected an expression, found: " + t.text);
        if (u == "CAST") {
          expect_sym("(");
          n->kind = ASTNode::SQLCast;
          n->left = parse_expr();
          expect_kw("AS");
          n->sql_type = parse_type(&n->id);
          expect_sym(")");
          return n;
        }
        if (accept_sym("(")) {  // function call
          n->kind = ASTNode::SQLFunction;
          n->id = t.text;
          // COUNT(DISTINCT expr); a column named "distinct" still reads as COUNT(distinct)
          if (is_kw("DISTINCT") && !(toks[pos + 1].kind == Token::Sym && toks[pos + 1].text == ")")) {
            pos++;
            if (upper(t.text) != "COUNT") perr("DISTINCT is only supported in COUNT(DISTINCT expr), not in " + t.text + "()");
            if (peek().kind == Token::Sym && peek().text == "*") perr("COUNT(DISTINCT *) is not supported");
            n->distinct = true;
          }
          if (!accept_sym(")")) {
            do { n->args.push_back(parse_expr()); } while (accept_sym(","));
            expect_sym(")");
          }
          if (is_kw("OVER") && toks[pos + 1].kind == Token::Sym && toks[pos + 1].text == "(") parse_window(*n);
          else if (is_kw("OVER") && toks[pos + 1].kind == Token::Ident) perr("named windows are not supported: write OVER (..)");
          return n;
        }
        n->kind = ASTNode::SQLIdentifier;
        n->id = t.text;
        if (accept_sym(".")) {  // qualifier.name
          Token c = next();
          if (c.kind != Token::Ident) perr("Expected a column name after " + t.text + ".");
          n->qualifier = t.text;
          n->id = c.text;
        }
        return n;
      }
      default: perr("Unexpected end of input");
    }
  }

  ASTRef parse_infix(ASTRef left, int precedence) {
    Token t = next();
    auto n = std::make_shared<ASTNode>();
    if (t.kind == Token::Ident) {
      std::string u = upper(t.text);
      if (u == "IS") {
        bool neg = accept_kw("NOT");
        expect_kw("NULL");
        n->kind = neg ? ASTNode::SQLIsNotNull : ASTNode::SQLIsNull;
        n->left = left;
        return n;
      }
      const bool not_in = u == "NOT" && is_kw("IN");
      if (u == "IN" || not_in) {  // x [NOT] IN (SELECT ..)
        if (not_in) pos++;
        if (!subquery_at(pos)) {
          if (peek().kind == Token::Sym && peek().text == "(")
            fail(DFGPU_ERR_NOT_IMPLEMENTED, "IN over a list of values is not supported: only IN (SELECT ..)");
          perr("Expected ( after IN, found: " + peek().text);
        }
        n->kind = ASTNode::SQLInSubquery;
        n->left = left;
        n->negated = not_in;
        n->subquery = parse_subquery();
        return n;
      }
      n->kind = ASTNode::SQLBinaryExpr;
      n->left = left;
      if (u == "AND") n->op = SQLOperator::And;
      else if (u == "OR") n->op = SQLOperator::Or;
      else if (u == "LIKE") n->op = SQLOperator::Like;
      else if (u == "NOT") {
        if (!accept_kw("LIKE")) perr("Expected LIKE or IN after NOT, found: " + peek().text);
        n->op = SQLOperator::NotLike;
      }
      else perr("No infix parser for token " + t.text);
      n->right = parse_expr(precedence);
      return n;
    }
    n->kind = ASTNode::SQLBinaryExpr;
    n->left = left;
    const std::string& s = t.text;
    if (s == "=") n->op = SQLOperator::Eq;
    else if (s == "!=" || s == "<>") n->op = SQLOperator::NotEq;
    else if (s == "<") n->op = SQLOperator::Lt;
    else if (s == "<=") n->op = SQLOperator::LtEq;
    else if (s == ">") n->op = SQLOperator::Gt;
    else if (s == ">=") n->op = SQLOperator::GtEq;
    else if (s == "+") n->op = SQLOperator::Plus;
    else if (s == "-") n->op = SQLOperator::Minus;
    else if (s == "*") n->op = SQLOperator::Multiply;
    else if (s == "/") n->op = SQLOperator::Divide;
    else if (s == "%") n->op = SQLOperator::Modulus;
    else perr("No infix parser for token " + s);
    n->right = parse_expr(precedence);
    return n;
  }

  // OVER ( [PARTITION BY e, ..] [ORDER BY e [ASC|DESC], ..] ) after a function call
  void parse_window(ASTNode& f) {
    expect_kw("OVER");
    expect_sym("(");
    f.over = true;
    if (is_kw("PARTITION") && toks[pos + 1].kind == Token::Ident && upper(toks[pos + 1].text) == "BY") {
      pos += 2;
      do { f.partition_by.push_back(parse_expr()); } while (accept_sym(","));
    }
    if (accept_kw("ORDER")) {
      expect_kw("BY");
      do {
        OrderByExpr o;
        o.expr = parse_expr();
        if (accept_kw("DESC")) o.asc = false;
        else accept_kw("ASC");
        f.window_order.push_back(o);
      } while (accept_sym(","));
    }
    if (is_kw("ROWS") || is_kw("RANGE") || is_kw("GROUPS")) fail(DFGPU_ERR_NOT_IMPLEMENTED, "window frame clauses are not supported");
    expect_sym(")");
  }

  // tokens i, i + 1 are `(` SELECT
  bool subquery_at(size_t i) const {
    return i + 1 < toks.size() && toks[i].kind == Token::Sym && toks[i].text == "(" && toks[i + 1].kind == Token::Ident &&
           upper(toks[i + 1].text) == "SELECT";
  }
  ASTRef parse_subquery() {
    expect_sym("(");
    ASTRef q = parse_select();
    expect_sym(")");
    return q;
  }

  // name [ [AS] alias ]
  ASTRef parse_table_ref(const char* after) {
    Token t = next();
    if (t.kind != Token::Ident || reserved(upper(t.text))) perr(std::string("Expected a table name after ") + after);
    auto r = std::make_shared<ASTNode>();
    r->kind = ASTNode::SQLIdentifier;
    r->id = t.text;
    const bool as = accept_kw("AS");
    if (peek().kind == Token::Ident && !reserved(upper(peek().text))) r->qualifier = next().text;
    else if (as) perr("Expected an alias after AS");
    return r;
  }

  ASTRef parse_select() {
    expect_kw("SELECT");
    auto n = std::make_shared<ASTNode>();
    n->kind = ASTNode::SQLSelect;
    do { n->projection.push_back(parse_expr()); } while (accept_sym(","));
    if (accept_kw("FROM")) {
      n->relation = parse_table_ref("FROM");
      for (;;) {
        for (const char* kind : {"LEFT", "RIGHT", "FULL", "OUTER", "CROSS", "NATURAL"})
          if (is_kw(kind)) fail(DFGPU_ERR_NOT_IMPLEMENTED, std::string(kind) + " JOIN is not supported: only [INNER] JOIN .. ON");
        if (accept_kw("INNER")) expect_kw("JOIN");
        else if (!accept_kw("JOIN")) break;
        JoinClause j;
        j.relation = parse_table_ref("JOIN");
        if (is_kw("USING")) perr("JOIN .. USING is not supported: use JOIN .. ON");
        expect_kw("ON");
        j.on = parse_expr();
        n->joins.push_back(j);
      }
    }
    if (accept_kw("WHERE")) n->selection = parse_expr();
    if (accept_kw("GROUP")) {
      expect_kw("BY");
      n->has_group_by = true;
      do { n->group_by.push_back(parse_expr()); } while (accept_sym(","));
    }
    if (accept_kw("HAVING")) n->having = parse_expr();
    if (accept_kw("ORDER")) {
      expect_kw("BY");
      n->has_order_by = true;
      do {
        OrderByExpr o;
        o.expr = parse_expr();
        if (accept_kw("DESC")) o.asc = false;
        else accept_kw("ASC");
        n->order_by.push_back(o);
      } while (accept_sym(","));
    }
    if (accept_kw("LIMIT")) n->limit = parse_expr();
    return n;
  }
};

}  // namespace

std::string ASTNode::debug() const {
  switch (kind) {
    case SQLIdentifier: return "SQLIdentifier(\"" + id + "\")";
    case SQLWildcard: return "SQLWildcard";
    case SQLLong: return "SQLValue(Long(" + std::to_string(lval) + "))";
    case SQLDouble: return "SQLValue(Double(" + rust_debug_f64(dval) + "))";
    case SQLString: return "SQLValue(SingleQuotedString(\"" + id + "\"))";
    case SQLBinaryExpr: return "SQLBinaryExpr { .. }";
    case SQLCast: return "SQLCast { .. }";
    case SQLIsNull: return "SQLIsNull(..)";
    case SQLIsNotNull: return "SQLIsNotNull(..)";
    case SQLFunction: return "SQLFunction { id: \"" + id + "\"" + (over ? ", over: Some(..)" : "") + ", .. }";
    case SQLSelect: return "SQLSelect { .. }";
    case SQLInSubquery: return negated ? "SQLInSubquery { negated: true, .. }" : "SQLInSubquery { .. }";
    case SQLExists: return negated ? "SQLExists { negated: true, .. }" : "SQLExists { .. }";
    case SQLCase: return "SQLCase { .. }";
  }
  return "?";
}

ASTRef parse_sql(const std::string& sql) {
  Parser p;
  p.toks = tokenize(sql);
  ASTRef e = p.parse_expr();
  p.accept_sym(";");
  if (p.peek().kind != Token::End) perr("Unexpected token after end of statement: " + p.peek().text);
  return e;
}

}  // namespace dfhost
