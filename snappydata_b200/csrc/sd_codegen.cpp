// sd_codegen.cpp -- plan analysis + generation of the PLAN struct consumed by sd_kernels.cuh.
//
// This is the CUDA counterpart of what the reference does in CodegenSupport.doProduce/doConsume:
// the reference emits Java for Janino per plan (ColumnTableScan.scala:186-672,
// SnappyHashAggregateExec.scala:240-263, 450-491, 1278-1580); we emit a ~30-line CUDA struct that
// plugs the plan's expressions into the hand-written kernel template.  The same generator feeds the
// ahead-of-time compiled benchmark plans (build step) and the NVRTC path for every other plan.
#include "sd_codegen.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <sstream>

namespace sd {

bool type_is_integral(int t) {
  return t == SD_BOOLEAN || t == SD_BYTE || t == SD_SHORT || t == SD_INT || t == SD_LONG || t == SD_DATE ||
         t == SD_TIMESTAMP || t == SD_DECIMAL;
}
bool type_is_fp(int t) { return t == SD_FLOAT || t == SD_DOUBLE; }
int sum_buffer_type(int t) { return type_is_fp(t) ? SD_DOUBLE : (t == SD_DECIMAL ? SD_DECIMAL : SD_LONG); }

int decimal_ps(const PlanSpec& p, int node) {
  const sd_expr& e = p.exprs[node];
  if (e.op == SD_OP_COL) return (p.cols[e.a].precision << 8) | p.cols[e.a].scale;
  if (e.op == SD_OP_NEG) return decimal_ps(p, e.a);
  return e.c;
}
bool node_is_wide(const PlanSpec& p, int node) {
  return p.exprs[node].type == SD_DECIMAL && (decimal_ps(p, node) >> 8) > 18;
}
int kind_of_column(const sd_column& c) { return wide_decimal(c.type, c.precision) ? K_CODE : kind_of_type(c.type); }
static const char* col_ctype(const sd_column& c);

int kind_of_type(int t) {
  switch (t) {
    case SD_BOOLEAN: return K_BOOL;
    case SD_BYTE: return K_I8;
    case SD_SHORT: return K_I16;
    case SD_INT: case SD_DATE: return K_I32;
    case SD_LONG: case SD_TIMESTAMP: case SD_DECIMAL: return K_I64;
    case SD_FLOAT: return K_F32;
    case SD_DOUBLE: return K_F64;
    case SD_STRING: return K_CODE;
  }
  return -1;
}

static const char* ctype_of(int t) {
  switch (t) {
    case SD_BOOLEAN: return "uint8_t";
    case SD_BYTE: return "int8_t";
    case SD_SHORT: return "int16_t";
    case SD_INT: case SD_DATE: return "int32_t";
    case SD_LONG: case SD_TIMESTAMP: case SD_DECIMAL: return "int64_t";
    case SD_FLOAT: return "float";
    case SD_DOUBLE: return "double";
    case SD_STRING: return "int32_t";
  }
  return "void";
}
static const char* col_ctype(const sd_column& c) { return wide_decimal(c.type, c.precision) ? "int32_t" : ctype_of(c.type); }
static const char* tname(int t) {
  static const char* n[] = {"?", "bool", "i8", "i16", "i32", "i64", "f32", "f64", "date", "ts", "str", "dec"};
  return (t >= 1 && t <= 11) ? n[t] : "?";
}
static const char* opname(int op) {
  switch (op) {
    case SD_OP_COL: return "col"; case SD_OP_LIT: return "lit"; case SD_OP_ADD: return "add"; case SD_OP_SUB: return "sub";
    case SD_OP_MUL: return "mul"; case SD_OP_DIV: return "div"; case SD_OP_NEG: return "neg"; case SD_OP_CAST: return "cast";
    case SD_OP_EQ: return "eq"; case SD_OP_NE: return "ne"; case SD_OP_LT: return "lt"; case SD_OP_LE: return "le";
    case SD_OP_GT: return "gt"; case SD_OP_GE: return "ge"; case SD_OP_AND: return "and"; case SD_OP_OR: return "or";
    case SD_OP_NOT: return "not"; case SD_OP_ISNULL: return "isnull"; case SD_OP_ISNOTNULL: return "isnotnull";
    case SD_OP_IN: return "in"; case SD_OP_STARTSWITH: return "startswith"; case SD_OP_PAIR: return "pair";
  }
  return "?";
}
static bool is_unary(int op) {
  return op == SD_OP_NEG || op == SD_OP_CAST || op == SD_OP_NOT || op == SD_OP_ISNULL || op == SD_OP_ISNOTNULL || op == SD_OP_IN;
}
static bool is_cmp(int op) { return op >= SD_OP_EQ && op <= SD_OP_GE; }
static bool is_grouping_node(int op) { return op == SD_OP_GROUPING_SET || op == SD_OP_GROUPING_ID; }
// AggFamily of an SD_AGG_* code (1..19), -1 when unknown
static int agg_family(int fn) {
  static const int family[] = {-1, AGG_COUNT, AGG_COUNT, AGG_SUM, AGG_AVG, AGG_MINMAX, AGG_MINMAX, AGG_MOMENT, AGG_MOMENT, AGG_MOMENT,
                               AGG_MOMENT, AGG_MOMENT, AGG_MOMENT, AGG_PAIR, AGG_PAIR, AGG_PAIR, AGG_ORDER, AGG_ORDER, AGG_ORDER, AGG_ORDER};
  return fn >= 1 && fn <= SD_AGG_LAST_IGNORE_NULLS ? family[fn] : -1;
}

sd_plan_desc PlanSpec::desc_view() const {
  sd_plan_desc d;
  memset(&d, 0, sizeof(d));
  d.abi_version = SD_ABI_VERSION;
  d.ncols = (int)cols.size(); d.cols = cols.data();
  d.nexprs = (int)exprs.size(); d.exprs = exprs.data();
  d.filter = filter;
  d.nkeys = (int)desc_keys.size(); d.keys = desc_keys.data();
  d.naggs = (int)aggs.size(); d.aggs = aggs.data();
  d.nproj = (int)proj.size(); d.proj = proj.data();
  d.nliterals = (int)literal_types.size(); d.literal_types = literal_types.data();
  d.flags = flags;
  return d;
}

// structural text of an expression subtree (CSE key and part of the plan signature)
static std::string expr_text(const PlanSpec& p, int node) {
  const sd_expr& e = p.exprs[node];
  std::ostringstream o;
  o << opname(e.op) << ":" << tname(e.type);
  if (e.type == SD_DECIMAL) o << "[" << decimal_ps(p, node) << "]";
  if (e.op == SD_OP_COL) o << "(c" << e.a << ")";
  else if (e.op == SD_OP_LIT) o << "(l" << e.a << ")";
  else if (e.op == SD_OP_IN) o << "(" << expr_text(p, e.a) << ",l" << e.b << "x" << e.c << ")";
  else if (is_unary(e.op)) o << "(" << expr_text(p, e.a) << ")";
  else o << "(" << expr_text(p, e.a) << "," << expr_text(p, e.b) << ")";
  return o.str();
}

// a predicate over (one STRING column, literals) that is evaluated per dictionary entry on the host
static bool string_predicate_col(const PlanSpec& p, int node, int* col) {
  const sd_expr& e = p.exprs[node];
  if (is_cmp(e.op)) {
    const sd_expr &a = p.exprs[e.a], &b = p.exprs[e.b];
    if (a.type != SD_STRING) return false;
    if (a.op == SD_OP_COL && b.op == SD_OP_LIT) { *col = a.a; return true; }
    if (b.op == SD_OP_COL && a.op == SD_OP_LIT) { *col = b.a; return true; }
    return false;
  }
  if (e.op == SD_OP_IN && p.exprs[e.a].type == SD_STRING && p.exprs[e.a].op == SD_OP_COL) { *col = p.exprs[e.a].a; return true; }
  if (e.op == SD_OP_STARTSWITH && p.exprs[e.a].op == SD_OP_COL && p.exprs[e.b].op == SD_OP_LIT) { *col = p.exprs[e.a].a; return true; }
  return false;
}

int cmp_bytes(const char* a, int la, const char* b, int lb) {
  int n = la < lb ? la : lb;
  int c = n ? memcmp(a, b, n) : 0;
  return c ? c : la - lb;
}

int eval_string_predicate(const PlanSpec& p, int node, const char* s, int slen, const sd_literal* lits) {
  const sd_expr& e = p.exprs[node];
  if (s == nullptr) return 2;                      // NULL operand => NULL (IN: null value => NULL)
  if (is_cmp(e.op)) {
    const sd_expr &a = p.exprs[e.a], &b = p.exprs[e.b];
    const bool col_left = a.op == SD_OP_COL;
    const sd_literal& l = lits[col_left ? b.a : a.a];
    if (l.is_null) return 2;
    int c = col_left ? cmp_bytes(s, slen, l.s, l.slen) : cmp_bytes(l.s, l.slen, s, slen);
    switch (e.op) {
      case SD_OP_EQ: return c == 0; case SD_OP_NE: return c != 0; case SD_OP_LT: return c < 0;
      case SD_OP_LE: return c <= 0; case SD_OP_GT: return c > 0; default: return c >= 0;
    }
  }
  if (e.op == SD_OP_IN) {
    bool has_null = false;
    for (int k = 0; k < e.c; k++) {
      const sd_literal& l = lits[e.b + k];
      if (l.is_null) { has_null = true; continue; }
      if (cmp_bytes(s, slen, l.s, l.slen) == 0) return 1;
    }
    return has_null ? 2 : 0;
  }
  if (e.op == SD_OP_STARTSWITH) {
    const sd_literal& l = lits[p.exprs[e.b].a];
    if (l.is_null) return 2;
    return slen >= l.slen && (l.slen == 0 || memcmp(s, l.s, l.slen) == 0);
  }
  return 2;
}

namespace {

struct Gen {
  PlanSpec& p;
  std::string& err;
  std::map<int, int> table_of_node;   // predicate node -> table index
  std::vector<int> keymap_table;      // key index -> table index
  Gen(PlanSpec& p_, std::string& e) : p(p_), err(e) {}

  int fail(int code, const std::string& m) { err = m; return code; }

  // GROUP BY ... WITH ROLLUP / CUBE / GROUPING SETS: a GROUPING_ID node as the last key lists the sets' masks; it is taken out of
  // `keys` so that everything generated from here on is the plain GROUP BY over the keys before it
  int grouping_sets() {
    const int ne = (int)p.exprs.size(), nk = (int)p.keys.size();
    std::vector<char> member(ne, 0);
    for (int i = 0; i < ne; i++) {
      const sd_expr& e = p.exprs[i];
      if (e.op == SD_OP_GROUPING_SET && e.type != SD_INT) return fail(SD_ERR_INVALID, "a GROUPING_SET node has type INT");
      if (e.op != SD_OP_GROUPING_ID) continue;
      if (e.type != SD_INT) return fail(SD_ERR_INVALID, "a GROUPING_ID node has type INT");
      if (e.b < 1) return fail(SD_ERR_INVALID, "a GROUPING_ID node lists at least one grouping set");
      if (e.a < 0 || e.a + (int64_t)e.b > i) return fail(SD_ERR_INVALID, "a GROUPING_ID node's sets must precede it");
      for (int j = e.a; j < e.a + e.b; j++) {
        if (p.exprs[j].op != SD_OP_GROUPING_SET) return fail(SD_ERR_INVALID, "a GROUPING_ID node lists consecutive GROUPING_SET nodes");
        member[j] = 1;
      }
    }
    for (int i = 0; i < ne; i++) {
      const sd_expr& e = p.exprs[i];
      if (e.op == SD_OP_GROUPING_SET && !member[i]) return fail(SD_ERR_INVALID, "a GROUPING_SET node outside a GROUPING_ID list");
      if (e.op == SD_OP_COL || e.op == SD_OP_LIT || is_grouping_node(e.op)) continue;
      const bool bin = !is_unary(e.op);
      auto bad = [&](int c) { return c >= 0 && c < ne && is_grouping_node(p.exprs[c].op); };
      if (bad(e.a) || (bin && bad(e.b))) return fail(SD_ERR_INVALID, "a GROUPING_SET / GROUPING_ID node is not an operand");
    }
    auto is_gid = [&](int n) { return n >= 0 && n < ne && is_grouping_node(p.exprs[n].op); };
    if (is_gid(p.filter)) return fail(SD_ERR_INVALID, "a GROUPING_ID node cannot be a filter");
    for (auto& a : p.aggs) if (is_gid(a.expr)) return fail(SD_ERR_INVALID, "a GROUPING_ID node cannot be an aggregate input");
    for (int k : p.proj) if (is_gid(k)) return fail(SD_ERR_INVALID, "a GROUPING_ID node cannot be projected or assigned");
    for (int k = 0; k < nk; k++) {
      if (!is_gid(p.keys[k])) continue;
      if (p.exprs[p.keys[k]].op != SD_OP_GROUPING_ID || k != nk - 1) return fail(SD_ERR_INVALID, "a GROUPING_ID node is only the last grouping key");
    }
    const int last = nk > 0 && is_gid(p.keys[nk - 1]) ? p.keys[nk - 1] : -1;
    for (int i = 0; i < ne; i++)
      if (p.exprs[i].op == SD_OP_GROUPING_ID && i != last) return fail(SD_ERR_INVALID, "a GROUPING_ID node is only the last grouping key");
    if (last < 0) return 0;
    if (p.flags & SD_PLAN_MUTATE) return fail(SD_ERR_UNSUPPORTED, "GROUPING_ID in an UPDATE / DELETE plan");
    if (p.aggs.empty() && nk == 1) return fail(SD_ERR_UNSUPPORTED, "GROUPING_ID in a projection plan");
    const sd_expr& g = p.exprs[p.keys[nk - 1]];
    const int n = nk - 1;
    if (n == 0) return fail(SD_ERR_UNSUPPORTED, "grouping sets without GROUP BY expressions");
    if (n > 31) return fail(SD_ERR_UNSUPPORTED, "grouping sets over more than 31 GROUP BY expressions (spark_grouping_id is an INT)");
    if (g.b > 4096) return fail(SD_ERR_UNSUPPORTED, "more than 4096 grouping sets");
    for (int j = g.a; j < g.a + g.b; j++) {
      const uint32_t m = (uint32_t)p.exprs[j].a;
      if (p.exprs[j].a < 0 || (n < 32 && (m >> n) != 0)) return fail(SD_ERR_INVALID, "a grouping-set mask has bits at or above the number of GROUP BY expressions");
      for (uint32_t q : p.sets) if (q == m) return fail(SD_ERR_UNSUPPORTED, "duplicate grouping sets (Expand would feed each row twice into one group)");
      p.sets.push_back(m);
    }
    p.gid_node = p.keys[nk - 1];
    p.keys.pop_back();
    return 0;
  }

  int validate() {
    const int ne = (int)p.exprs.size();
    if ((int)p.cols.size() > 64) return fail(SD_ERR_UNSUPPORTED, "more than 64 scan columns in one fused plan");
    if ((int)p.literal_types.size() > MAX_LITERALS) return fail(SD_ERR_UNSUPPORTED, "more than 64 literal slots");
    for (auto& c : p.cols) if (kind_of_type(c.type) < 0) return fail(SD_ERR_INVALID, "unknown column type");
    for (auto& c : p.cols) if (c.type == SD_DECIMAL && (c.precision < 1 || c.precision > 38 || c.scale < 0 || c.scale > c.precision))
      return fail(SD_ERR_INVALID, "DECIMAL scan column needs 1 <= precision <= 38 and 0 <= scale <= precision");
    for (int i = 0; i < ne; i++) {
      const sd_expr& e = p.exprs[i];
      if (is_grouping_node(e.op)) continue;   // checked by grouping_sets()
      if (e.op == SD_OP_COL) { if (e.a < 0 || e.a >= (int)p.cols.size()) return fail(SD_ERR_INVALID, "column reference out of range"); }
      else if (e.op == SD_OP_LIT) { if (e.a < 0 || e.a >= (int)p.literal_types.size()) return fail(SD_ERR_INVALID, "literal slot out of range"); }
      else {
        if (e.a < 0 || e.a >= i) return fail(SD_ERR_INVALID, "expression children must precede parents");
        if (!is_unary(e.op) && (e.b < 0 || e.b >= i)) return fail(SD_ERR_INVALID, "expression children must precede parents");
        if (e.op == SD_OP_IN && (e.b < 0 || e.c < 1 || e.b + e.c > (int)p.literal_types.size())) return fail(SD_ERR_INVALID, "IN list out of range");
      }
      if (kind_of_type(e.type) < 0) return fail(SD_ERR_INVALID, "unknown expression type");
      if (e.type == SD_DECIMAL) {
        const int ps = decimal_ps(p, i), pr = ps >> 8, sc = ps & 0xff;
        if (pr < 1 || pr > 38 || sc > pr) return fail(SD_ERR_INVALID, "DECIMAL expression needs 1 <= precision <= 38 and scale <= precision (sd_expr.c / sd_column)");
      }
      // DECIMAL wider than 18 digits: read, compared, cast up, grouped and aggregated; no arithmetic on it
      const bool wide_here = node_is_wide(p, i);
      const bool wide_a = e.op != SD_OP_COL && e.op != SD_OP_LIT && node_is_wide(p, e.a);
      const bool wide_b = e.op != SD_OP_COL && e.op != SD_OP_LIT && !is_unary(e.op) && node_is_wide(p, e.b);
      if ((e.op >= SD_OP_ADD && e.op <= SD_OP_NEG) && (wide_here || wide_a || wide_b))
        return fail(SD_ERR_UNSUPPORTED, "arithmetic on a DECIMAL wider than 18 digits");
      if (e.op == SD_OP_STARTSWITH && (wide_a || wide_b)) return fail(SD_ERR_UNSUPPORTED, "startsWith on a DECIMAL wider than 18 digits");
      if (e.op == SD_OP_CAST && wide_a && !(wide_here && (decimal_ps(p, i) & 0xff) >= (decimal_ps(p, e.a) & 0xff)))
        return fail(SD_ERR_UNSUPPORTED, "cast from a DECIMAL wider than 18 digits to anything but an equal or wider DECIMAL");
      if (e.op == SD_OP_CAST && wide_here && !wide_a && p.exprs[e.a].type != SD_DECIMAL)
        return fail(SD_ERR_UNSUPPORTED, "cast to a DECIMAL wider than 18 digits from a non-DECIMAL type");
      if (e.op == SD_OP_CAST) {   // refused casts are refused at plan creation, whether or not the node ends up in generated code
        const int from = p.exprs[e.a].type, to = e.type;
        const bool tf = from == SD_DATE || from == SD_TIMESTAMP, tt = to == SD_DATE || to == SD_TIMESTAMP;
        if (from == SD_STRING || to == SD_STRING) return fail(SD_ERR_UNSUPPORTED, "casts involving STRING");
        if ((tf || tt) && from != to) return fail(SD_ERR_UNSUPPORTED, "casts involving DATE / TIMESTAMP (time-zone dependent in Spark)");
        if (from == SD_DECIMAL && !(type_is_fp(to) || to == SD_DECIMAL)) return fail(SD_ERR_UNSUPPORTED, "this cast from DECIMAL");
        if (to == SD_DECIMAL && !(from == SD_BYTE || from == SD_SHORT || from == SD_INT || from == SD_LONG || from == SD_DECIMAL))
          return fail(SD_ERR_UNSUPPORTED, "this cast to DECIMAL");
        if (from == SD_DECIMAL && to == SD_DECIMAL && (decimal_ps(p, i) & 0xff) < (decimal_ps(p, e.a) & 0xff))
          return fail(SD_ERR_UNSUPPORTED, "DECIMAL cast that reduces the scale (needs HALF_UP rounding)");
      }
    }
    auto chk = [&](int n) { return n >= 0 && n < ne; };
    if (p.filter >= 0 && (!chk(p.filter) || p.exprs[p.filter].type != SD_BOOLEAN)) return fail(SD_ERR_INVALID, "filter must be a BOOLEAN expression");
    for (int k : p.keys) if (!chk(k)) return fail(SD_ERR_INVALID, "key expression out of range");
    for (auto& a : p.aggs) if (a.expr != -1 && !chk(a.expr)) return fail(SD_ERR_INVALID, "aggregate input out of range");
    for (int k : p.proj) if (!chk(k)) return fail(SD_ERR_INVALID, "projection expression out of range");
    if ((int)p.keys.size() > MAX_HASH_KEYS) return fail(SD_ERR_UNSUPPORTED, "more than 32 grouping keys");
    // SD_OP_PAIR: two DOUBLE inputs of COVAR_POP / COVAR_SAMP / CORR, and nothing else
    auto is_pair = [&](int n) { return p.exprs[n].op == SD_OP_PAIR; };
    for (int i = 0; i < ne; i++) {
      const sd_expr& e = p.exprs[i];
      if (is_grouping_node(e.op)) continue;
      if (e.op == SD_OP_PAIR && (e.type != SD_DOUBLE || p.exprs[e.a].type != SD_DOUBLE || p.exprs[e.b].type != SD_DOUBLE))
        return fail(SD_ERR_INVALID, "a PAIR node and both its inputs must be DOUBLE (cast them)");
      if (e.op != SD_OP_COL && e.op != SD_OP_LIT && (is_pair(e.a) || (!is_unary(e.op) && is_pair(e.b))))
        return fail(SD_ERR_INVALID, "a PAIR node is only the input of COVAR_POP / COVAR_SAMP / CORR, not of another operator");
    }
    if (p.filter >= 0 && is_pair(p.filter)) return fail(SD_ERR_INVALID, "a PAIR node cannot be a filter");
    for (int k : p.keys) if (is_pair(k)) return fail(SD_ERR_INVALID, "a PAIR node cannot be a grouping key");
    for (int k : p.proj) if (is_pair(k)) return fail(SD_ERR_INVALID, "a PAIR node cannot be projected or assigned");
    for (auto& a : p.aggs) {
      const bool pair_agg = agg_family(a.fn) == AGG_PAIR;
      if (pair_agg && (a.expr < 0 || !is_pair(a.expr))) return fail(SD_ERR_INVALID, "COVAR_POP / COVAR_SAMP / CORR need a PAIR node input");
      if (!pair_agg && a.expr >= 0 && is_pair(a.expr)) return fail(SD_ERR_INVALID, "a PAIR node is only the input of COVAR_POP / COVAR_SAMP / CORR");
    }
    return 0;
  }

  void nullability() {   // Catalyst Expression.nullable
    p.expr_nullable.assign(p.exprs.size(), 0);
    for (size_t i = 0; i < p.exprs.size(); i++) {
      const sd_expr& e = p.exprs[i];
      int n;
      switch (e.op) {
        case SD_OP_COL: n = p.cols[e.a].nullable; break;
        case SD_OP_LIT: n = 1; break;   // a ParamLiteral's value (incl. NULL) is only known at run time
        case SD_OP_DIV: n = 1; break;
        case SD_OP_ISNULL: case SD_OP_ISNOTNULL: case SD_OP_GROUPING_SET: case SD_OP_GROUPING_ID: n = 0; break;
        case SD_OP_CAST: n = p.expr_nullable[e.a] || e.type == SD_DECIMAL; break;   // Cast.forceNullable: -> DECIMAL may overflow to NULL
        case SD_OP_NEG: case SD_OP_NOT: n = p.expr_nullable[e.a]; break;
        case SD_OP_IN: n = 1; break;
        default: n = p.expr_nullable[e.a] || p.expr_nullable[e.b]; break;
      }
      p.expr_nullable[i] = n;
    }
  }

  // Static nullability as the reference sees it for buffer schemas: literals are non-null there
  // (TokenLiteral/ParamLiteral.nullable == false for non-null constants), so recompute ignoring LIT.
  int static_nullable(int node) {
    const sd_expr& e = p.exprs[node];
    switch (e.op) {
      case SD_OP_COL: return p.cols[e.a].nullable;
      case SD_OP_LIT: return 0;
      case SD_OP_DIV: return 1;
      case SD_OP_ISNULL: case SD_OP_ISNOTNULL: return 0;
      case SD_OP_CAST: return static_nullable(e.a) || e.type == SD_DECIMAL;
      case SD_OP_NEG: case SD_OP_NOT: case SD_OP_IN: return static_nullable(e.a);
      default: return static_nullable(e.a) || static_nullable(e.b);
    }
  }

  int add_slot(int op, int node, int gate) {
    std::string key = std::to_string(op) + "|" + std::to_string(gate) + "|" + (node >= 0 ? expr_text(p, node) : std::string("-"));
    for (size_t s = 0; s < p.slots.size(); s++) {
      const SlotSpec& x = p.slots[s];
      std::string k2 = std::to_string(x.op) + "|" + std::to_string(x.gate) + "|" + (x.node >= 0 ? expr_text(p, x.node) : std::string("-"));
      if (k2 == key) return (int)s;
    }
    p.slots.push_back(SlotSpec{op, node, gate});
    return (int)p.slots.size() - 1;
  }
  int count_slot_for(int node) {   // number of non-null inputs of `node`
    if (node < 0 || !static_nullable(node)) return add_slot(SLOT_ADD_I64, -1, GATE_ONE);
    return add_slot(SLOT_ADD_I64, node, GATE_NONNULL_COUNT);
  }

  // the buffer of SUM / MIN / MAX is nullable when its input is (grouped: SnappyHashAggregateExec.scala:174-210) and always
  // without keys (a plain Spark buffer, NULL until the first non-null input, :337-346); a nullable buffer counts its inputs
  void nullable_buffer(AggMap& m, int node, bool keyed) {
    m.buf_nullable = keyed ? static_nullable(node) : 1;
    if (m.buf_nullable) m.count_slot = count_slot_for(node);
  }
  // the STRING column's TABLE_KEYPTR table that aggregates share, added on first use
  int keyptr_table(int col) {
    for (size_t t = 0; t < p.tables.size(); t++)
      if (p.tables[t].kind == TABLE_KEYPTR && p.tables[t].col == col && p.tables[t].key < 0) return (int)t;
    p.tables.push_back(TableSpec{TABLE_KEYPTR, col, -1, -1});
    return (int)p.tables.size() - 1;
  }

  int build_slots() {
    const bool keyed = !p.keys.empty();
    for (auto& a : p.aggs) {
      AggMap m;
      memset(&m, 0, sizeof(m));
      m.fn = a.fn; m.family = agg_family(a.fn); m.hold = HOLD_WORD;
      m.value_slot = -1; m.value_slot2 = -1; m.count_slot = -1; m.shift = -1; m.shift_y = -1; m.order_slot = -1;
      for (int& l : m.limb_slot) l = -1;
      for (int& s : m.pow_slot) s = -1;
      for (int& s : m.pair_slot) s = -1;
      const int it = a.expr >= 0 ? p.exprs[a.expr].type : SD_LONG;
      if (a.fn != SD_AGG_COUNT_STAR && a.expr < 0) return fail(SD_ERR_INVALID, "aggregate without input expression");
      if (it == SD_DECIMAL) m.buf_ps = m.in_ps = decimal_ps(p, a.expr);   // MIN / MAX / FIRST / LAST keep the input type
      const bool wide = a.expr >= 0 && node_is_wide(p, a.expr);
      if (m.family == AGG_MOMENT) {
        // n = the non-null count, S_j = sum (x - K)^j around the group's shift K; the host turns them into Spark's buffers
        if (it != SD_DOUBLE) return fail(SD_ERR_INVALID, "STDDEV / VARIANCE / SKEWNESS / KURTOSIS need a DOUBLE input (cast it)");
        m.buf_type = SD_DOUBLE;
        m.hold = HOLD_SHIFTED;
        m.count_slot = count_slot_for(a.expr);
        const int order = moment_order(a.fn);
        for (int j = 0; j < order; j++) m.pow_slot[j] = add_slot(SLOT_ADD_F64, a.expr, GATE_POW1 + j);
        m.value_slot = m.pow_slot[0];
        for (size_t i = 0; i < p.shifts.size(); i++) if (p.shifts[i].pow_slot[0] == m.pow_slot[0]) m.shift = (int)i;   // same input
        if (m.shift < 0) { p.shifts.push_back(ShiftSpec{0, {-1, -1, -1, -1}}); m.shift = (int)p.shifts.size() - 1; }
        ShiftSpec* sh = &p.shifts[(size_t)m.shift];
        for (int j = 0; j < order; j++) sh->pow_slot[j] = m.pow_slot[j];
        sh->order = std::max(sh->order, order);
        p.agg_map.push_back(m);
        continue;
      }
      if (m.family == AGG_PAIR) {
        // n = the count of rows with x and y non-null; S_x, S_y, S_xy (+ CORR's S_xx, S_yy) around the group's (Kx, Ky)
        const bool corr = a.fn == SD_AGG_CORR;
        m.buf_type = SD_DOUBLE;
        m.hold = HOLD_SHIFTED;
        m.count_slot = count_slot_for(a.expr);   // the PAIR node is NULL when x or y is
        for (int j = 0; j < (corr ? 5 : 3); j++) m.pair_slot[j] = add_slot(SLOT_ADD_F64, a.expr, GATE_PAIR_X + j);
        m.value_slot = m.pair_slot[2];
        int q = -1;
        for (size_t i = 0; i < p.pairs.size(); i++) if (p.pairs[i].xy_slot == m.pair_slot[2]) q = (int)i;   // same PAIR input
        if (q < 0) {
          p.shifts.push_back(ShiftSpec{1, {m.pair_slot[0], -1, -1, -1}});
          p.shifts.push_back(ShiftSpec{1, {m.pair_slot[1], -1, -1, -1}});
          p.pairs.push_back(PairSpec{(int)p.shifts.size() - 2, (int)p.shifts.size() - 1, m.pair_slot[2]});
          q = (int)p.pairs.size() - 1;
        }
        m.shift = p.pairs[(size_t)q].shift_x;
        m.shift_y = p.pairs[(size_t)q].shift_y;
        if (corr) {   // the squares are the order-2 sums of the pair's x and y shifts
          ShiftSpec &sx = p.shifts[(size_t)m.shift], &sy = p.shifts[(size_t)m.shift_y];
          sx.order = sy.order = 2;
          sx.pow_slot[1] = m.pair_slot[3];
          sy.pow_slot[1] = m.pair_slot[4];
        }
        p.agg_map.push_back(m);
        continue;
      }
      if (m.family == AGG_ORDER) {
        // one (order key, value) pair at an even slot index; FIRST and LAST of one input, or one function with and without
        // ignoreNulls, keep pairs of their own
        const bool str = it == SD_STRING;
        if ((str || wide) && p.exprs[a.expr].op != SD_OP_COL)
          return fail(SD_ERR_UNSUPPORTED, "FIRST / LAST of a STRING or wide DECIMAL expression that is not a column");
        m.buf_type = it;
        m.hold = str || wide ? HOLD_REF : HOLD_WORD;
        m.buf_nullable = 1;
        const int op = a.fn == SD_AGG_LAST || a.fn == SD_AGG_LAST_IGNORE_NULLS ? SLOT_LAST : SLOT_FIRST;
        const int gate = a.fn == SD_AGG_FIRST_IGNORE_NULLS || a.fn == SD_AGG_LAST_IGNORE_NULLS ? GATE_ORDER_KEY_IGN : GATE_ORDER_KEY;
        const std::string in = expr_text(p, a.expr);
        for (size_t q = 0; q < p.slots.size(); q++)
          if (p.slots[q].op == op && p.slots[q].gate == gate && expr_text(p, p.slots[q].node) == in) m.order_slot = (int)q;
        if (m.order_slot < 0) {
          if (p.slots.size() % 2) p.slots.push_back(SlotSpec{SLOT_ADD_I64, -1, GATE_PAD});
          m.order_slot = (int)p.slots.size();
          p.slots.push_back(SlotSpec{op, a.expr, gate});
          p.slots.push_back(SlotSpec{SLOT_PAIR_VAL, a.expr, GATE_ORDER_VAL});
          // a STRING value is the address of the row's record, as for MIN / MAX over STRING
          if (str) p.slots.back().table = keyptr_table(p.exprs[a.expr].a);
          p.norder++;
        }
        m.value_slot = m.order_slot + 1;
        p.agg_map.push_back(m);
        continue;
      }
      if (a.expr >= 0 && it == SD_STRING && a.fn != SD_AGG_COUNT && (m.family != AGG_MINMAX || p.exprs[a.expr].op != SD_OP_COL))
        return fail(SD_ERR_UNSUPPORTED, "aggregates over STRING: only MIN / MAX / COUNT of a STRING column");
      switch (m.family) {
        case AGG_COUNT:
          m.value_slot = a.fn == SD_AGG_COUNT_STAR ? add_slot(SLOT_ADD_I64, -1, GATE_ONE) : count_slot_for(a.expr);
          m.buf_type = SD_LONG;
          break;
        case AGG_SUM: case AGG_AVG:
          if (it == SD_DECIMAL) {
            // Spark 2.1.1 Sum / Average over DECIMAL(p,s): buffer DECIMAL(min(38, p + 10), s) -- up to 28 digits from an input
            // of at most 18, i.e. wider than int64, so the value is summed in 32-bit parts (exact for < 2^31 rows) recombined on
            // the host: four limbs of a wide input, else the high / low halves
            m.buf_type = SD_DECIMAL;
            m.buf_ps = (std::min(38, (m.in_ps >> 8) + 10) << 8) | (m.in_ps & 0xff);
            m.hold = wide ? HOLD_LIMBS : HOLD_HILO;
            if (wide) for (int l = 0; l < 4; l++) m.value_slot = m.limb_slot[l] = add_slot(SLOT_ADD_I64, a.expr, GATE_LIMB0 + l);
            else { m.value_slot = add_slot(SLOT_ADD_I64, a.expr, GATE_VALUE_HI32); m.value_slot2 = add_slot(SLOT_ADD_I64, a.expr, GATE_VALUE_LO32); }
          } else {
            m.buf_type = m.family == AGG_AVG ? SD_DOUBLE : sum_buffer_type(it);
            m.value_slot = add_slot(m.buf_type == SD_DOUBLE ? SLOT_ADD_F64 : SLOT_ADD_I64, a.expr, GATE_VALUE);
          }
          if (m.family == AGG_SUM) nullable_buffer(m, a.expr, keyed);
          else m.count_slot = count_slot_for(a.expr);
          break;
        case AGG_MINMAX: {
          const bool str = it == SD_STRING, fp = type_is_fp(it), min = a.fn == SD_AGG_MIN;
          m.buf_type = it;
          if (str || wide) {   // the slot holds the address of the winning value's record, compared by bytes (STRING) or by value
            if (p.exprs[a.expr].op != SD_OP_COL) return fail(SD_ERR_UNSUPPORTED, "MIN / MAX of a wide DECIMAL expression that is not a column");
            m.hold = HOLD_REF;
            m.value_slot = add_slot(str ? (min ? SLOT_MIN_STR : SLOT_MAX_STR) : (min ? SLOT_MIN_DEC : SLOT_MAX_DEC), a.expr, str ? GATE_STRREF : GATE_DECREF);
            if (str) p.slots[m.value_slot].table = keyptr_table(p.exprs[a.expr].a);
          } else m.value_slot = add_slot(min ? (fp ? SLOT_MIN_F64 : SLOT_MIN_I64) : (fp ? SLOT_MAX_F64 : SLOT_MAX_I64), a.expr, GATE_VALUE);
          nullable_buffer(m, a.expr, keyed);
          break;
        }
        default: return fail(SD_ERR_INVALID, "unknown aggregate function");
      }
      p.agg_map.push_back(m);
    }
    p.rows_slot = add_slot(SLOT_ADD_I64, -1, GATE_ONE);
    if (p.norder > 0 && p.slots.size() % 2) p.slots.push_back(SlotSpec{SLOT_ADD_I64, -1, GATE_PAD});   // even group stride
    return 0;
  }

  // ---- expression emission ------------------------------------------------------------------------
  // value nodes:   const T vN = ...; const bool nN = ...;
  // BOOLEAN nodes additionally: const int tN (0 FALSE, 1 TRUE, 2 NULL)
  int emit_node(int node, std::vector<char>& done, std::ostringstream& o) {
    if (done[node]) return 0;
    const sd_expr& e = p.exprs[node];
    if (e.op != SD_OP_COL && e.op != SD_OP_LIT) {
      int col;
      if (!string_predicate_col(p, node, &col)) {
        int rc = emit_node(e.a, done, o);
        if (rc) return rc;
        if (!is_unary(e.op)) { rc = emit_node(e.b, done, o); if (rc) return rc; }
      }
    }
    done[node] = 1;
    const std::string N = std::to_string(node);
    const bool wide = node_is_wide(p, node);
    const char* T = wide ? "sd::i128" : ctype_of(e.type);
    auto V = [&](int n) { return "v" + std::to_string(n); };
    auto NL = [&](int n) { return "n" + std::to_string(n); };
    auto finish_bool = [&]() { o << "    const bool n" << N << " = t" << N << " == 2; const uint8_t v" << N << " = t" << N << " == 1;\n"; };
    switch (e.op) {
      case SD_OP_COL:
        if (wide) {   // the row holds the position of the value's record in the batch body
          const std::string C = std::to_string(e.a), nl = p.cols[e.a].nullable ? "r.n" + C : std::string("false");
          o << "    const bool n" << N << " = " << nl << "; const sd::i128 v" << N << " = n" << N
            << " ? (sd::i128)0 : sd::dec_rec(ctx.strbase[" << C << "] + (uint32_t)r.c" << C << ");\n";
          return 0;
        }
        o << "    const " << T << " v" << N << " = r.c" << e.a << "; const bool n" << N << " = "
          << (p.cols[e.a].nullable ? "r.n" + std::to_string(e.a) : std::string("false")) << ";\n";
        if (e.type == SD_BOOLEAN) o << "    const int t" << N << " = n" << N << " ? 2 : (v" << N << " ? 1 : 0);\n";
        return 0;
      case SD_OP_LIT: {
        if (e.type == SD_STRING) { o << "    const int32_t v" << N << " = 0; const bool n" << N << " = false;\n"; return 0; }
        if (wide) {
          o << "    const sd::i128 v" << N << " = sd::dec_lit(ctx.lit_bytes(" << e.a << ")); const bool n" << N << " = "
            << (p.lit_nullable ? "((ctx.L->nullmask >> " + std::to_string(e.a) + ") & 1ull) != 0" : std::string("false")) << ";\n";
          return 0;
        }
        std::string val = type_is_fp(e.type) ? "ctx.L->d[" + std::to_string(e.a) + "]" : "ctx.L->i[" + std::to_string(e.a) + "]";
        if (e.type == SD_BOOLEAN) val = "(" + val + " != 0)";
        o << "    const " << T << " v" << N << " = (" << T << ")" << val << "; const bool n" << N << " = "
          << (p.lit_nullable ? "((ctx.L->nullmask >> " + std::to_string(e.a) + ") & 1ull) != 0" : std::string("false")) << ";\n";
        if (e.type == SD_BOOLEAN) o << "    const int t" << N << " = n" << N << " ? 2 : (v" << N << " ? 1 : 0);\n";
        return 0;
      }
      case SD_OP_ADD: case SD_OP_SUB: case SD_OP_MUL: case SD_OP_DIV: {
        const char* sym = e.op == SD_OP_ADD ? "+" : e.op == SD_OP_SUB ? "-" : e.op == SD_OP_MUL ? "*" : "/";
        if (p.exprs[e.a].type != e.type || p.exprs[e.b].type != e.type)
          return fail(SD_ERR_INVALID, "arithmetic operands must be cast to the node type");
        if (type_is_fp(e.type)) {
          o << "    const " << T << " v" << N << " = " << V(e.a) << " " << sym << " " << V(e.b) << ";";
          if (e.op == SD_OP_DIV) o << " const bool n" << N << " = " << NL(e.a) << " || " << NL(e.b) << " || (" << V(e.b) << " == 0);\n";
          else o << " const bool n" << N << " = " << NL(e.a) << " || " << NL(e.b) << ";\n";
          return 0;
        }
        if (e.op == SD_OP_DIV) return fail(SD_ERR_UNSUPPORTED, "integral Divide (Catalyst casts it to double before it reaches the plan)");
        if (e.type == SD_STRING || e.type == SD_BOOLEAN || e.type == SD_DECIMAL) return fail(SD_ERR_UNSUPPORTED, "arithmetic on this type");
        const char* U = (e.type == SD_LONG || e.type == SD_TIMESTAMP) ? "uint64_t" : "uint32_t";
        o << "    const " << T << " v" << N << " = (" << T << ")((" << U << ")" << V(e.a) << " " << sym << " (" << U << ")" << V(e.b)
          << "); const bool n" << N << " = " << NL(e.a) << " || " << NL(e.b) << ";\n";
        return 0;
      }
      case SD_OP_NEG:
        if (type_is_fp(e.type)) o << "    const " << T << " v" << N << " = -" << V(e.a) << ";";
        else o << "    const " << T << " v" << N << " = (" << T << ")(0 - (uint64_t)" << V(e.a) << ");";
        o << " const bool n" << N << " = " << NL(e.a) << ";\n";
        return 0;
      case SD_OP_CAST: {   // Spark 2.1.1 Cast for the pairs listed in include/snappy_gpu.h; anything else is refused
        const int from = p.exprs[e.a].type, to = e.type;
        std::string v, extra_null;
        auto is_time = [](int t) { return t == SD_DATE || t == SD_TIMESTAMP; };
        auto pow10 = [](int k) { std::string r = "1"; for (int i = 0; i < k; i++) r += "0"; return r + "ll"; };
        if (from == SD_STRING || to == SD_STRING) return fail(SD_ERR_UNSUPPORTED, "casts involving STRING");
        if ((is_time(from) || is_time(to)) && from != to) return fail(SD_ERR_UNSUPPORTED, "casts involving DATE / TIMESTAMP (time-zone dependent in Spark)");
        if (wide) {   // DECIMAL(p1, s1) -> DECIMAL(p2 > 18, s2 >= s1) in 128 bits, NULL when it does not fit p2 digits
          const int ps0 = decimal_ps(p, e.a), ps1 = decimal_ps(p, node);
          const int up = (ps1 & 0xff) - (ps0 & 0xff), k = (ps1 >> 8) - up;
          const std::string a = "(sd::i128)" + V(e.a);
          o << "    const sd::i128 v" << N << " = (sd::i128)((unsigned __int128)" << a << " * (unsigned __int128)sd::p10w(" << up << ")); const bool n" << N
            << " = " << NL(e.a) << " || " << a << " >= sd::p10w(" << k << ") || " << a << " <= -sd::p10w(" << k << ");\n";
          return 0;
        }
        if (from == SD_DECIMAL || to == SD_DECIMAL) {
          if (from == SD_DECIMAL && type_is_fp(to)) {   // Decimal.toDouble: unscaled / 10^s
            const int sc = decimal_ps(p, e.a) & 0xff;
            v = std::string("(") + T + ")((double)" + V(e.a) + " / 1e" + std::to_string(sc) + ")";
          } else if (to == SD_DECIMAL && (from == SD_BYTE || from == SD_SHORT || from == SD_INT || from == SD_LONG)) {
            const int ps = decimal_ps(p, node), pr = ps >> 8, sc = ps & 0xff;   // v * 10^s, NULL when it needs more than p digits
            const std::string lim = pow10(pr - sc);
            v = "(int64_t)" + V(e.a) + " * " + pow10(sc);
            extra_null = " || (int64_t)" + V(e.a) + " >= " + lim + " || (int64_t)" + V(e.a) + " <= -" + lim;
          } else if (from == SD_DECIMAL && to == SD_DECIMAL) {
            const int ps0 = decimal_ps(p, e.a), ps1 = decimal_ps(p, node);
            const int up = (ps1 & 0xff) - (ps0 & 0xff);
            if (up < 0) return fail(SD_ERR_UNSUPPORTED, "DECIMAL cast that reduces the scale (needs HALF_UP rounding)");
            const std::string lim = pow10((ps1 >> 8) - up);
            v = V(e.a) + " * " + pow10(up);
            extra_null = " || " + V(e.a) + " >= " + lim + " || " + V(e.a) + " <= -" + lim;
          } else return fail(SD_ERR_UNSUPPORTED, "this cast to / from DECIMAL");
        }
        else if (to == SD_BOOLEAN) v = "(uint8_t)(" + V(e.a) + " != 0)";                       // castToBoolean: _ != 0
        else if (type_is_fp(from) && (to == SD_LONG)) v = "sd::f64_to_i64((double)" + V(e.a) + ")";
        else if (type_is_fp(from) && type_is_integral(to)) v = std::string("(") + T + ")sd::f64_to_i32((double)" + V(e.a) + ")";
        else v = std::string("(") + T + ")" + V(e.a);
        o << "    const " << T << " v" << N << " = " << v << "; const bool n" << N << " = " << NL(e.a) << extra_null << ";\n";
        if (to == SD_BOOLEAN) o << "    const int t" << N << " = n" << N << " ? 2 : (v" << N << " ? 1 : 0);\n";
        return 0;
      }
      case SD_OP_EQ: case SD_OP_NE: case SD_OP_LT: case SD_OP_LE: case SD_OP_GT: case SD_OP_GE:
      case SD_OP_IN: case SD_OP_STARTSWITH: {
        int col;
        if (string_predicate_col(p, node, &col)) {   // per-batch truth table indexed by the dictionary code
          int t;
          auto it = table_of_node.find(node);
          if (it == table_of_node.end()) {
            p.tables.push_back(TableSpec{TABLE_TRUTH, col, node, -1});
            t = (int)p.tables.size() - 1;
            table_of_node[node] = t;
          } else t = it->second;
          // dictionary batch: truth table indexed by the code.  Raw (variable-width) batch: compare the bytes on the device
          const std::string C = std::to_string(col), rec = "ctx.strbase[" + C + "] + (uint32_t)r.c" + C;
          const std::string rnull = p.cols[col].nullable ? "r.n" + C : std::string("false");
          auto lnull = [&](int slot) { return p.lit_nullable ? "(((ctx.L->nullmask >> " + std::to_string(slot) + ") & 1ull) != 0)" : std::string("false"); };
          std::string raw;
          if (is_cmp(e.op)) {
            const bool col_left = p.exprs[e.a].op == SD_OP_COL;
            const int slot = p.exprs[col_left ? e.b : e.a].a;
            int op = e.op;   // literal on the left: cmp(lit, col) = -cmp(col, lit)
            if (!col_left) op = op == SD_OP_LT ? SD_OP_GT : op == SD_OP_LE ? SD_OP_GE : op == SD_OP_GT ? SD_OP_LT : op == SD_OP_GE ? SD_OP_LE : op;
            const char* sym = op == SD_OP_EQ ? "==" : op == SD_OP_NE ? "!=" : op == SD_OP_LT ? "<" : op == SD_OP_LE ? "<=" : op == SD_OP_GT ? ">" : ">=";
            raw = "((" + rnull + " || " + lnull(slot) + ") ? 2 : (sd::str_cmp_rec(" + rec + ", ctx.lit_bytes(" + std::to_string(slot) + "), ctx.lit_len(" +
                  std::to_string(slot) + ")) " + sym + " 0 ? 1 : 0))";
          } else if (e.op == SD_OP_STARTSWITH) {
            const int slot = p.exprs[e.b].a;
            raw = "((" + rnull + " || " + lnull(slot) + ") ? 2 : (sd::str_starts_rec(" + rec + ", ctx.lit_bytes(" + std::to_string(slot) + "), ctx.lit_len(" +
                  std::to_string(slot) + ")) ? 1 : 0))";
          } else {   // IN: TRUE on a match, else NULL when a literal is NULL, else FALSE; NULL value -> NULL
            std::string any, anynull;
            for (int k = 0; k < e.c; k++) {
              const std::string S = std::to_string(e.b + k);
              any += std::string(k ? " || " : "") + "(!" + lnull(e.b + k) + " && sd::str_cmp_rec(" + rec + ", ctx.lit_bytes(" + S + "), ctx.lit_len(" + S + ")) == 0)";
              anynull += std::string(k ? " || " : "") + lnull(e.b + k);
            }
            raw = "(" + rnull + " ? 2 : ((" + any + ") ? 1 : ((" + anynull + ") ? 2 : 0)))";
          }
          o << "    const int t" << N << " = ctx.strbase[" << C << "] ? " << raw << " : (int)ctx.table(" << t << ")[r.c" << col << "];\n";
          finish_bool();
          return 0;
        }
        const int ot = p.exprs[e.a].type;
        if (ot == SD_STRING) return fail(SD_ERR_UNSUPPORTED, "string comparison that is not (dictionary column vs literal)");
        if (e.op == SD_OP_STARTSWITH) return fail(SD_ERR_UNSUPPORTED, "startsWith on a non-column operand");
        if (e.op == SD_OP_IN) {
          std::ostringstream any, anynull;
          for (int k = 0; k < e.c; k++) {
            const int s = e.b + k;
            std::string lv = type_is_fp(ot) ? std::string("(") + ctype_of(ot) + ")ctx.L->d[" + std::to_string(s) + "]"
                                            : std::string("(") + ctype_of(ot) + ")ctx.L->i[" + std::to_string(s) + "]";
            if (node_is_wide(p, e.a)) lv = "sd::dec_lit(ctx.lit_bytes(" + std::to_string(s) + "))";
            std::string nn = p.lit_nullable ? "(((ctx.L->nullmask >> " + std::to_string(s) + ") & 1ull) == 0)" : std::string("true");
            std::string eq = type_is_fp(ot) ? "sd::f_eq(" + V(e.a) + ", " + lv + ")" : "(" + V(e.a) + " == " + lv + ")";
            any << (k ? " || " : "") << "(" << nn << " && " << eq << ")";
            anynull << (k ? " || " : "") << "!" << nn;
          }
          o << "    const int t" << N << " = " << NL(e.a) << " ? 2 : ((" << any.str() << ") ? 1 : ((" << anynull.str() << ") ? 2 : 0));\n";
          finish_bool();
          return 0;
        }
        if (p.exprs[e.b].type != ot) return fail(SD_ERR_INVALID, "comparison operands must have the same type");
        if (ot == SD_DECIMAL && (decimal_ps(p, e.a) & 0xff) != (decimal_ps(p, e.b) & 0xff))
          return fail(SD_ERR_INVALID, "DECIMAL comparison operands must have the same scale (Catalyst casts them to a common type)");
        std::string c;
        if (type_is_fp(ot)) {
          const char* f = e.op == SD_OP_EQ ? "f_eq" : e.op == SD_OP_NE ? "f_eq" : e.op == SD_OP_LT ? "f_lt" : e.op == SD_OP_LE ? "f_le"
                        : e.op == SD_OP_GT ? "f_gt" : "f_ge";
          c = std::string(e.op == SD_OP_NE ? "!" : "") + "sd::" + f + "(" + V(e.a) + ", " + V(e.b) + ")";
        } else {
          const char* sym = e.op == SD_OP_EQ ? "==" : e.op == SD_OP_NE ? "!=" : e.op == SD_OP_LT ? "<" : e.op == SD_OP_LE ? "<="
                          : e.op == SD_OP_GT ? ">" : ">=";
          c = "(" + V(e.a) + " " + sym + " " + V(e.b) + ")";
        }
        o << "    const int t" << N << " = (" << NL(e.a) << " || " << NL(e.b) << ") ? 2 : (" << c << " ? 1 : 0);\n";
        finish_bool();
        return 0;
      }
      case SD_OP_AND: case SD_OP_OR:
        if (p.exprs[e.a].type != SD_BOOLEAN || p.exprs[e.b].type != SD_BOOLEAN) return fail(SD_ERR_INVALID, "AND/OR over non-boolean operands");
        o << "    const int t" << N << " = sd::" << (e.op == SD_OP_AND ? "tv_and" : "tv_or") << "(t" << e.a << ", t" << e.b << ");\n";
        finish_bool();
        return 0;
      case SD_OP_NOT:
        if (p.exprs[e.a].type != SD_BOOLEAN) return fail(SD_ERR_INVALID, "NOT over a non-boolean operand");
        o << "    const int t" << N << " = sd::tv_not(t" << e.a << ");\n";
        finish_bool();
        return 0;
      case SD_OP_ISNULL: case SD_OP_ISNOTNULL:
        o << "    const int t" << N << " = " << NL(e.a) << (e.op == SD_OP_ISNULL ? " ? 1 : 0;\n" : " ? 0 : 1;\n");
        finish_bool();
        return 0;
      case SD_OP_PAIR:   // x as its value; the slots read y from child b (GATE_PAIR_Y)
        o << "    const double v" << N << " = " << V(e.a) << "; const bool n" << N << " = " << NL(e.a) << " || " << NL(e.b) << ";\n";
        return 0;
    }
    return fail(SD_ERR_INVALID, "unknown expression operator");
  }

  int generate() {
    std::ostringstream sig;
    sig << "v2;cols=";
    for (size_t c = 0; c < p.cols.size(); c++) sig << (c ? "," : "") << p.kinds[c] << (p.cols[c].nullable ? "n" : "");
    sig << ";filter=" << (p.filter >= 0 ? expr_text(p, p.filter) : std::string("-")) << ";keys=";
    for (size_t k = 0; k < p.keys.size(); k++) sig << (k ? "," : "") << expr_text(p, p.keys[k]);

    // ---- bodies ---------------------------------------------------------------------------------
    std::ostringstream filt, grp, slt;
    std::vector<char> done(p.exprs.size(), 0);
    if (p.filter >= 0) {
      int rc = emit_node(p.filter, done, filt);
      if (rc) return rc;
      filt << "    return t" << p.filter << " == 1;\n";
    } else filt << "    return true;\n";

    if (p.mode == MODE_GROUPS) {
      std::fill(done.begin(), done.end(), 0);
      keymap_table.clear();
      std::string g;
      for (size_t k = 0; k < p.keys.size(); k++) {
        const sd_expr& e = p.exprs[p.keys[k]];
        if (!(e.op == SD_OP_COL && e.type == SD_STRING))
          return fail(SD_ERR_UNSUPPORTED, "GPU group-by currently needs dictionary-encoded STRING key columns");
        p.tables.push_back(TableSpec{TABLE_KEYMAP, e.a, -1, (int)k});
        const int t = (int)p.tables.size() - 1;
        keymap_table.push_back(t);
        std::string term = "ctx.key_id(" + std::to_string(t) + ", r.c" + std::to_string(e.a) + ")";
        g = k == 0 ? term : "(" + g + ") * ctx.radix[" + std::to_string(k) + "] + " + term;
      }
      grp << "    return " << g << ";\n";
    } else grp << "    return 0;\n";
    std::ostringstream projfn;
    if (p.mode == MODE_PROJECT || p.mode == MODE_MUTATE) {   // MODE_MUTATE: the SET values of an UPDATE (none for a DELETE)
      std::fill(done.begin(), done.end(), 0);
      sig << ";proj=";
      for (size_t j = 0; j < p.proj.size(); j++) {
        const sd_expr& e = p.exprs[p.proj[j]];
        sig << (j ? "," : "") << expr_text(p, p.proj[j]);
        if (node_is_wide(p, p.proj[j])) {   // a wide DECIMAL column: the device address of its record (the host reads the bytes)
          const std::string C = std::to_string(e.a);
          projfn << "    pv[" << j << "] = (uint64_t)(uintptr_t)(ctx.strbase[" << C << "] + (uint32_t)r.c" << C << ");";
          if (p.cols[e.a].nullable) projfn << " if (r.n" << C << ") pnull |= " << (1u << j) << "u;";
          projfn << "\n";
          continue;
        }
        int rc = emit_node(p.proj[j], done, projfn);
        if (rc) return rc;
        const std::string N = std::to_string(p.proj[j]);
        projfn << "    pv[" << j << "] = " << (type_is_fp(e.type) ? "sd::f2u((double)v" + N + ")" : "(uint64_t)(int64_t)v" + N)
               << "; if (n" << N << ") pnull |= " << (1u << j) << "u;\n";
      }
    }
    std::ostringstream keyfn;
    uint32_t strkeymask = 0;
    if (p.mode == MODE_HASH) {
      std::fill(done.begin(), done.end(), 0);
      for (size_t k = 0; k < p.keys.size(); k++) {
        const sd_expr& e = p.exprs[p.keys[k]];
        if (e.op == SD_OP_COL && e.type == SD_STRING) {   // held by reference: address of the value's [len][bytes] record
          p.tables.push_back(TableSpec{TABLE_KEYPTR, e.a, -1, (int)k});
          const int t = (int)p.tables.size() - 1;
          strkeymask |= 1u << k;
          if (p.cols[e.a].nullable) keyfn << "    if (r.n" << e.a << ") { knull |= " << (1u << k) << "u; kc[" << k << "] = 0; } else";
          keyfn << "    kc[" << k << "] = ctx.str_ref(" << e.a << ", " << t << ", r.c" << e.a << ");\n";
        } else if (node_is_wide(p, p.keys[k])) {   // by reference like a string: equal values have identical bytes
          strkeymask |= 1u << k;
          if (p.cols[e.a].nullable) keyfn << "    if (r.n" << e.a << ") { knull |= " << (1u << k) << "u; kc[" << k << "] = 0; } else";
          keyfn << "    kc[" << k << "] = (int64_t)(uintptr_t)(ctx.strbase[" << e.a << "] + (uint32_t)r.c" << e.a << ");\n";
        } else {
          int rc = emit_node(p.keys[k], done, keyfn);
          if (rc) return rc;
          const std::string N = std::to_string(p.keys[k]);
          if (type_is_fp(e.type))   // NaN-safe key equality: one NaN, -0.0 == 0.0 (SURVEY.md Appendix B.5)
            keyfn << "    { double d = (double)v" << N << "; if (d == 0.0) d = 0.0; kc[" << k << "] = n" << N
                  << " ? 0 : ((d != d) ? 0x7ff8000000000000ll : __double_as_longlong(d)); }";
          else
            keyfn << "    kc[" << k << "] = n" << N << " ? 0 : (int64_t)v" << N << ";";
          keyfn << " if (n" << N << ") knull |= " << (1u << k) << "u;\n";
        }
      }
    }

    std::fill(done.begin(), done.end(), 0);
    sig << ";slots=";
    for (size_t s = 0; s < p.slots.size(); s++) {
      const SlotSpec& x = p.slots[s];
      sig << (s ? "," : "") << x.op << "/" << x.gate << "/" << (x.node >= 0 ? expr_text(p, x.node) : std::string("-"));
      const bool order_gate = x.gate == GATE_ORDER_KEY || x.gate == GATE_ORDER_KEY_IGN || x.gate == GATE_ORDER_VAL;
      const bool by_ref = x.node >= 0 && (x.gate == GATE_DECREF || (order_gate && node_is_wide(p, x.node)));   // record address, not value
      if (x.node >= 0 && !by_ref) { int rc = emit_node(x.node, done, slt); if (rc) return rc; }
      const std::string V = "v" + std::to_string(x.node), NL = "n" + std::to_string(x.node);
      slt << "    sv[" << s << "] = ";
      if (x.gate == GATE_ONE) slt << "1ull;\n";
      else if (x.gate == GATE_NONNULL_COUNT) slt << NL << " ? 0ull : 1ull;\n";
      else if (x.gate == GATE_STRREF) {
        const int col = p.exprs[x.node].a;
        slt << NL << " ? 0ull : (uint64_t)ctx.str_ref(" << col << ", " << x.table << ", r.c" << col << ");\n";
      }
      else if (x.gate == GATE_DECREF) {
        const std::string C = std::to_string(p.exprs[x.node].a);
        slt << (p.cols[p.exprs[x.node].a].nullable ? "r.n" + C : std::string("false")) << " ? 0ull : (uint64_t)(uintptr_t)(ctx.strbase[" << C << "] + (uint32_t)r.c" << C << ");\n";
      }
      else if (x.gate == GATE_LIMB3) slt << NL << " ? 0ull : (uint64_t)(int64_t)(" << V << " >> 96);\n";
      else if (x.gate >= GATE_LIMB0 && x.gate <= GATE_LIMB2)
        slt << NL << " ? 0ull : (uint64_t)(uint32_t)((unsigned __int128)" << V << " >> " << 32 * (x.gate - GATE_LIMB0) << ");\n";
      else if (x.gate == GATE_VALUE_HI32) slt << NL << " ? 0ull : (uint64_t)((int64_t)" << V << " >> 32);\n";
      else if (x.gate == GATE_VALUE_LO32) slt << NL << " ? 0ull : ((uint64_t)(int64_t)" << V << " & 0xffffffffull);\n";
      else if (x.gate == GATE_POW1) slt << NL << " ? sd::SHIFT_EMPTY : sd::shift_cand((double)" << V << ");\n";
      else if (x.gate >= GATE_POW2 && x.gate <= GATE_POW4) slt << "0ull;\n";
      else if (x.gate == GATE_PAIR_X) slt << NL << " ? sd::SHIFT_EMPTY : sd::shift_cand(" << V << ");\n";
      else if (x.gate == GATE_PAIR_Y) slt << NL << " ? sd::SHIFT_EMPTY : sd::shift_cand(v" << p.exprs[x.node].b << ");\n";
      else if (x.gate >= GATE_PAIR_XY && x.gate <= GATE_PAIR_YY) slt << "0ull;\n";
      else if (x.gate == GATE_PAD) slt << "0ull;\n";
      else if (order_gate) {
        const int col = p.exprs[x.node].a;
        const std::string C = std::to_string(col);
        const std::string isnull = by_ref ? (p.cols[col].nullable ? "r.n" + C : std::string("false")) : NL;
        if (x.gate == GATE_ORDER_KEY) slt << "ctx.ord | (" << isnull << " ? 1ull : 0ull);\n";
        else if (x.gate == GATE_ORDER_KEY_IGN) slt << isnull << " ? " << (x.op == SLOT_FIRST ? "0xffffffffffffffffull" : "0ull") << " : ctx.ord;\n";
        else if (by_ref) slt << isnull << " ? 0ull : (uint64_t)(uintptr_t)(ctx.strbase[" << C << "] + (uint32_t)r.c" << C << ");\n";
        else if (p.exprs[x.node].type == SD_STRING) slt << isnull << " ? 0ull : (uint64_t)ctx.str_ref(" << C << ", " << x.table << ", r.c" << C << ");\n";
        else slt << isnull << " ? 0ull : " << (type_is_fp(p.exprs[x.node].type) ? "sd::f2u((double)" + V + ")" : "(uint64_t)(int64_t)" + V) << ";\n";
      }
      else {
        const bool f = x.op == SLOT_ADD_F64 || x.op == SLOT_MIN_F64 || x.op == SLOT_MAX_F64;
        char ident[32];
        snprintf(ident, sizeof(ident), "0x%llxull", (unsigned long long)(
            x.op == SLOT_ADD_F64 || x.op == SLOT_ADD_I64 ? 0ull : x.op == SLOT_MIN_I64 ? 0x7fffffffffffffffull
          : x.op == SLOT_MAX_I64 ? 0x8000000000000000ull : x.op == SLOT_MIN_F64 ? 0x7ff8000000000000ull : 0xfff0000000000000ull));
        slt << NL << " ? " << ident << " : " << (f ? "sd::f2u((double)" + V + ")" : "(uint64_t)(int64_t)" + V) << ";\n";
      }
    }
    if ((int)p.tables.size() > MAX_TABLES) return fail(SD_ERR_UNSUPPORTED, "more than 40 dictionary lookup tables in one plan");
    sig << ";mode=" << p.mode << ";tables=" << p.tables.size() << ";rpt=" << p.rpt << ";minctas=" << p.min_ctas << ";staged=" << (p.stages > 0 ? 1 : 0) << ";reggroups=" << p.reg_groups << ";litnull=" << p.lit_nullable << ";slow=" << p.slow_paths;
    if (const char* e = getenv("SD_JIT_DEFINES")) sig << ";defines=" << e;   // experiment switches compile (and cache) as distinct kernels
    p.signature = sig.str();
    char hbuf[32];
    snprintf(hbuf, sizeof(hbuf), "%016llx", (unsigned long long)std::hash<std::string>()(p.signature));
    // std::hash is not stable across libstdc++ builds: use FNV-1a for a reproducible name
    unsigned long long h = 1469598103934665603ull;
    for (unsigned char ch : p.signature) { h ^= ch; h *= 1099511628211ull; }
    snprintf(hbuf, sizeof(hbuf), "%016llx", h);
    p.struct_name = std::string("Plan_") + hbuf;

    // ---- the struct --------------------------------------------------------------------------------
    std::ostringstream o;
    const int nc = (int)p.cols.size(), ns = (int)p.slots.size();
    o << "// signature: " << p.signature << "\n";
    o << "struct " << p.struct_name << " {\n";
    o << "  static constexpr int NC = " << nc << ";\n  static constexpr int NSLOT = " << ns << ";\n";
    o << "  static constexpr int MODE = " << (p.mode == MODE_GROUPS ? "sd::MODE_GROUPS" : p.mode == MODE_HASH ? "sd::MODE_HASH" : p.mode == MODE_PROJECT ? "sd::MODE_PROJECT" : p.mode == MODE_MUTATE ? "sd::MODE_MUTATE" : "sd::MODE_NOKEY") << ";\n";
    o << "  static constexpr int NKEYS = " << p.keys.size() << ";\n";
    o << "  static constexpr int NPROJ = " << p.proj.size() << ";\n";
    o << "  static constexpr int MIN_CTAS = " << p.min_ctas << ";\n  static constexpr int RPT = " << p.rpt << ";\n";
    o << "  static constexpr int STAGES = " << (p.stages > 0 ? 1 : 0) << ";\n";
    o << "  static constexpr int REG_GROUPS = " << p.reg_groups << ";\n";
    o << "  static constexpr bool SLOW_PATHS = " << (p.slow_paths ? "true" : "false") << ";\n";
    o << "  static constexpr int NTABLES = " << p.tables.size() << ";\n";
    o << "  static constexpr unsigned STRKEYMASK = " << strkeymask << "u;\n";
    for (auto& x : p.slots)
      if (x.op == SLOT_MIN_DEC || x.op == SLOT_MAX_DEC) {   // slot_combine compares these by value only with 128-bit integers
        o << "  static_assert(sd::HAVE_I128, \"MIN / MAX of a wide DECIMAL needs 128-bit integers (NVRTC -device-int128)\");\n";
        break;
      }
    { bool anys = false; for (auto& c : p.cols) anys = anys || c.type == SD_STRING || wide_decimal(c.type, c.precision); o << "  static constexpr bool ANY_STRING = " << (anys ? "true" : "false") << ";\n"; }
    o << "  __host__ __device__ static constexpr int kind(int c) { return ";
    for (int c = 0; c < nc; c++) o << "c == " << c << " ? " << p.kinds[c] << " : ";
    o << "0; }\n";
    {   // columns the plan declares nullable: only those carry the NULL-aware staged path
      bool any = false;
      o << "  __host__ __device__ static constexpr bool col_nullable(int c) { return ";
      for (int c = 0; c < nc; c++) { if (p.cols[c].nullable) { o << "c == " << c << " || "; any = true; } }
      o << "false; }\n";
      o << "  static constexpr bool ANY_NULLABLE = " << (any ? "true" : "false") << ";\n";
    }
    o << "  __host__ __device__ static constexpr int slot_op(int s) { return ";
    for (int s = 0; s < ns; s++) o << "s == " << s << " ? " << p.slots[s].op << " : ";
    o << "0; }\n";
    o << "  __device__ static __forceinline__ int slot_op_rt(int s) { return slot_op(s); }\n";
    if (!p.shifts.empty()) {   // moment aggregates (sd_kernels.cuh apply_shifts)
      const int nsh = (int)p.shifts.size();
      o << "  static constexpr int NSHIFT = " << nsh << ";\n";
      o << "  __host__ __device__ static constexpr int order(int i) { return ";
      for (int i = 0; i < nsh; i++) o << "i == " << i << " ? " << p.shifts[i].order << " : ";
      o << "0; }\n";
      o << "  __host__ __device__ static constexpr int pow_slot(int i, int j) { return ";
      for (int i = 0; i < nsh; i++)
        for (int j = 1; j <= p.shifts[i].order; j++) o << "(i == " << i << " && j == " << j << ") ? " << p.shifts[i].pow_slot[j - 1] << " : ";
      o << "0; }\n";
    }
    if (p.norder > 0) o << "  static constexpr int NORDER = " << p.norder << ";\n";   // FIRST / LAST pairs (sd_kernels.cuh PlanOrders)
    if (!p.pairs.empty()) {   // two-input aggregates: S_xy of shifts (x, y) (sd_kernels.cuh apply_shifts)
      const int np = (int)p.pairs.size();
      o << "  static constexpr int NPAIR = " << np << ";\n";
      o << "  __host__ __device__ static constexpr int pair_shift(int q, int v) { return ";
      for (int q = 0; q < np; q++) o << "(q == " << q << ") ? (v ? " << p.pairs[q].shift_y << " : " << p.pairs[q].shift_x << ") : ";
      o << "0; }\n";
      o << "  __host__ __device__ static constexpr int pair_slot(int q) { return ";
      for (int q = 0; q < np; q++) o << "q == " << q << " ? " << p.pairs[q].xy_slot << " : ";
      o << "0; }\n";
    }
    o << "  struct Row {\n";
    for (int c = 0; c < nc; c++) o << "    " << col_ctype(p.cols[c]) << " c" << c << "; bool n" << c << ";\n";
    o << "    template <int C, class T> __device__ __forceinline__ void set(T v, bool isnull) {\n";
    for (int c = 0; c < nc; c++) o << "      if (C == " << c << ") { c" << c << " = (" << col_ctype(p.cols[c]) << ")v; n" << c << " = isnull; }\n";
    o << "    }\n  };\n";
    o << "  __device__ static __forceinline__ bool filter(const Row& r, const sd::RowCtx& ctx) {\n" << filt.str() << "  }\n";
    o << "  __device__ static __forceinline__ int group(const Row& r, const sd::RowCtx& ctx) {\n" << grp.str() << "  }\n";
    o << "  __device__ static __forceinline__ void project(const Row& r, const sd::RowCtx& ctx, uint64_t* pv, uint32_t& pnull) {\n" << projfn.str() << "  }\n";
    o << "  __device__ static __forceinline__ void keys(const Row& r, const sd::RowCtx& ctx, int64_t* kc, uint32_t& knull) {\n" << keyfn.str() << "  }\n";
    o << "  __device__ static __forceinline__ void slots(const Row& r, const sd::RowCtx& ctx, uint64_t* sv) {\n" << slt.str() << "  }\n";
    o << "};\n";
    p.source = o.str();
    return 0;
  }
};

}  // namespace

int analyze_plan(const sd_plan_desc* d, PlanSpec& out, std::string& err, const CodegenOptions* opt) {
  if (!d) { err = "null plan descriptor"; return SD_ERR_INVALID; }
  if (d->abi_version != SD_ABI_VERSION) { err = "sd_plan_desc.abi_version mismatch"; return SD_ERR_INVALID; }
  if (d->ncols < 0 || d->nexprs < 0 || d->nkeys < 0 || d->naggs < 0 || d->nproj < 0 || d->nliterals < 0) {
    err = "negative count in plan descriptor"; return SD_ERR_INVALID;
  }
  out = PlanSpec();
  out.cols.assign(d->cols, d->cols + d->ncols);
  out.exprs.assign(d->exprs, d->exprs + d->nexprs);
  out.keys.assign(d->keys, d->keys + d->nkeys);
  out.desc_keys = out.keys;
  out.aggs.assign(d->aggs, d->aggs + d->naggs);
  out.proj.assign(d->proj, d->proj + d->nproj);
  out.literal_types.assign(d->literal_types, d->literal_types + d->nliterals);
  out.filter = d->filter;
  const bool mutate = (d->flags & SD_PLAN_MUTATE) != 0;
  out.flags = mutate ? SD_PLAN_MUTATE : 0;
  Gen g(out, err);
  int rc = g.grouping_sets();
  if (rc) return rc;
  rc = g.validate();
  if (rc) return rc;
  for (auto& c : out.cols) out.kinds.push_back(kind_of_column(c));
  out.lit_wide.assign(out.literal_types.size(), 0);   // slots read by a wide LIT node or listed by an IN over a wide operand
  for (size_t i = 0; i < out.exprs.size(); i++) {
    const sd_expr& e = out.exprs[i];
    if (e.op == SD_OP_LIT && node_is_wide(out, (int)i)) out.lit_wide[(size_t)e.a] = 1;
    if (e.op == SD_OP_IN && node_is_wide(out, e.a)) for (int k = 0; k < e.c; k++) out.lit_wide[(size_t)(e.b + k)] = 1;
  }
  g.nullability();
  const bool projection = out.aggs.empty() && out.keys.empty();
  if (mutate && !projection) { err = "an UPDATE / DELETE plan has no grouping keys and no aggregates"; return SD_ERR_INVALID; }
  if (projection && out.proj.empty() && !mutate) { err = "plan has neither aggregates nor projection columns"; return SD_ERR_INVALID; }
  if (projection) {
    if (out.proj.size() > 32) { err = "more than 32 projected columns"; return SD_ERR_UNSUPPORTED; }
    for (int n : out.proj) {
      const sd_expr& e = out.exprs[n];
      if (e.type == SD_STRING && e.op != SD_OP_COL) { err = "projected STRING expression that is not a dictionary column"; return SD_ERR_UNSUPPORTED; }
      if (node_is_wide(out, n) && mutate) { err = "UPDATE with a SET value that is a DECIMAL wider than 18 digits"; return SD_ERR_UNSUPPORTED; }
      if (node_is_wide(out, n) && e.op != SD_OP_COL) { err = "projected wide DECIMAL expression that is not a column"; return SD_ERR_UNSUPPORTED; }
    }
  }
  out.mode = mutate ? MODE_MUTATE : projection ? MODE_PROJECT : MODE_NOKEY;
  if (!out.keys.empty()) {
    bool all_dict_strings = true;
    for (int k : out.keys) {
      const sd_expr& e = out.exprs[k];
      if (!(e.op == SD_OP_COL && e.type == SD_STRING)) all_dict_strings = false;
      if (e.type == SD_STRING && e.op != SD_OP_COL) { err = "STRING group key that is not a dictionary column"; return SD_ERR_UNSUPPORTED; }
      if (node_is_wide(out, k) && e.op != SD_OP_COL) { err = "wide DECIMAL group key that is not a column"; return SD_ERR_UNSUPPORTED; }
    }
    // dense table: <= 4 dictionary-string keys; anything else (other key types, more keys) goes through the hash table
    out.mode = (all_dict_strings && (int)out.keys.size() <= MAX_KEYS && !(opt && opt->force_hash)) ? MODE_GROUPS : MODE_HASH;
  }
  // kernel shape (see tools/sweep.sh for the measurements behind the defaults): staged fast path on;
  // 4 rows per thread per tile; narrow no-key scans run 3 CTAs per SM, register-table group-bys 1.
  {
    int row_bytes = 0;
    for (int k : out.kinds) row_bytes += kind_stage_width(k);
    CodegenOptions o;
    if (opt) o = *opt;
    out.reg_groups = out.mode == MODE_GROUPS ? std::max(0, o.reg_groups) : 0;
    out.lit_nullable = o.lit_nullable ? 1 : 0;
    out.slow_paths = o.slow_paths ? 1 : 0;
    out.rpt = 4;
    // group tables want the SM's shared memory; otherwise 2 CTAs per SM (H100 sweep, DESIGN.md section 5: Q6 at 2 is level
    // with 1 and ahead of 3), 3 only for very narrow rows whose tiles are too small to keep enough bytes in flight
    out.min_ctas = out.mode == MODE_GROUPS ? 1 : (row_bytes <= 8 ? 3 : 2);
    out.stages = 1;
    if (const char* e = getenv("SD_TUNE_RPT")) { int v = atoi(e); if (v == 2 || v == 4 || v == 8) out.rpt = v; }
    if (const char* e = getenv("SD_TUNE_MIN_CTAS")) { int v = atoi(e); if (v >= 1 && v <= 8) out.min_ctas = v; }
    if (const char* e = getenv("SD_TUNE_STAGES")) out.stages = atoi(e) > 0 ? 1 : 0;
    if (o.rpt == 2 || o.rpt == 4 || o.rpt == 8) out.rpt = o.rpt;
    if (o.min_ctas >= 1) out.min_ctas = o.min_ctas;
    if (o.stages >= 0) out.stages = o.stages > 0 ? 1 : 0;
    // a stage of the ring holds THREADS * RPT rows of every scan column (+ 128 bytes of alignment slack each): very wide
    // plans first halve the tile, then give the ring up for direct vector loads (the ring needs >= 2 stages in ~200 KB)
    auto stage_bytes = [&](int rpt) { return (size_t)THREADS * rpt * row_bytes + (size_t)128 * out.kinds.size(); };
    const size_t ring_budget = size_t(200) << 10;
    if (out.stages && 2 * stage_bytes(out.rpt) + (size_t)tile_smem_bytes((int)out.kinds.size(), out.rpt) > ring_budget && out.rpt > 2) out.rpt = 2;
    if (out.stages && 2 * stage_bytes(out.rpt) + (size_t)tile_smem_bytes((int)out.kinds.size(), out.rpt) > ring_budget) out.stages = 0;
    if (out.stages == 0) out.reg_groups = 0;   // the register tables are reduced through the ring's memory
  }
  if (!projection) { rc = g.build_slots(); if (rc) return rc; }
  if (!out.sets.empty() && out.shifts.size() > (size_t)ROLLUP_MAX_SHIFTS) {
    err = "grouping sets over more than 16 moment / covariance shifts";
    return SD_ERR_UNSUPPORTED;
  }
  if (!out.shifts.empty()) out.reg_groups = 0;   // register tables would need a K lookup per row and group: never built for them
  if (out.norder > 0) out.reg_groups = 0;        // nor for FIRST / LAST pairs
  return g.generate();
}

}  // namespace sd

// ---- C entry point: generated source + signature of a plan (build step, debugging, profiling) ------
extern "C" int sd_plan_codegen(const sd_plan_desc* desc, char* source, int64_t source_cap, int64_t* source_len,
                               char* signature, int64_t sig_cap, char* struct_name, int64_t name_cap, int32_t reg_groups,
                               int32_t lit_nullable, int32_t slow_paths) {
  sd::PlanSpec spec;
  std::string err;
  sd::CodegenOptions opt;
  opt.reg_groups = reg_groups;
  opt.lit_nullable = lit_nullable;
  opt.slow_paths = slow_paths;
  int rc = sd::analyze_plan(desc, spec, err, &opt);
  if (rc) {
    if (source && source_cap > 0) snprintf(source, (size_t)source_cap, "%s", err.c_str());
    return rc;
  }
  if (source_len) *source_len = (int64_t)spec.source.size();
  if ((int64_t)spec.source.size() + 1 > source_cap || (int64_t)spec.signature.size() + 1 > sig_cap ||
      (int64_t)spec.struct_name.size() + 1 > name_cap)
    return SD_ERR_OVERFLOW;
  memcpy(source, spec.source.c_str(), spec.source.size() + 1);
  memcpy(signature, spec.signature.c_str(), spec.signature.size() + 1);
  memcpy(struct_name, spec.struct_name.c_str(), spec.struct_name.size() + 1);
  return 0;
}
