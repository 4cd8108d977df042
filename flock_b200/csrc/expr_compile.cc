// expr_compile.cc -- lowers postfix PhysicalExpr programs (include/flockgpu.h: flockgpu_expr) to the
// term/chain programs of expr_program.h.
//
// The shapes follow what DataFusion's planner emits for the reference's queries: type coercion is
// already explicit (cast_expr / try_cast_expr nodes, flock/src/tests/data/plan/aggregate.json
// "predicate"; "CAST(auction@0 AS Int64) % 123 = 0", flock/src/distributed_plan/planner.rs:122), so
// both sides of a binary_expr normally carry the same type.  Where a caller of the C ABI omits the
// casts, the usual numeric promotion (Float64 > 64-bit ints > Int32) is applied.
#include "expr_compile.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <functional>
#include <map>
#include <set>

namespace fg {

namespace {

struct Node {
  int op = 0;
  int dtype = 0;  // result type
  int col = -1;
  int64_t i = 0;
  double d = 0;
  std::string s;
  int l = -1, r = -1;
  std::vector<int> kids;  // CASE: [base] (when, then)... [else]; IN_LIST: value, literals...
  int flags = 0;          // CASE: FLOCKGPU_CASE_HAS_*; IN_LIST: 1 = NOT IN
};

bool is_arith(int op) { return op >= FLOCKGPU_OP_ADD && op <= FLOCKGPU_OP_MOD; }
bool is_cmp(int op) { return op >= FLOCKGPU_OP_EQ && op <= FLOCKGPU_OP_GE; }
bool is_literal(const Node& n) { return n.op == FLOCKGPU_OP_LIT_I64 || n.op == FLOCKGPU_OP_LIT_F64 || n.op == FLOCKGPU_OP_LIT_UTF8; }
bool is_intlike(int dt) {
  return dt == FLOCKGPU_INT32 || dt == FLOCKGPU_INT64 || dt == FLOCKGPU_TIMESTAMP || dt == FLOCKGPU_UINT32 || dt == FLOCKGPU_UINT64;
}
bool is_unsigned(int dt) { return dt == FLOCKGPU_UINT32 || dt == FLOCKGPU_UINT64; }
bool is_numeric(int dt) { return is_intlike(dt) || dt == FLOCKGPU_FLOAT64; }
// Date32 is neither: it compares with Date32 only and takes part in no arithmetic or cast, and is lowered as Int32 is
bool same_ordered(int a, int b) { return a == b && (a == FLOCKGPU_UTF8 || a == FLOCKGPU_DATE32); }
bool is_i32(int dt) { return dt == FLOCKGPU_INT32 || dt == FLOCKGPU_DATE32; }

int promote(int a, int b) {
  if (a == b) return a;
  if (a == FLOCKGPU_FLOAT64 || b == FLOCKGPU_FLOAT64) return FLOCKGPU_FLOAT64;
  auto rank = [](int t) {
    switch (t) {
      case FLOCKGPU_INT32: return 1;
      case FLOCKGPU_UINT32: return 2;
      case FLOCKGPU_INT64: case FLOCKGPU_TIMESTAMP: return 3;
      default: return 4;  // UInt64
    }
  };
  return rank(a) >= rank(b) ? a : b;
}

// A CAST from `from` to `to` that some source value does not survive (cast_fits): Float64 to an integer type, an
// integer type to a narrower one or across signedness.  The tree form gives NULL for the values that do not fit.  The
// chain form has no NULLs of its own: compile_value and compile_predicate refuse an expression that holds one, and the
// operators evaluate it in the tree form.
bool lossy_cast(int from, int to) {
  if (from == to || to == FLOCKGPU_FLOAT64) return false;
  if (from == FLOCKGPU_FLOAT64) return true;
  if (to == FLOCKGPU_INT32 || to == FLOCKGPU_UINT32) return true;
  return to == FLOCKGPU_UINT64 ? !is_unsigned(from) : from == FLOCKGPU_UINT64;
}

struct Tree {
  std::vector<Node> nodes;
  int root = -1;
};

bool has_lossy_cast(const Tree& t) {
  for (const Node& n : t.nodes)
    if (n.op == FLOCKGPU_OP_CAST && lossy_cast(t.nodes[n.l].dtype, n.dtype)) return true;
  return false;
}

// The unit of date_part's Timestamp operand `idx`: that of the first Timestamp column it reads, as compile_value keeps
// the format of a computed Timestamp.  A timezone, or no Timestamp column at all (a literal), is refused.
int timestamp_unit(const Tree& t, int idx, const std::vector<ColInfo>& cols) {
  std::function<int(int)> first = [&](int i) -> int {
    if (i < 0) return -1;
    const Node& x = t.nodes[i];
    if (x.op == FLOCKGPU_OP_COLUMN) return x.dtype == FLOCKGPU_TIMESTAMP ? x.col : -1;
    for (int k : {x.l, x.r})
      if (int c = first(k); c >= 0) return c;
    for (int k : x.kids)
      if (int c = first(k); c >= 0) return c;
    return -1;
  };
  const int c = first(idx);
  FG_CHECK(c >= 0, FLOCKGPU_ERR_UNSUPPORTED, "expression: date_part of a Timestamp that reads no Timestamp column (its unit is unknown)");
  const std::string& f = cols[c].format;  // "ts" + unit letter + ':' + timezone
  FG_CHECK(f.size() >= 4 && f.compare(0, 2, "ts") == 0 && f[3] == ':', FLOCKGPU_ERR_INVALID, "expression: Timestamp column \"%s\" has format \"%s\"",
           cols[c].name.c_str(), f.c_str());
  FG_CHECK(f.size() == 4, FLOCKGPU_ERR_UNSUPPORTED, "expression: date_part of Timestamp with timezone %s (column \"%s\")", f.c_str() + 4,
           cols[c].name.c_str());
  switch (f[2]) {
    case 's': return DU_S;
    case 'm': return DU_MS;
    case 'u': return DU_US;
    case 'n': return DU_NS;
  }
  fail(FLOCKGPU_ERR_INVALID, "expression: Timestamp column \"%s\" has format \"%s\"", cols[c].name.c_str(), f.c_str());
}

Tree build_tree(const Expr& e, const std::vector<ColInfo>& cols) {
  Tree t;
  std::vector<int> stack;
  auto pop = [&]() {
    FG_CHECK(!stack.empty(), FLOCKGPU_ERR_INVALID, "expression: stack underflow (malformed postfix program)");
    int v = stack.back();
    stack.pop_back();
    return v;
  };
  for (const ExprTok& tok : e) {
    Node n;
    n.op = tok.op;
    switch (tok.op) {
      case FLOCKGPU_OP_COLUMN:
        FG_CHECK(tok.col >= 0 && tok.col < int(cols.size()), FLOCKGPU_ERR_INVALID, "expression: column index %d out of range (%zu columns)",
                 tok.col, cols.size());
        n.col = tok.col;
        n.dtype = cols[tok.col].dtype;
        break;
      case FLOCKGPU_OP_LIT_I64:
        n.i = tok.i64;
        n.dtype = (tok.dtype == FLOCKGPU_INT32 || tok.dtype == FLOCKGPU_UINT32 || tok.dtype == FLOCKGPU_UINT64 ||
                   tok.dtype == FLOCKGPU_TIMESTAMP || tok.dtype == FLOCKGPU_DATE32)
                      ? tok.dtype
                      : FLOCKGPU_INT64;
        break;
      case FLOCKGPU_OP_LIT_F64:
        n.d = tok.f64;
        n.dtype = FLOCKGPU_FLOAT64;
        break;
      case FLOCKGPU_OP_LIT_UTF8:
        n.s = tok.str;
        n.dtype = FLOCKGPU_UTF8;
        break;
      case FLOCKGPU_OP_CAST:
        n.l = pop();
        n.dtype = tok.dtype;
        FG_CHECK(is_numeric(n.dtype) && is_numeric(t.nodes[n.l].dtype), FLOCKGPU_ERR_UNSUPPORTED, "expression: CAST from %s to %s",
                 dtype_name(t.nodes[n.l].dtype), dtype_name(n.dtype));
        break;
      case FLOCKGPU_OP_NOT:
        n.l = pop();
        n.dtype = FLOCKGPU_BOOL;
        FG_CHECK(t.nodes[n.l].dtype == FLOCKGPU_BOOL, FLOCKGPU_ERR_INVALID, "expression: NOT of a non-boolean");
        break;
      case FLOCKGPU_OP_LIT_NULL:
        FG_CHECK(tok.dtype >= FLOCKGPU_BOOL && tok.dtype <= FLOCKGPU_DATE32, FLOCKGPU_ERR_INVALID, "expression: NULL literal of unknown type %d", tok.dtype);
        n.dtype = tok.dtype;
        break;
      case FLOCKGPU_OP_NEG:
        n.l = pop();
        n.dtype = t.nodes[n.l].dtype;
        FG_CHECK(is_numeric(n.dtype) && !is_unsigned(n.dtype), FLOCKGPU_ERR_UNSUPPORTED, "expression: unary minus on %s", dtype_name(n.dtype));
        break;
      case FLOCKGPU_OP_IS_NULL:
      case FLOCKGPU_OP_IS_NOT_NULL:
        n.l = pop();
        n.dtype = FLOCKGPU_BOOL;
        break;
      case FLOCKGPU_OP_CASE: {
        n.flags = tok.col;
        const bool has_base = tok.col & FLOCKGPU_CASE_HAS_BASE, has_else = tok.col & FLOCKGPU_CASE_HAS_ELSE;
        FG_CHECK(tok.i64 >= 1 && tok.i64 <= 64 && (tok.col & ~3) == 0, FLOCKGPU_ERR_INVALID, "expression: malformed CASE (%lld WHEN branches, flags %d)",
                 (long long)tok.i64, tok.col);
        const size_t need = size_t(2 * tok.i64) + has_base + has_else;
        FG_CHECK(stack.size() >= need, FLOCKGPU_ERR_INVALID, "expression: CASE needs %zu operands, %zu on the stack (malformed postfix program)", need,
                 stack.size());
        n.kids.assign(stack.end() - need, stack.end());
        stack.resize(stack.size() - need);
        // result type: the common type of the THEN / ELSE values that are not NULL literals
        int dt = -1;
        for (size_t k = has_base ? 1 : 0; k < n.kids.size(); ++k) {
          const bool is_value = k + 1 == n.kids.size() && has_else ? true : ((k - (has_base ? 1 : 0)) & 1) == 1;
          const Node& c = t.nodes[n.kids[k]];
          if (!is_value) {
            if (has_base) {
              const int bt = t.nodes[n.kids[0]].dtype;
              FG_CHECK((is_numeric(bt) && is_numeric(c.dtype)) || same_ordered(bt, c.dtype), FLOCKGPU_ERR_UNSUPPORTED,
                       "expression: CASE compares %s with %s", dtype_name(bt), dtype_name(c.dtype));
            } else {
              FG_CHECK(c.dtype == FLOCKGPU_BOOL, FLOCKGPU_ERR_INVALID, "expression: CASE WHEN condition is not boolean");
            }
            continue;
          }
          if (c.op == FLOCKGPU_OP_LIT_NULL) continue;
          if (dt < 0) dt = c.dtype;
          else if (is_numeric(dt) && is_numeric(c.dtype)) dt = promote(dt, c.dtype);
          else FG_CHECK(dt == c.dtype, FLOCKGPU_ERR_INVALID, "expression: CASE branches of types %s and %s", dtype_name(dt), dtype_name(c.dtype));
        }
        if (dt < 0) dt = t.nodes[n.kids.back()].dtype;  // every branch is a NULL literal
        n.dtype = dt;
        break;
      }
      case FLOCKGPU_OP_IN_LIST: {
        n.flags = tok.col;
        FG_CHECK(tok.i64 >= 1 && tok.i64 <= 64 && (tok.col & ~1) == 0, FLOCKGPU_ERR_INVALID, "expression: malformed IN list (%lld literals, flags %d)",
                 (long long)tok.i64, tok.col);
        const size_t need = size_t(tok.i64) + 1;
        FG_CHECK(stack.size() >= need, FLOCKGPU_ERR_INVALID, "expression: IN list needs %zu operands, %zu on the stack (malformed postfix program)", need,
                 stack.size());
        n.kids.assign(stack.end() - need, stack.end());
        stack.resize(stack.size() - need);
        const int vt = t.nodes[n.kids[0]].dtype;
        for (size_t k = 1; k < n.kids.size(); ++k) {
          const Node& c = t.nodes[n.kids[k]];
          FG_CHECK(is_literal(c) || c.op == FLOCKGPU_OP_LIT_NULL, FLOCKGPU_ERR_INVALID, "expression: IN list entry %zu is not a literal", k - 1);
          FG_CHECK(c.op == FLOCKGPU_OP_LIT_NULL || (is_numeric(vt) && is_numeric(c.dtype)) || same_ordered(vt, c.dtype),
                   FLOCKGPU_ERR_UNSUPPORTED, "expression: %s IN a list with a %s literal", dtype_name(vt), dtype_name(c.dtype));
        }
        n.dtype = FLOCKGPU_BOOL;
        break;
      }
      case FLOCKGPU_OP_LIKE:
      case FLOCKGPU_OP_NOT_LIKE: {
        n.r = pop();
        n.l = pop();
        const Node& v = t.nodes[n.l];
        const Node& pat = t.nodes[n.r];
        FG_CHECK(v.dtype == FLOCKGPU_UTF8 || v.op == FLOCKGPU_OP_LIT_NULL, FLOCKGPU_ERR_UNSUPPORTED, "expression: LIKE over %s", dtype_name(v.dtype));
        FG_CHECK(pat.op == FLOCKGPU_OP_LIT_UTF8 || pat.op == FLOCKGPU_OP_LIT_NULL, FLOCKGPU_ERR_UNSUPPORTED, "expression: LIKE needs a literal pattern");
        n.dtype = FLOCKGPU_BOOL;
        break;
      }
      case FLOCKGPU_OP_DATE_PART: {
        n.l = pop();
        n.flags = tok.col;
        FG_CHECK(tok.col == FLOCKGPU_DATE_PART_YEAR || tok.col == FLOCKGPU_DATE_PART_HOUR, FLOCKGPU_ERR_UNSUPPORTED,
                 "expression: date_part field %d (YEAR and HOUR only)", tok.col);
        const int xt = t.nodes[n.l].dtype;
        FG_CHECK(xt == FLOCKGPU_DATE32 || xt == FLOCKGPU_TIMESTAMP, FLOCKGPU_ERR_UNSUPPORTED, "expression: date_part of %s", dtype_name(xt));
        n.i = xt == FLOCKGPU_DATE32 ? DU_DAY : timestamp_unit(t, n.l, cols);
        n.dtype = FLOCKGPU_INT32;
        break;
      }
      default:
        if (is_arith(tok.op) || is_cmp(tok.op) || tok.op == FLOCKGPU_OP_AND || tok.op == FLOCKGPU_OP_OR) {
          n.r = pop();
          n.l = pop();
          int lt = t.nodes[n.l].dtype, rt = t.nodes[n.r].dtype;
          if (is_arith(tok.op)) {
            FG_CHECK(is_numeric(lt) && is_numeric(rt), FLOCKGPU_ERR_UNSUPPORTED, "expression: arithmetic on %s and %s", dtype_name(lt),
                     dtype_name(rt));
            n.dtype = promote(lt, rt);
          } else if (is_cmp(tok.op)) {
            FG_CHECK((is_numeric(lt) && is_numeric(rt)) || same_ordered(lt, rt), FLOCKGPU_ERR_UNSUPPORTED,
                     "expression: comparison of %s with %s", dtype_name(lt), dtype_name(rt));
            n.dtype = FLOCKGPU_BOOL;
          } else {
            FG_CHECK(lt == FLOCKGPU_BOOL && rt == FLOCKGPU_BOOL, FLOCKGPU_ERR_INVALID, "expression: AND/OR of non-boolean operands");
            n.dtype = FLOCKGPU_BOOL;
          }
        } else {
          fail(FLOCKGPU_ERR_INVALID, "expression: unknown opcode %d", tok.op);
        }
    }
    t.nodes.push_back(n);
    stack.push_back(int(t.nodes.size()) - 1);
  }
  FG_CHECK(stack.size() == 1, FLOCKGPU_ERR_INVALID, "expression: %zu values left on the stack (malformed postfix program)", stack.size());
  t.root = stack[0];
  return t;
}

// Literal value converted to the canonical representation of `dtype`.
Val literal_as(const Node& n, int dtype) {
  Val v;
  v.i = 0;
  if (dtype == FLOCKGPU_FLOAT64) {
    v.d = n.op == FLOCKGPU_OP_LIT_F64 ? n.d : (is_unsigned(n.dtype) ? double(uint64_t(n.i)) : double(n.i));
  } else {
    int64_t x = n.op == FLOCKGPU_OP_LIT_F64 ? int64_t(n.d) : n.i;
    if (is_i32(dtype)) x = int64_t(int32_t(uint32_t(uint64_t(x))));
    if (dtype == FLOCKGPU_UINT32) x = int64_t(uint64_t(uint32_t(uint64_t(x))));
    v.i = x;
  }
  return v;
}

struct ChainBuilder {
  const Tree& t;
  bool div_by_col = false;
  explicit ChainBuilder(const Tree& tree) : t(tree) {}

  static void push(Chain& c, ChainStep st) {
    FG_CHECK(c.n_steps < MAX_STEPS, FLOCKGPU_ERR_UNSUPPORTED, "expression: more than %d arithmetic steps in one chain", MAX_STEPS);
    c.steps[c.n_steps++] = st;
  }
  static void push_unary(Chain& c, int op) {
    ChainStep st{};
    st.op = int16_t(op);
    st.src = 2;
    push(c, st);
  }
  // steps converting the accumulator from `from` to `to`
  static void convert(Chain& c, int from, int to) {
    if (from == to) return;
    if (to == FLOCKGPU_FLOAT64) {
      push_unary(c, is_unsigned(from) ? C_U2F : C_I2F);
    } else if (from == FLOCKGPU_FLOAT64) {
      push_unary(c, to == FLOCKGPU_UINT64 ? C_F2U : C_F2I);
      if (to == FLOCKGPU_INT32) push_unary(c, C_WRAP_I32);
      if (to == FLOCKGPU_UINT32) push_unary(c, C_WRAP_U32);
    } else {
      if (to == FLOCKGPU_INT32) push_unary(c, C_WRAP_I32);
      else if (to == FLOCKGPU_UINT32) push_unary(c, C_WRAP_U32);
      else if (from == FLOCKGPU_UINT32 || from == FLOCKGPU_INT32) { /* canonical form already 64-bit */ }
    }
  }

  // A "simple" operand: literal, column, or CAST of either that needs at most a load-time conversion.
  // Returns false if `idx` is not simple.  On success fills (is_col, col, cvt, lit) for result type T.
  bool simple_operand(int idx, int T, bool* is_col, int* col, int8_t* cvt, Val* lit) const {
    const Node* n = &t.nodes[idx];
    int src_dtype = n->dtype;
    while (n->op == FLOCKGPU_OP_CAST) {
      const Node* inner = &t.nodes[n->l];
      // only casts that keep every value (widening, to Float64) keep the operand simple
      if (lossy_cast(inner->dtype, n->dtype)) return false;
      src_dtype = n->dtype;
      n = inner;
    }
    (void)src_dtype;
    if (is_literal(*n)) {
      if (n->op == FLOCKGPU_OP_LIT_UTF8) return false;
      // fold the cast chain on the host: evaluate through each cast level
      std::function<Val(int, int*)> fold = [&](int i, int* dt) -> Val {
        const Node& m = t.nodes[i];
        if (m.op == FLOCKGPU_OP_CAST) {
          int inner_dt;
          Val v = fold(m.l, &inner_dt);
          Node tmp;
          tmp.dtype = inner_dt;
          if (inner_dt == FLOCKGPU_FLOAT64) { tmp.op = FLOCKGPU_OP_LIT_F64; tmp.d = v.d; }
          else { tmp.op = FLOCKGPU_OP_LIT_I64; tmp.i = v.i; }
          *dt = m.dtype;
          return literal_as(tmp, m.dtype);
        }
        *dt = m.dtype;
        return literal_as(m, m.dtype);
      };
      int dt;
      Val v = fold(idx, &dt);
      Node tmp;
      tmp.dtype = dt;
      if (dt == FLOCKGPU_FLOAT64) { tmp.op = FLOCKGPU_OP_LIT_F64; tmp.d = v.d; }
      else { tmp.op = FLOCKGPU_OP_LIT_I64; tmp.i = v.i; }
      *is_col = false;
      *lit = literal_as(tmp, T);
      *cvt = CVT_NONE;
      return true;
    }
    if (n->op == FLOCKGPU_OP_COLUMN) {
      *is_col = true;
      *col = n->col;
      *cvt = CVT_NONE;
      if (T == FLOCKGPU_FLOAT64 && n->dtype != FLOCKGPU_FLOAT64) *cvt = is_unsigned(n->dtype) ? CVT_U2F : CVT_I2F;
      if (T != FLOCKGPU_FLOAT64 && n->dtype == FLOCKGPU_FLOAT64) return false;
      return true;
    }
    return false;
  }

  static int arith_opcode(int op, int T, bool reversed) {
    bool f = T == FLOCKGPU_FLOAT64, u = is_unsigned(T);
    switch (op) {
      case FLOCKGPU_OP_ADD: return f ? C_ADD_F : C_ADD_I;
      case FLOCKGPU_OP_MUL: return f ? C_MUL_F : C_MUL_I;
      case FLOCKGPU_OP_SUB: return f ? (reversed ? C_RSUB_F : C_SUB_F) : (reversed ? C_RSUB_I : C_SUB_I);
      case FLOCKGPU_OP_DIV: return f ? (reversed ? C_RDIV_F : C_DIV_F) : u ? (reversed ? C_RDIV_U : C_DIV_U) : (reversed ? C_RDIV_I : C_DIV_I);
      case FLOCKGPU_OP_MOD:
        FG_CHECK(!f, FLOCKGPU_ERR_UNSUPPORTED, "expression: %% on Float64");
        return u ? (reversed ? C_RMOD_U : C_MOD_U) : (reversed ? C_RMOD_I : C_MOD_I);
    }
    fail(FLOCKGPU_ERR_INVALID, "expression: bad arithmetic opcode %d", op);
  }

  // Builds the chain computing node `idx`; the accumulator ends in the canonical form of node.dtype.
  Chain build(int idx) {
    const Node& n = t.nodes[idx];
    Chain c{};
    c.start_col = -1;
    c.n_steps = 0;
    c.start_lit.i = 0;
    if (n.op == FLOCKGPU_OP_COLUMN) {
      FG_CHECK(n.dtype != FLOCKGPU_UTF8, FLOCKGPU_ERR_UNSUPPORTED, "expression: Utf8 column in an arithmetic context");
      c.start_col = n.col;
      return c;
    }
    if (is_literal(n)) {
      FG_CHECK(n.op != FLOCKGPU_OP_LIT_UTF8, FLOCKGPU_ERR_UNSUPPORTED, "expression: Utf8 literal in an arithmetic context");
      c.start_lit = literal_as(n, n.dtype);
      return c;
    }
    if (n.op == FLOCKGPU_OP_CAST) {
      c = build(n.l);
      convert(c, t.nodes[n.l].dtype, n.dtype);
      return c;
    }
    FG_CHECK(n.op != FLOCKGPU_OP_DATE_PART, FLOCKGPU_ERR_UNSUPPORTED, "expression: date_part runs in the tree form only");
    FG_CHECK(is_arith(n.op), FLOCKGPU_ERR_UNSUPPORTED, "expression: boolean sub-expression used as a value");
    int T = n.dtype;
    bool is_col = false;
    int col = -1;
    int8_t cvt = CVT_NONE;
    Val lit;
    lit.i = 0;
    bool reversed = false;
    if (simple_operand(n.r, T, &is_col, &col, &cvt, &lit)) {
      c = build(n.l);
      convert(c, t.nodes[n.l].dtype, T);
    } else if (simple_operand(n.l, T, &is_col, &col, &cvt, &lit)) {
      c = build(n.r);
      convert(c, t.nodes[n.r].dtype, T);
      reversed = true;
    } else {
      fail(FLOCKGPU_ERR_UNSUPPORTED,
           "expression: both operands of an arithmetic node are compound; the GPU path evaluates left-deep chains only");
    }
    ChainStep st{};
    st.op = int16_t(arith_opcode(n.op, T, reversed));
    st.src = is_col ? 1 : 0;
    st.cvt = cvt;
    st.col = col;
    st.lit = lit;
    bool divides = (n.op == FLOCKGPU_OP_DIV || n.op == FLOCKGPU_OP_MOD) && T != FLOCKGPU_FLOAT64;
    if (divides) {
      if (!reversed && !is_col)
        FG_CHECK(lit.i != 0, FLOCKGPU_ERR_EXECUTION, "Divide by zero");  // DataFusion's message for a zero divisor
      if (is_col || reversed) div_by_col = true;
    }
    push(c, st);
    if (T == FLOCKGPU_INT32) push_unary(c, C_WRAP_I32);
    if (T == FLOCKGPU_UINT32) push_unary(c, C_WRAP_U32);
    return c;
  }
};

int cmp_domain(int lt, int rt) {
  if (lt == FLOCKGPU_FLOAT64 || rt == FLOCKGPU_FLOAT64) return DOM_F64;
  if (is_unsigned(lt) && is_unsigned(rt)) return DOM_U64;
  if (is_unsigned(lt) || is_unsigned(rt)) return DOM_U64;  // DataFusion coerces both sides first
  return DOM_I64;
}

int swap_cmp(int cmp) {
  switch (cmp) {
    case FLOCKGPU_OP_LT: return FLOCKGPU_OP_GT;
    case FLOCKGPU_OP_LE: return FLOCKGPU_OP_GE;
    case FLOCKGPU_OP_GT: return FLOCKGPU_OP_LT;
    case FLOCKGPU_OP_GE: return FLOCKGPU_OP_LE;
    default: return cmp;
  }
}

}  // namespace

Expr tokens_to_expr(const flockgpu_expr* e) {
  Expr out;
  FG_CHECK(e && e->tokens && e->n_tokens > 0, FLOCKGPU_ERR_INVALID, "expression: empty program");
  for (int i = 0; i < e->n_tokens; ++i) {
    const flockgpu_expr_token& t = e->tokens[i];
    ExprTok k;
    k.op = t.op;
    k.dtype = t.dtype;
    k.col = t.col;
    k.i64 = t.i64;
    k.f64 = t.f64;
    if (t.op == FLOCKGPU_OP_LIT_UTF8) {
      FG_CHECK(t.str_len >= 0 && (t.str || t.str_len == 0), FLOCKGPU_ERR_INVALID, "expression: bad Utf8 literal");
      k.str.assign(t.str ? t.str : "", size_t(t.str_len));
    }
    out.push_back(std::move(k));
  }
  return out;
}

int infer_dtype(const Expr& e, const std::vector<ColInfo>& cols) {
  Tree t = build_tree(e, cols);
  return t.nodes[t.root].dtype;
}

CompiledValue compile_value(const Expr& e, const std::vector<ColInfo>& cols, int max_null_inputs) {
  Tree t = build_tree(e, cols);
  const Node& root = t.nodes[t.root];
  CompiledValue out;
  out.dtype = root.dtype;
  FG_CHECK(root.dtype != FLOCKGPU_BOOL, FLOCKGPU_ERR_UNSUPPORTED, "projection: boolean-valued output columns are not supported");
  if (root.op == FLOCKGPU_OP_COLUMN) {
    out.passthrough = true;
    out.src_col = root.col;
    out.format = cols[root.col].format;
    return out;
  }
  FG_CHECK(root.dtype != FLOCKGPU_UTF8, FLOCKGPU_ERR_UNSUPPORTED, "projection: computed Utf8 columns are not supported");
  ChainBuilder b(t);
  out.chain = b.build(t.root);
  out.has_div_by_col = b.div_by_col;
  auto note = [&](int col) {
    if (col >= 0 && cols[col].has_nulls) out.null_inputs.push_back(col);
  };
  note(out.chain.start_col);
  for (int st = 0; st < out.chain.n_steps; ++st)
    if (out.chain.steps[st].src == 1) note(out.chain.steps[st].col);
  FG_CHECK(int(out.null_inputs.size()) <= max_null_inputs, FLOCKGPU_ERR_UNSUPPORTED, "projection: more than %d inputs with NULLs for the chain form",
           max_null_inputs);
  // a NULL operand makes the quotient NULL, whatever value sits under it: the chain divides it all the same
  FG_CHECK(!out.has_div_by_col || out.null_inputs.empty(), FLOCKGPU_ERR_UNSUPPORTED, "projection: a division by a column over columns with NULLs");
  FG_CHECK(!has_lossy_cast(t), FLOCKGPU_ERR_UNSUPPORTED, "projection: a CAST that can give NULL");
  out.format = default_format(root.dtype);
  if (root.dtype == FLOCKGPU_TIMESTAMP) {
    // keep the unit/timezone of the first timestamp column the expression touches
    for (const Node& n : t.nodes)
      if (n.op == FLOCKGPU_OP_COLUMN && n.dtype == FLOCKGPU_TIMESTAMP) {
        out.format = cols[n.col].format;
        break;
      }
  }
  // fast shape: lit * CAST(i32 AS f64)
  const Chain& c = out.chain;
  if (root.dtype == FLOCKGPU_FLOAT64 && c.start_col >= 0 && cols[c.start_col].dtype == FLOCKGPU_INT32 && c.n_steps == 2 &&
      c.steps[0].op == C_I2F && c.steps[1].op == C_MUL_F && c.steps[1].src == 0) {
    out.fast = FAST_VAL_I32_TO_F64_MUL;
    out.fast_lit = c.steps[1].lit.d;
  }
  return out;
}

CompiledPredicate compile_predicate(const Expr& e, const std::vector<ColInfo>& cols) {
  Tree t = build_tree(e, cols);
  FG_CHECK(t.nodes[t.root].dtype == FLOCKGPU_BOOL, FLOCKGPU_ERR_INVALID, "filter: predicate is not boolean");
  CompiledPredicate out;
  memset(&out.prog, 0, sizeof out.prog);
  Predicate& p = out.prog;
  ChainBuilder b(t);
  int pool_used = 0;
  std::vector<int> term_of_node(t.nodes.size(), -1);

  std::function<void(int)> collect = [&](int idx) {
    const Node& n = t.nodes[idx];
    if (n.op == FLOCKGPU_OP_AND || n.op == FLOCKGPU_OP_OR) {
      collect(n.l);
      collect(n.r);
      return;
    }
    if (n.op == FLOCKGPU_OP_NOT) {
      collect(n.l);
      return;
    }
    FG_CHECK(is_cmp(n.op), FLOCKGPU_ERR_UNSUPPORTED, "filter: boolean leaf is not a comparison (opcode %d)", n.op);
    FG_CHECK(p.n_terms < MAX_TERMS, FLOCKGPU_ERR_UNSUPPORTED, "filter: more than %d comparison terms", MAX_TERMS);
    Term& term = p.terms[p.n_terms];
    term.cmp = n.op;
    const Node& l = t.nodes[n.l];
    const Node& r = t.nodes[n.r];
    if (l.dtype == FLOCKGPU_UTF8) {
      term.domain = DOM_UTF8;
      const Node* colside = &l;
      const Node* other = &r;
      if (l.op != FLOCKGPU_OP_COLUMN) {
        colside = &r;
        other = &l;
        term.cmp = swap_cmp(n.op);
      }
      FG_CHECK(colside->op == FLOCKGPU_OP_COLUMN, FLOCKGPU_ERR_UNSUPPORTED, "filter: Utf8 comparison needs a column operand");
      term.lhs_col = colside->col;
      if (other->op == FLOCKGPU_OP_COLUMN) {
        term.rhs_col = other->col;
      } else {
        FG_CHECK(other->op == FLOCKGPU_OP_LIT_UTF8, FLOCKGPU_ERR_UNSUPPORTED, "filter: Utf8 comparison with a computed operand");
        FG_CHECK(pool_used + int(other->s.size()) <= STRPOOL_BYTES, FLOCKGPU_ERR_UNSUPPORTED, "filter: Utf8 literals exceed %d bytes", STRPOOL_BYTES);
        term.rhs_col = -1;
        term.lit_off = pool_used;
        term.lit_len = int(other->s.size());
        memcpy(p.strpool + pool_used, other->s.data(), other->s.size());
        pool_used += int(other->s.size());
      }
    } else {
      term.domain = cmp_domain(l.dtype, r.dtype);
      term.lhs = b.build(n.l);
      term.rhs = b.build(n.r);
      if (term.domain == DOM_F64) {
        ChainBuilder::convert(term.lhs, l.dtype, FLOCKGPU_FLOAT64);
        ChainBuilder::convert(term.rhs, r.dtype, FLOCKGPU_FLOAT64);
      }
    }
    // which input columns make this comparison NULL
    {
      std::function<void(int)> cols_of = [&](int i) {
        const Node& x = t.nodes[i];
        if (x.op == FLOCKGPU_OP_COLUMN) {
          if (x.col >= 0 && x.col < 32 && cols[x.col].has_nulls) term.null_cols |= 1u << x.col;
          return;
        }
        if (x.l >= 0) cols_of(x.l);
        if (x.r >= 0) cols_of(x.r);
      };
      term.null_cols = 0;
      cols_of(n.l);
      cols_of(n.r);
    }
    term_of_node[idx] = p.n_terms++;
  };
  collect(t.root);
  p.has_div_by_col = b.div_by_col ? 1 : 0;
  FG_CHECK(!has_lossy_cast(t), FLOCKGPU_ERR_UNSUPPORTED, "filter: a CAST that can give NULL");
  bool any_null = false;
  for (int i = 0; i < p.n_terms; ++i) any_null |= p.terms[i].null_cols != 0;

  if (!any_null) {
    // truth table over the term bits
    std::function<bool(int, unsigned)> truth = [&](int idx, unsigned bits) -> bool {
      const Node& n = t.nodes[idx];
      if (n.op == FLOCKGPU_OP_AND) return truth(n.l, bits) && truth(n.r, bits);
      if (n.op == FLOCKGPU_OP_OR) return truth(n.l, bits) || truth(n.r, bits);
      if (n.op == FLOCKGPU_OP_NOT) return !truth(n.l, bits);
      return (bits >> term_of_node[idx]) & 1u;
    };
    for (unsigned bits = 0; bits < (1u << p.n_terms); ++bits)
      if (truth(t.root, bits)) p.lut[bits >> 5] |= 1u << (bits & 31);
  } else {
    // SQL three-valued logic (strong Kleene): 1 = TRUE, 0 = FALSE, 2 = NULL; the row is kept iff the root is TRUE
    FG_CHECK(p.n_terms <= 4, FLOCKGPU_ERR_UNSUPPORTED, "filter: more than 4 comparison terms over columns with NULLs");
    // the terms divide in the rows where an operand is NULL too
    FG_CHECK(!p.has_div_by_col, FLOCKGPU_ERR_UNSUPPORTED, "filter: a division by a column over columns with NULLs");
    p.kleene = 1;
    std::function<int(int, unsigned)> k3 = [&](int idx, unsigned bits) -> int {
      const Node& n = t.nodes[idx];
      if (n.op == FLOCKGPU_OP_AND) {
        const int a = k3(n.l, bits), c = k3(n.r, bits);
        return (a == 0 || c == 0) ? 0 : (a == 2 || c == 2) ? 2 : 1;
      }
      if (n.op == FLOCKGPU_OP_OR) {
        const int a = k3(n.l, bits), c = k3(n.r, bits);
        return (a == 1 || c == 1) ? 1 : (a == 2 || c == 2) ? 2 : 0;
      }
      if (n.op == FLOCKGPU_OP_NOT) {
        const int a = k3(n.l, bits);
        return a == 2 ? 2 : 1 - a;
      }
      const int tix = term_of_node[idx];
      return ((bits >> (4 + tix)) & 1u) ? 2 : int((bits >> tix) & 1u);
    };
    for (unsigned bits = 0; bits < 256; ++bits)
      if (k3(t.root, bits) == 1) p.lut[bits >> 5] |= 1u << (bits & 31);
    return out;  // no vectorised shape reads validity
  }

  // fast shapes: one term over one Int32 (or Date32) column against literals
  // (a single term has a 2-entry truth table: 0b10 = the term itself, 0b01 = NOT term; constants keep the interpreter)
  const unsigned table1 = p.lut[0] & 3u;
  auto negate_cmp = [](int cmp) {
    switch (cmp) {
      case FLOCKGPU_OP_EQ: return int(FLOCKGPU_OP_NE);
      case FLOCKGPU_OP_NE: return int(FLOCKGPU_OP_EQ);
      case FLOCKGPU_OP_LT: return int(FLOCKGPU_OP_GE);
      case FLOCKGPU_OP_LE: return int(FLOCKGPU_OP_GT);
      case FLOCKGPU_OP_GT: return int(FLOCKGPU_OP_LE);
      default: return int(FLOCKGPU_OP_LT);
    }
  };
  if (p.n_terms == 1 && p.terms[0].domain == DOM_I64 && (table1 == 2u || table1 == 1u)) {
    const Term& term = p.terms[0];
    const Chain& l = term.lhs;
    const Chain& r = term.rhs;
    if (r.start_col < 0 && r.n_steps == 0 && l.start_col >= 0 && is_i32(cols[l.start_col].dtype)) {
      if (l.n_steps == 0) {
        out.fast.kind = FAST_PRED_I32_CMP;
        out.fast.col = l.start_col;
        out.fast.cmp = term.cmp;
        out.fast.rhs = r.start_lit.i;
      } else if (l.n_steps == 1 && l.steps[0].op == C_MOD_I && l.steps[0].src == 0) {
        int64_t m = l.steps[0].lit.i;
        int64_t am = m < 0 ? -m : m;
        if (am > 0 && am < (int64_t(1) << 31)) {
          out.fast.kind = FAST_PRED_I32_MOD_CMP;
          out.fast.col = l.start_col;
          out.fast.cmp = term.cmp;
          out.fast.modulus = am;  // x % m == x % |m| (sign follows the dividend)
          out.fast.rhs = r.start_lit.i;
        }
      }
    }
    if (out.fast.kind != FAST_PRED_NONE && table1 == 1u) out.fast.cmp = negate_cmp(out.fast.cmp);
  }
  return out;
}

// ------------------------------------------------------------------------------------------------
// the tree form (expr_tree.h)
// ------------------------------------------------------------------------------------------------
namespace {

// A value of the program before registers are assigned.  Nodes are hash-consed: the same operation over the same
// operands is one node, across all the expressions of a program.
struct TNode {
  int op = 0, sub = 0;
  int a = -1, b = -1, c = -1;  // operand nodes
  int col = -1, col2 = -1;
  Val lit{};
  bool null_lit = false;
  bool may_null = false;
};

struct TreeBuilder {
  const std::vector<ColInfo>& cols;
  std::vector<TNode> ir;
  std::map<std::string, int> interned;
  std::string pool;
  bool may_fail = false;
  explicit TreeBuilder(const std::vector<ColInfo>& c) : cols(c) {}

  int intern(const TNode& n) {
    char key[160];
    snprintf(key, sizeof key, "%d.%d.%d.%d.%d.%d.%d.%llx.%d", n.op, n.sub, n.a, n.b, n.c, n.col, n.col2, (unsigned long long)n.lit.u, int(n.null_lit));
    auto it = interned.find(key);
    if (it != interned.end()) return it->second;
    ir.push_back(n);
    interned[key] = int(ir.size()) - 1;
    return int(ir.size()) - 1;
  }
  bool nullable(int id) const { return id >= 0 && ir[id].may_null; }

  int lit_node(Val v, bool is_null) {
    TNode n;
    n.op = T_LIT;
    n.lit = is_null ? Val{0} : v;
    n.null_lit = is_null;
    n.may_null = is_null;
    return intern(n);
  }
  int unary(int op, int sub, int a) {
    TNode n;
    n.op = op;
    n.sub = sub;
    n.a = a;
    n.may_null = (op == T_IS_NULL || op == T_IS_NOT_NULL) ? false : nullable(a);
    return intern(n);
  }
  int binary(int op, int sub, int a, int b) {
    TNode n;
    n.op = op;
    n.sub = sub;
    n.a = a;
    n.b = b;
    n.may_null = nullable(a) || nullable(b);
    return intern(n);
  }
  int select(int cond, int a, int b) {
    TNode n;
    n.op = T_SELECT;
    n.c = cond;
    n.a = a;
    n.b = b;
    n.may_null = nullable(a) || nullable(b);
    return intern(n);
  }
  // `id` (canonical form of `from`) converted to the canonical form of `to`: the steps ChainBuilder::convert pushes
  int convert(int id, int from, int to) {
    if (from == to || from == FLOCKGPU_BOOL || to == FLOCKGPU_BOOL) return id;
    if (to == FLOCKGPU_FLOAT64) return unary(T_ARITH, is_unsigned(from) ? C_U2F : C_I2F, id);
    if (from == FLOCKGPU_FLOAT64) id = unary(T_ARITH, C_F2I, id);
    if (to == FLOCKGPU_INT32) return unary(T_ARITH, C_WRAP_I32, id);
    if (to == FLOCKGPU_UINT32) return unary(T_ARITH, C_WRAP_U32, id);
    return id;
  }
  // An explicit CAST.  One that can lose its value checks the source (cast_fits) and is NULL where it does not fit;
  // a value that fits keeps its canonical form, except that a float is truncated toward zero.
  int cast(int id, int from, int to) {
    if (!lossy_cast(from, to)) return convert(id, from, to);
    TNode n;
    n.op = T_ARITH;
    n.sub = from != FLOCKGPU_FLOAT64 ? C_NOP : to == FLOCKGPU_UINT64 ? C_F2U : C_F2I;
    n.a = id;
    n.lit.i = cast_code(from == FLOCKGPU_FLOAT64 ? DOM_F64 : is_unsigned(from) ? DOM_U64 : DOM_I64, to);
    n.may_null = true;
    return intern(n);
  }
  int pooled(const std::string& s, Val* where) {
    size_t at = pool.find(s);
    if (at == std::string::npos || s.empty()) {
      at = s.empty() ? 0 : pool.size();
      if (!s.empty()) pool += s;
    }
    FG_CHECK(pool.size() <= size_t(TREE_POOL_BYTES), FLOCKGPU_ERR_UNSUPPORTED, "expression: Utf8 literals exceed %d bytes", TREE_POOL_BYTES);
    where->u = (uint64_t(at) << 32) | uint64_t(s.size());
    return 0;
  }

  // `l CMP r` over tree nodes li, ri
  int compare(const Tree& t, int cmp, int li, int ri, std::vector<int>& memo) {
    const Node& l = t.nodes[li];
    const Node& r = t.nodes[ri];
    if (l.op == FLOCKGPU_OP_LIT_NULL || r.op == FLOCKGPU_OP_LIT_NULL) return lit_node(Val{0}, true);  // x CMP NULL is NULL
    if (l.dtype == FLOCKGPU_UTF8) {
      const Node* colside = &l;
      const Node* other = &r;
      if (l.op != FLOCKGPU_OP_COLUMN) {
        colside = &r;
        other = &l;
        cmp = swap_cmp(cmp);
      }
      FG_CHECK(colside->op == FLOCKGPU_OP_COLUMN, FLOCKGPU_ERR_UNSUPPORTED, "expression: Utf8 comparison needs a column operand");
      TNode n;
      n.op = T_CMP_UTF8;
      n.sub = cmp;
      n.col = colside->col;
      n.may_null = cols[colside->col].has_nulls;
      if (other->op == FLOCKGPU_OP_COLUMN) {
        n.col2 = other->col;
        n.may_null |= cols[other->col].has_nulls;
      } else {
        FG_CHECK(other->op == FLOCKGPU_OP_LIT_UTF8, FLOCKGPU_ERR_UNSUPPORTED, "expression: Utf8 comparison with a computed operand");
        pooled(other->s, &n.lit);
      }
      return intern(n);
    }
    const int dom = cmp_domain(l.dtype, r.dtype);
    int a = lower(t, li, memo), b = lower(t, ri, memo);
    if (dom == DOM_F64) {
      a = convert(a, l.dtype, FLOCKGPU_FLOAT64);
      b = convert(b, r.dtype, FLOCKGPU_FLOAT64);
    }
    return binary(T_CMP, (dom << 8) | (cmp - FLOCKGPU_OP_EQ), a, b);
  }

  int lower(const Tree& t, int idx, std::vector<int>& memo) {
    if (memo[idx] >= 0) return memo[idx];
    const Node& n = t.nodes[idx];
    int id = -1;
    switch (n.op) {
      case FLOCKGPU_OP_COLUMN: {
        TNode x;
        x.op = T_COL;
        x.col = n.col;
        x.may_null = cols[n.col].has_nulls;
        id = intern(x);
        break;
      }
      case FLOCKGPU_OP_LIT_I64:
      case FLOCKGPU_OP_LIT_F64:
        id = lit_node(literal_as(n, n.dtype), false);
        break;
      case FLOCKGPU_OP_LIT_NULL:
        id = lit_node(Val{0}, true);
        break;
      case FLOCKGPU_OP_LIT_UTF8:
        fail(FLOCKGPU_ERR_UNSUPPORTED, "expression: a Utf8 literal is only supported as a comparison operand or in an IN list");
      case FLOCKGPU_OP_CAST:
        FG_CHECK(t.nodes[n.l].dtype != FLOCKGPU_BOOL, FLOCKGPU_ERR_UNSUPPORTED, "expression: CAST of a boolean");
        id = cast(lower(t, n.l, memo), t.nodes[n.l].dtype, n.dtype);
        break;
      case FLOCKGPU_OP_NEG:
        if (n.dtype == FLOCKGPU_FLOAT64) {
          Val m;
          m.d = -1.0;  // x * -1 flips the sign of every value, zeros included, in one exact operation
          id = binary(T_ARITH, C_MUL_F, lower(t, n.l, memo), lit_node(m, false));
        } else {
          id = binary(T_ARITH, C_RSUB_I, lower(t, n.l, memo), lit_node(Val{0}, false));
          if (n.dtype == FLOCKGPU_INT32) id = unary(T_ARITH, C_WRAP_I32, id);
        }
        break;
      case FLOCKGPU_OP_NOT:
        id = unary(T_NOT, 0, lower(t, n.l, memo));
        break;
      case FLOCKGPU_OP_IS_NULL:
      case FLOCKGPU_OP_IS_NOT_NULL: {
        FG_CHECK(t.nodes[n.l].op != FLOCKGPU_OP_LIT_UTF8, FLOCKGPU_ERR_UNSUPPORTED, "expression: IS NULL of a Utf8 literal");
        id = unary(n.op == FLOCKGPU_OP_IS_NULL ? T_IS_NULL : T_IS_NOT_NULL, 0, lower(t, n.l, memo));
        break;
      }
      case FLOCKGPU_OP_AND:
      case FLOCKGPU_OP_OR:
        id = binary(n.op == FLOCKGPU_OP_AND ? T_AND : T_OR, 0, lower(t, n.l, memo), lower(t, n.r, memo));
        break;
      case FLOCKGPU_OP_CASE: {
        FG_CHECK(n.dtype != FLOCKGPU_UTF8, FLOCKGPU_ERR_UNSUPPORTED, "expression: a CASE that returns Utf8 (computed Utf8 values are not supported)");
        const bool has_base = n.flags & FLOCKGPU_CASE_HAS_BASE, has_else = n.flags & FLOCKGPU_CASE_HAS_ELSE;
        const int first = has_base ? 1 : 0;
        const int n_when = int(n.kids.size() - first - (has_else ? 1 : 0)) / 2;
        auto value = [&](int kid) { return convert(lower(t, kid, memo), t.nodes[kid].dtype, n.dtype); };
        id = has_else ? value(n.kids.back()) : lit_node(Val{0}, true);
        for (int w = n_when - 1; w >= 0; --w) {
          const int when = n.kids[first + 2 * w], then = n.kids[first + 2 * w + 1];
          const int cond = has_base ? compare(t, FLOCKGPU_OP_EQ, n.kids[0], when, memo) : lower(t, when, memo);
          id = select(cond, value(then), id);
        }
        break;
      }
      case FLOCKGPU_OP_LIKE:
      case FLOCKGPU_OP_NOT_LIKE: {
        const Node& v = t.nodes[n.l];
        const Node& pat = t.nodes[n.r];
        if (v.op == FLOCKGPU_OP_LIT_NULL || pat.op == FLOCKGPU_OP_LIT_NULL) {
          id = lit_node(Val{0}, true);
          break;
        }
        FG_CHECK(v.op == FLOCKGPU_OP_COLUMN, FLOCKGPU_ERR_UNSUPPORTED, "expression: LIKE needs a column operand");
        TNode x;
        x.op = T_LIKE;
        x.sub = n.op == FLOCKGPU_OP_NOT_LIKE;
        x.col = v.col;
        x.may_null = cols[v.col].has_nulls;
        pooled(pat.s, &x.lit);
        id = intern(x);
        break;
      }
      case FLOCKGPU_OP_DATE_PART: {
        TNode x;
        x.op = T_DATE_PART;
        x.sub = n.flags;
        x.a = lower(t, n.l, memo);
        x.lit.i = n.i;
        // only a year of seconds can leave Int32: 2^31 years are some 6.8e16 s
        x.may_null = nullable(x.a) || (n.flags == FLOCKGPU_DATE_PART_YEAR && n.i == DU_S);
        id = intern(x);
        break;
      }
      case FLOCKGPU_OP_IN_LIST: {
        // x IN (a, b) is x = a OR x = b under Kleene's OR: exactly SQL's three-valued IN
        for (size_t k = 1; k < n.kids.size(); ++k) {
          const int eq = compare(t, FLOCKGPU_OP_EQ, n.kids[0], n.kids[k], memo);
          id = id < 0 ? eq : binary(T_OR, 0, id, eq);
        }
        if (n.flags & 1) id = unary(T_NOT, 0, id);
        break;
      }
      default:
        if (is_cmp(n.op)) {
          id = compare(t, n.op, n.l, n.r, memo);
        } else {
          FG_CHECK(is_arith(n.op), FLOCKGPU_ERR_INVALID, "expression: unknown opcode %d", n.op);
          const int T = n.dtype;
          const int a = convert(lower(t, n.l, memo), t.nodes[n.l].dtype, T);
          const int b = convert(lower(t, n.r, memo), t.nodes[n.r].dtype, T);
          id = binary(T_ARITH, ChainBuilder::arith_opcode(n.op, T, false), a, b);
          if ((n.op == FLOCKGPU_OP_DIV || n.op == FLOCKGPU_OP_MOD) && T != FLOCKGPU_FLOAT64) may_fail = true;
          if (T == FLOCKGPU_INT32) id = unary(T_ARITH, C_WRAP_I32, id);
          if (T == FLOCKGPU_UINT32) id = unary(T_ARITH, C_WRAP_U32, id);
        }
    }
    memo[idx] = id;
    return id;
  }

  // Registers and instruction order: post-order from each root, a register freed at its value's last use.
  // stores[k] >= 0: root k is written to output stores[k] as soon as it is computed.
  void emit(const std::vector<int>& roots, const std::vector<int>& stores, bool predicate, CompiledTree* out) {
    TreeProgram& p = out->prog;
    memset(&p, 0, sizeof p);
    p.result_reg = -1;
    std::vector<int> uses(ir.size(), 0), reg(ir.size(), -1);
    std::vector<char> seen(ir.size(), 0);
    std::function<void(int)> count = [&](int id) {
      if (id < 0) return;
      ++uses[id];
      if (seen[id]) return;
      seen[id] = 1;
      count(ir[id].a);
      count(ir[id].b);
      count(ir[id].c);
    };
    for (int r : roots) count(r);
    // registers a node's subtree needs when it is evaluated on its own (operands are interned before their users)
    std::vector<int> need(ir.size(), 1);
    for (size_t id = 0; id < ir.size(); ++id) {
      int k[3] = {ir[id].a < 0 ? 0 : need[ir[id].a], ir[id].b < 0 ? 0 : need[ir[id].b], ir[id].c < 0 ? 0 : need[ir[id].c]};
      std::sort(k, k + 3, std::greater<int>());
      need[id] = std::max({1, k[0], k[1] + (k[1] > 0), k[2] + 2 * (k[2] > 0)});
    }
    bool busy[TREE_REGS] = {};
    std::set<int> cols_read;
    auto push = [&](const TreeInstr& in) {
      FG_CHECK(p.n_instr < TREE_MAX_INSTR, FLOCKGPU_ERR_UNSUPPORTED, "expression: the program needs more than %d instructions", TREE_MAX_INSTR);
      p.ins[p.n_instr++] = in;
    };
    auto release = [&](int id) {
      if (id >= 0 && --uses[id] == 0) busy[reg[id]] = false;
    };
    std::function<void(int)> gen = [&](int id) {
      if (id < 0 || reg[id] >= 0) return;
      const TNode& n = ir[id];
      // the operand that needs the most registers first (Sethi-Ullman): the others' results are not held meanwhile
      int kids[3] = {n.c, n.a, n.b};
      std::stable_sort(kids, kids + 3, [&](int x, int y) { return (x < 0 ? 0 : need[x]) > (y < 0 ? 0 : need[y]); });
      for (int k : kids) gen(k);
      // the operands' last use may be this instruction: their registers are free for its result (every row reads its
      // operands before it writes)
      release(n.a);
      release(n.b);
      release(n.c);
      int r = 0;
      while (r < TREE_REGS && busy[r]) ++r;
      FG_CHECK(r < TREE_REGS, FLOCKGPU_ERR_UNSUPPORTED, "expression: the tree needs more than %d registers at once", TREE_REGS);
      busy[r] = true;
      out->n_regs = std::max(out->n_regs, r + 1);
      reg[id] = r;
      TreeInstr in{};
      in.op = int16_t(n.op);
      in.sub = int16_t(n.sub);
      in.d = int8_t(r);
      in.a = int8_t(n.a >= 0 ? reg[n.a] : -1);
      in.b = int8_t(n.b >= 0 ? reg[n.b] : -1);
      in.c = int8_t(n.c >= 0 ? reg[n.c] : -1);
      if (n.op == T_LIT) in.a = n.null_lit ? 1 : 0;
      in.col = n.col;
      in.col2 = n.col2;
      in.lit = n.lit;
      if (n.col >= 0) cols_read.insert(n.col);
      if (n.col2 >= 0) cols_read.insert(n.col2);
      push(in);
    };
    for (size_t k = 0; k < roots.size(); ++k) {
      gen(roots[k]);
      if (predicate) {
        p.result_reg = reg[roots[k]];
      } else {
        TreeInstr st{};
        st.op = T_STORE;
        st.a = int8_t(reg[roots[k]]);
        st.col = stores[k];
        push(st);
        release(roots[k]);
      }
    }
    memcpy(p.pool, pool.data(), pool.size());
    out->may_fail = may_fail;
    out->cols_read.assign(cols_read.begin(), cols_read.end());
  }
};

}  // namespace

CompiledTree compile_tree_values(const std::vector<Expr>& exprs, const std::vector<ColInfo>& cols) {
  CompiledTree out;
  TreeBuilder b(cols);
  std::vector<int> roots, stores;
  for (const Expr& e : exprs) {
    Tree t = build_tree(e, cols);
    const Node& root = t.nodes[t.root];
    TreeRoot r;
    r.dtype = root.dtype;
    FG_CHECK(root.dtype != FLOCKGPU_BOOL, FLOCKGPU_ERR_UNSUPPORTED, "projection: boolean-valued output columns are not supported");
    if (root.op == FLOCKGPU_OP_COLUMN) {
      r.passthrough = true;
      r.src_col = root.col;
      r.format = cols[root.col].format;
    } else {
      FG_CHECK(root.dtype != FLOCKGPU_UTF8, FLOCKGPU_ERR_UNSUPPORTED, "projection: computed Utf8 columns are not supported");
      FG_CHECK(out.n_outs < TREE_MAX_OUTS, FLOCKGPU_ERR_UNSUPPORTED, "expression: more than %d computed values in one program", TREE_MAX_OUTS);
      std::vector<int> memo(t.nodes.size(), -1);
      const int id = b.lower(t, t.root, memo);
      r.out = out.n_outs++;
      r.may_be_null = b.ir[id].may_null;
      r.format = default_format(root.dtype);
      if (root.dtype == FLOCKGPU_TIMESTAMP)
        for (const Node& n : t.nodes)
          if (n.op == FLOCKGPU_OP_COLUMN && n.dtype == FLOCKGPU_TIMESTAMP) {
            r.format = cols[n.col].format;
            break;
          }
      roots.push_back(id);
      stores.push_back(r.out);
    }
    out.roots.push_back(r);
  }
  b.emit(roots, stores, false, &out);
  return out;
}

CompiledTree compile_tree_predicate(const Expr& e, const std::vector<ColInfo>& cols) {
  CompiledTree out;
  TreeBuilder b(cols);
  Tree t = build_tree(e, cols);
  FG_CHECK(t.nodes[t.root].dtype == FLOCKGPU_BOOL, FLOCKGPU_ERR_INVALID, "filter: predicate is not boolean");
  std::vector<int> memo(t.nodes.size(), -1);
  const int id = b.lower(t, t.root, memo);
  b.emit({id}, {-1}, true, &out);
  return out;
}

std::string expr_to_string(const Expr& e, const std::vector<ColInfo>& cols) {
  std::vector<std::string> st;
  auto opname = [](int op) -> const char* {
    switch (op) {
      case FLOCKGPU_OP_ADD: return "+"; case FLOCKGPU_OP_SUB: return "-"; case FLOCKGPU_OP_MUL: return "*";
      case FLOCKGPU_OP_DIV: return "/"; case FLOCKGPU_OP_MOD: return "%"; case FLOCKGPU_OP_EQ: return "=";
      case FLOCKGPU_OP_NE: return "!="; case FLOCKGPU_OP_LT: return "<"; case FLOCKGPU_OP_LE: return "<=";
      case FLOCKGPU_OP_GT: return ">"; case FLOCKGPU_OP_GE: return ">="; case FLOCKGPU_OP_AND: return "AND";
      case FLOCKGPU_OP_OR: return "OR"; case FLOCKGPU_OP_LIKE: return "LIKE"; case FLOCKGPU_OP_NOT_LIKE: return "NOT LIKE";
      default: return "?";
    }
  };
  char buf[64];
  for (const ExprTok& t : e) {
    switch (t.op) {
      case FLOCKGPU_OP_COLUMN:
        st.push_back((t.col >= 0 && t.col < int(cols.size()) ? cols[t.col].name : std::string("?")) + "@" + std::to_string(t.col));
        break;
      case FLOCKGPU_OP_LIT_I64: st.push_back(std::to_string(t.i64)); break;
      case FLOCKGPU_OP_LIT_F64: snprintf(buf, sizeof buf, "%.17g", t.f64); st.push_back(buf); break;
      case FLOCKGPU_OP_LIT_UTF8: st.push_back(t.str); break;
      case FLOCKGPU_OP_CAST: {
        if (st.empty()) return "<malformed>";
        std::string a = st.back(); st.pop_back();
        st.push_back("CAST(" + a + " AS " + dtype_name(t.dtype) + ")");
        break;
      }
      case FLOCKGPU_OP_NOT: {
        if (st.empty()) return "<malformed>";
        std::string a = st.back(); st.pop_back();
        st.push_back("NOT " + a);
        break;
      }
      case FLOCKGPU_OP_LIT_NULL: st.push_back("NULL"); break;
      case FLOCKGPU_OP_NEG:
      case FLOCKGPU_OP_IS_NULL:
      case FLOCKGPU_OP_IS_NOT_NULL: {
        if (st.empty()) return "<malformed>";
        std::string a = st.back(); st.pop_back();
        st.push_back(t.op == FLOCKGPU_OP_NEG ? "(- " + a + ")" : a + (t.op == FLOCKGPU_OP_IS_NULL ? " IS NULL" : " IS NOT NULL"));
        break;
      }
      case FLOCKGPU_OP_CASE: {
        const bool has_base = t.col & FLOCKGPU_CASE_HAS_BASE, has_else = t.col & FLOCKGPU_CASE_HAS_ELSE;
        const size_t need = size_t(2 * t.i64) + has_base + has_else;
        if (t.i64 < 1 || st.size() < need) return "<malformed>";
        const size_t at = st.size() - need;
        std::string s = "CASE ";
        if (has_base) s += st[at] + " ";
        for (int64_t w = 0; w < t.i64; ++w) s += "WHEN " + st[at + has_base + 2 * w] + " THEN " + st[at + has_base + 2 * w + 1] + " ";
        if (has_else) s += "ELSE " + st.back() + " ";
        st.resize(at);
        st.push_back(s + "END");
        break;
      }
      case FLOCKGPU_OP_DATE_PART: {
        if (st.empty()) return "<malformed>";
        std::string a = st.back(); st.pop_back();
        st.push_back(std::string("date_part(") + (t.col == FLOCKGPU_DATE_PART_HOUR ? "HOUR" : t.col == FLOCKGPU_DATE_PART_YEAR ? "YEAR" : "?") + ", " + a + ")");
        break;
      }
      case FLOCKGPU_OP_IN_LIST: {
        const size_t need = size_t(t.i64) + 1;
        if (t.i64 < 1 || st.size() < need) return "<malformed>";
        const size_t at = st.size() - need;
        std::string s = st[at] + (t.col ? " NOT IN ([" : " IN ([");
        for (size_t k = 1; k < need; ++k) s += (k > 1 ? ", " : "") + st[at + k];
        st.resize(at);
        st.push_back(s + "])");
        break;
      }
      default: {
        if (st.size() < 2) return "<malformed>";
        std::string r = st.back(); st.pop_back();
        std::string l = st.back(); st.pop_back();
        st.push_back(l + " " + opname(t.op) + " " + r);
      }
    }
  }
  return st.empty() ? "" : st.back();
}

}  // namespace fg
