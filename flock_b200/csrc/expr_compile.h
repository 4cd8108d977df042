// expr_compile.h -- host-side lowering of postfix PhysicalExpr programs to device programs.
#pragma once

#include <string>
#include <vector>

#include "expr_program.h"
#include "expr_tree.h"
#include "internal.h"

namespace fg {

// Input column description the compiler needs (decoupled from Table so it can be unit-tested).
struct ColInfo {
  int dtype;
  std::string name;
  std::string format;
  bool has_nulls = false;  // the column carries validity bytes: comparisons over it are three-valued
};

// Shapes with a hand-specialised kernel (everything else runs the generic term interpreter).
enum FastPredKind {
  FAST_PRED_NONE = 0,
  FAST_PRED_I32_MOD_CMP = 1,  // CAST(i32col AS Int64) % m  CMP  c   (NEXMark q2, planner.rs:122)
  FAST_PRED_I32_CMP = 2       // CAST(i32col AS Int64)      CMP  c   (NEXMark q3 auction side, planner.rs:155)
};
struct FastPred {
  int kind = FAST_PRED_NONE;
  int col = -1;
  int cmp = 0;
  int64_t modulus = 0;
  int64_t rhs = 0;
};

struct CompiledPredicate {
  Predicate prog;
  FastPred fast;
};

enum FastValueKind {
  FAST_VAL_NONE = 0,
  FAST_VAL_I32_TO_F64_MUL = 1  // lit * CAST(i32col AS Float64)   (NEXMark q1, planner.rs:90)
};
struct CompiledValue {
  bool passthrough = false;
  int src_col = -1;
  Chain chain{};
  int dtype = FLOCKGPU_INT64;
  std::string format;  // Arrow format of the result
  bool has_div_by_col = false;
  std::vector<int> null_inputs;  // the columns with NULLs the chain reads, once per read: the value is NULL where one is
  int fast = FAST_VAL_NONE;
  double fast_lit = 0;
};

// The tree form (expr_tree.h): one register program for several value expressions, or for one predicate.
struct TreeRoot {
  bool passthrough = false;  // a plain column: nothing is computed
  int src_col = -1;
  int out = -1;              // computed: index of its TreeOut (T_STORE's `col`)
  int dtype = FLOCKGPU_INT64;
  std::string format;
  bool may_be_null = false;  // computed: the result needs validity bytes
};
struct CompiledTree {
  TreeProgram prog;
  std::vector<TreeRoot> roots;
  int n_outs = 0;
  int n_regs = 0;             // registers the program uses
  bool may_fail = false;      // contains an integer division or modulo: the error flag must be read back
  std::vector<int> cols_read; // input columns the program loads, ascending
};
// Both fail with FLOCKGPU_ERR_UNSUPPORTED naming the limit when the program exceeds TREE_REGS registers,
// TREE_MAX_INSTR instructions or TREE_POOL_BYTES of Utf8 literals, and for Boolean or computed Utf8 results.
CompiledTree compile_tree_values(const std::vector<Expr>& exprs, const std::vector<ColInfo>& cols);
CompiledTree compile_tree_predicate(const Expr& e, const std::vector<ColInfo>& cols);

// ColInfo / ColRef views of a table's columns (filter_project.cu); filter_colrefs refuses more than MAX_IN_COLS columns
// and a column that is NULL as a whole.
std::vector<ColInfo> col_infos(const Table& t);
void filter_colrefs(const Table& t, ColRef* refs);

// A value in the chain form is NULL where a column it reads is: a pure projection ANDs the validity of at most this many
// reads (and_validity_kernel).  The fused filter kernel writes no validity, so a value computed there reads none.
constexpr int PROJECT_MAX_NULL_INPUTS = 4;

// The term and chain forms.  Both fail with FLOCKGPU_ERR_UNSUPPORTED, naming the reason, on what they cannot evaluate
// exactly, and the operators then take the tree form: a CAST that can give NULL, a division by a column over columns
// with NULLs, and in compile_value more than `max_null_inputs` reads of columns with NULLs (a plain column passes).
Expr tokens_to_expr(const flockgpu_expr* e);
CompiledPredicate compile_predicate(const Expr& e, const std::vector<ColInfo>& cols);
CompiledValue compile_value(const Expr& e, const std::vector<ColInfo>& cols, int max_null_inputs);
// Result type of a value expression without building the chain (used for output schemas).
int infer_dtype(const Expr& e, const std::vector<ColInfo>& cols);
std::string expr_to_string(const Expr& e, const std::vector<ColInfo>& cols);

}  // namespace fg
