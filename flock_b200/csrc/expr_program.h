// expr_program.h -- the device form of DataFusion PhysicalExpr trees.
//
// A FilterExec predicate (flock/src/distributed_plan/planner.rs:122,155,162) is lowered to at most
// 8 comparison TERMS plus a 256-bit truth table over them (any AND/OR/NOT structure is one table
// look-up); each side of a comparison, and each computed ProjectionExec column (planner.rs:90), is a
// CHAIN: load a column (or literal), then apply up to MAX_STEPS typed steps `acc = acc OP operand`
// where the operand is a literal or a column.  The program is uniform across the grid, so its
// interpretation costs one uniform branch per step per thread-tile, not per row.
//
// Value representation ("canonical 64-bit"): Int32/Int64/Timestamp as sign-extended int64, UInt32/
// UInt64 as uint64, Float64 as double.  Int32 arithmetic wraps (C_WRAP_I32) like arrow-rs release
// builds; f64 arithmetic uses __dmul_rn/__dadd_rn so that no FMA contraction changes a rounding
// (SURVEY.md Appendix C.2).
#pragma once

#include <stdint.h>

#include "../../include/flockgpu.h"

namespace fg {

constexpr int MAX_STEPS = 6;
constexpr int MAX_TERMS = 8;
constexpr int MAX_IN_COLS = 16;
constexpr int MAX_OUT_COLS = 16;
constexpr int STRPOOL_BYTES = 256;

enum Domain : int32_t { DOM_I64 = 0, DOM_U64 = 1, DOM_F64 = 2, DOM_UTF8 = 3 };

enum ChainOp : int16_t {
  C_NOP = 0,
  C_ADD_I, C_SUB_I, C_RSUB_I, C_MUL_I, C_DIV_I, C_RDIV_I, C_MOD_I, C_RMOD_I,
  C_DIV_U, C_RDIV_U, C_MOD_U, C_RMOD_U,
  C_ADD_F, C_SUB_F, C_RSUB_F, C_MUL_F, C_DIV_F, C_RDIV_F,
  C_I2F, C_U2F, C_F2I, C_WRAP_I32, C_WRAP_U32, C_F2U
};

enum Cvt : int8_t { CVT_NONE = 0, CVT_I2F = 1, CVT_U2F = 2 };

union Val {
  int64_t i;
  uint64_t u;
  double d;
};

struct ColRef {
  const void* data;        // fixed width values / Utf8 bytes (NULL for a host-resident chunked column)
  const int32_t* offsets;  // Utf8 only
  int32_t dtype;
  int32_t chunk_shift;     // chunked: rows per chunk = 1 << chunk_shift
  const void* const* chunks;  // chunked: base pointer of every chunk (device-accessible host memory)
  const uint8_t* validity;  // one byte per row, 1 = valid; NULL when the column has no NULLs
};

struct ChainStep {
  int16_t op;     // ChainOp
  int8_t src;     // 0 = literal, 1 = column, 2 = none (unary step)
  int8_t cvt;     // conversion applied to the loaded column operand
  int32_t col;
  Val lit;
};

struct Chain {
  int32_t start_col;  // -1: start from the literal
  int32_t n_steps;
  Val start_lit;
  ChainStep steps[MAX_STEPS];
};

struct Term {
  int32_t domain;  // Domain
  int32_t cmp;     // FLOCKGPU_OP_EQ .. FLOCKGPU_OP_GE
  // numeric domains
  Chain lhs, rhs;
  // DOM_UTF8: column lhs_col compared with a pooled literal (rhs_col < 0) or another column
  int32_t lhs_col, rhs_col;
  int32_t lit_off, lit_len;
  uint32_t null_cols;  // bit c: a NULL in input column c makes this comparison NULL (Predicate::kleene)
  int32_t pad;
};

struct Predicate {
  int32_t n_terms;
  int32_t has_div_by_col;  // a division/modulo by a column: the kernel reports divide-by-zero
  // kleene = 1 (some referenced column has NULLs; at most 4 terms): the table is indexed by the terms' VALUE bits
  // (0 where the term is NULL) | their NULL bits << 4, and holds "the predicate is TRUE under SQL's three-valued
  // logic" -- FilterExec keeps a row only then (a NULL predicate drops the row, SURVEY.md Appendix C.3)
  int32_t kleene;
  int32_t pad;
  uint32_t lut[8];         // bit (b) of the table = truth value when the term bits spell b
  Term terms[MAX_TERMS];
  char strpool[STRPOOL_BYTES];
};

enum OutKind : int32_t { OUT_PASS = 0, OUT_COMPUTED = 1 };

struct OutCol {
  int32_t kind;       // OutKind
  int32_t src_col;    // OUT_PASS: input column
  int32_t out_dtype;  // storage type of the output column
  int32_t width;      // bytes per output value
  void* dst;
  Chain chain;        // OUT_COMPUTED
};

#include <cuda_runtime.h>
#define FG_HD __host__ __device__ __forceinline__
#ifdef __CUDA_ARCH__
#define FG_DADD(a, b) __dadd_rn(a, b)
#define FG_DSUB(a, b) __dsub_rn(a, b)
#define FG_DMUL(a, b) __dmul_rn(a, b)
#define FG_DDIV(a, b) __ddiv_rn(a, b)
#define FG_I2F(a) __ll2double_rn(a)
#define FG_U2F(a) __ull2double_rn(a)
#define FG_F2I(a) __double2ll_rz(a)
#define FG_F2U(a) __double2ull_rz(a)
#else  // host build of the same interpreter (flockgpu_selftest_* only; never on the product path)
// Float -> integer conversions only run on values that fit (cast_fits); the host forms still clamp, so that no input
// is undefined behaviour.
inline int64_t host_f2i(double d) {
  return d != d ? 0 : d >= 9223372036854775808.0 ? INT64_MAX : d < -9223372036854775808.0 ? INT64_MIN : static_cast<int64_t>(d);
}
inline uint64_t host_f2u(double d) { return !(d > -1.0) ? 0 : d >= 18446744073709551616.0 ? UINT64_MAX : static_cast<uint64_t>(d); }
#define FG_DADD(a, b) ((a) + (b))
#define FG_DSUB(a, b) ((a) - (b))
#define FG_DMUL(a, b) ((a) * (b))
#define FG_DDIV(a, b) ((a) / (b))
#define FG_I2F(a) static_cast<double>(a)
#define FG_U2F(a) static_cast<double>(a)
#define FG_F2I(a) host_f2i(a)
#define FG_F2U(a) host_f2u(a)
#endif

FG_HD Val load_val(const ColRef& c, int64_t row) {
  Val v;
  switch (c.dtype) {
    case FLOCKGPU_INT32: case FLOCKGPU_DATE32: v.i = static_cast<const int32_t*>(c.data)[row]; break;
    case FLOCKGPU_UINT32: v.u = static_cast<const uint32_t*>(c.data)[row]; break;
    case FLOCKGPU_FLOAT64: v.d = static_cast<const double*>(c.data)[row]; break;
    default: v.i = static_cast<const int64_t*>(c.data)[row]; break;  // Int64 / UInt64 / Timestamp
  }
  return v;
}

FG_HD void store_val(void* dst, int dtype, int64_t pos, Val v) {
  switch (dtype) {
    case FLOCKGPU_INT32: case FLOCKGPU_UINT32: case FLOCKGPU_DATE32: static_cast<int32_t*>(dst)[pos] = int32_t(v.i); break;
    case FLOCKGPU_FLOAT64: static_cast<double*>(dst)[pos] = v.d; break;
    default: static_cast<int64_t*>(dst)[pos] = v.i; break;
  }
}

FG_HD Val apply_step(int op, Val a, Val b, int* err) {
  Val r = a;
  switch (op) {
    case C_ADD_I: r.i = int64_t(uint64_t(a.i) + uint64_t(b.i)); break;
    case C_SUB_I: r.i = int64_t(uint64_t(a.i) - uint64_t(b.i)); break;
    case C_RSUB_I: r.i = int64_t(uint64_t(b.i) - uint64_t(a.i)); break;
    case C_MUL_I: r.i = int64_t(uint64_t(a.i) * uint64_t(b.i)); break;
    case C_DIV_I: if (b.i == 0) { *err = 1; r.i = 0; } else r.i = (b.i == -1) ? int64_t(0 - uint64_t(a.i)) : a.i / b.i; break;
    case C_RDIV_I: if (a.i == 0) { *err = 1; r.i = 0; } else r.i = (a.i == -1) ? int64_t(0 - uint64_t(b.i)) : b.i / a.i; break;
    case C_MOD_I: if (b.i == 0) { *err = 1; r.i = 0; } else r.i = (b.i == -1) ? 0 : a.i % b.i; break;
    case C_RMOD_I: if (a.i == 0) { *err = 1; r.i = 0; } else r.i = (a.i == -1) ? 0 : b.i % a.i; break;
    case C_DIV_U: if (b.u == 0) { *err = 1; r.u = 0; } else r.u = a.u / b.u; break;
    case C_RDIV_U: if (a.u == 0) { *err = 1; r.u = 0; } else r.u = b.u / a.u; break;
    case C_MOD_U: if (b.u == 0) { *err = 1; r.u = 0; } else r.u = a.u % b.u; break;
    case C_RMOD_U: if (a.u == 0) { *err = 1; r.u = 0; } else r.u = b.u % a.u; break;
    case C_ADD_F: r.d = FG_DADD(a.d, b.d); break;
    case C_SUB_F: r.d = FG_DSUB(a.d, b.d); break;
    case C_RSUB_F: r.d = FG_DSUB(b.d, a.d); break;
    case C_MUL_F: r.d = FG_DMUL(a.d, b.d); break;
    case C_DIV_F: r.d = FG_DDIV(a.d, b.d); break;
    case C_RDIV_F: r.d = FG_DDIV(b.d, a.d); break;
    case C_I2F: r.d = FG_I2F(a.i); break;
    case C_U2F: r.d = FG_U2F(a.u); break;
    case C_F2I: r.i = FG_F2I(a.d); break;
    case C_F2U: r.u = FG_F2U(a.d); break;
    case C_WRAP_I32: r.i = int64_t(int32_t(uint32_t(a.u))); break;
    case C_WRAP_U32: r.u = uint64_t(uint32_t(a.u)); break;
    default: break;
  }
  return r;
}

// An explicit CAST that can lose its value (Float64 to an integer type, an integer type to a narrower one or across
// signedness) yields NULL where the target type cannot hold the source value, as arrow-rs's numeric cast does
// (num::cast::cast returns None: NaN, +-inf, a float outside the range once truncated toward zero, an integer outside
// the range).  code = cast_code(domain of the source, target dtype); `v` is in the canonical form of the source.
FG_HD int64_t cast_code(int dom, int to) { return (int64_t(to) << 2) | dom; }

FG_HD bool cast_fits(int64_t code, Val v) {
  const int dom = int(code & 3), to = int(code >> 2);
  const bool wide = to != FLOCKGPU_INT32 && to != FLOCKGPU_UINT32 && to != FLOCKGPU_DATE32;
  const bool uns = to == FLOCKGPU_UINT32 || to == FLOCKGPU_UINT64;
  if (dom == DOM_F64) {
    // truncation toward zero keeps the open interval (min - 1, max + 1); every bound below is an exact double, and
    // -9223372036854777856 is the next double below -2^63
    const double below = uns ? -1.0 : wide ? -9223372036854777856.0 : -2147483649.0;
    const double above = wide ? (uns ? 18446744073709551616.0 : 9223372036854775808.0) : (uns ? 4294967296.0 : 2147483648.0);
    return v.d > below && v.d < above;  // false for NaN
  }
  if (dom == DOM_U64) return v.u <= (wide ? (uns ? UINT64_MAX : uint64_t(INT64_MAX)) : (uns ? uint64_t(UINT32_MAX) : uint64_t(INT32_MAX)));
  if (uns) return v.i >= 0 && (wide || v.i <= int64_t(UINT32_MAX));
  return wide || (v.i >= INT32_MIN && v.i <= INT32_MAX);
}

// Evaluates `c` for R rows at once: row[j] (j < R); rows < 0 are skipped.  The switch on the step
// opcode is outside the row loop.
template <int R>
FG_HD void eval_chain(const Chain& c, const ColRef* cols, const int64_t (&rows)[R], Val (&acc)[R], int* err) {
  if (c.start_col >= 0) {
    const ColRef col = cols[c.start_col];
#pragma unroll
    for (int j = 0; j < R; ++j) acc[j] = rows[j] >= 0 ? load_val(col, rows[j]) : Val{0};
  } else {
#pragma unroll
    for (int j = 0; j < R; ++j) acc[j] = c.start_lit;
  }
  for (int s = 0; s < c.n_steps; ++s) {
    const ChainStep st = c.steps[s];
    if (st.src == 1) {
      const ColRef col = cols[st.col];
#pragma unroll
      for (int j = 0; j < R; ++j) {
        if (rows[j] < 0) continue;
        Val b = load_val(col, rows[j]);
        if (st.cvt == CVT_I2F) b.d = FG_I2F(b.i);
        else if (st.cvt == CVT_U2F) b.d = FG_U2F(b.u);
        acc[j] = apply_step(st.op, acc[j], b, err);
      }
    } else {
#pragma unroll
      for (int j = 0; j < R; ++j) {
        // padded rows carry acc = 0: a reversed literal step (`lit / (col*k)`, `lit % (col*k)`) would raise a
        // spurious divide-by-zero on them
        if (rows[j] < 0) continue;
        acc[j] = apply_step(st.op, acc[j], st.lit, err);
      }
    }
  }
}

FG_HD bool compare_vals(int domain, int cmp, Val a, Val b) {
  int lt, eq;
  if (domain == DOM_I64) { lt = a.i < b.i; eq = a.i == b.i; }
  else if (domain == DOM_U64) { lt = a.u < b.u; eq = a.u == b.u; }
  else { lt = a.d < b.d; eq = a.d == b.d; if (a.d != a.d || b.d != b.d) { return cmp == FLOCKGPU_OP_NE; } }
  switch (cmp) {
    case FLOCKGPU_OP_EQ: return eq;
    case FLOCKGPU_OP_NE: return !eq;
    case FLOCKGPU_OP_LT: return lt;
    case FLOCKGPU_OP_LE: return lt || eq;
    case FLOCKGPU_OP_GT: return !(lt || eq);
    default: return !lt;  // GE
  }
}

// bytewise compare (UTF-8 byte order == code point order == Rust `str` Ord): <0, 0, >0
FG_HD int compare_bytes(const uint8_t* a, int na, const uint8_t* b, int nb) {
  int n = na < nb ? na : nb;
  for (int i = 0; i < n; ++i) {
    int d = int(a[i]) - int(b[i]);
    if (d) return d;
  }
  return na - nb;
}

FG_HD bool cmp_result(int cmp, int c) {
  switch (cmp) {
    case FLOCKGPU_OP_EQ: return c == 0;
    case FLOCKGPU_OP_NE: return c != 0;
    case FLOCKGPU_OP_LT: return c < 0;
    case FLOCKGPU_OP_LE: return c <= 0;
    case FLOCKGPU_OP_GT: return c > 0;
    default: return c >= 0;
  }
}

// Evaluates the whole predicate for R rows; bit j of the result = row j selected.
template <int R>
FG_HD unsigned eval_predicate(const Predicate& p, const ColRef* cols, const int64_t (&rows)[R], int* err) {
  unsigned bits[R];
#pragma unroll
  for (int j = 0; j < R; ++j) bits[j] = 0;
  for (int t = 0; t < p.n_terms; ++t) {
    const Term& term = p.terms[t];
    if (term.domain == DOM_UTF8) {
      const ColRef lc = cols[term.lhs_col];
#pragma unroll
      for (int j = 0; j < R; ++j) {
        if (rows[j] < 0) continue;
        int32_t lo = lc.offsets[rows[j]], hi = lc.offsets[rows[j] + 1];
        const uint8_t* a = static_cast<const uint8_t*>(lc.data) + lo;
        int c;
        if (term.rhs_col < 0) {
          c = compare_bytes(a, hi - lo, reinterpret_cast<const uint8_t*>(p.strpool) + term.lit_off, term.lit_len);
        } else {
          const ColRef rc = cols[term.rhs_col];
          int32_t rlo = rc.offsets[rows[j]], rhi = rc.offsets[rows[j] + 1];
          c = compare_bytes(a, hi - lo, static_cast<const uint8_t*>(rc.data) + rlo, rhi - rlo);
        }
        bits[j] |= unsigned(cmp_result(term.cmp, c)) << t;
      }
    } else {
      Val a[R], b[R];
      eval_chain<R>(term.lhs, cols, rows, a, err);
      eval_chain<R>(term.rhs, cols, rows, b, err);
#pragma unroll
      for (int j = 0; j < R; ++j) bits[j] |= unsigned(compare_vals(term.domain, term.cmp, a[j], b[j])) << t;
    }
  }
  if (p.kleene) {
#pragma unroll
    for (int j = 0; j < R; ++j) {
      if (rows[j] < 0) continue;
      unsigned nulls = 0;
      for (int t = 0; t < p.n_terms; ++t) {
        const unsigned m = p.terms[t].null_cols;
        for (int c = 0; m >> c; ++c)
          if (((m >> c) & 1u) && cols[c].validity && !cols[c].validity[rows[j]]) nulls |= 1u << t;
      }
      bits[j] = (bits[j] & ~nulls & 0xfu) | (nulls << 4);
    }
  }
  unsigned sel = 0;
#pragma unroll
  for (int j = 0; j < R; ++j) {
    unsigned b = bits[j];
    if (rows[j] >= 0) sel |= ((p.lut[b >> 5] >> (b & 31)) & 1u) << j;
  }
  return sel;
}

// ---- host-side compiler (expr_compile.cc) ---------------------------------------------------------
struct ExprTok;
struct Table;
}  // namespace fg
