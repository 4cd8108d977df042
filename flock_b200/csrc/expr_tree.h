// expr_tree.h -- the TREE form of the device expression program: a register program.
//
// expr_program.h runs two shapes: a left-deep CHAIN and a PREDICATE of comparison terms under a truth table.  Whatever
// does not fit them -- arithmetic over two compound operands, CASE, IN lists, IS [NOT] NULL, unary minus, NULL
// literals, booleans used as values, any number of nullable columns -- is lowered (expr_compile.cc) to a flat list of
// typed instructions  r[d] = op(r[a], r[b])  over TREE_REGS per-row registers.  One program may have several roots
// (every computed output of an operator); common sub-expressions are computed once and a register is re-used as
// soon as its value is dead.
//
// A register is the canonical 64-bit Val of expr_program.h plus a flag byte: TF_NULL (SQL NULL) and TF_ERR.  TF_ERR
// is "this value is the result of an integer division by zero": it travels with the value instead of raising the
// error at once, so that a CASE branch that is not taken, or a row whose divisor is NULL, raises nothing.  A root
// that carries TF_ERR sets the error flag (FLOCKGPU_ERR_EXECUTION, "Divide by zero").
//
// The register file is addressed by the program, so it cannot live in hardware registers without local-memory
// indexing: the kernels keep it in shared memory, [register][row][thread], which is conflict free and costs no
// stack; the host build of the same interpreter (flockgpu_selftest_eval_tree) keeps it in a local array.
// Arithmetic is apply_step's: same wrap, truncation and single-rounding rules as the chain form.
#pragma once

#include "expr_program.h"

namespace fg {

constexpr int TREE_REGS = 10;
constexpr int TREE_MAX_INSTR = 160;
constexpr int TREE_MAX_OUTS = 16;
constexpr int TREE_POOL_BYTES = 512;

enum TreeOp : int16_t {
  T_COL = 1,      // r[d] = column `col` (a Utf8 column loads its NULL flag only)
  T_LIT,          // r[d] = lit; a != 0: a NULL literal
  T_ARITH,        // r[d] = apply_step(sub, r[a], r[b]); b < 0: unary (conversions, wraps); lit != 0: an explicit CAST
                  // that can lose its value, lit = its cast_code: NULL where !cast_fits
  T_CMP,          // r[d] = r[a] CMP r[b]; sub = domain << 8 | (cmp - FLOCKGPU_OP_EQ)
  T_CMP_UTF8,     // r[d] = column `col` CMP (column `col2` | pooled literal lit = offset << 32 | length); sub = cmp
  T_AND, T_OR,    // Kleene
  T_NOT,
  T_IS_NULL, T_IS_NOT_NULL,
  T_SELECT,       // r[d] = r[c] is TRUE ? r[a] : r[b]   (a NULL condition takes r[b]: CASE falls through)
  T_STORE,        // output `col` = r[a]
  T_LIKE,         // r[d] = Utf8 column `col` LIKE pooled pattern lit (offset << 32 | length); sub = 1: NOT LIKE
  T_DATE_PART     // r[d] = date_part(sub = FLOCKGPU_DATE_PART_*, r[a]); lit = the operand's unit (DateUnit)
};

constexpr uint8_t TF_NULL = 1, TF_ERR = 2;

struct TreeInstr {
  int16_t op, sub;
  int8_t d, a, b, c;
  int32_t col, col2;
  Val lit;
};

struct TreeOut {
  void* dst;
  uint8_t* validity;  // one byte per row, or NULL when the result cannot be NULL
  int32_t dtype;
  int32_t pad;
};

struct TreeProgram {
  int32_t n_instr;
  int32_t result_reg;  // predicate programs: the register holding the verdict; -1 otherwise
  TreeInstr ins[TREE_MAX_INSTR];
  char pool[TREE_POOL_BYTES];
};

// The register file of one thread: R rows per register, consecutive slots STRIDE apart (the thread count when it is
// shared memory interleaved by thread, 1 for a private array).
template <int R, int STRIDE>
struct TreeRegs {
  Val* v;
  uint8_t* f;
  FG_HD Val& val(int reg, int j) const { return v[(reg * R + j) * STRIDE]; }
  FG_HD uint8_t& flag(int reg, int j) const { return f[(reg * R + j) * STRIDE]; }
};

// SQL LIKE without an escape character: '%' matches any run of characters, '_' exactly one UTF-8 code point, every
// other byte itself.  Greedy two-pointer match that backtracks to the last '%' only, so it needs no stack: the
// pattern up to that '%' is already matched, and a later '%' makes every earlier choice final.
FG_HD int next_code_point(const uint8_t* s, int i, int n) {
  ++i;
  while (i < n && (s[i] & 0xc0) == 0x80) ++i;
  return i;
}

FG_HD bool like_match(const uint8_t* s, int n, const uint8_t* p, int m) {
  int si = 0, pi = 0, star = -1, mark = 0;
  while (si < n) {
    if (pi < m && p[pi] == '%') {
      star = ++pi;
      mark = si;
    } else if (pi < m && p[pi] == '_') {
      ++pi;
      si = next_code_point(s, si, n);
    } else if (pi < m && p[pi] == s[si]) {
      ++pi;
      ++si;
    } else if (star >= 0) {
      pi = star;
      si = mark = next_code_point(s, mark, n);
    } else {
      return false;
    }
  }
  while (pi < m && p[pi] == '%') ++pi;
  return pi == m;
}

// The unit of a date_part operand: a Date32 counts days, a Timestamp seconds, milli-, micro- or nanoseconds.
enum DateUnit : int { DU_DAY = 0, DU_S, DU_MS, DU_US, DU_NS };

// Proleptic Gregorian year of `day` (days since 1970-01-01), year 0 included: civil_from_days (H. Hinnant), the
// inverse of the plan reader's days_from_civil, in 64-bit so that every day an Int64 timestamp can name is exact.
FG_HD int64_t year_of_day(int64_t day) {
  const int64_t z = day + 719468;
  const int64_t era = (z >= 0 ? z : z - 146096) / 146097;
  const int64_t doe = z - era * 146097;                                    // [0, 146096]
  const int64_t yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;  // [0, 399]
  const int64_t doy = doe - (365 * yoe + yoe / 4 - yoe / 100);             // [0, 365], from March 1st
  const int64_t mp = (5 * doy + 2) / 153;                                  // [0, 11], March = 0
  return yoe + era * 400 + (mp >= 10);                                     // January and February close the year
}

// date_part(field, v) for v counted in units of which PER_DAY make a day and PER_HOUR an hour.  The day is the floor
// of v / PER_DAY, so an instant before 1970 falls on its own day.  false: the result is NULL (a year beyond Int32).
template <int64_t PER_DAY, int64_t PER_HOUR>
FG_HD bool date_part_in(int field, int64_t v, int64_t* out) {
  int64_t day = v / PER_DAY, rem = v % PER_DAY;
  if (rem < 0) {
    --day;
    rem += PER_DAY;
  }
  if (field == FLOCKGPU_DATE_PART_HOUR) {
    *out = rem / PER_HOUR;
    return true;
  }
  const int64_t y = year_of_day(day);
  *out = y;
  return y >= INT32_MIN && y <= INT32_MAX;
}

// One switch on the unit, so that every divisor is a compile-time constant.
FG_HD bool date_part(int field, int unit, int64_t v, int64_t* out) {
  switch (unit) {
    case DU_S: return date_part_in<86400, 3600>(field, v, out);
    case DU_MS: return date_part_in<86400000, 3600000>(field, v, out);
    case DU_US: return date_part_in<86400000000ll, 3600000000ll>(field, v, out);
    case DU_NS: return date_part_in<86400000000000ll, 3600000000000ll>(field, v, out);
    default: return date_part_in<1, 1>(field, v, out);
  }
}

// Runs the program for R rows (rows[j] < 0: no row); returns bit j = the verdict register is TRUE for row j.
// `vec`: rows[0..4) are four consecutive rows starting at a multiple of four (R == 4): fixed-width columns are
// read and results written 16 bytes at a time where the buffers are aligned.
template <int R, class Regs>
FG_HD unsigned eval_tree(const TreeProgram& p, const ColRef* cols, const TreeOut* outs, const int64_t (&rows)[R], bool vec, const Regs& rf,
                         int* err) {
  for (int pc = 0; pc < p.n_instr; ++pc) {
    const TreeInstr in = p.ins[pc];
    switch (in.op) {
      case T_COL: {
        const ColRef col = cols[in.col];
        bool done = false;
#ifdef __CUDA_ARCH__
        if (R == 4 && vec && col.dtype != FLOCKGPU_UTF8) {
          const int w = (col.dtype == FLOCKGPU_INT32 || col.dtype == FLOCKGPU_UINT32 || col.dtype == FLOCKGPU_DATE32) ? 4 : 8;
          const char* src = static_cast<const char*>(col.data) + rows[0] * w;
          if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) {
            if (w == 4) {
              const int4 x = *reinterpret_cast<const int4*>(src);
              const int32_t xs[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
              for (int j = 0; j < R; ++j) {
                Val v;
                if (col.dtype != FLOCKGPU_UINT32) v.i = xs[j];
                else v.u = uint32_t(xs[j]);
                rf.val(in.d, j) = v;
              }
            } else {
              const longlong2 x = *reinterpret_cast<const longlong2*>(src);
              const longlong2 y = *reinterpret_cast<const longlong2*>(src + 16);
              const long long xs[4] = {x.x, x.y, y.x, y.y};
#pragma unroll
              for (int j = 0; j < R; ++j) {
                Val v;
                v.i = xs[j];
                rf.val(in.d, j) = v;
              }
            }
            done = true;
          }
        }
#endif
        if (!done) {
#pragma unroll
          for (int j = 0; j < R; ++j) {
            Val v;
            v.i = 0;
            if (rows[j] >= 0 && col.dtype != FLOCKGPU_UTF8) v = load_val(col, rows[j]);
            rf.val(in.d, j) = v;
          }
        }
#pragma unroll
        for (int j = 0; j < R; ++j)
          rf.flag(in.d, j) = (rows[j] < 0 || (col.validity && !col.validity[rows[j]])) ? TF_NULL : uint8_t(0);
        break;
      }
      case T_LIT:
#pragma unroll
        for (int j = 0; j < R; ++j) {
          rf.val(in.d, j) = in.lit;
          rf.flag(in.d, j) = (in.a || rows[j] < 0) ? TF_NULL : uint8_t(0);
        }
        break;
      case T_ARITH:
#pragma unroll
        for (int j = 0; j < R; ++j) {
          const uint8_t f = rf.flag(in.a, j) | (in.b >= 0 ? rf.flag(in.b, j) : uint8_t(0));
          Val v;
          v.i = 0;
          uint8_t nf = f;
          if (!(f & TF_NULL) && in.lit.i && !cast_fits(in.lit.i, rf.val(in.a, j))) {
            nf |= TF_NULL;
          } else if (!(f & TF_NULL)) {
            int e = 0;
            v = apply_step(in.sub, rf.val(in.a, j), in.b >= 0 ? rf.val(in.b, j) : v, &e);
            if (e) nf |= TF_ERR;
          }
          rf.val(in.d, j) = v;
          rf.flag(in.d, j) = nf;
        }
        break;
      case T_CMP:
#pragma unroll
        for (int j = 0; j < R; ++j) {
          const uint8_t f = rf.flag(in.a, j) | rf.flag(in.b, j);
          Val v;
          v.i = (f & TF_NULL) ? 0 : int64_t(compare_vals(in.sub >> 8, FLOCKGPU_OP_EQ + (in.sub & 0xff), rf.val(in.a, j), rf.val(in.b, j)));
          rf.val(in.d, j) = v;
          rf.flag(in.d, j) = f;
        }
        break;
      case T_CMP_UTF8: {
        const ColRef lc = cols[in.col];
#pragma unroll
        for (int j = 0; j < R; ++j) {
          Val v;
          v.i = 0;
          uint8_t f = TF_NULL;
          if (rows[j] >= 0) {
            const int64_t r = rows[j];
            f = (lc.validity && !lc.validity[r]) ? TF_NULL : uint8_t(0);
            const uint8_t* b = reinterpret_cast<const uint8_t*>(p.pool) + (in.lit.u >> 32);
            int nb = int(in.lit.u & 0xffffffffu);
            if (in.col2 >= 0) {
              const ColRef rc = cols[in.col2];
              if (rc.validity && !rc.validity[r]) f = TF_NULL;
              b = static_cast<const uint8_t*>(rc.data) + rc.offsets[r];
              nb = rc.offsets[r + 1] - rc.offsets[r];
            }
            if (!f) {
              const int32_t lo = lc.offsets[r], hi = lc.offsets[r + 1];
              v.i = int64_t(cmp_result(in.sub, compare_bytes(static_cast<const uint8_t*>(lc.data) + lo, hi - lo, b, nb)));
            }
          }
          rf.val(in.d, j) = v;
          rf.flag(in.d, j) = f;
        }
        break;
      }
      case T_LIKE: {
        const ColRef c = cols[in.col];
        const uint8_t* pat = reinterpret_cast<const uint8_t*>(p.pool) + (in.lit.u >> 32);
        const int np = int(in.lit.u & 0xffffffffu);
#pragma unroll
        for (int j = 0; j < R; ++j) {
          Val v;
          v.i = 0;
          uint8_t f = TF_NULL;
          if (rows[j] >= 0 && !(c.validity && !c.validity[rows[j]])) {
            f = 0;
            const int32_t lo = c.offsets[rows[j]], hi = c.offsets[rows[j] + 1];
            v.i = int64_t(like_match(static_cast<const uint8_t*>(c.data) + lo, hi - lo, pat, np) != (in.sub != 0));
          }
          rf.val(in.d, j) = v;
          rf.flag(in.d, j) = f;
        }
        break;
      }
      case T_DATE_PART:
#pragma unroll
        for (int j = 0; j < R; ++j) {
          uint8_t f = rf.flag(in.a, j);
          Val v;
          v.i = 0;
          if (!(f & TF_NULL) && !date_part(in.sub, int(in.lit.i), rf.val(in.a, j).i, &v.i)) {
            v.i = 0;
            f |= TF_NULL;
          }
          rf.val(in.d, j) = v;
          rf.flag(in.d, j) = f;
        }
        break;
      case T_AND:
      case T_OR:
#pragma unroll
        for (int j = 0; j < R; ++j) {
          const uint8_t fa = rf.flag(in.a, j), fb = rf.flag(in.b, j);
          const bool na = fa & TF_NULL, nb = fb & TF_NULL;
          const bool va = rf.val(in.a, j).i != 0, vb = rf.val(in.b, j).i != 0;
          // the value that decides on its own: FALSE for AND, TRUE for OR
          const bool dom = in.op == T_OR;
          const bool decided = (!na && va == dom) || (!nb && vb == dom);
          Val v;
          v.i = decided ? int64_t(dom) : ((na || nb) ? 0 : int64_t(!dom));
          rf.val(in.d, j) = v;
          rf.flag(in.d, j) = uint8_t(((fa | fb) & TF_ERR) | ((!decided && (na || nb)) ? TF_NULL : 0));
        }
        break;
      case T_NOT:
#pragma unroll
        for (int j = 0; j < R; ++j) {
          const uint8_t f = rf.flag(in.a, j);
          Val v;
          v.i = (f & TF_NULL) ? 0 : int64_t(rf.val(in.a, j).i == 0);
          rf.val(in.d, j) = v;
          rf.flag(in.d, j) = f;
        }
        break;
      case T_IS_NULL:
      case T_IS_NOT_NULL:
#pragma unroll
        for (int j = 0; j < R; ++j) {
          const uint8_t f = rf.flag(in.a, j);
          Val v;
          v.i = int64_t(((f & TF_NULL) != 0) == (in.op == T_IS_NULL));
          rf.val(in.d, j) = v;
          rf.flag(in.d, j) = uint8_t(f & TF_ERR);
        }
        break;
      case T_SELECT:
#pragma unroll
        for (int j = 0; j < R; ++j) {
          const uint8_t fc = rf.flag(in.c, j);
          const int src = (!(fc & TF_NULL) && rf.val(in.c, j).i != 0) ? in.a : in.b;
          const Val v = rf.val(src, j);
          const uint8_t f = rf.flag(src, j);
          rf.val(in.d, j) = v;
          rf.flag(in.d, j) = uint8_t((fc & TF_ERR) | f);
        }
        break;
      case T_STORE: {
        const TreeOut o = outs[in.col];
        bool done = false;
#pragma unroll
        for (int j = 0; j < R; ++j)
          if (rows[j] >= 0 && (rf.flag(in.a, j) & TF_ERR)) *err = 1;
#ifdef __CUDA_ARCH__
        if (R == 4 && vec) {
          // rows[0] is a multiple of four and output buffers are fresh allocations: 16-byte aligned stores
          if (o.dtype == FLOCKGPU_INT32 || o.dtype == FLOCKGPU_UINT32 || o.dtype == FLOCKGPU_DATE32) {
            int4 x;
            x.x = int32_t(rf.val(in.a, 0).i); x.y = int32_t(rf.val(in.a, 1 % R).i);
            x.z = int32_t(rf.val(in.a, 2 % R).i); x.w = int32_t(rf.val(in.a, 3 % R).i);
            *reinterpret_cast<int4*>(static_cast<int32_t*>(o.dst) + rows[0]) = x;
          } else {
            longlong2 x, y;
            x.x = rf.val(in.a, 0).i; x.y = rf.val(in.a, 1 % R).i;
            y.x = rf.val(in.a, 2 % R).i; y.y = rf.val(in.a, 3 % R).i;
            longlong2* q = reinterpret_cast<longlong2*>(static_cast<int64_t*>(o.dst) + rows[0]);
            q[0] = x;
            q[1] = y;
          }
          if (o.validity) {
            uint32_t w = 0;
#pragma unroll
            for (int j = 0; j < R; ++j) w |= uint32_t(!(rf.flag(in.a, j) & TF_NULL)) << (8 * j);
            *reinterpret_cast<uint32_t*>(o.validity + rows[0]) = w;
          }
          done = true;
        }
#endif
        if (!done) {
#pragma unroll
          for (int j = 0; j < R; ++j) {
            if (rows[j] < 0) continue;
            store_val(o.dst, o.dtype, rows[j], rf.val(in.a, j));
            if (o.validity) o.validity[rows[j]] = !(rf.flag(in.a, j) & TF_NULL);
          }
        }
        break;
      }
      default: break;
    }
  }
  unsigned sel = 0;
  if (p.result_reg >= 0) {
#pragma unroll
    for (int j = 0; j < R; ++j) {
      if (rows[j] < 0) continue;
      const uint8_t f = rf.flag(p.result_reg, j);
      if (f & TF_ERR) *err = 1;
      if (!(f & TF_NULL) && rf.val(p.result_reg, j).i != 0) sel |= 1u << j;
    }
  }
  return sel;
}

}  // namespace fg
