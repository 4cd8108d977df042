// oracle.cc -- CPU restatement of the DataFusion-6 operators on Flock's per-batch hot path.
//
// TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is linked, imported or executed by the product
// (flock_b200/, libflockgpu.so); only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
// `--impl reference` legs use it -- as the checker, never as the thing shipped.
//
// PARITY UNPINNED for NEXMark outputs: the reference's operators live in an un-vendored git dependency
// (datafusion = { git = "https://github.com/flock-lab/arrow-datafusion", branch = "flock" },
// flock/Cargo.toml:21, no Cargo.lock) and no Rust toolchain exists here, so the reference binary was
// never executed.  This file restates the PUBLISHED algorithms of apache/arrow-datafusion 6.0 /
// arrow-rs 6 (SURVEY.md Appendix C) and is pinned against (a) the reference's own toy goldens
// (flock/src/runtime/context.rs:428-592, flock/src/launcher/local.rs:169-234) and (b) an independent
// second implementation on Arrow C++ compute (oracle/acero_ref.py); see tests/test_oracle.py.
//
// Algorithms restated (each function cites the reference call site that exercises it):
//   eval_expr        PhysicalExpr::evaluate, vector-at-a-time with materialised intermediates like the
//                    arrow-rs kernels (cast / arithmetic / comparison / boolean), planner.rs:90,122,155,162
//   filter           arrow `filter` (order preserving), FilterExec
//   partition_ids    RepartitionExec::Hash: hash(keys) % n (shuffle_writer.rs:105-146); ahash is replaced
//                    by SplitMix64 -- hash values are unobservable (Appendix C.6)
//   group_by         HashAggregateExec: hash map keyed by the group values, groups in first-seen order,
//                    accumulators COUNT(u64) / SUM / MIN / MAX / AVG(sum f64, count u64) (Appendix C.7)
//   hash_join        HashJoinExec Inner: build map on the left, probe right rows in order, verify equality,
//                    emit (left, right) index pairs probe-row-major (Appendix C.8)
#include <algorithm>
#include <atomic>
#include <thread>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

extern "C" {

enum { T_BOOL = 0, T_I32 = 1, T_I64 = 2, T_U64 = 3, T_F64 = 4, T_TS = 5, T_UTF8 = 6, T_U32 = 7 };
enum {
  OP_COLUMN = 1, OP_LIT_I64 = 2, OP_LIT_F64 = 3, OP_LIT_UTF8 = 4, OP_CAST = 5,
  OP_ADD = 10, OP_SUB = 11, OP_MUL = 12, OP_DIV = 13, OP_MOD = 14,
  OP_EQ = 20, OP_NE = 21, OP_LT = 22, OP_LE = 23, OP_GT = 24, OP_GE = 25,
  OP_AND = 30, OP_OR = 31, OP_NOT = 32
};

struct OCol {
  int32_t dtype;
  int32_t pad;
  int64_t len;
  const void* data;        // values, or Utf8 bytes
  const int32_t* offsets;  // Utf8: offsets[0..len] (absolute into data)
};

struct OTok {
  int32_t op, dtype, col, str_len;
  int64_t i64;
  double f64;
  const char* str;
};

}  // extern "C"

namespace {

// A materialised intermediate array (or a scalar literal broadcast lazily).
struct Arr {
  int dtype = T_I64;
  bool scalar = false;
  int64_t si = 0;
  double sd = 0;
  std::string ss;
  std::vector<int64_t> i;   // I32 (widened) / I64 / U64 (bit pattern) / TS / U32 / BOOL(0,1)
  std::vector<double> d;    // F64
  const OCol* utf8 = nullptr;
};

bool is_float(int t) { return t == T_F64; }
bool is_unsigned(int t) { return t == T_U64 || t == T_U32; }

inline int64_t geti(const Arr& a, int64_t r) { return a.scalar ? a.si : a.i[r]; }
inline double getd(const Arr& a, int64_t r) { return a.scalar ? a.sd : a.d[r]; }

Arr load_col(const OCol& c) {
  Arr a;
  a.dtype = c.dtype;
  switch (c.dtype) {
    case T_I32: {
      a.i.resize(c.len);
      const int32_t* p = static_cast<const int32_t*>(c.data);
      for (int64_t r = 0; r < c.len; ++r) a.i[r] = p[r];
      break;
    }
    case T_U32: {
      a.i.resize(c.len);
      const uint32_t* p = static_cast<const uint32_t*>(c.data);
      for (int64_t r = 0; r < c.len; ++r) a.i[r] = p[r];
      break;
    }
    case T_I64: case T_U64: case T_TS: {
      a.i.assign(static_cast<const int64_t*>(c.data), static_cast<const int64_t*>(c.data) + c.len);
      break;
    }
    case T_F64:
      a.d.assign(static_cast<const double*>(c.data), static_cast<const double*>(c.data) + c.len);
      break;
    case T_UTF8:
      a.utf8 = &c;
      break;
    default: break;
  }
  return a;
}

// arrow-rs `cast` kernel for the numeric pairs DataFusion's coercion inserts
Arr cast_to(const Arr& x, int to, int64_t n) {
  Arr r;
  r.dtype = to;
  r.scalar = x.scalar;
  auto conv_i = [&](int64_t v) -> int64_t {
    if (to == T_I32) return int64_t(int32_t(uint32_t(uint64_t(v))));
    if (to == T_U32) return int64_t(uint64_t(uint32_t(uint64_t(v))));
    return v;
  };
  if (is_float(to)) {
    if (is_float(x.dtype)) return x;
    if (x.scalar) { r.sd = is_unsigned(x.dtype) ? double(uint64_t(x.si)) : double(x.si); return r; }
    r.d.resize(n);
    if (is_unsigned(x.dtype)) for (int64_t k = 0; k < n; ++k) r.d[k] = double(uint64_t(x.i[k]));
    else for (int64_t k = 0; k < n; ++k) r.d[k] = double(x.i[k]);
    return r;
  }
  if (is_float(x.dtype)) {
    if (x.scalar) { r.si = conv_i(int64_t(x.sd)); return r; }
    r.i.resize(n);
    for (int64_t k = 0; k < n; ++k) r.i[k] = conv_i(int64_t(x.d[k]));
    return r;
  }
  if (x.scalar) { r.si = conv_i(x.si); return r; }
  r.i.resize(n);
  for (int64_t k = 0; k < n; ++k) r.i[k] = conv_i(x.i[k]);
  return r;
}

int promote(int a, int b) {
  if (a == b) return a;
  if (a == T_F64 || b == T_F64) return T_F64;
  auto rank = [](int t) { return t == T_I32 ? 1 : t == T_U32 ? 2 : (t == T_I64 || t == T_TS) ? 3 : 4; };
  return rank(a) >= rank(b) ? a : b;
}

int arith(int op, const Arr& l0, const Arr& r0, int64_t n, Arr* out) {
  int T = promote(l0.dtype, r0.dtype);
  Arr l = cast_to(l0, T, n), r = cast_to(r0, T, n);
  out->dtype = T;
  out->scalar = false;
  if (T == T_F64) {
    if (op == OP_MOD) return -2;
    out->d.resize(n);
    for (int64_t k = 0; k < n; ++k) {
      double a = getd(l, k), b = getd(r, k);
      out->d[k] = op == OP_ADD ? a + b : op == OP_SUB ? a - b : op == OP_MUL ? a * b : a / b;
    }
    return 0;
  }
  out->i.resize(n);
  const bool u = is_unsigned(T);
  for (int64_t k = 0; k < n; ++k) {
    int64_t a = geti(l, k), b = geti(r, k), v;
    switch (op) {
      case OP_ADD: v = int64_t(uint64_t(a) + uint64_t(b)); break;
      case OP_SUB: v = int64_t(uint64_t(a) - uint64_t(b)); break;
      case OP_MUL: v = int64_t(uint64_t(a) * uint64_t(b)); break;
      case OP_DIV:
        if (b == 0) return -5;  // DataFusion: "Divide by zero"
        v = u ? int64_t(uint64_t(a) / uint64_t(b)) : (b == -1 ? int64_t(0 - uint64_t(a)) : a / b);
        break;
      default:
        if (b == 0) return -5;
        v = u ? int64_t(uint64_t(a) % uint64_t(b)) : (b == -1 ? 0 : a % b);  // truncated remainder (Rust %)
    }
    if (T == T_I32) v = int64_t(int32_t(uint32_t(uint64_t(v))));
    if (T == T_U32) v = int64_t(uint64_t(uint32_t(uint64_t(v))));
    out->i[k] = v;
  }
  return 0;
}

template <typename T>
inline bool cmp_op(int op, T a, T b) {
  switch (op) {
    case OP_EQ: return a == b;
    case OP_NE: return a != b;
    case OP_LT: return a < b;
    case OP_LE: return a <= b;
    case OP_GT: return a > b;
    default: return a >= b;
  }
}

inline int cmp_bytes(const char* a, int64_t na, const char* b, int64_t nb) {
  int c = memcmp(a, b, size_t(std::min(na, nb)));
  if (c) return c;
  return na < nb ? -1 : na > nb ? 1 : 0;
}

int compare(int op, const Arr& l0, const Arr& r0, int64_t n, Arr* out) {
  out->dtype = T_BOOL;
  out->scalar = false;
  out->i.resize(n);
  if (l0.dtype == T_UTF8 || r0.dtype == T_UTF8) {
    if (l0.dtype != T_UTF8 || r0.dtype != T_UTF8) return -2;
    auto str_at = [](const Arr& a, int64_t k, const char** p, int64_t* len) {
      if (a.utf8) {
        *p = static_cast<const char*>(a.utf8->data) + a.utf8->offsets[k];
        *len = a.utf8->offsets[k + 1] - a.utf8->offsets[k];
      } else {
        *p = a.ss.data();
        *len = int64_t(a.ss.size());
      }
    };
    for (int64_t k = 0; k < n; ++k) {
      const char *pa, *pb;
      int64_t la, lb;
      str_at(l0, k, &pa, &la);
      str_at(r0, k, &pb, &lb);
      out->i[k] = cmp_op<int>(op, cmp_bytes(pa, la, pb, lb), 0);
    }
    return 0;
  }
  int T = promote(l0.dtype, r0.dtype);
  Arr l = cast_to(l0, T, n), r = cast_to(r0, T, n);
  if (T == T_F64) for (int64_t k = 0; k < n; ++k) out->i[k] = cmp_op<double>(op, getd(l, k), getd(r, k));
  else if (is_unsigned(T)) for (int64_t k = 0; k < n; ++k) out->i[k] = cmp_op<uint64_t>(op, uint64_t(geti(l, k)), uint64_t(geti(r, k)));
  else for (int64_t k = 0; k < n; ++k) out->i[k] = cmp_op<int64_t>(op, geti(l, k), geti(r, k));
  return 0;
}

int eval_tokens(const OCol* cols, int n_cols, int64_t n, const OTok* toks, int n_toks, Arr* result) {
  std::vector<Arr> st;
  for (int t = 0; t < n_toks; ++t) {
    const OTok& k = toks[t];
    switch (k.op) {
      case OP_COLUMN:
        if (k.col < 0 || k.col >= n_cols) return -1;
        st.push_back(load_col(cols[k.col]));
        break;
      case OP_LIT_I64: {
        Arr a;
        a.scalar = true;
        a.dtype = (k.dtype == T_I32 || k.dtype == T_U32 || k.dtype == T_U64 || k.dtype == T_TS) ? k.dtype : T_I64;
        a.si = k.i64;
        st.push_back(a);
        break;
      }
      case OP_LIT_F64: {
        Arr a;
        a.scalar = true;
        a.dtype = T_F64;
        a.sd = k.f64;
        st.push_back(a);
        break;
      }
      case OP_LIT_UTF8: {
        Arr a;
        a.scalar = true;
        a.dtype = T_UTF8;
        a.ss.assign(k.str ? k.str : "", size_t(k.str_len));
        st.push_back(a);
        break;
      }
      case OP_CAST: {
        if (st.empty()) return -1;
        Arr x = std::move(st.back());
        st.pop_back();
        if (x.dtype == T_UTF8 || k.dtype == T_UTF8 || k.dtype == T_BOOL) return -2;
        st.push_back(cast_to(x, k.dtype, n));
        break;
      }
      case OP_NOT: {
        if (st.empty()) return -1;
        Arr& x = st.back();
        for (auto& v : x.i) v = !v;
        break;
      }
      default: {
        if (st.size() < 2) return -1;
        Arr r = std::move(st.back());
        st.pop_back();
        Arr l = std::move(st.back());
        st.pop_back();
        Arr o;
        int rc = 0;
        if (k.op >= OP_ADD && k.op <= OP_MOD) rc = arith(k.op, l, r, n, &o);
        else if (k.op >= OP_EQ && k.op <= OP_GE) rc = compare(k.op, l, r, n, &o);
        else if (k.op == OP_AND || k.op == OP_OR) {
          o.dtype = T_BOOL;
          o.i.resize(n);
          for (int64_t q = 0; q < n; ++q) o.i[q] = k.op == OP_AND ? (geti(l, q) && geti(r, q)) : (geti(l, q) || geti(r, q));
        } else return -1;
        if (rc) return rc;
        st.push_back(std::move(o));
      }
    }
  }
  if (st.size() != 1) return -1;
  *result = std::move(st[0]);
  return 0;
}

inline uint64_t splitmix(uint64_t x) {
  x += 0x9e3779b97f4a7c15ull;
  x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
  x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}

// Serialises the key columns of row r into a byte string (fixed width raw, Utf8 length-prefixed).
inline void key_bytes(const OCol* cols, const int32_t* keys, int n_keys, int64_t r, std::string* out) {
  out->clear();
  for (int k = 0; k < n_keys; ++k) {
    const OCol& c = cols[keys[k]];
    if (c.dtype == T_UTF8) {
      int32_t lo = c.offsets[r], len = c.offsets[r + 1] - lo;
      out->append(reinterpret_cast<const char*>(&len), 4);
      out->append(static_cast<const char*>(c.data) + lo, size_t(len));
    } else if (c.dtype == T_I32 || c.dtype == T_U32) {
      out->append(static_cast<const char*>(c.data) + r * 4, 4);
    } else {
      out->append(static_cast<const char*>(c.data) + r * 8, 8);
    }
  }
}

inline uint64_t hash_bytes(const std::string& s) {
  uint64_t h = 0x243f6a8885a308d3ull;
  size_t i = 0;
  for (; i + 8 <= s.size(); i += 8) {
    uint64_t w;
    memcpy(&w, s.data() + i, 8);
    h = splitmix(h ^ w);
  }
  uint64_t w = 0;
  memcpy(&w, s.data() + i, s.size() - i);
  return splitmix(h ^ w ^ (uint64_t(s.size()) << 56));
}

struct StrHash {
  size_t operator()(const std::string& s) const { return size_t(hash_bytes(s)); }
};

}  // namespace

extern "C" {

// ---- PhysicalExpr::evaluate ---------------------------------------------------------------------------
// Predicate: out_mask[n] (0/1).  Returns 0, or <0 (-1 malformed, -2 unsupported, -5 divide by zero).
int orc_eval_predicate(const OCol* cols, int n_cols, int64_t n, const OTok* toks, int n_toks, uint8_t* out_mask) {
  Arr r;
  int rc = eval_tokens(cols, n_cols, n, toks, n_toks, &r);
  if (rc) return rc;
  if (r.dtype != T_BOOL) return -1;
  for (int64_t k = 0; k < n; ++k) out_mask[k] = uint8_t(r.scalar ? r.si != 0 : r.i[k] != 0);
  return 0;
}

// Value expression: writes the result with its natural storage width; *out_dtype receives the type.
int orc_eval_value(const OCol* cols, int n_cols, int64_t n, const OTok* toks, int n_toks, void* out, int32_t* out_dtype) {
  Arr r;
  int rc = eval_tokens(cols, n_cols, n, toks, n_toks, &r);
  if (rc) return rc;
  *out_dtype = r.dtype;
  if (r.dtype == T_F64) {
    double* o = static_cast<double*>(out);
    for (int64_t k = 0; k < n; ++k) o[k] = getd(r, k);
  } else if (r.dtype == T_I32 || r.dtype == T_U32) {
    int32_t* o = static_cast<int32_t*>(out);
    for (int64_t k = 0; k < n; ++k) o[k] = int32_t(geti(r, k));
  } else if (r.dtype == T_UTF8 || r.dtype == T_BOOL) {
    return -2;
  } else {
    int64_t* o = static_cast<int64_t*>(out);
    for (int64_t k = 0; k < n; ++k) o[k] = geti(r, k);
  }
  return 0;
}

int32_t orc_infer_dtype(const OCol* cols, int n_cols, const OTok* toks, int n_toks) {
  Arr r;
  // evaluate on zero rows: types propagate without touching data
  std::vector<OCol> empty(cols, cols + n_cols);
  for (auto& c : empty) c.len = 0;
  if (eval_tokens(empty.data(), n_cols, 0, toks, n_toks, &r)) return -1;
  return r.dtype;
}

// ---- arrow `filter`: indices of the set mask entries ---------------------------------------------------
int64_t orc_mask_to_indices(const uint8_t* mask, int64_t n, int64_t* out_idx) {
  int64_t m = 0;
  for (int64_t k = 0; k < n; ++k)
    if (mask[k]) out_idx[m++] = k;
  return m;
}

// ---- RepartitionExec::Hash ------------------------------------------------------------------------------
int orc_partition_ids(const OCol* cols, const int32_t* keys, int n_keys, int64_t n, int n_parts, int32_t* out_pid) {
  std::string kb;
  for (int64_t r = 0; r < n; ++r) {
    key_bytes(cols, keys, n_keys, r, &kb);
    out_pid[r] = int32_t(hash_bytes(kb) % uint64_t(n_parts));
  }
  return 0;
}

// ---- HashAggregateExec -----------------------------------------------------------------------------------
// accumulator kinds
enum { A_COUNT = 0, A_SUM_I = 1, A_SUM_F = 2, A_MIN_I = 3, A_MAX_I = 4, A_MIN_U = 5, A_MAX_U = 6, A_MIN_F = 7, A_MAX_F = 8 };
struct OAcc {
  int32_t kind;
  int32_t col;  // value column (-1: COUNT(*)); int columns are read widened to int64, f64 as double
};

// Groups rows by the key columns (first-seen order).  out_first_row[g] = first row of group g;
// out_state[a * n + g] = accumulator a of group g (int64 / uint64 / double bit patterns).
// Returns the number of groups.
int64_t orc_group_by(const OCol* cols, const int32_t* keys, int n_keys, int64_t n, const OAcc* accs, int n_accs, int64_t* out_first_row,
                     uint64_t* out_state) {
  std::unordered_map<std::string, int64_t, StrHash> map;
  map.reserve(size_t(n / 4 + 16));
  std::string kb;
  int64_t n_groups = 0;
  auto load_i = [&](const OCol& c, int64_t r) -> int64_t {
    switch (c.dtype) {
      case T_I32: return static_cast<const int32_t*>(c.data)[r];
      case T_U32: return static_cast<const uint32_t*>(c.data)[r];
      default: return static_cast<const int64_t*>(c.data)[r];
    }
  };
  auto load_d = [&](const OCol& c, int64_t r) -> double {
    if (c.dtype == T_F64) return static_cast<const double*>(c.data)[r];
    if (c.dtype == T_U64 || c.dtype == T_U32) return double(uint64_t(load_i(c, r)));
    return double(load_i(c, r));
  };
  auto f64_bits = [](double d) {
    uint64_t b;
    memcpy(&b, &d, 8);
    return b;
  };
  // the IEEE total order as an unsigned order: a set sign bit flips every bit, a clear one only the sign
  auto total_key = [](uint64_t b) { return (b >> 63) ? ~b : (b ^ (uint64_t(1) << 63)); };
  for (int64_t r = 0; r < n; ++r) {
    int64_t g;
    if (n_keys == 0) {
      g = 0;
      if (n_groups == 0) {
        n_groups = 1;
        out_first_row[0] = r;
        g = -1;
      }
    } else {
      key_bytes(cols, keys, n_keys, r, &kb);
      auto it = map.find(kb);
      if (it == map.end()) {
        map.emplace(kb, n_groups);
        out_first_row[n_groups] = r;
        g = -1;
      } else {
        g = it->second;
      }
    }
    const bool fresh = g < 0;
    if (fresh) g = n_keys == 0 ? 0 : n_groups++;
    for (int a = 0; a < n_accs; ++a) {
      uint64_t* s = &out_state[int64_t(a) * n + g];
      const OAcc& ac = accs[a];
      switch (ac.kind) {
        case A_COUNT: *s = fresh ? 1 : *s + 1; break;
        case A_SUM_I: { int64_t v = load_i(cols[ac.col], r); *s = fresh ? uint64_t(v) : *s + uint64_t(v); break; }
        // SUM starts at +0.0: a group of -0.0 sums to +0.0 (Appendix C.7)
        case A_SUM_F: { double v = load_d(cols[ac.col], r), cur; memcpy(&cur, s, 8); cur = (fresh ? 0.0 : cur) + v; memcpy(s, &cur, 8); break; }
        case A_MIN_I: { int64_t v = load_i(cols[ac.col], r); if (fresh || v < int64_t(*s)) *s = uint64_t(v); break; }
        case A_MAX_I: { int64_t v = load_i(cols[ac.col], r); if (fresh || v > int64_t(*s)) *s = uint64_t(v); break; }
        case A_MIN_U: { uint64_t v = uint64_t(load_i(cols[ac.col], r)); if (fresh || v < *s) *s = v; break; }
        case A_MAX_U: { uint64_t v = uint64_t(load_i(cols[ac.col], r)); if (fresh || v > *s) *s = v; break; }
        // MIN / MAX of Float64 follow the IEEE total order (f64::total_cmp): -NaN < -inf < -0.0 < +0.0 < +inf < +NaN
        case A_MIN_F: { uint64_t v = f64_bits(load_d(cols[ac.col], r)); if (fresh || total_key(v) < total_key(*s)) *s = v; break; }
        case A_MAX_F: { uint64_t v = f64_bits(load_d(cols[ac.col], r)); if (fresh || total_key(v) > total_key(*s)) *s = v; break; }
      }
    }
  }
  return n_groups;
}

// ---- HashJoinExec (Inner) ------------------------------------------------------------------------------------
// A key with a NaN component matches nothing, NaN itself included (DataFusion confirms hash candidates with `==`);
// other Float64 components compare by bit pattern, so -0.0 and +0.0 do not meet.
inline bool key_has_nan(const OCol* cols, const int32_t* keys, int n_keys, int64_t r) {
  for (int k = 0; k < n_keys; ++k) {
    const OCol& c = cols[keys[k]];
    if (c.dtype == T_F64 && std::isnan(static_cast<const double*>(c.data)[r])) return true;
  }
  return false;
}

// Returns the number of pairs; writes up to `cap` pairs (call once with cap = 0 to size the output).
int64_t orc_hash_join(const OCol* lcols, const int32_t* lkeys, int64_t ln, const OCol* rcols, const int32_t* rkeys, int64_t rn, int n_keys,
                      int64_t* out_left, int64_t* out_right, int64_t cap) {
  std::unordered_map<std::string, std::vector<int64_t>, StrHash> map;
  map.reserve(size_t(ln + 16));
  std::string kb;
  for (int64_t r = 0; r < ln; ++r) {
    if (key_has_nan(lcols, lkeys, n_keys, r)) continue;
    key_bytes(lcols, lkeys, n_keys, r, &kb);
    map[kb].push_back(r);
  }
  int64_t m = 0;
  for (int64_t r = 0; r < rn; ++r) {
    if (key_has_nan(rcols, rkeys, n_keys, r)) continue;
    key_bytes(rcols, rkeys, n_keys, r, &kb);
    auto it = map.find(kb);
    if (it == map.end()) continue;
    for (int64_t l : it->second) {
      if (m < cap) {
        out_left[m] = l;
        out_right[m] = r;
      }
      ++m;
    }
  }
  return m;
}

// ---- fused CPU pipelines timed as bench.py's cpu_baseline ----------------------------------------------------
// NEXMark q2 on ONE record batch, step by step as DataFusion executes it (planner.rs:120-124):
//   CAST(auction AS Int64) -> `% 123` -> `= 0` (three materialised arrow kernels) -> filter(auction), filter(price).
// Returns the number of surviving rows; out_* need room for n values.
int64_t orc_q2_batch(const int32_t* auction, const int32_t* price, int64_t n, int64_t modulus, int64_t rhs, int64_t* scratch_i64,
                     uint8_t* scratch_mask, int32_t* out_auction, int32_t* out_price) {
  for (int64_t k = 0; k < n; ++k) scratch_i64[k] = int64_t(auction[k]);          // cast kernel
  for (int64_t k = 0; k < n; ++k) scratch_i64[k] = scratch_i64[k] % modulus;      // modulus kernel
  for (int64_t k = 0; k < n; ++k) scratch_mask[k] = scratch_i64[k] == rhs;        // eq kernel
  int64_t m = 0;
  for (int64_t k = 0; k < n; ++k)                                                 // filter kernel, column 1
    if (scratch_mask[k]) out_auction[m++] = auction[k];
  m = 0;
  for (int64_t k = 0; k < n; ++k)                                                 // filter kernel, column 2
    if (scratch_mask[k]) out_price[m++] = price[k];
  return m;
}


// NEXMark q2 over a whole relation, partition-parallel the way DataFusion runs the plan (planner.rs:120-124 with
// target_partitions = n, flock/src/configs/flock.toml:113): RepartitionExec(RoundRobinBatch(n)) deals batch b to
// partition b % n, every partition is one task (here: drawn by a pool of native threads) running FilterExec batch by batch through the
// same three materialised kernels as orc_q2_batch, CoalesceBatchesExec + ProjectionExec append the survivors to the
// partition's output, and `collect` concatenates the partitions in partition order.  No Python inside the timed call.
//   auction[b] / price[b] / rows[b]: the record batches; out_*: room for the total row count.
//   part_rows[p] receives the output rows of partition p (for the caller's checks).  Returns the output row count.
int64_t orc_q2_collect(const int32_t* const* auction, const int32_t* const* price, const int64_t* rows, int32_t n_batches, int64_t modulus, int64_t rhs,
                       int32_t n_partitions, int32_t n_threads, int32_t* out_auction, int32_t* out_price, int64_t* part_rows) {
  if (n_partitions < 1) n_partitions = 1;
  if (n_threads < 1) n_threads = 1;
  std::vector<std::vector<int32_t>> pa(n_partitions), pp(n_partitions);
  int64_t max_rows = 0;
  for (int32_t b = 0; b < n_batches; ++b) max_rows = std::max(max_rows, rows[b]);
  // a pool of n_threads workers draws partitions from a shared counter (this image's gcc ships without libgomp, so
  // the "OpenMP" arm of BASELINE.md section 3 is std::thread; the schedule is the same dynamic one)
  std::atomic<int32_t> next{0};
  auto worker = [&]() {
    std::vector<int64_t> scratch(size_t(max_rows) + 1);
    std::vector<uint8_t> mask(size_t(max_rows) + 1);
    std::vector<int32_t> oa(size_t(max_rows) + 1), op(size_t(max_rows) + 1);
    for (int32_t p = next.fetch_add(1); p < n_partitions; p = next.fetch_add(1)) {
      for (int32_t b = p; b < n_batches; b += n_partitions) {
        const int64_t m = orc_q2_batch(auction[b], price[b], rows[b], modulus, rhs, scratch.data(), mask.data(), oa.data(), op.data());
        pa[p].insert(pa[p].end(), oa.begin(), oa.begin() + m);
        pp[p].insert(pp[p].end(), op.begin(), op.begin() + m);
      }
    }
  };
  const int32_t n_workers = std::min(n_threads, n_partitions);
  std::vector<std::thread> pool;
  for (int32_t t = 1; t < n_workers; ++t) pool.emplace_back(worker);
  worker();
  for (std::thread& t : pool) t.join();
  int64_t total = 0;
  for (int32_t p = 0; p < n_partitions; ++p) {
    std::copy(pa[p].begin(), pa[p].end(), out_auction + total);
    std::copy(pp[p].begin(), pp[p].end(), out_price + total);
    if (part_rows) part_rows[p] = int64_t(pa[p].size());
    total += int64_t(pa[p].size());
  }
  return total;
}


// ---- the N > 1 CPU arm of bench.py: NEXMark q8 over one rank's share, executed natively the way the plan runs ----------
// Plan (benchmarks/src/nexmark/query/q8.sql, q8_plan.fmt; shapes planner.rs:152-171, stage.rs:535-543, :597-601):
//   P = DISTINCT (p_id, name) over person, A = DISTINCT seller over auction, P JOIN A ON p_id = seller -> (p_id, name).
//   Each DISTINCT is HashAggregate(Partial) per input partition -> RepartitionExec(Hash) -> HashAggregate(FinalPartitioned);
//   the join is Partitioned on the same routing.  Input batches are dealt round-robin to n_partitions input partitions
//   (RepartitionExec(RoundRobinBatch)); a pool of native threads draws the partitions of each phase from a counter.
// Output: p_id / name (offsets + bytes) of the join result, partitions in order; returns the row count.
}  // extern "C" (the helpers below are templates)
namespace {

struct RowRef {
  int32_t batch, row;
};
inline uint64_t q8_mix(uint64_t k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdull;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ull;
  k ^= k >> 33;
  return k;
}
// open-addressing set of row references; equality and hash are supplied by the caller
template <class Hash, class Eq>
struct RefSet {
  std::vector<int64_t> slot;  // (batch << 32) | row, -1 = free
  uint64_t mask;
  Hash hash;
  Eq eq;
  RefSet(size_t n, Hash h, Eq e) : hash(h), eq(e) {
    size_t cap = 16;
    while (cap < 2 * n) cap <<= 1;
    slot.assign(cap, -1);
    mask = cap - 1;
  }
  // true when (b, r) was new
  bool insert(int32_t b, int32_t r) {
    uint64_t i = hash(b, r) & mask;
    while (true) {
      const int64_t cur = slot[i];
      if (cur < 0) {
        slot[i] = (int64_t(b) << 32) | uint32_t(r);
        return true;
      }
      if (eq(int32_t(cur >> 32), int32_t(cur & 0xffffffff), b, r)) return false;
      i = (i + 1) & mask;
    }
  }
};

}  // namespace

extern "C" {

int64_t orc_q8_collect(const int32_t* const* p_id, const int32_t* const* name_off, const uint8_t* const* name_data, const int64_t* p_rows, int32_t n_p_batches,
                       const int32_t* const* seller, const int64_t* a_rows, int32_t n_a_batches, int32_t n_partitions, int32_t n_threads, int32_t* out_pid,
                       int32_t* out_name_off, uint8_t* out_name_data) {
  const int32_t P = std::max(1, n_partitions);
  const int32_t T = std::max(1, std::min(n_threads, P));
  auto run = [&](auto&& task) {
    std::atomic<int32_t> next{0};
    auto worker = [&]() {
      for (int32_t p = next.fetch_add(1); p < P; p = next.fetch_add(1)) task(p);
    };
    std::vector<std::thread> pool;
    for (int32_t t = 1; t < T; ++t) pool.emplace_back(worker);
    worker();
    for (std::thread& t : pool) t.join();
  };
  auto name_len = [&](int32_t b, int32_t r) { return name_off[b][r + 1] - name_off[b][r]; };
  auto p_hash = [&](int32_t b, int32_t r) {
    uint64_t h = q8_mix(uint32_t(p_id[b][r]));
    const uint8_t* s = name_data[b] + name_off[b][r];
    for (int32_t i = 0, n = name_len(b, r); i < n; ++i) h = (h ^ s[i]) * 0x100000001b3ull;
    return q8_mix(h);
  };
  auto p_eq = [&](int32_t b1, int32_t r1, int32_t b2, int32_t r2) {
    if (p_id[b1][r1] != p_id[b2][r2]) return false;
    const int32_t n = name_len(b1, r1);
    return n == name_len(b2, r2) && !memcmp(name_data[b1] + name_off[b1][r1], name_data[b2] + name_off[b2][r2], size_t(n));
  };
  auto route = [&](int32_t key) { return int32_t((q8_mix(uint32_t(key)) >> 32) * uint64_t(P) >> 32); };
  // ---- phase 1: Partial DISTINCT per input partition, then the hash repartition of its groups
  const size_t np = size_t(P);
  std::vector<std::vector<std::vector<RowRef>>> p_parts{np, std::vector<std::vector<RowRef>>{np}};   // [source][destination]
  std::vector<std::vector<std::vector<int32_t>>> a_parts{np, std::vector<std::vector<int32_t>>{np}};
  run([&](int32_t p) {
    size_t rows = 0;
    for (int32_t b = p; b < n_p_batches; b += P) rows += size_t(p_rows[b]);
    RefSet<decltype(p_hash), decltype(p_eq)> groups(rows, p_hash, p_eq);
    for (int32_t b = p; b < n_p_batches; b += P)
      for (int32_t r = 0; r < int32_t(p_rows[b]); ++r)
        if (groups.insert(b, r)) p_parts[size_t(p)][size_t(route(p_id[b][r]))].push_back(RowRef{b, r});
    size_t arows = 0;
    for (int32_t b = p; b < n_a_batches; b += P) arows += size_t(a_rows[b]);
    size_t cap = 16;
    while (cap < 2 * arows) cap <<= 1;
    std::vector<int64_t> set(cap, -1);
    for (int32_t b = p; b < n_a_batches; b += P)
      for (int64_t r = 0; r < a_rows[b]; ++r) {
        const int32_t k = seller[b][r];
        uint64_t i = q8_mix(uint32_t(k)) & (cap - 1);
        while (set[i] >= 0 && int32_t(set[i]) != k) i = (i + 1) & (cap - 1);
        if (set[i] < 0) {
          set[i] = int64_t(uint32_t(k));
          a_parts[size_t(p)][size_t(route(k))].push_back(k);
        }
      }
  });
  // ---- phase 2: FinalPartitioned DISTINCTs of one output partition, then its join (build P, probe A: probe = membership)
  std::vector<std::vector<int32_t>> o_pid{np}, o_len{np};
  std::vector<std::vector<uint8_t>> o_bytes{np};
  run([&](int32_t q) {
    size_t n_p = 0, n_a = 0;
    for (int32_t p = 0; p < P; ++p) {
      n_p += p_parts[size_t(p)][size_t(q)].size();
      n_a += a_parts[size_t(p)][size_t(q)].size();
    }
    size_t cap = 16;
    while (cap < 2 * n_a) cap <<= 1;
    std::vector<int64_t> sellers(cap, -1);
    for (int32_t p = 0; p < P; ++p)
      for (int32_t k : a_parts[size_t(p)][size_t(q)]) {
        uint64_t i = q8_mix(uint32_t(k)) & (cap - 1);
        while (sellers[i] >= 0 && int32_t(sellers[i]) != k) i = (i + 1) & (cap - 1);
        sellers[i] = int64_t(uint32_t(k));
      }
    RefSet<decltype(p_hash), decltype(p_eq)> groups(n_p, p_hash, p_eq);
    for (int32_t p = 0; p < P; ++p)
      for (const RowRef& ref : p_parts[size_t(p)][size_t(q)]) {
        if (!groups.insert(ref.batch, ref.row)) continue;
        const int32_t k = p_id[ref.batch][ref.row];
        uint64_t i = q8_mix(uint32_t(k)) & (cap - 1);
        while (sellers[i] >= 0 && int32_t(sellers[i]) != k) i = (i + 1) & (cap - 1);
        if (sellers[i] < 0) continue;
        o_pid[size_t(q)].push_back(k);
        const int32_t n = name_len(ref.batch, ref.row);
        o_len[size_t(q)].push_back(n);
        const uint8_t* sp = name_data[ref.batch] + name_off[ref.batch][ref.row];
        o_bytes[size_t(q)].insert(o_bytes[size_t(q)].end(), sp, sp + n);
      }
  });
  // ---- collect: the partitions one behind the other
  int64_t rows = 0, bytes = 0;
  out_name_off[0] = 0;
  for (int32_t q = 0; q < P; ++q) {
    std::copy(o_pid[size_t(q)].begin(), o_pid[size_t(q)].end(), out_pid + rows);
    for (size_t i = 0; i < o_len[size_t(q)].size(); ++i) {
      bytes += o_len[size_t(q)][i];
      out_name_off[rows + int64_t(i) + 1] = int32_t(bytes);
    }
    std::copy(o_bytes[size_t(q)].begin(), o_bytes[size_t(q)].end(), out_name_data + (bytes - int64_t(o_bytes[size_t(q)].size())));
    rows += int64_t(o_pid[size_t(q)].size());
  }
  return rows;
}


// ---- NEXMark q5 over one window, natively (the CPU figure beside bench.py's `queries.q5`) -------------------------------------
// Plan (benchmarks/src/nexmark/query/q5.sql, q5_plan.fmt; shapes stage.rs:535-543, :597-601): AuctionBids = COUNT(*) GROUP BY
// auction as HashAggregate(Partial) per input partition -> RepartitionExec(Hash[auction]) -> HashAggregate(FinalPartitioned);
// MaxBids = MAX(num) over it; join num = maxn.  The duplicated COUNT subtree of the reference plan is evaluated once
// (SURVEY.md 8d allows the CSE).  Output: every (auction, num) with num = MAX(num); returns the row count.
int64_t orc_q5_collect(const int32_t* const* auction, const int64_t* rows, int32_t n_batches, int32_t n_partitions, int32_t n_threads, int32_t* out_auction,
                       uint64_t* out_num, int64_t out_capacity) {
  const int32_t P = std::max(1, n_partitions);
  const int32_t T = std::max(1, std::min(n_threads, P));
  const size_t np = size_t(P);
  auto run = [&](auto&& task) {
    std::atomic<int32_t> next{0};
    auto worker = [&]() {
      for (int32_t p = next.fetch_add(1); p < P; p = next.fetch_add(1)) task(p);
    };
    std::vector<std::thread> pool;
    for (int32_t t = 1; t < T; ++t) pool.emplace_back(worker);
    worker();
    for (std::thread& t : pool) t.join();
  };
  auto mix = [](uint64_t k) {
    k ^= k >> 33;
    k *= 0xff51afd7ed558ccdull;
    k ^= k >> 33;
    k *= 0xc4ceb9fe1a85ec53ull;
    k ^= k >> 33;
    return k;
  };
  struct Counts {  // open addressing, key = auction, grows by doubling
    std::vector<int64_t> key;  // -1 = free
    std::vector<uint64_t> cnt;
    size_t used = 0;
    Counts() : key(1024, -1), cnt(1024, 0) {}
  };
  auto add = [&](Counts& c, int32_t k, uint64_t n, auto&& self) -> void {
    if (2 * (c.used + 1) > c.key.size()) {
      Counts bigger;
      bigger.key.assign(c.key.size() * 4, -1);
      bigger.cnt.assign(c.key.size() * 4, 0);
      for (size_t i = 0; i < c.key.size(); ++i)
        if (c.key[i] >= 0) self(bigger, int32_t(c.key[i]), c.cnt[i], self);
      c = std::move(bigger);
    }
    uint64_t i = mix(uint32_t(k)) & (c.key.size() - 1);
    while (c.key[i] >= 0 && int32_t(c.key[i]) != k) i = (i + 1) & (c.key.size() - 1);
    if (c.key[i] < 0) {
      c.key[i] = int64_t(uint32_t(k));
      ++c.used;
    }
    c.cnt[i] += n;
  };
  auto route = [&](int32_t key) { return int32_t((mix(uint32_t(key)) >> 32) * uint64_t(P) >> 32); };
  // phase 1: Partial COUNT per input partition, its groups routed by hash(auction)
  std::vector<std::vector<std::vector<std::pair<int32_t, uint64_t>>>> parts{np, std::vector<std::vector<std::pair<int32_t, uint64_t>>>{np}};
  run([&](int32_t p) {
    Counts c;
    for (int32_t b = p; b < n_batches; b += P)
      for (int64_t r = 0; r < rows[b]; ++r) add(c, auction[b][r], 1, add);
    for (size_t i = 0; i < c.key.size(); ++i)
      if (c.key[i] >= 0) parts[size_t(p)][size_t(route(int32_t(c.key[i])))].emplace_back(int32_t(c.key[i]), c.cnt[i]);
  });
  // phase 2: FinalPartitioned COUNT per output partition; its MAX
  std::vector<Counts> finals{np};
  std::vector<uint64_t> part_max(np, 0);
  run([&](int32_t q) {
    Counts& c = finals[size_t(q)];
    for (int32_t p = 0; p < P; ++p)
      for (const auto& kv : parts[size_t(p)][size_t(q)]) add(c, kv.first, kv.second, add);
    uint64_t m = 0;
    for (size_t i = 0; i < c.key.size(); ++i)
      if (c.key[i] >= 0) m = std::max(m, c.cnt[i]);
    part_max[size_t(q)] = m;
  });
  // MaxBids (Partial MAX per partition above, Final here) and the join num = maxn
  uint64_t maxn = 0;
  bool any = false;
  for (int32_t q = 0; q < P; ++q) {
    maxn = std::max(maxn, part_max[size_t(q)]);
    any = any || finals[size_t(q)].used > 0;
  }
  int64_t out = 0;
  if (any)
    for (int32_t q = 0; q < P; ++q) {
      const Counts& c = finals[size_t(q)];
      for (size_t i = 0; i < c.key.size(); ++i)
        if (c.key[i] >= 0 && c.cnt[i] == maxn && out < out_capacity) {
          out_auction[out] = int32_t(c.key[i]);
          out_num[out] = c.cnt[i];
          ++out;
        }
    }
  return out;
}


// ---- NEXMark q1 natively: ProjectionExec [auction, bidder, 0.908 * CAST(price AS Float64), b_date_time] (planner.rs:90-92).
// The pass-through columns are Arc clones in the reference; the work is the computed column, batch by batch, the batches
// dealt round-robin to n_partitions tasks.  out_price[b] receives batch b's Float64 column.
void orc_q1_collect(const int32_t* const* price, const int64_t* rows, int32_t n_batches, int32_t n_partitions, int32_t n_threads, double* const* out_price) {
  const int32_t P = std::max(1, n_partitions);
  const int32_t T = std::max(1, std::min(n_threads, P));
  std::atomic<int32_t> next{0};
  auto worker = [&]() {
    for (int32_t p = next.fetch_add(1); p < P; p = next.fetch_add(1))
      for (int32_t b = p; b < n_batches; b += P) {
        const int32_t* in = price[b];
        double* out = out_price[b];
        for (int64_t r = 0; r < rows[b]; ++r) out[r] = 0.908 * double(in[r]);
      }
  };
  std::vector<std::thread> pool;
  for (int32_t t = 1; t < T; ++t) pool.emplace_back(worker);
  worker();
  for (std::thread& t : pool) t.join();
}

// ---- NEXMark q3 natively (planner.rs:151-171): auction' = FilterExec(category = 10) over (a_id, seller, category), person' =
// FilterExec(state = 'or' OR 'id' OR 'ca') over (p_id, name, city, state); both hash-repartitioned on the join key; per
// partition HashJoinExec(build auction', probe person') on seller = p_id; ProjectionExec -> (name, city, state, a_id).
// Strings are (offsets, bytes) pairs per batch.  Output columns are written one partition behind the other; returns rows,
// or -1 when the output does not fit out_capacity rows / out_bytes_capacity bytes per string column.
int64_t orc_q3_collect(const int32_t* const* a_id, const int32_t* const* a_seller, const int32_t* const* a_category, const int64_t* a_rows, int32_t n_a_batches,
                       const int32_t* const* p_id, const int32_t* const* name_off, const uint8_t* const* name_dat, const int32_t* const* city_off,
                       const uint8_t* const* city_dat, const int32_t* const* state_off, const uint8_t* const* state_dat, const int64_t* p_rows,
                       int32_t n_p_batches, int32_t n_partitions, int32_t n_threads, int32_t* out_a_id, int32_t* out_name_off, uint8_t* out_name,
                       int32_t* out_city_off, uint8_t* out_city, int32_t* out_state_off, uint8_t* out_state, int64_t out_capacity, int64_t out_bytes_capacity) {
  const int32_t P = std::max(1, n_partitions);
  const int32_t T = std::max(1, std::min(n_threads, P));
  const size_t np = size_t(P);
  auto run = [&](auto&& task) {
    std::atomic<int32_t> next{0};
    auto worker = [&]() {
      for (int32_t p = next.fetch_add(1); p < P; p = next.fetch_add(1)) task(p);
    };
    std::vector<std::thread> pool;
    for (int32_t t = 1; t < T; ++t) pool.emplace_back(worker);
    worker();
    for (std::thread& t : pool) t.join();
  };
  auto mix = [](uint64_t k) {
    k ^= k >> 33;
    k *= 0xff51afd7ed558ccdull;
    k ^= k >> 33;
    k *= 0xc4ceb9fe1a85ec53ull;
    k ^= k >> 33;
    return k;
  };
  auto route = [&](int32_t key) { return int32_t((mix(uint32_t(key)) >> 32) * uint64_t(P) >> 32); };
  struct Ref {
    int32_t batch, row;
  };
  // phase 1: the two filters, survivors routed by hash(join key)
  std::vector<std::vector<std::vector<Ref>>> a_parts{np, std::vector<std::vector<Ref>>{np}}, p_parts{np, std::vector<std::vector<Ref>>{np}};
  run([&](int32_t p) {
    for (int32_t b = p; b < n_a_batches; b += P)
      for (int32_t r = 0; r < int32_t(a_rows[b]); ++r)
        if (int64_t(a_category[b][r]) == 10) a_parts[size_t(p)][size_t(route(a_seller[b][r]))].push_back(Ref{b, r});
    for (int32_t b = p; b < n_p_batches; b += P)
      for (int32_t r = 0; r < int32_t(p_rows[b]); ++r) {
        const int32_t lo = state_off[b][r], n = state_off[b][r + 1] - lo;
        const uint8_t* st = state_dat[b] + lo;
        const bool keep = n == 2 && ((st[0] == 'o' && st[1] == 'r') || (st[0] == 'i' && st[1] == 'd') || (st[0] == 'c' && st[1] == 'a'));
        if (keep) p_parts[size_t(p)][size_t(route(p_id[b][r]))].push_back(Ref{b, r});
      }
  });
  // phase 2: per partition, build on auction' (seller -> chain of rows), probe with person' in order
  struct Out {
    std::vector<int32_t> a, name_len, city_len, state_len;
    std::vector<uint8_t> name, city, state;
  };
  std::vector<Out> outs{np};
  run([&](int32_t q) {
    std::vector<Ref> build;
    for (int32_t p = 0; p < P; ++p) build.insert(build.end(), a_parts[size_t(p)][size_t(q)].begin(), a_parts[size_t(p)][size_t(q)].end());
    size_t cap = 16;
    while (cap < 2 * build.size()) cap <<= 1;
    std::vector<int32_t> head(cap, -1), nxt(build.size(), -1);
    std::vector<int64_t> key(cap, -1);
    for (size_t i = 0; i < build.size(); ++i) {
      const int32_t k = a_seller[build[i].batch][build[i].row];
      uint64_t s = mix(uint32_t(k)) & (cap - 1);
      while (key[s] >= 0 && int32_t(key[s]) != k) s = (s + 1) & (cap - 1);
      key[s] = int64_t(uint32_t(k));
      nxt[i] = head[s];
      head[s] = int32_t(i);
    }
    Out& o = outs[size_t(q)];
    auto put = [](std::vector<uint8_t>& bytes, std::vector<int32_t>& lens, const int32_t* off, const uint8_t* dat, int32_t r) {
      const int32_t n = off[r + 1] - off[r];
      lens.push_back(n);
      bytes.insert(bytes.end(), dat + off[r], dat + off[r] + n);
    };
    for (int32_t p = 0; p < P; ++p)
      for (const Ref& ref : p_parts[size_t(p)][size_t(q)]) {
        const int32_t k = p_id[ref.batch][ref.row];
        uint64_t s = mix(uint32_t(k)) & (cap - 1);
        while (key[s] >= 0 && int32_t(key[s]) != k) s = (s + 1) & (cap - 1);
        if (key[s] < 0) continue;
        for (int32_t i = head[s]; i >= 0; i = nxt[size_t(i)]) {
          o.a.push_back(a_id[build[size_t(i)].batch][build[size_t(i)].row]);
          put(o.name, o.name_len, name_off[ref.batch], name_dat[ref.batch], ref.row);
          put(o.city, o.city_len, city_off[ref.batch], city_dat[ref.batch], ref.row);
          put(o.state, o.state_len, state_off[ref.batch], state_dat[ref.batch], ref.row);
        }
      }
  });
  int64_t rows = 0;
  int64_t nb = 0, cb = 0, sb = 0;
  out_name_off[0] = out_city_off[0] = out_state_off[0] = 0;
  for (int32_t q = 0; q < P; ++q) {
    const Out& o = outs[size_t(q)];
    if (rows + int64_t(o.a.size()) > out_capacity) return -1;  // the caller retries with more room
    if (nb + int64_t(o.name.size()) > out_bytes_capacity || cb + int64_t(o.city.size()) > out_bytes_capacity || sb + int64_t(o.state.size()) > out_bytes_capacity) return -1;
    std::copy(o.a.begin(), o.a.end(), out_a_id + rows);
    std::copy(o.name.begin(), o.name.end(), out_name + nb);
    std::copy(o.city.begin(), o.city.end(), out_city + cb);
    std::copy(o.state.begin(), o.state.end(), out_state + sb);
    for (size_t i = 0; i < o.a.size(); ++i) {
      nb += o.name_len[i];
      cb += o.city_len[i];
      sb += o.state_len[i];
      out_name_off[rows + int64_t(i) + 1] = int32_t(nb);
      out_city_off[rows + int64_t(i) + 1] = int32_t(cb);
      out_state_off[rows + int64_t(i) + 1] = int32_t(sb);
    }
    rows += int64_t(o.a.size());
  }
  return rows;
}

}  // extern "C"
