// rowkeys.cuh -- key handling shared by the hash operators (aggregate, join, repartition).
//
//   packed keys : up to two fixed-width key columns of <= 8 bytes together, folded into one uint64
//                 (Int32 keys zero-extended; (Int32, Int32) as hi:lo).  Equal keys <=> equal words.
//   row keys    : anything else (Utf8, wide or > 2 columns): hash and compare the key columns of rows.
//
// The hash is Murmur3-fmix / FNV based.  DataFusion hashes with ahash (RandomState::with_seeds(0,0,0,0),
// playground/src/distributed_plan/shuffle_writer.rs:109-124); hash values are never observable in
// results (SURVEY.md Appendix C.6), only the grouping / co-location they induce.
#pragma once

#include "device_utils.cuh"
#include "expr_program.h"

namespace fg {

constexpr int MAX_KEY_COLS = 8;

struct KeyPack {
  int32_t n;         // 1 or 2 columns
  int32_t width[2];  // bytes
  int32_t col[2];
};

struct RowKeys {
  int32_t n;
  int32_t col[MAX_KEY_COLS];
};

__device__ __forceinline__ unsigned long long pack_key(const KeyPack& k, const ColRef* cols, int64_t row) {
  // The two-column case is kept as two independent 32-bit loads combined at the end: ptxas 12.9 turned the
  // earlier "a = (a << 32) | second" form into a load that overwrote `a` before its old value had been moved to
  // the high half (tests/test_gpu_ops.py::test_hash_aggregate_single[*-group1] caught it).
  if (k.n == 2) {
    const uint32_t hi = __ldg(static_cast<const uint32_t*>(cols[k.col[0]].data) + row);
    const uint32_t lo = __ldg(static_cast<const uint32_t*>(cols[k.col[1]].data) + row);
    return (static_cast<unsigned long long>(hi) << 32) | lo;
  }
  if (k.width[0] == 4) return static_cast<const uint32_t*>(cols[k.col[0]].data)[row];
  return static_cast<const unsigned long long*>(cols[k.col[0]].data)[row];
}

__device__ __forceinline__ unsigned long long hash_row(const RowKeys& k, const ColRef* cols, int64_t row) {
  unsigned long long h = 0x9e3779b97f4a7c15ull;
  for (int i = 0; i < k.n; ++i) {
    const ColRef& c = cols[k.col[i]];
    if (c.validity && !c.validity[row]) {  // NULL: one fixed contribution, whatever bytes lie underneath
      h = fmix64(h ^ 0x6e756c6c6e756c6cull);
      continue;
    }
    if (c.dtype == FLOCKGPU_UTF8) {
      int32_t lo = c.offsets[row], hi = c.offsets[row + 1];
      h = hash_bytes(static_cast<const uint8_t*>(c.data) + lo, hi - lo, h);
    } else {
      h = fmix64(h ^ (unsigned long long)load_val(c, row).u);
    }
  }
  return h;
}

// Key equality of row r1 of (k1, cols1) and row r2 of (k2, cols2); the i-th key columns have equal types.
__device__ __forceinline__ bool rows_equal(const RowKeys& k1, const ColRef* cols1, int64_t r1, const RowKeys& k2, const ColRef* cols2, int64_t r2) {
  for (int i = 0; i < k1.n; ++i) {
    const ColRef& c1 = cols1[k1.col[i]];
    const ColRef& c2 = cols2[k2.col[i]];
    // grouping semantics: NULL equals NULL and nothing else (joins never get here with a NULL key: they skip such rows)
    const bool v1 = !c1.validity || c1.validity[r1], v2 = !c2.validity || c2.validity[r2];
    if (v1 != v2) return false;
    if (!v1) continue;
    if (c1.dtype == FLOCKGPU_UTF8) {
      int32_t lo1 = c1.offsets[r1], n1 = c1.offsets[r1 + 1] - lo1;
      int32_t lo2 = c2.offsets[r2], n2 = c2.offsets[r2 + 1] - lo2;
      if (n1 != n2) return false;
      const uint8_t* p1 = static_cast<const uint8_t*>(c1.data) + lo1;
      const uint8_t* p2 = static_cast<const uint8_t*>(c2.data) + lo2;
      for (int b = 0; b < n1; ++b)
        if (p1[b] != p2[b]) return false;
    } else if (load_val(c1, r1).u != load_val(c2, r2).u) {
      return false;
    }
  }
  return true;
}

// Host-side classification: can these key columns be packed into 64 bits?
inline bool keys_packable(const int* widths, int n) {
  if (n < 1 || n > 2) return false;
  int total = 0;
  for (int i = 0; i < n; ++i) {
    if (widths[i] != 4 && widths[i] != 8) return false;
    total += widths[i];
  }
  return n == 1 ? true : total == 8;
}

}  // namespace fg
