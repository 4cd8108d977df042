// hash_agg.cu -- K5/K6/K7: HashAggregateExec {Partial, Final, FinalPartitioned} (+ the fused SINGLE mode).
//
// Reference operator (DataFusion fork, not in tree): group-by hash table over the group columns with
// per-group accumulators; Partial emits (keys, state columns "<name>[count|sum|max|min]"), Final*
// merges states (COUNT = sum of counts, AVG = sum / count) -- shapes at
// flock/src/distributed_plan/stage.rs:535-543, :597-600, planner.rs:235, :246-254; state-column names
// in flock/src/tests/data/plan/aggregate.json.
//
// GPU design
//   packed keys   up to two fixed-width group columns (<= 8 bytes together) become one 64-bit key.
//     level 1     (raw rows, large inputs) every CTA owns a contiguous row range and pre-aggregates it in SHARED
//                 MEMORY -- the reference's Partial stage with the CTA in the role of the partition:
//                   agg_hist32_kernel   one 4-byte key + COUNT / DISTINCT: sliding direct-address histogram (NEXMark
//                                       ids are consecutive and local in time), 32-bit (key, count) partials;
//                   agg_local32_kernel  its hash-table fallback when the keys are not dense;
//                   agg_local_kernel    any packed key / accumulators: 64 KB hash table, 64-bit CAS + shared atomics.
//     level 2     agg_insert_kernel: partials (or raw rows when the input is small, or partial STATES in the Final*
//                 modes) are merged into a global table -- direct-address when one key column fills its range,
//                 open addressing with 64-bit CAS otherwise; its size comes from the partial count.
//     emit        agg_emit_kernel: stable single-pass compaction of the occupied slots (compact.cuh), four
//                 contiguous slots per vector load.
//   row keys      Utf8 or wide group keys: the table stores the index of a representative input row
//                 (agg_insert_rows_kernel); key equality is checked against the input columns.
//   no keys       agg_global_kernel: register accumulators -> warp shuffle -> one atomic per warp.
#include <algorithm>
#include <functional>

#include "compact.cuh"
#include "expr_program.h"
#include "internal.h"
#include "rowkeys.cuh"

namespace fg {

constexpr int MAX_ACC = 8;
constexpr unsigned long long EMPTY_KEY = ~0ull;
constexpr unsigned EMPTY_OWNER = ~0u;

// ACC_MIN_F / ACC_MAX_F hold f64_order_key(value): the IEEE total order becomes an unsigned one, so they are
// ACC_MIN_U / ACC_MAX_U on the encoded bits (a NaN is a value like any other, -0.0 < +0.0, and the result is always
// the bit pattern of one input row).  Values are encoded on load and decoded on emit.
enum AccOp : int32_t { ACC_COUNT = 0, ACC_ADD_I, ACC_ADD_F, ACC_MIN_I, ACC_MAX_I, ACC_MIN_U, ACC_MAX_U, ACC_MIN_F, ACC_MAX_F };

struct AccDesc {
  int32_t op;   // AccOp applied to raw input rows
  int32_t col;  // input column (-1: none, COUNT(*))
  int32_t cvt;  // Cvt applied to the loaded value (AVG / SUM over ints into f64)
  int32_t pad;
};

enum EmitKind : int32_t { EMIT_RAW = 0, EMIT_AVG = 1, EMIT_F64_ORDER = 2 };  // EMIT_F64_ORDER: decode f64_order_key
struct EmitDesc {
  int32_t kind;
  int32_t a0, a1;     // accumulator indices (AVG: a0 = count, a1 = sum)
  int32_t out_dtype;
  void* dst;
  uint8_t* valid_dst;  // not NULL: the output is NULL for groups whose accumulator `valid_acc` (a count of non-NULL inputs) is 0
  int32_t valid_acc, pad;
};

__host__ __device__ __forceinline__ unsigned long long acc_identity(int op) {
  switch (op) {
    case ACC_MIN_I: return 0x7fffffffffffffffull;
    case ACC_MAX_I: return 0x8000000000000000ull;
    case ACC_MIN_U:
    case ACC_MIN_F: return ~0ull;
    default: return 0ull;  // COUNT / ADD_I / ADD_F (+0.0) / MAX_U / MAX_F
  }
}

// The operation that merges two partial states of accumulator `op`.
__host__ __device__ __forceinline__ int acc_merge_op(int op) { return op == ACC_COUNT ? ACC_ADD_I : op; }

// Atomic accumulate into a (shared or global) 64-bit state word.
__device__ __forceinline__ void acc_apply(unsigned long long* p, int op, Val v) {
  switch (op) {
    case ACC_COUNT: atomicAdd(p, 1ull); break;
    case ACC_ADD_I: atomicAdd(p, v.u); break;
    case ACC_ADD_F: atomicAdd(reinterpret_cast<double*>(p), v.d); break;
    case ACC_MIN_I: atomicMin(reinterpret_cast<long long*>(p), (long long)v.i); break;
    case ACC_MAX_I: atomicMax(reinterpret_cast<long long*>(p), (long long)v.i); break;
    case ACC_MIN_U:
    case ACC_MIN_F: atomicMin(p, (unsigned long long)v.u); break;
    default: atomicMax(p, (unsigned long long)v.u); break;  // MAX_U / MAX_F
  }
}

// Non-atomic combine (register accumulators of the no-group kernel).
__device__ __forceinline__ Val acc_combine(int op, Val a, Val b) {
  Val r = a;
  switch (op) {
    case ACC_COUNT: r.u = a.u + 1; break;
    case ACC_ADD_I: r.u = a.u + b.u; break;
    case ACC_ADD_F: r.d = a.d + b.d; break;
    case ACC_MIN_I: r.i = b.i < a.i ? b.i : a.i; break;
    case ACC_MAX_I: r.i = b.i > a.i ? b.i : a.i; break;
    case ACC_MIN_U:
    case ACC_MIN_F: r.u = b.u < a.u ? b.u : a.u; break;
    default: r.u = b.u > a.u ? b.u : a.u; break;  // MAX_U / MAX_F
  }
  return r;
}

// false: the argument is NULL in this row, and NULL arguments are skipped by every aggregate (SURVEY.md Appendix C.7)
__device__ __forceinline__ bool acc_input_valid(const AccDesc& d, const ColRef* cols, int64_t row) {
  return d.col < 0 || !cols[d.col].validity || cols[d.col].validity[row] != 0;
}

__device__ __forceinline__ Val load_acc_input(const AccDesc& d, const ColRef* cols, int64_t row) {
  Val v;
  v.u = 0;
  if (d.col >= 0 && d.op != ACC_COUNT) {
    v = load_val(cols[d.col], row);
    if (d.cvt == CVT_I2F) v.d = __ll2double_rn(v.i);
    else if (d.cvt == CVT_U2F) v.d = __ull2double_rn(v.u);
    if (d.op == ACC_MIN_F || d.op == ACC_MAX_F) v.u = f64_order_key(v.u);  // raw rows and MIN / MAX states alike
  }
  return v;
}

__device__ __forceinline__ unsigned hash_key(unsigned long long k) { return unsigned(fmix64(k) >> 20); }

// ================================================================================================
// level 1: CTA-local pre-aggregation in shared memory
// ================================================================================================
constexpr int AL_THREADS = 256;
constexpr int AL_UNROLL = 4;
constexpr int AL_SLOTS = 4096;  // >= 4 * AL_THREADS * AL_UNROLL so a 3/4-full table absorbs one iteration

struct AggLocalArgs {
  int64_t n_rows;
  KeyPack keys;
  int32_t n_acc;
  int32_t pad;
  AccDesc acc[MAX_ACC];
  ColRef cols[MAX_IN_COLS];
  unsigned long long* part_keys;    // [part_capacity]
  unsigned long long* part_acc;     // [n_acc][part_capacity]
  int64_t part_capacity;
  unsigned long long* part_cursor;  // number of partial entries written so far
  unsigned long long* key_minmax;   // [0] = min, [1] = max packed key seen (decides the dense level-2 table)
};

__device__ __forceinline__ void local_flush(const AggLocalArgs& a, unsigned long long* s_keys, unsigned long long* s_acc, unsigned* s_warp,
                                            unsigned long long* s_base, unsigned* s_occ) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int PER = AL_SLOTS / AL_THREADS;
  // thread owns slots [tid * PER, tid * PER + PER)
  unsigned cnt = 0;
#pragma unroll
  for (int j = 0; j < PER; ++j) cnt += s_keys[tid * PER + j] != EMPTY_KEY;
  unsigned incl = warp_inclusive_sum(cnt);
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  unsigned warp_base = 0, total = 0;
#pragma unroll
  for (int w = 0; w < AL_THREADS / 32; ++w) {
    unsigned v = s_warp[w];
    if (w < warp) warp_base += v;
    total += v;
  }
  if (tid == 0) *s_base = total ? atomicAdd(a.part_cursor, (unsigned long long)total) : 0ull;
  __syncthreads();
  unsigned long long pos = *s_base + warp_base + (incl - cnt);
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    const int slot = tid * PER + j;
    const unsigned long long k = s_keys[slot];
    if (k != EMPTY_KEY) {
      a.part_keys[pos] = k;
      for (int c = 0; c < a.n_acc; ++c) {
        a.part_acc[int64_t(c) * a.part_capacity + pos] = s_acc[c * AL_SLOTS + slot];
        s_acc[c * AL_SLOTS + slot] = acc_identity(a.acc[c].op);
      }
      s_keys[slot] = EMPTY_KEY;
      ++pos;
    }
  }
  if (tid == 0) *s_occ = 0;
  __syncthreads();
}

__global__ void __launch_bounds__(AL_THREADS) agg_local_kernel(const __grid_constant__ AggLocalArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned long long* s_keys = reinterpret_cast<unsigned long long*>(smem_raw);
  unsigned long long* s_acc = s_keys + AL_SLOTS;  // [n_acc][AL_SLOTS]
  __shared__ unsigned s_warp[AL_THREADS / 32];
  __shared__ unsigned long long s_base;
  __shared__ unsigned s_occ;
  const int tid = threadIdx.x;

  for (int s = tid; s < AL_SLOTS; s += AL_THREADS) {
    s_keys[s] = EMPTY_KEY;
    for (int c = 0; c < a.n_acc; ++c) s_acc[c * AL_SLOTS + s] = acc_identity(a.acc[c].op);
  }
  if (tid == 0) s_occ = 0;
  __syncthreads();

  constexpr int STEP = AL_THREADS * AL_UNROLL;
  int64_t per_cta = (a.n_rows + gridDim.x - 1) / gridDim.x;
  per_cta = (per_cta + STEP - 1) / STEP * STEP;
  const int64_t begin = int64_t(blockIdx.x) * per_cta;
  const int64_t end = begin + per_cta < a.n_rows ? begin + per_cta : a.n_rows;

  unsigned long long kmin = ~0ull, kmax = 0ull;
  for (int64_t base = begin; base < end; base += STEP) {
    unsigned long long key[AL_UNROLL];
    int64_t row[AL_UNROLL];
#pragma unroll
    for (int u = 0; u < AL_UNROLL; ++u) {
      row[u] = base + int64_t(u) * AL_THREADS + tid;
      if (row[u] < end) {
        key[u] = pack_key(a.keys, a.cols, row[u]);
        kmin = key[u] < kmin ? key[u] : kmin;
        kmax = key[u] > kmax ? key[u] : kmax;
      }
    }
#pragma unroll
    for (int u = 0; u < AL_UNROLL; ++u) {
      if (row[u] >= end) continue;
      if (key[u] == EMPTY_KEY) {
        // the one key value that collides with the empty marker bypasses the shared table
        unsigned long long pos = atomicAdd(a.part_cursor, 1ull);
        a.part_keys[pos] = key[u];
        for (int c = 0; c < a.n_acc; ++c) {
          Val v = load_acc_input(a.acc[c], a.cols, row[u]);
          Val id;
          id.u = acc_identity(a.acc[c].op);
          a.part_acc[int64_t(c) * a.part_capacity + pos] = acc_input_valid(a.acc[c], a.cols, row[u]) ? acc_combine(a.acc[c].op, id, v).u : id.u;
        }
        continue;
      }
      unsigned slot = hash_key(key[u]) & (AL_SLOTS - 1);
      while (true) {
        unsigned long long cur = s_keys[slot];
        if (cur == key[u]) break;
        if (cur == EMPTY_KEY) {
          unsigned long long old = atomicCAS(&s_keys[slot], EMPTY_KEY, key[u]);
          if (old == EMPTY_KEY) {
            atomicAdd(&s_occ, 1u);
            break;
          }
          if (old == key[u]) break;
        }
        slot = (slot + 1) & (AL_SLOTS - 1);
      }
      for (int c = 0; c < a.n_acc; ++c)
        if (acc_input_valid(a.acc[c], a.cols, row[u])) acc_apply(&s_acc[c * AL_SLOTS + slot], a.acc[c].op, load_acc_input(a.acc[c], a.cols, row[u]));
    }
    // the decision must be CTA-uniform: s_occ is bumped again by fast warps in the next step, so every thread
    // reads it between two barriers
    __syncthreads();
    const bool do_flush = s_occ > AL_SLOTS * 3 / 4 - STEP;
    __syncthreads();
    if (do_flush) local_flush(a, s_keys, s_acc, s_warp, &s_base, &s_occ);
  }
  local_flush(a, s_keys, s_acc, s_warp, &s_base, &s_occ);
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    unsigned long long o1 = __shfl_xor_sync(FULL_MASK, kmin, d), o2 = __shfl_xor_sync(FULL_MASK, kmax, d);
    kmin = o1 < kmin ? o1 : kmin;
    kmax = o2 > kmax ? o2 : kmax;
  }
  if ((tid & 31) == 0 && kmin <= kmax) {
    atomicMin(a.key_minmax, kmin);
    atomicMax(a.key_minmax + 1, kmax);
  }
}


// ================================================================================================
// level 1, specialised: ONE 4-byte key column, COUNT(*) or no aggregate (NEXMark q5 / q8 seller)
// ================================================================================================
// Same structure as agg_local_kernel, but the table is (u32 key, u32 count): native 32-bit shared atomics
// (the generic kernel's 64-bit shared atomicAdd / CAS are the slower path on q5), 128-bit loads, and a per-warp HOT KEY: NEXMark's bid stream puts about half of the
// rows of a batch on one auction id (event.rs:355-359), so every warp remembers the key that dominated its
// last step and folds all lanes carrying it into one atomicAdd of popc(ballot).
constexpr int A32_THREADS = 256;
constexpr int A32_SLOTS = 8192;
constexpr int A32_STEP = A32_THREADS * 16;  // rows per CTA iteration (4 x int4 per thread)
constexpr unsigned EMPTY32 = ~0u;

struct AggLocal32Args {
  int64_t n_rows;
  const uint32_t* key_col;
  int32_t has_count;
  int32_t pad;
  uint32_t* part_keys;  // 32-bit partials: 8 B per (key, count) instead of 16 -- half the traffic of q5's 4.9 M partials
  uint32_t* part_acc;   // next to the 58 MB level-2 table ([part_capacity], unused without COUNT)
  int64_t part_capacity;
  unsigned long long* part_cursor;
  unsigned long long* key_minmax;
};

__device__ __forceinline__ unsigned a32_find_or_insert(unsigned* s_keys, unsigned* s_occ, unsigned key) {
  unsigned slot = fmix32(key) & (A32_SLOTS - 1);
  while (true) {
    unsigned cur = s_keys[slot];
    if (cur == key) return slot;
    if (cur == EMPTY32) {
      unsigned old = atomicCAS(&s_keys[slot], EMPTY32, key);
      if (old == EMPTY32) {
        atomicAdd(s_occ, 1u);
        return slot;
      }
      if (old == key) return slot;
    }
    slot = (slot + 1) & (A32_SLOTS - 1);
  }
}

__global__ void __launch_bounds__(A32_THREADS) agg_local32_kernel(const __grid_constant__ AggLocal32Args a) {
  extern __shared__ __align__(16) unsigned a32_smem[];  // keys[A32_SLOTS] | counts[A32_SLOTS] = 64 KB (dynamic: > 48 KB)
  unsigned* s_keys = a32_smem;
  unsigned* s_cnt = a32_smem + A32_SLOTS;
  __shared__ unsigned s_warp[A32_THREADS / 32];
  __shared__ unsigned long long s_base;
  __shared__ unsigned s_occ;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int s = tid; s < A32_SLOTS; s += A32_THREADS) {
    s_keys[s] = EMPTY32;
    s_cnt[s] = 0;
  }
  if (tid == 0) s_occ = 0;
  __syncthreads();

  int64_t per_cta = (a.n_rows + gridDim.x - 1) / gridDim.x;
  per_cta = (per_cta + A32_STEP - 1) / A32_STEP * A32_STEP;
  const int64_t begin = int64_t(blockIdx.x) * per_cta;
  const int64_t end = begin + per_cta < a.n_rows ? begin + per_cta : a.n_rows;
  unsigned kmin = ~0u, kmax = 0u;
  unsigned hot = EMPTY32, hot_slot = 0;  // warp-uniform

  auto flush = [&]() {
    constexpr int PER = A32_SLOTS / A32_THREADS;
    unsigned cnt = 0;
#pragma unroll
    for (int j = 0; j < PER; ++j) cnt += s_keys[tid * PER + j] != EMPTY32;
    unsigned incl = warp_inclusive_sum(cnt);
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    unsigned warp_base = 0, total = 0;
#pragma unroll
    for (int w = 0; w < A32_THREADS / 32; ++w) {
      unsigned v = s_warp[w];
      if (w < warp) warp_base += v;
      total += v;
    }
    if (tid == 0) s_base = total ? atomicAdd(a.part_cursor, (unsigned long long)total) : 0ull;
    __syncthreads();
    unsigned long long pos = s_base + warp_base + (incl - cnt);
#pragma unroll
    for (int j = 0; j < PER; ++j) {
      const int slot = tid * PER + j;
      const unsigned k = s_keys[slot];
      if (k != EMPTY32) {
        a.part_keys[pos] = k;
        if (a.has_count) a.part_acc[pos] = s_cnt[slot];
        s_keys[slot] = EMPTY32;
        s_cnt[slot] = 0;
        ++pos;
      }
    }
    if (tid == 0) s_occ = 0;
    hot = EMPTY32;
    __syncthreads();
  };

  for (int64_t base = begin; base < end; base += A32_STEP) {
    uint4 v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int64_t r0 = base + (int64_t(j) * A32_THREADS + tid) * 4;
      if (r0 + 3 < end) {
        int4 t = ldg_stream_v4(a.key_col + r0);
        v[j] = make_uint4(unsigned(t.x), unsigned(t.y), unsigned(t.z), unsigned(t.w));
      } else {
        v[j] = make_uint4(EMPTY32, EMPTY32, EMPTY32, EMPTY32);  // EMPTY32 doubles as "no row" inside the step
        if (r0 + 0 < end) v[j].x = a.key_col[r0 + 0];
        if (r0 + 1 < end) v[j].y = a.key_col[r0 + 1];
        if (r0 + 2 < end) v[j].z = a.key_col[r0 + 2];
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int64_t r0 = base + (int64_t(j) * A32_THREADS + tid) * 4;
      const unsigned ks[4] = {v[j].x, v[j].y, v[j].z, v[j].w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const unsigned k = ks[e];
        const bool valid = r0 + e < end;
        if (valid) {
          kmin = k < kmin ? k : kmin;
          kmax = k > kmax ? k : kmax;
        }
        // --- hot key: all lanes carrying it become one atomic
        unsigned m = __ballot_sync(FULL_MASK, valid && k == hot && hot != EMPTY32);
        bool done = !valid || (m >> lane) & 1u;
        if (m && lane == __ffs(m) - 1 && a.has_count) atomicAdd(&s_cnt[hot_slot], (unsigned)__popc(m));
        if (__popc(m) < 8) {
          // the remembered key no longer dominates: try the key of the first still-pending lane
          const unsigned pending = __ballot_sync(FULL_MASK, !done && k != EMPTY32);
          if (pending) {
            const unsigned cand = __shfl_sync(FULL_MASK, k, __ffs(pending) - 1);
            const unsigned m2 = __ballot_sync(FULL_MASK, !done && k == cand);
            if (__popc(m2) >= 8) {
              unsigned slot = 0;
              if (lane == __ffs(m2) - 1) {
                slot = a32_find_or_insert(s_keys, &s_occ, cand);
                if (a.has_count) atomicAdd(&s_cnt[slot], (unsigned)__popc(m2));
              }
              hot = cand;
              hot_slot = __shfl_sync(FULL_MASK, slot, __ffs(m2) - 1);
              done = done || (m2 >> lane) & 1u;
            }
          }
        }
        if (!done) {
          if (k == EMPTY32) {
            // the one key equal to the empty marker bypasses the shared table
            unsigned long long pos = atomicAdd(a.part_cursor, 1ull);
            a.part_keys[pos] = k;
            if (a.has_count) a.part_acc[pos] = 1;
          } else {
            const unsigned slot = a32_find_or_insert(s_keys, &s_occ, k);
            if (a.has_count) atomicAdd(&s_cnt[slot], 1u);
          }
        }
      }
    }
    __syncthreads();
    const bool do_flush = s_occ > A32_SLOTS * 3 / 4 - A32_STEP;  // CTA-uniform: read between two barriers
    __syncthreads();
    if (do_flush) flush();
  }
  flush();
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    unsigned o1 = __shfl_xor_sync(FULL_MASK, kmin, d), o2 = __shfl_xor_sync(FULL_MASK, kmax, d);
    kmin = o1 < kmin ? o1 : kmin;
    kmax = o2 > kmax ? o2 : kmax;
  }
  if (lane == 0 && kmin <= kmax) {
    atomicMin(a.key_minmax, (unsigned long long)kmin);
    atomicMax(a.key_minmax + 1, (unsigned long long)kmax);
  }
}

// ================================================================================================
// level 1, dense variant: a sliding DIRECT-ADDRESS histogram in shared memory
// ================================================================================================
// NEXMark ids are consecutive integers and a bid references one of the ~110 most recent auctions
// (event.rs:354-371), so the keys of a CTA's contiguous row range fall into a narrow, slowly advancing window.
// The CTA keeps counts[key - base] for an 8 Ki-key window: ONE native shared atomicAdd per row, no hashing, no
// CAS, no probing (the hash kernel above spends ~129 instructions per row; shared atomics keep their rate even with half
// of the lanes on one hot key).  When a row falls outside the window the histogram is flushed as
// (key, count) partials and re-based at the smallest key of the current step; rows below the base go to the
// partial buffer one by one.  `slow_rows` counts those exceptions: if the data is not dense the caller re-runs
// the hash kernel instead.
constexpr int H32_THREADS = 256;
constexpr int H32_WINDOW = 8192;              // 32 KB of u32 counters: 4 CTAs per SM (a CTA of q5 spans ~15 K auction ids: 2-3 re-bases)
constexpr int H32_LOADS = 4;                  // 16-byte loads per thread and step; the NEXT step's loads are issued before this
                                              // step's atomics (two register stages), so 64-128 B per thread are always in flight
constexpr int H32_ROWS = H32_LOADS * 4;       // rows per thread and step
constexpr int H32_STEP = H32_THREADS * H32_ROWS;  // rows per CTA iteration (4096)

struct AggHist32Args {
  int64_t n_rows;
  const uint32_t* key_col;
  int32_t has_count;
  int32_t pad;
  uint32_t* part_keys;  // 32-bit partials (see AggLocal32Args)
  uint32_t* part_acc;
  int64_t part_capacity;
  unsigned long long* part_cursor;
  unsigned long long* key_minmax;
  unsigned long long* slow_rows;
  // DENSE variant: the flushed counters are added straight into a direct-address table in global memory (L2-resident
  // for NEXMark: q5's 6.5 M auctions are 26 MB) instead of being written out as (key, count) partials
  uint32_t* dense;                          // [dense_cap] counts; slot = key - dense_meta[0]
  unsigned long long* dense_meta;           // [0] key of slot 0 (decided on the device by CTA 0 of the scan)
  unsigned long long dense_cap;
  unsigned long long* overflow;             // rows whose key fell outside the table (the caller then starts over)
};

// meta words of a direct-address count table
enum DenseMeta : int { DM_FIRST_KEY = 0, DM_OVERFLOW = 1, DM_SAMPLE = 2, DM_SLOTS = 3, DM_MAX = 4, DM_BARRIER1 = 5, DM_BARRIER2 = 6, DM_MATCHES = 7,
                       DM_READY = 8, DM_CLEARED = 9, DM_WORDS = 16 };

// Decides, ON THE DEVICE (CTA 0 of the scan kernel itself), which keys the direct-address table covers: the range of a SAMPLE of the key column (the
// first and last 256 rows -- ids grow with time, so the extremes sit at the ends -- and 512 rows spread over the
// rest) widened by a sixteenth of its span (at least 4096 keys) on both sides, cut to the table's capacity.  The host
// never learns the range: every later kernel reads it from `meta`, so there is no round trip before the scan starts.
// Executed by one whole CTA (any block size that is a multiple of 32, at most 1024 threads).
__device__ __forceinline__ void dense_sample_range(const uint32_t* __restrict__ keys, int64_t n, unsigned long long* meta, unsigned long long cap, unsigned* s_min,
                                                   unsigned* s_max) {
  const int tid = threadIdx.x, nthr = blockDim.x;
  unsigned lo = ~0u, hi = 0u;
  // one round of independent loads per thread: the first and last `nthr` rows and 2 x nthr rows spread over the rest
  const int64_t stride = n / (2 * nthr) > 0 ? n / (2 * nthr) : 1;
  {
    const int64_t at[4] = {int64_t(tid), n - 1 - tid, int64_t(tid) * stride, int64_t(tid + nthr) * stride};
    unsigned k[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) k[j] = (at[j] >= 0 && at[j] < n) ? keys[at[j]] : keys[0];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      lo = min(lo, k[j]);
      hi = max(hi, k[j]);
    }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    lo = min(lo, __shfl_xor_sync(FULL_MASK, lo, d));
    hi = max(hi, __shfl_xor_sync(FULL_MASK, hi, d));
  }
  if ((tid & 31) == 0) {
    s_min[tid >> 5] = lo;
    s_max[tid >> 5] = hi;
  }
  __syncthreads();
  if (tid < 32) {
    const int nw = nthr >> 5;
    lo = tid < nw ? s_min[tid] : ~0u;
    hi = tid < nw ? s_max[tid] : 0u;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      lo = min(lo, __shfl_xor_sync(FULL_MASK, lo, d));
      hi = max(hi, __shfl_xor_sync(FULL_MASK, hi, d));
    }
    if (tid == 0) {
      const unsigned long long span = (unsigned long long)hi - lo + 1;
      unsigned long long margin = span / 16 > 4096 ? span / 16 : 4096;
      const unsigned long long first = lo > margin ? lo - margin : 0ull;
      unsigned long long slots = ((unsigned long long)hi - first + 1 + margin + 3) & ~3ull;
      if (slots > cap) slots = cap;  // keys beyond it count as overflow and the caller starts over
      meta[DM_FIRST_KEY] = first;
      meta[DM_SAMPLE] = ((unsigned long long)hi << 32) | lo;
      meta[DM_SLOTS] = slots;
    }
  }
  __syncthreads();
}

template <bool DENSE>
__global__ void __launch_bounds__(H32_THREADS, 4) agg_hist32_kernel(const __grid_constant__ AggHist32Args a) {
  extern __shared__ __align__(128) unsigned h32_cnt[];  // [H32_WINDOW]
  __shared__ unsigned s_warp[H32_THREADS / 32];
  __shared__ unsigned long long s_base_pos;
  __shared__ unsigned s_min;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int s = tid; s < H32_WINDOW; s += H32_THREADS) h32_cnt[s] = 0;

  int64_t per_cta = (a.n_rows + gridDim.x - 1) / gridDim.x;
  per_cta = (per_cta + H32_STEP - 1) / H32_STEP * H32_STEP;
  const int64_t begin = int64_t(blockIdx.x) * per_cta;
  const int64_t end = begin + per_cta < a.n_rows ? begin + per_cta : a.n_rows;
  unsigned base = 0;     // CTA-uniform: key of counter 0
  bool have_base = false;
  unsigned kmin = ~0u, kmax = 0u;
  unsigned long long slow = 0, overflow = 0;
  unsigned top = 0;  // DENSE: largest count this thread has produced in the table
  const bool has_count = a.has_count != 0;
  __syncthreads();

  // DENSE: the table's key range is decided by CTA 0 from a sample, every CTA then clears its slice of the table, and
  // nobody touches the table before all slices are clear.  None of that holds up the scan: a CTA only needs the table
  // at its first flush, thousands of rows in, and by then the 5 us of sampling and 1 us of clearing are long over.
  // (The launch is cooperative: all CTAs are co-resident, so waiting for each other cannot deadlock.)
  bool table_ready = !DENSE;
  if (DENSE && blockIdx.x == 0) {
    __shared__ unsigned s_lo[H32_THREADS / 32], s_hi[H32_THREADS / 32];
    dense_sample_range(a.key_col, a.n_rows, a.dense_meta, a.dense_cap, s_lo, s_hi);
    if (tid == 0) {
      __threadfence();
      st_relaxed_u64(a.dense_meta + DM_READY, 1ull);
    }
  }
  // clears this CTA's slice as soon as CTA 0 has published the range (called once, with the first loads in flight)
  auto clear_my_slice = [&]() {
    unsigned long long* meta = a.dense_meta;
    if (tid == 0) {
      while (ld_relaxed_u64(meta + DM_READY) == 0ull) __nanosleep(100);
      __threadfence();
    }
    __syncthreads();
    const unsigned long long n4 = ld_relaxed_u64(meta + DM_SLOTS) >> 2;
    const unsigned long long per_cta = (n4 + gridDim.x - 1) / gridDim.x;
    const unsigned long long lo4 = blockIdx.x * per_cta, hi4 = lo4 + per_cta < n4 ? lo4 + per_cta : n4;
    for (unsigned long long i = lo4 + tid; i < hi4; i += H32_THREADS) reinterpret_cast<uint4*>(a.dense)[i] = make_uint4(0, 0, 0, 0);
    __threadfence();
    __syncthreads();
    if (tid == 0) atomicAdd(meta + DM_CLEARED, 1ull);
  };
  // before the first access to the table: every CTA's slice must be clear (they all cleared at their start, so this
  // hardly ever waits)
  auto ensure_table = [&]() {
    if (table_ready) return;  // CTA-uniform
    unsigned long long* meta = a.dense_meta;
    if (tid == 0) {
      while (ld_relaxed_u64(meta + DM_CLEARED) < gridDim.x) __nanosleep(100);
      __threadfence();
    }
    __syncthreads();
    table_ready = true;
  };

  // Writes the non-zero counters as partials and clears them.  Thread t owns counters (j * 256 + t) * 4 .. + 3
  // (128-bit, conflict-free shared accesses; the first version let a thread walk 32 consecutive counters = a 32-way
  // bank conflict on every access, 21 M conflict cycles per q5 launch); partial writes are compacted per warp and
  // iteration with a ballot so that a warp writes consecutive entries.
  auto flush = [&]() {
    constexpr int VEC = H32_WINDOW / (H32_THREADS * 4);  // uint4 per thread
    const uint4* cnt4 = reinterpret_cast<const uint4*>(h32_cnt);
    if (DENSE) {
      ensure_table();
      // every non-zero counter becomes one global atomic on the direct-address table (4.9 M per 100 M bids, spread
      // over the whole scan: they hide behind the streaming loads)
      const unsigned gbase = unsigned(ld_relaxed_u64(a.dense_meta + DM_FIRST_KEY)), gslots = unsigned(ld_relaxed_u64(a.dense_meta + DM_SLOTS));
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        const int v4 = j * H32_THREADS + tid;
        const uint4 c = cnt4[v4];
        if (!(c.x | c.y | c.z | c.w)) continue;
        const unsigned cs[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if (!cs[e]) continue;
          const unsigned idx = base + unsigned(v4) * 4u + unsigned(e) - gbase;
          if (idx < gslots) {
            // counts only grow, so the largest value any add ever produced is the largest final count: MAX(count)
            // falls out of the scan for free (NEXMark q5 asks for exactly that next)
            if (has_count) top = max(top, atomicAdd(&a.dense[idx], cs[e]) + cs[e]);
            else a.dense[idx] = 1u;
          } else {
            overflow += has_count ? cs[e] : 1u;  // summed per warp at the end: a sparse column must not serialise on one word
          }
        }
        reinterpret_cast<uint4*>(h32_cnt)[v4] = make_uint4(0, 0, 0, 0);
      }
      __syncthreads();
      return;
    }
    unsigned cnt = 0;
    unsigned smin = ~0u, smax = 0u;
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const uint4 c = cnt4[j * H32_THREADS + tid];
      const unsigned nz = unsigned(c.x != 0) + unsigned(c.y != 0) + unsigned(c.z != 0) + unsigned(c.w != 0);
      cnt += nz;
      if (nz) {
        const unsigned s0 = unsigned(j * H32_THREADS + tid) * 4u;
        const unsigned first = c.x ? 0u : c.y ? 1u : c.z ? 2u : 3u, last = c.w ? 3u : c.z ? 2u : c.y ? 1u : 0u;
        smin = min(smin, s0 + first);
        smax = max(smax, s0 + last);
      }
    }
    if (cnt) {
      kmin = min(kmin, base + smin);
      kmax = max(kmax, base + smax);
    }
    const unsigned warp_total = warp_sum(cnt);
    if (lane == 0) s_warp[warp] = warp_total;
    __syncthreads();
    unsigned warp_base = 0, total = 0;
#pragma unroll
    for (int w = 0; w < H32_THREADS / 32; ++w) {
      unsigned v = s_warp[w];
      if (w < warp) warp_base += v;
      total += v;
    }
    if (tid == 0) s_base_pos = total ? atomicAdd(a.part_cursor, (unsigned long long)total) : 0ull;
    __syncthreads();
    unsigned long long pos = s_base_pos + warp_base;  // warp-uniform running position
    const unsigned lt = lanemask_lt();
#pragma unroll
    for (int j = 0; j < VEC; ++j) {
      const int v4 = j * H32_THREADS + tid;
      const uint4 c = cnt4[v4];
      const unsigned cs[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const unsigned b = __ballot_sync(FULL_MASK, cs[e] != 0);
        if (cs[e]) {
          const unsigned long long p = pos + __popc(b & lt);
          a.part_keys[p] = base + unsigned(v4) * 4u + unsigned(e);
          if (has_count) a.part_acc[p] = cs[e];
        }
        pos += __popc(b);
      }
      if (c.x | c.y | c.z | c.w) reinterpret_cast<uint4*>(h32_cnt)[v4] = make_uint4(0, 0, 0, 0);
    }
    __syncthreads();
  };

  // one row at a time, any key: inside the window -> counter, outside -> its own partial
  auto add_checked = [&](unsigned k) {
    const unsigned idx = k - base;
    if (idx < unsigned(H32_WINDOW)) {
      if (has_count) atomicAdd(&h32_cnt[idx], 1u);
      else h32_cnt[idx] = 1u;
    } else if (DENSE) {
      const unsigned idx2 = k - unsigned(ld_relaxed_u64(a.dense_meta + DM_FIRST_KEY));
      if (idx2 < unsigned(ld_relaxed_u64(a.dense_meta + DM_SLOTS))) {
        if (has_count) top = max(top, atomicAdd(&a.dense[idx2], 1u) + 1u);
        else a.dense[idx2] = 1u;
      } else {
        ++overflow;
      }
      ++slow;
    } else {
      // outside the window even after re-basing (the step spans more than 8 Ki keys)
      unsigned long long pos = atomicAdd(a.part_cursor, 1ull);
      a.part_keys[pos] = k;
      if (has_count) a.part_acc[pos] = 1;
      kmin = k < kmin ? k : kmin;
      kmax = k > kmax ? k : kmax;
      ++slow;
    }
  };

  // re-base at the smallest key of the step (keys below a later base take the slow path)
  auto rebase = [&](unsigned lo) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      unsigned o = __shfl_xor_sync(FULL_MASK, lo, d);
      lo = o < lo ? o : lo;
    }
    if (tid == 0) s_min = ~0u;
    __syncthreads();
    if (lane == 0) atomicMin(&s_min, lo);
    __syncthreads();
    const unsigned new_base = s_min;
    if (have_base) flush();  // uniform: have_base is CTA-uniform
    base = new_base;
    have_base = true;
  };

  int64_t step = begin;
  // ---- full steps: every thread owns H32_ROWS valid rows; two register stages
  auto load_step = [&](uint4 (&v)[H32_LOADS], int64_t at) {
#pragma unroll
    for (int j = 0; j < H32_LOADS; ++j) {
      int4 t = ldg_stream_v4(a.key_col + at + (int64_t(j) * H32_THREADS + tid) * 4);
      v[j] = make_uint4(unsigned(t.x), unsigned(t.y), unsigned(t.z), unsigned(t.w));
    }
  };
  uint4 v[H32_LOADS], nxt[H32_LOADS];
  if (step + H32_STEP <= end) load_step(v, step);
  if (DENSE) clear_my_slice();  // the first step's loads are in flight meanwhile
  for (; step + H32_STEP <= end; step += H32_STEP) {
    const bool more = step + 2 * int64_t(H32_STEP) <= end;
    if (more) load_step(nxt, step + H32_STEP);  // in flight while this step waits at the barrier and counts
    unsigned ored = 0;
#pragma unroll
    for (int j = 0; j < H32_LOADS; ++j) ored |= (v[j].x - base) | (v[j].y - base) | (v[j].z - base) | (v[j].w - base);
    const int in_window = __syncthreads_and(have_base && ored < unsigned(H32_WINDOW));
    if (in_window) {
      if (has_count) {
#pragma unroll
        for (int j = 0; j < H32_LOADS; ++j) {
          atomicAdd(&h32_cnt[v[j].x - base], 1u);
          atomicAdd(&h32_cnt[v[j].y - base], 1u);
          atomicAdd(&h32_cnt[v[j].z - base], 1u);
          atomicAdd(&h32_cnt[v[j].w - base], 1u);
        }
      } else {
#pragma unroll
        for (int j = 0; j < H32_LOADS; ++j) {
          h32_cnt[v[j].x - base] = 1u;
          h32_cnt[v[j].y - base] = 1u;
          h32_cnt[v[j].z - base] = 1u;
          h32_cnt[v[j].w - base] = 1u;
        }
      }
    } else {
      unsigned lo = ~0u;
#pragma unroll
      for (int j = 0; j < H32_LOADS; ++j) lo = min(min(lo, min(v[j].x, v[j].y)), min(v[j].z, v[j].w));
      rebase(lo);
      if (DENSE) ensure_table();  // add_checked may touch the table directly
#pragma unroll
      for (int j = 0; j < H32_LOADS; ++j) {
        add_checked(v[j].x);
        add_checked(v[j].y);
        add_checked(v[j].z);
        add_checked(v[j].w);
      }
    }
    if (more) {
#pragma unroll
      for (int j = 0; j < H32_LOADS; ++j) v[j] = nxt[j];
    }
  }
  // ---- ragged tail of the CTA's range (at most one step): row by row
  if (step < end) {
    unsigned lo = ~0u;
    for (int64_t r = step + tid; r < end; r += H32_THREADS) lo = min(lo, a.key_col[r]);
    unsigned ok = 1;
    for (int64_t r = step + tid; r < end; r += H32_THREADS) ok &= unsigned(a.key_col[r] - base < unsigned(H32_WINDOW));
    if (!__syncthreads_and(have_base && ok)) rebase(lo);
    if (DENSE) ensure_table();
    for (int64_t r = step + tid; r < end; r += H32_THREADS) add_checked(a.key_col[r]);
  }
  __syncthreads();
  if (have_base) flush();
  if (DENSE) ensure_table();  // a CTA without rows still owes its slice of the clearing
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    unsigned o1 = __shfl_xor_sync(FULL_MASK, kmin, d), o2 = __shfl_xor_sync(FULL_MASK, kmax, d);
    kmin = o1 < kmin ? o1 : kmin;
    kmax = o2 > kmax ? o2 : kmax;
    slow += __shfl_xor_sync(FULL_MASK, slow, d);
    overflow += __shfl_xor_sync(FULL_MASK, overflow, d);
    top = max(top, __shfl_xor_sync(FULL_MASK, top, d));
  }
  if (lane == 0) {
    if (DENSE && overflow) atomicAdd(a.overflow, overflow);
    if (DENSE && top) atomicMax(a.dense_meta + DM_MAX, (unsigned long long)top);
    if (!DENSE && kmin <= kmax) {
      atomicMin(a.key_minmax, (unsigned long long)kmin);
      atomicMax(a.key_minmax + 1, (unsigned long long)kmax);
    }
    if (slow) atomicAdd(a.slow_rows, slow);
  }
}

// ================================================================================================
// the direct-address count table as a relation of its own (DeferredTable): emit / MAX / "count = v"
// ================================================================================================
struct DenseScanArgs {
  CompactScratch sc;
  const uint32_t* table;
  unsigned long long n_slots;
  const unsigned long long* meta;      // [0] key of slot 0
  const unsigned long long* eq_value;  // SELECT: keep slots whose count equals *eq_value
  uint32_t* key_dst;                   // may be NULL
  unsigned long long* count_dst;       // may be NULL
  int32_t n_bcast, pad;                // SELECT: columns of the one-row side, repeated for every survivor
  const void* bcast_src[MAX_IN_COLS];
  void* bcast_dst[MAX_IN_COLS];
  int32_t bcast_width[MAX_IN_COLS];
};

// SELECT = false: every non-empty slot; true: the slots whose count equals *eq_value.  Stable (ascending key).
template <bool SELECT>
__global__ void __launch_bounds__(CP_THREADS) dense_scan_kernel(const __grid_constant__ DenseScanArgs a) {
  constexpr int E = 4, I = 64, G = I / E, TILE = CP_THREADS * I;
  __shared__ CompactSmem<E, I> sm;
  const int tid = threadIdx.x, warp = tid >> 5;
  const unsigned long long want = SELECT ? *a.eq_value : 0ull;
  const unsigned gbase = unsigned(a.meta[DM_FIRST_KEY]);
  const unsigned long long used = a.meta[DM_SLOTS];  // slots in use (device-decided, <= n_slots): the tiles behind them are empty
  long long tile;
  for (int it = 0; (tile = cp_next_tile(sm, a.sc, it)) >= 0; ++it) {
    const unsigned long long tile_base = (unsigned long long)tile * TILE;
    unsigned long long bits = 0;
    uint4 c[G];
#pragma unroll
    for (int g = 0; g < G; ++g) {
      const unsigned long long slot0 = tile_base + ((unsigned long long)g * CP_THREADS + tid) * E;
      c[g] = make_uint4(0, 0, 0, 0);
      if (slot0 < used) c[g] = *reinterpret_cast<const uint4*>(a.table + slot0);  // slot counts are multiples of 4
      unsigned nib;
      if (SELECT) nib = unsigned(c[g].x == want && c[g].x) | (unsigned(c[g].y == want && c[g].y) << 1) | (unsigned(c[g].z == want && c[g].z) << 2) | (unsigned(c[g].w == want && c[g].w) << 3);
      else nib = unsigned(c[g].x != 0) | (unsigned(c[g].y != 0) << 1) | (unsigned(c[g].z != 0) << 2) | (unsigned(c[g].w != 0) << 3);
      bits |= (unsigned long long)nib << (g * E);
    }
    unsigned lane_prefix[G];
    cp_rank_tile<E, I>(sm, a.sc, tile, bits, lane_prefix);
    if (bits && sm.tile_total) {
#pragma unroll
      for (int g = 0; g < G; ++g) {
        const unsigned nib = unsigned(bits >> (g * E)) & 0xfu;
        if (!nib) continue;
        const unsigned long long slot0 = tile_base + ((unsigned long long)g * CP_THREADS + tid) * E;
        const int64_t pos0 = int64_t(sm.excl) + sm.group_warp[g][warp] + lane_prefix[g];
        const unsigned cs[4] = {c[g].x, c[g].y, c[g].z, c[g].w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if (!((nib >> e) & 1u)) continue;
          const int64_t pos = pos0 + __popc(nib & ((1u << e) - 1u));
          if (a.key_dst) a.key_dst[pos] = gbase + unsigned(slot0) + unsigned(e);
          if (a.count_dst) a.count_dst[pos] = cs[e];
          if (SELECT) {
            for (int b = 0; b < a.n_bcast; ++b) {
              if (a.bcast_width[b] == 4) static_cast<uint32_t*>(a.bcast_dst[b])[pos] = *static_cast<const uint32_t*>(a.bcast_src[b]);
              else static_cast<unsigned long long*>(a.bcast_dst[b])[pos] = *static_cast<const unsigned long long*>(a.bcast_src[b]);
            }
          }
        }
      }
    }
    __syncthreads();
  }
}

// "count = MAX(count)" (NEXMark q5's join with its MaxBids subquery) in one cooperative launch.  MAX(count) is a
// by-product of the scan (meta[DM_MAX]); every CTA owns a contiguous range of the table, (1) counts its slots that
// reach the maximum, (2) after a grid-wide barrier writes them behind those of the CTAs before it -- ascending key
// order, like the row-by-row path.  The table is L2-resident (it was just built); what is saved against the
// operator-by-operator plan is a MAX pass, a 8-byte relation, a join launch and the host's wait in between.
struct DenseArgmaxArgs {
  const uint32_t* table;
  unsigned long long* meta;   // DM_MAX from the scan; DM_BARRIER2 is zero on entry (the caller zeroed the meta words before the scan)
  unsigned* cta_counts;       // [gridDim.x]
  uint32_t* key_dst;          // may be NULL
  unsigned long long* count_dst;
  int32_t n_max_dst, pad;
  unsigned long long* max_dst[4];  // columns that repeat the maximum for every output row (the one-row side of the join)
  unsigned long long* out_count;   // device
  unsigned long long* host_count;  // page-locked copy (PendingRows)
};

__device__ __forceinline__ void dense_grid_barrier(unsigned long long* word, unsigned n_ctas) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(word, 1ull);
    while (ld_relaxed_u64(word) < n_ctas) __nanosleep(64);
    __threadfence();
  }
  __syncthreads();
}

constexpr int AM_REGS = 16;  // uint4 a thread keeps in registers between the phases (covers 592 x 256 x 16 x 4 = 9.7 M slots)

__global__ void __launch_bounds__(256, 3) dense_argmax_kernel(const __grid_constant__ DenseArgmaxArgs a) {
  __shared__ unsigned s_cnt[AM_REGS][8];
  __shared__ unsigned s_part[8];
  __shared__ unsigned long long s_excl;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned long long n4 = a.meta[DM_SLOTS] >> 2;
  const unsigned long long per_cta = (n4 + gridDim.x - 1) / gridDim.x;
  const unsigned long long lo4 = blockIdx.x * per_cta, hi4 = lo4 + per_cta < n4 ? lo4 + per_cta : n4;
  const uint4* t4 = reinterpret_cast<const uint4*>(a.table);
  // element (k, tid) of the CTA's range is uint4 number lo4 + k * 256 + tid: coalesced, and (k, tid) order = key order.
  // The first AM_REGS rounds stay in registers between the two phases; longer ranges are read again.
  // (MAX(count) itself is already in meta[DM_MAX]: the scan kernel tracked it through its atomics.)
  const bool in_regs = per_cta <= 256ull * AM_REGS;
  uint4 c[AM_REGS];
#pragma unroll
  for (int k = 0; k < AM_REGS; ++k) {
    const unsigned long long i = lo4 + (unsigned long long)k * 256 + tid;
    c[k] = i < hi4 ? t4[i] : make_uint4(0, 0, 0, 0);
  }
  const unsigned top = unsigned(a.meta[DM_MAX]);
  auto hits = [&](const uint4& v) { return unsigned(v.x == top) + unsigned(v.y == top) + unsigned(v.z == top) + unsigned(v.w == top); };
  // ---- how many of my slots reach the maximum.  Nearly always none or one in the whole grid: decide per CTA first.
  unsigned mine = 0;
  if (top) {
#pragma unroll
    for (int k = 0; k < AM_REGS; ++k) mine += hits(c[k]);
    if (!in_regs)
      for (unsigned long long i = lo4 + 256ull * AM_REGS + tid; i < hi4; i += 256) mine += hits(t4[i]);
  }
  const int any = __syncthreads_or(mine != 0);
  unsigned total = 0;
  if (any) {
    const unsigned w = warp_sum(mine);
    if (lane == 0) s_part[warp] = w;
    __syncthreads();
#pragma unroll
    for (int x = 0; x < 8; ++x) total += s_part[x];
  }
  if (tid == 0) a.cta_counts[blockIdx.x] = total;
  dense_grid_barrier(a.meta + DM_BARRIER2, gridDim.x);
  // ---- exclusive prefix over the CTAs
  unsigned long long part = 0;
  for (unsigned b = tid; b < blockIdx.x; b += 256) part += *reinterpret_cast<volatile unsigned*>(a.cta_counts + b);
  part = warp_sum(part);
  if (lane == 0) s_part[warp] = unsigned(part);
  __syncthreads();
  if (tid == 0) {
    unsigned long long e = 0;
    for (int x = 0; x < 8; ++x) e += s_part[x];
    s_excl = e;
    if (blockIdx.x == gridDim.x - 1) {
      *a.out_count = e + total;
      if (a.host_count) *reinterpret_cast<volatile unsigned long long*>(a.host_count) = e + total;
    }
  }
  __syncthreads();
  if (!any) return;
  // ---- the rare CTA that holds a maximum: write its hits in (k, tid) order
  const unsigned gbase = unsigned(a.meta[DM_FIRST_KEY]);
  unsigned long long pos = s_excl;
  const unsigned long long rounds = (per_cta + 255) / 256;
  for (unsigned long long k = 0; k < rounds; ++k) {
    const unsigned long long i = lo4 + k * 256 + tid;
    const uint4 v = i < hi4 ? t4[i] : make_uint4(0, 0, 0, 0);  // L2 / L1 hit: this CTA just read it
    const unsigned h = top ? hits(v) : 0u;
    const unsigned incl = warp_inclusive_sum(h);
    __syncthreads();
    if (lane == 31) s_part[warp] = incl;
    __syncthreads();
    unsigned before = 0, round_total = 0;
#pragma unroll
    for (int x = 0; x < 8; ++x) {
      if (x < warp) before += s_part[x];
      round_total += s_part[x];
    }
    if (h) {
      unsigned long long p = pos + before + (incl - h);
      const unsigned cs[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (cs[e] == top) {
          if (a.key_dst) a.key_dst[p] = gbase + unsigned(i * 4) + unsigned(e);
          if (a.count_dst) a.count_dst[p] = top;
          for (int q = 0; q < a.n_max_dst; ++q) a.max_dst[q][p] = top;
          ++p;
        }
    }
    pos += round_total;
  }
  (void)s_cnt;
}

// ================================================================================================
// level 2: global table (packed 64-bit keys)
// ================================================================================================
struct AggTable {
  unsigned long long* keys;  // [cap + 1]; slot `cap` is reserved for the key equal to EMPTY_KEY (NULL when dense)
  unsigned long long* acc;   // [n_acc][cap + 1]
  unsigned long long cap;    // hashed: power of two; dense: max_key - min_key + 1
  // dense (direct-address) table: slot = key - dense_base.  NEXMark ids are dense ranges (auction ids of a window
  // are consecutive integers), so level 2 needs no hashing, no CAS and a table that mostly lives in L2
  // (q5: 6.5 M auctions x 9 B = 58 MB), where random 64-bit atomics run several times faster than in DRAM.
  unsigned char* present;    // [cap + 1] dense only
  unsigned long long dense_base;
  unsigned long long stride; // slots between accumulator columns: cap + 1 rounded up to 4 (the emit kernel reads 4 slots per load)
};

__global__ void agg_init_kernel(AggTable t, int n_acc, unsigned long long ident0, unsigned long long ident1, unsigned long long ident2,
                                unsigned long long ident3, unsigned long long ident4, unsigned long long ident5, unsigned long long ident6,
                                unsigned long long ident7) {
  const unsigned long long ident[MAX_ACC] = {ident0, ident1, ident2, ident3, ident4, ident5, ident6, ident7};
  const unsigned long long n = t.cap + 1;
  for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
    if (t.keys) t.keys[i] = EMPTY_KEY;
    for (int c = 0; c < n_acc; ++c) t.acc[c * t.stride + i] = ident[c];
  }
}

struct AggInsertArgs {
  int64_t n;  // rows or partial entries
  KeyPack keys;
  int32_t n_acc;
  int32_t from_partials;
  AccDesc acc[MAX_ACC];
  ColRef cols[MAX_IN_COLS];
  const unsigned long long* part_keys;
  const unsigned long long* part_acc;
  int64_t part_capacity;
  int32_t part32;  // from_partials: keys / single accumulator are uint32_t arrays (the 4-byte-key level-1 kernels)
  int32_t pad2;
  AggTable table;
};

__device__ __forceinline__ unsigned long long table_find_or_insert(const AggTable& t, unsigned long long key) {
  if (t.present) {
    const unsigned long long slot = key - t.dense_base;
    t.present[slot] = 1;  // idempotent plain store
    return slot;
  }
  if (key == EMPTY_KEY) {
    t.keys[t.cap] = 0;  // marks the reserved slot occupied (idempotent plain store)
    return t.cap;
  }
  unsigned long long slot = fmix64(key) & (t.cap - 1);
  while (true) {
    unsigned long long cur = t.keys[slot];
    if (cur == key) return slot;
    if (cur == EMPTY_KEY) {
      unsigned long long old = atomicCAS(&t.keys[slot], EMPTY_KEY, key);
      if (old == EMPTY_KEY || old == key) return slot;
    }
    slot = (slot + 1) & (t.cap - 1);
  }
}

__global__ void __launch_bounds__(256) agg_insert_kernel(const __grid_constant__ AggInsertArgs a) {
  const unsigned long long stride_n = a.table.stride;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < a.n; i += int64_t(gridDim.x) * blockDim.x) {
    const unsigned long long key = !a.from_partials ? pack_key(a.keys, a.cols, i)
                                   : a.part32       ? (unsigned long long)reinterpret_cast<const uint32_t*>(a.part_keys)[i]
                                                    : a.part_keys[i];
    const unsigned long long slot = table_find_or_insert(a.table, key);
    for (int c = 0; c < a.n_acc; ++c) {
      Val v;
      int op;
      if (a.from_partials) {
        v.u = a.part32 ? (unsigned long long)reinterpret_cast<const uint32_t*>(a.part_acc)[i] : a.part_acc[int64_t(c) * a.part_capacity + i];
        op = acc_merge_op(a.acc[c].op);
      } else {
        if (!acc_input_valid(a.acc[c], a.cols, i)) continue;
        v = load_acc_input(a.acc[c], a.cols, i);
        op = a.acc[c].op;
      }
      acc_apply(&a.table.acc[c * stride_n + slot], op, v);
    }
  }
}

// ================================================================================================
// row-representative table (Utf8 / wide keys)
// ================================================================================================
struct AggRowsArgs {
  int64_t n_rows;
  RowKeys keys;
  int32_t n_acc;
  AccDesc acc[MAX_ACC];
  ColRef cols[MAX_IN_COLS];
  unsigned* owner;          // [cap]
  unsigned long long* tacc; // [n_acc][cap]
  unsigned long long cap;
  unsigned long long* n_groups;  // number of slots claimed = number of distinct keys
};

__global__ void agg_rows_init_kernel(unsigned* owner, unsigned long long* tacc, unsigned long long cap, int n_acc, unsigned long long ident0,
                                     unsigned long long ident1, unsigned long long ident2, unsigned long long ident3, unsigned long long ident4,
                                     unsigned long long ident5, unsigned long long ident6, unsigned long long ident7) {
  const unsigned long long ident[MAX_ACC] = {ident0, ident1, ident2, ident3, ident4, ident5, ident6, ident7};
  for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < cap; i += (unsigned long long)gridDim.x * blockDim.x) {
    owner[i] = EMPTY_OWNER;
    for (int c = 0; c < n_acc; ++c) tacc[c * cap + i] = ident[c];
  }
}

__global__ void __launch_bounds__(256) agg_insert_rows_kernel(const __grid_constant__ AggRowsArgs a) {
  unsigned claimed = 0;
  for (int64_t row = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; row < a.n_rows; row += int64_t(gridDim.x) * blockDim.x) {
    unsigned long long slot = hash_row(a.keys, a.cols, row) & (a.cap - 1);
    while (true) {
      unsigned cur = a.owner[slot];
      if (cur == EMPTY_OWNER) {
        cur = atomicCAS(&a.owner[slot], EMPTY_OWNER, unsigned(row));
        if (cur == EMPTY_OWNER) {  // we own the slot: `row` is the group's representative
          ++claimed;
          break;
        }
      }
      if (rows_equal(a.keys, a.cols, int64_t(cur), a.keys, a.cols, row)) break;
      slot = (slot + 1) & (a.cap - 1);
    }
    for (int c = 0; c < a.n_acc; ++c)
      if (acc_input_valid(a.acc[c], a.cols, row)) acc_apply(&a.tacc[c * a.cap + slot], a.acc[c].op, load_acc_input(a.acc[c], a.cols, row));
  }
  claimed = warp_sum(claimed);
  if ((threadIdx.x & 31) == 0 && claimed) atomicAdd(a.n_groups, (unsigned long long)claimed);
}

// ---- level 1 for row keys: CTA-local pre-aggregation (TPC-H q1: ~6 M rows per SF into 4 (Utf8, Utf8) groups, where
// agg_insert_rows_kernel would send every thread of the GPU to the same four slots).  Each CTA owns a contiguous row
// range and keeps an open-addressing table of RL_SLOTS slots in shared memory: one 64-bit word (hash tag << 32 | the
// group's representative row) and one accumulator per aggregate.  A probe compares the tag first, then the key columns
// (rows_equal).  Lanes of a warp that land on the same slot combine their values first (__match_any_sync on the slot,
// then the leader folds its peers' values in), so a warp step costs one shared atomic per distinct slot and
// accumulator.  Before a tile could take the table past 3/4 full, and at the end, the CTA merges its entries into the
// level-2 row table (agg_insert_rows_kernel's table, keyed by representative row) with the merge operation of each
// accumulator; agg_emit_kernel<2> then runs unchanged.
constexpr int RL_SLOTS = 1024;
constexpr int RL_THREADS = 256;
constexpr unsigned long long RL_EMPTY = ~0ull;

__device__ __forceinline__ void rows_table_merge(const AggRowsArgs& a, unsigned rep, const unsigned long long* s_acc, int s, unsigned* claimed) {
  unsigned long long slot = hash_row(a.keys, a.cols, rep) & (a.cap - 1);
  while (true) {
    unsigned cur = a.owner[slot];
    if (cur == EMPTY_OWNER) {
      cur = atomicCAS(&a.owner[slot], EMPTY_OWNER, rep);
      if (cur == EMPTY_OWNER) {
        ++*claimed;
        break;
      }
    }
    if (rows_equal(a.keys, a.cols, int64_t(cur), a.keys, a.cols, rep)) break;
    slot = (slot + 1) & (a.cap - 1);
  }
  for (int c = 0; c < a.n_acc; ++c) {
    Val v;
    v.u = s_acc[c * RL_SLOTS + s];
    acc_apply(&a.tacc[c * a.cap + slot], acc_merge_op(a.acc[c].op), v);
  }
}

__global__ void __launch_bounds__(RL_THREADS) agg_rows_local_kernel(const __grid_constant__ AggRowsArgs a, int64_t rows_per_cta) {
  extern __shared__ unsigned long long rl_smem[];
  unsigned long long* s_word = rl_smem;              // [RL_SLOTS]
  unsigned long long* s_acc = rl_smem + RL_SLOTS;    // [n_acc][RL_SLOTS]
  const int lane = threadIdx.x & 31;
  for (int s = threadIdx.x; s < RL_SLOTS; s += blockDim.x) {
    s_word[s] = RL_EMPTY;
    for (int c = 0; c < a.n_acc; ++c) s_acc[c * RL_SLOTS + s] = acc_identity(a.acc[c].op);
  }
  __syncthreads();
  unsigned claimed = 0;
  int used = 0;  // slots in use, the same in every thread (__syncthreads_count)
  auto flush = [&]() {
    __syncthreads();
    for (int s = threadIdx.x; s < RL_SLOTS; s += blockDim.x) {
      const unsigned long long w = s_word[s];
      if (w == RL_EMPTY) continue;
      rows_table_merge(a, unsigned(w), s_acc, s, &claimed);
      s_word[s] = RL_EMPTY;
      for (int c = 0; c < a.n_acc; ++c) s_acc[c * RL_SLOTS + s] = acc_identity(a.acc[c].op);
    }
    used = 0;
    __syncthreads();
  };
  const int64_t begin = int64_t(blockIdx.x) * rows_per_cta;
  const int64_t end = begin + rows_per_cta < a.n_rows ? begin + rows_per_cta : a.n_rows;
  for (int64_t base = begin; base < end; base += RL_THREADS) {
    // a tile claims at most RL_THREADS slots: flush first when that could pass 3/4 of the table
    if (used + RL_THREADS > RL_SLOTS * 3 / 4) flush();
    const int64_t row = base + threadIdx.x;
    const bool live = row < end;
    unsigned slot = 0xffffffffu;
    bool new_slot = false;
    if (live) {
      const unsigned long long h = hash_row(a.keys, a.cols, row);
      const unsigned long long mine = ((h >> 32) << 32) | (unsigned long long)unsigned(row);
      unsigned s = unsigned(h) & (RL_SLOTS - 1);
      while (true) {
        unsigned long long w = s_word[s];
        if (w == RL_EMPTY) {
          w = atomicCAS(&s_word[s], RL_EMPTY, mine);
          if (w == RL_EMPTY) {
            new_slot = true;
            break;
          }
        }
        if ((w >> 32) == (h >> 32) && rows_equal(a.keys, a.cols, int64_t(unsigned(w)), a.keys, a.cols, row)) break;
        s = (s + 1) & (RL_SLOTS - 1);
      }
      slot = s;
    }
    const unsigned peers = __match_any_sync(FULL_MASK, slot);
    const int leader = __ffs(peers) - 1;
    // lanes whose value a leader folds in: every live lane that is not its group's leader (warp-uniform)
    const unsigned others = __ballot_sync(FULL_MASK, live && lane != leader);
    for (int c = 0; c < a.n_acc; ++c) {
      const AccDesc d = a.acc[c];
      const int op = d.op == ACC_COUNT ? ACC_ADD_I : d.op;  // a count adds 1 per row with a non-NULL argument
      Val v;
      v.u = acc_identity(op);
      if (live && acc_input_valid(d, a.cols, row)) {
        if (d.op == ACC_COUNT) v.u = 1;
        else v = load_acc_input(d, a.cols, row);
      }
      for (unsigned m = others; m; m &= m - 1) {
        const int k = __ffs(m) - 1;
        Val o;
        o.u = __shfl_sync(FULL_MASK, v.u, k);
        if (lane == leader && ((peers >> k) & 1u)) v = acc_combine(op, v, o);
      }
      if (live && lane == leader) acc_apply(&s_acc[c * RL_SLOTS + slot], op, v);
    }
    used += __syncthreads_count(new_slot);
  }
  flush();
  claimed = warp_sum(claimed);
  if (lane == 0 && claimed) atomicAdd(a.n_groups, (unsigned long long)claimed);
}

// ================================================================================================
// emit: compaction of the occupied slots
// ================================================================================================
struct AggEmitArgs {
  CompactScratch sc;
  unsigned long long n_slots;       // slots to scan (cap + 1 packed, cap rows mode)
  unsigned long long acc_stride;    // slots between accumulator columns (multiple of 4, >= n_slots)
  const unsigned long long* keys;   // packed hashed mode (NULL otherwise)
  const unsigned char* present;     // packed dense mode: key = dense_base + slot
  unsigned long long dense_base;
  const unsigned* owner;            // rows mode
  const unsigned long long* acc;    // [n_acc][acc_stride]
  int32_t n_emit;
  int32_t n_key_out;                // packed mode: 1 or 2 key columns
  int32_t key_width[2];
  void* key_dst[2];
  unsigned* rep_rows;               // rows mode: representative row per group
  EmitDesc emit[2 * MAX_ACC];
};

__device__ __forceinline__ void emit_values(const EmitDesc* emit, int n_emit, const unsigned long long* acc, unsigned long long stride,
                                            unsigned long long slot, int64_t pos) {
  for (int e = 0; e < n_emit; ++e) {
    const EmitDesc& d = emit[e];
    Val v;
    v.u = acc[d.a0 * stride + slot];
    if (d.kind == EMIT_AVG) {
      Val s;
      s.u = acc[d.a1 * stride + slot];
      v.d = __ddiv_rn(s.d, __ull2double_rn(v.u));
    } else if (d.kind == EMIT_F64_ORDER) {
      v.u = f64_from_order_key(v.u);
    }
    store_val(d.dst, d.out_dtype, pos, v);
    if (d.valid_dst) d.valid_dst[pos] = acc[d.valid_acc * stride + slot] != 0ull;
  }
}

// MODE 0: hashed packed keys, 1: dense (direct-address) table, 2: row-representative table.
// A thread owns groups of FOUR CONTIGUOUS slots: the occupancy test is one vector load per group (32 B of keys,
// 4 present bytes or 16 B of owners), the ranking is the packed SWAR scan of compact.cuh, and a group's accumulators
// are read with two 16-byte loads per column whatever its occupancy.  (The first version tested and emitted slot by
// slot: 138 lane-instructions per slot and one dependent accumulator load per survivor.)
// EMIT_ITEMS = slots per thread and tile: 64 for large tables (16 Ki-slot tiles: q5's 6.5 M-slot table is 397 tiles =
// ONE wave with the cheap single-wave prefix instead of 1587 tiles in three waves of look-back), 16 for small
// tables so that they still spread over the SMs.
template <int MODE, int EMIT_ITEMS>
__global__ void __launch_bounds__(CP_THREADS) agg_emit_kernel(const __grid_constant__ AggEmitArgs a) {
  constexpr int E = 4;
  constexpr int CP_ITEMS = EMIT_ITEMS;
  constexpr int G = CP_ITEMS / E;
  constexpr int CP_TILE = CP_THREADS * CP_ITEMS;
  __shared__ CompactSmem<E, CP_ITEMS> sm;
  const int tid = threadIdx.x, warp = tid >> 5;
  long long tile;
  for (int it = 0; (tile = cp_next_tile(sm, a.sc, it)) >= 0; ++it) {
    const unsigned long long tile_base = (unsigned long long)tile * CP_TILE;
    unsigned long long bits = 0;
#pragma unroll
    for (int g = 0; g < G; ++g) {
      const unsigned long long slot0 = tile_base + ((unsigned long long)g * CP_THREADS + tid) * E;
      unsigned nib = 0;
      if (slot0 < a.n_slots) {
        if (MODE == 0) {
          const ulonglong2 k01 = *reinterpret_cast<const ulonglong2*>(a.keys + slot0);
          const ulonglong2 k23 = *reinterpret_cast<const ulonglong2*>(a.keys + slot0 + 2);
          nib = unsigned(k01.x != EMPTY_KEY) | (unsigned(k01.y != EMPTY_KEY) << 1) | (unsigned(k23.x != EMPTY_KEY) << 2) | (unsigned(k23.y != EMPTY_KEY) << 3);
        } else if (MODE == 1) {
          const unsigned p4 = *reinterpret_cast<const unsigned*>(a.present + slot0);
          nib = unsigned((p4 & 0xffu) != 0) | (unsigned((p4 & 0xff00u) != 0) << 1) | (unsigned((p4 & 0xff0000u) != 0) << 2) | (unsigned((p4 >> 24) != 0) << 3);
        } else {
          const uint4 o = *reinterpret_cast<const uint4*>(a.owner + slot0);
          nib = unsigned(o.x != EMPTY_OWNER) | (unsigned(o.y != EMPTY_OWNER) << 1) | (unsigned(o.z != EMPTY_OWNER) << 2) | (unsigned(o.w != EMPTY_OWNER) << 3);
        }
        const unsigned long long left = a.n_slots - slot0;  // the padding slots behind the table are not part of it
        if (left < 4) nib &= (1u << left) - 1u;
      }
      bits |= (unsigned long long)nib << (g * E);
    }
    unsigned lane_prefix[G];
    cp_rank_tile<E, CP_ITEMS>(sm, a.sc, tile, bits, lane_prefix);
    if (bits && sm.tile_total) {
#pragma unroll
      for (int g = 0; g < G; ++g) {
        const unsigned nib = unsigned(bits >> (g * E)) & 0xfu;
        if (!nib) continue;
        const unsigned long long slot0 = tile_base + ((unsigned long long)g * CP_THREADS + tid) * E;
        const int64_t pos0 = int64_t(sm.excl) + sm.group_warp[g][warp] + lane_prefix[g];
        // output position of element e of the group: pos0 + number of survivors below it
        int64_t pos[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) pos[e] = pos0 + __popc(nib & ((1u << e) - 1u));
        if (MODE == 2) {
          const uint4 o = *reinterpret_cast<const uint4*>(a.owner + slot0);
          const unsigned r[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if ((nib >> e) & 1u) a.rep_rows[pos[e]] = r[e];
        } else {
          unsigned long long key[4];
          if (MODE == 0) {
            const ulonglong2 k01 = *reinterpret_cast<const ulonglong2*>(a.keys + slot0);
            const ulonglong2 k23 = *reinterpret_cast<const ulonglong2*>(a.keys + slot0 + 2);
            key[0] = k01.x; key[1] = k01.y; key[2] = k23.x; key[3] = k23.y;
#pragma unroll
            for (int e = 0; e < 4; ++e)
              if (slot0 + e == a.n_slots - 1) key[e] = EMPTY_KEY;  // the reserved slot of the key that equals EMPTY_KEY
          } else {
#pragma unroll
            for (int e = 0; e < 4; ++e) key[e] = a.dense_base + slot0 + e;
          }
          if (a.n_key_out == 2) {
#pragma unroll
            for (int e = 0; e < 4; ++e)
              if ((nib >> e) & 1u) {
                static_cast<uint32_t*>(a.key_dst[0])[pos[e]] = uint32_t(key[e] >> 32);
                static_cast<uint32_t*>(a.key_dst[1])[pos[e]] = uint32_t(key[e]);
              }
          } else if (a.key_width[0] == 4) {
#pragma unroll
            for (int e = 0; e < 4; ++e)
              if ((nib >> e) & 1u) static_cast<uint32_t*>(a.key_dst[0])[pos[e]] = uint32_t(key[e]);
          } else {
#pragma unroll
            for (int e = 0; e < 4; ++e)
              if ((nib >> e) & 1u) static_cast<unsigned long long*>(a.key_dst[0])[pos[e]] = key[e];
          }
        }
        for (int c = 0; c < a.n_emit; ++c) {
          const EmitDesc& d = a.emit[c];
          const unsigned long long* p0 = a.acc + d.a0 * a.acc_stride + slot0;
          const ulonglong2 v01 = *reinterpret_cast<const ulonglong2*>(p0), v23 = *reinterpret_cast<const ulonglong2*>(p0 + 2);
          Val v[4];
          v[0].u = v01.x; v[1].u = v01.y; v[2].u = v23.x; v[3].u = v23.y;
          if (d.kind == EMIT_AVG) {
            const unsigned long long* p1 = a.acc + d.a1 * a.acc_stride + slot0;
            const ulonglong2 s01 = *reinterpret_cast<const ulonglong2*>(p1), s23 = *reinterpret_cast<const ulonglong2*>(p1 + 2);
            Val sv[4];
            sv[0].u = s01.x; sv[1].u = s01.y; sv[2].u = s23.x; sv[3].u = s23.y;
#pragma unroll
            for (int e = 0; e < 4; ++e) v[e].d = __ddiv_rn(sv[e].d, __ull2double_rn(v[e].u));
          }
          if (d.valid_dst) {
            const unsigned long long* pv = a.acc + d.valid_acc * a.acc_stride + slot0;
#pragma unroll
            for (int e = 0; e < 4; ++e)
              if ((nib >> e) & 1u) d.valid_dst[pos[e]] = pv[e] != 0ull;
          }
          // one uniform width branch per column instead of a type switch per element
          if (d.out_dtype == FLOCKGPU_INT32 || d.out_dtype == FLOCKGPU_UINT32 || d.out_dtype == FLOCKGPU_DATE32) {
#pragma unroll
            for (int e = 0; e < 4; ++e)
              if ((nib >> e) & 1u) static_cast<uint32_t*>(d.dst)[pos[e]] = uint32_t(v[e].u);
          } else {
            // decoded at the store: MIN / MAX of Float64 leave their order-key form here
            const bool decode = d.kind == EMIT_F64_ORDER;
#pragma unroll
            for (int e = 0; e < 4; ++e)
              if ((nib >> e) & 1u) static_cast<unsigned long long*>(d.dst)[pos[e]] = decode ? f64_from_order_key(v[e].u) : v[e].u;
          }
        }
      }
    }
    __syncthreads();
  }
}

// ================================================================================================
// no group columns: one global accumulator row
// ================================================================================================
struct AggGlobalArgs {
  int64_t n_rows;
  int32_t n_acc;
  int32_t pad;
  AccDesc acc[MAX_ACC];
  ColRef cols[MAX_IN_COLS];
  unsigned long long* state;  // [n_acc], pre-initialised to the identities
};

__global__ void __launch_bounds__(256) agg_global_kernel(const __grid_constant__ AggGlobalArgs a) {
  Val local[MAX_ACC];
#pragma unroll
  for (int c = 0; c < MAX_ACC; ++c) local[c].u = c < a.n_acc ? acc_identity(a.acc[c].op) : 0ull;
  // four rows per thread and iteration: their loads are independent and in flight together
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  int64_t row = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
  for (; row + 3 * stride < a.n_rows; row += 4 * stride) {
#pragma unroll
    for (int c = 0; c < MAX_ACC; ++c) {
      if (c >= a.n_acc) continue;
      Val v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = load_acc_input(a.acc[c], a.cols, row + u * stride);
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (acc_input_valid(a.acc[c], a.cols, row + u * stride)) local[c] = acc_combine(a.acc[c].op, local[c], v[u]);
    }
  }
  for (; row < a.n_rows; row += stride) {
#pragma unroll
    for (int c = 0; c < MAX_ACC; ++c)
      if (c < a.n_acc && acc_input_valid(a.acc[c], a.cols, row)) local[c] = acc_combine(a.acc[c].op, local[c], load_acc_input(a.acc[c], a.cols, row));
  }
#pragma unroll
  for (int c = 0; c < MAX_ACC; ++c) {
    if (c >= a.n_acc) break;
    const int mop = acc_merge_op(a.acc[c].op);
    Val v = local[c];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      Val o;
      o.u = __shfl_xor_sync(FULL_MASK, v.u, d);
      v = acc_combine(mop, v, o);
    }
    if ((threadIdx.x & 31) == 0) acc_apply(&a.state[c], mop, v);
  }
}

struct AggEmitOneArgs {
  const unsigned long long* state;
  int32_t n_emit;
  EmitDesc emit[2 * MAX_ACC];
};
__global__ void agg_emit_one_kernel(const __grid_constant__ AggEmitOneArgs a) {
  if (threadIdx.x == 0 && blockIdx.x == 0) emit_values(a.emit, a.n_emit, a.state, 1, 0, 0);
}

// ================================================================================================
// host
// ================================================================================================
namespace {

bool is_unsigned_dt(int dt) { return dt == FLOCKGPU_UINT32 || dt == FLOCKGPU_UINT64; }
bool is_signed_dt(int dt) { return dt == FLOCKGPU_INT32 || dt == FLOCKGPU_INT64 || dt == FLOCKGPU_TIMESTAMP || dt == FLOCKGPU_DATE32; }

struct OutPlan {
  std::string name;
  int dtype;
  std::string format;
  int kind, a0, a1;
  int valid_acc = -1;  // accumulator counting the non-NULL inputs of this aggregate: 0 at the end = the result is NULL
};

struct AggPlan {
  std::vector<AccDesc> accs;
  std::vector<OutPlan> outs;
  unsigned long long ident[MAX_ACC] = {};  // identity of each accumulator
  int n_acc() const { return int(accs.size()); }
};

const char* func_name(int f) {
  switch (f) {
    case FLOCKGPU_AGG_COUNT: return "COUNT";
    case FLOCKGPU_AGG_SUM: return "SUM";
    case FLOCKGPU_AGG_MIN: return "MIN";
    case FLOCKGPU_AGG_MAX: return "MAX";
    default: return "AVG";
  }
}

int minmax_op(int dtype, bool is_min, const char* what) {
  if (dtype == FLOCKGPU_FLOAT64) return is_min ? ACC_MIN_F : ACC_MAX_F;
  if (is_unsigned_dt(dtype)) return is_min ? ACC_MIN_U : ACC_MAX_U;
  if (is_signed_dt(dtype)) return is_min ? ACC_MIN_I : ACC_MAX_I;
  fail(FLOCKGPU_ERR_UNSUPPORTED, "hash_aggregate: %s over %s", what, dtype_name(dtype));
}

// Translates (mode, aggregate list) into accumulators + output columns.
AggPlan plan_aggregates(const Table& in, int mode, const std::vector<AggSpec>& aggs) {
  AggPlan plan;
  std::vector<AccDesc>* accs = &plan.accs;
  std::vector<OutPlan>* outs = &plan.outs;
  const bool from_states = mode == FLOCKGPU_AGG_FINAL || mode == FLOCKGPU_AGG_FINAL_PARTITIONED;
  const bool partial_out = mode == FLOCKGPU_AGG_PARTIAL;
  auto add_acc = [&](int op, int col, int cvt) {
    // identical accumulators are one: "how many non-NULL values of column c" is wanted by COUNT(c) and by the validity
    // of SUM / MIN / MAX / AVG over c, COUNT(*) by every AVG over a non-nullable column, SUM(x) by AVG(x) (TPC-H q1's
    // eleven accumulators are six)
    for (size_t i = 0; i < accs->size(); ++i)
      if ((*accs)[i].op == op && (*accs)[i].col == col && (*accs)[i].cvt == cvt) return int(i);
    FG_CHECK(accs->size() < size_t(MAX_ACC), FLOCKGPU_ERR_UNSUPPORTED, "hash_aggregate: more than %d accumulators", MAX_ACC);
    accs->push_back(AccDesc{op, col, cvt, 0});
    return int(accs->size()) - 1;
  };
  auto col_dtype = [&](int col, const char* what) {
    FG_CHECK(col >= 0 && col < int(in.cols.size()), FLOCKGPU_ERR_INVALID, "hash_aggregate: %s column %d out of range", what, col);
    FG_CHECK(!in.cols[col].all_null, FLOCKGPU_ERR_UNSUPPORTED, "hash_aggregate: NULL input column");
    return in.cols[col].dtype;
  };
  // an argument (or state) column with NULLs: the aggregate skips them, and a group that saw nothing else is NULL
  auto nulls_in = [&](int col) { return col >= 0 && col < int(in.cols.size()) && in.cols[col].validity != nullptr; };
  auto valid_counter = [&](int col) { return nulls_in(col) ? add_acc(ACC_COUNT, col, CVT_NONE) : -1; };
  for (const AggSpec& s : aggs) {
    const std::string base = s.name.empty() ? std::string(func_name(s.func)) : s.name;
    switch (s.func) {
      case FLOCKGPU_AGG_COUNT: {
        int a;
        if (from_states) {
          FG_CHECK(col_dtype(s.col, "COUNT state") == FLOCKGPU_UINT64, FLOCKGPU_ERR_INVALID, "hash_aggregate: COUNT state must be UInt64");
          a = add_acc(ACC_ADD_I, s.col, CVT_NONE);
        } else {
          if (s.col >= 0) col_dtype(s.col, "COUNT");
          a = add_acc(ACC_COUNT, nulls_in(s.col) ? s.col : -1, CVT_NONE);  // COUNT(col) counts the non-NULL values
        }
        outs->push_back({partial_out ? base + "[count]" : base, FLOCKGPU_UINT64, "L", EMIT_RAW, a, 0});
        break;
      }
      case FLOCKGPU_AGG_SUM: {
        int dt = col_dtype(s.col, "SUM");
        int out_dt, op;
        if (dt == FLOCKGPU_FLOAT64) { out_dt = FLOCKGPU_FLOAT64; op = ACC_ADD_F; }
        else if (is_unsigned_dt(dt)) { out_dt = FLOCKGPU_UINT64; op = ACC_ADD_I; }
        else if (dt == FLOCKGPU_INT32 || dt == FLOCKGPU_INT64) { out_dt = FLOCKGPU_INT64; op = ACC_ADD_I; }
        else fail(FLOCKGPU_ERR_UNSUPPORTED, "hash_aggregate: SUM over %s", dtype_name(dt));
        int a = add_acc(op, s.col, CVT_NONE);
        outs->push_back({partial_out ? base + "[sum]" : base, out_dt, default_format(out_dt), EMIT_RAW, a, 0, valid_counter(s.col)});
        break;
      }
      case FLOCKGPU_AGG_MIN:
      case FLOCKGPU_AGG_MAX: {
        bool is_min = s.func == FLOCKGPU_AGG_MIN;
        int dt = col_dtype(s.col, is_min ? "MIN" : "MAX");
        int a = add_acc(minmax_op(dt, is_min, is_min ? "MIN" : "MAX"), s.col, CVT_NONE);
        const int kind = dt == FLOCKGPU_FLOAT64 ? EMIT_F64_ORDER : EMIT_RAW;  // the state columns of `partial` are decoded too
        outs->push_back({partial_out ? base + (is_min ? "[min]" : "[max]") : base, dt, in.cols[s.col].format, kind, a, 0, valid_counter(s.col)});
        break;
      }
      case FLOCKGPU_AGG_AVG: {
        int a_cnt, a_sum;
        if (from_states) {
          FG_CHECK(col_dtype(s.col, "AVG count state") == FLOCKGPU_UINT64 && col_dtype(s.col + 1, "AVG sum state") == FLOCKGPU_FLOAT64,
                   FLOCKGPU_ERR_INVALID, "hash_aggregate: AVG states must be (UInt64 count, Float64 sum)");
          a_cnt = add_acc(ACC_ADD_I, s.col, CVT_NONE);
          a_sum = add_acc(ACC_ADD_F, s.col + 1, CVT_NONE);
        } else {
          int dt = col_dtype(s.col, "AVG");
          FG_CHECK(dt != FLOCKGPU_UTF8 && dt != FLOCKGPU_TIMESTAMP && dt != FLOCKGPU_DATE32, FLOCKGPU_ERR_UNSUPPORTED, "hash_aggregate: AVG over %s", dtype_name(dt));
          a_cnt = add_acc(ACC_COUNT, nulls_in(s.col) ? s.col : -1, CVT_NONE);  // AVG divides by the number of non-NULL values
          a_sum = add_acc(ACC_ADD_F, s.col, dt == FLOCKGPU_FLOAT64 ? CVT_NONE : (is_unsigned_dt(dt) ? CVT_U2F : CVT_I2F));
        }
        if (partial_out) {
          outs->push_back({base + "[count]", FLOCKGPU_UINT64, "L", EMIT_RAW, a_cnt, 0});
          // like SUM's state: NULL for a group that saw no non-NULL value (a nullable argument only), so that the final
          // stage sees a nullable state column and knows the merged count can be 0
          outs->push_back({base + "[sum]", FLOCKGPU_FLOAT64, "g", EMIT_RAW, a_sum, 0, nulls_in(s.col) ? a_cnt : -1});
        } else {
          // no non-NULL value at all: AVG is NULL (0 / 0 otherwise); with states, the merged count tells
          const bool maybe_empty = from_states ? (nulls_in(s.col) || nulls_in(s.col + 1)) : nulls_in(s.col);
          outs->push_back({base, FLOCKGPU_FLOAT64, "g", EMIT_AVG, a_cnt, a_sum, maybe_empty ? a_cnt : -1});
        }
        break;
      }
      default:
        fail(FLOCKGPU_ERR_INVALID, "hash_aggregate: unknown aggregate function %d", s.func);
    }
  }
  for (int c = 0; c < plan.n_acc(); ++c) plan.ident[c] = acc_identity(plan.accs[c].op);
  return plan;
}

void fill_cols(const Table& t, ColRef* refs) {
  FG_CHECK(t.cols.size() <= size_t(MAX_IN_COLS), FLOCKGPU_ERR_UNSUPPORTED, "hash_aggregate: more than %d input columns", MAX_IN_COLS);
  fill_colrefs(t, refs);
}

int grid_for(const CtxPtr& ctx, int64_t items, int threads, int per_sm) {
  return int(std::max<int64_t>(1, std::min<int64_t>((items + threads - 1) / threads, int64_t(ctx->sm_count) * per_sm)));
}

// A CTA per `step` rows, but no more CTAs than fit on the device at once (the level-1 kernels loop over their range).
int resident_grid(const CtxPtr& ctx, const void* kernel, int threads, size_t smem, int64_t n, int64_t step) {
  return int(std::max<int64_t>(1, std::min<int64_t>(resident_ctas(ctx, kernel, threads, smem), (n + step - 1) / step)));
}

unsigned long long pow2_at_least(unsigned long long n) {
  unsigned long long c = 1024;
  while (c < n) c <<= 1;
  return c;
}

}  // namespace

static TablePtr hash_aggregate_impl(const CtxPtr& ctx, const TablePtr& in_ptr, int mode, const std::vector<int>& group_cols, const std::vector<AggSpec>& aggs,
                                    bool allow_dense);

// ---- how much would a DISTINCT over `group_cols` shrink the relation?  (plan layer: is a Partial stage worth it) -----
struct DistinctSampleArgs {
  int64_t n;
  RowKeys keys;
  ColRef cols[MAX_IN_COLS];
  unsigned long long* tags;  // [cap] zero = free
  unsigned long long cap;    // power of two
  unsigned long long* dups;
};

__global__ void __launch_bounds__(256) distinct_sample_kernel(const __grid_constant__ DistinctSampleArgs a) {
  unsigned mine = 0;
  for (int64_t row = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; row < a.n; row += int64_t(gridDim.x) * blockDim.x) {
    const unsigned long long h = hash_row(a.keys, a.cols, row) | 1ull;  // never the free marker
    unsigned long long slot = (h >> 7) & (a.cap - 1);
    for (int probe = 0; probe < 16; ++probe) {
      const unsigned long long old = atomicCAS(&a.tags[slot], 0ull, h);
      if (old == 0ull) break;
      if (old == h) {  // the same 64-bit hash: the same key for the purpose of an estimate
        ++mine;
        break;
      }
      slot = (slot + 1) & (a.cap - 1);
    }
  }
  mine = warp_sum(mine);
  if ((threadIdx.x & 31) == 0 && mine) atomicAdd(a.dups, (unsigned long long)mine);
}

// Fraction of the first min(n, 65536) rows that repeat a key seen earlier in that sample (0 = all different).
double distinct_sample_duplicates(const CtxPtr& ctx, const TablePtr& in_ptr, const std::vector<int>& group_cols) {
  in_ptr->dense();
  const Table& in = *in_ptr;
  const int64_t n = std::min<int64_t>(in.num_rows, 65536);
  if (n <= 0 || group_cols.empty() || group_cols.size() > size_t(MAX_KEY_COLS) || in.cols.size() > size_t(MAX_IN_COLS)) return 1.0;
  DistinctSampleArgs a{};
  a.n = n;
  a.keys.n = int(group_cols.size());
  for (size_t i = 0; i < group_cols.size(); ++i) a.keys.col[i] = group_cols[i];
  for (size_t i = 0; i < in.cols.size(); ++i) {
    a.cols[i].data = in.cols[i].values();
    a.cols[i].offsets = in.cols[i].offs();
    a.cols[i].dtype = in.cols[i].dtype;
  }
  a.cap = 1ull << 18;
  BufferPtr tags = alloc(ctx, size_t(a.cap) * 8);
  FG_CUDA(cudaMemsetAsync(tags->ptr, 0, size_t(a.cap) * 8, ctx->stream));
  a.tags = tags->as<unsigned long long>();
  a.dups = ctx->d_scalars + 10;
  FG_CUDA(cudaMemsetAsync(a.dups, 0, 8, ctx->stream));
  {
    LaunchTimer lt(ctx, "distinct_sample_kernel");
    distinct_sample_kernel<<<int((n + 255) / 256), 256, 0, ctx->stream>>>(a);
  }
  FG_CUDA(cudaGetLastError());
  count_launch(ctx);
  unsigned long long dups = 0;
  read_scalars(ctx, 10, 1, &dups);
  return double(dups) / double(n);
}

// ---- COUNT(*) / DISTINCT by one 4-byte key kept in its direct-address table --------------------------------------
namespace {

struct DenseCore {
  CtxPtr ctx;
  TablePtr input;  // kept for the generic path: taken when a key fell outside the table (overflow != 0)
  int mode = FLOCKGPU_AGG_SINGLE;
  std::vector<int> group_cols;
  std::vector<AggSpec> aggs;
  BufferPtr table, meta;
  unsigned long long cap = 0;  // capacity in slots; how many are in use is decided on the device (meta[DM_SLOTS])
  bool has_count = false;
  std::shared_ptr<PendingRows> overflow;
  TablePtr full;  // the materialised (key [, count]) rows, produced at most once
  bool valid() { return overflow->wait() == 0; }
  TablePtr materialise_full();
  // the visible columns `kinds` (0 = key, 1 = count) of the materialised relation under `names`
  TablePtr materialise_as(const std::vector<int>& kinds, const std::vector<std::string>& names, const std::string& metadata) {
    TablePtr f = materialise_full();
    auto t = std::make_shared<Table>();
    t->ctx = ctx;
    t->metadata = metadata;
    t->num_rows = f->num_rows;
    for (size_t i = 0; i < kinds.size(); ++i) {
      Column c = f->cols[kinds[i]];
      c.name = names[i];
      t->cols.push_back(std::move(c));
    }
    return t;
  }
};

struct DeferredAgg : DeferredTable {
  std::shared_ptr<DenseCore> core;
  std::vector<int> kinds;  // per visible column: 0 = the key, 1 = the count
  void materialise(const Table& self) override;
  TablePtr project(const Table& self, const std::vector<int>& src_cols, const std::vector<std::string>& names) override;
  TablePtr global_max(const Table& self, int col, const std::string& out_name) override;
  TablePtr select_equal(const Table& self, int key_col, const TablePtr& one_row, int one_key, bool self_is_left) override;
};

// MAX(count) of a DenseCore that nobody has asked the value of yet (one row, one UInt64 column).
struct DeferredMax : DeferredTable {
  std::shared_ptr<DenseCore> core;
  void materialise(const Table& self) override;
  TablePtr project(const Table& self, const std::vector<int>& src_cols, const std::vector<std::string>& names) override;
};

// The output of a selection over the table: its buffers are written, its row count is in flight, and whether the
// table was complete is only known once the overflow word has arrived.  Resolving waits for both; an incomplete
// table makes it run `fallback` (the same operator on materialised rows) instead.
struct DeferredChecked : DeferredTable {
  std::shared_ptr<DenseCore> core;
  std::shared_ptr<PendingRows> rows;
  std::function<TablePtr()> fallback;
  void materialise(const Table& self) override {
    const int64_t n = rows->wait();
    if (core->valid()) {
      self.num_rows = n;
      for (Column& c : self.cols) c.length = n;
      return;
    }
    TablePtr g = fallback();
    g->dense();
    self.num_rows = g->num_rows;
    for (size_t i = 0; i < self.cols.size(); ++i) {
      Column c = g->cols[i];
      c.name = self.cols[i].name;
      self.cols[i] = std::move(c);
    }
  }
};

DenseScanArgs dense_scan_args(const DenseCore& c) {
  DenseScanArgs a{};
  a.table = c.table->as<uint32_t>();
  a.n_slots = c.cap;
  a.meta = c.meta->as<unsigned long long>();
  return a;
}

template <bool SELECT>
void launch_dense_scan(const CtxPtr& ctx, DenseScanArgs& a, unsigned long long* out_count, unsigned long long* host_count) {
  const long long tiles = (long long)((a.n_slots + CP_THREADS * 64 - 1) / (CP_THREADS * 64));
  auto kernel = dense_scan_kernel<SELECT>;
  a.sc = prepare_compact(ctx, tiles, resident_ctas(ctx, reinterpret_cast<const void*>(kernel), CP_THREADS), out_count);
  a.sc.host_count = host_count;
  {
    LaunchTimer lt(ctx, SELECT ? "dense_select_kernel" : "dense_emit_kernel");
    launch_compact(ctx, kernel, a.sc, a);
  }
  FG_CUDA(cudaGetLastError());
  count_launch(ctx);
}

TablePtr DenseCore::materialise_full() {
  if (full) return full;
  if (!valid()) {
    // a key outside the sampled range: the table is incomplete, aggregate again the general way
    full = hash_aggregate_impl(ctx, input, mode, group_cols, aggs, false);
    return full;
  }
  const Table& in = *input;
  const Column& kc = in.cols[group_cols[0]];
  const int64_t max_groups = int64_t(std::min<unsigned long long>(cap, (unsigned long long)in.num_rows));
  auto t = std::make_shared<Table>();
  t->ctx = ctx;
  t->metadata = in.metadata;
  Column key;
  key.name = kc.name;
  key.dtype = kc.dtype;
  key.format = kc.format;
  key.nullable = kc.nullable;
  key.data = alloc(ctx, size_t(max_groups) * 4);
  DenseScanArgs a = dense_scan_args(*this);
  a.key_dst = key.data->as<uint32_t>();
  Column cnt;
  if (has_count) {
    cnt.dtype = FLOCKGPU_UINT64;
    cnt.format = "L";
    cnt.nullable = true;
    cnt.data = alloc(ctx, size_t(max_groups) * 8);
    a.count_dst = cnt.data->as<unsigned long long>();
  }
  launch_dense_scan<false>(ctx, a, ctx->d_scalars + 3, nullptr);
  unsigned long long n_groups = 0;
  read_scalars(ctx, 3, 1, &n_groups);
  FG_CHECK(int64_t(n_groups) <= max_groups, FLOCKGPU_ERR_CUDA, "hash_aggregate: corrupt group count %llu", n_groups);
  t->num_rows = int64_t(n_groups);
  key.length = t->num_rows;
  t->cols.push_back(std::move(key));
  if (has_count) {
    cnt.length = t->num_rows;
    cnt.name = "count";
    t->cols.push_back(std::move(cnt));
  }
  full = t;
  return full;
}

void DeferredAgg::materialise(const Table& self) {
  TablePtr f = core->materialise_full();
  self.num_rows = f->num_rows;
  for (size_t i = 0; i < kinds.size(); ++i) {
    Column c = f->cols[kinds[i]];
    c.name = self.cols[i].name;
    self.cols[i] = std::move(c);
  }
}

TablePtr deferred_table(const CtxPtr& ctx, const std::shared_ptr<DenseCore>& core, const std::vector<int>& kinds, const std::vector<std::string>& names,
                        const std::string& metadata) {
  auto t = std::make_shared<Table>();
  t->ctx = ctx;
  t->metadata = metadata;
  t->num_rows = -1;
  const Column& kc = core->input->cols[core->group_cols[0]];
  for (size_t i = 0; i < kinds.size(); ++i) {
    Column c;
    c.name = names[i];
    c.length = -1;
    if (kinds[i] == 0) {
      c.dtype = kc.dtype;
      c.format = kc.format;
      c.nullable = kc.nullable;
    } else {
      c.dtype = FLOCKGPU_UINT64;
      c.format = "L";
      c.nullable = true;
    }
    t->cols.push_back(std::move(c));
  }
  auto d = std::make_shared<DeferredAgg>();
  d->core = core;
  d->kinds = kinds;
  t->deferred = d;
  return t;
}

TablePtr DeferredAgg::project(const Table& self, const std::vector<int>& src_cols, const std::vector<std::string>& names) {
  std::vector<int> k;
  for (int c : src_cols) k.push_back(kinds[c]);
  return deferred_table(core->ctx, core, k, names, self.metadata);
}

TablePtr deferred_max_table(const std::shared_ptr<DenseCore>& core, const std::string& name, const std::string& metadata) {
  auto t = std::make_shared<Table>();
  t->ctx = core->ctx;
  t->metadata = metadata;
  t->num_rows = 1;
  Column c;
  c.name = name;
  c.dtype = FLOCKGPU_UINT64;
  c.format = "L";
  c.nullable = true;
  c.length = 1;
  t->cols.push_back(std::move(c));
  auto d = std::make_shared<DeferredMax>();
  d->core = core;
  t->deferred = d;
  return t;
}

TablePtr DeferredAgg::global_max(const Table& self, int col, const std::string& out_name) {
  if (col < 0 || col >= int(kinds.size()) || kinds[col] != 1 || !core->has_count) return nullptr;
  return deferred_max_table(core, out_name, self.metadata);  // nothing runs until somebody needs the number
}

void DeferredMax::materialise(const Table& self) {
  const CtxPtr& ctx = core->ctx;
  Column& c = self.cols[0];
  c.data = alloc(ctx, 8);
  // the scan kernel tracked the largest count it produced: MAX(count) is one word of its meta block
  FG_CUDA(cudaMemcpyAsync(c.data->ptr, core->meta->as<unsigned long long>() + DM_MAX, 8, cudaMemcpyDeviceToDevice, ctx->stream));
  if (!core->valid()) {
    // the table was incomplete: MAX over the materialised counts instead
    TablePtr f = core->materialise_full();
    TablePtr m = hash_aggregate_impl(ctx, f, FLOCKGPU_AGG_SINGLE, {}, {AggSpec{FLOCKGPU_AGG_MAX, 1, c.name}}, false);
    const std::string name = c.name;
    c = m->cols[0];
    c.name = name;
  }
  self.num_rows = 1;
  c.length = 1;
}

TablePtr DeferredMax::project(const Table& self, const std::vector<int>& src_cols, const std::vector<std::string>& names) {
  if (src_cols.size() != 1 || src_cols[0] != 0) return nullptr;
  return deferred_max_table(core, names[0], self.metadata);
}

TablePtr DeferredAgg::select_equal(const Table& self, int key_col, const TablePtr& one_ptr, int one_key, bool self_is_left) {
  if (key_col < 0 || key_col >= int(kinds.size()) || kinds[key_col] != 1 || !core->has_count) return nullptr;
  const Table& one_row = *one_ptr;
  // the other side: MAX(count) of this very table, not computed yet (fused below), or any resolved one-row relation
  auto* dmax = dynamic_cast<DeferredMax*>(one_row.deferred.get());
  const bool fused = dmax && dmax->core == core && one_key == 0;
  if (!fused) one_row.dense();
  if (one_row.num_rows != 1 || one_row.cols.size() > size_t(fused ? 4 : MAX_IN_COLS)) return nullptr;
  if (one_key < 0 || one_key >= int(one_row.cols.size()) || one_row.cols[one_key].dtype != FLOCKGPU_UINT64) return nullptr;
  if (!fused)
    for (const Column& c : one_row.cols)
      if (c.all_null || c.validity || c.dtype == FLOCKGPU_UTF8 || (c.width() != 4 && c.width() != 8) || c.chunks) return nullptr;
  const CtxPtr& ctx = core->ctx;
  const int64_t max_rows = int64_t(std::min<unsigned long long>(core->cap, (unsigned long long)core->input->num_rows));
  std::vector<Column> mine(kinds.size()), theirs(one_row.cols.size());
  BufferPtr key_buf, cnt_buf;
  for (size_t i = 0; i < kinds.size(); ++i) {
    Column& c = mine[i];
    c = self.cols[i];
    c.length = -1;
    BufferPtr& shared = kinds[i] == 0 ? key_buf : cnt_buf;  // the same logical column twice shares one buffer
    if (!shared) shared = alloc(ctx, size_t(max_rows) * (kinds[i] == 0 ? 4 : 8));
    c.data = shared;
  }
  for (size_t i = 0; i < one_row.cols.size(); ++i) {
    Column& c = theirs[i];
    c = one_row.cols[i];
    c.length = -1;
    c.data = alloc(ctx, size_t(max_rows) * c.width());
  }
  std::shared_ptr<PendingRows> pending = reserve_row_count(ctx);
  if (fused) {
    DenseArgmaxArgs a{};
    a.table = core->table->as<uint32_t>();
    a.meta = core->meta->as<unsigned long long>();
    const void* kernel = reinterpret_cast<const void*>(dense_argmax_kernel);
    const int grid = int(std::min<int64_t>(resident_ctas(ctx, kernel, 256), int64_t(ctx->sm_count) * 4));
    BufferPtr cta_counts = alloc(ctx, size_t(grid) * 4);
    a.cta_counts = cta_counts->as<unsigned>();
    a.key_dst = key_buf ? key_buf->as<uint32_t>() : nullptr;
    a.count_dst = cnt_buf ? cnt_buf->as<unsigned long long>() : nullptr;
    a.n_max_dst = int(theirs.size());
    for (size_t i = 0; i < theirs.size(); ++i) a.max_dst[i] = theirs[i].data->as<unsigned long long>();
    a.out_count = ctx->d_scalars + 4;
    a.host_count = pending->host_slot();
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(unsigned(grid));
    cfg.blockDim = dim3(256);
    cfg.stream = ctx->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;  // the CTAs wait for each other: co-residency must be guaranteed
    attr[0].val.cooperative = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    {
      LaunchTimer lt(ctx, "dense_argmax_kernel");
      FG_CUDA(cudaLaunchKernelEx(&cfg, dense_argmax_kernel, a));
    }
    count_launch(ctx);
    // `cta_counts` may be released now: the block allocator hands it out again in stream order only
  } else {
    DenseScanArgs a = dense_scan_args(*core);
    a.eq_value = static_cast<const unsigned long long*>(one_row.cols[one_key].values());
    if (key_buf) a.key_dst = key_buf->as<uint32_t>();
    if (cnt_buf) a.count_dst = cnt_buf->as<unsigned long long>();
    a.n_bcast = int(one_row.cols.size());
    for (size_t i = 0; i < one_row.cols.size(); ++i) {
      a.bcast_src[i] = one_row.cols[i].values();
      a.bcast_dst[i] = theirs[i].data->ptr;
      a.bcast_width[i] = theirs[i].width();
    }
    launch_dense_scan<true>(ctx, a, ctx->d_scalars + 4, pending->host_slot());
  }
  commit_row_count(pending);
  auto t = std::make_shared<Table>();
  t->ctx = ctx;
  t->metadata = self_is_left ? self.metadata : one_row.metadata;
  t->num_rows = -1;
  for (Column& c : (self_is_left ? mine : theirs)) t->cols.push_back(std::move(c));
  for (Column& c : (self_is_left ? theirs : mine)) t->cols.push_back(std::move(c));
  auto chk = std::make_shared<DeferredChecked>();
  chk->core = core;
  chk->rows = pending;
  std::vector<std::string> my_names;
  for (const Column& c : self.cols) my_names.push_back(c.name);
  std::shared_ptr<DenseCore> core_ref = core;
  std::vector<int> my_kinds = kinds;
  const std::string md = self.metadata;
  chk->fallback = [core_ref, my_kinds, my_names, md, one_ptr, key_col, one_key, self_is_left]() {
    TablePtr me = core_ref->materialise_as(my_kinds, my_names, md);
    one_ptr->dense();  // a DeferredMax over an incomplete table computes MAX over the materialised rows
    return self_is_left ? hash_join(core_ref->ctx, me, one_ptr, {key_col}, {one_key}) : hash_join(core_ref->ctx, one_ptr, me, {one_key}, {key_col});
  };
  t->deferred = chk;
  return t;
}

}  // namespace

TablePtr hash_aggregate(const CtxPtr& ctx, const TablePtr& in_ptr, int mode, const std::vector<int>& group_cols, const std::vector<AggSpec>& aggs) {
  // MAX over the count column of a group-by that still lives in its direct-address table (NEXMark q5: MAX(num))
  if (in_ptr->deferred && group_cols.empty() && aggs.size() == 1 && aggs[0].func == FLOCKGPU_AGG_MAX &&
      (mode == FLOCKGPU_AGG_PARTIAL || mode == FLOCKGPU_AGG_SINGLE)) {
    std::string name = aggs[0].name.empty() ? std::string("MAX") : aggs[0].name;
    if (mode == FLOCKGPU_AGG_PARTIAL) name += "[max]";
    std::shared_ptr<DeferredTable> d = in_ptr->deferred;
    if (TablePtr t = d->global_max(*in_ptr, aggs[0].col, name)) return t;
  }
  return hash_aggregate_impl(ctx, in_ptr, mode, group_cols, aggs, true);
}

// One pass over a 4-byte key column: the sliding shared-memory histogram adds straight into the direct-address count
// table `table` (capacity `cap` slots) whose first key a sample of the column decides ON THE DEVICE.  `meta`
// (DM_WORDS words, zeroed by the caller on the stream) receives the range, the rows that fell outside (DM_OVERFLOW)
// and, with has_count, the largest count (DM_MAX).
static void launch_dense_hist(const CtxPtr& ctx, const uint32_t* key_col, int64_t n, int has_count, uint32_t* table, unsigned long long* meta,
                              unsigned long long cap) {
  AggHist32Args h{};
  h.n_rows = n;
  h.key_col = key_col;
  h.has_count = has_count;
  h.slow_rows = ctx->d_scalars + 9;
  h.dense = table;
  h.dense_meta = meta;
  h.dense_cap = cap;  // (the kernels use meta[DM_SLOTS] <= cap)
  h.overflow = meta + DM_OVERFLOW;
  FG_CUDA(cudaMemsetAsync(h.slow_rows, 0, 8, ctx->stream));
  constexpr size_t h_bytes = size_t(H32_WINDOW) * 4;
  FG_CUDA(cudaFuncSetAttribute(agg_hist32_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(h_bytes)));
  const int grid = resident_grid(ctx, reinterpret_cast<const void*>(agg_hist32_kernel<true>), H32_THREADS, h_bytes, n, H32_STEP);
  {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(unsigned(grid));
    cfg.blockDim = dim3(H32_THREADS);
    cfg.dynamicSmemBytes = h_bytes;
    cfg.stream = ctx->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;  // the CTAs wait for each other's slice of the clearing
    attr[0].val.cooperative = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    LaunchTimer lt(ctx, "agg_hist32_dense_kernel");
    FG_CUDA(cudaLaunchKernelEx(&cfg, agg_hist32_kernel<true>, h));
  }
  FG_CUDA(cudaGetLastError());
  count_launch(ctx);
}

namespace {

std::shared_ptr<Table> result_table(const CtxPtr& ctx, const Table& in) {
  auto t = std::make_shared<Table>();
  t->ctx = ctx;
  t->metadata = in.metadata;
  return t;
}

Column make_out_col(const CtxPtr& ctx, const OutPlan& p, int64_t rows) {
  Column c;
  c.name = p.name;
  c.dtype = p.dtype;
  c.format = p.format;
  c.nullable = true;  // aggregate outputs are nullable in the reference schema (aggregate.json)
  c.length = rows;
  c.data = alloc(ctx, size_t(rows) * dtype_width(p.dtype));
  return c;
}

// Column `g` of the input as a group column of the output (no data yet).
Column key_out_col(const Table& in, int g, int64_t rows) {
  Column c;
  c.name = in.cols[g].name;
  c.dtype = in.cols[g].dtype;
  c.format = in.cols[g].format;
  c.nullable = in.cols[g].nullable;
  c.length = rows;
  return c;
}

void fill_emit(const CtxPtr& ctx, const std::vector<OutPlan>& outs, EmitDesc* emit, int32_t* n_emit, std::vector<Column>& cols) {
  FG_CHECK(outs.size() <= size_t(2 * MAX_ACC), FLOCKGPU_ERR_UNSUPPORTED, "hash_aggregate: too many output columns");
  *n_emit = int(outs.size());
  for (size_t i = 0; i < outs.size(); ++i) {
    emit[i] = EmitDesc{outs[i].kind, outs[i].a0, outs[i].a1, outs[i].dtype, cols[i].data->ptr, nullptr, 0, 0};
    if (outs[i].valid_acc >= 0) {
      cols[i].validity = alloc(ctx, size_t(std::max<int64_t>(cols[i].length, 1)));
      emit[i].valid_dst = cols[i].validity->as<uint8_t>();
      emit[i].valid_acc = outs[i].valid_acc;
    }
  }
}

// Groups stay on the rank their rows were routed to: the input's routing survives when its columns are group columns.
void keep_routing(const Table& in, const std::vector<int>& group_cols, Table* out) {
  if (in.partitioned_on.empty()) return;
  for (const std::string& p : in.partitioned_on) {
    bool found = false;
    for (int g : group_cols) found |= in.cols[g].name == p;
    if (!found) return;
  }
  out->partitioned_on = in.partitioned_on;
  out->partition_world = in.partition_world;
}

// DISTINCT over rows that are all different: the result IS the input's group columns (zero-copy) -- any order is a
// valid group order.
TablePtr input_groups(const CtxPtr& ctx, const Table& in, const std::vector<int>& group_cols) {
  auto out = result_table(ctx, in);
  out->num_rows = in.num_rows;
  for (int g : group_cols) out->cols.push_back(in.cols[g]);
  keep_routing(in, group_cols, out.get());
  return out;
}

// Up to two fixed-width group columns of at most 8 bytes together (two: exactly 8) become one 64-bit key.  A NULL key
// is a group of its own, so a nullable column goes to the row-representative table, which compares validity too.
bool pack_keys(const Table& in, const std::vector<int>& group_cols, KeyPack* kp) {
  if (group_cols.size() > 2) return false;
  int key_bytes = 0;
  for (int g : group_cols) {
    if (in.cols[g].width() == 0 || in.cols[g].validity) return false;
    key_bytes += in.cols[g].width();
  }
  if (key_bytes > 8 || (group_cols.size() == 2 && key_bytes != 8)) return false;
  kp->n = int(group_cols.size());
  for (int i = 0; i < kp->n; ++i) {
    kp->col[i] = group_cols[i];
    kp->width[i] = in.cols[group_cols[i]].width();
  }
  return true;
}

// Level-1 output: (key, accumulators) entries of CTA-local pre-aggregation, or nothing (keys == NULL) when level 2
// takes the input rows themselves.
struct Partials {
  BufferPtr keys, acc;
  int64_t count = 0;
  bool part32 = false;  // uint32 keys / counts (the 4-byte-key kernels)
  unsigned long long key_min = 1, key_max = 0;
};

// A level-2 table ready to be emitted: the emit kernel's arguments except the outputs, and the buffers behind them.
struct GroupTable {
  AggEmitArgs ea{};
  int mode = 0;  // agg_emit_kernel MODE: 0 hashed packed keys, 1 dense, 2 row representatives
  std::vector<BufferPtr> buffers;
};

}  // namespace

// ---- no group columns: one row
static TablePtr aggregate_ungrouped(const CtxPtr& ctx, const Table& in, int mode, const std::vector<AggSpec>& aggs, const AggPlan& p) {
  const int64_t n = in.num_rows;
  auto out = result_table(ctx, in);
  out->num_rows = 1;
  std::vector<Column> cols;
  for (const OutPlan& o : p.outs) cols.push_back(make_out_col(ctx, o, 1));
  BufferPtr state = alloc(ctx, sizeof(unsigned long long) * MAX_ACC);
  FG_CUDA(cudaMemcpyAsync(state->ptr, p.ident, sizeof p.ident, cudaMemcpyHostToDevice, ctx->stream));
  if (n > 0) {
    AggGlobalArgs ga{};
    ga.n_rows = n;
    ga.n_acc = p.n_acc();
    for (int c = 0; c < p.n_acc(); ++c) ga.acc[c] = p.accs[c];
    fill_cols(in, ga.cols);
    ga.state = state->as<unsigned long long>();
    {
      LaunchTimer lt(ctx, "agg_global_kernel");
      agg_global_kernel<<<grid_for(ctx, n, 256, 8), 256, 0, ctx->stream>>>(ga);
    }
    FG_CUDA(cudaGetLastError());
    count_launch(ctx);
  }
  AggEmitOneArgs ea{};
  ea.state = state->as<unsigned long long>();
  fill_emit(ctx, p.outs, ea.emit, &ea.n_emit, cols);
  {
    LaunchTimer lt(ctx, "agg_emit_one_kernel");
    agg_emit_one_kernel<<<1, 32, 0, ctx->stream>>>(ea);
  }
  FG_CUDA(cudaGetLastError());
  count_launch(ctx);
  // aggregates other than COUNT over zero rows are NULL (SURVEY.md Appendix C.7); the same holds for a Final merge
  // that received no state row at all (every producer's partition was empty): COUNT merges to 0, the rest is NULL
  if (n == 0) {
    size_t o = 0;
    for (const AggSpec& s : aggs) {
      const size_t width = (s.func == FLOCKGPU_AGG_AVG && mode == FLOCKGPU_AGG_PARTIAL) ? 2 : 1;
      for (size_t k = 0; k < width; ++k, ++o) {
        const bool is_count_state = s.func == FLOCKGPU_AGG_COUNT || (s.func == FLOCKGPU_AGG_AVG && mode == FLOCKGPU_AGG_PARTIAL && k == 0);
        if (!is_count_state) cols[o].all_null = true;
      }
    }
  }
  out->cols = std::move(cols);
  // keep `state` alive until the kernels have run: stream-ordered free does that
  return out;
}

// ---- group columns, empty input: empty output
static TablePtr empty_grouped(const CtxPtr& ctx, const Table& in, const std::vector<int>& group_cols, const AggPlan& p) {
  auto out = result_table(ctx, in);
  out->num_rows = 0;
  for (int g : group_cols) {
    Column c = key_out_col(in, g, 0);
    c.data = alloc(ctx, 0);
    if (c.dtype == FLOCKGPU_UTF8) {
      c.offsets = alloc(ctx, 4);
      FG_CUDA(cudaMemsetAsync(c.offsets->ptr, 0, 4, ctx->stream));
    }
    out->cols.push_back(std::move(c));
  }
  for (const OutPlan& o : p.outs) out->cols.push_back(make_out_col(ctx, o, 0));
  return out;
}

// ---- COUNT(*) / DISTINCT by one 4-byte key in one pass: the sliding shared-memory histogram adds straight into a
// direct-address table whose first key a sample of the column decides ON THE DEVICE (no host round trip); the result
// stays in table form (DeferredTable) until somebody needs rows.  A key outside the table counts as overflow, and the
// first consumer that finds overflow != 0 aggregates again the general way.
static TablePtr count_table(const CtxPtr& ctx, const TablePtr& in_ptr, int mode, const std::vector<int>& group_cols, const std::vector<AggSpec>& aggs,
                            const AggPlan& p) {
  const Table& in = *in_ptr;
  const int64_t n = in.num_rows;
  const Column& key = in.cols[group_cols[0]];
  auto core = std::make_shared<DenseCore>();
  core->ctx = ctx;
  core->input = in_ptr;
  core->mode = mode;
  core->group_cols = group_cols;
  core->aggs = aggs;
  core->has_count = p.n_acc() == 1;
  // capacity: a direct-address table pays off while it is not much larger than the input; only the slots the
  // device decides to use are ever cleared or scanned, so a generous capacity costs address space, not time
  core->cap = (std::min<unsigned long long>(std::max<unsigned long long>(2ull * (unsigned long long)n, 1ull << 16), 1ull << 26) + 3) & ~3ull;
  core->table = alloc(ctx, size_t(core->cap) * 4);
  core->meta = alloc(ctx, DM_WORDS * 8);
  FG_CUDA(cudaMemsetAsync(core->meta->ptr, 0, DM_WORDS * 8, ctx->stream));
  launch_dense_hist(ctx, static_cast<const uint32_t*>(key.values()), n, p.n_acc(), core->table->as<uint32_t>(), core->meta->as<unsigned long long>(),
                    core->cap);
  core->overflow = reserve_row_count(ctx);
  FG_CUDA(cudaMemcpyAsync(core->overflow->host_slot(), core->meta->as<unsigned long long>() + DM_OVERFLOW, 8, cudaMemcpyDeviceToHost, ctx->stream));
  commit_row_count(core->overflow);
  std::vector<int> kinds{0};
  std::vector<std::string> names{key.name};
  if (core->has_count) {
    kinds.push_back(1);
    names.push_back(p.outs[0].name);
  }
  return deferred_table(ctx, core, kinds, names, in.metadata);
}

// ---- level 1 (large inputs of raw rows): every CTA pre-aggregates its row range in shared memory into partials.  One
// 4-byte key with COUNT(*) or no aggregate (`count32`) first tries the sliding histogram without a table; when more
// than an eighth of the rows miss its window, the shared-memory hash table starts over.
static Partials level1_partials(const CtxPtr& ctx, const Table& in, const KeyPack& kp, const AggPlan& p, bool count32) {
  const int64_t n = in.num_rows;
  const int n_acc = p.n_acc();
  Partials l1;
  l1.keys = alloc(ctx, size_t(n) * 8);
  l1.acc = alloc(ctx, size_t(n) * 8 * std::max(n_acc, 1));
  l1.part32 = count32;
  unsigned long long* cursor = ctx->d_scalars + 2;      // partial entries written
  unsigned long long* key_minmax = ctx->d_scalars + 6;  // [0] = min, [1] = max key seen
  auto reset = [&]() {
    FG_CUDA(cudaMemsetAsync(cursor, 0, 8, ctx->stream));
    FG_CUDA(cudaMemsetAsync(key_minmax, 0xff, 8, ctx->stream));   // min = ~0
    FG_CUDA(cudaMemsetAsync(key_minmax + 1, 0, 8, ctx->stream));  // max = 0
  };
  reset();
  const uint32_t* key_col = static_cast<const uint32_t*>(in.cols[kp.col[0]].values());
  bool hist_ok = false;
  if (count32) {
    AggHist32Args h{};
    h.n_rows = n;
    h.key_col = key_col;
    h.has_count = n_acc;
    h.part_keys = l1.keys->as<uint32_t>();
    h.part_acc = l1.acc->as<uint32_t>();
    h.part_capacity = n;
    h.part_cursor = cursor;
    h.key_minmax = key_minmax;
    h.slow_rows = ctx->d_scalars + 9;
    FG_CUDA(cudaMemsetAsync(h.slow_rows, 0, 8, ctx->stream));
    constexpr size_t h_bytes = size_t(H32_WINDOW) * 4;
    FG_CUDA(cudaFuncSetAttribute(agg_hist32_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(h_bytes)));
    const int grid = resident_grid(ctx, reinterpret_cast<const void*>(agg_hist32_kernel<false>), H32_THREADS, h_bytes, n, H32_STEP);
    {
      LaunchTimer lt(ctx, "agg_hist32_kernel");
      agg_hist32_kernel<false><<<grid, H32_THREADS, h_bytes, ctx->stream>>>(h);
    }
    FG_CUDA(cudaGetLastError());
    count_launch(ctx);
    unsigned long long slow = 0;
    read_scalars(ctx, 9, 1, &slow);
    hist_ok = slow * 8 <= (unsigned long long)n;
    if (!hist_ok) reset();
  }
  if (count32 && !hist_ok) {
    AggLocal32Args l32{};
    l32.n_rows = n;
    l32.key_col = key_col;
    l32.has_count = n_acc;
    l32.part_keys = l1.keys->as<uint32_t>();
    l32.part_acc = l1.acc->as<uint32_t>();
    l32.part_capacity = n;
    l32.part_cursor = cursor;
    l32.key_minmax = key_minmax;
    constexpr size_t a32_bytes = size_t(A32_SLOTS) * 8;
    FG_CUDA(cudaFuncSetAttribute(agg_local32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(a32_bytes)));
    const int grid = resident_grid(ctx, reinterpret_cast<const void*>(agg_local32_kernel), A32_THREADS, a32_bytes, n, A32_STEP);
    {
      LaunchTimer lt(ctx, "agg_local32_kernel");
      agg_local32_kernel<<<grid, A32_THREADS, a32_bytes, ctx->stream>>>(l32);
    }
    FG_CUDA(cudaGetLastError());
    count_launch(ctx);
  } else if (!count32) {
    AggLocalArgs la{};
    la.n_rows = n;
    la.keys = kp;
    la.n_acc = n_acc;
    for (int c = 0; c < n_acc; ++c) la.acc[c] = p.accs[c];
    fill_cols(in, la.cols);
    la.part_keys = l1.keys->as<unsigned long long>();
    la.part_acc = l1.acc->as<unsigned long long>();
    la.part_capacity = n;
    la.part_cursor = cursor;
    la.key_minmax = key_minmax;
    const size_t local_smem = size_t(AL_SLOTS) * 8 * (1 + n_acc);
    FG_CUDA(cudaFuncSetAttribute(agg_local_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(local_smem)));
    const int grid = resident_grid(ctx, reinterpret_cast<const void*>(agg_local_kernel), AL_THREADS, local_smem, n, AL_THREADS * AL_UNROLL);
    {
      LaunchTimer lt(ctx, "agg_local_kernel");
      agg_local_kernel<<<grid, AL_THREADS, local_smem, ctx->stream>>>(la);
    }
    FG_CUDA(cudaGetLastError());
    count_launch(ctx);
  }
  unsigned long long sc6[6] = {};
  read_scalars(ctx, 2, 6, sc6);
  FG_CHECK(int64_t(sc6[0]) <= n, FLOCKGPU_ERR_CUDA, "hash_aggregate: corrupt partial count");
  l1.count = int64_t(sc6[0]);
  l1.key_min = sc6[4];
  l1.key_max = sc6[5];
  return l1;
}

// ---- level 2 over packed keys: the partials (or the raw rows, or the partial STATES of a Final*) merge into one global
// table.  Direct-address when the keys of a single column fill their range well, open addressing otherwise.
static GroupTable packed_table(const CtxPtr& ctx, const Table& in, const KeyPack& kp, const AggPlan& p, const Partials& l1) {
  const int64_t n = in.num_rows;
  const int n_acc = p.n_acc();
  const bool from_partials = l1.keys != nullptr;
  const int64_t n_entries = from_partials ? l1.count : n;
  bool dense = false;
  if (from_partials && kp.n == 1 && l1.key_max >= l1.key_min && l1.key_max != EMPTY_KEY) {
    const unsigned long long range = l1.key_max - l1.key_min + 1;
    dense = range <= std::max<unsigned long long>(4ull * (unsigned long long)n_entries, 1ull << 16) && range < (1ull << 31);
  }
  const unsigned long long cap = dense ? l1.key_max - l1.key_min + 1 : pow2_at_least(2ull * (unsigned long long)n_entries);
  GroupTable t;
  t.mode = dense ? 1 : 0;
  t.ea.n_slots = cap + 1;
  t.ea.acc_stride = (t.ea.n_slots + 3) & ~3ull;  // the emit kernel reads whole groups of four slots
  const unsigned long long stride = t.ea.acc_stride;
  BufferPtr tkeys, tpresent;
  if (dense) {
    tpresent = alloc(ctx, size_t(stride));
    FG_CUDA(cudaMemsetAsync(tpresent->ptr, 0, size_t(stride), ctx->stream));
  } else {
    tkeys = alloc(ctx, size_t(stride) * 8);
  }
  BufferPtr tacc = alloc(ctx, size_t(stride) * 8 * std::max(n_acc, 1));
  t.buffers = {tkeys, tpresent, tacc};
  AggTable tab{dense ? nullptr : tkeys->as<unsigned long long>(), tacc->as<unsigned long long>(), cap,
               dense ? tpresent->as<unsigned char>() : nullptr, l1.key_min, stride};
  const unsigned long long* ident = p.ident;
  {
    LaunchTimer lt(ctx, "agg_init_kernel");
    agg_init_kernel<<<grid_for(ctx, int64_t(t.ea.n_slots), 256, 8), 256, 0, ctx->stream>>>(tab, n_acc, ident[0], ident[1], ident[2], ident[3], ident[4],
                                                                                         ident[5], ident[6], ident[7]);
  }
  FG_CUDA(cudaGetLastError());
  count_launch(ctx);
  AggInsertArgs ia{};
  ia.n = n_entries;
  ia.keys = kp;
  ia.n_acc = n_acc;
  ia.from_partials = from_partials ? 1 : 0;
  for (int c = 0; c < n_acc; ++c) ia.acc[c] = p.accs[c];
  fill_cols(in, ia.cols);
  ia.part32 = l1.part32 ? 1 : 0;
  ia.part_keys = from_partials ? l1.keys->as<unsigned long long>() : nullptr;
  ia.part_acc = from_partials ? l1.acc->as<unsigned long long>() : nullptr;
  ia.part_capacity = n;
  ia.table = tab;
  if (n_entries > 0) {
    {
      LaunchTimer lt(ctx, "agg_insert_kernel");
      agg_insert_kernel<<<grid_for(ctx, n_entries, 256, 8), 256, 0, ctx->stream>>>(ia);
    }
    FG_CUDA(cudaGetLastError());
    count_launch(ctx);
  }
  t.ea.keys = tab.keys;
  t.ea.present = tab.present;
  t.ea.dense_base = tab.dense_base;
  t.ea.acc = tab.acc;
  t.ea.n_key_out = kp.n;
  t.ea.key_width[0] = kp.width[0];
  t.ea.key_width[1] = kp.width[1];
  return t;
}

// ---- Utf8, wide or nullable keys: a table of representative input rows (key equality against the input columns).
// Returns the result itself when a DISTINCT finds every row different, else NULL with `t` ready to be emitted.
// agg_rows_local_kernel is taken when at least this share of a 64 Ki-row sample repeats an earlier key of the sample
constexpr double ROWS_LOCAL_MIN_DUPLICATES = 0.5;

static TablePtr row_table(const CtxPtr& ctx, const TablePtr& in_ptr, const std::vector<int>& group_cols, const AggPlan& p, GroupTable* t) {
  const Table& in = *in_ptr;
  FG_CHECK(group_cols.size() <= size_t(MAX_KEY_COLS), FLOCKGPU_ERR_UNSUPPORTED, "hash_aggregate: more than %d group columns", MAX_KEY_COLS);
  const int64_t n = in.num_rows;
  const int n_acc = p.n_acc();
  // ---- DISTINCT whose key holds a 4-byte column: if THAT column alone never repeats, no key does, and the answer is
  // the input.  One streaming count of the column into a direct-address table (the q5 kernel: MAX(count) == 1 and no
  // row outside the table) settles it for a quarter of what hashing and comparing the Utf8 keys costs (q8's persons
  // by (p_id, name): 2.5 M rows); when the column does repeat, the general path
  // below runs as before.
  // (not behind an exchange over more than two ranks: a rank then holds every W-th key of the whole range, a
  // 4096-row step spans more ids than the sliding window and the table W x the rows -- at N = 8 the probe
  // overflowed and the row table ran anyway)
  if (n_acc == 0 && n >= (int64_t(1) << 18) && n < (int64_t(1) << 32) && in.partition_world <= 2) {
    int probe_col = -1;
    for (int g : group_cols)
      if (in.cols[g].dtype != FLOCKGPU_UTF8 && in.cols[g].width() == 4 && !in.cols[g].validity) {
        probe_col = g;
        break;
      }
    if (probe_col >= 0) {
      constexpr int kProbeMeta = 64;  // d_scalars[64 .. 64 + DM_WORDS)
      // capacity 4 n: behind a two-rank exchange a rank holds every second key of the WHOLE range (2 n ids plus the
      // sampled margins); at 2 n the probe overflowed on one rank of two and that rank then reached every
      // exchange late.  Only the slots the device decides to use are cleared and scanned.
      const unsigned long long pcap = (std::min<unsigned long long>(std::max<unsigned long long>(4ull * (unsigned long long)n, 1ull << 16), 1ull << 26) + 3) & ~3ull;
      BufferPtr ptable = alloc(ctx, size_t(pcap) * 4);
      unsigned long long* pmeta = ctx->d_scalars + kProbeMeta;
      FG_CUDA(cudaMemsetAsync(pmeta, 0, DM_WORDS * 8, ctx->stream));
      launch_dense_hist(ctx, static_cast<const uint32_t*>(in.cols[probe_col].values()), n, 1, ptable->as<uint32_t>(), pmeta, pcap);
      unsigned long long m[DM_WORDS] = {};
      read_scalars(ctx, kProbeMeta, DM_WORDS, m);
      if (m[DM_OVERFLOW] == 0 && m[DM_MAX] == 1) return input_groups(ctx, in, group_cols);
    }
  }
  const unsigned long long cap = std::max<unsigned long long>(4, pow2_at_least(2ull * (unsigned long long)n));
  BufferPtr towner = alloc(ctx, size_t(cap) * 4);
  BufferPtr tacc = alloc(ctx, size_t(cap) * 8 * std::max(n_acc, 1));
  const unsigned long long* ident = p.ident;
  {
    LaunchTimer lt(ctx, "agg_rows_init_kernel");
    agg_rows_init_kernel<<<grid_for(ctx, int64_t(cap), 256, 8), 256, 0, ctx->stream>>>(towner->as<unsigned>(), tacc->as<unsigned long long>(), cap, n_acc,
                                                                                     ident[0], ident[1], ident[2], ident[3], ident[4], ident[5],
                                                                                     ident[6], ident[7]);
  }
  FG_CUDA(cudaGetLastError());
  count_launch(ctx);
  AggRowsArgs ra{};
  ra.n_rows = n;
  ra.keys.n = int(group_cols.size());
  for (size_t i = 0; i < group_cols.size(); ++i) ra.keys.col[i] = group_cols[i];
  ra.n_acc = n_acc;
  for (int c = 0; c < n_acc; ++c) ra.acc[c] = p.accs[c];
  fill_cols(in, ra.cols);
  ra.owner = towner->as<unsigned>();
  ra.tacc = tacc->as<unsigned long long>();
  ra.cap = cap;
  ra.n_groups = ctx->d_scalars + 7;
  FG_CUDA(cudaMemsetAsync(ra.n_groups, 0, 8, ctx->stream));
  // Mostly repeated keys over a large input (TPC-H q1, q5 and q12 at scale): pre-aggregate per CTA first.  The cut-off
  // (DESIGN.md K6r) keeps inputs whose keys are mostly distinct, and small ones, on the direct insert.
  if (n >= (int64_t(1) << 18) && n < int64_t(EMPTY_OWNER) && distinct_sample_duplicates(ctx, in_ptr, group_cols) >= ROWS_LOCAL_MIN_DUPLICATES) {
    const size_t smem = size_t(RL_SLOTS) * 8 * (1 + n_acc);
    FG_CUDA(cudaFuncSetAttribute(agg_rows_local_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    const int grid = resident_grid(ctx, reinterpret_cast<const void*>(agg_rows_local_kernel), RL_THREADS, smem, n, RL_THREADS * 16);
    const int64_t per_cta = ((n + grid - 1) / grid + RL_THREADS - 1) / RL_THREADS * RL_THREADS;
    LaunchTimer lt(ctx, "agg_rows_local_kernel");
    agg_rows_local_kernel<<<grid, RL_THREADS, smem, ctx->stream>>>(ra, per_cta);
  } else {
    LaunchTimer lt(ctx, "agg_insert_rows_kernel");
    agg_insert_rows_kernel<<<grid_for(ctx, n, 256, 8), 256, 0, ctx->stream>>>(ra);
  }
  FG_CUDA(cudaGetLastError());
  count_launch(ctx);
  if (n_acc == 0) {
    // DISTINCT over rows that are all different (q8: persons by (p_id, name)): nothing needs to be emitted or gathered
    // (the take() of the Utf8 names cost more than building the table)
    unsigned long long distinct = 0;
    read_scalars(ctx, 7, 1, &distinct);
    if (int64_t(distinct) == n) return input_groups(ctx, in, group_cols);
  }
  BufferPtr rep_rows = alloc(ctx, size_t(std::min<unsigned long long>(cap, (unsigned long long)n)) * 4);
  t->mode = 2;
  t->ea.n_slots = cap;
  t->ea.acc_stride = cap;
  t->ea.owner = towner->as<unsigned>();
  t->ea.acc = tacc->as<unsigned long long>();
  t->ea.rep_rows = rep_rows->as<unsigned>();
  t->buffers = {towner, tacc, rep_rows};
  return nullptr;
}

// ---- emit: stable compaction of the occupied slots into the output columns (worst case: every input row is its own
// group).  Row representatives become key columns through a gather.
static TablePtr emit_groups(const CtxPtr& ctx, const Table& in, const std::vector<int>& group_cols, const AggPlan& p, GroupTable& t) {
  const int64_t max_groups = in.num_rows;
  AggEmitArgs& ea = t.ea;
  std::vector<Column> key_cols, val_cols;
  if (t.mode != 2) {
    for (size_t i = 0; i < group_cols.size(); ++i) {
      Column c = key_out_col(in, group_cols[i], 0);
      c.data = alloc(ctx, size_t(max_groups) * c.width());
      ea.key_dst[i] = c.data->ptr;
      key_cols.push_back(std::move(c));
    }
  }
  for (const OutPlan& o : p.outs) val_cols.push_back(make_out_col(ctx, o, max_groups));
  fill_emit(ctx, p.outs, ea.emit, &ea.n_emit, val_cols);
  {
    const bool big = ea.n_slots > (unsigned long long)ctx->sm_count * 4 * CP_THREADS * 16;
    const int items = big ? 64 : 16;
    const long long tiles = (long long)((ea.n_slots + CP_THREADS * items - 1) / (CP_THREADS * items));
    auto launch = [&](auto kernel) {
      ea.sc = prepare_compact(ctx, tiles, resident_ctas(ctx, reinterpret_cast<const void*>(kernel), CP_THREADS), ctx->d_scalars + 3);
      LaunchTimer lt(ctx, t.mode == 1 ? "agg_emit_dense_kernel" : "agg_emit_kernel");  // the profile tells the direct-address table apart
      launch_compact(ctx, kernel, ea.sc, ea);
    };
    if (t.mode == 0) big ? launch(agg_emit_kernel<0, 64>) : launch(agg_emit_kernel<0, 16>);
    else if (t.mode == 1) big ? launch(agg_emit_kernel<1, 64>) : launch(agg_emit_kernel<1, 16>);
    else big ? launch(agg_emit_kernel<2, 64>) : launch(agg_emit_kernel<2, 16>);
    FG_CUDA(cudaGetLastError());
    count_launch(ctx);
  }
  unsigned long long n_groups = 0;
  read_scalars(ctx, 3, 1, &n_groups);
  FG_CHECK(int64_t(n_groups) <= max_groups, FLOCKGPU_ERR_CUDA, "hash_aggregate: corrupt group count %llu", n_groups);
  auto out = result_table(ctx, in);
  out->num_rows = int64_t(n_groups);
  if (t.mode != 2) {
    for (Column& c : key_cols) {
      c.length = int64_t(n_groups);
      out->cols.push_back(std::move(c));
    }
  } else {
    std::vector<const Column*> src;
    for (int g : group_cols) src.push_back(&in.cols[g]);
    for (Column& c : gather_columns(ctx, src, ea.rep_rows, int64_t(n_groups))) out->cols.push_back(std::move(c));
  }
  for (Column& c : val_cols) {
    c.length = int64_t(n_groups);
    out->cols.push_back(std::move(c));
  }
  keep_routing(in, group_cols, out.get());
  return out;
}

// ---- a SINGLE aggregate by one 4-byte key with MIN / MAX whose level-2 table is direct-address stays in that table
// (NEXMark q9: each auction's MAX(price), which the outer join on (auction, price) reads back per bid).  The join asks
// select_group_match for one selection over its other side; every other consumer materialises exactly the rows the
// emit path writes.
namespace {

struct GroupsCore {
  CtxPtr ctx;
  TablePtr input;
  std::vector<int> group_cols;
  std::vector<AggSpec> aggs;
  AggPlan plan;
  GroupTable table;
  TablePtr full;  // the emitted rows, produced at most once
  TablePtr materialise_full() {
    if (!full) full = emit_groups(ctx, *input, group_cols, plan, table);
    return full;
  }
};

struct DeferredGroups : DeferredTable {
  std::shared_ptr<GroupsCore> core;
  std::vector<int> kinds;  // per visible column: its column of the emitted relation (0 = the key, 1 + j = output j)
  void materialise(const Table& self) override {
    TablePtr f = core->materialise_full();
    self.num_rows = f->num_rows;
    for (size_t i = 0; i < kinds.size(); ++i) {
      Column c = f->cols[kinds[i]];
      c.name = self.cols[i].name;
      self.cols[i] = std::move(c);
    }
  }
  TablePtr project(const Table& self, const std::vector<int>& src_cols, const std::vector<std::string>& names) override;
  TablePtr select_group_match(const Table& self, const int (&self_keys)[2], const TablePtr& other, const int (&other_keys)[2],
                              bool self_is_left) override;
};

TablePtr groups_table(const std::shared_ptr<GroupsCore>& core, const std::vector<int>& kinds, const std::vector<std::string>& names,
                      const std::string& metadata) {
  auto t = std::make_shared<Table>();
  t->ctx = core->ctx;
  t->metadata = metadata;
  t->num_rows = -1;
  for (size_t i = 0; i < kinds.size(); ++i) {
    Column c;
    if (kinds[i] == 0) {
      c = key_out_col(*core->input, core->group_cols[0], -1);
    } else {
      const OutPlan& o = core->plan.outs[kinds[i] - 1];
      c.dtype = o.dtype;
      c.format = o.format;
      c.nullable = true;
      c.length = -1;
    }
    c.name = names[i];
    t->cols.push_back(std::move(c));
  }
  auto d = std::make_shared<DeferredGroups>();
  d->core = core;
  d->kinds = kinds;
  t->deferred = d;
  return t;
}

TablePtr DeferredGroups::project(const Table& self, const std::vector<int>& src_cols, const std::vector<std::string>& names) {
  std::vector<int> k;
  for (int c : src_cols) k.push_back(kinds[c]);
  return groups_table(core, k, names, self.metadata);
}

TablePtr DeferredGroups::select_group_match(const Table& self, const int (&self_keys)[2], const TablePtr& other_ptr, const int (&other_keys)[2],
                                            bool self_is_left) {
  for (int i = 0; i < 2; ++i)
    if (self_keys[i] < 0 || self_keys[i] >= int(kinds.size())) return nullptr;
  // which of the two key pairs is (group column, other column) and which (aggregate, other column)
  const int kp = kinds[self_keys[0]] == 0 ? 0 : 1, vp = 1 - kp;
  if (kinds[self_keys[kp]] != 0 || kinds[self_keys[vp]] == 0) return nullptr;
  const int out_col = kinds[self_keys[vp]];
  const OutPlan& o = core->plan.outs[out_col - 1];
  const int func = core->aggs[out_col - 1].func;
  if ((func != FLOCKGPU_AGG_MIN && func != FLOCKGPU_AGG_MAX) || o.kind != EMIT_RAW || o.dtype == FLOCKGPU_FLOAT64) return nullptr;
  // every column of self must be one of the two: both are the survivors' own values
  for (int k : kinds)
    if (k != 0 && k != out_col) return nullptr;
  const Table& other = *other_ptr;
  other.dense();
  const int ok = other_keys[kp], ov = other_keys[vp];
  if (ok < 0 || ok >= int(other.cols.size()) || ov < 0 || ov >= int(other.cols.size())) return nullptr;
  // hash_join has already checked both key pairs with join_key_types_match (Timestamp unit and zone included) before
  // it asked for this selection, so the types of other's two columns are those of self's
  if (other.cols[ok].all_null || other.cols[ov].all_null) return nullptr;
  const AggEmitArgs& ea = core->table.ea;
  GroupMatchTable gt{ea.present, ea.acc + o.a0 * ea.acc_stride, o.valid_acc >= 0 ? ea.acc + o.valid_acc * ea.acc_stride : nullptr, ea.dense_base,
                     ea.n_slots - 1};
  TablePtr rows = select_group_match_rows(core->ctx, other, ok, ov, gt);
  // self's columns are views of the survivors' key and value columns (equal by the join condition, and never NULL)
  std::vector<Column> mine;
  for (size_t i = 0; i < kinds.size(); ++i) {
    Column c = rows->cols[kinds[i] == 0 ? ok : ov];
    c.name = self.cols[i].name;
    c.format = self.cols[i].format;
    c.nullable = self.cols[i].nullable;
    c.validity = nullptr;
    mine.push_back(std::move(c));
  }
  auto t = std::make_shared<Table>();
  t->ctx = core->ctx;
  t->metadata = self_is_left ? self.metadata : other.metadata;
  t->num_rows = rows->num_rows;
  if (self_is_left) {
    t->cols = std::move(mine);
    for (const Column& c : rows->cols) t->cols.push_back(c);
  } else {
    t->cols = rows->cols;
    for (Column& c : mine) t->cols.push_back(std::move(c));
  }
  return t;
}

bool has_minmax(const std::vector<AggSpec>& aggs) {
  for (const AggSpec& s : aggs)
    if (s.func == FLOCKGPU_AGG_MIN || s.func == FLOCKGPU_AGG_MAX) return true;
  return false;
}

}  // namespace

// The decision tree of DESIGN.md K5-K7: no group columns -> one row; empty input -> empty output; packed keys -> the
// direct-address count table, else level-1 partials (large raw inputs) and the level-2 table; other keys -> the
// row-representative table.
static TablePtr hash_aggregate_impl(const CtxPtr& ctx, const TablePtr& in_ptr, int mode, const std::vector<int>& group_cols, const std::vector<AggSpec>& aggs,
                                    bool allow_dense) {
  HostSpan agg_span("hash_aggregate (host)");
  in_ptr->dense();
  FG_CHECK(mode >= FLOCKGPU_AGG_PARTIAL && mode <= FLOCKGPU_AGG_SINGLE, FLOCKGPU_ERR_INVALID, "hash_aggregate: bad mode %d", mode);
  const bool states_in = mode == FLOCKGPU_AGG_FINAL || mode == FLOCKGPU_AGG_FINAL_PARTITIONED;
  // A NULL state column (the state row of an aggregate over no input) merges as "absent": Final over such a row is
  // Final over no row (the reference skips NULL states; COUNT's state is 0 there, the identity).
  if (states_in && group_cols.empty()) {
    bool null_state = false;
    for (const Column& c : in_ptr->cols) null_state |= c.all_null;
    if (null_state) return hash_aggregate_impl(ctx, empty_like(ctx, *in_ptr), mode, group_cols, aggs, allow_dense);
  }
  const Table& in = *in_ptr;
  for (int g : group_cols) {
    FG_CHECK(g >= 0 && g < int(in.cols.size()), FLOCKGPU_ERR_INVALID, "hash_aggregate: group column %d out of range", g);
    FG_CHECK(!in.cols[g].all_null, FLOCKGPU_ERR_UNSUPPORTED, "hash_aggregate: NULL group column");
  }
  const AggPlan p = plan_aggregates(in, mode, aggs);
  const int n_acc = p.n_acc();
  const int64_t n = in.num_rows;
  if (group_cols.empty()) return aggregate_ungrouped(ctx, in, mode, aggs, p);
  if (n == 0) return empty_grouped(ctx, in, group_cols, p);
  KeyPack kp{};
  GroupTable t;
  if (pack_keys(in, group_cols, &kp)) {
    // Final* inputs are partial states: every key occurs at most once per producer, so a CTA-local pre-aggregation
    // finds nothing to merge (agg_local_kernel would cost a full pass on q5's 2-GPU final stage for no reduction)
    // (also right for the Final* stage of a DISTINCT, which has no states: its input arrives hash-routed, 1/W of the
    // keys spread over the WHOLE key range -- no locality for a sliding window, no density for a direct-address table;
    // when tried, the dense table overflowed and the stage paid both paths)
    Partials l1;
    if (n >= (int64_t(1) << 18) && size_t(AL_SLOTS) * 8 * (1 + n_acc) <= 200 * 1024 && !states_in) {
      const bool count32 = kp.n == 1 && kp.width[0] == 4 && p.outs.size() <= 1 && (n_acc == 0 || (n_acc == 1 && p.accs[0].op == ACC_COUNT && p.accs[0].col < 0));
      if (count32 && allow_dense && n < (int64_t(1) << 32)) return count_table(ctx, in_ptr, mode, group_cols, aggs, p);
      l1 = level1_partials(ctx, in, kp, p, count32);
    }
    t = packed_table(ctx, in, kp, p, l1);
    if (t.mode == 1 && allow_dense && mode == FLOCKGPU_AGG_SINGLE && kp.n == 1 && kp.width[0] == 4 && has_minmax(aggs) && comm_world(ctx) == 1) {
      auto core = std::make_shared<GroupsCore>();
      core->ctx = ctx;
      core->input = in_ptr;
      core->group_cols = group_cols;
      core->aggs = aggs;
      core->plan = p;
      core->table = std::move(t);
      std::vector<int> kinds{0};
      std::vector<std::string> names{in.cols[group_cols[0]].name};
      for (size_t j = 0; j < p.outs.size(); ++j) {
        kinds.push_back(int(j) + 1);
        names.push_back(p.outs[j].name);
      }
      return groups_table(core, kinds, names, in.metadata);
    }
  } else if (TablePtr distinct = row_table(ctx, in_ptr, group_cols, p, &t)) {
    return distinct;
  }
  return emit_groups(ctx, in, group_cols, p, t);
}

}  // namespace fg

// ================================================================================================
using namespace fg;

extern "C" int flockgpu_hash_aggregate(flockgpu_ctx* ctx, const flockgpu_table* in, int32_t mode, const int32_t* group_cols, int32_t n_group_cols,
                                       const flockgpu_agg_spec* aggs, int32_t n_aggs, flockgpu_table** out) {
  return guarded([&] {
    auto c = core_of(ctx);
    FG_CHECK(out && in && in->table, FLOCKGPU_ERR_INVALID, "hash_aggregate: null argument");
    FG_CHECK(n_group_cols >= 0 && n_aggs >= 0 && (n_group_cols == 0 || group_cols) && (n_aggs == 0 || aggs), FLOCKGPU_ERR_INVALID,
             "hash_aggregate: bad column lists");
    std::lock_guard<std::recursive_mutex> g(c->mu);
    FG_CUDA(cudaSetDevice(c->device));
    std::vector<int> gc(group_cols, group_cols + n_group_cols);
    std::vector<AggSpec> as;
    for (int i = 0; i < n_aggs; ++i) as.push_back(AggSpec{aggs[i].func, aggs[i].col, aggs[i].name ? aggs[i].name : ""});
    *out = wrap_table(hash_aggregate(c, in->table, mode, gc, as));
  });
}
