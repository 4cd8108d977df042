// filter_project.cu -- K1: FilterExec + CoalesceBatchesExec + ProjectionExec as one pass over HBM.
//
// Reference operators replaced (DataFusion fork, not in tree; shapes evidenced at
// flock/src/distributed_plan/planner.rs:90-92 (q1), :120-124 (q2), :151-163 (q3 filters)):
//   FilterExec:     predicate.evaluate(batch) -> BooleanArray -> arrow filter_record_batch (stable)
//   ProjectionExec: per-batch expression evaluation; plain Column exprs are zero-copy
//
// filter_compact_kernel: ONE launch for the whole relation (all 64 Ki-row batches: a 1.3 MB batch is
// 0.2 us of HBM traffic, far below launch latency, so per-batch launches cannot work).  CTAs take tiles of
// 256 x {4, 16, 32} rows, evaluate the predicate (PredI32: one multiply-add + compare per row for the NEXMark shapes;
// the generic term interpreter otherwise), rank the survivors (compact.cuh), obtain the tile's global output offset
// from the grid-wide prefix protocol (each input byte is read once, no second pass), and write the surviving rows of
// every fixed-width output column in input order.  PredI32 walks cooperative rounds with the next tile's column bytes
// in flight (see the kernel).  Utf8 outputs leave through the selection vector and gather.cu.
// Host-resident (page-locked, zero-copy fed) predicate columns are read in place over PCIe.
#include <algorithm>
#include <cstdlib>
#include <type_traits>

#include "compact.cuh"
#include "expr_compile.h"
#include "internal.h"
#include "pred_i32.h"

namespace fg {

constexpr int FP_THREADS = CP_THREADS;

struct FilterArgs {
  int64_t n_rows;
  int32_t n_out;
  int32_t pad;
  CompactScratch sc;                 // tickets / prefix scratch of this launch (compact.cuh)
  uint32_t* sel_out;                 // optional: indices of surviving rows
  unsigned long long* out_count;     // total surviving rows
  unsigned long long* host_count;    // pinned host slot that also receives the total (NULL: none)
  int* err_flag;                     // set to 1 on divide-by-zero
  unsigned long long* trace;         // debug (FLOCKGPU_TRACE): 8 globaltimer stamps per tile, else NULL
  ColRef cols[MAX_IN_COLS];
  OutCol outs[MAX_OUT_COLS];
};

// ---- predicate functors ---------------------------------------------------------------------------
// A functor evaluates this thread's I rows of a tile and returns one bit per item, in two steps: load() issues the
// tile's loads into a Staged value (a shared-memory variable of the kernel) and test() turns it into the verdicts.
// Between the two the kernel works on the previous tile, so a functor that stages asynchronous copies keeps them in
// flight across that work.  E = rows a
// thread loads contiguously (vector width); item k is row
//   tile_base + ((k / E) * FP_THREADS + tid) * E + k % E.
// ROWS = rows per thread per tile: 16 for large inputs; 4 for small ones, where 4 Ki-row tiles would leave most SMs
// idle and every thread would walk 16 rows' worth of dependent loads (NEXMark q3: 200 K persons = 49 tiles)
template <int ROWS>
struct PredGenericT {
  static constexpr int E = 1;
  static constexpr int I = ROWS;
  static constexpr int MIN_CTAS = 1;
  static constexpr bool ROUNDS = false;  // the interpreter's loads depend on each other: nothing to stage ahead
  struct Staged {};
  Predicate p;
  __device__ __forceinline__ void load(Staged&, int64_t, int64_t, int) const {}
  __device__ __forceinline__ unsigned long long test(const Staged&, const ColRef* cols, int64_t tile_base, int64_t n_rows, int tid, int* err) const {
    int64_t rows[I];
#pragma unroll
    for (int k = 0; k < I; ++k) {
      int64_t r = tile_base + int64_t(k) * FP_THREADS + tid;
      rows[k] = r < n_rows ? r : -1;
    }
    return eval_predicate<I>(p, cols, rows, err);
  }
};

// A predicate in the tree form (expr_tree.h): the verdict is the register program's result.  The register file sits in
// the functor's shared staging area, two rows per thread at a time.
template <int ROWS>
struct PredTreeT {
  static constexpr int E = 1;
  static constexpr int I = ROWS;
  static constexpr int MIN_CTAS = 1;
  static constexpr bool ROUNDS = false;
  static constexpr int R = 2;
  struct Staged {  // thread t only touches slots [.][t]
    Val v[TREE_REGS * R * FP_THREADS];
    uint8_t f[TREE_REGS * R * FP_THREADS];
  };
  TreeProgram p;
  __device__ __forceinline__ void load(Staged&, int64_t, int64_t, int) const {}
  __device__ __forceinline__ unsigned long long test(const Staged& st, const ColRef* cols, int64_t tile_base, int64_t n_rows, int tid, int* err) const {
    Staged& s = const_cast<Staged&>(st);  // the kernel's own shared variable
    const TreeRegs<R, FP_THREADS> regs{s.v + tid, s.f + tid};
    unsigned long long bits = 0;
    for (int k = 0; k < I; k += R) {
      int64_t rows[R];
#pragma unroll
      for (int j = 0; j < R; ++j) {
        const int64_t r = tile_base + int64_t(k + j) * FP_THREADS + tid;
        rows[j] = r < n_rows ? r : -1;
      }
      bits |= (unsigned long long)eval_tree<R>(p, cols, nullptr, rows, false, regs, err) << k;
    }
    return bits;
  }
};

// other JOIN (group key, MIN / MAX) ON (k, v) against a direct-address group table (NEXMark q9: bids back to each
// auction's top price): a row survives when k is inside the table's range, its slot is present and the slot's value
// equals v; a NULL k or v matches nothing.  The table (q9: 600 K auctions, a byte and a word each) stays in L2 while
// the two columns stream once.  Every thread issues all its rows' loads before it tests any of them.
struct PredGroupMatch {
  static constexpr int E = 1;
  static constexpr int I = 16;
  static constexpr int MIN_CTAS = 2;
  static constexpr bool ROUNDS = false;
  struct Staged {};
  const uint32_t* key;
  const void* val;
  const uint8_t* key_valid;
  const uint8_t* val_valid;
  int32_t val_width;  // 4 or 8
  int32_t pad;
  GroupMatchTable t;
  __device__ __forceinline__ void load(Staged&, int64_t, int64_t, int) const {}
  __device__ __forceinline__ unsigned long long test(const Staged&, const ColRef*, int64_t tile_base, int64_t n_rows, int tid, int*) const {
    unsigned long long slot[I], v[I];
    unsigned ok = 0;
#pragma unroll
    for (int k = 0; k < I; ++k) {
      const int64_t r = tile_base + int64_t(k) * FP_THREADS + tid;
      slot[k] = ~0ull;
      v[k] = 0;
      if (r < n_rows) {
        slot[k] = (unsigned long long)key[r] - t.base;  // keys below the base wrap to huge slots
        v[k] = val_width == 4 ? (unsigned long long)static_cast<const uint32_t*>(val)[r] : static_cast<const unsigned long long*>(val)[r];
        const bool null_row = (key_valid && !key_valid[r]) || (val_valid && !val_valid[r]);
        if (!null_row && slot[k] < t.n_slots) ok |= 1u << k;
      }
    }
#pragma unroll
    for (int k = 0; k < I; ++k)
      if (((ok >> k) & 1u) && !t.present[slot[k]]) ok &= ~(1u << k);
    unsigned long long bits = 0;
#pragma unroll
    for (int k = 0; k < I; ++k) {
      if (!((ok >> k) & 1u)) continue;
      const unsigned long long a = t.acc[slot[k]];
      const bool eq = val_width == 4 ? uint32_t(a) == uint32_t(v[k]) : a == v[k];
      if (eq && (!t.valid || t.valid[slot[k]] != 0ull)) bits |= 1ull << k;
    }
    return bits;
  }
};

// One tile = 8 Ki rows: every thread copies eight 16-byte pieces of the column per tile into shared memory with
// cp.async, and the kernel keeps the next tile's copies in flight while it ranks, publishes and writes the current
// one (cooperative rounds, compact.cuh).  Staging in shared memory instead of registers keeps the loads in flight
// without costing registers, so more CTAs stay resident and each round covers more of the relation.
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, int src_bytes) {
  // src_bytes < 16 zero-fills the rest of the 16 bytes (rows past the end of the relation)
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(unsigned(__cvta_generic_to_shared(smem))), "l"(gmem), "r"(src_bytes)
               : "memory");
}

template <int MODE>
struct PredI32 {
  static constexpr int E = 4;
  static constexpr int L = 8;          // 16-byte copies per thread and tile
  static constexpr int I = 4 * L;      // rows per thread per tile
  static constexpr int MIN_CTAS = 4;   // <= 64 registers
  static constexpr bool ROUNDS = true;
  struct Staged {                      // in shared memory; thread t only touches v[.][t], so no barrier is needed
    int4 v[L][FP_THREADS];
  };
  const int32_t* col;
  PredI32Consts k;
  const void* const* chunks;  // host-resident column (zero-copy feed): chunk bases, else NULL
  int32_t chunk_shift;
  // address of rows [row0, row0 + 4): row0 is a multiple of 4 and chunk lengths are powers of two >= 4096
  __device__ __forceinline__ const int32_t* at(int64_t row0) const {
    if (!chunks) return col + row0;
    return static_cast<const int32_t*>(chunks[row0 >> chunk_shift]) + (row0 & ((int64_t(1) << chunk_shift) - 1));
  }
  __device__ __forceinline__ bool test(int32_t x) const { return pred_i32_test<MODE>(k, x); }
  __device__ __forceinline__ unsigned test4(const int4& v) const {
    return unsigned(test(v.x)) | (unsigned(test(v.y)) << 1) | (unsigned(test(v.z)) << 2) | (unsigned(test(v.w)) << 3);
  }
  __device__ __forceinline__ void load(Staged& st, int64_t tile_base, int64_t n_rows, int tid) const {
    if (!chunks && tile_base + int64_t(FP_THREADS) * I <= n_rows) {
      // full tile of a device-resident column (every tile but the last): no bounds, no chunk lookup
      const int4* p = reinterpret_cast<const int4*>(col + tile_base) + tid;
#pragma unroll
      for (int j = 0; j < L; ++j) cp_async16(&st.v[j][tid], p + j * FP_THREADS, 16);
    } else {
#pragma unroll
      for (int j = 0; j < L; ++j) {
        const int64_t row0 = tile_base + (int64_t(j) * FP_THREADS + tid) * 4;
        const int64_t left = n_rows - row0;
        cp_async16(&st.v[j][tid], at(left > 0 ? row0 : 0), left >= 4 ? 16 : left > 0 ? int(left) * 4 : 0);
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  // Only the one-bit verdicts outlive test(): the values of the ~1 % survivors are re-read from L2 when they are written.
  __device__ __forceinline__ unsigned long long test(const Staged& st, const ColRef*, int64_t tile_base, int64_t n_rows, int tid, int*) const {
    asm volatile("cp.async.wait_all;" ::: "memory");
    unsigned bits = 0;
#pragma unroll
    for (int j = 0; j < L; ++j) bits |= test4(st.v[j][tid]) << (4 * j);
    if (tile_base + int64_t(FP_THREADS) * I > n_rows) {
#pragma unroll
      for (int j = 0; j < L; ++j) {
        const int64_t left = n_rows - (tile_base + (int64_t(j) * FP_THREADS + tid) * 4);  // mask rows past the end
        if (left < 4) bits &= ~((left <= 0 ? 0xfu : (0xfu << left) & 0xfu) << (4 * j));
      }
    }
    return bits;
  }
};

// Pulls the survivors' pass-through values (one dependent ~1 us DRAM read each) into L2 ahead of the write phase,
// which then finds them there.  Every survivor is prefetched, not only the first four of a thread: in the cooperative
// rounds a tile is written one whole iteration after it is ranked, so even a thread whose 32 rows all survive (the hot
// auction id) has its values in L2 by then, and a prefetch costs the thread one instruction.
template <int E>
__device__ __forceinline__ void prefetch_survivors(const FilterArgs& a, unsigned long long bits, int64_t tile_base, int tid) {
  if (!bits) return;
  for (int c = 0; c < a.n_out; ++c) {
    const OutCol& oc = a.outs[c];
    if (oc.kind != OUT_PASS) continue;
    const ColRef& src = a.cols[oc.src_col];
    if (src.chunks) continue;  // host-resident: fetched once, when written
    unsigned long long m = bits;
#pragma unroll 1
    while (m) {
      const int k = __ffsll((long long)m) - 1;
      m &= m - 1;
      prefetch_l2(static_cast<const char*>(src.data) + (tile_base + cp_item_index<E>(k, tid)) * oc.width);
    }
  }
}

// Writes this thread's survivors of the tile to their output positions, in input order.  A thread may own many
// survivors (NEXMark's hot auction id: when it satisfies the predicate half of the rows of a stretch survive), and
// every pass-through value is a dependent ~1 us DRAM read: gather four survivors at a time so that their loads are in
// flight together.  COMPUTED: some output is an expression (eval_chain), compiled only into the kernels that need it.
template <int E, int I, bool COMPUTED>
__device__ __forceinline__ void write_survivors(const FilterArgs& a, const CompactSmem<E, I>& sm, unsigned long long bits, int64_t tile_base,
                                                const unsigned (&lane_prefix)[I / E], int tid, int* err) {
  // positions and rows are kept as 32-bit offsets from the tile's output and input bases until used: the 64-bit
  // forms of four survivors would not fit the register budget next to the next tile's loads in flight
  const long long excl = (long long)sm.excl;
  unsigned long long m = bits;
  while (m) {
    unsigned lpos[4], item[4];
    int nb = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      lpos[q] = 0;
      item[q] = 0;
      if (m) {
        const int k = __ffsll((long long)m) - 1;
        m &= m - 1;
        lpos[q] = cp_local_position<E, I>(sm, bits, k, lane_prefix);
        item[q] = unsigned(cp_item_index<E>(k, tid));
        nb = q + 1;
      }
    }
    if (a.sel_out) {
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (q < nb) a.sel_out[excl + lpos[q]] = uint32_t(tile_base + item[q]);
    }
    for (int c = 0; c < a.n_out; ++c) {
      const OutCol& oc = a.outs[c];
      if (!COMPUTED || oc.kind == OUT_PASS) {
        const ColRef& sc_col = a.cols[oc.src_col];
        if (sc_col.chunks) {
          // host-resident source: one PCIe read per survivor
          const int64_t mask = (int64_t(1) << sc_col.chunk_shift) - 1;
          uint64_t v[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            v[q] = 0;
            if (q < nb) {
              const int64_t row = tile_base + item[q];
              const char* base = static_cast<const char*>(sc_col.chunks[row >> sc_col.chunk_shift]) + (row & mask) * oc.width;
              v[q] = oc.width == 4 ? uint64_t(*reinterpret_cast<const uint32_t*>(base)) : *reinterpret_cast<const uint64_t*>(base);
            }
          }
#pragma unroll
          for (int q = 0; q < 4; ++q)
            if (q < nb) {
              if (oc.width == 4) static_cast<uint32_t*>(oc.dst)[excl + lpos[q]] = uint32_t(v[q]);
              else static_cast<uint64_t*>(oc.dst)[excl + lpos[q]] = v[q];
            }
        } else if (oc.width == 4) {
          const uint32_t* src = static_cast<const uint32_t*>(sc_col.data) + tile_base;
          uint32_t* dst = static_cast<uint32_t*>(oc.dst) + excl;
          uint32_t v[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) v[q] = q < nb ? src[item[q]] : 0u;
#pragma unroll
          for (int q = 0; q < 4; ++q)
            if (q < nb) dst[lpos[q]] = v[q];
        } else {
          const uint64_t* src = static_cast<const uint64_t*>(sc_col.data) + tile_base;
          uint64_t* dst = static_cast<uint64_t*>(oc.dst) + excl;
          uint64_t v[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) v[q] = q < nb ? src[item[q]] : 0ull;
#pragma unroll
          for (int q = 0; q < 4; ++q)
            if (q < nb) dst[lpos[q]] = v[q];
        }
      } else if constexpr (COMPUTED) {
        int64_t row[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) row[q] = q < nb ? tile_base + item[q] : -1;
        Val acc[4];
        eval_chain<4>(oc.chain, a.cols, row, acc, err);
#pragma unroll
        for (int q = 0; q < 4; ++q)
          if (q < nb) store_val(oc.dst, oc.out_dtype, excl + lpos[q], acc[q]);
      }
    }
  }
}

// Trace (FLOCKGPU_TRACE): 8 %globaltimer stamps per tile, written by thread 0 of the CTA that owns the tile:
//   0 the CTA turns to the tile, 1 verdicts known (the tile's loads have landed), 2 ranked within the tile, 3 output
//   offset known, 4 survivors written, 5 CTA end (its last tile only), 6 CTA index, 7 SM id.  In the cooperative
//   rounds 3 and 4 come one iteration after 2: tile r is written after tile r + 1 is published.
constexpr int FP_TRACE_WORDS = 8;

// The expression interpreter of computed outputs needs more registers than MIN_CTAS allows: kernels that have it
// trade residency for no spills (the cooperative rounds take any grid).
template <class PredFn, bool COMPUTED>
__global__ void __launch_bounds__(FP_THREADS, COMPUTED && PredFn::MIN_CTAS > 2 ? 2 : PredFn::MIN_CTAS) filter_compact_kernel(const __grid_constant__ PredFn pred, const __grid_constant__ FilterArgs a) {
  constexpr int E = PredFn::E;
  constexpr int I = PredFn::I;
  constexpr int TILE = FP_THREADS * I;
  const int tid = threadIdx.x;
  const CompactScratch& sc = a.sc;
  int err = 0;

  auto now = [] {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
  };
  auto stamp = [&](long long tile, int k) {
    if (a.trace && tid == 0) a.trace[tile * FP_TRACE_WORDS + k] = now();
  };
  auto stamp_ids = [&](long long tile) {
    if (a.trace && tid == 0) {
      unsigned smid;
      asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
      a.trace[tile * FP_TRACE_WORDS + 5] = 0;  // the CTA's last tile stamps its end afterwards
      a.trace[tile * FP_TRACE_WORDS + 6] = blockIdx.x;
      a.trace[tile * FP_TRACE_WORDS + 7] = smid;
    }
  };

  __shared__ typename PredFn::Staged st;
  if (sc.single_wave) {
    // Cooperative rounds (compact.cuh): tile blockIdx.x + r * grid in round r.  Iteration r tests tile r (its loads
    // were issued one iteration earlier), issues tile r + 1's loads, ranks and publishes tile r, and only then reads
    // the offset of tile r - 1 and writes its survivors.  So the loads stream while the CTA ranks, waits and writes,
    // and a round's counts are published without waiting for anybody's writes.  Tile indices are 32-bit here (2^31
    // tiles are far beyond any relation): 64-bit loop state would not fit the 64-register budget of four CTAs per SM.
    //
    // A launch may start while the filter launched ahead of it drains (compact.cuh: EarlyStart, launch_compact_early).
    // Until griddepcontrol.wait, right before its first publish, a CTA only streams its first tiles into shared memory,
    // tests and ranks the first one and prefetches its survivors: nothing there touches the scan scratch (the previous
    // launch may still poll those words), the outputs (their blocks may have been released while it ran) or
    // d_scalars.  Past the wait the previous launch has completed and its memory is visible.  The CTA lets the next
    // launch start (launch_dependents) once it has passed its wait and issued its last tile's loads, so at most one
    // launch runs ahead of the current one.  Without the launch attribute both instructions do nothing.
    __shared__ CompactSmem<E, I> rank_sm[2];  // tile r is ranked into rank_sm[r & 1] and written from it one iteration later
    __shared__ unsigned long long rounds_done;
    const int num_tiles = int(sc.num_tiles);
    int tile = blockIdx.x;
    if (tile < num_tiles) pred.load(st, int64_t(tile) * TILE, a.n_rows, tid);
    // A thread's group prefixes are at most 31 x E < 256: the tile waiting for its writes keeps them as bytes (group g
    // in byte g % 4 of register g / 4), which keeps the kernel within its register budget.
    constexpr int G = I / E, P = (G + 3) / 4;
    static_assert(31 * E < 256 && I <= 32, "group prefixes do not fit a byte, or verdicts a word");
    unsigned prev_bits = 0, prev_packed[P] = {};
    for (int it = 0;; ++it, tile += sc.grid) {
      const int prev = tile - sc.grid;
      unsigned bits = 0, packed[P] = {};
      if (tile < num_tiles) {
        stamp(tile, 0);
        bits = unsigned(pred.test(st, a.cols, int64_t(tile) * TILE, a.n_rows, tid, &err));
        stamp(tile, 1);
        if (tile + sc.grid < num_tiles) pred.load(st, int64_t(tile + sc.grid) * TILE, a.n_rows, tid);
        unsigned lane_prefix[I / E];
        cp_rank_local<E, I>(rank_sm[it & 1], bits, lane_prefix);
#pragma unroll
        for (int g = 0; g < G; ++g) packed[g >> 2] |= lane_prefix[g] << ((g & 3) * 8);
        stamp(tile, 2);
        prefetch_survivors<E>(a, bits, int64_t(tile) * TILE, tid);
        if (it == 0) asm volatile("griddepcontrol.wait;" ::: "memory");
        cp_round_publish(sc, tile, rank_sm[it & 1].tile_total);
        // the first iteration with no loads left to issue (tile + grid, if any, was issued above)
        if (tile + 2 * sc.grid >= num_tiles && (it == 0 || tile + sc.grid < num_tiles)) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
      }
      if (it > 0) {
        CompactSmem<E, I>& ps = rank_sm[(it - 1) & 1];
        cp_round_offset<E, I>(ps, sc, prev, prev - int(blockIdx.x), rounds_done);
        stamp(prev, 3);
        if (prev_bits) {
          unsigned prev_prefix[G];
#pragma unroll
          for (int g = 0; g < G; ++g) prev_prefix[g] = (prev_packed[g >> 2] >> ((g & 3) * 8)) & 0xffu;
          write_survivors<E, I, COMPUTED>(a, ps, prev_bits, int64_t(prev) * TILE, prev_prefix, tid, &err);
        }
        __syncthreads();  // ps is reused by the next tile
        stamp(prev, 4);
        stamp_ids(prev);
        if (tile >= num_tiles) stamp(prev, 5);
      }
      if (tile >= num_tiles) break;
      prev_bits = bits;
#pragma unroll
      for (int i = 0; i < P; ++i) prev_packed[i] = packed[i];
    }
  } else {
    // decoupled look-back: tiles drawn from the ticket counter, one at a time
    __shared__ CompactSmem<E, I> sm;
    long long tile, last = -1;
    for (int it = 0; (tile = cp_next_tile(sm, sc, it)) >= 0; ++it) {
      last = tile;
      const int64_t tile_base = tile * TILE;
      stamp(tile, 0);
      pred.load(st, tile_base, a.n_rows, tid);
      const unsigned long long bits = pred.test(st, a.cols, tile_base, a.n_rows, tid, &err);
      stamp(tile, 1);
      unsigned lane_prefix[I / E];
      cp_rank_local<E, I>(sm, bits, lane_prefix);
      stamp(tile, 2);
      prefetch_survivors<E>(a, bits, tile_base, tid);
      cp_block_lookback<E, I>(sm, sc, tile, sm.tile_total);
      stamp(tile, 3);
      if (bits) write_survivors<E, I, COMPUTED>(a, sm, bits, tile_base, lane_prefix, tid, &err);
      __syncthreads();  // sm is reused by the next tile
      stamp(tile, 4);
      stamp_ids(tile);
    }
    if (last >= 0) stamp(last, 5);
  }
  if (err) *a.err_flag = 1;
}

// ---- pure projection (no predicate): streaming evaluation of the computed columns ----------------
struct ProjectArgs {
  int64_t n_rows;
  int32_t n_out;
  int32_t pad;
  int* err_flag;
  ColRef cols[MAX_IN_COLS];
  OutCol outs[MAX_OUT_COLS];
};

constexpr int PJ_THREADS = 256;
constexpr int PJ_ROWS = 4;

__global__ void __launch_bounds__(PJ_THREADS) project_generic_kernel(const __grid_constant__ ProjectArgs a) {
  int err = 0;
  const int64_t stride = int64_t(gridDim.x) * PJ_THREADS * PJ_ROWS;
  for (int64_t base = int64_t(blockIdx.x) * PJ_THREADS * PJ_ROWS; base < a.n_rows; base += stride) {
    int64_t rows[PJ_ROWS];
#pragma unroll
    for (int j = 0; j < PJ_ROWS; ++j) {
      int64_t r = base + int64_t(j) * PJ_THREADS + threadIdx.x;
      rows[j] = r < a.n_rows ? r : -1;
    }
    for (int c = 0; c < a.n_out; ++c) {
      const OutCol& oc = a.outs[c];
      Val acc[PJ_ROWS];
      eval_chain<PJ_ROWS>(oc.chain, a.cols, rows, acc, &err);
#pragma unroll
      for (int j = 0; j < PJ_ROWS; ++j)
        if (rows[j] >= 0) store_val(oc.dst, oc.out_dtype, rows[j], acc[j]);
    }
  }
  if (err) *a.err_flag = 1;
}

// NEXMark q1: price' = lit * CAST(price AS Float64).  One IEEE multiply per row (__dmul_rn: the i32 ->
// f64 conversion is exact, so the product has a single rounding, SURVEY.md Appendix C.2).
// 16 B in, 32 B out per thread-iteration; 4 B + 8 B per row is all the traffic there is.
__global__ void __launch_bounds__(PJ_THREADS) project_i32_to_f64_mul_kernel(const int32_t* __restrict__ in, double* __restrict__ out,
                                                                            int64_t n_rows, double lit) {
  const int64_t n4 = n_rows >> 2;
  const int64_t stride = int64_t(gridDim.x) * PJ_THREADS;
  for (int64_t i = int64_t(blockIdx.x) * PJ_THREADS + threadIdx.x; i < n4; i += stride) {
    int4 v = ldg_stream_v4(in + i * 4);
    stg_stream_v2f64(out + i * 4, __dmul_rn(lit, double(v.x)), __dmul_rn(lit, double(v.y)));
    stg_stream_v2f64(out + i * 4 + 2, __dmul_rn(lit, double(v.z)), __dmul_rn(lit, double(v.w)));
  }
  if (blockIdx.x == 0 && threadIdx.x < (n_rows & 3)) {
    int64_t r = (n4 << 2) + threadIdx.x;
    out[r] = __dmul_rn(lit, double(in[r]));
  }
}

__global__ void __launch_bounds__(256) and_validity_kernel(const uint8_t* a, const uint8_t* b, const uint8_t* c, const uint8_t* d, uint8_t* out, int64_t n) {
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x) {
    uint8_t v = a[i];
    if (b) v &= b[i];
    if (c) v &= c[i];
    if (d) v &= d[i];
    out[i] = v;
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
std::vector<ColInfo> col_infos(const Table& t) {
  std::vector<ColInfo> v;
  for (const Column& c : t.cols) v.push_back({c.dtype, c.name, c.format, c.validity != nullptr});
  return v;
}

ColRef colref_of(const Column& c) {
  ColRef r{};
  r.data = c.values();
  r.offsets = c.offs();
  r.dtype = c.dtype;
  r.chunk_shift = c.chunks ? c.chunks->shift : 0;
  r.chunks = c.chunks ? static_cast<const void* const*>(c.chunks->table->ptr) : nullptr;
  r.validity = c.valid();
  return r;
}

void fill_colrefs(const Table& t, ColRef* refs) {
  for (size_t i = 0; i < t.cols.size(); ++i) refs[i] = colref_of(t.cols[i]);
}

void filter_colrefs(const Table& t, ColRef* refs) {
  FG_CHECK(t.cols.size() <= size_t(MAX_IN_COLS), FLOCKGPU_ERR_UNSUPPORTED, "filter_project: more than %d input columns", MAX_IN_COLS);
  for (const Column& c : t.cols) FG_CHECK(!c.all_null, FLOCKGPU_ERR_UNSUPPORTED, "filter_project: NULL input column \"%s\"", c.name.c_str());
  fill_colrefs(t, refs);
}

// Launches the filter over the whole relation in tiles of FP_THREADS x PredFn::I rows.  The grid is the resident CTAs
// of the instantiation launched: functors with ROUNDS walk any number of cooperative rounds; the others run one
// wave when the tiles fit it and fall back to decoupled look-back beyond it.
template <class PredFn, bool COMPUTED>
static void launch_filter(const CtxPtr& ctx, const PredFn& pred, FilterArgs args, const char* profile_name = "filter_compact_kernel",
                          const EarlyStart* early = nullptr) {
  constexpr int64_t TILE = int64_t(FP_THREADS) * PredFn::I;
  const int64_t num_tiles = (args.n_rows + TILE - 1) / TILE;
  auto* kernel = &filter_compact_kernel<PredFn, COMPUTED>;
  args.sc = prepare_compact(ctx, num_tiles, resident_ctas(ctx, reinterpret_cast<const void*>(kernel), FP_THREADS), args.out_count, PredFn::ROUNDS);
  args.sc.host_count = args.host_count;
  BufferPtr trace_buf;
  static const char* trace_path = getenv("FLOCKGPU_TRACE");
  if (trace_path) {
    // every word of every tile is stamped by the kernel: no memset, which would stand between two launches
    trace_buf = alloc(ctx, size_t(num_tiles) * FP_TRACE_WORDS * 8);
    args.trace = trace_buf->as<unsigned long long>();
  }
  const int64_t overlapped0 = ctx->overlapped.load(std::memory_order_relaxed);
  {
    LaunchTimer lt(ctx, profile_name);
    // only the rounds path waits for the previous grid before it touches shared state
    launch_compact_early(ctx, kernel, args.sc, PredFn::ROUNDS ? early : nullptr, pred, args);
  }
  FG_CUDA(cudaGetLastError());
  count_launch(ctx);
  if (trace_path)
    ctx->filter_traces.push_back({trace_buf, (long long)num_tiles, args.sc.grid, args.sc.single_wave,
                                  int(ctx->overlapped.load(std::memory_order_relaxed) != overlapped0)});
}

void dump_filter_traces(const CtxPtr& ctx) {
  static const char* trace_path = getenv("FLOCKGPU_TRACE");
  if (!trace_path || ctx->filter_traces.empty()) return;
  // debug only: the per-tile time stamps of the launches since the last dump, in launch order (overwrites the file).
  // Per launch a header: tiles, grid, 1 when tile t ran in round t / grid of the cooperative mode (0: decoupled
  // look-back), 1 when the launch was allowed to overlap the one before it; then one line of stamps per tile.
  std::vector<CtxCore::FilterTrace> traces;
  traces.swap(ctx->filter_traces);
  FG_CUDA(cudaStreamSynchronize(ctx->stream));
  FILE* f = fopen(trace_path, "w");
  if (!f) return;
  for (const CtxCore::FilterTrace& t : traces) {
    std::vector<unsigned long long> h(size_t(t.tiles) * FP_TRACE_WORDS);
    FG_CUDA(cudaMemcpy(h.data(), t.stamps->ptr, h.size() * 8, cudaMemcpyDeviceToHost));
    fprintf(f, "%lld %d %d %d\n", t.tiles, t.grid, t.rounds, t.overlapped);
    for (size_t i = 0; i < h.size() / FP_TRACE_WORDS; ++i) {
      for (int j = 0; j < FP_TRACE_WORDS; ++j) fprintf(f, "%llu ", h[i * FP_TRACE_WORDS + j]);
      fprintf(f, "\n");
    }
  }
  fclose(f);
}

TablePtr filter_project(const CtxPtr& ctx, const TablePtr& in_ptr, const Expr* predicate, const std::vector<Expr>& projections,
                        const std::vector<std::string>& names) {
  const Table& in = *in_ptr;
  // a pure column selection / renaming of a relation that is still in table form (DeferredTable) keeps it there
  if (in_ptr->deferred && !predicate && !projections.empty()) {
    std::vector<ColInfo> dinfos = col_infos(in);
    std::vector<int> src;
    std::vector<std::string> out_names;
    bool plain = true;
    for (size_t i = 0; i < projections.size() && plain; ++i) {
      CompiledValue v;
      try {
        v = compile_value(projections[i], dinfos, PROJECT_MAX_NULL_INPUTS);
      } catch (const Error& err) {
        if (err.code != FLOCKGPU_ERR_UNSUPPORTED) throw;  // not a plain column: compiled again, for the tree form, below
      }
      plain = v.passthrough;
      src.push_back(v.src_col);
      out_names.push_back(i < names.size() && !names[i].empty() ? names[i] : (plain ? in.cols[v.src_col].name : std::string()));
    }
    if (plain) {
      std::shared_ptr<DeferredTable> d = in_ptr->deferred;
      if (TablePtr t = d->project(in, src, out_names)) return t;
    }
  }
  in.resolve();
  std::vector<ColInfo> infos = col_infos(in);
  // ---- compile
  std::vector<CompiledValue> vals;
  std::vector<bool> tree_vals;  // vals[i] is computed by the tree form
  if (projections.empty()) {
    for (size_t i = 0; i < in.cols.size(); ++i) {
      CompiledValue v;
      v.passthrough = true;
      v.src_col = int(i);
      v.dtype = in.cols[i].dtype;
      v.format = in.cols[i].format;
      vals.push_back(v);
    }
  } else {
    // an expression the chain form refuses is evaluated in the tree form (expr_eval.cu)
    bool tree = false;
    for (const Expr& e : projections) {
      try {
        vals.push_back(compile_value(e, infos, predicate ? 0 : PROJECT_MAX_NULL_INPUTS));
        tree_vals.push_back(false);
      } catch (const Error& err) {
        if (err.code != FLOCKGPU_ERR_UNSUPPORTED) throw;
        const CompiledTree ct = compile_tree_values({e}, infos);  // fails when the tree form refuses it too
        CompiledValue v;
        v.dtype = ct.roots[0].dtype;
        v.format = ct.roots[0].format;
        vals.push_back(v);
        tree_vals.push_back(true);
        tree = true;
      }
    }
    if (tree && predicate) {
      // tree-form values are evaluated over the surviving rows only (a division by zero in a dropped row raises nothing)
      TablePtr kept = filter_project(ctx, in_ptr, predicate, {}, {});
      return filter_project(ctx, kept, nullptr, projections, names);
    }
  }
  tree_vals.resize(vals.size(), false);
  auto out_name = [&](size_t i) -> std::string {
    if (i < names.size() && !names[i].empty()) return names[i];
    if (vals[i].passthrough) return in.cols[vals[i].src_col].name;
    return projections.empty() ? std::string() : expr_to_string(projections[i], infos);
  };

  auto out = std::make_shared<Table>();
  out->ctx = ctx;
  out->metadata = in.metadata;
  // rows stay on their rank: the routing property of an exchanged input survives when its columns pass through by name
  if (!in.partitioned_on.empty()) {
    bool kept = true;
    for (const std::string& p : in.partitioned_on) {
      bool found = false;
      for (size_t i = 0; i < vals.size(); ++i) found |= vals[i].passthrough && in.cols[vals[i].src_col].name == p && out_name(i) == p;
      kept &= found;
    }
    if (kept) {
      out->partitioned_on = in.partitioned_on;
      out->partition_world = in.partition_world;
    }
  }

  int* err_flag = reinterpret_cast<int*>(ctx->d_scalars + 8);
  bool check_err = false;

  if (!predicate) {
    // ------------------------------------------------------------------ ProjectionExec only
    in.dense();
    out->num_rows = in.num_rows;
    ProjectArgs pa{};
    pa.n_rows = in.num_rows;
    pa.err_flag = err_flag;
    filter_colrefs(in, pa.cols);
    for (size_t i = 0; i < vals.size(); ++i) {
      const CompiledValue& v = vals[i];
      Column c;
      c.name = out_name(i);
      c.dtype = v.dtype;
      c.format = v.format;
      c.length = in.num_rows;
      if (tree_vals[i]) {
        // filled in below: every tree-form column of the projection comes from one expr_eval_kernel launch
      } else if (v.passthrough) {
        const Column& s = in.cols[v.src_col];
        c.nullable = s.nullable;
        c.data = s.data;  // zero-copy, like the Arc clone in ProjectionExec
        c.offsets = s.offsets;
        c.values_bytes = s.values_bytes;
        c.all_null = s.all_null;
        c.validity = s.validity;
      } else {
        // a computed value is NULL where any column it reads is NULL
        std::vector<const uint8_t*> srcs;
        for (int col : v.null_inputs) srcs.push_back(in.cols[col].valid());
        if (!srcs.empty() && in.num_rows > 0) {
          c.validity = alloc(ctx, size_t(in.num_rows));
          c.nullable = true;
          int grid = int(std::min<int64_t>((in.num_rows + 255) / 256, int64_t(ctx->sm_count) * 8));
          {
            LaunchTimer lt(ctx, "and_validity_kernel");
            and_validity_kernel<<<grid, 256, 0, ctx->stream>>>(srcs[0], srcs.size() > 1 ? srcs[1] : nullptr, srcs.size() > 2 ? srcs[2] : nullptr,
                                                           srcs.size() > 3 ? srcs[3] : nullptr, c.validity->as<uint8_t>(), in.num_rows);
          }
          FG_CUDA(cudaGetLastError());
          count_launch(ctx);
        }
        c.data = alloc(ctx, size_t(in.num_rows) * dtype_width(v.dtype));
        if (in.num_rows > 0) {
          if (v.fast == FAST_VAL_I32_TO_F64_MUL) {
            int64_t n4 = std::max<int64_t>(1, in.num_rows / 4);
            int grid = int(std::min<int64_t>((n4 + PJ_THREADS - 1) / PJ_THREADS, int64_t(ctx->sm_count) * 8));
            {
              LaunchTimer lt(ctx, "project_i32_to_f64_mul_kernel");
              project_i32_to_f64_mul_kernel<<<grid, PJ_THREADS, 0, ctx->stream>>>(
                static_cast<const int32_t*>(in.cols[v.chain.start_col].values()), c.data->as<double>(), in.num_rows, v.fast_lit);
            }
            FG_CUDA(cudaGetLastError());
            count_launch(ctx);
          } else {
            FG_CHECK(pa.n_out < MAX_OUT_COLS, FLOCKGPU_ERR_UNSUPPORTED, "projection: more than %d computed columns", MAX_OUT_COLS);
            OutCol& oc = pa.outs[pa.n_out++];
            oc.kind = OUT_COMPUTED;
            oc.src_col = -1;
            oc.out_dtype = v.dtype;
            oc.width = dtype_width(v.dtype);
            oc.dst = c.data->ptr;
            oc.chain = v.chain;
            check_err |= v.has_div_by_col;
          }
        }
      }
      out->cols.push_back(std::move(c));
    }
    {
      std::vector<Expr> tree_exprs;
      std::vector<std::string> tree_names;
      for (size_t i = 0; i < vals.size(); ++i)
        if (tree_vals[i]) {
          tree_exprs.push_back(projections[i]);
          tree_names.push_back(out->cols[i].name);
        }
      if (!tree_exprs.empty()) {
        std::vector<Column> computed = eval_exprs(ctx, in, tree_exprs, tree_names);
        size_t k = 0;
        for (size_t i = 0; i < vals.size(); ++i)
          if (tree_vals[i]) out->cols[i] = std::move(computed[k++]);
      }
    }
    if (pa.n_out > 0 && in.num_rows > 0) {
      int64_t per_block = int64_t(PJ_THREADS) * PJ_ROWS;
      int grid = int(std::min<int64_t>((in.num_rows + per_block - 1) / per_block, int64_t(ctx->sm_count) * 8));
      if (check_err) FG_CUDA(cudaMemsetAsync(err_flag, 0, sizeof(int), ctx->stream));
      {
        LaunchTimer lt(ctx, "project_generic_kernel");
        project_generic_kernel<<<grid, PJ_THREADS, 0, ctx->stream>>>(pa);
      }
      FG_CUDA(cudaGetLastError());
      count_launch(ctx);
      if (check_err) {
        unsigned long long flag = 0;
        read_scalars(ctx, 8, 1, &flag);
        FG_CHECK((flag & 0xffffffffull) == 0, FLOCKGPU_ERR_EXECUTION, "Divide by zero");
      }
    }
    return out;
  }

  // -------------------------------------------------------------------- FilterExec (+ projection)
  CompiledPredicate cp;
  CompiledTree tree_pred;  // the predicate in the tree form, when the term form refuses it
  bool use_tree = false;
  try {
    cp = compile_predicate(*predicate, infos);
  } catch (const Error& err) {
    if (err.code != FLOCKGPU_ERR_UNSUPPORTED) throw;
    tree_pred = compile_tree_predicate(*predicate, infos);
    use_tree = true;
    cp = CompiledPredicate{};
    memset(&cp.prog, 0, sizeof cp.prog);
  }
  check_err = use_tree ? tree_pred.may_fail : cp.prog.has_div_by_col != 0;
  // host-resident (zero-copy) columns can be consumed in place only by the vectorised predicate with plain
  // pass-through fixed-width outputs; anything else scans the relation more than once and copies it to HBM first
  if (in.has_host_columns()) {
    bool in_place = cp.fast.kind != FAST_PRED_NONE;
    for (const CompiledValue& v : vals) in_place &= v.passthrough && v.dtype != FLOCKGPU_UTF8;
    if (!in_place) in.dense();
  }
  if (in.num_rows == 0) {
    // nothing to scan: an empty table with the output schema
    out->num_rows = 0;
    for (size_t i = 0; i < vals.size(); ++i) {
      Column c;
      c.name = out_name(i);
      c.dtype = vals[i].dtype;
      c.format = vals[i].format;
      c.length = 0;
      c.data = alloc(ctx, 0);
      if (c.dtype == FLOCKGPU_UTF8) {
        c.offsets = alloc(ctx, 4);
        FG_CUDA(cudaMemsetAsync(c.offsets->ptr, 0, 4, ctx->stream));
      }
      out->cols.push_back(std::move(c));
    }
    return out;
  }

  FilterArgs fa{};
  fa.n_rows = in.num_rows;
  fa.out_count = ctx->d_scalars + 0;
  fa.err_flag = err_flag;
  filter_colrefs(in, fa.cols);
  // What a launch that starts before the kernel ahead of it completes reads early (compact.cuh: EarlyStart): the
  // relation's device-resident buffers, all older than the outputs allocated below.
  EarlyStart early{0, ++ctx->alloc_seq};
  bool may_start_early = true;
  for (const Column& c : in.cols) {
    may_start_early &= !c.chunks;
    for (const BufferPtr& b : {c.data, c.offsets, c.validity})
      if (b) early.newest_input = std::max(early.newest_input, b->seq);
  }

  bool need_sel = false;
  std::vector<int> utf8_outs;
  for (size_t i = 0; i < vals.size(); ++i) {
    const CompiledValue& v = vals[i];
    Column c;
    c.name = out_name(i);
    c.dtype = v.dtype;
    c.format = v.format;
    if (v.passthrough) c.nullable = in.cols[v.src_col].nullable;
    if (v.dtype == FLOCKGPU_UTF8 || (v.passthrough && in.cols[v.src_col].validity)) {
      // Utf8 outputs and outputs with validity bytes are taken through the selection vector behind the kernel
      need_sel = true;
      utf8_outs.push_back(int(i));
    } else {
      FG_CHECK(fa.n_out < MAX_OUT_COLS, FLOCKGPU_ERR_UNSUPPORTED, "filter: more than %d fixed-width output columns", MAX_OUT_COLS);
      c.data = alloc(ctx, size_t(in.num_rows) * dtype_width(v.dtype));  // worst case: every row survives
      OutCol& oc = fa.outs[fa.n_out++];
      oc.kind = v.passthrough ? OUT_PASS : OUT_COMPUTED;
      oc.src_col = v.src_col;
      oc.out_dtype = v.dtype;
      oc.width = dtype_width(v.dtype);
      oc.dst = c.data->ptr;
      oc.chain = v.chain;
      check_err |= v.has_div_by_col;
    }
    out->cols.push_back(std::move(c));
  }
  BufferPtr sel;
  if (need_sel) {
    sel = alloc(ctx, size_t(in.num_rows) * 4);
    fa.sel_out = sel->as<uint32_t>();
  }
  if (check_err) FG_CUDA(cudaMemsetAsync(err_flag, 0, sizeof(int), ctx->stream));
  // fixed-width outputs only: the survivor count stays in flight.  The kernel stores it straight into a pinned host
  // slot (no 8-byte D2H copy on the stream); the first consumer that needs the number waits for the event
  // recorded behind the launch (Table::resolve).
  std::shared_ptr<PendingRows> pending;
  if (!check_err && utf8_outs.empty()) {
    pending = reserve_row_count(ctx);
    fa.host_count = pending->host_slot();
  }
  // zero-copy feed: what this launch reads over the host link (flockgpu_bytes_moved) -- the predicate column whole,
  // the pass-through columns once per survivor
  int64_t zc_bytes_per_survivor = 0;
  if (in.has_host_columns()) {
    if (cp.fast.kind != FAST_PRED_NONE && in.cols[cp.fast.col].chunks)
      ctx->h2d_bytes.fetch_add(in.num_rows * int64_t(in.cols[cp.fast.col].width()), std::memory_order_relaxed);
    for (const CompiledValue& v : vals)
      if (v.passthrough && in.cols[v.src_col].chunks) zc_bytes_per_survivor += in.cols[v.src_col].width();
    if (pending) pending->h2d_bytes_per_row = zc_bytes_per_survivor;
  }

  // computed outputs (eval_chain) are compiled only into the kernels that have them
  bool computed = false;
  for (int c = 0; c < fa.n_out; ++c) computed |= fa.outs[c].kind != OUT_PASS;
  auto launch = [&](const auto& pred) {
    using PredFn = std::decay_t<decltype(pred)>;
    const EarlyStart* e = may_start_early && !check_err ? &early : nullptr;  // check_err: a memset goes first
    if (computed) launch_filter<PredFn, true>(ctx, pred, fa, "filter_compact_kernel", e);
    else launch_filter<PredFn, false>(ctx, pred, fa, "filter_compact_kernel", e);
  };
  auto launch_i32 = [&](int64_t modulus) {
    const Column& pc = in.cols[cp.fast.col];
    const int32_t* col = static_cast<const int32_t*>(pc.values());
    const void* const* chunks = pc.chunks ? static_cast<const void* const*>(pc.chunks->table->ptr) : nullptr;
    const int32_t chunk_shift = pc.chunks ? pc.chunks->shift : 0;
    PredI32Consts k;
    const int mode = pred_i32_consts(modulus, cp.fast.cmp, cp.fast.rhs, &k);
    if (mode == 0) launch(PredI32<0>{col, k, chunks, chunk_shift});
    else if (mode == 1) launch(PredI32<1>{col, k, chunks, chunk_shift});
    else launch(PredI32<2>{col, k, chunks, chunk_shift});
  };
  switch (cp.fast.kind) {
    case FAST_PRED_I32_MOD_CMP:
      launch_i32(cp.fast.modulus);
      break;
    case FAST_PRED_I32_CMP:
      launch_i32(0);
      break;
    default: {
      const bool large = in.num_rows >= int64_t(ctx->sm_count) * 4 * FP_THREADS * 16;
      if (use_tree) {
        if (large) launch(PredTreeT<16>{tree_pred.prog});
        else launch(PredTreeT<4>{tree_pred.prog});
      } else if (large) {
        launch(PredGenericT<16>{cp.prog});
      } else {
        launch(PredGenericT<4>{cp.prog});
      }
    }
  }

  if (pending) {
    commit_row_count(pending);
    out->pending = pending;
    out->num_rows = -1;
    for (Column& c : out->cols) c.length = -1;
    return out;
  }
  unsigned long long scalars[9];
  read_scalars(ctx, 0, 9, scalars);
  if (check_err) FG_CHECK((scalars[8] & 0xffffffffull) == 0, FLOCKGPU_ERR_EXECUTION, "Divide by zero");
  int64_t n_sel = int64_t(scalars[0]);
  FG_CHECK(n_sel >= 0 && n_sel <= in.num_rows, FLOCKGPU_ERR_CUDA, "filter: corrupt survivor count %lld", (long long)n_sel);
  ctx->h2d_bytes.fetch_add(n_sel * zc_bytes_per_survivor, std::memory_order_relaxed);
  out->num_rows = n_sel;
  for (Column& c : out->cols) c.length = n_sel;
  if (!utf8_outs.empty()) {
    std::vector<const Column*> src;
    for (int i : utf8_outs) src.push_back(&in.cols[vals[i].src_col]);
    std::vector<Column> g = gather_columns(ctx, src, fa.sel_out, n_sel);  // one host round trip for all byte totals
    for (size_t u = 0; u < utf8_outs.size(); ++u) {
      g[u].name = out->cols[utf8_outs[u]].name;
      out->cols[utf8_outs[u]] = std::move(g[u]);
    }
  }
  return out;
}

TablePtr select_group_match_rows(const CtxPtr& ctx, const Table& in, int key_col, int val_col, const GroupMatchTable& t) {
  in.dense();
  if (in.num_rows == 0) return empty_like(ctx, in);
  FilterArgs fa{};
  fa.n_rows = in.num_rows;
  fa.out_count = ctx->d_scalars + 0;
  fa.err_flag = reinterpret_cast<int*>(ctx->d_scalars + 8);
  filter_colrefs(in, fa.cols);
  auto out = std::make_shared<Table>();
  out->ctx = ctx;
  out->metadata = in.metadata;
  std::vector<int> sel_outs;  // Utf8 columns and columns with validity bytes leave through the selection vector
  for (size_t i = 0; i < in.cols.size(); ++i) {
    const Column& s = in.cols[i];
    Column c;
    c.name = s.name;
    c.dtype = s.dtype;
    c.format = s.format;
    c.nullable = s.nullable;
    if (s.dtype == FLOCKGPU_UTF8 || s.validity) {
      sel_outs.push_back(int(i));
    } else {
      FG_CHECK(fa.n_out < MAX_OUT_COLS, FLOCKGPU_ERR_UNSUPPORTED, "join: more than %d fixed-width output columns", MAX_OUT_COLS);
      c.data = alloc(ctx, size_t(in.num_rows) * s.width());
      OutCol& oc = fa.outs[fa.n_out++];
      oc.kind = OUT_PASS;
      oc.src_col = int(i);
      oc.out_dtype = s.dtype;
      oc.width = s.width();
      oc.dst = c.data->ptr;
    }
    out->cols.push_back(std::move(c));
  }
  BufferPtr sel;
  if (!sel_outs.empty()) {
    sel = alloc(ctx, size_t(in.num_rows) * 4);
    fa.sel_out = sel->as<uint32_t>();
  }
  const Column& k = in.cols[key_col];
  const Column& v = in.cols[val_col];
  PredGroupMatch pred{static_cast<const uint32_t*>(k.values()), v.values(), k.valid(), v.valid(), v.width(), 0, t};
  launch_filter<PredGroupMatch, false>(ctx, pred, fa, "group_match_kernel");  // its own name in the launch profile
  unsigned long long n_sel = 0;
  read_scalars(ctx, 0, 1, &n_sel);
  FG_CHECK(int64_t(n_sel) <= in.num_rows, FLOCKGPU_ERR_CUDA, "join: corrupt survivor count %llu", n_sel);
  out->num_rows = int64_t(n_sel);
  for (Column& c : out->cols) c.length = out->num_rows;
  if (!sel_outs.empty()) {
    std::vector<const Column*> src;
    for (int i : sel_outs) src.push_back(&in.cols[i]);
    std::vector<Column> g = gather_columns(ctx, src, fa.sel_out, out->num_rows);
    for (size_t u = 0; u < sel_outs.size(); ++u) {
      g[u].name = out->cols[sel_outs[u]].name;
      out->cols[sel_outs[u]] = std::move(g[u]);
    }
  }
  return out;
}

}  // namespace fg

// ================================================================================================
using namespace fg;

extern "C" int flockgpu_filter_project(flockgpu_ctx* ctx, const flockgpu_table* in, const flockgpu_expr* predicate,
                                       const flockgpu_expr* projections, const char* const* out_names, int32_t n_projections,
                                       flockgpu_table** out) {
  return guarded([&] {
    auto c = core_of(ctx);
    FG_CHECK(out, FLOCKGPU_ERR_INVALID, "filter_project: null out pointer");
    FG_CHECK(in && in->table, FLOCKGPU_ERR_INVALID, "filter_project: null input table");
    FG_CHECK(n_projections >= 0 && (n_projections == 0 || projections), FLOCKGPU_ERR_INVALID, "filter_project: bad projection list");
    std::lock_guard<std::recursive_mutex> g(c->mu);
    FG_CUDA(cudaSetDevice(c->device));
    Expr pred;
    if (predicate) pred = tokens_to_expr(predicate);
    std::vector<Expr> projs;
    std::vector<std::string> names;
    for (int i = 0; i < n_projections; ++i) {
      projs.push_back(tokens_to_expr(&projections[i]));
      names.push_back(out_names && out_names[i] ? out_names[i] : "");
    }
    *out = wrap_table(filter_project(c, in->table, predicate ? &pred : nullptr, projs, names));
  });
}
