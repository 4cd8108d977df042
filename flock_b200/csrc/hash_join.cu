// hash_join.cu -- K3/K4: HashJoinExec { mode: Partitioned, join_type: Inner | Semi | Anti }.
//
// Reference operator (DataFusion fork, not in tree; used at flock/src/distributed_plan/planner.rs:169,
// :239 and serialised in flock/src/tests/data/plan/join.json): build a hash map over ALL left batches
// (hash -> row indices), then for every right batch emit (left_idx, right_idx) for each pair of equal
// keys and materialise `take(left columns) ++ take(right columns)`.  A key with a NULL or a NaN component
// never matches; duplicate keys on both sides give the full cross product.
//
// GPU design: an open-addressing table with ONE slot per DISTINCT build key -- the slot holds a
// representative build row (key equality is checked against the immutable build columns, so there is no
// publish race), the head of a linked list threading all build rows of that key (`next[row]`), and their
// count.  Heavily duplicated keys (NEXMark q5 joins 6.5 M (auction, num) rows on `num`, ~850 distinct
// values; q3's hot sellers) therefore cost one probe step, not one per duplicate.  The SMALLER input is
// the build side (the reference always builds on the left; which side is hashed is not observable).
//   join_build_kernel        claim / find the key's slot, push the row on its list
//   join_count_scan_kernel   per probe row: number of matches -> exclusive offsets (the grid-wide prefix
//                            protocol of compact.cuh, single pass) and the total pair count
//   join_emit_kernel         second walk (table lines are L2-hot) writes the (build, probe) index pairs
//   join_one_kernel          build side of ONE row (q5 / q7 join with a global aggregate): a stable equality
//                            compaction over the probe side, no table
//   semi_mark_kernel         Semi / Anti with the left side hashed: marks the slots the right rows find
//   semi_select_kernel       Semi / Anti: stable compaction of the left rows whose key is (Semi) / is not (Anti) matched
// and gather.cu materialises the output columns (Utf8 included).  The kernels are instantiated per key shape:
// one 4-byte key, one 8-byte key, or the general form (two packed columns / row comparison for Utf8 keys).
#include <algorithm>

#include "compact.cuh"
#include "device_utils.cuh"
#include "internal.h"
#include "rowkeys.cuh"

namespace fg {

constexpr unsigned JOIN_EMPTY = ~0u;

struct JoinSide {
  int64_t n_rows;
  int32_t packed;
  int32_t pad;
  const void* key0;  // the key column when the join has ONE fixed-width key (kernels instantiated with KW = 4 / 8)
  int32_t n_null_cols;  // key columns that carry validity bytes: a row with a NULL key matches nothing (NULL != NULL)
  int32_t n_nan_cols;   // Float64 key columns: a row with a NaN key matches nothing (NaN != NaN)
  const uint8_t* key_valid[MAX_KEY_COLS];
  const double* key_f64[MAX_KEY_COLS];
  KeyPack pack;
  RowKeys rk;
  ColRef cols[MAX_IN_COLS];
};

struct JoinTable {
  unsigned* rep;           // [cap] representative build row of the slot's key, JOIN_EMPTY = free
  unsigned* head;          // [cap] most recently pushed build row of that key
  unsigned* cnt;           // [cap] number of build rows with that key
  unsigned* next;          // [build rows] next build row with the same key, JOIN_EMPTY = end
  unsigned long long cap;  // power of two
  struct JoinSlot* slots;  // KW = 4: the table proper (below); rep / head / cnt are unused, `next` holds row + 1
};

// One 4-byte key (every NEXMark join but q5's): the KEY LIVES IN THE SLOT.  A probe is one 16-byte load -- key, list
// head and count arrive together -- where the representative-row table needs three dependent reads (rep[slot], the
// build key column at that row, cnt[slot]) in three cache lines; the build claims a slot with one CAS that returns the
// resident key.  The representative-row kernels spend most of their time stalled on those dependent loads.  All-zero = empty, so the table is
// initialised by one memset: `tag_key` carries an occupied bit above the key, `head` and next[] hold row + 1.
struct __align__(16) JoinSlot {
  unsigned long long tag_key;  // 0 = free, else (1 << 63) | key
  unsigned head;               // most recently pushed build row + 1
  unsigned cnt;                // build rows with this key
};
constexpr unsigned long long JOIN_TAG = 1ull << 63;
// Capacity stays a power of two >= 2 x build rows (load 0.3 - 0.5).  A table at load 0.6 of any capacity (slot = high
// half of hash x capacity: half the footprint for q8's 2.5 M persons) was measured and is SLOWER: linear probing at that load makes 2-3 x the dependent accesses, and
// those, not the table's footprint, are what the kernels wait for.
// KW = 4 / 8: one fixed-width key column, read straight from JoinSide::key0 (every NEXMark join); KW = 0: the general
// form (two packed columns, or row comparison for Utf8 / wide keys).  The general form cost ~140 lane-instructions per
// probe row on q5 (dynamic indexing of the column table in parameter space, width and mode branches).
// A key with a NULL or a NaN component equals no key, its own included: such a row never enters the table and never
// probes.  Past those two, Float64 components compare by bit pattern (-0.0 != +0.0, +inf == +inf), as DataFusion's
// hash-then-compare does.  A join without Float64 keys has n_nan_cols = 0 and runs the NULL test alone.
__device__ __forceinline__ bool key_matches_nothing(const JoinSide& s, int64_t row) {
  for (int i = 0; i < s.n_null_cols; ++i)
    if (!s.key_valid[i][row]) return true;
  for (int i = 0; i < s.n_nan_cols; ++i)
    if (isnan(s.key_f64[i][row])) return true;
  return false;
}

template <int KW>
__device__ __forceinline__ unsigned long long side_hash(const JoinSide& s, int64_t row, unsigned long long* key) {
  if (KW == 4) {
    *key = static_cast<const uint32_t*>(s.key0)[row];
    return fmix64(*key);
  }
  if (KW == 8) {
    *key = static_cast<const unsigned long long*>(s.key0)[row];
    return fmix64(*key);
  }
  if (s.packed) {
    *key = pack_key(s.pack, s.cols, row);
    return fmix64(*key);
  }
  *key = 0;
  return hash_row(s.rk, s.cols, row);
}

// Does build row `r` carry the key (`key` / row `row` of side `other`)?
template <int KW>
__device__ __forceinline__ bool build_row_matches(const JoinSide& build, unsigned r, const JoinSide& other, int64_t row, unsigned long long key) {
  if (KW == 4) return static_cast<const uint32_t*>(build.key0)[r] == uint32_t(key);
  if (KW == 8) return static_cast<const unsigned long long*>(build.key0)[r] == key;
  return build.packed ? pack_key(build.pack, build.cols, int64_t(r)) == key : rows_equal(build.rk, build.cols, int64_t(r), other.rk, other.cols, row);
}

template <int KW>
__global__ void __launch_bounds__(256) join_build_kernel(const __grid_constant__ JoinSide build, const JoinTable t) {
  for (int64_t row = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; row < build.n_rows; row += int64_t(gridDim.x) * blockDim.x) {
    if (key_matches_nothing(build, row)) continue;  // never enters the table: nothing can match it
    unsigned long long key;
    unsigned long long slot = side_hash<KW>(build, row, &key) & (t.cap - 1);
    if (KW == 4) {
      const unsigned long long want = JOIN_TAG | key;
      while (true) {
        unsigned long long cur = t.slots[slot].tag_key;
        if (cur == 0ull) cur = atomicCAS(&t.slots[slot].tag_key, 0ull, want);
        if (cur == 0ull || cur == want) break;
        slot = (slot + 1) & (t.cap - 1);
      }
      t.next[row] = atomicExch(&t.slots[slot].head, unsigned(row) + 1u);
      atomicAdd(&t.slots[slot].cnt, 1u);
      continue;
    }
    while (true) {
      unsigned r = t.rep[slot];
      if (r == JOIN_EMPTY) {
        r = atomicCAS(&t.rep[slot], JOIN_EMPTY, unsigned(row));
        if (r == JOIN_EMPTY) break;  // claimed: this row represents the key
      }
      if (build_row_matches<KW>(build, r, build, row, key)) break;
      slot = (slot + 1) & (t.cap - 1);
    }
    t.next[row] = atomicExch(&t.head[slot], unsigned(row));
    atomicAdd(&t.cnt[slot], 1u);
  }
}

// Slot of the key of probe row `row`, or ~0 when no build row has it.
// (KW = 4: *head receives the list head (row + 1) and *cnt the number of build rows of the key, from the same load)
template <int KW>
__device__ __forceinline__ unsigned long long find_slot(const JoinSide& build, const JoinSide& probe, const JoinTable& t, int64_t row, unsigned* head,
                                                        unsigned* cnt) {
  if (key_matches_nothing(probe, row)) return ~0ull;
  unsigned long long key;
  unsigned long long slot = side_hash<KW>(probe, row, &key) & (t.cap - 1);
  if (KW == 4) {
    const unsigned long long want = JOIN_TAG | key;
    while (true) {
      const uint4 s = *reinterpret_cast<const uint4*>(&t.slots[slot]);
      const unsigned long long tag = ((unsigned long long)s.y << 32) | s.x;
      if (tag == 0ull) return ~0ull;
      if (tag == want) {
        *head = s.z;
        *cnt = s.w;
        return slot;
      }
      slot = (slot + 1) & (t.cap - 1);
    }
  }
  while (true) {
    const unsigned r = t.rep[slot];
    if (r == JOIN_EMPTY) return ~0ull;
    if (build_row_matches<KW>(build, r, probe, row, key)) return slot;
    slot = (slot + 1) & (t.cap - 1);
  }
}

constexpr int JC_THREADS = 256;
constexpr int JC_ITEMS = 4;
constexpr int JC_TILE = JC_THREADS * JC_ITEMS;

struct JoinCountArgs {
  JoinSide build, probe;
  JoinTable table;
  unsigned* out_off;  // [probe rows + 1] exclusive pair offsets
  CompactScratch sc;  // grid-wide exclusive prefix of the tiles' pair counts (compact.cuh); sc.out_count = total pairs
};

template <int KW>
__global__ void __launch_bounds__(JC_THREADS) join_count_scan_kernel(const __grid_constant__ JoinCountArgs a) {
  __shared__ CompactSmem<1, 16> sm;
  __shared__ unsigned long long s_warp[JC_THREADS / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t n = a.probe.n_rows;
  long long tile;
  for (int it = 0; (tile = cp_next_tile(sm, a.sc, it)) >= 0; ++it) {
    const int64_t i0 = tile * JC_TILE + int64_t(tid) * JC_ITEMS;
    unsigned cnt[JC_ITEMS];
    unsigned long long local = 0;
#pragma unroll
    for (int k = 0; k < JC_ITEMS; ++k) {
      unsigned c = 0;
      if (i0 + k < n) {
        unsigned head = 0, in_slot = 0;
        const unsigned long long slot = find_slot<KW>(a.build, a.probe, a.table, i0 + k, &head, &in_slot);
        if (slot != ~0ull) c = KW == 4 ? in_slot : a.table.cnt[slot];
      }
      cnt[k] = c;
      local += c;
    }
    unsigned long long incl = warp_inclusive_sum(local);
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    unsigned long long warp_base = 0, tile_total = 0;
#pragma unroll
    for (int w = 0; w < JC_THREADS / 32; ++w) {
      unsigned long long v = s_warp[w];
      if (w < warp) warp_base += v;
      tile_total += v;
    }
    // exclusive prefix over the tiles: the whole CTA looks back (256 predecessors per step) or, when every tile is
    // resident, reads its predecessors' self-validating count words
    if (a.sc.single_wave) cp_grid_prefix(sm, a.sc, tile, tile_total);
    else cp_block_lookback(sm, a.sc, tile, tile_total);
    unsigned long long run = sm.excl + warp_base + (incl - local);
#pragma unroll
    for (int k = 0; k < JC_ITEMS; ++k) {
      if (i0 + k < n) a.out_off[i0 + k] = unsigned(run);
      run += cnt[k];
    }
    if (tile == a.sc.num_tiles - 1 && tid == 0) a.out_off[n] = unsigned(sm.excl + tile_total);
    __syncthreads();  // sm / s_warp are reused by the next tile
  }
}

// ---- build side of ONE row (NEXMark q5 / q7 join a relation with a global aggregate): no table, no chains -- the
// probe is an equality filter.  One stable compaction pass writes the matching probe rows; every pair's build row is 0.
struct JoinOneArgs {
  CompactScratch sc;
  const void* probe_key;
  const void* build_key;  // device pointer to the single build key
  int64_t n_rows;
  unsigned* probe_idx;
};

template <int KW>
__global__ void __launch_bounds__(CP_THREADS) join_one_kernel(const __grid_constant__ JoinOneArgs a) {
  constexpr int E = 4, I = 16, G = I / E;
  constexpr int TILE = CP_THREADS * I;
  __shared__ CompactSmem<E, I> sm;
  const int tid = threadIdx.x, warp = tid >> 5;
  const unsigned long long want = KW == 4 ? (unsigned long long)*static_cast<const uint32_t*>(a.build_key) : *static_cast<const unsigned long long*>(a.build_key);
  long long tile;
  for (int it = 0; (tile = cp_next_tile(sm, a.sc, it)) >= 0; ++it) {
    const int64_t tile_base = tile * TILE;
    unsigned long long bits = 0;
#pragma unroll
    for (int g = 0; g < G; ++g) {
      const int64_t r0 = tile_base + (int64_t(g) * CP_THREADS + tid) * E;
      unsigned nib = 0;
      if (r0 + 3 < a.n_rows) {
        if (KW == 4) {
          const uint4 k = *reinterpret_cast<const uint4*>(static_cast<const uint32_t*>(a.probe_key) + r0);
          nib = unsigned(k.x == uint32_t(want)) | (unsigned(k.y == uint32_t(want)) << 1) | (unsigned(k.z == uint32_t(want)) << 2) | (unsigned(k.w == uint32_t(want)) << 3);
        } else {
          const unsigned long long* p = static_cast<const unsigned long long*>(a.probe_key) + r0;
          const ulonglong2 k01 = *reinterpret_cast<const ulonglong2*>(p), k23 = *reinterpret_cast<const ulonglong2*>(p + 2);
          nib = unsigned(k01.x == want) | (unsigned(k01.y == want) << 1) | (unsigned(k23.x == want) << 2) | (unsigned(k23.y == want) << 3);
        }
      } else {
        for (int e = 0; e < E; ++e) {
          if (r0 + e >= a.n_rows) break;
          const unsigned long long k = KW == 4 ? (unsigned long long)static_cast<const uint32_t*>(a.probe_key)[r0 + e]
                                               : static_cast<const unsigned long long*>(a.probe_key)[r0 + e];
          nib |= unsigned(k == want) << e;
        }
      }
      bits |= (unsigned long long)nib << (g * E);
    }
    unsigned lane_prefix[G];
    cp_rank_tile<E, I>(sm, a.sc, tile, bits, lane_prefix);
    if (bits && sm.tile_total) {
#pragma unroll
      for (int g = 0; g < G; ++g) {
        const unsigned nib = unsigned(bits >> (g * E)) & 0xfu;
        if (!nib) continue;
        const int64_t r0 = tile_base + (int64_t(g) * CP_THREADS + tid) * E;
        const int64_t pos0 = int64_t(sm.excl) + sm.group_warp[g][warp] + lane_prefix[g];
#pragma unroll
        for (int e = 0; e < E; ++e)
          if ((nib >> e) & 1u) a.probe_idx[pos0 + __popc(nib & ((1u << e) - 1u))] = unsigned(r0 + e);
      }
    }
    __syncthreads();
  }
}

struct JoinEmitArgs {
  JoinSide build, probe;
  JoinTable table;
  const unsigned* off;
  unsigned* build_idx;
  unsigned* probe_idx;
};

template <int KW>
__global__ void __launch_bounds__(256) join_emit_kernel(const __grid_constant__ JoinEmitArgs a) {
  for (int64_t row = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; row < a.probe.n_rows; row += int64_t(gridDim.x) * blockDim.x) {
    unsigned pos = a.off[row];
    if (a.off[row + 1] == pos) continue;
    unsigned head = 0, in_slot = 0;
    const unsigned long long slot = find_slot<KW>(a.build, a.probe, a.table, row, &head, &in_slot);
    if (KW == 4) {
      for (unsigned r1 = head; r1 != 0u; r1 = a.table.next[r1 - 1u]) {  // row + 1 links, 0 ends the list
        a.build_idx[pos] = r1 - 1u;
        a.probe_idx[pos] = unsigned(row);
        ++pos;
      }
      continue;
    }
    for (unsigned r = a.table.head[slot]; r != JOIN_EMPTY; r = a.table.next[r]) {
      a.build_idx[pos] = r;
      a.probe_idx[pos] = unsigned(row);
      ++pos;
    }
  }
}

// ---- Semi / Anti: the left rows whose key tuple does (Semi) or does not (Anti) occur on the right, each at most once,
// in left order.  The smaller side is hashed, as for the inner join; either way one stable compaction over the left rows
// (compact.cuh) writes the kept rows' indices.  A row is "matched" when
//   right side built: its key has a slot in the table;
//   left side built:  its key's slot was marked by semi_mark_kernel (some right row probed it).  The left row finds its
//                     slot again by a re-probe of its own key: the table lines are L2-hot, and the build kernel stays
//                     the inner join's.
// A left row with a NULL / NaN key component has no slot (find_slot), so it is never matched: out of Semi, in Anti.
struct SemiMarkArgs {
  JoinSide build, probe;  // build = the left side, probe = the right side
  JoinTable table;
  unsigned char* marked;  // [table.cap] 1 = a right row has the slot's key
};

template <int KW>
__global__ void __launch_bounds__(256) semi_mark_kernel(const __grid_constant__ SemiMarkArgs a) {
  for (int64_t row = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; row < a.probe.n_rows; row += int64_t(gridDim.x) * blockDim.x) {
    unsigned head = 0, in_slot = 0;
    const unsigned long long slot = find_slot<KW>(a.build, a.probe, a.table, row, &head, &in_slot);
    if (slot != ~0ull) a.marked[slot] = 1;  // every writer stores the same value: no atomic needed
  }
}

struct SemiSelectArgs {
  JoinSide build, left;          // build: the hashed side (the left side itself when `marked` is set)
  JoinTable table;
  const unsigned char* marked;   // left side built: semi_mark_kernel's bytes; nullptr: right side built
  int keep_matched;              // 1 Semi, 0 Anti
  CompactScratch sc;
  unsigned* out_idx;             // the kept left rows, ascending
};

template <int KW>
__global__ void __launch_bounds__(CP_THREADS) semi_select_kernel(const __grid_constant__ SemiSelectArgs a) {
  constexpr int E = 4, I = 16, G = I / E;
  constexpr int TILE = CP_THREADS * I;
  __shared__ CompactSmem<E, I> sm;
  const int tid = threadIdx.x, warp = tid >> 5;
  const int64_t n = a.left.n_rows;
  long long tile;
  for (int it = 0; (tile = cp_next_tile(sm, a.sc, it)) >= 0; ++it) {
    const int64_t tile_base = tile * TILE;
    unsigned long long bits = 0;
#pragma unroll 1
    for (int k = 0; k < I; ++k) {
      const int64_t row = tile_base + cp_item_index<E>(k, tid);
      if (row >= n) continue;
      unsigned head = 0, in_slot = 0;
      const unsigned long long slot = find_slot<KW>(a.build, a.left, a.table, row, &head, &in_slot);
      const bool matched = slot != ~0ull && (!a.marked || a.marked[slot]);
      bits |= (unsigned long long)(int(matched) == a.keep_matched) << k;
    }
    unsigned lane_prefix[G];
    cp_rank_tile<E, I>(sm, a.sc, tile, bits, lane_prefix);
    if (bits && sm.tile_total) {
#pragma unroll
      for (int g = 0; g < G; ++g) {
        const unsigned nib = unsigned(bits >> (g * E)) & 0xfu;
        if (!nib) continue;
        const int64_t r0 = tile_base + (int64_t(g) * CP_THREADS + tid) * E;
        const int64_t pos0 = int64_t(sm.excl) + sm.group_warp[g][warp] + lane_prefix[g];
#pragma unroll
        for (int e = 0; e < E; ++e)
          if ((nib >> e) & 1u) a.out_idx[pos0 + __popc(nib & ((1u << e) - 1u))] = unsigned(r0 + e);
      }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------
// The kernels read the key columns only, so a side carries those alone: key i in slot i.  The other columns of the side,
// however many, reach the output through gather_columns.
static void fill_side(const Table& t, const std::vector<int>& keys, bool packed, JoinSide* s) {
  s->n_rows = t.num_rows;
  s->packed = packed ? 1 : 0;
  s->rk.n = int(keys.size());
  s->n_null_cols = 0;
  s->n_nan_cols = 0;
  for (size_t i = 0; i < keys.size(); ++i) {
    const Column& c = t.cols[keys[i]];
    s->cols[i].data = c.values();
    s->cols[i].offsets = c.offs();
    s->cols[i].dtype = c.dtype;
    s->cols[i].chunk_shift = 0;
    s->cols[i].chunks = nullptr;
    s->cols[i].validity = nullptr;  // key equality between the sides is value equality: rows with NULL keys are skipped up front
    s->rk.col[i] = int(i);
    if (c.validity) s->key_valid[s->n_null_cols++] = c.valid();
    if (c.dtype == FLOCKGPU_FLOAT64) s->key_f64[s->n_nan_cols++] = static_cast<const double*>(c.values());
  }
  if (packed) {
    s->pack.n = int(keys.size());
    for (size_t i = 0; i < keys.size(); ++i) {
      s->pack.col[i] = int(i);
      s->pack.width[i] = t.cols[keys[i]].width();
    }
  }
}

static int grid_for(const CtxPtr& ctx, int64_t items, int threads, int per_sm) {
  return int(std::max<int64_t>(1, std::min<int64_t>((items + threads - 1) / threads, int64_t(ctx->sm_count) * per_sm)));
}

// Every join type accepts and refuses the same key lists.
static void check_join_keys(const Table& L, const Table& R, const std::vector<int>& left_keys, const std::vector<int>& right_keys) {
  FG_CHECK(!left_keys.empty() && left_keys.size() == right_keys.size(), FLOCKGPU_ERR_INVALID, "hash_join: key lists must be non-empty and of equal length");
  FG_CHECK(left_keys.size() <= size_t(MAX_KEY_COLS), FLOCKGPU_ERR_UNSUPPORTED, "hash_join: more than %d key columns", MAX_KEY_COLS);
  for (size_t i = 0; i < left_keys.size(); ++i) {
    const int lk = left_keys[i], rk = right_keys[i];
    FG_CHECK(lk >= 0 && lk < int(L.cols.size()) && rk >= 0 && rk < int(R.cols.size()), FLOCKGPU_ERR_INVALID, "hash_join: key column out of range");
    check_join_key_types("hash_join", L.cols[lk], R.cols[rk]);
  }
}

// kernel flavour: one fixed-width key column (KW = 4 / 8) or the general form (KW = 0)
template <class F>
static void by_width(int kw, F&& f) {
  if (kw == 4) f(std::integral_constant<int, 4>{});
  else if (kw == 8) f(std::integral_constant<int, 8>{});
  else f(std::integral_constant<int, 0>{});
}

// The open-addressing table over the `bs.n_rows` rows of the build side, filled by join_build_kernel; *tbuf owns it.
static JoinTable build_join_table(const CtxPtr& ctx, const JoinSide& bs, int kw, BufferPtr* tbuf) {
  unsigned long long cap = 1024;
  while (cap < 2ull * (unsigned long long)bs.n_rows) cap <<= 1;
  JoinTable tab{};
  if (kw == 4) {
    // 16-byte slots (key, head, count), all-zero = empty, then next[build rows]
    *tbuf = alloc(ctx, size_t(cap) * sizeof(JoinSlot) + size_t(bs.n_rows) * 4);
    FG_CUDA(cudaMemsetAsync((*tbuf)->ptr, 0, size_t(cap) * sizeof(JoinSlot), ctx->stream));
    tab.slots = (*tbuf)->as<JoinSlot>();
    tab.next = reinterpret_cast<unsigned*>(tab.slots + cap);
    tab.cap = cap;
  } else {
    // rep | head | cnt in one allocation (cap words each), then next[build rows]
    *tbuf = alloc(ctx, size_t(cap) * 12 + size_t(bs.n_rows) * 4);
    FG_CUDA(cudaMemsetAsync((*tbuf)->ptr, 0xff, size_t(cap) * 8, ctx->stream));                                  // rep, head = EMPTY
    FG_CUDA(cudaMemsetAsync(static_cast<char*>((*tbuf)->ptr) + size_t(cap) * 8, 0, size_t(cap) * 4, ctx->stream));  // cnt = 0
    unsigned* w = (*tbuf)->as<unsigned>();
    tab = JoinTable{w, w + cap, w + 2 * cap, w + 3 * cap, cap, nullptr};
  }
  {
    LaunchTimer lt(ctx, "join_build_kernel");
    by_width(kw, [&](auto w) { join_build_kernel<decltype(w)::value><<<grid_for(ctx, bs.n_rows, 256, 8), 256, 0, ctx->stream>>>(bs, tab); });
  }
  FG_CUDA(cudaGetLastError());
  count_launch(ctx);
  return tab;
}

TablePtr hash_join(const CtxPtr& ctx, const TablePtr& left_ptr, const TablePtr& right_ptr, const std::vector<int>& left_keys,
                   const std::vector<int>& right_keys) {
  const Table& L = *left_ptr;
  const Table& R = *right_ptr;
  // the key columns are checked before any fast path, so every path accepts and refuses the same joins
  check_join_keys(L, R, left_keys, right_keys);
  // one side is a single row and the other a group-by result still in table form (NEXMark q5: num = MAX(num)):
  // an equality selection over the table, no rows are materialised for the join
  if (left_keys.size() == 1 && right_keys.size() == 1) {
    if (std::shared_ptr<DeferredTable> d = left_ptr->deferred)
      if (TablePtr t = d->select_equal(L, left_keys[0], right_ptr, right_keys[0], true)) return t;
    if (std::shared_ptr<DeferredTable> d = right_ptr->deferred)
      if (TablePtr t = d->select_equal(R, right_keys[0], left_ptr, left_keys[0], false)) return t;
  }
  // one side is a (key, MIN / MAX) group-by still in its direct-address table and the join is on (key, MIN / MAX)
  // (NEXMark q9: bids back to each auction's top price): one selection over the other side, no hash table
  if (left_keys.size() == 2 && right_keys.size() == 2) {
    const int lk[2] = {left_keys[0], left_keys[1]}, rk[2] = {right_keys[0], right_keys[1]};
    if (std::shared_ptr<DeferredTable> d = right_ptr->deferred)
      if (TablePtr t = d->select_group_match(R, rk, left_ptr, lk, false)) return t;
    if (std::shared_ptr<DeferredTable> d = left_ptr->deferred)
      if (TablePtr t = d->select_group_match(L, lk, right_ptr, rk, true)) return t;
  }
  L.dense();
  R.dense();
  std::vector<int> widths;
  for (int lk : left_keys) widths.push_back(L.cols[lk].width());
  const bool packed = keys_packable(widths.data(), int(widths.size()));

  auto out = std::make_shared<Table>();
  out->ctx = ctx;
  out->metadata = L.metadata;

  // a NULL key column (one-row global aggregate over empty input) matches nothing
  bool null_key = false;
  for (size_t i = 0; i < left_keys.size(); ++i) null_key |= L.cols[left_keys[i]].all_null || R.cols[right_keys[i]].all_null;

  int64_t n_pairs = 0;
  BufferPtr build_idx, probe_idx;
  // hash the smaller input, stream the larger one through it
  const bool swap_sides = R.num_rows < L.num_rows;
  const Table& B = swap_sides ? R : L;
  const Table& P = swap_sides ? L : R;
  if (L.num_rows > 0 && R.num_rows > 0 && !null_key) {
    JoinSide bs{}, ps{};
    fill_side(B, swap_sides ? right_keys : left_keys, packed, &bs);
    fill_side(P, swap_sides ? left_keys : right_keys, packed, &ps);
    // kernel flavour: one fixed-width key column (4 / 8 bytes) or the general form
    const int kw = (packed && widths.size() == 1) ? widths[0] : 0;
    if (kw) {
      bs.key0 = B.cols[(swap_sides ? right_keys : left_keys)[0]].values();
      ps.key0 = P.cols[(swap_sides ? left_keys : right_keys)[0]].values();
    }
    if (kw && B.num_rows == 1 && bs.n_null_cols == 0 && ps.n_null_cols == 0 && ps.n_nan_cols == 0) {
      // one build row: equality filter over the probe side (see join_one_kernel), which compares bits only -- NULL and
      // NaN keys (a Float64 key column) take the table path, which skips them
      probe_idx = alloc(ctx, size_t(P.num_rows) * 4);
      JoinOneArgs oa{};
      oa.probe_key = ps.key0;
      oa.build_key = bs.key0;
      oa.n_rows = P.num_rows;
      oa.probe_idx = probe_idx->as<unsigned>();
      const int64_t num_tiles = (P.num_rows + CP_THREADS * 16 - 1) / (CP_THREADS * 16);
      by_width(kw, [&](auto w) {
        constexpr int KW = decltype(w)::value == 8 ? 8 : 4;
        auto kernel = join_one_kernel<KW>;
        oa.sc = prepare_compact(ctx, num_tiles, resident_ctas(ctx, reinterpret_cast<const void*>(kernel), CP_THREADS), ctx->d_scalars + 4);
        LaunchTimer lt(ctx, "join_one_kernel");
        launch_compact(ctx, kernel, oa.sc, oa);
      });
      FG_CUDA(cudaGetLastError());
      count_launch(ctx);
      unsigned long long total = 0;
      read_scalars(ctx, 4, 1, &total);
      FG_CHECK(total <= (unsigned long long)P.num_rows, FLOCKGPU_ERR_CUDA, "hash_join: corrupt match count");
      n_pairs = int64_t(total);
      if (n_pairs > 0) {
        build_idx = alloc(ctx, size_t(n_pairs) * 4);
        FG_CUDA(cudaMemsetAsync(build_idx->ptr, 0, size_t(n_pairs) * 4, ctx->stream));
      }
    } else {
    BufferPtr tbuf;
    const JoinTable tab = build_join_table(ctx, bs, kw, &tbuf);

    BufferPtr off = alloc(ctx, size_t(P.num_rows + 1) * 4);
    JoinCountArgs ca{};
    ca.build = bs;
    ca.probe = ps;
    ca.table = tab;
    ca.out_off = off->as<unsigned>();
    const int64_t num_tiles = (P.num_rows + JC_TILE - 1) / JC_TILE;
    by_width(kw, [&](auto w) {
      auto kernel = join_count_scan_kernel<decltype(w)::value>;
      ca.sc = prepare_compact(ctx, num_tiles, resident_ctas(ctx, reinterpret_cast<const void*>(kernel), JC_THREADS), ctx->d_scalars + 4);
      LaunchTimer lt(ctx, "join_count_scan_kernel");
      launch_compact(ctx, kernel, ca.sc, ca);
    });
    FG_CUDA(cudaGetLastError());
    count_launch(ctx);
    unsigned long long total = 0;
    read_scalars(ctx, 4, 1, &total);
    FG_CHECK(total < (1ull << 32) - 1, FLOCKGPU_ERR_UNSUPPORTED, "hash_join: %llu output rows exceed 2^32-2", total);
    n_pairs = int64_t(total);
    if (n_pairs > 0) {
      build_idx = alloc(ctx, size_t(n_pairs) * 4);
      probe_idx = alloc(ctx, size_t(n_pairs) * 4);
      JoinEmitArgs ea{};
      ea.build = bs;
      ea.probe = ps;
      ea.table = tab;
      ea.off = off->as<unsigned>();
      ea.build_idx = build_idx->as<unsigned>();
      ea.probe_idx = probe_idx->as<unsigned>();
      {
        LaunchTimer lt(ctx, "join_emit_kernel");
        by_width(kw, [&](auto w) { join_emit_kernel<decltype(w)::value><<<grid_for(ctx, P.num_rows, 256, 8), 256, 0, ctx->stream>>>(ea); });
      }
      FG_CUDA(cudaGetLastError());
      count_launch(ctx);
    }
    }  // general build / probe
  }
  out->num_rows = n_pairs;
  if (n_pairs == 0) {
    TablePtr le = empty_like(ctx, L), re = empty_like(ctx, R);
    for (const Column& c : le->cols) out->cols.push_back(c);
    for (const Column& c : re->cols) out->cols.push_back(c);
    return out;
  }
  // output schema is always left ++ right, whichever side was hashed
  const uint32_t* l_idx = (swap_sides ? probe_idx : build_idx)->as<uint32_t>();
  const uint32_t* r_idx = (swap_sides ? build_idx : probe_idx)->as<uint32_t>();
  std::vector<const Column*> lsrc, rsrc;
  for (const Column& c : L.cols) lsrc.push_back(&c);
  for (const Column& c : R.cols) rsrc.push_back(&c);
  for (Column& c : gather_columns(ctx, lsrc, l_idx, n_pairs)) out->cols.push_back(std::move(c));
  for (Column& c : gather_columns(ctx, rsrc, r_idx, n_pairs)) out->cols.push_back(std::move(c));
  return out;
}

TablePtr hash_semi_join(const CtxPtr& ctx, const TablePtr& left_ptr, const TablePtr& right_ptr, const std::vector<int>& left_keys,
                        const std::vector<int>& right_keys, bool anti) {
  const Table& L = *left_ptr;
  const Table& R = *right_ptr;
  check_join_keys(L, R, left_keys, right_keys);
  L.dense();
  R.dense();
  // a NULL key column (one-row global aggregate over empty input) matches nothing
  bool null_key = false;
  for (size_t i = 0; i < left_keys.size(); ++i) null_key |= L.cols[left_keys[i]].all_null || R.cols[right_keys[i]].all_null;
  // the output is a subset of the left rows in their order: all of them is the left input itself, rows and routing
  if (L.num_rows == 0) return left_ptr;
  if (R.num_rows == 0 || null_key) return anti ? left_ptr : empty_like(ctx, L);

  std::vector<int> widths;
  for (int lk : left_keys) widths.push_back(L.cols[lk].width());
  const bool packed = keys_packable(widths.data(), int(widths.size()));
  const int kw = (packed && widths.size() == 1) ? widths[0] : 0;
  JoinSide ls{}, rs{};
  fill_side(L, left_keys, packed, &ls);
  fill_side(R, right_keys, packed, &rs);
  if (kw) {
    ls.key0 = L.cols[left_keys[0]].values();
    rs.key0 = R.cols[right_keys[0]].values();
  }
  // hash the smaller input, as the inner join does
  const bool build_left = L.num_rows <= R.num_rows;
  BufferPtr tbuf, marked;
  const JoinTable tab = build_join_table(ctx, build_left ? ls : rs, kw, &tbuf);
  if (build_left) {
    marked = alloc(ctx, size_t(tab.cap));
    FG_CUDA(cudaMemsetAsync(marked->ptr, 0, size_t(tab.cap), ctx->stream));
    SemiMarkArgs ma{ls, rs, tab, marked->as<unsigned char>()};
    {
      LaunchTimer lt(ctx, "semi_mark_kernel");
      by_width(kw, [&](auto w) { semi_mark_kernel<decltype(w)::value><<<grid_for(ctx, R.num_rows, 256, 8), 256, 0, ctx->stream>>>(ma); });
    }
    FG_CUDA(cudaGetLastError());
    count_launch(ctx);
  }
  BufferPtr idx = alloc(ctx, size_t(L.num_rows) * 4);
  SemiSelectArgs sa{};
  sa.build = build_left ? ls : rs;
  sa.left = ls;
  sa.table = tab;
  sa.marked = build_left ? marked->as<unsigned char>() : nullptr;
  sa.keep_matched = anti ? 0 : 1;
  sa.out_idx = idx->as<unsigned>();
  const int64_t num_tiles = (L.num_rows + CP_THREADS * 16 - 1) / (CP_THREADS * 16);
  by_width(kw, [&](auto w) {
    auto kernel = semi_select_kernel<decltype(w)::value>;
    sa.sc = prepare_compact(ctx, num_tiles, resident_ctas(ctx, reinterpret_cast<const void*>(kernel), CP_THREADS), ctx->d_scalars + 4);
    LaunchTimer lt(ctx, "semi_select_kernel");
    launch_compact(ctx, kernel, sa.sc, sa);
  });
  FG_CUDA(cudaGetLastError());
  count_launch(ctx);
  unsigned long long total = 0;
  read_scalars(ctx, 4, 1, &total);
  FG_CHECK(total <= (unsigned long long)L.num_rows, FLOCKGPU_ERR_CUDA, "hash_join: corrupt semi / anti row count");
  if (total == (unsigned long long)L.num_rows) return left_ptr;
  if (total == 0) return empty_like(ctx, L);
  auto out = std::make_shared<Table>();
  out->ctx = ctx;
  out->metadata = L.metadata;
  out->num_rows = int64_t(total);
  // the kept rows stay on the rank they were routed to
  out->partitioned_on = L.partitioned_on;
  out->partition_world = L.partition_world;
  std::vector<const Column*> src;
  for (const Column& c : L.cols) src.push_back(&c);
  out->cols = gather_columns(ctx, src, idx->as<uint32_t>(), out->num_rows);
  return out;
}

}  // namespace fg

using namespace fg;

extern "C" int flockgpu_hash_join(flockgpu_ctx* ctx, const flockgpu_table* left, const flockgpu_table* right, const int32_t* left_keys,
                                  const int32_t* right_keys, int32_t n_keys, flockgpu_table** out) {
  return guarded([&] {
    auto c = core_of(ctx);
    FG_CHECK(out && left && left->table && right && right->table && left_keys && right_keys && n_keys > 0, FLOCKGPU_ERR_INVALID,
             "hash_join: null or empty argument");
    std::lock_guard<std::recursive_mutex> g(c->mu);
    FG_CUDA(cudaSetDevice(c->device));
    std::vector<int> lk(left_keys, left_keys + n_keys), rk(right_keys, right_keys + n_keys);
    *out = wrap_table(hash_join(c, left->table, right->table, lk, rk));
  });
}
