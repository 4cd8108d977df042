// compact.cuh -- the single-pass stable compaction / scan skeleton shared by FilterExec (filter_project.cu), the
// hash-table emitter (hash_agg.cu), the partition selector (partition.cu), the join's pair-count scan and
// one-row-build probe (hash_join.cu) and the Utf8 length scan (gather.cu).
//
// A CTA processes tiles of CP_THREADS x I items.  For each tile it gets one bit per item ("survives"), ranks the
// survivors in item order (packed SWAR scan for four-item groups, ballots otherwise), obtains the tile's global
// output offset and hands every survivor its output position.  Three ways to get that offset:
//
//   single wave   (tiles <= resident CTAs; cooperative launch, tile = blockIdx.x):
//                 every tile needs the counts of ALL its predecessors and they all finish counting at about the same
//                 time, so a chained look-back degenerates into everybody polling everybody (the largest share of
//                 the kernel's stall samples).  Instead each CTA publishes one self-validating word
//                 {launch epoch, count}, bumps ONE arrival counter, ONE thread per CTA polls that counter until all
//                 tiles have arrived, then the CTA sums its predecessors' words with one strided read.
//   rounds        (the vectorised filter, any number of tiles; cooperative launch): the single wave walks tiles
//                 blockIdx.x + r * grid, publishing round r before it reads round r - 1 (cp_round_publish / _offset).
//   many waves    persistent CTAs draw tiles from an atomic ticket; decoupled look-back with the whole CTA (thread i
//                 inspects predecessor i): earlier waves have long published their inclusive prefixes, so one 256-wide
//                 window almost always suffices.
//
// Nothing is reset between launches: tickets and arrivals are monotonic counters (the host passes the base value of
// the launch), status words carry a 20-bit launch epoch and a stale epoch reads as "invalid".  That removes the
// end-of-kernel fence + atomic + reset loop.
#pragma once

#include <utility>

#include "device_utils.cuh"
#include "internal.h"

namespace fg {

constexpr int CP_THREADS = 256;
constexpr int CP_WARPS = CP_THREADS / 32;

// look-back word: [63:44] launch epoch, [43:42] flag (1 = partial, 2 = inclusive prefix), [41:0] value
constexpr int EP_VALUE_BITS = 42;
constexpr unsigned long long EP_VALUE_MASK = (1ull << EP_VALUE_BITS) - 1;
constexpr unsigned long long EP_PARTIAL = 1ull << EP_VALUE_BITS;
constexpr unsigned long long EP_PREFIX = 2ull << EP_VALUE_BITS;
constexpr unsigned long long EP_FLAG_MASK = 3ull << EP_VALUE_BITS;

struct CompactScratch {
  unsigned long long* tile_state;  // epoch-tagged look-back words (many-wave mode)
  unsigned long long* counts;      // per-tile survivor counts, epoch-tagged like the look-back words, dense (single-wave mode)
  int grid;                        // CTAs to launch
  unsigned int* counters;          // [0] tickets issued (many-wave mode), [1] tiles arrived (single-wave mode) -- monotonic across launches
  unsigned long long* out_count;   // receives the total number of survivors
  unsigned long long* host_count;  // optional second copy in page-locked host memory (saves the 8-byte D2H copy per launch)
  long long num_tiles;
  unsigned ticket_base;            // value of counters[0] when this launch starts
  unsigned arrived_base;           // value of counters[1] when this launch starts
  unsigned epoch;                  // 20-bit launch epoch of the look-back words
  int single_wave;
  int stride;                      // u64 words between look-back words of consecutive tiles (32 = one 256-byte L2 chunk each)
  int poll_sleep_ns;               // back-off of a polling thread (0 = spin)
};

// Item k of thread `tid` is item index  ((k / E) * CP_THREADS + tid) * E + k % E  of the tile: E = items
// a thread loads contiguously (vector width).  Survivors are ordered (group = k / E, thread, k % E),
// which is ascending item index.
template <int E>
__device__ __forceinline__ long long cp_item_index(int k, int tid) {
  return ((long long)(k / E) * CP_THREADS + tid) * E + (k % E);
}

template <int E, int I>
struct CompactSmem {
  static constexpr int G = I / E;
  unsigned group_warp[G][CP_WARPS];
  unsigned long long lb_sum[CP_WARPS];
  int lb_has[CP_WARPS];
  int lb_done;
  long long tile;
  unsigned long long excl;
  unsigned tile_total;
};

// Fetches the next tile index for the CTA (or -1 when the work is exhausted); `iteration` counts the CTA's calls.
// Many-wave mode: every CTA draws exactly one ticket past the end, so a launch consumes num_tiles + gridDim.x
// tickets (the host advances its base by that).
template <int E, int I>
__device__ __forceinline__ long long cp_next_tile(CompactSmem<E, I>& s, const CompactScratch& sc, int iteration) {
  if (sc.single_wave) {
    // one tile per CTA, all CTAs resident (cooperative launch, grid == num_tiles): the block index is the tile
    return iteration == 0 && (long long)blockIdx.x < sc.num_tiles ? (long long)blockIdx.x : -1;
  }
  if (threadIdx.x == 0) s.tile = (long long)(atomicAdd(sc.counters, 1u) - sc.ticket_base);
  __syncthreads();
  long long t = s.tile;
  return t < sc.num_tiles ? t : -1;
}

template <int E, int I>
__device__ __forceinline__ unsigned long long cp_block_sum(CompactSmem<E, I>& s, unsigned long long v) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_sum(v);
  if (lane == 0) s.lb_sum[warp] = v;
  __syncthreads();
  unsigned long long tot = 0;
#pragma unroll
  for (int w = 0; w < CP_WARPS; ++w) tot += s.lb_sum[w];
  return tot;
}

// ---- single wave ------------------------------------------------------------------------------------------------
// All CTAs are resident (cooperative launch), so a tile may simply wait for the counts of its predecessors.
//   publish   one relaxed store of a self-validating word {20-bit launch epoch, count} + one relaxed `red` on a
//             monotonic arrival counter.  No fence: the arrival only says "now is a good time to read", the epoch
//             tag in each word says whether that word is this launch's.
//   wait      thread 0 polls the arrival counter -- one word, T pollers -- until every tile has arrived;
//   read      the CTA reads its predecessors' words (thread i: tiles i, i + 256, ...: dense coalesced 2 KB reads of
//             an L2-resident array) and re-polls the rare word whose store is not visible yet.
// Alternatives that were slower on the 611 tiles of a 10 M-row relation: polling the count words directly from the
// start (every thread spins on not-yet-valid words), and a dedicated scanner CTA that publishes per-tile prefix
// words (two more L2 hops).  Nothing is reset between launches.
__device__ __forceinline__ unsigned ld_relaxed_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_relaxed_add_u32(unsigned* p, unsigned v) {
  asm volatile("red.relaxed.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// `group_base`: the launch may run several independent scans at once (gather.cu: the length scans of all Utf8 columns
// of a take()): tile `tile` of a group only sums the words [group_base, group_base + tile) but everybody waits for
// all sc.num_tiles arrivals.  `is_last` marks the tile that reports the group's total.
template <int E, int I>
__device__ __forceinline__ void cp_grid_prefix(CompactSmem<E, I>& s, const CompactScratch& sc, long long tile, unsigned long long total,
                                               long long group_base = 0, int is_last = -1, unsigned long long* group_out = nullptr) {
  const int tid = threadIdx.x;
  const unsigned long long tag = (unsigned long long)(sc.epoch & 0xfffffu) << 44;
  if (tid == 0) {
    st_relaxed_u64(sc.counts + group_base + tile, tag | EP_PREFIX | total);
    red_relaxed_add_u32(sc.counters + 1, 1u);
    const unsigned target = sc.arrived_base + unsigned(sc.num_tiles);
    while (int(ld_relaxed_u32(sc.counters + 1) - target) < 0) {
      if (sc.poll_sleep_ns) __nanosleep(sc.poll_sleep_ns);
    }
  }
  __syncthreads();
  unsigned long long part = 0;
  for (long long i = tid; i < tile; i += CP_THREADS) {
    unsigned long long w = ld_relaxed_u64(sc.counts + group_base + i);
    while ((w >> 44) != (tag >> 44)) w = ld_relaxed_u64(sc.counts + group_base + i);  // arrival seen before the count: rare
    part += w & EP_VALUE_MASK;
  }
  const unsigned long long excl = cp_block_sum(s, part);
  if (tid == 0) {
    s.excl = excl;
    const bool last = is_last < 0 ? tile == sc.num_tiles - 1 : is_last != 0;
    if (last) {
      unsigned long long* out = group_out ? group_out : sc.out_count;
      *out = excl + total;
      if (sc.host_count && !group_out) *reinterpret_cast<volatile unsigned long long*>(sc.host_count) = excl + total;
    }
  }
  __syncthreads();
}

// ---- many waves: decoupled look-back, 256 predecessors per step, epoch-tagged words -------------------------
template <int E, int I>
__device__ __forceinline__ void cp_block_lookback(CompactSmem<E, I>& s, const CompactScratch& sc, long long tile, unsigned long long total) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const unsigned long long tag = (unsigned long long)(sc.epoch & 0xfffffu) << 44;
  unsigned long long excl = 0;  // meaningful in thread 0 only
  if (tile == 0) {
    if (tid == 0) st_relaxed_u64(sc.tile_state, tag | EP_PREFIX | (unsigned long long)total);
  } else {
    if (tid == 0) st_relaxed_u64(sc.tile_state + tile * sc.stride, tag | EP_PARTIAL | (unsigned long long)total);
    long long base = tile - 1;
    while (true) {
      const long long t = base - tid;
      unsigned long long st = tag | EP_PREFIX;  // virtual tiles before the first one: inclusive prefix 0
      if (t >= 0) {
        while (true) {
          st = ld_relaxed_u64(sc.tile_state + t * sc.stride);
          if ((st >> 44) == (tag >> 44) && (st & EP_FLAG_MASK) != 0) break;  // published in THIS launch
          if (sc.poll_sleep_ns) __nanosleep(sc.poll_sleep_ns);
        }
      }
      const unsigned pm = __ballot_sync(FULL_MASK, (st & EP_FLAG_MASK) == EP_PREFIX);
      const int first = pm ? __ffs(pm) - 1 : 32;
      const unsigned long long wsum = warp_sum(lane <= first ? (st & EP_VALUE_MASK) : 0ull);
      if (lane == 0) {
        s.lb_sum[warp] = wsum;
        s.lb_has[warp] = pm != 0;
      }
      __syncthreads();
      if (tid == 0) {
        int done = 0;
        for (int w = 0; w < CP_WARPS && !done; ++w) {  // warp 0 holds the nearest predecessors
          excl += s.lb_sum[w];
          done = s.lb_has[w];
        }
        s.lb_done = done;
      }
      __syncthreads();
      if (s.lb_done) break;
      base -= CP_THREADS;
    }
    if (tid == 0) st_relaxed_u64(sc.tile_state + tile * sc.stride, tag | EP_PREFIX | (excl + total));
  }
  if (tid == 0) {
    s.excl = excl;
    if (tile == sc.num_tiles - 1) {
      *sc.out_count = excl + total;
      if (sc.host_count) *reinterpret_cast<volatile unsigned long long*>(sc.host_count) = excl + total;
    }
  }
  __syncthreads();
}

// ---- cooperative rounds: one wave of resident CTAs, CTA b takes tiles b, b + grid, b + 2 grid, ... --------------
// Round r is the contiguous band of tiles [r * grid, min((r + 1) * grid, num_tiles)).  A CTA publishes its tile's
// word of round r as soon as the tile is ranked (cp_round_publish) and only then asks for the offset of its tile of
// round r - 1 (cp_round_offset) and writes that tile: the publish of one round never waits behind the writes of the
// previous one, so a CTA that is slow to write does not hold up everybody's next round.  With publishes one round
// ahead, an arrival count cannot tell which round is complete, so the reader polls the epoch-tagged words themselves;
// by the time a round is read its words were published about one tile earlier, and a stale word is rare.  The
// arrival counter is still bumped once per tile, which keeps it in step with the host's count (launch_compact).
__device__ __forceinline__ void cp_round_publish(const CompactScratch& sc, long long tile, unsigned long long total) {
  if (threadIdx.x == 0) {
    const unsigned long long tag = (unsigned long long)(sc.epoch & 0xfffffu) << 44;
    st_relaxed_u64(sc.counts + tile, tag | EP_PREFIX | total);
    red_relaxed_add_u32(sc.counters + 1, 1u);
  }
}

// Reads the words of `tile`'s round once, summing those before the tile and the whole round.  `done` (shared) holds the
// survivors of the rounds the CTA has already read; the CTA reads its rounds in order, starting at round0 == 0.
// On return s.excl is the tile's output offset.
template <int E, int I>
__device__ __forceinline__ void cp_round_offset(CompactSmem<E, I>& s, const CompactScratch& sc, long long tile, long long round0,
                                                unsigned long long& done) {
  // a round's survivors (at most grid x tile items) fit the 32-bit halves of the packed sum below
  static_assert(CP_THREADS * I <= (1 << 16), "tile too large for the packed round sums");
  const int tid = threadIdx.x;
  const unsigned long long tag = (unsigned long long)(sc.epoch & 0xfffffu) << 44;
  const long long round_end = round0 + sc.grid < sc.num_tiles ? round0 + sc.grid : sc.num_tiles;
  unsigned long long part = 0;  // [31:0] words before `tile`, [63:32] all words of the round
  for (long long i = round0 + tid; i < round_end; i += CP_THREADS) {
    unsigned long long w = ld_relaxed_u64(sc.counts + i);
    while ((w >> 44) != (tag >> 44)) {
      if (sc.poll_sleep_ns) __nanosleep(sc.poll_sleep_ns);
      w = ld_relaxed_u64(sc.counts + i);
    }
    const unsigned long long c = w & EP_VALUE_MASK;
    part += (c << 32) | (i < tile ? c : 0ull);
  }
  const unsigned long long sums = cp_block_sum(s, part);
  if (tid == 0) {
    const unsigned long long before = round0 == 0 ? 0ull : done;
    const unsigned long long excl = before + (sums & 0xffffffffull);
    s.excl = excl;
    done = before + (sums >> 32);
    if (tile == sc.num_tiles - 1) {
      *sc.out_count = excl + s.tile_total;
      if (sc.host_count) *reinterpret_cast<volatile unsigned long long*>(sc.host_count) = excl + s.tile_total;
    }
  }
  __syncthreads();
}

// Ranks the survivors of one tile within the tile (bit k of `bits` = item k survives): on return (after the internal
// barriers) s.group_warp, lane_prefix and s.tile_total hold everything cp_local_position() needs.
template <int E, int I>
__device__ __forceinline__ void cp_rank_local(CompactSmem<E, I>& s, unsigned long long bits, unsigned (&lane_prefix)[I / E]) {
  constexpr int G = I / E;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if constexpr (E == 4) {
    // Group g is nibble g of `bits`.  SWAR: per-nibble popcounts (0..4), spread to byte fields of up to four
    // registers, ONE 5-step warp scan over the packed fields (a field holds at most 32 x 4 = 128): ~60
    // instructions per thread for 64 rows instead of one ballot + two popcounts per row.
    static_assert(G <= 16, "packed ranking covers 64 items per thread");
    constexpr int R = G > 8 ? 4 : 2;
    auto nibble_counts = [](unsigned x) {
      x = x - ((x >> 1) & 0x55555555u);
      return (x & 0x33333333u) + ((x >> 2) & 0x33333333u);
    };
    const unsigned lo = nibble_counts(unsigned(bits)), hi = nibble_counts(unsigned(bits >> 32));
    // register r, byte i holds group (r >> 1) * 8 + 2 * i + (r & 1)
    unsigned own[4] = {lo & 0x0f0f0f0fu, (lo >> 4) & 0x0f0f0f0fu, hi & 0x0f0f0f0fu, (hi >> 4) & 0x0f0f0f0fu};
    unsigned incl[4] = {own[0], own[1], own[2], own[3]};
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const unsigned t = __shfl_up_sync(FULL_MASK, incl[r], d);
        if (lane >= d) incl[r] += t;
      }
    }
#pragma unroll
    for (int g = 0; g < G; ++g) {
      const int r = (g >> 3) * 2 + (g & 1), sh = ((g & 7) >> 1) * 8;
      lane_prefix[g] = ((incl[r] - own[r]) >> sh) & 0xffu;
      if (lane == 31) s.group_warp[g][warp] = (incl[r] >> sh) & 0xffu;
    }
  } else {
    const unsigned lt = lanemask_lt();
#pragma unroll
    for (int g = 0; g < G; ++g) {
      unsigned pre = 0, tot = 0;
#pragma unroll
      for (int e = 0; e < E; ++e) {
        unsigned b = __ballot_sync(FULL_MASK, (bits >> (g * E + e)) & 1ull);
        pre += __popc(b & lt);
        tot += __popc(b);
      }
      lane_prefix[g] = pre;
      if (lane == 0) s.group_warp[g][warp] = tot;
    }
  }
  __syncthreads();
  if (warp == 0) {
    constexpr int N = G * CP_WARPS;
    constexpr int PER = (N + 31) / 32;
    unsigned* flat = &s.group_warp[0][0];
    unsigned v[PER], sum = 0;
#pragma unroll
    for (int i = 0; i < PER; ++i) {
      int idx = lane * PER + i;
      v[i] = idx < N ? flat[idx] : 0u;
      sum += v[i];
    }
    unsigned incl = warp_inclusive_sum(sum);
    unsigned run = incl - sum;
#pragma unroll
    for (int i = 0; i < PER; ++i) {
      int idx = lane * PER + i;
      if (idx < N) flat[idx] = run;
      run += v[i];
    }
    unsigned total = __shfl_sync(FULL_MASK, incl, 31);
    if (lane == 0) s.tile_total = total;
  }
  __syncthreads();
}

// Ranks the survivors of one tile (bit k of `bits` = item k survives).  On return (after the internal
// barriers) cp_position() gives every survivor its output slot and s.tile_total the tile's survivor count.
struct CpNoHook {
  __device__ __forceinline__ void operator()() const {}
};

// `before_wait` runs after the tile-local ranking and before the wait for the grid-wide prefix: work that does not
// need output positions (prefetching the survivors' pass-through values) hides behind that wait.
template <int E, int I, class Hook = CpNoHook>
__device__ __forceinline__ void cp_rank_tile(CompactSmem<E, I>& s, const CompactScratch& sc, long long tile, unsigned long long bits,
                                             unsigned (&lane_prefix)[I / E], Hook before_wait = Hook{}) {
  cp_rank_local<E, I>(s, bits, lane_prefix);
  before_wait();
  if (sc.single_wave) cp_grid_prefix(s, sc, tile, s.tile_total);
  else cp_block_lookback(s, sc, tile, s.tile_total);
}

// Host side (core.cu): sizes the scratch and fills a CompactScratch for ONE launch over `num_tiles` tiles by a kernel of
// which `resident_ctas` fit on the device at once; chooses the mode and the grid (sc.grid) and draws a launch epoch.
// `rounds`: the kernel walks cooperative rounds (cp_round_publish / cp_round_offset), so the single-wave mode also covers num_tiles >
// resident_ctas.  Call it right before launch_compact(), which advances the ticket / arrival bookkeeping once the launch
// is accepted.
CompactScratch prepare_compact(const CtxPtr& ctx, long long num_tiles, long long resident_ctas, unsigned long long* out_count, bool rounds = false);

// A launch of a kernel built to start while the kernel enqueued ahead of it drains (filter_compact_kernel<PredI32>):
// before griddepcontrol.wait it only reads its input buffers and its own shared memory, and it touches the shared
// scan scratch, its outputs and d_scalars only after the wait, which returns once that kernel has completed and its
// memory is visible.
struct EarlyStart {
  int64_t newest_input;  // the largest Buffer::seq among the device buffers the launch reads
  int64_t outputs;       // Buffer::seq of its outputs (ctx->alloc_seq, advanced before they were allocated)
};

// Whether this launch may take programmatic stream serialization (core.cu; the whole policy).  Only when ALL hold:
//   - it is a single-wave (cooperative rounds) launch of an EarlyStart kernel;
//   - the last kernel enqueued on ctx->stream was a single-wave EarlyStart launch of the same kernel (ctx->launches
//     has advanced by that one launch since), and prepare_compact enqueued no scratch reset since;
//   - every buffer it reads is older than that launch's outputs (Buffer::seq).  No kernel writes into a table column
//     it did not allocate at its own enqueue: a column is written only by work its operator enqueues before it returns,
//     and outputs are fresh blocks.  So such a buffer was complete before the previous launch started, and since that
//     launch's CTAs pass their own wait before they let this one start, everything ahead of it has completed.  A
//     chained input (the previous filter's output) is not older, and that launch waits as before.
bool overlap_previous(const CtxPtr& ctx, const void* kernel, const CompactScratch& sc, const EarlyStart* early);
// Records an accepted launch for the next overlap_previous() decision.
void note_compact_launch(const CtxPtr& ctx, const void* kernel, const CompactScratch& sc, const EarlyStart* early, bool overlapped);

// Launches a compaction kernel with sc.grid CTAs.  Single-wave launches wait for data of other CTAs, which only
// arrives when EVERY CTA of the grid is running, so they go through the cooperative-launch path: the driver then
// guarantees co-residency (or fails the launch) instead of us assuming the GPU is otherwise idle.
//
// A launch that overlaps its predecessor (overlap_previous) drops the cooperative attribute: a launch that carries both
// is accepted but never starts before its predecessor has ended (measured on an H100 80GB HBM3, CUDA 12.9).  It
// stays live without it: the previous grid never waits on this one, and this grid is the same kernel with the same
// grid (resident_ctas of the same instantiation), so every one of its CTAs is resident once the previous grid exits.
template <class Kernel, class... Args>
inline void launch_compact_early(const CtxPtr& ctx, Kernel kernel, const CompactScratch& sc, const EarlyStart* early, Args&&... args) {
  HostSpan span("launch_compact");
  const bool overlap = overlap_previous(ctx, reinterpret_cast<const void*>(kernel), sc, early);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(unsigned(sc.grid));
  cfg.blockDim = dim3(CP_THREADS);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = ctx->stream;
  cudaLaunchAttribute attr[1];
  if (overlap) {
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
  } else {
    attr[0].id = cudaLaunchAttributeCooperative;
    attr[0].val.cooperative = sc.single_wave ? 1 : 0;
  }
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  FG_CUDA(cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...));
  // Only a launch that was accepted consumes arrivals / tickets: if anything fails between prepare_compact() and here,
  // the host's view of the monotonic device counters stays exact (a mismatch would make the next launch wait forever).
  ScanScratch& s = ctx->scan;
  if (sc.single_wave) s.arrived += unsigned(sc.num_tiles);                      // one arrival per tile, no tickets
  else s.tickets_issued += unsigned(sc.num_tiles) + unsigned(sc.grid);          // every CTA draws exactly one ticket past the end
  note_compact_launch(ctx, reinterpret_cast<const void*>(kernel), sc, early, overlap);
}

template <class Kernel, class... Args>
inline void launch_compact(const CtxPtr& ctx, Kernel kernel, const CompactScratch& sc, Args&&... args) {
  launch_compact_early(ctx, kernel, sc, static_cast<const EarlyStart*>(nullptr), std::forward<Args>(args)...);
}

// Rank of survivor item k among the survivors of its tile (0 .. tile_total - 1) / its global output position.
template <int E, int I>
__device__ __forceinline__ unsigned cp_local_position(const CompactSmem<E, I>& s, unsigned long long bits, int k, const unsigned (&lane_prefix)[I / E]) {
  constexpr int G = I / E;
  const int g = k / E, e = k % E;
  const unsigned within = __popcll(bits & (((1ull << e) - 1ull) << (g * E)));
  unsigned lp;
  if constexpr (G <= 8) {
    // selects instead of a run-time index: the array stays in registers instead of going to local memory
    lp = lane_prefix[0];
#pragma unroll
    for (int i = 1; i < G; ++i) lp = g == i ? lane_prefix[i] : lp;
  } else {
    lp = lane_prefix[g];
  }
  return s.group_warp[g][threadIdx.x >> 5] + lp + within;
}

template <int E, int I>
__device__ __forceinline__ long long cp_position(const CompactSmem<E, I>& s, unsigned long long bits, int k, const unsigned (&lane_prefix)[I / E]) {
  return (long long)s.excl + cp_local_position<E, I>(s, bits, k, lane_prefix);
}

}  // namespace fg
