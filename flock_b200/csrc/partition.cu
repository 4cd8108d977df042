// partition.cu -- K2: RepartitionExec: partitioning = Hash([keys], n) as ONE multi-way pass (see partition.h).
//
// Reference operator (DataFusion fork; used at flock/src/distributed_plan/planner.rs:153, :160, :223,
// :234; standalone helper flock/src/transmute.rs:77-109; the call shape is spelled out in
// playground/src/distributed_plan/shuffle_writer.rs:105-146): create_hashes(key arrays) ->
// partition = hash % n -> per-partition index lists -> arrow `take` of every column.  Rows keep their
// input order inside a partition.
//
// Here: count (+ scan in its last CTA for up to 64 histogram columns, else a scan launch) -> place -> scatter, three or
// four launches whatever n is; the n output tables are VIEWS of one
// partition-ordered set of buffers (every partition starts on a 16-byte boundary so that vector loads keep working).
#include "partition.h"

#include <algorithm>
#include <cstdlib>

#include "device_utils.cuh"

namespace fg {

__host__ __device__ __forceinline__ uint32_t partition_of(uint64_t hash, uint32_t n_parts) {
  return uint32_t(((hash >> 32) * uint64_t(n_parts)) >> 32);
}

// ================================================================================================
// step 1: destinations + per-CTA histograms
// ================================================================================================
struct PartCountArgs {
  int64_t n_rows, chunk;
  int32_t n_parts, packed, dest_rank, n_utf8, grid, key_nulls;
  int32_t digit_col, digit_shift;  // digit_col >= 0: destination = byte `digit_shift / 8` of that UInt64 column (a radix-sort pass)
  KeyPack pack;
  RowKeys rk;
  ColRef cols[MAX_IN_COLS];
  const int32_t* uoff[PT_MAX_UTF8];
  uint8_t* pid;
  uint32_t* hist;  // [(1 + n_utf8)][grid][n_parts]
  // fused scan (step 2 inside this kernel): the CTA that arrives last scans the histograms of all CTAs
  unsigned* arrive;           // zero on entry, left zero (NULL: the scan is a launch of its own)
  uint32_t* cta_pos;
  unsigned long long* totals;
};

constexpr int kPartitionArriveSlot = 80;  // d_scalars[80]: arrival counter of the fused scan (zero between launches)
constexpr int PT_FUSED_SCAN_COLS = 64;  // (1 + n_utf8) * n_parts up to which the last CTA scans (>= 4 row blocks of threads)

// Step 2 by ONE CTA of PT_THREADS threads, for matrices of few columns (an exchange over <= 16 ranks): thread (g, c)
// sums a block of rows of column c, the blocks' sums are combined through shared memory, a second sweep writes the
// exclusive prefixes.  `s_part` holds PT_THREADS words.
__device__ __forceinline__ void scan_hist_cta(const uint32_t* hist, uint32_t* cta_pos, unsigned long long* totals, int grid, int P, int kinds,
                                              unsigned long long* s_part) {
  const int tid = threadIdx.x;
  const int C = kinds * P, G = PT_THREADS / C;
  const int c = tid % C, g = tid / C;
  const int kind = c / P, p = c - kind * P;
  const int R = (grid + G - 1) / G;
  const int r0 = g * R, r1 = g < G ? min(grid, r0 + R) : r0;
  const uint32_t* h = hist + int64_t(kind) * grid * P + p;
  uint32_t* o = cta_pos + int64_t(kind) * grid * P + p;
  unsigned long long sum = 0;
  for (int r = r0; r < r1; ++r) sum += __ldcg(h + int64_t(r) * P);
  s_part[tid] = sum;
  __syncthreads();
  if (g < G) {
    unsigned long long before = 0, total = 0;
    for (int gg = 0; gg < G; ++gg) {
      const unsigned long long v = s_part[gg * C + c];
      if (gg < g) before += v;
      total += v;
    }
    unsigned long long run = before;
    for (int r = r0; r < r1; ++r) {
      const unsigned v = __ldcg(h + int64_t(r) * P);
      o[int64_t(r) * P] = uint32_t(run);
      run += v;
    }
    if (g == 0) totals[kind * P + p] = total;
  }
}

__global__ void __launch_bounds__(PT_THREADS) partition_count_kernel(const __grid_constant__ PartCountArgs a) {
  extern __shared__ __align__(16) unsigned pc_smem[];
  const int P = a.n_parts;
  unsigned* h_rows = pc_smem;                  // [PT_WARPS][P] private to a warp: plain updates by one leader lane per value
  unsigned* h_bytes = pc_smem + PT_WARPS * P;  // [n_utf8][P] shared atomics
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < (PT_WARPS + a.n_utf8) * P; i += PT_THREADS) pc_smem[i] = 0;
  __syncthreads();
  const int64_t begin = int64_t(blockIdx.x) * a.chunk;
  const int64_t end = begin + a.chunk < a.n_rows ? begin + a.chunk : a.n_rows;
  const unsigned lt = lanemask_lt();
  unsigned* mine = h_rows + warp * P;
  (void)lt;
  constexpr int UNROLL = 4;  // rows per thread and iteration: their key loads are independent and in flight together
  const bool small = P <= 8;
  unsigned long long acc8 = 0;
  int since = 0;
  auto flush_acc8 = [&]() {
    for (int p = 0; p < P; ++p) {
      const unsigned total = __reduce_add_sync(FULL_MASK, unsigned(acc8 >> (8 * p)) & 0xffu);
      if (lane == 0) mine[p] += total;
    }
    acc8 = 0;
  };
  for (int64_t base = begin; base < end; base += PT_THREADS * UNROLL) {
    unsigned pid[UNROLL];
    bool valid[UNROLL];
#pragma unroll
    for (int j = 0; j < UNROLL; ++j) {
      const int64_t row = base + j * PT_THREADS + tid;
      valid[j] = row < end;
      pid[j] = 0;
      if (valid[j]) {
        if (a.dest_rank >= 0) {
          pid[j] = unsigned(a.dest_rank);
        } else if (a.digit_col >= 0) {
          pid[j] = unsigned(static_cast<const unsigned long long*>(a.cols[a.digit_col].data)[row] >> a.digit_shift) & 0xffu;
        } else {
          // a row with a NULL key takes hash_row's fixed NULL contribution on every rank; any other row of a packable
          // key hashes its packed word whether or not the column carries validity HERE (a peer's slice of the same
          // column may hold no NULL and so no validity: both must route a key alike)
          bool null_key = false;
          if (a.packed && a.key_nulls)
            for (int i = 0; i < a.rk.n; ++i) {
              const uint8_t* v = a.cols[a.rk.col[i]].validity;
              null_key |= v && !v[row];
            }
          const unsigned long long h = a.packed && !null_key ? fmix64(pack_key(a.pack, a.cols, row)) : hash_row(a.rk, a.cols, row);
          pid[j] = partition_of(h, uint32_t(P));
        }
      }
    }
#pragma unroll
    for (int j = 0; j < UNROLL; ++j) {
      const int64_t row = base + j * PT_THREADS + tid;
      if (valid[j]) {
        a.pid[row] = uint8_t(pid[j]);
        for (int u = 0; u < a.n_utf8; ++u) atomicAdd(&h_bytes[u * P + pid[j]], unsigned(a.uoff[u][row + 1] - a.uoff[u][row]));
      }
      if (small) {  // up to 8 destinations: eight 8-bit counters in one register, emptied before any can wrap
        if (valid[j]) acc8 += 1ull << (8 * pid[j]);
        continue;
      }
      const unsigned vmask = __ballot_sync(FULL_MASK, valid[j]);
      unsigned m = 0, before = 0;
      if (valid[j]) {
        m = __match_any_sync(vmask, pid[j]);
        before = mine[pid[j]];
      }
      __syncwarp();
      if (valid[j] && lane == __ffs(m) - 1) mine[pid[j]] = before + __popc(m);
      __syncwarp();
    }
    if (small && ++since == 255 / UNROLL) {
      flush_acc8();
      since = 0;
    }
  }
  if (small) flush_acc8();
  __syncthreads();
  for (int p = tid; p < P; p += PT_THREADS) {
    unsigned rows = 0;
#pragma unroll
    for (int w = 0; w < PT_WARPS; ++w) rows += h_rows[w * P + p];
    a.hist[(int64_t(0) * a.grid + blockIdx.x) * P + p] = rows;
    for (int u = 0; u < a.n_utf8; ++u) a.hist[(int64_t(1 + u) * a.grid + blockIdx.x) * P + p] = h_bytes[u * P + p];
  }
  if (a.arrive) {
    // the histograms of this CTA are visible before its arrival is; whoever counts the last arrival reads them all
    __shared__ unsigned s_last;
    __shared__ unsigned long long s_part[PT_THREADS];
    __threadfence();
    __syncthreads();
    if (tid == 0) s_last = atomicAdd(a.arrive, 1u) == gridDim.x - 1 ? 1u : 0u;
    __syncthreads();
    if (s_last) {
      __threadfence();
      scan_hist_cta(a.hist, a.cta_pos, a.totals, a.grid, P, 1 + a.n_utf8, s_part);
      if (tid == 0) *a.arrive = 0u;  // ready for the next pass on this context's stream
    }
  }
}

// ================================================================================================
// step 2: per destination (and per kind: rows, bytes of Utf8 column u) exclusive scan over the CTAs
// ================================================================================================
__global__ void __launch_bounds__(1024) partition_scan_kernel(const uint32_t* __restrict__ hist, uint32_t* __restrict__ cta_pos,
                                                              unsigned long long* __restrict__ totals, int grid, int n_parts, int n_kinds) {
  // One kind (rows, or the bytes of one Utf8 column) is a grid x n_parts matrix, row-major; wanted: the exclusive
  // prefix down every column.  Warp w owns the rows [w * R, (w + 1) * R), lane l the column c0 + l of a block of 32
  // columns: a thread first sums its R entries (independent loads), the 32 partial sums of a column are combined
  // through shared memory, and a second sweep writes the prefixes.  (The first version walked each column with one
  // warp, 32 CTAs per dependent step, and was several times slower.)
  __shared__ unsigned long long s_part[32][33];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int R = (grid + 31) / 32;
  const int r0 = warp * R, r1 = min(grid, r0 + R);
  for (int k = 0; k < n_kinds; ++k) {
    const uint32_t* h = hist + int64_t(k) * grid * n_parts;
    uint32_t* o = cta_pos + int64_t(k) * grid * n_parts;
    for (int c0 = 0; c0 < n_parts; c0 += 32) {
      const int c = c0 + lane;
      unsigned long long sum = 0;
      if (c < n_parts)
        for (int r = r0; r < r1; ++r) sum += h[int64_t(r) * n_parts + c];
      s_part[warp][lane] = sum;
      __syncthreads();
      unsigned long long before = 0, total = 0;
#pragma unroll 8
      for (int w = 0; w < 32; ++w) {
        const unsigned long long v = s_part[w][lane];
        if (w < warp) before += v;
        total += v;
      }
      if (c < n_parts) {
        unsigned long long run = before;
        for (int r = r0; r < r1; ++r) {
          const unsigned v = h[int64_t(r) * n_parts + c];
          o[int64_t(r) * n_parts + c] = unsigned(run);
          run += v;
        }
        if (warp == 0) totals[k * n_parts + c] = total;
      }
      __syncthreads();
    }
  }
}

// ================================================================================================
// step 4: stable scatter through shared memory
// ================================================================================================
struct PartScatterArgs {
  int64_t n_rows, chunk;
  int32_t n_parts, n_fixed, n_utf8, grid;
  const uint8_t* pid;
  const void* fsrc[MAX_IN_COLS];
  int32_t fwidth[MAX_IN_COLS];
  const int32_t* uoff[PT_MAX_UTF8];
  const uint8_t* udata[PT_MAX_UTF8];
  const uint32_t* cta_pos;
  const PartDest* dest;
  const unsigned* abort_flag;
};

// dynamic shared memory layout of the scatter kernel (P destinations, U Utf8 columns)
struct ScatterSmem {
  size_t wcnt, woff, seg, tot, run, runb, segb, sege, row, pid, wscan, dest, stage, src, total;
  __host__ __device__ ScatterSmem(int P, int U, bool dest_in_smem) {
    size_t o = 0;
    auto take = [&](size_t bytes) {
      size_t at = o;
      o = (o + bytes + 15) & ~size_t(15);
      return at;
    };
    wcnt = take(size_t(PT_WARPS) * P * 2);
    woff = take(size_t(PT_WARPS) * P * 2);
    seg = take(size_t(P + 1) * 2);
    tot = take(size_t(P) * 2);
    run = take(size_t(P) * 4);
    runb = take(size_t(U ? U : 1) * P * 4);
    segb = take(size_t(P) * 4);
    sege = take(size_t(P) * 4);
    row = take(size_t(PT_TILE) * 2);
    pid = take(size_t(PT_TILE));
    wscan = take(size_t(PT_WARPS + 1) * 4);
    dest = take(dest_in_smem ? size_t(P) * sizeof(PartDest) : 0);
    stage = take(U ? size_t(PT_STAGE_BYTES) : 0);
    src = take(U ? size_t(PT_STAGE_BYTES) + 32 : 0);
    total = o;
  }
};
constexpr int PT_DEST_SMEM_PARTS = 16;  // up to this many destinations the PartDest table is copied to shared memory

__global__ void __launch_bounds__(PT_THREADS, 3) partition_scatter_kernel(const __grid_constant__ PartScatterArgs a) {
  extern __shared__ __align__(16) unsigned char ps_smem[];
  if (a.abort_flag && *reinterpret_cast<const volatile unsigned*>(a.abort_flag)) return;
  const int P = a.n_parts, U = a.n_utf8;
  const bool dest_in_smem = P <= PT_DEST_SMEM_PARTS;
  const ScatterSmem L(P, U, dest_in_smem);
  unsigned short* s_wcnt = reinterpret_cast<unsigned short*>(ps_smem + L.wcnt);
  unsigned short* s_woff = reinterpret_cast<unsigned short*>(ps_smem + L.woff);
  unsigned short* s_seg = reinterpret_cast<unsigned short*>(ps_smem + L.seg);
  unsigned short* s_tot = reinterpret_cast<unsigned short*>(ps_smem + L.tot);
  unsigned* s_run = reinterpret_cast<unsigned*>(ps_smem + L.run);
  unsigned* s_runb = reinterpret_cast<unsigned*>(ps_smem + L.runb);
  unsigned* s_segb = reinterpret_cast<unsigned*>(ps_smem + L.segb);
  unsigned* s_sege = reinterpret_cast<unsigned*>(ps_smem + L.sege);
  unsigned short* s_row = reinterpret_cast<unsigned short*>(ps_smem + L.row);
  unsigned char* s_pid = ps_smem + L.pid;
  unsigned* s_wscan = reinterpret_cast<unsigned*>(ps_smem + L.wscan);
  unsigned char* s_stage = ps_smem + L.stage;
  unsigned char* s_src = ps_smem + L.src;
  const PartDest* dest = a.dest;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t begin = int64_t(blockIdx.x) * a.chunk;
  const int64_t end = begin + a.chunk < a.n_rows ? begin + a.chunk : a.n_rows;
  if (begin >= end) return;
  if (dest_in_smem) {
    unsigned long long* d = reinterpret_cast<unsigned long long*>(ps_smem + L.dest);
    const unsigned long long* s = reinterpret_cast<const unsigned long long*>(a.dest);
    for (int i = tid; i < int(P * sizeof(PartDest) / 8); i += PT_THREADS) d[i] = s[i];
    dest = reinterpret_cast<const PartDest*>(ps_smem + L.dest);
  }
  for (int p = tid; p < P; p += PT_THREADS) {
    s_run[p] = a.cta_pos[(int64_t(0) * a.grid + blockIdx.x) * P + p];
    for (int u = 0; u < U; ++u) s_runb[u * P + p] = a.cta_pos[(int64_t(1 + u) * a.grid + blockIdx.x) * P + p];
  }
  const unsigned lt = lanemask_lt();
  unsigned short* my_wcnt = s_wcnt + warp * P;

  for (int64_t tile0 = begin; tile0 < end; tile0 += PT_TILE) {
    const int rows = int(end - tile0 < PT_TILE ? end - tile0 : PT_TILE);
    for (int p = lane; p < P; p += 32) my_wcnt[p] = 0;
    __syncthreads();  // also: s_run / dest are initialised, the previous tile's readers of s_row / s_pid are done
    // ---- rank of every row among the rows of its warp with the same destination (rows in input order)
    unsigned char mypid[8];
    unsigned short myrank[8];
    // the eight destination bytes first: independent loads, all in flight before the (warp-synchronous) ranking starts
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int local = warp * 256 + j * 32 + lane;
      mypid[j] = local < rows ? a.pid[tile0 + local] : (unsigned char)0;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int local = warp * 256 + j * 32 + lane;
      const bool valid = local < rows;
      unsigned pid = mypid[j], m = 0, before = 0;
      const unsigned vmask = __ballot_sync(FULL_MASK, valid);
      if (valid) {
        m = __match_any_sync(vmask, pid);
        before = my_wcnt[pid];
      }
      __syncwarp();
      if (valid && lane == __ffs(m) - 1) my_wcnt[pid] = (unsigned short)(before + __popc(m));
      __syncwarp();
      myrank[j] = (unsigned short)(before + __popc(m & lt));
    }
    __syncthreads();
    // ---- per destination: offsets of the warps, the tile's total
    for (int p = tid; p < P; p += PT_THREADS) {
      unsigned run = 0;
#pragma unroll
      for (int w = 0; w < PT_WARPS; ++w) {
        s_woff[w * P + p] = (unsigned short)run;
        run += s_wcnt[w * P + p];
      }
      s_tot[p] = (unsigned short)run;
    }
    __syncthreads();
    if (warp == 0) {  // exclusive scan of the totals over the destinations: where each segment starts in the tile
      unsigned run = 0;
      for (int p0 = 0; p0 < P; p0 += 32) {
        const int p = p0 + lane;
        const unsigned v = p < P ? s_tot[p] : 0u;
        const unsigned incl = warp_inclusive_sum(v);
        if (p < P) s_seg[p] = (unsigned short)(run + incl - v);
        run += __shfl_sync(FULL_MASK, incl, 31);
      }
      if (lane == 0) s_seg[P] = (unsigned short)run;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int local = warp * 256 + j * 32 + lane;
      if (local < rows) {
        const unsigned p = mypid[j];
        const unsigned s = unsigned(s_seg[p]) + s_woff[warp * P + p] + myrank[j];
        s_row[s] = (unsigned short)local;
        s_pid[s] = (unsigned char)p;
      }
    }
    __syncthreads();
    // ---- fixed-width columns: consecutive threads write consecutive rows of one destination
    {
      // slot s = tid + 256 k of the ordered tile: where it goes and where it comes from, for all eight k at once, then
      // column by column eight loads in flight before their eight stores
      unsigned pp[8];
      int64_t pos[8], row[8];
      bool on[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int sx = tid + k * PT_THREADS;
        on[k] = sx < rows;
        pp[k] = on[k] ? s_pid[sx] : 0u;
        pos[k] = on[k] ? int64_t(s_run[pp[k]]) + (sx - int(s_seg[pp[k]])) : 0;
        row[k] = on[k] ? tile0 + s_row[sx] : tile0;
      }
      for (int f = 0; f < a.n_fixed; ++f) {
        if (a.fwidth[f] == 1) {
          uint8_t v[8];
#pragma unroll
          for (int k = 0; k < 8; ++k) v[k] = on[k] ? static_cast<const uint8_t*>(a.fsrc[f])[row[k]] : uint8_t(0);
#pragma unroll
          for (int k = 0; k < 8; ++k)
            if (on[k]) static_cast<uint8_t*>(dest[pp[k]].val[f])[pos[k]] = v[k];
        } else if (a.fwidth[f] == 4) {
          uint32_t v[8];
#pragma unroll
          for (int k = 0; k < 8; ++k) v[k] = on[k] ? static_cast<const uint32_t*>(a.fsrc[f])[row[k]] : 0u;
#pragma unroll
          for (int k = 0; k < 8; ++k)
            if (on[k]) static_cast<uint32_t*>(dest[pp[k]].val[f])[pos[k]] = v[k];
        } else {
          unsigned long long v[8];
#pragma unroll
          for (int k = 0; k < 8; ++k) v[k] = on[k] ? static_cast<const unsigned long long*>(a.fsrc[f])[row[k]] : 0ull;
#pragma unroll
          for (int k = 0; k < 8; ++k)
            if (on[k]) static_cast<unsigned long long*>(dest[pp[k]].val[f])[pos[k]] = v[k];
        }
      }
    }
    // ---- Utf8 columns: a thread owns 8 consecutive slots of the ordered tile
    for (int u = 0; u < U; ++u) {
      for (int p = tid; p < P; p += PT_THREADS) {
        s_segb[p] = 0;
        s_sege[p] = 0;
      }
      int len[8], src[8];
      unsigned local_sum = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int s = tid * 8 + k;
        len[k] = 0;
        src[k] = 0;
        if (s < rows) {
          const int64_t row = tile0 + s_row[s];
          src[k] = a.uoff[u][row];
          len[k] = a.uoff[u][row + 1] - src[k];
        }
        local_sum += unsigned(len[k]);
      }
      const unsigned incl = warp_inclusive_sum(local_sum);
      if (lane == 31) s_wscan[warp] = incl;
      __syncthreads();  // s_segb / s_sege zeroed, warp sums published
      unsigned warp_base = 0, tile_bytes = 0;
#pragma unroll
      for (int w = 0; w < PT_WARPS; ++w) {
        const unsigned v = s_wscan[w];
        if (w < warp) warp_base += v;
        tile_bytes += v;
      }
      unsigned bytepos[8];
      unsigned run = warp_base + incl - local_sum;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        bytepos[k] = run;
        run += unsigned(len[k]);
        const int s = tid * 8 + k;
        if (s < rows) {
          const unsigned p = s_pid[s];
          if (s == int(s_seg[p])) s_segb[p] = bytepos[k];
          if (s == int(s_seg[p]) + int(s_tot[p]) - 1) s_sege[p] = bytepos[k] + unsigned(len[k]);
        }
      }
      __syncthreads();
      const bool staged = tile_bytes <= unsigned(PT_STAGE_BYTES);
      // The tile's strings are CONTIGUOUS in the source (rows tile0 .. tile0 + rows): the CTA fetches that byte range
      // with coalesced 16-byte loads into shared memory, and the per-string shuffling into destination order then runs
      // from shared to shared.  (Fetching string by string from global memory chained ~24 dependent loads per
      // thread and took most of the kernel's time on q8's 2.5 M names.)
      const int32_t sb0 = a.uoff[u][tile0];
      unsigned shift = 0;
      if (staged) {
        const uintptr_t addr = reinterpret_cast<uintptr_t>(a.udata[u] + sb0);
        const uint4* aligned = reinterpret_cast<const uint4*>(addr & ~uintptr_t(15));
        shift = unsigned(addr & 15);
        const unsigned n16 = (shift + tile_bytes + 15) >> 4;
        for (unsigned i = tid; i < n16; i += PT_THREADS) reinterpret_cast<uint4*>(s_src)[i] = __ldg(aligned + i);
        __syncthreads();
      }
      // The offsets entries are NOT stored from here: a thread owns 8 consecutive slots, so the lanes of a warp would
      // write 4 bytes each into addresses 32 bytes apart -- 32 partial sectors per store instruction.  HBM absorbs
      // that; NVLink sends every partial sector as a packet of its own, and with 7/8 of the rows leaving the GPU the
      // scatter of q8's persons took about twice as long at 8 ranks as at 2.  The
      // values go through shared memory (the source staging area is free again after the shuffle) and are written
      // out below with consecutive lanes on consecutive slots, like the fixed-width columns.
      int32_t offv[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int s = tid * 8 + k;
        offv[k] = 0;
        if (s >= rows) continue;
        const unsigned p = s_pid[s];
        const unsigned rel = s_runb[u * P + p] + (bytepos[k] - s_segb[p]);
        offv[k] = int32_t(dest[p].byte_origin[u] + (long long)rel);
        if (staged) {
          const unsigned char* from = s_src + shift + (src[k] - sb0);
          unsigned char* to = s_stage + bytepos[k];
          for (int b = 0; b < len[k]; ++b) to[b] = from[b];
        } else {  // a tile of long strings: straight to the destination
          const uint8_t* from = a.udata[u] + src[k];
          uint8_t* to = dest[p].bytes[u] + rel;
          for (int b = 0; b < len[k]; ++b) to[b] = from[b];
        }
      }
      __syncthreads();
      int32_t* s_offv = reinterpret_cast<int32_t*>(s_src);  // every read of the source staging area is behind the barrier
#pragma unroll
      for (int k = 0; k < 8; ++k) s_offv[tid * 8 + k] = offv[k];
      if (staged) {
        // a warp per destination segment: the lanes write consecutive bytes (full sectors on the wire)
        for (int p = warp; p < P; p += PT_WARPS) {
          const unsigned b0 = s_segb[p], b1 = s_sege[p];
          uint8_t* to = dest[p].bytes[u] + s_runb[u * P + p];
          // head up to a 4-byte boundary of the destination, aligned words, tail
          unsigned head = unsigned(-(long long)reinterpret_cast<uintptr_t>(to)) & 3u;
          if (head > b1 - b0) head = b1 - b0;
          if (lane < head) to[lane] = s_stage[b0 + lane];
          const unsigned words = (b1 - b0 - head) >> 2;
          for (unsigned w = lane; w < words; w += 32) {
            const unsigned char* sp = s_stage + b0 + head + 4 * w;
            const unsigned v = unsigned(sp[0]) | (unsigned(sp[1]) << 8) | (unsigned(sp[2]) << 16) | (unsigned(sp[3]) << 24);
            *reinterpret_cast<unsigned*>(to + head + 4 * w) = v;
          }
          const unsigned done = head + 4 * words;
          if (lane < (b1 - b0) - done) to[done + lane] = s_stage[b0 + done + lane];
        }
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int sx = tid + k * PT_THREADS;
        if (sx < rows) {
          const unsigned p = s_pid[sx];
          dest[p].off[u][int64_t(s_run[p]) + (sx - int(s_seg[p]))] = s_offv[sx];
        }
      }
      __syncthreads();  // s_offv aliases the source staging area of the next column / tile
      for (int p = tid; p < P; p += PT_THREADS) s_runb[u * P + p] += s_sege[p] - s_segb[p];
    }
    __syncthreads();
    for (int p = tid; p < P; p += PT_THREADS) s_run[p] += s_tot[p];
  }
}

// ================================================================================================
// host: steps 1, 2 and 4
// ================================================================================================
std::vector<int> routing_columns(const Table& in, const std::vector<int>& keys) {
  std::vector<int> fixed;
  for (int k : keys)
    if (in.cols[k].dtype != FLOCKGPU_UTF8) fixed.push_back(k);
  return fixed.empty() ? keys : fixed;
}

PartPass partition_count_scan(const CtxPtr& ctx, const Table& in, const std::vector<int>& routing_cols, int n_parts, int dest_rank, int digit_col,
                              int digit_shift, bool ship_nullable) {
  FG_CHECK(n_parts >= 1 && n_parts <= PT_MAX_PARTS, FLOCKGPU_ERR_INVALID, "hash_partition: n_parts must be in [1, %d], got %d", PT_MAX_PARTS, n_parts);
  FG_CHECK(in.cols.size() <= size_t(MAX_IN_COLS), FLOCKGPU_ERR_UNSUPPORTED, "hash_partition: more than %d columns", MAX_IN_COLS);
  FG_CHECK(dest_rank >= 0 || digit_col >= 0 || (!routing_cols.empty() && routing_cols.size() <= size_t(MAX_KEY_COLS)), FLOCKGPU_ERR_INVALID,
           "hash_partition: 1..%d key columns", MAX_KEY_COLS);
  PartPass ps;
  ps.n_rows = in.num_rows;
  ps.n_parts = n_parts;
  for (size_t i = 0; i < in.cols.size(); ++i) {
    FG_CHECK(!in.cols[i].all_null, FLOCKGPU_ERR_UNSUPPORTED, "hash_partition: NULL column \"%s\"", in.cols[i].name.c_str());
    if (in.cols[i].dtype == FLOCKGPU_UTF8) ps.utf8_cols.push_back(int(i));
    else {
      FG_CHECK(in.cols[i].width() == 4 || in.cols[i].width() == 8, FLOCKGPU_ERR_UNSUPPORTED, "hash_partition: column width %d", in.cols[i].width());
      ps.fixed_cols.push_back(int(i));
    }
  }
  FG_CHECK(ps.utf8_cols.size() <= size_t(PT_MAX_UTF8), FLOCKGPU_ERR_UNSUPPORTED, "hash_partition: more than %d Utf8 columns", PT_MAX_UTF8);
  for (size_t i = 0; i < in.cols.size(); ++i) {
    const Column& c = in.cols[i];
    if (!c.validity && !(ship_nullable && c.nullable)) continue;
    ps.valid_cols.push_back(int(i));
    if (c.validity) {
      ps.valid_src.push_back(c.validity);
    } else {
      BufferPtr ones = alloc(ctx, size_t(std::max<int64_t>(in.num_rows, 1)));
      FG_CUDA(cudaMemsetAsync(ones->ptr, 1, size_t(std::max<int64_t>(in.num_rows, 1)), ctx->stream));
      ps.valid_src.push_back(ones);
    }
  }
  FG_CHECK(ps.fixed_cols.size() + ps.valid_cols.size() <= size_t(MAX_IN_COLS), FLOCKGPU_ERR_UNSUPPORTED, "hash_partition: more than %d value + validity columns",
           MAX_IN_COLS);
  const int U = int(ps.utf8_cols.size());
  // geometry: as many CTAs as stay resident, each owning a contiguous, tile-aligned range of rows
  const ScatterSmem L(n_parts, U, n_parts <= PT_DEST_SMEM_PARTS);
  FG_CUDA(cudaFuncSetAttribute(partition_scatter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(L.total)));
  const int64_t resident = resident_ctas(ctx, reinterpret_cast<const void*>(partition_scatter_kernel), PT_THREADS, L.total);
  // neither the count nor the scatter kernel waits for another CTA, so several waves are fine: small chunks keep
  // every SM busy on relations of a few million rows (2.5 M persons are 1221 tiles)
  const int64_t tiles = std::max<int64_t>(1, (ps.n_rows + PT_TILE - 1) / PT_TILE);
  const int64_t tiles_per_cta = (tiles + resident * 4 - 1) / (resident * 4);
  ps.chunk = tiles_per_cta * PT_TILE;
  ps.grid = int((tiles + tiles_per_cta - 1) / tiles_per_cta);
  const size_t cells = size_t(1 + U) * ps.grid * n_parts;
  ps.pid = alloc(ctx, size_t(ps.n_rows) + 16);
  ps.hist = alloc(ctx, cells * 4);
  ps.cta_pos = alloc(ctx, cells * 4);
  ps.totals = alloc(ctx, size_t(1 + U) * n_parts * 8);
  ps.dest = alloc(ctx, size_t(n_parts) * sizeof(PartDest));

  PartCountArgs ca{};
  ca.n_rows = ps.n_rows;
  ca.chunk = ps.chunk;
  ca.n_parts = n_parts;
  ca.dest_rank = dest_rank;
  ca.digit_col = digit_col;
  ca.digit_shift = digit_shift;
  ca.n_utf8 = U;
  ca.grid = ps.grid;
  fill_colrefs(in, ca.cols);
  if (dest_rank < 0 && digit_col < 0) {
    std::vector<int> widths;
    for (int k : routing_cols) {
      FG_CHECK(k >= 0 && k < int(in.cols.size()), FLOCKGPU_ERR_INVALID, "hash_partition: key column %d out of range", k);
      widths.push_back(in.cols[k].width());
    }
    ca.packed = keys_packable(widths.data(), int(widths.size())) ? 1 : 0;
    for (int k : routing_cols)
      if (in.cols[k].validity) ca.key_nulls = 1;  // a NULL key routes by hash_row's fixed NULL contribution, not by the bytes underneath
    ca.rk.n = int(routing_cols.size());
    for (size_t i = 0; i < routing_cols.size(); ++i) ca.rk.col[i] = routing_cols[i];
    if (ca.packed) {
      ca.pack.n = int(routing_cols.size());
      for (size_t i = 0; i < routing_cols.size(); ++i) {
        ca.pack.col[i] = routing_cols[i];
        ca.pack.width[i] = widths[i];
      }
    }
  }
  for (int u = 0; u < U; ++u) ca.uoff[u] = in.cols[ps.utf8_cols[u]].offs();
  ca.pid = ps.pid->as<uint8_t>();
  ca.hist = ps.hist->as<uint32_t>();
  const size_t count_smem = size_t(PT_WARPS + U) * n_parts * 4;
  // few destinations (an exchange): the CTA that finishes last also scans -- one launch, no 1-CTA kernel in the chain
  static const bool no_fused_scan = getenv("FLOCKGPU_NO_FUSED_SCAN") != nullptr;
  const bool fused_scan = !no_fused_scan && (1 + U) * n_parts <= PT_FUSED_SCAN_COLS;
  if (fused_scan) {
    ca.arrive = reinterpret_cast<unsigned*>(ctx->d_scalars + kPartitionArriveSlot);
    // (the last CTA leaves the word at zero, but a launch that died half-way would not: never trust it)
    FG_CUDA(cudaMemsetAsync(ca.arrive, 0, 8, ctx->stream));
    ca.cta_pos = ps.cta_pos->as<uint32_t>();
    ca.totals = ps.totals->as<unsigned long long>();
  }
  {
    LaunchTimer lt(ctx, "partition_count_kernel");
    partition_count_kernel<<<ps.grid, PT_THREADS, count_smem, ctx->stream>>>(ca);
  }
  FG_CUDA(cudaGetLastError());
  count_launch(ctx);
  if (!fused_scan) {
    {
      LaunchTimer lt(ctx, "partition_scan_kernel");
      partition_scan_kernel<<<1, 1024, 0, ctx->stream>>>(ps.hist->as<uint32_t>(), ps.cta_pos->as<uint32_t>(), ps.totals->as<unsigned long long>(), ps.grid,
                                                         n_parts, 1 + U);
    }
    FG_CUDA(cudaGetLastError());
    count_launch(ctx);
  }
  return ps;
}

void partition_scatter(const CtxPtr& ctx, const Table& in, const PartPass& ps, const unsigned* abort_flag) {
  const int U = int(ps.utf8_cols.size());
  PartScatterArgs sa{};
  sa.n_rows = ps.n_rows;
  sa.chunk = ps.chunk;
  sa.n_parts = ps.n_parts;
  sa.n_fixed = int(ps.fixed_cols.size());
  sa.n_utf8 = U;
  sa.grid = ps.grid;
  sa.pid = ps.pid->as<uint8_t>();
  for (size_t f = 0; f < ps.fixed_cols.size(); ++f) {
    sa.fsrc[f] = in.cols[ps.fixed_cols[f]].values();
    sa.fwidth[f] = in.cols[ps.fixed_cols[f]].width();
  }
  for (size_t k = 0; k < ps.valid_cols.size(); ++k) {  // validity bytes: one more column of width 1 each
    sa.fsrc[ps.fixed_cols.size() + k] = ps.valid_src[k]->ptr;
    sa.fwidth[ps.fixed_cols.size() + k] = 1;
  }
  sa.n_fixed = int(ps.fixed_cols.size() + ps.valid_cols.size());
  for (int u = 0; u < U; ++u) {
    sa.uoff[u] = in.cols[ps.utf8_cols[u]].offs();
    sa.udata[u] = static_cast<const uint8_t*>(in.cols[ps.utf8_cols[u]].values());
  }
  sa.cta_pos = ps.cta_pos->as<uint32_t>();
  sa.dest = ps.dest->as<PartDest>();
  sa.abort_flag = abort_flag;
  const ScatterSmem L(ps.n_parts, U, ps.n_parts <= PT_DEST_SMEM_PARTS);
  if (ps.n_rows > 0) {
    {
      LaunchTimer lt(ctx, "partition_scatter_kernel");
      partition_scatter_kernel<<<ps.grid, PT_THREADS, L.total, ctx->stream>>>(sa);
    }
    FG_CUDA(cudaGetLastError());
    count_launch(ctx);
  }
}

// ================================================================================================
// one GPU: the partitions one behind the other in local buffers, handed out as views
// ================================================================================================
// Partition p starts at row base[p] of every output column: base[0] = 0, base[p + 1] = align4(base[p] + rows[p] + 1).
// The alignment keeps 16-byte vector loads working on a view; the spare row keeps the terminal offsets entry of a
// Utf8 partition apart from the first entry of the next one.
__host__ __device__ __forceinline__ unsigned long long next_partition_base(unsigned long long base, unsigned long long rows) {
  return (base + rows + 1 + 3) & ~3ull;
}

struct PlaceLocalArgs {
  int32_t n_parts, n_fixed, n_utf8, dense;  // dense: partitions back to back, no alignment gaps (radix-sort passes)
  const unsigned long long* totals;  // [(1 + n_utf8)][n_parts]
  void* fdst[MAX_IN_COLS];
  int32_t fwidth[MAX_IN_COLS];
  int32_t* uoff_dst[PT_MAX_UTF8];
  uint8_t* ubytes_dst[PT_MAX_UTF8];
  PartDest* dest;
};

__global__ void partition_place_local_kernel(const __grid_constant__ PlaceLocalArgs a) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  unsigned long long base = 0;
  unsigned long long byte_base[PT_MAX_UTF8] = {};
  for (int p = 0; p < a.n_parts; ++p) {
    const unsigned long long rows = a.totals[p];
    PartDest d{};
    for (int f = 0; f < a.n_fixed; ++f) d.val[f] = static_cast<char*>(a.fdst[f]) + base * a.fwidth[f];
    for (int u = 0; u < a.n_utf8; ++u) {
      const unsigned long long bytes = a.totals[(1 + u) * a.n_parts + p];
      d.off[u] = a.uoff_dst[u] + base;
      d.bytes[u] = a.ubytes_dst[u] + byte_base[u];
      d.byte_origin[u] = 0;  // a partition's offsets are relative to its own view of the value bytes
      a.uoff_dst[u][base + rows] = int32_t(bytes);  // terminal entry (also the only entry of an empty partition)
      byte_base[u] += bytes;
    }
    a.dest[p] = d;
    base = a.dense ? base + rows : next_partition_base(base, rows);
  }
}

std::vector<TablePtr> hash_partition(const CtxPtr& ctx, const TablePtr& in_ptr, const std::vector<int>& keys, int n_parts) {
  const Table& in = *in_ptr;
  in.dense();
  FG_CHECK(n_parts >= 1 && n_parts <= PT_MAX_PARTS, FLOCKGPU_ERR_INVALID, "hash_partition: n_parts must be in [1, %d], got %d", PT_MAX_PARTS, n_parts);
  FG_CHECK(!keys.empty() && keys.size() <= size_t(MAX_KEY_COLS), FLOCKGPU_ERR_INVALID, "hash_partition: 1..%d key columns", MAX_KEY_COLS);
  for (int k : keys) {
    FG_CHECK(k >= 0 && k < int(in.cols.size()), FLOCKGPU_ERR_INVALID, "hash_partition: key column %d out of range", k);
    FG_CHECK(!in.cols[k].all_null, FLOCKGPU_ERR_UNSUPPORTED, "hash_partition: NULL key column");
  }
  std::vector<TablePtr> out;
  if (n_parts == 1) {
    out.push_back(in_ptr);
    return out;
  }
  if (in.num_rows == 0) {
    for (int p = 0; p < n_parts; ++p) out.push_back(empty_like(ctx, in));
    return out;
  }
  const int64_t n = in.num_rows;
  PartPass ps = partition_count_scan(ctx, in, routing_columns(in, keys), n_parts);
  const int U = int(ps.utf8_cols.size());
  // ---- output buffers: every column once, partitions one behind the other (5 spare rows per partition at most)
  const size_t cap_rows = size_t(n) + 5 * size_t(n_parts) + 4;
  std::vector<BufferPtr> fbuf(ps.fixed_cols.size()), obuf(U), bbuf(U), vbuf(ps.valid_cols.size());
  PlaceLocalArgs pa{};
  pa.n_parts = n_parts;
  pa.n_fixed = int(ps.fixed_cols.size() + ps.valid_cols.size());
  for (size_t k = 0; k < ps.valid_cols.size(); ++k) {
    vbuf[k] = alloc(ctx, cap_rows);
    pa.fdst[ps.fixed_cols.size() + k] = vbuf[k]->ptr;
    pa.fwidth[ps.fixed_cols.size() + k] = 1;
  }
  pa.n_utf8 = U;
  pa.totals = ps.totals->as<unsigned long long>();
  for (size_t f = 0; f < ps.fixed_cols.size(); ++f) {
    const int w = in.cols[ps.fixed_cols[f]].width();
    fbuf[f] = alloc(ctx, cap_rows * w);
    pa.fdst[f] = fbuf[f]->ptr;
    pa.fwidth[f] = w;
  }
  for (int u = 0; u < U; ++u) {
    obuf[u] = alloc(ctx, cap_rows * 4);
    bbuf[u] = alloc(ctx, size_t(in.cols[ps.utf8_cols[u]].values_bytes));
    pa.uoff_dst[u] = obuf[u]->as<int32_t>();
    pa.ubytes_dst[u] = bbuf[u]->as<uint8_t>();
  }
  pa.dest = ps.dest->as<PartDest>();
  {
    LaunchTimer lt(ctx, "partition_place_local_kernel");
    partition_place_local_kernel<<<1, 32, 0, ctx->stream>>>(pa);
  }
  FG_CUDA(cudaGetLastError());
  count_launch(ctx);
  partition_scatter(ctx, in, ps, nullptr);
  // ---- the partition sizes are the one thing the host needs: views are cut from them
  std::vector<unsigned long long> tot(size_t(1 + U) * n_parts);
  FG_CUDA(cudaMemcpyAsync(tot.data(), ps.totals->ptr, tot.size() * 8, cudaMemcpyDeviceToHost, ctx->stream));
  FG_CUDA(cudaStreamSynchronize(ctx->stream));
  unsigned long long sum = 0;
  for (int p = 0; p < n_parts; ++p) sum += tot[p];
  FG_CHECK(int64_t(sum) == n, FLOCKGPU_ERR_CUDA, "hash_partition: partition sizes sum to %llu, expected %lld", sum, (long long)n);
  unsigned long long base = 0;
  std::vector<unsigned long long> byte_base(U, 0);
  for (int p = 0; p < n_parts; ++p) {
    const int64_t rows = int64_t(tot[p]);
    auto t = std::make_shared<Table>();
    t->ctx = ctx;
    t->metadata = in.metadata;
    t->num_rows = rows;
    t->cols.resize(in.cols.size());
    for (size_t f = 0; f < ps.fixed_cols.size(); ++f) {
      const Column& src = in.cols[ps.fixed_cols[f]];
      Column& c = t->cols[ps.fixed_cols[f]];
      c.dtype = src.dtype;
      c.name = src.name;
      c.format = src.format;
      c.nullable = src.nullable;
      c.length = rows;
      c.data = view_of(fbuf[f], size_t(base) * src.width(), size_t(rows) * src.width());
    }
    for (int u = 0; u < U; ++u) {
      const Column& src = in.cols[ps.utf8_cols[u]];
      Column& c = t->cols[ps.utf8_cols[u]];
      const unsigned long long bytes = tot[size_t(1 + u) * n_parts + p];
      c.dtype = src.dtype;
      c.name = src.name;
      c.format = src.format;
      c.nullable = src.nullable;
      c.length = rows;
      c.offsets = view_of(obuf[u], size_t(base) * 4, size_t(rows + 1) * 4);
      c.data = view_of(bbuf[u], size_t(byte_base[u]), size_t(bytes));
      c.values_bytes = int64_t(bytes);
      byte_base[u] += bytes;
    }
    for (size_t k = 0; k < ps.valid_cols.size(); ++k) t->cols[ps.valid_cols[k]].validity = view_of(vbuf[k], size_t(base), size_t(rows));
    out.push_back(std::move(t));
    base = next_partition_base(base, tot[p]);
  }
  return out;
}

// One stable radix pass: the rows of `in` (fixed-width columns only) reordered by byte `shift / 8` of the UInt64 column
// `digit_col`, ties in input order -- the multi-way partition with 256 destinations laid out back to back (sort.cu).
TablePtr radix_pass(const CtxPtr& ctx, const TablePtr& in_ptr, int digit_col, int shift) {
  const Table& in = *in_ptr;
  const int64_t n = in.num_rows;
  if (n <= 1) return in_ptr;
  PartPass ps = partition_count_scan(ctx, in, {}, 256, -1, digit_col, shift);
  FG_CHECK(ps.utf8_cols.empty(), FLOCKGPU_ERR_UNSUPPORTED, "radix_pass: Utf8 columns");
  auto t = std::make_shared<Table>();
  t->ctx = ctx;
  t->metadata = in.metadata;
  t->num_rows = n;
  t->cols.resize(in.cols.size());
  PlaceLocalArgs pa{};
  pa.n_parts = 256;
  pa.n_fixed = int(ps.fixed_cols.size());
  pa.n_utf8 = 0;
  pa.dense = 1;
  pa.totals = ps.totals->as<unsigned long long>();
  for (size_t f = 0; f < ps.fixed_cols.size(); ++f) {
    const Column& src = in.cols[ps.fixed_cols[f]];
    Column& c = t->cols[ps.fixed_cols[f]];
    c = src;
    c.data = alloc(ctx, size_t(n) * src.width());
    pa.fdst[f] = c.data->ptr;
    pa.fwidth[f] = src.width();
  }
  pa.dest = ps.dest->as<PartDest>();
  {
    LaunchTimer lt(ctx, "partition_place_local_kernel");
    partition_place_local_kernel<<<1, 32, 0, ctx->stream>>>(pa);
  }
  FG_CUDA(cudaGetLastError());
  count_launch(ctx);
  partition_scatter(ctx, in, ps, nullptr);
  return t;
}

}  // namespace fg

using namespace fg;

extern "C" int flockgpu_hash_partition(flockgpu_ctx* ctx, const flockgpu_table* in, const int32_t* key_cols, int32_t n_keys, int32_t n_parts,
                                       flockgpu_table** out_parts) {
  return guarded([&] {
    auto c = core_of(ctx);
    FG_CHECK(out_parts && in && in->table && key_cols && n_keys > 0, FLOCKGPU_ERR_INVALID, "hash_partition: null or empty argument");
    std::lock_guard<std::recursive_mutex> g(c->mu);
    FG_CUDA(cudaSetDevice(c->device));
    std::vector<int> keys(key_cols, key_cols + n_keys);
    std::vector<TablePtr> parts = hash_partition(c, in->table, keys, n_parts);
    for (int p = 0; p < n_parts; ++p) out_parts[p] = wrap_table(parts[p]);
  });
}
