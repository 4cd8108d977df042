// dim_count.cu -- K13: COUNT(*) of an inner join with a small dimension, grouped by dimension columns, in one pass.
//
// Shape (YSB, benchmarks/src/ysb/ysb.sql): SELECT campaign_id, COUNT(*) FROM ad_event JOIN campaign ON ad_id = c_ad_id
// WHERE event_type = 'view' GROUP BY campaign_id.  Millions of fact rows, filtered, join a dimension of ~1 000 rows and
// end up as ~100 counters.  The generic path writes the surviving keys (K1 + K4), probes the join table with row
// comparisons (K3), gathers the group string of every joined row (K4) and hashes it again (K6).  None of those rows is
// needed: each fact row adds one to the counter of every dimension row it joins.  So:
//   dim_count_build_kernel  the dimension's keys into a hash table of dimension rows (HBM, `cap` 32-bit slots)
//   dim_count_kernel        ONE launch over the fact relation.  Every CTA copies the table into shared memory next to
//                           one 32-bit counter per dimension row; per fact row it evaluates the fact's filter predicate
//                           (the K1 interpreter, eval_predicate), and only for a row that passes reads its key, hashes
//                           it, probes the table and confirms equality against the dimension's key column (rows_equal);
//                           every equal dimension row gets one increment (duplicate dimension keys: the join's cross
//                           product).  The CTA adds its counters into a uint64 count per dimension row at the end.
// The plan layer (HashAggregateExec) then selects the dimension rows with a count above zero (K1) and groups them by
// the group columns, summing the counts (K6): ~1 000 rows, whatever the size of the fact relation.
//
// NULLs (DESIGN §3): a NULL predicate drops the row (Kleene table of the interpreter); a NULL key on either side
// matches nothing (NULL dimension keys never enter the table, NULL fact keys are not probed); a NULL group value is a
// group of its own (the grouping step compares validity).
//
// Counter widths: a fact row increments a given dimension row's counter at most once (one slot per dimension row), so a
// CTA's 32-bit counter never exceeds the rows the CTA scanned since its last flush, and the CTA flushes before that
// number could pass 2^32 - 1.  The uint64 totals are bounded by the fact's row count.
#include <algorithm>

#include "expr_compile.h"
#include "internal.h"
#include "rowkeys.cuh"

namespace fg {

constexpr int DC_THREADS = 256;
constexpr int DC_ROWS = 2;                   // fact rows per thread per tile (the interpreter evaluates them together)
constexpr int DC_MIN_CTAS = 4;               // 48 KiB of shared memory each at D_MAX: four fit an SM; <= 64 registers
constexpr int DC_TILE = DC_THREADS * DC_ROWS;
constexpr int DC_ROW_BITS = 13;              // slot word = tag << 13 | (dimension row + 1); row + 1 <= 4096 < 2^13
static_assert(DIM_COUNT_MAX_ROWS < (1 << DC_ROW_BITS), "a dimension row index must fit the slot word");

__device__ __forceinline__ unsigned dc_slot_word(unsigned long long h, unsigned row) {
  return unsigned(h >> (64 - (32 - DC_ROW_BITS))) << DC_ROW_BITS | (row + 1u);  // tag: the hash's top 19 bits
}

struct DimBuildArgs {
  int32_t n_dim, cap;  // cap: a power of two >= 2 n_dim
  unsigned* table;     // [cap], zeroed: 0 = free
  RowKeys key;         // one column: cols[0]
  ColRef cols[1];
};

__global__ void __launch_bounds__(256) dim_count_build_kernel(const __grid_constant__ DimBuildArgs a) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < a.n_dim; r += gridDim.x * blockDim.x) {
    if (a.cols[0].validity && !a.cols[0].validity[r]) continue;  // a NULL key matches nothing
    const unsigned long long h = hash_row(a.key, a.cols, r);
    const unsigned word = dc_slot_word(h, unsigned(r));
    unsigned slot = unsigned(h) & unsigned(a.cap - 1);
    while (atomicCAS(&a.table[slot], 0u, word) != 0u) slot = (slot + 1u) & unsigned(a.cap - 1);
  }
}

struct DimCountArgs {
  int64_t n_fact;
  int32_t n_dim, cap;
  int32_t has_pred, pad;
  const unsigned* table;          // [cap] from dim_count_build_kernel
  unsigned long long* counts;     // [n_dim], zeroed: matches per dimension row
  RowKeys fact_key;               // one column of fact_cols
  RowKeys dim_key;                // cols[0] of dim_cols
  ColRef dim_cols[1];
  ColRef fact_cols[MAX_IN_COLS];
  Predicate pred;                 // the fact's filter (has_pred)
};

__global__ void __launch_bounds__(DC_THREADS, DC_MIN_CTAS) dim_count_kernel(const __grid_constant__ DimCountArgs a) {
  extern __shared__ unsigned dc_smem[];
  unsigned* tab = dc_smem;             // [cap]
  unsigned* cnt = dc_smem + a.cap;     // [n_dim]
  const int tid = threadIdx.x;
  for (int i = tid; i < a.cap; i += DC_THREADS) tab[i] = a.table[i];
  for (int i = tid; i < a.n_dim; i += DC_THREADS) cnt[i] = 0u;
  __syncthreads();
  const unsigned mask = unsigned(a.cap - 1);
  const ColRef& fk = a.fact_cols[a.fact_key.col[0]];
  auto flush = [&] {
    __syncthreads();
    for (int i = tid; i < a.n_dim; i += DC_THREADS) {
      const unsigned c = cnt[i];
      if (c) {
        atomicAdd(&a.counts[i], (unsigned long long)c);
        cnt[i] = 0u;
      }
    }
    __syncthreads();
  };
  unsigned long long since_flush = 0;  // fact rows this CTA scanned since its counters were last flushed
  int err = 0;                         // (the plan layer keeps predicates that can divide by zero out of this kernel)
  for (int64_t base = int64_t(blockIdx.x) * DC_TILE; base < a.n_fact; base += int64_t(gridDim.x) * DC_TILE) {
    if (since_flush + DC_TILE > 0xffffffffull) {
      flush();
      since_flush = 0;
    }
    since_flush += DC_TILE;
    int64_t rows[DC_ROWS];
    unsigned sel = 0;
#pragma unroll
    for (int k = 0; k < DC_ROWS; ++k) {
      const int64_t r = base + int64_t(k) * DC_THREADS + tid;
      rows[k] = r < a.n_fact ? r : -1;
      if (r < a.n_fact) sel |= 1u << k;
    }
    if (a.has_pred) sel = eval_predicate<DC_ROWS>(a.pred, a.fact_cols, rows, &err);
#pragma unroll
    for (int k = 0; k < DC_ROWS; ++k) {
      if (!((sel >> k) & 1u)) continue;
      const int64_t row = rows[k];
      if (fk.validity && !fk.validity[row]) continue;  // a NULL key matches nothing
      const unsigned long long h = hash_row(a.fact_key, a.fact_cols, row);
      const unsigned tag = dc_slot_word(h, 0u) >> DC_ROW_BITS;
      for (unsigned slot = unsigned(h) & mask;; slot = (slot + 1u) & mask) {
        const unsigned w = tab[slot];
        if (w == 0u) break;
        if ((w >> DC_ROW_BITS) != tag) continue;
        const unsigned d = (w & ((1u << DC_ROW_BITS) - 1u)) - 1u;
        if (rows_equal(a.dim_key, a.dim_cols, d, a.fact_key, a.fact_cols, row)) atomicAdd(&cnt[d], 1u);
      }
    }
  }
  flush();
}

// ------------------------------------------------------------------------------------------------
bool dim_count_key_type(int dtype) {
  return dtype == FLOCKGPU_INT32 || dtype == FLOCKGPU_DATE32 || dtype == FLOCKGPU_INT64 || dtype == FLOCKGPU_UINT64 || dtype == FLOCKGPU_TIMESTAMP || dtype == FLOCKGPU_UTF8;
}

TablePtr dim_count_aggregate(const CtxPtr& ctx, const TablePtr& fact_ptr, int fact_key, const Expr* predicate, const TablePtr& dim_ptr, int dim_key,
                             const std::vector<int>& group_cols, const std::vector<std::string>& count_names, const std::string& metadata) {
  const Table& fact = *fact_ptr;
  const Table& dim = *dim_ptr;
  fact.dense();
  dim.dense();
  FG_CHECK(dim.num_rows <= DIM_COUNT_MAX_ROWS, FLOCKGPU_ERR_INVALID, "dim_count: %lld dimension rows exceed %lld", (long long)dim.num_rows,
           (long long)DIM_COUNT_MAX_ROWS);
  FG_CHECK(fact.cols.size() <= size_t(MAX_IN_COLS), FLOCKGPU_ERR_UNSUPPORTED, "dim_count: more than %d fact columns", MAX_IN_COLS);
  const Column& fk = fact.cols[fact_key];
  const Column& dk = dim.cols[dim_key];
  check_join_key_types("dim_count", fk, dk);
  FG_CHECK(dim_count_key_type(fk.dtype), FLOCKGPU_ERR_UNSUPPORTED, "dim_count: key type %s", dtype_name(fk.dtype));
  const int n_dim = int(dim.num_rows);
  BufferPtr counts = alloc(ctx, size_t(std::max(n_dim, 1)) * 8);
  FG_CUDA(cudaMemsetAsync(counts->ptr, 0, size_t(std::max(n_dim, 1)) * 8, ctx->stream));
  if (n_dim > 0 && fact.num_rows > 0) {
    int cap = 64;
    while (cap < 2 * n_dim) cap <<= 1;
    BufferPtr table = alloc(ctx, size_t(cap) * 4);
    FG_CUDA(cudaMemsetAsync(table->ptr, 0, size_t(cap) * 4, ctx->stream));
    DimBuildArgs b{};
    b.n_dim = n_dim;
    b.cap = cap;
    b.table = table->as<unsigned>();
    b.key.n = 1;
    b.key.col[0] = 0;
    b.cols[0] = colref_of(dk);
    {
      LaunchTimer lt(ctx, "dim_count_build_kernel");
      dim_count_build_kernel<<<(n_dim + 255) / 256, 256, 0, ctx->stream>>>(b);
    }
    FG_CUDA(cudaGetLastError());
    count_launch(ctx);

    DimCountArgs a{};
    a.n_fact = fact.num_rows;
    a.n_dim = n_dim;
    a.cap = cap;
    a.table = table->as<unsigned>();
    a.counts = counts->as<unsigned long long>();
    a.fact_key.n = 1;
    a.fact_key.col[0] = fact_key;
    a.dim_key = b.key;
    a.dim_cols[0] = b.cols[0];
    fill_colrefs(fact, a.fact_cols);
    if (predicate) {
      CompiledPredicate cp = compile_predicate(*predicate, col_infos(fact));
      // the kernel never reports a division by zero
      FG_CHECK(!cp.prog.has_div_by_col, FLOCKGPU_ERR_INVALID, "dim_count: a predicate that divides by a column stays in its own filter");
      a.has_pred = 1;
      a.pred = cp.prog;
    }
    const size_t smem = size_t(cap + n_dim) * 4;  // <= 48 KiB at D_MAX: no opt-in needed
    const int64_t tiles = (fact.num_rows + DC_TILE - 1) / DC_TILE;
    const int grid = int(std::max<int64_t>(1, std::min<int64_t>(tiles, resident_ctas(ctx, reinterpret_cast<const void*>(dim_count_kernel), DC_THREADS, smem))));
    {
      LaunchTimer lt(ctx, "dim_count_kernel");
      dim_count_kernel<<<grid, DC_THREADS, smem, ctx->stream>>>(a);
    }
    FG_CUDA(cudaGetLastError());
    count_launch(ctx);
  }

  // emit: the dimension rows with a count above zero (K1), grouped by the group columns with their counts summed (K6)
  auto counted = std::make_shared<Table>();
  counted->ctx = ctx;
  counted->metadata = metadata;
  counted->num_rows = n_dim;
  std::vector<int> out_groups;
  for (int g : group_cols) {
    out_groups.push_back(int(counted->cols.size()));
    counted->cols.push_back(dim.cols[g]);
  }
  Column c;
  c.name = count_names.at(0);
  c.dtype = FLOCKGPU_UINT64;
  c.format = "L";
  c.length = n_dim;
  c.data = counts;
  const int cnt_col = int(counted->cols.size());
  counted->cols.push_back(std::move(c));
  ExprTok col_tok{}, zero{}, gt{};
  col_tok.op = FLOCKGPU_OP_COLUMN;
  col_tok.col = cnt_col;
  zero.op = FLOCKGPU_OP_LIT_I64;
  zero.dtype = FLOCKGPU_UINT64;
  gt.op = FLOCKGPU_OP_GT;
  const Expr above_zero{col_tok, zero, gt};
  TablePtr matched = filter_project(ctx, counted, &above_zero, {}, {});
  TablePtr grouped = hash_aggregate(ctx, matched, FLOCKGPU_AGG_SINGLE, out_groups, {AggSpec{FLOCKGPU_AGG_SUM, cnt_col, count_names[0]}});
  grouped->resolve();
  auto out = std::make_shared<Table>(*grouped);
  // the group columns keep the dimension's nullability when no row survives (an empty selection carries none)
  for (size_t i = 0; i < group_cols.size(); ++i) out->cols[i].nullable = dim.cols[group_cols[i]].nullable;
  for (size_t i = 1; i < count_names.size(); ++i) {  // COUNT(*) listed again: the same values under its own name
    Column again = out->cols[group_cols.size()];
    again.name = count_names[i];
    out->cols.push_back(std::move(again));
  }
  return out;
}

}  // namespace fg
