// sort.cu -- SortExec, WindowAggExec(ROW_NUMBER) and GlobalLimitExec: what NEXMark q6 adds to the operator set
// (benchmarks/src/nexmark/query/q6.sql, q6_plan.fmt; flock-function/src/aws/arch/ops/sort.sql; the serialised form of
// sort_exec / global_limit_exec is in flock/src/tests/data/plan/join.json).
//
// SortExec    LSD radix sort of a row permutation.  Column by column from the least significant sort key to the
//             most significant one, the column's values become order-preserving UInt64 keys (sign bit flipped for
//             signed integers, the IEEE total order for Float64 (f64_order_key), complemented for DESC) and every byte of the key that
//             actually varies is one stable 256-way partition pass over (key, row) pairs -- the very kernels of
//             RepartitionExec (partition.cu), with the destinations laid out back to back.  Ties the reference leaves
//             undefined are broken by the remaining columns, ascending, in column order: the total order the oracle
//             uses (oracle/__init__.py: sort_batch), so results do not depend on the order the join emitted its rows in.
//             A Utf8 column is a sequence of sub-keys: its length, then its bytes eight at a time as big-endian words.
// ROW_NUMBER  over an input sorted by (PARTITION BY .., ORDER BY ..): rows of a window partition are contiguous, so a
//             row's number is its index minus the index of the first row that carries its partition key -- a binary
//             search per row on "same key as mine" (monotone thanks to contiguity).
// LIMIT n     the first n rows of the (single) partition: a view.
#include <algorithm>

#include "device_utils.cuh"
#include "internal.h"
#include "partition.h"

namespace fg {

// ---- order-preserving UInt64 image of a value ------------------------------------------------------------------------
// Utf8: `chunk` >= 0 selects bytes [8 chunk, 8 chunk + 8) of the string as a big-endian word (zero padded: byte order
// = string order), chunk == -1 the string's length (the last tie-breaker: "a" sorts before "a\0").
__device__ __forceinline__ unsigned long long sortable_u64(const ColRef& c, int64_t row, bool descending, int chunk = 0) {
  unsigned long long k;
  unsigned long long mask = ~0ull;
  if (c.dtype == FLOCKGPU_UTF8) {
    const int32_t lo = c.offsets[row], len = c.offsets[row + 1] - lo;
    if (chunk < 0) {
      k = (unsigned long long)len;
    } else {
      k = 0;
      const uint8_t* p = static_cast<const uint8_t*>(c.data) + lo;
#pragma unroll
      for (int b = 0; b < 8; ++b) {
        const int at = chunk * 8 + b;
        k = (k << 8) | (at < len ? (unsigned long long)p[at] : 0ull);
      }
    }
    return descending ? ~k : k;
  }
  switch (c.dtype) {
    case FLOCKGPU_INT32:
    case FLOCKGPU_DATE32:
      k = (unsigned long long)(static_cast<const uint32_t*>(c.data)[row] ^ 0x80000000u);
      mask = 0xffffffffull;
      break;
    case FLOCKGPU_UINT32:
      k = static_cast<const uint32_t*>(c.data)[row];
      mask = 0xffffffffull;
      break;
    case FLOCKGPU_FLOAT64:
      k = f64_order_key(static_cast<const unsigned long long*>(c.data)[row]);
      break;
    case FLOCKGPU_UINT64:
      k = static_cast<const unsigned long long*>(c.data)[row];
      break;
    default:  // Int64 / Timestamp
      k = static_cast<const unsigned long long*>(c.data)[row] ^ (1ull << 63);
      break;
  }
  return descending ? (~k & mask) : k;
}

// keys[i] = image of col[perm[i]]; or_and[0] |= key, or_and[1] &= key (which bytes of the key vary at all?)
__global__ void __launch_bounds__(256) sort_keys_kernel(ColRef col, const uint32_t* __restrict__ perm, int64_t n, int descending, int chunk,
                                                        unsigned long long* __restrict__ keys, unsigned long long* or_and) {
  unsigned long long o = 0, a = ~0ull;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x) {
    const unsigned long long k = sortable_u64(col, int64_t(perm[i]), descending != 0, chunk);
    keys[i] = k;
    o |= k;
    a &= k;
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    o |= __shfl_xor_sync(FULL_MASK, o, d);
    a &= __shfl_xor_sync(FULL_MASK, a, d);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicOr(or_and, o);
    atomicAnd(or_and + 1, a);
  }
}

__global__ void __launch_bounds__(256) utf8_max_len_kernel(const int32_t* __restrict__ off, int64_t n, unsigned long long* out) {
  unsigned m = 0;
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x) m = max(m, unsigned(off[i + 1] - off[i]));
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) m = max(m, __shfl_xor_sync(FULL_MASK, m, d));
  if ((threadIdx.x & 31) == 0) atomicMax(out, (unsigned long long)m);
}

__global__ void __launch_bounds__(256) iota_kernel(uint32_t* p, int64_t n) {
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < n; i += int64_t(gridDim.x) * blockDim.x) p[i] = uint32_t(i);
}

static int grid_for(const CtxPtr& ctx, int64_t items) {
  return int(std::max<int64_t>(1, std::min<int64_t>((items + 255) / 256, int64_t(ctx->sm_count) * 8)));
}

TablePtr sort_table(const CtxPtr& ctx, const TablePtr& in_ptr, const std::vector<SortKey>& keys) {
  in_ptr->dense();
  const Table& in = *in_ptr;
  const int64_t n = in.num_rows;
  FG_CHECK(!keys.empty(), FLOCKGPU_ERR_INVALID, "sort: no sort expressions");
  FG_CHECK(n < (int64_t(1) << 32) - 1, FLOCKGPU_ERR_UNSUPPORTED, "sort: more than 2^32-2 rows");
  // the total order: the sort expressions, then every other column ascending (ties are undefined in the reference)
  std::vector<SortKey> order = keys;
  for (const SortKey& k : keys) {
    FG_CHECK(k.col >= 0 && k.col < int(in.cols.size()), FLOCKGPU_ERR_INVALID, "sort: column %d out of range", k.col);
  }
  for (int c = 0; c < int(in.cols.size()); ++c) {
    bool used = false;
    for (const SortKey& k : keys) used |= k.col == c;
    if (!used) order.push_back(SortKey{c, false, false});
  }
  for (const SortKey& k : order) {
    const Column& c = in.cols[k.col];
    FG_CHECK(!c.all_null, FLOCKGPU_ERR_UNSUPPORTED, "sort: NULL column \"%s\"", c.name.c_str());
    FG_CHECK(!c.chunks, FLOCKGPU_ERR_INVALID, "sort: host-resident column");
    require_no_nulls(c, "sort");
  }
  if (n <= 1) return in_ptr;

  // (key, row) pairs: column 0 = UInt64 key of the current sort column, column 1 = the permutation so far
  auto pairs = std::make_shared<Table>();
  pairs->ctx = ctx;
  pairs->num_rows = n;
  pairs->cols.resize(2);
  pairs->cols[0].dtype = FLOCKGPU_UINT64;
  pairs->cols[0].format = "L";
  pairs->cols[0].name = "key";
  pairs->cols[0].length = n;
  pairs->cols[0].data = alloc(ctx, size_t(n) * 8);
  pairs->cols[1].dtype = FLOCKGPU_UINT32;
  pairs->cols[1].format = "I";
  pairs->cols[1].name = "row";
  pairs->cols[1].length = n;
  pairs->cols[1].data = alloc(ctx, size_t(n) * 4);
  {
    LaunchTimer lt(ctx, "iota_kernel");
    iota_kernel<<<grid_for(ctx, n), 256, 0, ctx->stream>>>(pairs->cols[1].data->as<uint32_t>(), n);
  }
  FG_CUDA(cudaGetLastError());
  count_launch(ctx);
  TablePtr cur = pairs;
  unsigned long long* or_and = ctx->d_scalars + 11;  // [11] OR, [12] AND of the keys
  for (auto it = order.rbegin(); it != order.rend(); ++it) {
    const Column& c = in.cols[it->col];
    ColRef ref{};
    ref.data = c.values();
    ref.offsets = c.offs();
    ref.dtype = c.dtype;
    // the sub-keys of this column, least significant first: a fixed-width column is one word; a Utf8 column is its
    // length, then its 8-byte chunks from the last one to the first
    std::vector<int> chunks{0};
    if (c.dtype == FLOCKGPU_UTF8) {
      FG_CUDA(cudaMemsetAsync(or_and, 0, 8, ctx->stream));
      {
        LaunchTimer lt(ctx, "utf8_max_len_kernel");
        utf8_max_len_kernel<<<grid_for(ctx, n), 256, 0, ctx->stream>>>(c.offs(), n, or_and);
      }
      FG_CUDA(cudaGetLastError());
      count_launch(ctx);
      unsigned long long max_len = 0;
      read_scalars(ctx, 11, 1, &max_len);
      chunks.assign(1, -1);
      for (int ch = int((max_len + 7) / 8) - 1; ch >= 0; --ch) chunks.push_back(ch);
    }
    for (int chunk : chunks) {
      const unsigned long long init[2] = {0ull, ~0ull};
      FG_CUDA(cudaMemcpyAsync(or_and, init, 16, cudaMemcpyHostToDevice, ctx->stream));
      // the keys are rebuilt in the CURRENT order of the permutation (the pair table of the previous sub-key is consumed)
      auto next = std::make_shared<Table>(*cur);
      next->cols[0].data = alloc(ctx, size_t(n) * 8);
      {
        LaunchTimer lt(ctx, "sort_keys_kernel");
        sort_keys_kernel<<<grid_for(ctx, n), 256, 0, ctx->stream>>>(ref, cur->cols[1].data->as<uint32_t>(), n, it->descending ? 1 : 0, chunk,
                                                                   next->cols[0].data->as<unsigned long long>(), or_and);
      }
      FG_CUDA(cudaGetLastError());
      count_launch(ctx);
      unsigned long long oa[2];
      read_scalars(ctx, 11, 2, oa);
      const unsigned long long varying = oa[0] ^ oa[1];  // bit set = not the same in every key
      cur = next;
      for (int shift = 0; shift < 64; shift += 8)
        if ((varying >> shift) & 0xffull) cur = radix_pass(ctx, cur, 0, shift);
    }
  }
  std::vector<int> all;
  for (int c = 0; c < int(in.cols.size()); ++c) all.push_back(c);
  TablePtr out = gather_rows(ctx, in, all, cur->cols[1].data->as<uint32_t>(), n);
  // `cur` must outlive the gather: the block allocator hands its buffers out again in stream order only
  return out;
}

// ---- ROW_NUMBER() OVER (PARTITION BY ...) on an input sorted by the partition columns --------------------------------
struct RowNumberArgs {
  int64_t n;
  int32_t n_keys, pad;
  ColRef key[2];
  unsigned long long* out;
};

__device__ __forceinline__ bool same_partition(const RowNumberArgs& a, int64_t i, int64_t j) {
  for (int k = 0; k < a.n_keys; ++k) {
    const ColRef& c = a.key[k];
    if (c.dtype == FLOCKGPU_INT32 || c.dtype == FLOCKGPU_UINT32 || c.dtype == FLOCKGPU_DATE32) {
      if (static_cast<const uint32_t*>(c.data)[i] != static_cast<const uint32_t*>(c.data)[j]) return false;
    } else if (static_cast<const unsigned long long*>(c.data)[i] != static_cast<const unsigned long long*>(c.data)[j]) {
      return false;
    }
  }
  return true;
}

__global__ void __launch_bounds__(256) row_number_kernel(const __grid_constant__ RowNumberArgs a) {
  for (int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; i < a.n; i += int64_t(gridDim.x) * blockDim.x) {
    // smallest j in [0, i] whose partition key equals row i's: rows of one partition are contiguous, so "equal" is
    // false ... false true ... true over that range.  Gallop backwards first (windows are short), then bisect.
    int64_t hi = i, step = 1;
    while (hi - step >= 0 && same_partition(a, hi - step, i)) {
      hi -= step;
      step <<= 1;
    }
    int64_t lo = hi - step < -1 ? -1 : hi - step;  // lo: known NOT equal (or -1), hi: known equal
    while (hi - lo > 1) {
      const int64_t mid = lo + ((hi - lo) >> 1);
      if (same_partition(a, mid, i)) hi = mid;
      else lo = mid;
    }
    a.out[i] = (unsigned long long)(i - hi + 1);
  }
}

TablePtr row_number(const CtxPtr& ctx, const TablePtr& in_ptr, const std::vector<int>& partition_cols, const std::string& name) {
  in_ptr->dense();
  const Table& in = *in_ptr;
  FG_CHECK(partition_cols.size() <= 2, FLOCKGPU_ERR_UNSUPPORTED, "ROW_NUMBER: more than two PARTITION BY columns");
  RowNumberArgs a{};
  a.n = in.num_rows;
  a.n_keys = int(partition_cols.size());
  for (size_t k = 0; k < partition_cols.size(); ++k) {
    const int c = partition_cols[k];
    FG_CHECK(c >= 0 && c < int(in.cols.size()), FLOCKGPU_ERR_INVALID, "ROW_NUMBER: partition column %d out of range", c);
    FG_CHECK(in.cols[c].dtype != FLOCKGPU_UTF8 && !in.cols[c].all_null, FLOCKGPU_ERR_UNSUPPORTED, "ROW_NUMBER: PARTITION BY column \"%s\" must be fixed width",
             in.cols[c].name.c_str());
    require_no_nulls(in.cols[c], "ROW_NUMBER: PARTITION BY");
    a.key[k].data = in.cols[c].values();
    a.key[k].dtype = in.cols[c].dtype;
  }
  auto out = std::make_shared<Table>();
  out->ctx = ctx;
  out->metadata = in.metadata;
  out->num_rows = in.num_rows;
  out->partitioned_on = in.partitioned_on;
  out->partition_world = in.partition_world;
  Column rn;
  rn.name = name;
  rn.dtype = FLOCKGPU_UINT64;
  rn.format = "L";
  rn.nullable = true;
  rn.length = in.num_rows;
  rn.data = alloc(ctx, size_t(in.num_rows) * 8);
  a.out = rn.data->as<unsigned long long>();
  if (in.num_rows > 0) {
    {
      LaunchTimer lt(ctx, "row_number_kernel");
      row_number_kernel<<<grid_for(ctx, in.num_rows), 256, 0, ctx->stream>>>(a);
    }
    FG_CUDA(cudaGetLastError());
    count_launch(ctx);
  }
  out->cols.push_back(std::move(rn));  // window columns come first (DataFusion's WindowAggExec schema)
  for (const Column& c : in.cols) out->cols.push_back(c);
  return out;
}

TablePtr limit_rows(const CtxPtr& ctx, const TablePtr& in_ptr, int64_t limit) {
  in_ptr->dense();
  const Table& in = *in_ptr;
  FG_CHECK(limit >= 0, FLOCKGPU_ERR_INVALID, "limit: negative row count");
  if (in.num_rows <= limit) return in_ptr;
  // a Utf8 column's byte count is part of its description (export, exchange): with strings the rows are taken, not viewed
  bool has_utf8 = false;
  for (const Column& c : in.cols) has_utf8 |= c.dtype == FLOCKGPU_UTF8;
  if (has_utf8) {
    BufferPtr idx = alloc(ctx, size_t(std::max<int64_t>(limit, 1)) * 4);
    if (limit > 0) {
      LaunchTimer lt(ctx, "iota_kernel");
      iota_kernel<<<grid_for(ctx, limit), 256, 0, ctx->stream>>>(idx->as<uint32_t>(), limit);
      count_launch(ctx);
    }
    std::vector<int> all;
    for (int c = 0; c < int(in.cols.size()); ++c) all.push_back(c);
    return gather_rows(ctx, in, all, idx->as<uint32_t>(), limit);
  }
  auto out = std::make_shared<Table>(in);  // fixed-width columns: the first `limit` rows of the same buffers
  out->num_rows = limit;
  for (Column& c : out->cols) c.length = limit;
  return out;
}

}  // namespace fg

using namespace fg;

extern "C" {

int flockgpu_sort(flockgpu_ctx* ctx, const flockgpu_table* in, const int32_t* cols, const int32_t* descending, int32_t n_keys, flockgpu_table** out) {
  return guarded([&] {
    auto c = core_of(ctx);
    FG_CHECK(out && in && in->table && cols && n_keys > 0, FLOCKGPU_ERR_INVALID, "sort: bad arguments");
    std::lock_guard<std::recursive_mutex> g(c->mu);
    FG_CUDA(cudaSetDevice(c->device));
    std::vector<SortKey> keys;
    for (int i = 0; i < n_keys; ++i) keys.push_back(SortKey{cols[i], descending && descending[i] != 0, false});
    *out = wrap_table(sort_table(c, in->table, keys));
  });
}

int flockgpu_row_number(flockgpu_ctx* ctx, const flockgpu_table* in, const int32_t* partition_cols, int32_t n_cols, const char* name, flockgpu_table** out) {
  return guarded([&] {
    auto c = core_of(ctx);
    FG_CHECK(out && in && in->table && n_cols >= 0 && (n_cols == 0 || partition_cols), FLOCKGPU_ERR_INVALID, "row_number: bad arguments");
    std::lock_guard<std::recursive_mutex> g(c->mu);
    FG_CUDA(cudaSetDevice(c->device));
    std::vector<int> pc(partition_cols, partition_cols + n_cols);
    *out = wrap_table(row_number(c, in->table, pc, name ? name : "ROW_NUMBER()"));
  });
}

int flockgpu_limit(flockgpu_ctx* ctx, const flockgpu_table* in, int64_t limit, flockgpu_table** out) {
  return guarded([&] {
    auto c = core_of(ctx);
    FG_CHECK(out && in && in->table, FLOCKGPU_ERR_INVALID, "limit: bad arguments");
    std::lock_guard<std::recursive_mutex> g(c->mu);
    FG_CUDA(cudaSetDevice(c->device));
    *out = wrap_table(limit_rows(c, in->table, limit));
  });
}

}  // extern "C"
