// internal.h -- host-side C++ types shared by every translation unit of libflockgpu.
//
// Nothing here is part of the ABI (include/flockgpu.h is).  Data model:
//   Ctx      one CUDA device + stream + stream-ordered memory pool + scratch state
//   Buffer   a reference-counted HBM allocation (freed stream-ordered when the last owner drops it)
//   Column   one Arrow column resident in HBM: fixed-width values, or Utf8 = int32 offsets + bytes
//   Table    an immutable relation = columns of equal length (the device form of Vec<RecordBatch>)
#pragma once

#include <cuda_runtime.h>

#include <atomic>
#include <condition_variable>
#include <cstdint>
#include <functional>
#include <thread>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/flockgpu.h"

namespace fg {

// ------------------------------------------------------------------------------------------------
// errors: thrown inside the library, converted to return codes at the extern "C" boundary
// ------------------------------------------------------------------------------------------------
struct Error {
  int code;
  std::string msg;
};
[[noreturn]] void fail(int code, const char* fmt, ...) __attribute__((format(printf, 2, 3)));
void set_last_error(const std::string& msg);

#define FG_CUDA(expr)                                                                          \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess)                                                                     \
      ::fg::fail(FLOCKGPU_ERR_CUDA, "%s:%d: %s -> %s", __FILE__, __LINE__, #expr,              \
                 cudaGetErrorString(_e));                                                      \
  } while (0)

#define FG_CHECK(cond, code, ...)                 \
  do {                                            \
    if (!(cond)) ::fg::fail((code), __VA_ARGS__); \
  } while (0)

// Runs `body` and maps fg::Error / std::exception to an ABI return code.
template <typename F>
int guarded(F&& body) noexcept {
  try {
    body();
    return FLOCKGPU_OK;
  } catch (const Error& e) {
    set_last_error(e.msg);
    return e.code;
  } catch (const std::exception& e) {
    set_last_error(std::string("internal error: ") + e.what());
    return FLOCKGPU_ERR_INVALID;
  } catch (...) {
    set_last_error("internal error: unknown exception");
    return FLOCKGPU_ERR_INVALID;
  }
}

// ------------------------------------------------------------------------------------------------
// context
// ------------------------------------------------------------------------------------------------
struct Comm;  // comm.cc

// Scratch of the single-pass compaction / scan kernels (compact.cuh).  Never reset between launches: tickets are a
// monotonic counter whose base the host tracks, status words carry the launch epoch.
struct ScanScratch {
  unsigned long long* ep_state = nullptr;    // [ep_capacity * stride] {epoch:20, flag:2, value:42}
  unsigned long long* ep_counts = nullptr;   // [ep_capacity] dense epoch-tagged per-tile counts (single-wave mode)
  unsigned* ep_counters = nullptr;           // [0] tickets issued, [1] tiles arrived
  int64_t ep_capacity = 0;
  unsigned tickets_issued = 0, arrived = 0, epoch = 0;
};

// Host threads that stage pageable batch buffers into page-locked memory (core.cu: import_batches).  Kept alive
// between feeds: creating eight threads costs more than copying their share of a 10 M-row relation.
struct StagePool {
  std::vector<std::thread> threads;
  std::mutex mu;
  std::condition_variable wake, idle;
  const std::function<void()>* job = nullptr;
  uint64_t generation = 0;
  int active = 0, running = 0;
  bool stop = false;
  void start(int n, const std::function<void()>* fn);  // the first n workers run *fn once
  void wait();                                         // until all of them have returned
  ~StagePool();
};

struct CtxCore {
  int device = 0;
  cudaStream_t stream = nullptr;
  // H2D fan-out (import_batches): one 256 KB copy per record batch and column leaves microseconds of dead time between
  // dependent copies on ONE stream, far below the link's rate; dealt over several streams they overlap and fill the link.
  static constexpr int kCopyStreams = 4;
  cudaStream_t copy_streams[kCopyStreams] = {};
  cudaEvent_t copy_fork = nullptr, copy_join[kCopyStreams] = {};
  cudaMemPool_t pool = nullptr;
  // Freed device blocks by rounded size.  cudaMallocAsync on the stream-ordered pool takes a microsecond most of the
  // time and milliseconds every so often, which no sub-millisecond query survives; every kernel of a context runs on ONE stream, so a block released by its last owner can be handed to
  // the next operator at once -- stream order does the rest.  Blocks go back to CUDA when the context closes (or
  // when a fresh allocation fails).
  StagePool stage_pool;
  std::mutex block_mu;
  std::unordered_map<size_t, std::vector<void*>> free_blocks;
  size_t cached_bytes = 0;
  void* take_block(size_t rounded);
  void give_block(void* p, size_t rounded);
  void drop_cached_blocks();
  int sm_count = 132;  // replaced by the device's multiProcessorCount when the context opens
  std::recursive_mutex mu;

  // small pinned buffer for device->host scalar read-backs and device scalars
  // d_scalars[0, kScalars): counters / totals written by kernels; read_scalars() mirrors a range into h_scalars at the
  // same indices.  h_scalars[kScalars, kScalars + kPendingSlots): the pinned row-count slots of PendingRows.
  static constexpr int kScalars = 512;
  unsigned long long* h_scalars = nullptr;  // pinned, kScalars + kPendingSlots x u64
  unsigned long long* d_scalars = nullptr;  // device, kScalars x u64

  ScanScratch scan;
  void* l2_flush = nullptr;
  size_t l2_flush_bytes = 0;

  cudaEvent_t timer_start[16] = {};
  cudaEvent_t timer_stop[16] = {};
  std::atomic<int64_t> launches{0};
  // Back-to-back PredI32 filter launches overlap (programmatic dependent launch, compact.cuh: launch_compact_early).
  // overlap_kernel: the kernel of the last launch that its successor may overlap (nullptr: none), with `launches`
  // just before it was enqueued and the Buffer::seq of its outputs.
  const void* overlap_kernel = nullptr;
  int64_t overlap_launches = 0, overlap_outputs = 0;
  int64_t alloc_seq = 0;               // Buffer::seq of new buffers; a filter advances it before it allocates its outputs
  std::atomic<int64_t> overlapped{0};  // launches that took the attribute (flockgpu_overlapped_launches)
  // FLOCKGPU_TRACE: per-tile stamp buffers of the filter launches enqueued since the stream last synchronised
  // (filter_project.cu), written to the trace file at the next synchronising call so that launches may overlap
  struct FilterTrace {
    std::shared_ptr<struct Buffer> stamps;
    long long tiles;
    int grid, rounds, overlapped;
  };
  std::vector<FilterTrace> filter_traces;
  // bytes that crossed the host link on behalf of this context (flockgpu_bytes_moved): copies issued by import /
  // export plus what kernels read in place from page-locked batches (zero-copy feed)
  std::atomic<int64_t> h2d_bytes{0}, d2h_bytes{0};

  // pinned host blocks handed out by flockgpu_host_alloc and by table export
  std::mutex pin_mu;
  std::unordered_map<void*, size_t> pinned;
  // flockgpu_host_alloc sub-allocates from page-locked SLABS: record batches allocated one after the other end up
  // contiguous in one large registration (few, large GPU mappings) instead of thousands of 256 KB registrations --
  // the in-place PCIe read of such batches is markedly slower over 153 separate allocations than over one 40 MB
  // allocation.
  struct PinSlab {
    char* base = nullptr;
    size_t size = 0, used = 0;
    int64_t live = 0;
  };
  static constexpr size_t kPinSlabBytes = size_t(64) << 20;
  std::vector<PinSlab> pin_slabs;
  std::unordered_map<void*, size_t> pin_owner;  // allocation -> slab index

  std::shared_ptr<Comm> comm;  // comm.cc (shared_ptr: Comm is incomplete here)

  // row counts still in flight (see PendingRows): pinned slots h_scalars[kScalars + i]
  static constexpr int kPendingSlots = 256;
  std::weak_ptr<struct PendingRows> pending_owner[kPendingSlots];
  int pending_next = 0;

  // per-kernel CUDA-event profile (flockgpu_profile_begin / _end; bench.py's roofline numerator)
  bool profiling = false;
  struct ProfiledLaunch {
    const char* kernel;
    cudaEvent_t start, stop;
  };
  std::vector<ProfiledLaunch> profile;

  // feed_data_sources keeps page-locked, uniformly batched fixed-width columns in host memory (flockgpu_set_option)
  bool feed_zero_copy = false;
  // with feed_zero_copy: page-lock ordinary (pageable) batch buffers in place at feed time (cudaHostRegister) and
  // release them when the fed relation is dropped -- for callers whose Arrow allocator cannot be hooked
  bool feed_register = false;
  // pageable sources of a copy feed are staged into a page-locked block by this many host threads, each issuing the
  // DMA of a batch as soon as it has copied it (0: hand the pageable pointer to cudaMemcpyAsync)
  int feed_stream_stores = 1;  // non-temporal stores into the staging ring (host/stream_copy.cpp); 0: memcpy
  int feed_stage_threads = 8;  // fewer threads leave the copy short of bandwidth, more contend for memory bandwidth
  // grid-wide prefix protocol of the compaction kernels: 0 = automatic (single wave when every tile is resident,
  // decoupled look-back otherwise), 1 = always decoupled look-back (flockgpu_set_option "compact_mode"; the parity
  // tests run both)
  int compact_mode = 0;
  // size of this rank's NVLink receive window (exchange.cu), fixed when the communicator is attached
  int64_t exchange_window_mb = 4096;

  // recycled CUDA events (creating one costs about a microsecond; a q2 step is one ~10 us kernel)
  std::vector<cudaEvent_t> sync_events;    // cudaEventDisableTiming
  std::vector<cudaEvent_t> timing_events;
  cudaEvent_t get_event(bool timing);
  void put_event(cudaEvent_t e, bool timing) { (timing ? timing_events : sync_events).push_back(e); }

  ~CtxCore();
};
using CtxPtr = std::shared_ptr<CtxCore>;

// Host-side wall time per named span, accumulated process-wide when FLOCKGPU_HOST_TRACE is set and printed to stderr
// by flockgpu_close (where does a 0.3 ms step spend its host time: allocation, waits, launches?).
struct HostSpan {
  const char* name;
  long long t0;
  explicit HostSpan(const char* n);
  ~HostSpan();
};
void host_trace_dump(bool reset);

// RAII: when profiling is on, brackets ONE kernel launch with events on the context stream.
struct LaunchTimer {
  CtxCore* ctx;
  cudaEvent_t stop = nullptr;
  LaunchTimer(const CtxPtr& c, const char* kernel);
  ~LaunchTimer();
};

// A survivor count that a kernel is still producing.  The operator enqueues an async copy of the device
// counter into a pinned slot and returns at once; the first consumer that needs the number waits.
struct PendingRows {
  CtxPtr ctx;
  int slot = 0;
  int64_t h2d_bytes_per_row = 0;  // zero-copy feed: bytes a survivor's pass-through values cost on the host link
  cudaEvent_t ev = nullptr;
  bool done = false;
  int64_t value = 0;
  int64_t wait();
  unsigned long long* host_slot() const;  // pinned (device-accessible) slot the count lands in
  ~PendingRows();
};
// reserve a pinned host slot (the compaction kernel stores the count there itself: CompactScratch::host_count),
// launch, then commit (records the event wait() blocks on)
std::shared_ptr<PendingRows> reserve_row_count(const CtxPtr& ctx);
void commit_row_count(const std::shared_ptr<PendingRows>& p);

struct Buffer {
  CtxPtr ctx;
  void* ptr = nullptr;
  size_t bytes = 0;
  size_t block_bytes = 0;  // size class of an owned block (CtxCore::take_block)
  // ctx->alloc_seq when the buffer was allocated (a view: when its owner was): a launch may read the buffer before the
  // kernel enqueued ahead of it completes only when the buffer is older than that kernel's outputs (compact.cuh)
  int64_t seq = 0;
  // A VIEW (a slice of another allocation: one partition of a partition-ordered relation, a column inside a
  // peer-exchange window) keeps its owner alive through `parent` and frees nothing itself.
  std::shared_ptr<const void> parent;
  Buffer(CtxPtr c, size_t n);
  Buffer(CtxPtr c, void* p, size_t n, std::shared_ptr<const void> owner)
      : ctx(std::move(c)), ptr(p), bytes(n), seq(ctx->alloc_seq), parent(std::move(owner)) {}
  ~Buffer();
  Buffer(const Buffer&) = delete;
  Buffer& operator=(const Buffer&) = delete;
  template <typename T>
  T* as() const {
    return static_cast<T*>(ptr);
  }
};
using BufferPtr = std::shared_ptr<Buffer>;
BufferPtr alloc(const CtxPtr& ctx, size_t bytes);  // bytes == 0 still yields a valid (tiny) buffer
// `bytes` bytes of `b` starting at byte `off`; the caller keeps `off` 16-byte aligned when vector loads will read it
inline BufferPtr view_of(const BufferPtr& b, size_t off, size_t bytes) {
  auto v = std::make_shared<Buffer>(b->ctx, static_cast<char*>(b->ptr) + off, bytes, std::static_pointer_cast<const void>(b));
  v->seq = b->seq;
  return v;
}

// Grid-prefix tuning (FLOCKGPU_LB_STRIDE / FLOCKGPU_LB_SLEEP override): 64-bit words between the look-back words of
// consecutive tiles (32 = one 256-byte L2 chunk each), back-off of a polling thread in ns.
int scan_stride();
int scan_poll_sleep_ns();
// CTAs of `kernel` (block size `threads`, `smem` dynamic shared bytes) that fit on the context's device at once.  The
// occupancy query costs microseconds per call and most kernels here run ~10 us, so the answer is cached per
// (device, kernel, smem): processes that drive unlike GPUs get the right value for each.
int resident_ctas(const CtxPtr& ctx, const void* kernel, int threads, size_t smem = 0);
// Host copy into memory a device reads next (host/stream_copy.cpp).
void stage_copy(void* dst, const void* src, size_t n, int streaming);
// Copies `n` u64 scalars from d_scalars[first..] to the host and waits.
void read_scalars(const CtxPtr& ctx, int first, int n, unsigned long long* out);
// FLOCKGPU_TRACE: writes the stamps of the filter launches enqueued since the last call to the trace file
// (filter_project.cu); called where the stream synchronises anyway.  No-op when there are none.
void dump_filter_traces(const CtxPtr& ctx);

// ------------------------------------------------------------------------------------------------
// columns and tables
// ------------------------------------------------------------------------------------------------
int dtype_width(int dtype);                 // bytes per value; 0 for Utf8
const char* dtype_name(int dtype);
int dtype_from_format(const char* format);  // -1 if unsupported
std::string default_format(int dtype);

// A fixed-width column that still lives in page-locked HOST memory, one chunk per fed record batch.  The filter
// kernel reads such a column straight over PCIe (UVA), so a q2 invocation moves each input byte once and never
// stages the relation in HBM; every other operator materialises it first (Table::dense()).
// Host ranges this library page-locked on behalf of a fed relation (feed_register); released with the last column.
struct HostRegistration {
  std::vector<std::pair<void*, size_t>> ranges;
  ~HostRegistration();
};

struct HostChunks {
  std::shared_ptr<HostRegistration> registration;  // keeps cudaHostRegister'ed sources locked while the column lives
  BufferPtr table;                // device array of chunk base pointers (device-accessible host addresses)
  std::vector<const void*> ptrs;  // the same pointers on the host
  std::vector<int64_t> rows;      // rows per chunk
  int shift = 16;                 // rows per chunk = 1 << shift for every chunk but the last
};

struct Column {
  int dtype = FLOCKGPU_INT32;
  std::string name;
  std::string format;  // Arrow C format string ("i", "tsm:", "u", ...)
  bool nullable = false;
  int64_t length = 0;
  BufferPtr data;      // fixed width: values; Utf8: value bytes (NULL while `chunks` is set)
  std::shared_ptr<HostChunks> chunks;  // host-resident form (zero-copy feed); see HostChunks
  BufferPtr offsets;   // Utf8 only: int32[length + 1]; offsets[0] may be > 0
  int64_t values_bytes = 0;  // Utf8: number of value bytes addressed by offsets
  // The one-row result of a global aggregate over empty input is NULL as a whole (SURVEY App. C.7).
  bool all_null = false;
  // Row-wise NULLs: one byte per row, 1 = valid; no buffer = no NULL in the column.  (Arrow's bit-packed bitmap is
  // expanded at import and packed again at export: every kernel that moves rows moves these bytes like one more
  // 1-byte column.)
  BufferPtr validity;
  const uint8_t* valid() const { return validity ? validity->as<uint8_t>() : nullptr; }

  const void* values() const { return data ? data->ptr : nullptr; }
  const int32_t* offs() const { return offsets ? offsets->as<int32_t>() : nullptr; }
  int width() const { return dtype_width(dtype); }
  std::string arrow_format() const { return format.empty() ? default_format(dtype) : format; }
};

// Can a key column of one join input meet a key column of the other?  Only when both have one type: the same dtype
// and, for a Timestamp, the same Arrow format (unit and timezone), since equal integers of unlike units are unlike
// instants.  Date32 and Int32 are different dtypes, so they never meet.  DataFusion inserts casts before the join.
bool join_key_types_match(const Column& a, const Column& b);
// Fails with FLOCKGPU_ERR_UNSUPPORTED, naming both formats, when join_key_types_match(a, b) is false.
void check_join_key_types(const char* op, const Column& a, const Column& b);

struct Table;
using TablePtr = std::shared_ptr<const Table>;

// A relation whose rows have not been written out yet: a group-by result that still lives in its direct-address
// table (hash_agg.cu).  Table::resolve() materialises it; the operators that can work on the table form directly
// (NEXMark q5: MAX over the counts, then "count = max") ask for that instead and never pay for the 78 MB of
// (auction, count) rows that the plan would otherwise write and read twice.
struct DeferredTable {
  virtual ~DeferredTable() = default;
  virtual void materialise(const Table& self) = 0;  // fills self.cols / self.num_rows
  // Fast paths: each returns nullptr when it does not apply (the caller then resolves and takes the generic path).
  // `out = SELECT self.src_cols AS names`:
  virtual TablePtr project(const Table& self, const std::vector<int>& src_cols, const std::vector<std::string>& names) { return nullptr; }
  // one-row relation MAX(self.col) (mode: FLOCKGPU_AGG_PARTIAL state or a final value -- the same number):
  virtual TablePtr global_max(const Table& self, int col, const std::string& out_name) { return nullptr; }
  // self JOIN one_row ON self.key_col = one_row.one_key, output columns self ++ one_row (or the reverse):
  virtual TablePtr select_equal(const Table& self, int key_col, const TablePtr& one_row, int one_key, bool self_is_left) { return nullptr; }
  // other JOIN self ON other.keys[0] = self.self_keys[0] AND other.keys[1] = self.self_keys[1], where the pair is
  // (group column, MIN / MAX column) in either order; output columns other ++ self (or the reverse):
  virtual TablePtr select_group_match(const Table& self, const int (&self_keys)[2], const TablePtr& other, const int (&other_keys)[2],
                                      bool self_is_left) { return nullptr; }
};

// A direct-address (key, MIN / MAX) table as the matching selection reads it: slot = key - base for a 4-byte key,
// present[slot] != 0 for a group that exists, acc[slot] its MIN / MAX (int64 for a signed column: compared in the
// value column's width) and, when the aggregated column had NULLs, valid[slot] = its non-NULL count (0: the MAX is NULL).
struct GroupMatchTable {
  const unsigned char* present;
  const unsigned long long* acc;
  const unsigned long long* valid;
  unsigned long long base, n_slots;
};
// The rows of `other` whose column `key_col` names a group of `t` and whose `val_col` equals that group's value, in
// row order, with every column of `other` (filter_project.cu: filter_compact_kernel with the group_match predicate).
TablePtr select_group_match_rows(const CtxPtr& ctx, const Table& other, int key_col, int val_col, const GroupMatchTable& t);

struct Table {
  CtxPtr ctx;
  // `cols[i].length` and `num_rows` are -1 while `pending` is set (a filter's survivor count that has not
  // been read back yet); resolve() waits for it and fills them in.  Every operator resolves its inputs.
  mutable std::vector<Column> cols;
  mutable int64_t num_rows = 0;
  mutable std::shared_ptr<PendingRows> pending;
  mutable std::shared_ptr<DeferredTable> deferred;  // see DeferredTable; cols carry names / types only until resolved
  std::string metadata;  // raw Arrow schema metadata block (may be empty)
  // Set on the output of a multi-GPU hash exchange: the NAMES of the columns whose values routed the rows (the
  // routing function of partition.cu over exactly these columns, `partition_world` ranks).  Operators that keep those
  // columns under the same names hand the property on; a later RepartitionExec(Hash) over the same routing columns
  // finds its input already in place and moves nothing (q8 plans Hash([p_id, name]) and then Hash([p_id])).
  std::vector<std::string> partitioned_on;
  int partition_world = 0;
  int64_t nbytes() const;
  void resolve() const {
    if (deferred) {
      std::shared_ptr<DeferredTable> d = deferred;
      d->materialise(*this);
      deferred.reset();
    }
    if (!pending) return;
    num_rows = pending->wait();
    for (Column& c : cols) c.length = num_rows;
    pending.reset();
  }
  // resolve() + copy host-resident columns into HBM (every operator except the vectorised filter needs this)
  void dense() const;
  bool has_host_columns() const {
    for (const Column& c : cols)
      if (c.chunks) return true;
    return false;
  }
};

}  // namespace fg

// ABI handles ------------------------------------------------------------------------------------
struct flockgpu_ctx {
  fg::CtxPtr core;
};
struct flockgpu_table {
  fg::TablePtr table;
  std::atomic<int> refs{1};
};

namespace fg {
flockgpu_table* wrap_table(TablePtr t);
inline const Table& deref(const flockgpu_table* t) {
  if (!t || !t->table) fail(FLOCKGPU_ERR_INVALID, "null table handle");
  t->table->resolve();
  return *t->table;
}
inline CtxPtr core_of(flockgpu_ctx* c) {
  if (!c || !c->core) fail(FLOCKGPU_ERR_INVALID, "null context handle");
  return c->core;
}

// Operators that do not implement NULL semantics for some input refuse it (FLOCKGPU_ERR_UNSUPPORTED): the Rust shim then
// keeps the CPU plan for that data.  Never a silent wrong answer.
inline void require_no_nulls(const Column& c, const char* what) {
  if (c.validity) fail(FLOCKGPU_ERR_UNSUPPORTED, "%s: column \"%s\" contains NULLs, which this operator does not handle on the GPU path", what, c.name.c_str());
}

// The kernels' view of a column (expr_program.h); fill_colrefs writes refs[i] for every column i of `t`, and each caller
// checks first that they fit its argument block (filter_project.cu).
struct ColRef;
ColRef colref_of(const Column& c);
void fill_colrefs(const Table& t, ColRef* refs);

// ---- operators (implemented in the .cu files; called by the ABI layer and by the plan layer) ----
struct ExprTok {
  int op, dtype, col;
  int64_t i64;
  double f64;
  std::string str;
};
using Expr = std::vector<ExprTok>;  // postfix

TablePtr import_batches(const CtxPtr& ctx, const ArrowSchema* schema, const ArrowArray* const* batches,
                        int n_batches, const int* projection, int n_projection, bool zero_copy = false);
// Host -> device copies, page-locked staging of pageable sources included (the copy path of import_batches); returns
// once the copies have landed.
struct HostPiece {
  char* dst;
  const char* src;
  size_t bytes;
  size_t stage_off;  // offset in the staging block: the pieces' running byte total
};
void upload_host_pieces(const CtxPtr& ctx, const std::vector<HostPiece>& pieces, size_t total_bytes);
std::string copy_metadata(const char* md);  // the Arrow schema metadata block, verbatim

// Arrow IPC record-batch messages (host/ipc.cc)
struct FrameLayout {
  int64_t length = 0;
  int64_t body_length = -1;                          // Message.bodyLength (-1: absent)
  std::vector<std::pair<int64_t, int64_t>> nodes;    // (length, null_count) per field
  std::vector<std::pair<int64_t, int64_t>> buffers;  // (offset, length) into the body
};
FrameLayout parse_record_batch_message(const uint8_t* header, int64_t header_len);
// Index of each field's first buffer in FrameLayout::buffers (Utf8: validity, offsets, values; every other type:
// validity, values); the last entry is the buffer count.
std::vector<size_t> field_buffers(const ArrowSchema* schema);
void check_frame_layout(const ArrowSchema* schema, int f, const FrameLayout& L, int64_t body_len);
void check_utf8_extent(int f, const char* column, int32_t first, int32_t last, int64_t value_bytes);

// The bodies of frames of `t` (dense), one per (first row, row count), laid out and packed on the device:
// payload_layout_kernel reads the Utf8 extents and null counts (one small read-back, none when every range is empty),
// then one segment launch writes every body.  Each body is exactly what an Arrow IPC writer gives for its rows.
struct PackedFrames {
  BufferPtr bodies;                           // every frame's body in HBM, 16-byte aligned, back to back, zero padding
  std::vector<int64_t> body_at, body_len;
  std::vector<std::vector<uint8_t>> headers;  // the uncompressed Message { RecordBatch } of each frame
};
PackedFrames pack_frames(const CtxPtr& ctx, const Table& t, const std::vector<std::pair<int64_t, int64_t>>& row_ranges);

// One CTA's piece of ipc_segment_kernel, which moves bytes between IPC bodies and column buffers (import assemble,
// export pack).  kCopy: n bytes; kOffsets: n int32 words, each + arg (the source may be unaligned); kBitsToBytes:
// n validity bits -> n bytes; kBytesToBits: n validity bytes -> ceil(n / 8) bitmap bytes; kFill: n bytes = arg;
// kSetI32: one int32 = arg.
struct Seg {
  enum Kind : int32_t { kCopy, kOffsets, kBitsToBytes, kBytesToBits, kFill, kSetI32 };
  const uint8_t* src;
  uint8_t* dst;
  int64_t n;
  int32_t kind, arg;
};
// Appends the segments of n elements (bytes, words or rows), cut into pieces of at most 64 KiB.
void add_segs(std::vector<Seg>& segs, int kind, const uint8_t* src, uint8_t* dst, int64_t n, int32_t arg = 0);
// Uploads `segs` and runs them: exactly one launch, even for an empty list.  The launch is profiled under `stage`
// ("payload_assemble_kernel" at import, "payload_pack_kernel" at export), so a profile that spans an export and an
// import keeps the two apart.
void launch_segments(const CtxPtr& ctx, const std::vector<Seg>& segs, const char* stage);

// zstd payload frames (zstd.cu).  zstd_decode_host: every frame of src[0, n) serially on the host (headers, self test);
// returns a zstd::Z_* code, 0 on success.
int zstd_decode_host(const uint8_t* src, int64_t n, int64_t max_out, std::vector<uint8_t>* out);
// One zstd frame of src[0, n) appended to *out, by the export kernel's encoder phases run serially (zstd_enc.cu).
void zstd_compress_host(const uint8_t* src, int64_t n, std::vector<uint8_t>* out);
TablePtr import_payload_zstd(flockgpu_ctx* ctx, const ArrowSchema* schema, const uint8_t* const* headers, const int64_t* header_lens,
                             const uint8_t* const* bodies, const int64_t* body_lens, int n_frames, const int* projection, int n_projection);
void export_table(const CtxPtr& ctx, const Table& t, int64_t row_begin, int64_t row_count,
                  ArrowSchema* out_schema, ArrowArray* out_array);
void export_schema(const Table& t, ArrowSchema* out_schema);
TablePtr concat_tables(const CtxPtr& ctx, const std::vector<TablePtr>& tables);
TablePtr empty_like(const CtxPtr& ctx, const Table& t);

TablePtr filter_project(const CtxPtr& ctx, const TablePtr& in, const Expr* predicate,
                        const std::vector<Expr>& projections, const std::vector<std::string>& names);

// The values of `exprs` over `in`, one column each (named names[i], or derived), with ONE expr_eval_kernel launch for
// all of them (expr_eval.cu); plain columns share the input's buffers.  Runs the tree form (expr_tree.h).
std::vector<Column> eval_exprs(const CtxPtr& ctx, const Table& in, const std::vector<Expr>& exprs, const std::vector<std::string>& names);

struct AggSpec {
  int func;
  int col;
  std::string name;
};
TablePtr hash_aggregate(const CtxPtr& ctx, const TablePtr& in, int mode, const std::vector<int>& group_cols,
                        const std::vector<AggSpec>& aggs);
// Estimate from the first 64 Ki rows: fraction of rows that repeat an earlier group key (hash_agg.cu).
double distinct_sample_duplicates(const CtxPtr& ctx, const TablePtr& in, const std::vector<int>& group_cols);
TablePtr hash_join(const CtxPtr& ctx, const TablePtr& left, const TablePtr& right,
                   const std::vector<int>& left_keys, const std::vector<int>& right_keys);
// HashJoinExec { join_type: Semi } (anti = false) / { Anti } (anti = true): the rows of `left` whose key tuple occurs
// (does not occur) in `right`, each at most once, in left order, with the left schema.  Key equality and the key type
// checks are hash_join's: a NULL or NaN component matches nothing.
TablePtr hash_semi_join(const CtxPtr& ctx, const TablePtr& left, const TablePtr& right,
                        const std::vector<int>& left_keys, const std::vector<int>& right_keys, bool anti);
// COUNT(*) of `fact JOIN dim ON fact.fact_key = dim.dim_key` (inner) [WHERE `predicate` over the fact's columns],
// grouped by the dimension's `group_cols`, in one pass over the fact (dim_count.cu).  Output: the group columns under
// their dimension names, then one UInt64 count column per name of `count_names` (COUNT(*) listed n times: n equal
// columns); schema metadata `metadata`.  The dimension holds at most
// DIM_COUNT_MAX_ROWS rows: its key table (2 slots per row) and one counter per row fill 48 KiB of shared memory.
constexpr int64_t DIM_COUNT_MAX_ROWS = 4096;
bool dim_count_key_type(int dtype);  // Int32, Int64, UInt64, Timestamp, Utf8
TablePtr dim_count_aggregate(const CtxPtr& ctx, const TablePtr& fact, int fact_key, const Expr* predicate, const TablePtr& dim, int dim_key,
                             const std::vector<int>& group_cols, const std::vector<std::string>& count_names, const std::string& metadata);
std::vector<TablePtr> hash_partition(const CtxPtr& ctx, const TablePtr& in, const std::vector<int>& keys,
                                     int n_parts);
// The columns of `keys` that actually route a row: the fixed-width ones when there are any (hashing `p_id` routes
// (p_id, name) groups just as well as hashing the name bytes too, and lets a later Hash([p_id]) stay in place).
std::vector<int> routing_columns(const Table& in, const std::vector<int>& keys);
// RepartitionExec(Hash(keys, world)) + the inter-GPU shuffle in one step (exchange.cu): rows travel straight from the
// partition kernel into the receivers' windows over NVLink peer memory; `dest` >= 0 sends every row to that rank
// instead (CoalescePartitionsExec).  Falls back to hash_partition + the NCCL all-to-all when peer windows are
// unavailable.
TablePtr hash_exchange(const CtxPtr& ctx, const TablePtr& in, const std::vector<int>& keys, int dest = -1);
// SortExec / WindowAggExec(ROW_NUMBER) / GlobalLimitExec (sort.cu)
struct SortKey {
  int col;
  bool descending;
  bool nulls_first;  // no effect: columns with NULLs are not sortable on the GPU path
};
TablePtr sort_table(const CtxPtr& ctx, const TablePtr& in, const std::vector<SortKey>& keys);
TablePtr row_number(const CtxPtr& ctx, const TablePtr& in, const std::vector<int>& partition_cols, const std::string& name);
TablePtr limit_rows(const CtxPtr& ctx, const TablePtr& in, int64_t limit);
// Row gather: out.col[c][i] = in.col[c][idx[i]] for every column (fixed width and Utf8).
TablePtr gather_rows(const CtxPtr& ctx, const Table& in, const std::vector<int>& cols, const uint32_t* d_idx,
                     int64_t n_idx);
// Gathers single columns (used by filter for Utf8 pass-through and by join).
Column gather_column(const CtxPtr& ctx, const Column& in, const uint32_t* d_idx, int64_t n_idx);
std::vector<Column> gather_columns(const CtxPtr& ctx, const std::vector<const Column*>& in, const uint32_t* d_idx, int64_t n);

TablePtr all_to_all(const CtxPtr& ctx, const std::vector<TablePtr>& parts);
void comm_unique_id(uint8_t* out);
void comm_init(const CtxPtr& ctx, const uint8_t* id, int rank, int world);
int comm_world(const CtxPtr& ctx);  // 1 when no communicator is attached
int comm_rank(const CtxPtr& ctx);   // 0 when no communicator is attached

inline void count_launch(const CtxPtr& ctx, int n = 1) { ctx->launches.fetch_add(n, std::memory_order_relaxed); }

}  // namespace fg
