// core.cu -- context, HBM buffers, and the Arrow C Data Interface boundary (host <-> HBM).
//
// Replaces, on the reference side: MemoryExec::set_partitions fed by
// ExecutionContext::feed_data_sources (flock/src/runtime/context.rs:257-325) for the way in, and the
// Vec<RecordBatch> returned by `collect` (context.rs:172-191) for the way out.
#include <algorithm>
#include <map>
#include <memory>
#include <tuple>
#include <thread>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>

#include "compact.cuh"
#include "device_utils.cuh"
#include "internal.h"

namespace fg {

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
static thread_local std::string g_last_error;

void set_last_error(const std::string& msg) { g_last_error = msg; }

void fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  throw Error{code, buf};
}

// ------------------------------------------------------------------------------------------------
// dtypes
// ------------------------------------------------------------------------------------------------
int dtype_width(int dtype) {
  switch (dtype) {
    case FLOCKGPU_BOOL: return 1;
    case FLOCKGPU_INT32: case FLOCKGPU_UINT32: case FLOCKGPU_DATE32: return 4;
    case FLOCKGPU_INT64: case FLOCKGPU_UINT64: case FLOCKGPU_FLOAT64: case FLOCKGPU_TIMESTAMP: return 8;
    default: return 0;
  }
}

const char* dtype_name(int dtype) {
  switch (dtype) {
    case FLOCKGPU_BOOL: return "Boolean";
    case FLOCKGPU_INT32: return "Int32";
    case FLOCKGPU_UINT32: return "UInt32";
    case FLOCKGPU_INT64: return "Int64";
    case FLOCKGPU_UINT64: return "UInt64";
    case FLOCKGPU_FLOAT64: return "Float64";
    case FLOCKGPU_TIMESTAMP: return "Timestamp";
    case FLOCKGPU_DATE32: return "Date32";
    case FLOCKGPU_UTF8: return "Utf8";
    default: return "?";
  }
}

int dtype_from_format(const char* f) {
  if (!f) return -1;
  if (!strcmp(f, "i")) return FLOCKGPU_INT32;
  if (!strcmp(f, "I")) return FLOCKGPU_UINT32;
  if (!strcmp(f, "l")) return FLOCKGPU_INT64;
  if (!strcmp(f, "L")) return FLOCKGPU_UINT64;
  if (!strcmp(f, "g")) return FLOCKGPU_FLOAT64;
  if (!strcmp(f, "u")) return FLOCKGPU_UTF8;
  if (!strcmp(f, "tdD")) return FLOCKGPU_DATE32;
  if (!strncmp(f, "ts", 2) && strlen(f) >= 4 && f[3] == ':') return FLOCKGPU_TIMESTAMP;
  return -1;
}

std::string default_format(int dtype) {
  switch (dtype) {
    case FLOCKGPU_INT32: return "i";
    case FLOCKGPU_UINT32: return "I";
    case FLOCKGPU_INT64: return "l";
    case FLOCKGPU_UINT64: return "L";
    case FLOCKGPU_FLOAT64: return "g";
    case FLOCKGPU_UTF8: return "u";
    case FLOCKGPU_TIMESTAMP: return "tsm:";
    case FLOCKGPU_DATE32: return "tdD";
    default: return "n";
  }
}

bool join_key_types_match(const Column& a, const Column& b) {
  return a.dtype == b.dtype && (a.dtype != FLOCKGPU_TIMESTAMP || a.arrow_format() == b.arrow_format());
}

void check_join_key_types(const char* op, const Column& a, const Column& b) {
  FG_CHECK(join_key_types_match(a, b), FLOCKGPU_ERR_UNSUPPORTED, "%s: key types differ (%s \"%s\" vs %s \"%s\"); DataFusion inserts casts before the join", op,
           dtype_name(a.dtype), a.arrow_format().c_str(), dtype_name(b.dtype), b.arrow_format().c_str());
}

// ------------------------------------------------------------------------------------------------
// context
// ------------------------------------------------------------------------------------------------
CtxCore::~CtxCore() {
  cudaSetDevice(device);
  if (stream) cudaStreamSynchronize(stream);
  drop_cached_blocks();
  for (auto& kv : pinned) cudaFreeHost(kv.first);
  pinned.clear();
  for (PinSlab& sl : pin_slabs)
    if (sl.base) cudaFreeHost(sl.base);
  pin_slabs.clear();
  if (scan.ep_state) cudaFree(scan.ep_state);
  if (scan.ep_counts) cudaFree(scan.ep_counts);
  if (scan.ep_counters) cudaFree(scan.ep_counters);
  if (l2_flush) cudaFree(l2_flush);
  if (h_scalars) cudaFreeHost(h_scalars);
  if (d_scalars) cudaFree(d_scalars);
  for (int i = 0; i < 16; ++i) {
    if (timer_start[i]) cudaEventDestroy(timer_start[i]);
    if (timer_stop[i]) cudaEventDestroy(timer_stop[i]);
  }
  for (auto& p : profile) {
    cudaEventDestroy(p.start);
    cudaEventDestroy(p.stop);
  }
  for (cudaEvent_t e : sync_events) cudaEventDestroy(e);
  for (cudaEvent_t e : timing_events) cudaEventDestroy(e);
  for (int i = 0; i < kCopyStreams; ++i) {
    if (copy_streams[i]) cudaStreamDestroy(copy_streams[i]);
    if (copy_join[i]) cudaEventDestroy(copy_join[i]);
  }
  if (copy_fork) cudaEventDestroy(copy_fork);
  if (stream) cudaStreamDestroy(stream);
}

static const bool g_host_trace = getenv("FLOCKGPU_HOST_TRACE") != nullptr;
static std::mutex g_trace_mu;
static std::map<std::string, std::pair<long long, long long>> g_trace;  // name -> (calls, ns)
static long long now_ns() {
  timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return (long long)ts.tv_sec * 1000000000ll + ts.tv_nsec;
}
HostSpan::HostSpan(const char* n) : name(n), t0(g_host_trace ? now_ns() : 0) {}
HostSpan::~HostSpan() {
  if (!g_host_trace) return;
  const long long dt = now_ns() - t0;
  std::lock_guard<std::mutex> g(g_trace_mu);
  auto& e = g_trace[name];
  e.first += 1;
  e.second += dt;
}
void host_trace_dump(bool reset) {
  if (!g_host_trace) return;
  std::lock_guard<std::mutex> g(g_trace_mu);
  for (auto& kv : g_trace)
    fprintf(stderr, "[flockgpu host] %-28s calls %8lld  total %10.3f ms  mean %9.3f us\n", kv.first.c_str(), kv.second.first, kv.second.second * 1e-6,
            kv.second.first ? kv.second.second * 1e-3 / kv.second.first : 0.0);
  if (reset) g_trace.clear();
}

void StagePool::start(int n, const std::function<void()>* fn) {
  std::unique_lock<std::mutex> g(mu);
  while (int(threads.size()) < n) {
    const int index = int(threads.size());
    threads.emplace_back([this, index] {
      uint64_t seen = 0;
      std::unique_lock<std::mutex> lk(mu);
      while (true) {
        wake.wait(lk, [&] { return stop || (generation != seen && index < active); });
        if (stop) return;
        seen = generation;
        const std::function<void()>* fn = job;
        lk.unlock();
        (*fn)();
        lk.lock();
        if (--running == 0) idle.notify_all();
      }
    });
  }
  job = fn;
  active = n;
  running = n;
  ++generation;
  g.unlock();
  wake.notify_all();
}

void StagePool::wait() {
  std::unique_lock<std::mutex> g(mu);
  idle.wait(g, [&] { return running == 0; });
  active = 0;
}

StagePool::~StagePool() {
  {
    std::lock_guard<std::mutex> g(mu);
    stop = true;
  }
  wake.notify_all();
  for (std::thread& t : threads) t.join();
}

// size classes: eight per power of two (at most 12.5 % slack), 512 bytes at least
static size_t round_block(size_t n) {
  if (n <= 512) return 512;
  size_t p = 512;
  while (p < n) p <<= 1;       // smallest power of two >= n
  const size_t step = p >> 4;  // sixteenths of it = eighths of the octave below
  return (n + step - 1) / step * step;
}

void* CtxCore::take_block(size_t rounded) {
  {
    std::lock_guard<std::mutex> g(block_mu);
    auto it = free_blocks.find(rounded);
    if (it != free_blocks.end() && !it->second.empty()) {
      void* p = it->second.back();
      it->second.pop_back();
      cached_bytes -= rounded;
      return p;
    }
  }
  HostSpan span("alloc (cudaMallocAsync)");
  void* p = nullptr;
  cudaError_t e = cudaMallocAsync(&p, rounded, stream);
  if (e == cudaErrorMemoryAllocation) {
    cudaGetLastError();
    drop_cached_blocks();
    e = cudaMallocAsync(&p, rounded, stream);
  }
  if (e != cudaSuccess) fail(FLOCKGPU_ERR_CUDA, "cudaMallocAsync(%zu bytes) -> %s", rounded, cudaGetErrorString(e));
  return p;
}

void CtxCore::give_block(void* p, size_t rounded) {
  std::lock_guard<std::mutex> g(block_mu);
  free_blocks[rounded].push_back(p);
  cached_bytes += rounded;
}

void CtxCore::drop_cached_blocks() {
  std::lock_guard<std::mutex> g(block_mu);
  for (auto& kv : free_blocks)
    for (void* p : kv.second) cudaFreeAsync(p, stream);
  free_blocks.clear();
  cached_bytes = 0;
  cudaStreamSynchronize(stream);
}

Buffer::Buffer(CtxPtr c, size_t n) : ctx(std::move(c)), bytes(n), seq(ctx->alloc_seq) {
  HostSpan span("alloc");
  size_t want = n ? n : 16;
  want = (want + 255) & ~size_t(255);  // room for vector tails: kernels may read up to 16 B past the end
  block_bytes = round_block(want + 256);
  ptr = ctx->take_block(block_bytes);
}

Buffer::~Buffer() {
  if (ptr && !parent) ctx->give_block(ptr, block_bytes);
}

BufferPtr alloc(const CtxPtr& ctx, size_t bytes) { return std::make_shared<Buffer>(ctx, bytes); }

int scan_stride() {
  static const int v = [] {
    const char* e = getenv("FLOCKGPU_LB_STRIDE");
    int x = e ? atoi(e) : 32;
    return x >= 1 && x <= 64 ? x : 32;
  }();
  return v;
}

int scan_poll_sleep_ns() {
  static const int v = [] {
    const char* e = getenv("FLOCKGPU_LB_SLEEP");
    int x = e ? atoi(e) : 100;
    return x >= 0 && x <= 10000 ? x : 100;
  }();
  return v;
}

CompactScratch prepare_compact(const CtxPtr& ctx, long long num_tiles, long long resident_ctas, unsigned long long* out_count, bool rounds) {
  ScanScratch& s = ctx->scan;
  const int stride = scan_stride();
  if (!s.ep_counters) {
    FG_CUDA(cudaMalloc(&s.ep_counters, 16 * sizeof(unsigned)));
    FG_CUDA(cudaMemsetAsync(s.ep_counters, 0, 16 * sizeof(unsigned), ctx->stream));
  }
  if (num_tiles > s.ep_capacity) {
    int64_t cap = 1 << 12;
    while (cap < num_tiles) cap <<= 1;
    FG_CUDA(cudaStreamSynchronize(ctx->stream));
    if (s.ep_state) FG_CUDA(cudaFree(s.ep_state));
    if (s.ep_counts) FG_CUDA(cudaFree(s.ep_counts));
    FG_CUDA(cudaMalloc(&s.ep_state, size_t(cap) * stride * sizeof(unsigned long long)));
    FG_CUDA(cudaMalloc(&s.ep_counts, size_t(cap) * sizeof(unsigned long long)));
    FG_CUDA(cudaMemsetAsync(s.ep_state, 0, size_t(cap) * stride * sizeof(unsigned long long), ctx->stream));
    FG_CUDA(cudaMemsetAsync(s.ep_counts, 0, size_t(cap) * sizeof(unsigned long long), ctx->stream));
    s.ep_capacity = cap;
    ctx->overlap_kernel = nullptr;  // the next launch must not start before these memsets
  }
  s.epoch = (s.epoch + 1) & 0xfffffu;
  if (s.epoch == 0) {
    // 2^20 launches later a stale word could carry the current epoch again: wipe them once per wrap
    FG_CUDA(cudaMemsetAsync(s.ep_state, 0, size_t(s.ep_capacity) * stride * sizeof(unsigned long long), ctx->stream));
    FG_CUDA(cudaMemsetAsync(s.ep_counts, 0, size_t(s.ep_capacity) * sizeof(unsigned long long), ctx->stream));
    s.epoch = 1;
    ctx->overlap_kernel = nullptr;
  }
  CompactScratch sc{};
  sc.tile_state = s.ep_state;
  sc.counts = s.ep_counts;
  sc.counters = s.ep_counters;
  sc.out_count = out_count;
  sc.num_tiles = num_tiles;
  sc.ticket_base = s.tickets_issued;
  sc.arrived_base = s.arrived;
  sc.epoch = s.epoch;
  static const bool env_lookback = getenv("FLOCKGPU_FORCE_LOOKBACK") != nullptr;
  const bool force_lookback = env_lookback || ctx->compact_mode == 1;
  if (resident_ctas < 1) resident_ctas = 1;
  sc.single_wave = ((rounds || num_tiles <= resident_ctas) && !force_lookback) ? 1 : 0;
  sc.grid = int(std::max<long long>(1, std::min<long long>(resident_ctas, num_tiles)));
  sc.stride = stride;
  sc.poll_sleep_ns = scan_poll_sleep_ns();
  // the arrival / ticket bases advance in launch_compact(), after the launch has been accepted
  return sc;
}

bool overlap_previous(const CtxPtr& ctx, const void* kernel, const CompactScratch& sc, const EarlyStart* early) {
  return early && sc.single_wave && kernel == ctx->overlap_kernel && ctx->launches.load(std::memory_order_relaxed) == ctx->overlap_launches + 1 &&
         early->newest_input < ctx->overlap_outputs;
}

void note_compact_launch(const CtxPtr& ctx, const void* kernel, const CompactScratch& sc, const EarlyStart* early, bool overlapped) {
  ctx->overlap_kernel = early && sc.single_wave ? kernel : nullptr;
  ctx->overlap_launches = ctx->launches.load(std::memory_order_relaxed);
  ctx->overlap_outputs = early ? early->outputs : 0;
  if (overlapped) ctx->overlapped.fetch_add(1, std::memory_order_relaxed);
}

int resident_ctas(const CtxPtr& ctx, const void* kernel, int threads, size_t smem) {
  struct Key {
    int device;
    const void* kernel;
    size_t smem;
    bool operator<(const Key& o) const { return std::tie(device, kernel, smem) < std::tie(o.device, o.kernel, o.smem); }
  };
  static std::mutex mu;
  static std::map<Key, int> cache;
  const Key key{ctx->device, kernel, smem};
  {
    std::lock_guard<std::mutex> g(mu);
    auto it = cache.find(key);
    if (it != cache.end()) return int(int64_t(ctx->sm_count) * it->second);
  }
  int per_sm = 0;
  FG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem));
  if (per_sm < 1) per_sm = 1;
  std::lock_guard<std::mutex> g(mu);
  cache[key] = per_sm;
  return int(int64_t(ctx->sm_count) * per_sm);
}

void read_scalars(const CtxPtr& ctx, int first, int n, unsigned long long* out) {
  HostSpan span("read_scalars (sync)");
  FG_CUDA(cudaMemcpyAsync(ctx->h_scalars + first, ctx->d_scalars + first, sizeof(unsigned long long) * n,
                          cudaMemcpyDeviceToHost, ctx->stream));
  FG_CUDA(cudaStreamSynchronize(ctx->stream));
  for (int i = 0; i < n; ++i) out[i] = ctx->h_scalars[first + i];
  dump_filter_traces(ctx);
}

// ---- row counts in flight ------------------------------------------------------------------------
int64_t PendingRows::wait() {
  if (!done) {
    HostSpan span("pending wait (sync)");
    cudaSetDevice(ctx->device);
    FG_CUDA(cudaEventSynchronize(ev));
    value = int64_t(ctx->h_scalars[CtxCore::kScalars + slot]);
    done = true;
    dump_filter_traces(ctx);
    if (h2d_bytes_per_row) ctx->h2d_bytes.fetch_add(value * h2d_bytes_per_row, std::memory_order_relaxed);
  }
  return value;
}

PendingRows::~PendingRows() {
  if (ev) ctx->put_event(ev, false);
}

cudaEvent_t CtxCore::get_event(bool timing) {
  std::vector<cudaEvent_t>& pool = timing ? timing_events : sync_events;
  if (!pool.empty()) {
    cudaEvent_t e = pool.back();
    pool.pop_back();
    return e;
  }
  cudaEvent_t e = nullptr;
  FG_CUDA(timing ? cudaEventCreate(&e) : cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  return e;
}

unsigned long long* PendingRows::host_slot() const { return ctx->h_scalars + CtxCore::kScalars + slot; }

std::shared_ptr<PendingRows> reserve_row_count(const CtxPtr& ctx) {
  const int slot = ctx->pending_next;
  ctx->pending_next = (ctx->pending_next + 1) % CtxCore::kPendingSlots;
  if (auto old = ctx->pending_owner[slot].lock()) old->wait();  // the pinned slot is about to be overwritten
  auto p = std::make_shared<PendingRows>();
  p->ctx = ctx;
  p->slot = slot;
  p->ev = ctx->get_event(false);
  ctx->pending_owner[slot] = p;
  return p;
}

void commit_row_count(const std::shared_ptr<PendingRows>& p) {
  FG_CUDA(cudaEventRecord(p->ev, p->ctx->stream));
}

// ---- per-kernel profile ----------------------------------------------------------------------------
LaunchTimer::LaunchTimer(const CtxPtr& c, const char* kernel) : ctx(c.get()) {
  if (!ctx->profiling) return;
  cudaEvent_t start = ctx->get_event(true);
  stop = ctx->get_event(true);
  cudaEventRecord(start, ctx->stream);
  ctx->profile.push_back({kernel, start, stop});
}

LaunchTimer::~LaunchTimer() {
  if (stop) cudaEventRecord(stop, ctx->stream);
}

int64_t Table::nbytes() const {
  resolve();
  int64_t n = 0;
  for (const Column& c : cols) {
    if (c.dtype == FLOCKGPU_UTF8)
      n += c.values_bytes + (c.length + 1) * 4;
    else
      n += c.length * c.width();
  }
  return n;
}

flockgpu_table* wrap_table(TablePtr t) {
  auto* h = new flockgpu_table();
  h->table = std::move(t);
  return h;
}

// ------------------------------------------------------------------------------------------------
// small kernels used by import / concat
// ------------------------------------------------------------------------------------------------
__global__ void rebase_offsets_kernel(int32_t* __restrict__ offs, int64_t n, int32_t delta) {
  int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
  int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (; i < n; i += stride) offs[i] += delta;
}

__global__ void set_i32_kernel(int32_t* p, int32_t v) { *p = v; }

static void rebase_offsets(const CtxPtr& ctx, int32_t* offs, int64_t n, int32_t delta) {
  if (n <= 0 || delta == 0) return;
  int blocks = int(std::min<int64_t>((n + 255) / 256, ctx->sm_count * 8));
  {
    LaunchTimer lt(ctx, "rebase_offsets_kernel");
    rebase_offsets_kernel<<<blocks, 256, 0, ctx->stream>>>(offs, n, delta);
  }
  count_launch(ctx);
}

static void set_i32(const CtxPtr& ctx, int32_t* p, int32_t v) {
  {
    LaunchTimer lt(ctx, "set_i32_kernel");
    set_i32_kernel<<<1, 1, 0, ctx->stream>>>(p, v);
  }
  count_launch(ctx);
}

// ------------------------------------------------------------------------------------------------
// import: Arrow C Data (host) -> Table (HBM)
// ------------------------------------------------------------------------------------------------
static bool range_has_null(const uint8_t* bitmap, int64_t off, int64_t len) {
  for (int64_t i = off; i < off + len; ++i)
    if (!((bitmap[i >> 3] >> (i & 7)) & 1)) return true;
  return false;
}

std::string copy_metadata(const char* md) {
  // Arrow metadata block: int32 n, then n x (int32 klen, key, int32 vlen, value)
  if (!md) return std::string();
  const char* p = md;
  int32_t n;
  memcpy(&n, p, 4);
  p += 4;
  for (int32_t i = 0; i < n; ++i) {
    for (int k = 0; k < 2; ++k) {
      int32_t l;
      memcpy(&l, p, 4);
      p += 4 + l;
    }
  }
  return std::string(md, p - md);
}

// Can this fixed-width column stay in host memory?  Needs page-locked sources (CUDA knows the pointer), uniform
// power-of-two batch lengths (row -> chunk is a shift) and 16-byte aligned chunk bases (128-bit loads).
// Deals host->device copies over the context's copy streams.  fork() orders them after everything already queued
// on the main stream (the stream-ordered allocations of their destinations), join() makes the main stream wait for
// all of them.
struct CopyFan {
  CtxCore* ctx;
  int next = 0;
  bool used[CtxCore::kCopyStreams] = {};
  explicit CopyFan(const CtxPtr& c) : ctx(c.get()) {}
  void fork() {
    FG_CUDA(cudaEventRecord(ctx->copy_fork, ctx->stream));
    for (int i = 0; i < CtxCore::kCopyStreams; ++i) FG_CUDA(cudaStreamWaitEvent(ctx->copy_streams[i], ctx->copy_fork, 0));
  }
  void copy(void* dst, const void* src, size_t bytes) {
    const int i = next;
    next = (next + 1) % CtxCore::kCopyStreams;
    used[i] = true;
    ctx->h2d_bytes.fetch_add(int64_t(bytes), std::memory_order_relaxed);
    FG_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->copy_streams[i]));
  }
  void join() {
    for (int i = 0; i < CtxCore::kCopyStreams; ++i) {
      if (!used[i]) continue;
      FG_CUDA(cudaEventRecord(ctx->copy_join[i], ctx->copy_streams[i]));
      FG_CUDA(cudaStreamWaitEvent(ctx->stream, ctx->copy_join[i], 0));
      used[i] = false;
    }
  }
};

HostRegistration::~HostRegistration() {
  for (auto& r : ranges) cudaHostUnregister(r.first);
}

static bool is_pageable(const void* p) {
  cudaPointerAttributes attr;
  if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) {
    cudaGetLastError();
    return true;
  }
  return attr.type == cudaMemoryTypeUnregistered;
}

// feed_register: page-locks, in place, the value buffers of the fixed-width columns `cols` of every batch.  Buffers of
// neighbouring batches may share pages, so the page-aligned ranges are merged before they are registered.
static std::shared_ptr<HostRegistration> register_sources(const ArrowArray* const* batches, int n_batches, const std::vector<std::pair<int, int>>& cols) {
  std::vector<std::pair<uintptr_t, uintptr_t>> ranges;
  const uintptr_t page = 4096;
  for (const auto& cw : cols)
    for (int b = 0; b < n_batches; ++b) {
      const ArrowArray* a = batches[b]->children[cw.first];
      if (batches[b]->length == 0 || a->n_buffers < 2 || !a->buffers[1]) continue;
      const char* src = static_cast<const char*>(a->buffers[1]) + (batches[b]->offset + a->offset) * cw.second;
      if (!is_pageable(src)) continue;
      const uintptr_t lo = reinterpret_cast<uintptr_t>(src) & ~(page - 1);
      const uintptr_t hi = (reinterpret_cast<uintptr_t>(src) + size_t(batches[b]->length) * cw.second + page - 1) & ~(page - 1);
      ranges.emplace_back(lo, hi);
    }
  if (ranges.empty()) return nullptr;
  std::sort(ranges.begin(), ranges.end());
  auto reg = std::make_shared<HostRegistration>();
  uintptr_t lo = ranges[0].first, hi = ranges[0].second;
  auto flush = [&]() {
    cudaError_t e = cudaHostRegister(reinterpret_cast<void*>(lo), hi - lo, cudaHostRegisterMapped | cudaHostRegisterPortable);
    if (e == cudaSuccess) reg->ranges.emplace_back(reinterpret_cast<void*>(lo), hi - lo);
    else cudaGetLastError();  // e.g. a page that is locked already: the column then simply takes the copy path
  };
  for (size_t i = 1; i < ranges.size(); ++i) {
    if (ranges[i].first <= hi) {
      hi = std::max(hi, ranges[i].second);
    } else {
      flush();
      lo = ranges[i].first;
      hi = ranges[i].second;
    }
  }
  flush();
  return reg;
}

static std::shared_ptr<HostChunks> try_host_chunks(const CtxPtr& ctx, const ArrowArray* const* batches, int n_batches, int p, int w) {
  if (n_batches < 1) return nullptr;
  const int64_t L = batches[0]->length;
  if (L < 4096 || (L & (L - 1)) != 0) return nullptr;
  auto hc = std::make_shared<HostChunks>();
  hc->shift = 0;
  while ((int64_t(1) << hc->shift) < L) ++hc->shift;
  for (int b = 0; b < n_batches; ++b) {
    const ArrowArray* a = batches[b]->children[p];
    const int64_t len = batches[b]->length, off = batches[b]->offset + a->offset;
    if (b + 1 < n_batches ? len != L : (len > L || len == 0)) return nullptr;
    if (a->n_buffers < 2 || !a->buffers[1]) return nullptr;
    const char* src = static_cast<const char*>(a->buffers[1]) + off * w;
    if (reinterpret_cast<uintptr_t>(src) & 15) return nullptr;
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, src) != cudaSuccess) {
      cudaGetLastError();
      return nullptr;
    }
    if (attr.type != cudaMemoryTypeHost || !attr.devicePointer) return nullptr;
    hc->ptrs.push_back(attr.devicePointer);
    hc->rows.push_back(len);
  }
  hc->table = alloc(ctx, hc->ptrs.size() * sizeof(void*));
  FG_CUDA(cudaMemcpyAsync(hc->table->ptr, hc->ptrs.data(), hc->ptrs.size() * sizeof(void*), cudaMemcpyHostToDevice, ctx->stream));
  return hc;
}

void Table::dense() const {
  resolve();
  for (Column& c : cols) {
    if (!c.chunks) continue;
    const int w = c.width();
    c.data = alloc(ctx, size_t(c.length) * w);
    CopyFan fan(ctx);
    fan.fork();
    int64_t row = 0;
    for (size_t k = 0; k < c.chunks->ptrs.size(); ++k) {
      fan.copy(static_cast<char*>(c.data->ptr) + row * w, c.chunks->ptrs[k], size_t(c.chunks->rows[k]) * w);
      row += c.chunks->rows[k];
    }
    fan.join();
    c.chunks.reset();
  }
}

namespace {
void* pin_get(size_t bytes);
void pin_put(void* p, size_t bytes);
}  // namespace

namespace {
// Page-locked staging blocks of one import; they return to the cache when the import is done with them.
struct PinnedBlocks {
  std::vector<std::pair<void*, size_t>> v;
  void emplace_back(void* p, size_t n) { v.emplace_back(p, n); }
  ~PinnedBlocks() {
    for (auto& b : v) pin_put(b.first, b.second);
  }
};

// Issues the host -> device copies of `pieces` (fixed_bytes in all) on the copy streams and joins them into the main
// stream.  The staging blocks it takes go to `staged`: the caller keeps them until the copies have drained.
void issue_pieces(const CtxPtr& ctx, CopyFan& fan, const std::vector<HostPiece>& pieces, size_t fixed_bytes, PinnedBlocks& staged) {
  fan.fork();
  const int n_thr = int(std::min<size_t>(size_t(ctx->feed_stage_threads), pieces.size()));
  if (n_thr >= 1 && fixed_bytes >= (size_t(1) << 20) && is_pageable(pieces[0].src)) {
    // Pageable sources (what arrow-rs hands over): cudaMemcpyAsync would bounce every batch through the driver's own
    // staging buffer on ONE thread.  Host threads copy the batches into a page-locked block instead and each issues
    // the DMA of a batch as soon as it has copied it, so the host copies run in parallel with each other and with
    // the link.
    char* stage = static_cast<char*>(pin_get(fixed_bytes));
    staged.emplace_back(stage, fixed_bytes);
    // DMA chunks: runs of consecutive pieces that are contiguous on both sides (one column's batches), about 4 MB
    // each.  The workers only copy; THIS thread issues a chunk's DMA as soon as its last piece has been staged
    // (one cudaMemcpyAsync per chunk: 306 per-batch calls from many threads serialised on the driver's lock).
    struct Chunk {
      char* dst;
      size_t stage_off, bytes;
      int pieces;
    };
    std::vector<Chunk> chunks;
    std::vector<int> chunk_of(pieces.size());
    for (size_t i = 0; i < pieces.size(); ++i) {
      const bool extend = !chunks.empty() && chunks.back().dst + chunks.back().bytes == pieces[i].dst &&
                          chunks.back().stage_off + chunks.back().bytes == pieces[i].stage_off && chunks.back().bytes < (size_t(4) << 20);
      if (!extend) chunks.push_back({pieces[i].dst, pieces[i].stage_off, 0, 0});
      chunks.back().bytes += pieces[i].bytes;
      chunks.back().pieces += 1;
      chunk_of[i] = int(chunks.size()) - 1;
    }
    std::unique_ptr<std::atomic<int>[]> remaining(new std::atomic<int>[chunks.size()]);
    for (size_t c = 0; c < chunks.size(); ++c) remaining[c].store(chunks[c].pieces);
    std::atomic<size_t> next{0};
    const int stream_stores = ctx->feed_stream_stores;
    const std::function<void()> worker = [&]() {
      for (size_t i = next.fetch_add(1); i < pieces.size(); i = next.fetch_add(1)) {
        stage_copy(stage + pieces[i].stage_off, pieces[i].src, pieces[i].bytes, stream_stores);
        remaining[chunk_of[i]].fetch_sub(1, std::memory_order_release);
      }
    };
    ctx->stage_pool.start(n_thr, &worker);
    cudaError_t issue_err = cudaSuccess;
    for (size_t c = 0; c < chunks.size(); ++c) {
      while (remaining[c].load(std::memory_order_acquire) > 0) {
      }
      cudaError_t e = cudaMemcpyAsync(chunks[c].dst, stage + chunks[c].stage_off, chunks[c].bytes, cudaMemcpyHostToDevice,
                                      ctx->copy_streams[c % CtxCore::kCopyStreams]);
      if (e != cudaSuccess && issue_err == cudaSuccess) issue_err = e;
    }
    ctx->stage_pool.wait();
    FG_CHECK(issue_err == cudaSuccess, FLOCKGPU_ERR_CUDA, "table_import: staged host-to-device copy failed: %s", cudaGetErrorString(issue_err));
    for (int i = 0; i < CtxCore::kCopyStreams; ++i) fan.used[i] = true;
    ctx->h2d_bytes.fetch_add(int64_t(fixed_bytes), std::memory_order_relaxed);
  } else {
    for (const HostPiece& pc : pieces) fan.copy(pc.dst, pc.src, pc.bytes);
  }
  fan.join();
}
}  // namespace

void upload_host_pieces(const CtxPtr& ctx, const std::vector<HostPiece>& pieces, size_t total_bytes) {
  CopyFan fan(ctx);
  PinnedBlocks staged;
  if (!pieces.empty()) issue_pieces(ctx, fan, pieces, total_bytes, staged);
  FG_CUDA(cudaStreamSynchronize(ctx->stream));
}

TablePtr import_batches(const CtxPtr& ctx, const ArrowSchema* schema, const ArrowArray* const* batches,
                        int n_batches, const int* projection, int n_projection, bool zero_copy) {
  FG_CHECK(schema && schema->format && !strcmp(schema->format, "+s"), FLOCKGPU_ERR_INVALID,
           "table_import: schema must be a struct (\"+s\"), got \"%s\"", schema && schema->format ? schema->format : "null");
  FG_CHECK(n_batches >= 0 && (n_batches == 0 || batches), FLOCKGPU_ERR_INVALID, "table_import: bad batch list");
  std::vector<int> proj;
  if (projection) {
    proj.assign(projection, projection + n_projection);
  } else {
    for (int i = 0; i < schema->n_children; ++i) proj.push_back(i);
  }
  CopyFan fan(ctx);
  // page-locked staging blocks of this call (pageable sources); they return to the cache once the copies have drained
  PinnedBlocks staged;
  int64_t total = 0;
  for (int b = 0; b < n_batches; ++b) {
    FG_CHECK(batches[b] && batches[b]->n_children == schema->n_children, FLOCKGPU_ERR_INVALID,
             "table_import: batch %d has %lld children, schema has %lld", b,
             (long long)(batches[b] ? batches[b]->n_children : -1), (long long)schema->n_children);
    FG_CHECK(batches[b]->null_count <= 0, FLOCKGPU_ERR_UNSUPPORTED, "table_import: struct-level nulls");
    total += batches[b]->length;
  }
  FG_CHECK(total < (int64_t(1) << 32) - 1, FLOCKGPU_ERR_UNSUPPORTED, "table_import: more than 2^32-2 rows in one relation");

  auto t = std::make_shared<Table>();
  t->ctx = ctx;
  t->num_rows = total;
  t->metadata = copy_metadata(schema->metadata);
  // host -> device copies of the fixed-width columns: collected for ALL columns, then issued together
  std::vector<HostPiece> pieces;
  size_t fixed_bytes = 0;
  std::shared_ptr<HostRegistration> registration;
  if (zero_copy && ctx->feed_register && total > 0) {
    std::vector<std::pair<int, int>> fixed;
    for (int p : proj) {
      if (p < 0 || p >= schema->n_children) continue;
      const int dt = dtype_from_format(schema->children[p]->format);
      if (dt >= 0 && dt != FLOCKGPU_UTF8) fixed.emplace_back(p, dtype_width(dt));
    }
    registration = register_sources(batches, n_batches, fixed);
  }
  for (int p : proj) {
    FG_CHECK(p >= 0 && p < schema->n_children, FLOCKGPU_ERR_INVALID, "table_import: projection index %d out of range", p);
    const ArrowSchema* cs = schema->children[p];
    int dt = dtype_from_format(cs->format);
    FG_CHECK(dt >= 0, FLOCKGPU_ERR_UNSUPPORTED, "table_import: column \"%s\" has unsupported Arrow format \"%s\"",
             cs->name ? cs->name : "", cs->format ? cs->format : "");
    FG_CHECK(cs->dictionary == nullptr, FLOCKGPU_ERR_UNSUPPORTED, "table_import: dictionary-encoded column \"%s\"", cs->name);
    Column col;
    col.dtype = dt;
    col.name = cs->name ? cs->name : "";
    col.format = cs->format;
    col.nullable = (cs->flags & ARROW_FLAG_NULLABLE) != 0;
    col.length = total;
    // validity: Arrow's bitmaps (bit offset = array offset) become one byte per row, only when some batch has a NULL
    bool has_null = false;
    for (int b = 0; b < n_batches && !has_null; ++b) {
      const ArrowArray* a = batches[b]->children[p];
      int64_t off = batches[b]->offset + a->offset, len = batches[b]->length;
      has_null = a->null_count > 0;
      if (a->null_count < 0 && a->n_buffers > 0 && a->buffers[0]) has_null = range_has_null(static_cast<const uint8_t*>(a->buffers[0]), off, len);
    }
    if (has_null) {
      uint8_t* bytes = static_cast<uint8_t*>(pin_get(size_t(total)));
      staged.emplace_back(bytes, size_t(total));
      int64_t row = 0;
      for (int b = 0; b < n_batches; ++b) {
        const ArrowArray* a = batches[b]->children[p];
        const int64_t off = batches[b]->offset + a->offset, len = batches[b]->length;
        const uint8_t* bits = a->n_buffers > 0 ? static_cast<const uint8_t*>(a->buffers[0]) : nullptr;
        if (!bits || a->null_count == 0) memset(bytes + row, 1, size_t(len));
        else
          for (int64_t i = 0; i < len; ++i) bytes[row + i] = (bits[(off + i) >> 3] >> ((off + i) & 7)) & 1;
        row += len;
      }
      col.validity = alloc(ctx, size_t(total));
      ctx->h2d_bytes.fetch_add(total, std::memory_order_relaxed);
      FG_CUDA(cudaMemcpyAsync(col.validity->ptr, bytes, size_t(total), cudaMemcpyHostToDevice, ctx->stream));
    }
    if (dt != FLOCKGPU_UTF8 && zero_copy && !has_null && total > 0 && (col.chunks = try_host_chunks(ctx, batches, n_batches, p, dtype_width(dt)))) {
      // stays in page-locked host memory; kernels read it over PCIe or Table::dense() copies it later
      col.chunks->registration = registration;
    } else if (dt != FLOCKGPU_UTF8) {
      int w = dtype_width(dt);
      col.data = alloc(ctx, size_t(total) * w);
      int64_t row = 0;
      for (int b = 0; b < n_batches; ++b) {
        const ArrowArray* a = batches[b]->children[p];
        int64_t off = batches[b]->offset + a->offset, len = batches[b]->length;
        if (len == 0) continue;
        FG_CHECK(a->n_buffers >= 2 && a->buffers[1], FLOCKGPU_ERR_INVALID, "table_import: column \"%s\" has no data buffer", col.name.c_str());
        pieces.push_back({static_cast<char*>(col.data->ptr) + row * w, static_cast<const char*>(a->buffers[1]) + off * w, size_t(len) * w, fixed_bytes});
        fixed_bytes += size_t(len) * w;
        row += len;
      }
    } else {
      int64_t bytes = 0;
      for (int b = 0; b < n_batches; ++b) {
        const ArrowArray* a = batches[b]->children[p];
        int64_t off = batches[b]->offset + a->offset, len = batches[b]->length;
        if (len == 0) continue;
        FG_CHECK(a->n_buffers >= 3 && a->buffers[1], FLOCKGPU_ERR_INVALID, "table_import: Utf8 column \"%s\" has no offsets", col.name.c_str());
        const int32_t* o = static_cast<const int32_t*>(a->buffers[1]) + off;
        bytes += int64_t(o[len]) - int64_t(o[0]);
      }
      FG_CHECK(bytes < (int64_t(1) << 31), FLOCKGPU_ERR_UNSUPPORTED,
               "table_import: Utf8 column \"%s\" holds %lld bytes; at most 2^31-1 per relation", col.name.c_str(), (long long)bytes);
      col.offsets = alloc(ctx, size_t(total + 1) * 4);
      col.data = alloc(ctx, size_t(bytes));
      col.values_bytes = bytes;
      int64_t row = 0, byte = 0;
      for (int b = 0; b < n_batches; ++b) {
        const ArrowArray* a = batches[b]->children[p];
        int64_t off = batches[b]->offset + a->offset, len = batches[b]->length;
        if (len == 0) continue;
        const int32_t* o = static_cast<const int32_t*>(a->buffers[1]) + off;
        int64_t nb = int64_t(o[len]) - int64_t(o[0]);
        ctx->h2d_bytes.fetch_add(int64_t(len) * 4 + nb, std::memory_order_relaxed);
        FG_CUDA(cudaMemcpyAsync(col.offsets->as<int32_t>() + row, o, size_t(len) * 4, cudaMemcpyHostToDevice, ctx->stream));
        rebase_offsets(ctx, col.offsets->as<int32_t>() + row, len, int32_t(byte - int64_t(o[0])));
        if (nb > 0) {
          FG_CHECK(a->buffers[2], FLOCKGPU_ERR_INVALID, "table_import: Utf8 column \"%s\" has no value buffer", col.name.c_str());
          FG_CUDA(cudaMemcpyAsync(static_cast<char*>(col.data->ptr) + byte, static_cast<const char*>(a->buffers[2]) + o[0],
                                  size_t(nb), cudaMemcpyHostToDevice, ctx->stream));
        }
        row += len;
        byte += nb;
      }
      set_i32(ctx, col.offsets->as<int32_t>() + total, int32_t(bytes));
    }
    t->cols.push_back(std::move(col));
  }
  if (!pieces.empty()) issue_pieces(ctx, fan, pieces, fixed_bytes, staged);
  // inputs are only borrowed for the call: every copy must have left the host buffers before we return
  FG_CUDA(cudaStreamSynchronize(ctx->stream));
  return t;
}

// ------------------------------------------------------------------------------------------------
// export: Table (HBM) -> Arrow C Data (host)
// ------------------------------------------------------------------------------------------------
namespace {

// Pinned blocks are recycled through a per-context cache: cudaHostAlloc costs ~1 ms per call.
struct PinCache {
  std::mutex mu;
  std::unordered_multimap<size_t, void*> free_blocks;  // rounded size -> block
  ~PinCache() {
    for (auto& kv : free_blocks) cudaFreeHost(kv.second);
  }
};
std::shared_ptr<PinCache> pin_cache() {
  static std::shared_ptr<PinCache> c = std::make_shared<PinCache>();
  return c;
}
size_t round_pin(size_t n) {
  size_t r = 4096;
  while (r < n) r <<= 1;
  return r;
}
void* pin_get(size_t bytes) {
  size_t r = round_pin(bytes);
  auto c = pin_cache();
  {
    std::lock_guard<std::mutex> g(c->mu);
    auto it = c->free_blocks.find(r);
    if (it != c->free_blocks.end()) {
      void* p = it->second;
      c->free_blocks.erase(it);
      return p;
    }
  }
  void* p = nullptr;
  FG_CUDA(cudaHostAlloc(&p, r, cudaHostAllocDefault));
  return p;
}
void pin_put(void* p, size_t bytes) {
  auto c = pin_cache();
  std::lock_guard<std::mutex> g(c->mu);
  c->free_blocks.emplace(round_pin(bytes), p);
}

struct ArrayPrivate {
  std::vector<std::pair<void*, size_t>> blocks;  // pinned blocks owned by this array
  std::vector<const void*> buffers;
  std::vector<ArrowArray*> child_ptrs;
  std::vector<ArrowArray> children;
};

void release_array(ArrowArray* a) {
  if (!a || !a->release) return;
  auto* priv = static_cast<ArrayPrivate*>(a->private_data);
  if (priv) {
    for (auto& ch : priv->children)
      if (ch.release) ch.release(&ch);
    for (auto& b : priv->blocks) pin_put(b.first, b.second);
    delete priv;
  }
  a->release = nullptr;
}

struct SchemaPrivate {
  std::string format, name, metadata;
  std::vector<ArrowSchema*> child_ptrs;
  std::vector<ArrowSchema> children;
};

void release_schema(ArrowSchema* s) {
  if (!s || !s->release) return;
  auto* priv = static_cast<SchemaPrivate*>(s->private_data);
  if (priv) {
    for (auto& ch : priv->children)
      if (ch.release) ch.release(&ch);
    delete priv;
  }
  s->release = nullptr;
}

void fill_schema(ArrowSchema* s, const std::string& format, const std::string& name, const std::string& metadata,
                 bool nullable, size_t n_children) {
  auto* priv = new SchemaPrivate();
  priv->format = format;
  priv->name = name;
  priv->metadata = metadata;
  priv->children.resize(n_children);
  for (auto& c : priv->children) {
    memset(&c, 0, sizeof c);
    priv->child_ptrs.push_back(&c);
  }
  memset(s, 0, sizeof *s);
  s->format = priv->format.c_str();
  s->name = priv->name.c_str();
  s->metadata = priv->metadata.empty() ? nullptr : priv->metadata.data();
  s->flags = nullable ? ARROW_FLAG_NULLABLE : 0;
  s->n_children = int64_t(n_children);
  s->children = n_children ? priv->child_ptrs.data() : nullptr;
  s->release = release_schema;
  s->private_data = priv;
}

}  // namespace

void export_schema(const Table& t, ArrowSchema* out) {
  fill_schema(out, "+s", "", t.metadata, false, t.cols.size());
  auto* priv = static_cast<SchemaPrivate*>(out->private_data);
  for (size_t i = 0; i < t.cols.size(); ++i) {
    const Column& c = t.cols[i];
    fill_schema(&priv->children[i], c.format.empty() ? default_format(c.dtype) : c.format, c.name, "", c.nullable || c.all_null, 0);
  }
}

__global__ void shift_offsets_kernel(const int32_t* __restrict__ src, int32_t* __restrict__ dst, int64_t n) {
  int32_t base = src[0];
  int64_t i = blockIdx.x * int64_t(blockDim.x) + threadIdx.x;
  int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (; i < n; i += stride) dst[i] = src[i] - base;
}

void export_table(const CtxPtr& ctx, const Table& t, int64_t row_begin, int64_t row_count, ArrowSchema* out_schema,
                  ArrowArray* out_array) {
  FG_CHECK(out_schema && out_array, FLOCKGPU_ERR_INVALID, "table_export: null output");
  t.dense();
  if (row_count < 0) row_count = t.num_rows - row_begin;
  FG_CHECK(row_begin >= 0 && row_begin + row_count <= t.num_rows, FLOCKGPU_ERR_INVALID,
           "table_export: rows [%lld, %lld) outside table of %lld rows", (long long)row_begin,
           (long long)(row_begin + row_count), (long long)t.num_rows);
  auto top = std::make_unique<ArrayPrivate>();
  top->children.resize(t.cols.size());
  for (auto& c : top->children) memset(&c, 0, sizeof c);

  // Utf8: the first/last offsets of the exported row range decide how many bytes travel
  std::vector<int32_t> first_off(t.cols.size(), 0), last_off(t.cols.size(), 0);
  bool need_sync = false;
  int32_t* h_i32 = reinterpret_cast<int32_t*>(ctx->h_scalars);
  int k = 0;
  for (size_t i = 0; i < t.cols.size(); ++i) {
    const Column& c = t.cols[i];
    if (c.dtype == FLOCKGPU_UTF8 && row_count > 0) {
      FG_CHECK(k + 2 <= 512, FLOCKGPU_ERR_UNSUPPORTED, "table_export: too many Utf8 columns");
      FG_CUDA(cudaMemcpyAsync(h_i32 + k, c.offs() + row_begin, 4, cudaMemcpyDeviceToHost, ctx->stream));
      FG_CUDA(cudaMemcpyAsync(h_i32 + k + 1, c.offs() + row_begin + row_count, 4, cudaMemcpyDeviceToHost, ctx->stream));
      k += 2;
      need_sync = true;
    }
  }
  if (need_sync) {
    FG_CUDA(cudaStreamSynchronize(ctx->stream));
    k = 0;
    for (size_t i = 0; i < t.cols.size(); ++i)
      if (t.cols[i].dtype == FLOCKGPU_UTF8 && row_count > 0) {
        first_off[i] = h_i32[k];
        last_off[i] = h_i32[k + 1];
        k += 2;
      }
  }

  std::vector<BufferPtr> keep;  // device temporaries alive until the final sync
  struct PackJob {
    const uint8_t* bytes;
    uint8_t* bits;
    int64_t n;
    ArrowArray* array;
  };
  std::vector<PackJob> pack_jobs;
  for (size_t i = 0; i < t.cols.size(); ++i) {
    const Column& c = t.cols[i];
    auto priv = std::make_unique<ArrayPrivate>();
    ArrowArray& a = top->children[i];
    a.length = row_count;
    a.null_count = 0;
    a.offset = 0;
    void* validity = nullptr;
    if (c.all_null && row_count > 0) {
      size_t nb = size_t((row_count + 7) / 8);
      validity = pin_get(nb);
      memset(validity, 0, nb);
      priv->blocks.emplace_back(validity, nb);
      a.null_count = row_count;
    } else if (c.validity && row_count > 0) {
      // bytes to the host now, packed into Arrow's bitmap after the final sync (pack_jobs)
      uint8_t* bytes = static_cast<uint8_t*>(pin_get(size_t(row_count)));
      priv->blocks.emplace_back(bytes, size_t(row_count));
      size_t nb = size_t((row_count + 7) / 8);
      validity = pin_get(nb);
      memset(validity, 0, nb);
      priv->blocks.emplace_back(validity, nb);
      ctx->d2h_bytes.fetch_add(row_count, std::memory_order_relaxed);
      FG_CUDA(cudaMemcpyAsync(bytes, c.valid() + row_begin, size_t(row_count), cudaMemcpyDeviceToHost, ctx->stream));
      pack_jobs.push_back({bytes, static_cast<uint8_t*>(validity), row_count, &a});
    }
    if (c.dtype != FLOCKGPU_UTF8) {
      int w = c.width();
      size_t nb = size_t(row_count) * w;
      void* h = pin_get(nb ? nb : 8);
      priv->blocks.emplace_back(h, nb ? nb : 8);
      if (nb) {
        if (c.all_null) {
          memset(h, 0, nb);
        } else {
          ctx->d2h_bytes.fetch_add(int64_t(nb), std::memory_order_relaxed);
          FG_CUDA(cudaMemcpyAsync(h, static_cast<const char*>(c.values()) + row_begin * w, nb, cudaMemcpyDeviceToHost, ctx->stream));
        }
      }
      priv->buffers = {validity, h};
    } else {
      size_t nb_off = size_t(row_count + 1) * 4;
      int32_t* h_off = static_cast<int32_t*>(pin_get(nb_off));
      priv->blocks.emplace_back(h_off, nb_off);
      size_t nb_val = size_t(last_off[i] - first_off[i]);
      void* h_val = pin_get(nb_val ? nb_val : 8);
      priv->blocks.emplace_back(h_val, nb_val ? nb_val : 8);
      if (row_count > 0) {
        if (first_off[i] == 0) {
          ctx->d2h_bytes.fetch_add(int64_t(nb_off), std::memory_order_relaxed);
          FG_CUDA(cudaMemcpyAsync(h_off, c.offs() + row_begin, nb_off, cudaMemcpyDeviceToHost, ctx->stream));
        } else {
          BufferPtr tmp = alloc(ctx, nb_off);
          keep.push_back(tmp);
          int blocks = int(std::min<int64_t>((row_count + 256) / 256, ctx->sm_count * 8));
          {
            LaunchTimer lt(ctx, "shift_offsets_kernel");
            shift_offsets_kernel<<<blocks, 256, 0, ctx->stream>>>(c.offs() + row_begin, tmp->as<int32_t>(), row_count + 1);
          }
          count_launch(ctx);
          ctx->d2h_bytes.fetch_add(int64_t(nb_off), std::memory_order_relaxed);
          FG_CUDA(cudaMemcpyAsync(h_off, tmp->ptr, nb_off, cudaMemcpyDeviceToHost, ctx->stream));
        }
        if (nb_val) {
          ctx->d2h_bytes.fetch_add(int64_t(nb_val), std::memory_order_relaxed);
          FG_CUDA(cudaMemcpyAsync(h_val, static_cast<const char*>(c.values()) + first_off[i], nb_val, cudaMemcpyDeviceToHost, ctx->stream));
        }
      } else {
        h_off[0] = 0;
      }
      priv->buffers = {validity, h_off, h_val};
    }
    a.n_buffers = int64_t(priv->buffers.size());
    a.buffers = priv->buffers.data();
    a.n_children = 0;
    a.children = nullptr;
    a.dictionary = nullptr;
    a.release = release_array;
    a.private_data = priv.release();
  }
  FG_CUDA(cudaStreamSynchronize(ctx->stream));
  for (const PackJob& j : pack_jobs) {
    int64_t nulls = 0;
    for (int64_t r = 0; r < j.n; ++r) {
      if (j.bytes[r]) j.bits[r >> 3] |= uint8_t(1u << (r & 7));
      else ++nulls;
    }
    j.array->null_count = nulls;
  }

  for (auto& c : top->children) top->child_ptrs.push_back(&c);
  top->buffers = {nullptr};
  memset(out_array, 0, sizeof *out_array);
  out_array->length = row_count;
  out_array->null_count = 0;
  out_array->offset = 0;
  out_array->n_buffers = 1;
  out_array->buffers = top->buffers.data();
  out_array->n_children = int64_t(t.cols.size());
  out_array->children = top->child_ptrs.data();
  out_array->release = release_array;
  out_array->private_data = top.release();
  export_schema(t, out_schema);
}

// ------------------------------------------------------------------------------------------------
// concat / empty
// ------------------------------------------------------------------------------------------------
TablePtr empty_like(const CtxPtr& ctx, const Table& src) {
  auto t = std::make_shared<Table>();
  t->ctx = ctx;
  t->metadata = src.metadata;
  t->num_rows = 0;
  for (const Column& c : src.cols) {
    Column e;
    e.dtype = c.dtype;
    e.name = c.name;
    e.format = c.format;
    e.nullable = c.nullable;
    e.length = 0;
    e.data = alloc(ctx, 0);
    if (c.dtype == FLOCKGPU_UTF8) {
      e.offsets = alloc(ctx, 4);
      FG_CUDA(cudaMemsetAsync(e.offsets->ptr, 0, 4, ctx->stream));
    }
    t->cols.push_back(std::move(e));
  }
  return t;
}

TablePtr concat_tables(const CtxPtr& ctx, const std::vector<TablePtr>& tables) {
  FG_CHECK(!tables.empty(), FLOCKGPU_ERR_INVALID, "concat: no tables");
  if (tables.size() == 1) return tables[0];
  for (const TablePtr& t : tables) t->dense();
  const Table& first = *tables[0];
  int64_t total = 0;
  for (const TablePtr& t : tables) {
    FG_CHECK(t->cols.size() == first.cols.size(), FLOCKGPU_ERR_INVALID, "concat: column count differs");
    for (size_t i = 0; i < first.cols.size(); ++i)
      FG_CHECK(t->cols[i].dtype == first.cols[i].dtype, FLOCKGPU_ERR_INVALID, "concat: column %zu type differs", i);
    total += t->num_rows;
  }
  FG_CHECK(total < (int64_t(1) << 32) - 1, FLOCKGPU_ERR_UNSUPPORTED, "concat: more than 2^32-2 rows");
  auto out = std::make_shared<Table>();
  out->ctx = ctx;
  out->metadata = first.metadata;
  out->num_rows = total;
  for (size_t i = 0; i < first.cols.size(); ++i) {
    Column c;
    c.dtype = first.cols[i].dtype;
    c.name = first.cols[i].name;
    c.format = first.cols[i].format;
    c.nullable = first.cols[i].nullable;
    c.length = total;
    bool any_validity = false;
    for (const TablePtr& t : tables) any_validity |= t->cols[i].validity != nullptr;
    if (any_validity) {
      c.validity = alloc(ctx, size_t(total));
      int64_t row = 0;
      for (const TablePtr& t : tables) {
        const Column& s = t->cols[i];
        if (s.length) {
          if (s.validity) FG_CUDA(cudaMemcpyAsync(c.validity->as<uint8_t>() + row, s.valid(), size_t(s.length), cudaMemcpyDeviceToDevice, ctx->stream));
          else FG_CUDA(cudaMemsetAsync(c.validity->as<uint8_t>() + row, 1, size_t(s.length), ctx->stream));
        }
        row += s.length;
      }
    }
    if (c.dtype != FLOCKGPU_UTF8) {
      int w = c.width();
      c.data = alloc(ctx, size_t(total) * w);
      int64_t row = 0;
      for (const TablePtr& t : tables) {
        const Column& s = t->cols[i];
        FG_CHECK(!s.all_null, FLOCKGPU_ERR_UNSUPPORTED, "concat: NULL column");
        if (s.length)
          FG_CUDA(cudaMemcpyAsync(static_cast<char*>(c.data->ptr) + row * w, s.values(), size_t(s.length) * w,
                                  cudaMemcpyDeviceToDevice, ctx->stream));
        row += s.length;
      }
    } else {
      // value-byte totals are host-known (values_bytes), so no read-back is needed
      int64_t bytes = 0;
      for (const TablePtr& t : tables) bytes += t->cols[i].values_bytes;
      FG_CHECK(bytes < (int64_t(1) << 31), FLOCKGPU_ERR_UNSUPPORTED, "concat: Utf8 column exceeds 2^31-1 bytes");
      c.offsets = alloc(ctx, size_t(total + 1) * 4);
      c.data = alloc(ctx, size_t(bytes));
      c.values_bytes = bytes;
      int64_t row = 0, byte = 0;
      for (const TablePtr& t : tables) {
        const Column& s = t->cols[i];
        if (s.length) {
          // s.offsets may start at a non-zero base: shift to `byte`
          int blocks = int(std::min<int64_t>((s.length + 255) / 256, ctx->sm_count * 8));
          {
            LaunchTimer lt(ctx, "shift_offsets_kernel");
            shift_offsets_kernel<<<blocks, 256, 0, ctx->stream>>>(s.offs(), c.offsets->as<int32_t>() + row, s.length);
          }
          count_launch(ctx);
          rebase_offsets(ctx, c.offsets->as<int32_t>() + row, s.length, int32_t(byte));
          if (s.values_bytes) {
            // value bytes of `s` start at s.offsets[0]; tables built by this library always start at 0
            FG_CUDA(cudaMemcpyAsync(static_cast<char*>(c.data->ptr) + byte, s.values(), size_t(s.values_bytes),
                                    cudaMemcpyDeviceToDevice, ctx->stream));
          }
        }
        row += s.length;
        byte += s.values_bytes;
      }
      set_i32(ctx, c.offsets->as<int32_t>() + total, int32_t(bytes));
    }
    out->cols.push_back(std::move(c));
  }
  return out;
}

}  // namespace fg

// ================================================================================================
// extern "C": context + table entry points
// ================================================================================================
using namespace fg;

extern "C" {

const char* flockgpu_last_error(void) { return g_last_error.c_str(); }

const char* flockgpu_version(void) { return "flockgpu 0.1 (sm_90a, CUDA " FG_STR(CUDART_VERSION) ")"; }

int flockgpu_open(int device, flockgpu_ctx** out) {
  return guarded([&] {
    FG_CHECK(out, FLOCKGPU_ERR_INVALID, "open: null out pointer");
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
      fail(FLOCKGPU_ERR_NO_DEVICE, "open: no CUDA device available (%s); this library has no CPU fallback",
           e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    FG_CHECK(device >= 0 && device < n, FLOCKGPU_ERR_INVALID, "open: device %d out of range (have %d)", device, n);
    FG_CUDA(cudaSetDevice(device));
    auto core = std::make_shared<CtxCore>();
    core->device = device;
    cudaDeviceProp prop;
    FG_CUDA(cudaGetDeviceProperties(&prop, device));
    core->sm_count = prop.multiProcessorCount;
    // the single-wave prefix needs co-resident CTAs (cooperative launch); without it every compaction uses look-back
    int coop = 0;
    FG_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, device));
    if (!coop) core->compact_mode = 1;
    FG_CUDA(cudaStreamCreateWithFlags(&core->stream, cudaStreamNonBlocking));
    for (int i = 0; i < CtxCore::kCopyStreams; ++i) {
      FG_CUDA(cudaStreamCreateWithFlags(&core->copy_streams[i], cudaStreamNonBlocking));
      FG_CUDA(cudaEventCreateWithFlags(&core->copy_join[i], cudaEventDisableTiming));
    }
    FG_CUDA(cudaEventCreateWithFlags(&core->copy_fork, cudaEventDisableTiming));
    FG_CUDA(cudaDeviceGetDefaultMemPool(&core->pool, device));
    uint64_t threshold = UINT64_MAX;  // keep freed blocks in the pool: allocation is on the hot path
    FG_CUDA(cudaMemPoolSetAttribute(core->pool, cudaMemPoolAttrReleaseThreshold, &threshold));
    FG_CUDA(cudaHostAlloc(&core->h_scalars, (CtxCore::kScalars + CtxCore::kPendingSlots) * sizeof(unsigned long long), cudaHostAllocDefault));
    FG_CUDA(cudaMalloc(&core->d_scalars, CtxCore::kScalars * sizeof(unsigned long long)));
    FG_CUDA(cudaMemset(core->d_scalars, 0, CtxCore::kScalars * sizeof(unsigned long long)));
    for (int i = 0; i < 16; ++i) {
      FG_CUDA(cudaEventCreate(&core->timer_start[i]));
      FG_CUDA(cudaEventCreate(&core->timer_stop[i]));
    }
    *out = new flockgpu_ctx{core};
  });
}

int flockgpu_close(flockgpu_ctx* ctx) {
  return guarded([&] {
    if (!ctx) return;
    if (ctx->core && ctx->core->stream) {
      cudaSetDevice(ctx->core->device);
      cudaStreamSynchronize(ctx->core->stream);
      dump_filter_traces(ctx->core);
    }
    delete ctx;
    host_trace_dump(false);
  });
}

int flockgpu_synchronize(flockgpu_ctx* ctx) {
  return guarded([&] {
    auto c = core_of(ctx);
    FG_CUDA(cudaStreamSynchronize(c->stream));
    dump_filter_traces(c);
  });
}

int flockgpu_timer_start(flockgpu_ctx* ctx, int slot) {
  return guarded([&] {
    auto c = core_of(ctx);
    FG_CHECK(slot >= 0 && slot < 16, FLOCKGPU_ERR_INVALID, "timer slot out of range");
    FG_CUDA(cudaEventRecord(c->timer_start[slot], c->stream));
  });
}

int flockgpu_timer_stop(flockgpu_ctx* ctx, int slot) {
  return guarded([&] {
    auto c = core_of(ctx);
    FG_CHECK(slot >= 0 && slot < 16, FLOCKGPU_ERR_INVALID, "timer slot out of range");
    FG_CUDA(cudaEventRecord(c->timer_stop[slot], c->stream));
  });
}

int flockgpu_timer_elapsed_ms(flockgpu_ctx* ctx, int slot, float* ms) {
  return guarded([&] {
    auto c = core_of(ctx);
    FG_CHECK(slot >= 0 && slot < 16 && ms, FLOCKGPU_ERR_INVALID, "timer slot out of range");
    FG_CUDA(cudaEventSynchronize(c->timer_stop[slot]));
    FG_CUDA(cudaEventElapsedTime(ms, c->timer_start[slot], c->timer_stop[slot]));
  });
}

int64_t flockgpu_kernel_launches(flockgpu_ctx* ctx) { return ctx && ctx->core ? ctx->core->launches.load() : -1; }

int64_t flockgpu_overlapped_launches(flockgpu_ctx* ctx) { return ctx && ctx->core ? ctx->core->overlapped.load() : -1; }

int64_t flockgpu_bytes_moved(flockgpu_ctx* ctx, int32_t direction) {
  if (!ctx || !ctx->core) return -1;
  return direction == 0 ? ctx->core->h2d_bytes.load() : ctx->core->d2h_bytes.load();
}

int flockgpu_host_alloc(flockgpu_ctx* ctx, int64_t bytes, void** out) {
  return guarded([&] {
    auto c = core_of(ctx);
    FG_CHECK(out && bytes >= 0, FLOCKGPU_ERR_INVALID, "host_alloc: bad arguments");
    const size_t need = (size_t(bytes ? bytes : 8) + 255) & ~size_t(255);  // Arrow wants 64-byte alignment; kernels read 16-byte vectors
    std::lock_guard<std::mutex> g(c->pin_mu);
    size_t slab = c->pin_slabs.size();
    for (size_t i = c->pin_slabs.size(); i-- > 0;) {  // newest first: consecutive allocations stay contiguous
      CtxCore::PinSlab& sl = c->pin_slabs[i];
      if (sl.base && sl.size - sl.used >= need) {
        slab = i;
        break;
      }
    }
    if (slab == c->pin_slabs.size()) {
      CtxCore::PinSlab sl;
      sl.size = std::max(need, CtxCore::kPinSlabBytes);
      FG_CUDA(cudaSetDevice(c->device));
      void* p = nullptr;
      FG_CUDA(cudaHostAlloc(&p, sl.size, cudaHostAllocDefault));
      sl.base = static_cast<char*>(p);
      // reuse the table entry of a released slab if there is one
      slab = c->pin_slabs.size();
      for (size_t i = 0; i < c->pin_slabs.size(); ++i)
        if (!c->pin_slabs[i].base) {
          slab = i;
          break;
        }
      if (slab == c->pin_slabs.size()) c->pin_slabs.push_back(sl);
      else c->pin_slabs[slab] = sl;
    }
    CtxCore::PinSlab& sl = c->pin_slabs[slab];
    void* p = sl.base + sl.used;
    sl.used += need;
    ++sl.live;
    c->pin_owner.emplace(p, slab);
    *out = p;
  });
}

int flockgpu_host_free(flockgpu_ctx* ctx, void* ptr) {
  return guarded([&] {
    auto c = core_of(ctx);
    std::lock_guard<std::mutex> g(c->pin_mu);
    auto it = c->pin_owner.find(ptr);
    FG_CHECK(it != c->pin_owner.end(), FLOCKGPU_ERR_INVALID, "host_free: pointer was not allocated by host_alloc");
    CtxCore::PinSlab& sl = c->pin_slabs[it->second];
    c->pin_owner.erase(it);
    if (--sl.live == 0) {
      // the slab is empty again: keep one standard slab for reuse, give everything else back
      size_t idle = 0;
      for (const CtxCore::PinSlab& o : c->pin_slabs) idle += (o.base && o.live == 0 && &o != &sl) ? 1 : 0;
      if (sl.size > CtxCore::kPinSlabBytes || idle >= 1) {
        FG_CUDA(cudaFreeHost(sl.base));
        sl = CtxCore::PinSlab{};
      } else {
        sl.used = 0;
      }
    }
  });
}

int flockgpu_flush_l2(flockgpu_ctx* ctx) {
  return guarded([&] {
    auto c = core_of(ctx);
    std::lock_guard<std::recursive_mutex> g(c->mu);
    if (!c->l2_flush) {
      int l2_bytes = 0;
      FG_CUDA(cudaDeviceGetAttribute(&l2_bytes, cudaDevAttrL2CacheSize, c->device));
      c->l2_flush_bytes = 3 * size_t(std::max(l2_bytes, 1 << 20));  // 3x the L2 (150 MB on an H100's 50 MB)
      FG_CUDA(cudaMalloc(&c->l2_flush, c->l2_flush_bytes));
    }
    FG_CUDA(cudaMemsetAsync(c->l2_flush, 0x5a, c->l2_flush_bytes, c->stream));
  });
}

int flockgpu_table_import(flockgpu_ctx* ctx, const struct ArrowSchema* schema, const struct ArrowArray* const* batches,
                          int32_t n_batches, const int32_t* projection, int32_t n_projection, flockgpu_table** out) {
  return guarded([&] {
    auto c = core_of(ctx);
    FG_CHECK(out, FLOCKGPU_ERR_INVALID, "table_import: null out pointer");
    std::lock_guard<std::recursive_mutex> g(c->mu);
    FG_CUDA(cudaSetDevice(c->device));
    *out = wrap_table(import_batches(c, schema, batches, n_batches, projection, n_projection));
  });
}

int flockgpu_table_export(flockgpu_ctx* ctx, const flockgpu_table* table, int64_t row_begin, int64_t row_count,
                          struct ArrowSchema* out_schema, struct ArrowArray* out_array) {
  return guarded([&] {
    auto c = core_of(ctx);
    std::lock_guard<std::recursive_mutex> g(c->mu);
    FG_CUDA(cudaSetDevice(c->device));
    export_table(c, deref(table), row_begin, row_count, out_schema, out_array);
  });
}

int flockgpu_table_schema(flockgpu_ctx* ctx, const flockgpu_table* table, struct ArrowSchema* out_schema) {
  return guarded([&] {
    (void)ctx;
    FG_CHECK(out_schema, FLOCKGPU_ERR_INVALID, "table_schema: null output");
    export_schema(deref(table), out_schema);
  });
}

int flockgpu_table_retain(flockgpu_table* table) {
  return guarded([&] {
    FG_CHECK(table, FLOCKGPU_ERR_INVALID, "null table handle");
    table->refs.fetch_add(1);
  });
}

int flockgpu_table_release(flockgpu_table* table) {
  return guarded([&] {
    if (!table) return;
    if (table->refs.fetch_sub(1) == 1) {
      if (table->table && table->table->ctx) cudaSetDevice(table->table->ctx->device);
      delete table;
    }
  });
}

int64_t flockgpu_table_num_rows(const flockgpu_table* table) {
  if (!table || !table->table) return -1;
  int64_t n = -1;
  guarded([&] {
    table->table->resolve();  // waits for a survivor count that is still in flight
    n = table->table->num_rows;
  });
  return n;
}

int flockgpu_set_option(flockgpu_ctx* ctx, const char* name, int64_t value) {
  return guarded([&] {
    auto c = core_of(ctx);
    FG_CHECK(name, FLOCKGPU_ERR_INVALID, "set_option: null name");
    std::lock_guard<std::recursive_mutex> g(c->mu);
    if (!strcmp(name, "feed_zero_copy")) c->feed_zero_copy = value != 0;
    else if (!strcmp(name, "compact_mode")) c->compact_mode = int(value);
    else if (!strcmp(name, "feed_register")) c->feed_register = value != 0;
    else if (!strcmp(name, "host_trace_dump")) host_trace_dump(value != 0);
    else if (!strcmp(name, "feed_stream_stores")) c->feed_stream_stores = value != 0;
    else if (!strcmp(name, "feed_stage_threads")) c->feed_stage_threads = int(std::max<int64_t>(0, std::min<int64_t>(value, 64)));
    else if (!strcmp(name, "exchange_window_mb")) c->exchange_window_mb = value;
    else fail(FLOCKGPU_ERR_INVALID, "set_option: unknown option \"%s\"", name);
  });
}

int flockgpu_profile_begin(flockgpu_ctx* ctx) {
  return guarded([&] {
    auto c = core_of(ctx);
    std::lock_guard<std::recursive_mutex> g(c->mu);
    for (auto& p : c->profile) {
      c->put_event(p.start, true);
      c->put_event(p.stop, true);
    }
    c->profile.clear();
    c->profiling = true;
  });
}

int flockgpu_profile_end(flockgpu_ctx* ctx, char* out_json, int32_t capacity) {
  return guarded([&] {
    auto c = core_of(ctx);
    FG_CHECK(out_json && capacity > 2, FLOCKGPU_ERR_INVALID, "profile_end: bad output buffer");
    std::lock_guard<std::recursive_mutex> g(c->mu);
    FG_CUDA(cudaSetDevice(c->device));
    c->profiling = false;
    FG_CUDA(cudaStreamSynchronize(c->stream));
    struct Acc {
      double ms = 0;
      int64_t n = 0;
    };
    std::vector<std::pair<std::string, Acc>> acc;
    for (auto& p : c->profile) {
      float ms = 0;
      FG_CUDA(cudaEventElapsedTime(&ms, p.start, p.stop));
      auto it = std::find_if(acc.begin(), acc.end(), [&](const std::pair<std::string, Acc>& kv) { return kv.first == p.kernel; });
      if (it == acc.end()) {
        acc.emplace_back(p.kernel, Acc{});
        it = acc.end() - 1;
      }
      it->second.ms += ms;
      it->second.n += 1;
      c->put_event(p.start, true);
      c->put_event(p.stop, true);
    }
    c->profile.clear();
    std::string s = "{";
    for (size_t i = 0; i < acc.size(); ++i) {
      char buf[256];
      snprintf(buf, sizeof buf, "%s\"%s\": {\"launches\": %lld, \"ms\": %.6f}", i ? ", " : "", acc[i].first.c_str(), (long long)acc[i].second.n,
               acc[i].second.ms);
      s += buf;
    }
    s += "}";
    FG_CHECK(int(s.size()) < capacity, FLOCKGPU_ERR_INVALID, "profile_end: output buffer too small (%zu bytes needed)", s.size() + 1);
    memcpy(out_json, s.c_str(), s.size() + 1);
  });
}

int32_t flockgpu_table_num_columns(const flockgpu_table* table) {
  return table && table->table ? int32_t(table->table->cols.size()) : -1;
}

int64_t flockgpu_table_nbytes(const flockgpu_table* table) { return table && table->table ? table->table->nbytes() : -1; }

int flockgpu_table_concat(flockgpu_ctx* ctx, flockgpu_table* const* tables, int32_t n, flockgpu_table** out) {
  return guarded([&] {
    auto c = core_of(ctx);
    FG_CHECK(out && tables && n > 0, FLOCKGPU_ERR_INVALID, "table_concat: bad arguments");
    std::lock_guard<std::recursive_mutex> g(c->mu);
    FG_CUDA(cudaSetDevice(c->device));
    std::vector<TablePtr> ts;
    for (int i = 0; i < n; ++i) ts.push_back(tables[i] ? tables[i]->table : nullptr);
    for (auto& t : ts) FG_CHECK(t, FLOCKGPU_ERR_INVALID, "table_concat: null table");
    *out = wrap_table(concat_tables(c, ts));
  });
}

}  // extern "C"
