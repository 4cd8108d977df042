// ipc.cc -- Arrow IPC record-batch messages <-> device tables: the payload decode / encode that brackets every hot call.
//
// In the reference a function's input arrives as `DataFrame { header, body }` pairs = the `data_header` / `data_body` of
// Arrow-Flight messages (flock/src/runtime/payload.rs:116-124): `Payload::to_record_batch` runs
// `flight_data_to_arrow_batch` on every frame (payload.rs:161-192; the arena hands the frames over,
// flock/src/runtime/arena/mod.rs:114-169) and `to_payload` / `to_bytes` run `flight_data_from_arrow_batch` on the
// way out (flock/src/transmute.rs:178-247).  A frame's header is the flatbuffer `Message { RecordBatch { length,
// nodes[], buffers[] } }`, its body the 8-byte-aligned concatenation of the column buffers.
//
// Import: the body buffers ARE the column buffers, so nothing is decoded -- the flatbuffer is read for the buffer
// extents, the extents become Arrow C arrays that point INTO the bodies, and the ordinary import (core.cu:
// import_batches) moves them to HBM (projection pushdown, staging of pageable memory and the zero-copy feed of
// page-locked bodies included).  Export: pack_frames is the one place that lays out and writes frames, for export_ipc
// (one frame, copied to the host) and export_payload (zstd_enc.cu: many frames, copied out or compressed first):
// payload_layout_kernel reads the Utf8 extents and null counts, the host writes the flatbuffer headers by hand, and
// ipc_segment_kernel packs every body in HBM (values, validity bytes into bitmaps, Utf8 offsets rebased to the frame).
// The same segment kernel assembles the columns of decoded zstd bodies at import (zstd.cu); a profile names the two
// uses payload_pack_kernel and payload_assemble_kernel.  Encoding::None only
// here; lz4 / snappy / zlib are not restated (DESIGN.md section 7).
#include <algorithm>
#include <cstring>
#include <memory>
#include <vector>

#include "../internal.h"

namespace fg {

namespace {

// ---- the few flatbuffer accessors an Arrow Message needs ---------------------------------------------------------------
struct Fb {
  const uint8_t* p;
  size_t n;
  template <typename T>
  T rd(size_t at) const {
    FG_CHECK(at <= n && sizeof(T) <= n - at, FLOCKGPU_ERR_INVALID, "IPC header: truncated or corrupt flatbuffer (offset %zu of %zu)", at, n);
    T v;
    memcpy(&v, p + at, sizeof(T));
    return v;
  }
  // position of field `id` of the table at `table`, 0 when absent
  size_t field(size_t table, int id) const {
    const int32_t soff = rd<int32_t>(table);
    const size_t vt = size_t(int64_t(table) - soff);
    const uint16_t vt_len = rd<uint16_t>(vt);
    const size_t slot = 4 + size_t(id) * 2;
    if (slot + 2 > vt_len) return 0;
    const uint16_t off = rd<uint16_t>(vt + slot);
    return off ? table + off : 0;
  }
  size_t indirect(size_t at) const { return at + rd<uint32_t>(at); }
};

}  // namespace

FrameLayout parse_record_batch_message(const uint8_t* header, int64_t header_len) {
  FG_CHECK(header && header_len >= 8, FLOCKGPU_ERR_INVALID, "IPC header: empty");
  Fb fb{header, size_t(header_len)};
  const size_t msg = fb.indirect(0);
  const size_t f_type = fb.field(msg, 1), f_header = fb.field(msg, 2);
  FG_CHECK(f_type && f_header, FLOCKGPU_ERR_INVALID, "IPC header: Message without a header union");
  FrameLayout L;
  const uint8_t type = fb.rd<uint8_t>(f_type);
  FG_CHECK(type == 3, FLOCKGPU_ERR_UNSUPPORTED, "IPC header: message type %d (only RecordBatch = 3 frames carry data; dictionaries are not supported)", int(type));
  if (size_t f = fb.field(msg, 3)) L.body_length = fb.rd<int64_t>(f);
  const size_t rb = fb.indirect(f_header);
  if (size_t f = fb.field(rb, 0)) L.length = fb.rd<int64_t>(f);
  FG_CHECK(!fb.field(rb, 3), FLOCKGPU_ERR_UNSUPPORTED, "IPC header: compressed record batch bodies (BodyCompression) are not supported");
  if (size_t f = fb.field(rb, 1)) {
    const size_t v = fb.indirect(f);
    const uint32_t n = fb.rd<uint32_t>(v);
    for (uint32_t i = 0; i < n; ++i) L.nodes.emplace_back(fb.rd<int64_t>(v + 4 + size_t(i) * 16), fb.rd<int64_t>(v + 4 + size_t(i) * 16 + 8));
  }
  if (size_t f = fb.field(rb, 2)) {
    const size_t v = fb.indirect(f);
    const uint32_t n = fb.rd<uint32_t>(v);
    for (uint32_t i = 0; i < n; ++i) L.buffers.emplace_back(fb.rd<int64_t>(v + 4 + size_t(i) * 16), fb.rd<int64_t>(v + 4 + size_t(i) * 16 + 8));
  }
  return L;
}

namespace {

// ---- writing the header of one record batch --------------------------------------------------------------------------------
struct Out {
  std::vector<uint8_t> b;
  template <typename T>
  void put(size_t at, T v) {
    if (b.size() < at + sizeof(T)) b.resize(at + sizeof(T), 0);
    memcpy(b.data() + at, &v, sizeof(T));
  }
};

// The flatbuffer Message { RecordBatch } of one frame: (length, null_count) per field, (offset, length) per buffer.
std::vector<uint8_t> build_record_batch_message(int64_t length, const std::vector<std::pair<int64_t, int64_t>>& nodes,
                                                const std::vector<std::pair<int64_t, int64_t>>& buffers, int64_t body_len) {
  // fixed layout, every offset pointing forward:
  //   0 root -> 16 | 4 Message vtable (12 B) | 16 Message table (24 B) | 40 RecordBatch vtable (10 B) | 56 RecordBatch table
  //   (24 B) | 84 nodes: u32 n, n x {i64 length, i64 null_count} | buffers: u32 n (at 4 mod 8), n x {i64 offset, i64 length}
  Out o;
  const size_t MT = 16, RT = 56, NODES = 84;
  const size_t BUFS = NODES + 4 + nodes.size() * 16 + 4;  // the elements of both vectors are 8-byte aligned
  o.put<uint32_t>(0, uint32_t(MT));
  // Message vtable: version, header_type, header, bodyLength
  o.put<uint16_t>(4, 12);
  o.put<uint16_t>(6, 24);
  o.put<uint16_t>(8, 16);   // version      @ MT + 16
  o.put<uint16_t>(10, 18);  // header_type  @ MT + 18
  o.put<uint16_t>(12, 4);   // header       @ MT + 4
  o.put<uint16_t>(14, 8);   // bodyLength   @ MT + 8
  o.put<int32_t>(MT, int32_t(MT - 4));
  o.put<uint32_t>(MT + 4, uint32_t(RT - (MT + 4)));
  o.put<int64_t>(MT + 8, body_len);
  o.put<int16_t>(MT + 16, 4);  // MetadataVersion::V5 (what arrow-rs 6 and pyarrow write)
  o.put<uint8_t>(MT + 18, 3);  // MessageHeader::RecordBatch
  // RecordBatch vtable: length, nodes, buffers
  o.put<uint16_t>(40, 10);
  o.put<uint16_t>(42, 24);
  o.put<uint16_t>(44, 8);   // length  @ RT + 8
  o.put<uint16_t>(46, 4);   // nodes   @ RT + 4
  o.put<uint16_t>(48, 16);  // buffers @ RT + 16
  o.put<int32_t>(RT, int32_t(RT - 40));
  o.put<uint32_t>(RT + 4, uint32_t(NODES - (RT + 4)));
  o.put<int64_t>(RT + 8, length);
  o.put<uint32_t>(RT + 16, uint32_t(BUFS - (RT + 16)));
  o.put<uint32_t>(NODES, uint32_t(nodes.size()));
  for (size_t i = 0; i < nodes.size(); ++i) {
    o.put<int64_t>(NODES + 4 + i * 16, nodes[i].first);
    o.put<int64_t>(NODES + 4 + i * 16 + 8, nodes[i].second);
  }
  o.put<uint32_t>(BUFS, uint32_t(buffers.size()));
  for (size_t i = 0; i < buffers.size(); ++i) {
    o.put<int64_t>(BUFS + 4 + i * 16, buffers[i].first);
    o.put<int64_t>(BUFS + 4 + i * 16 + 8, buffers[i].second);
  }
  o.b.resize((o.b.size() + 7) & ~size_t(7), 0);
  return o.b;
}

}  // namespace

std::vector<size_t> field_buffers(const ArrowSchema* schema) {
  std::vector<size_t> first(size_t(schema->n_children) + 1, 0);
  for (int64_t c = 0; c < schema->n_children; ++c)
    first[size_t(c) + 1] = first[size_t(c)] + (dtype_from_format(schema->children[c]->format) == FLOCKGPU_UTF8 ? 3 : 2);
  return first;
}

// Everything about frame `f` that its header alone decides, against the schema and a body of `body_len` bytes: field
// count, batch and field lengths, null counts, and every buffer extent.  The Utf8 offsets live in the body; the caller
// checks them (check_utf8_extent).
void check_frame_layout(const ArrowSchema* schema, int f, const FrameLayout& L, int64_t body_len) {
  const int64_t n_fields = schema->n_children;
  FG_CHECK(int64_t(L.nodes.size()) == n_fields, FLOCKGPU_ERR_INVALID, "table_import_ipc: frame %d describes %zu fields, the schema has %lld", f, L.nodes.size(),
           (long long)n_fields);
  FG_CHECK(L.length >= 0 && L.length < (int64_t(1) << 31), FLOCKGPU_ERR_INVALID, "table_import_ipc: frame %d: batch length %lld", f, (long long)L.length);
  const std::vector<size_t> first_buf = field_buffers(schema);
  for (int64_t c = 0; c < n_fields; ++c) {
    const char* fmt = schema->children[c]->format;
    const int dt = dtype_from_format(fmt);
    FG_CHECK(dt >= 0, FLOCKGPU_ERR_UNSUPPORTED, "table_import_ipc: column \"%s\" has unsupported Arrow format \"%s\"", schema->children[c]->name, fmt ? fmt : "");
    const size_t next = first_buf[size_t(c)];
    FG_CHECK(first_buf[size_t(c) + 1] <= L.buffers.size(), FLOCKGPU_ERR_INVALID, "table_import_ipc: frame %d lists too few buffers", f);
    const int64_t length = L.nodes[size_t(c)].first, null_count = L.nodes[size_t(c)].second;
    FG_CHECK(length == L.length, FLOCKGPU_ERR_INVALID, "table_import_ipc: frame %d: field length %lld differs from the batch length %lld", f,
             (long long)length, (long long)L.length);
    FG_CHECK(null_count >= 0 && null_count <= length, FLOCKGPU_ERR_INVALID, "table_import_ipc: frame %d: null count %lld of %lld rows", f,
             (long long)null_count, (long long)length);
    for (size_t b = next; b < first_buf[size_t(c) + 1]; ++b) {
      const auto& ext = L.buffers[b];
      FG_CHECK(ext.first >= 0 && ext.second >= 0 && ext.first <= body_len && ext.second <= body_len - ext.first, FLOCKGPU_ERR_INVALID,
               "table_import_ipc: frame %d: buffer [%lld, +%lld) outside the %lld-byte body", f, (long long)ext.first, (long long)ext.second,
               (long long)body_len);
    }
    // every buffer holds what `length` rows need (a frame that claims more rows than it carries would be read past its end)
    const auto& validity = L.buffers[next];
    FG_CHECK(validity.second == 0 ? null_count == 0 : validity.second >= (length + 7) / 8, FLOCKGPU_ERR_INVALID,
             "table_import_ipc: frame %d, column \"%s\": validity bitmap of %lld bytes for %lld rows with %lld nulls", f, schema->children[c]->name,
             (long long)validity.second, (long long)length, (long long)null_count);
    if (dt == FLOCKGPU_UTF8) {
      const auto& offs = L.buffers[next + 1];
      FG_CHECK(length == 0 || offs.second >= (length + 1) * 4, FLOCKGPU_ERR_INVALID, "table_import_ipc: frame %d, column \"%s\": offsets buffer of %lld bytes for %lld rows", f,
               schema->children[c]->name, (long long)offs.second, (long long)length);
    } else {
      const auto& data = L.buffers[next + 1];
      FG_CHECK(data.second >= length * int64_t(dtype_width(dt)), FLOCKGPU_ERR_INVALID, "table_import_ipc: frame %d, column \"%s\": %lld value bytes for %lld rows", f,
               schema->children[c]->name, (long long)data.second, (long long)length);
    }
  }
}

void check_utf8_extent(int f, const char* column, int32_t first, int32_t last, int64_t value_bytes) {
  FG_CHECK(first >= 0 && last >= first && int64_t(last) <= value_bytes, FLOCKGPU_ERR_INVALID, "table_import_ipc: frame %d, column \"%s\": offsets [%d, %d] outside the %lld value bytes", f,
           column, first, last, (long long)value_bytes);
}

// Arrow C arrays whose buffers point INTO the frames' bodies: pure host work, no device, no context -- every offset and
// length a frame claims is checked against the bytes it came with before anything dereferences them.
struct IpcFrame {
  ArrowArray top;
  std::vector<ArrowArray> kids;
  std::vector<ArrowArray*> kid_ptrs;
  std::vector<std::vector<const void*>> bufs;
  const void* top_buf[1] = {nullptr};
};
struct IpcFrames {
  std::vector<std::unique_ptr<IpcFrame>> frames;
  std::vector<const ArrowArray*> tops;
};

IpcFrames view_ipc_frames(const ArrowSchema* schema, const uint8_t* const* headers, const int64_t* header_lens, const uint8_t* const* bodies,
                          const int64_t* body_lens, int n_frames) {
  FG_CHECK(schema && schema->format && !strcmp(schema->format, "+s"), FLOCKGPU_ERR_INVALID, "table_import_ipc: schema must be a struct (\"+s\")");
  FG_CHECK(n_frames >= 0 && (n_frames == 0 || (headers && header_lens && bodies && body_lens)), FLOCKGPU_ERR_INVALID, "table_import_ipc: bad frame list");
  const int64_t n_fields = schema->n_children;
  const std::vector<size_t> first_buf = field_buffers(schema);
  IpcFrames out;
  for (int f = 0; f < n_frames; ++f) {
    FG_CHECK(body_lens[f] >= 0 && (body_lens[f] == 0 || bodies[f]), FLOCKGPU_ERR_INVALID, "table_import_ipc: frame %d has no body", f);
    const FrameLayout L = parse_record_batch_message(headers[f], header_lens[f]);
    check_frame_layout(schema, f, L, body_lens[f]);
    auto fr = std::make_unique<IpcFrame>();
    fr->kids.resize(size_t(n_fields));
    fr->bufs.resize(size_t(n_fields));
    for (int64_t c = 0; c < n_fields; ++c) {
      const size_t next = first_buf[size_t(c)], want = first_buf[size_t(c) + 1] - next;
      ArrowArray& a = fr->kids[size_t(c)];
      memset(&a, 0, sizeof a);
      a.length = L.nodes[size_t(c)].first;
      a.null_count = L.nodes[size_t(c)].second;
      for (size_t b = 0; b < want; ++b) {
        const auto& ext = L.buffers[next + b];
        // a zero-length validity buffer means "no nulls"; zero-length data buffers of empty batches still get an address
        const bool absent = ext.second == 0 && b == 0;
        fr->bufs[size_t(c)].push_back(absent ? nullptr : static_cast<const void*>(bodies[f] + ext.first));
      }
      if (dtype_from_format(schema->children[c]->format) == FLOCKGPU_UTF8 && a.length > 0) {
        const auto& offs = L.buffers[next + 1];
        int32_t first, last;
        memcpy(&first, bodies[f] + offs.first, 4);
        memcpy(&last, bodies[f] + offs.first + a.length * 4, 4);
        check_utf8_extent(f, schema->children[c]->name, first, last, L.buffers[next + 2].second);
      }
      a.n_buffers = int64_t(want);
      a.buffers = fr->bufs[size_t(c)].data();
    }
    for (ArrowArray& a : fr->kids) fr->kid_ptrs.push_back(&a);
    memset(&fr->top, 0, sizeof fr->top);
    fr->top.length = L.length;
    fr->top.n_buffers = 1;
    fr->top.buffers = fr->top_buf;
    fr->top.n_children = n_fields;
    fr->top.children = fr->kid_ptrs.data();
    out.tops.push_back(&fr->top);
    out.frames.push_back(std::move(fr));
  }
  return out;
}

namespace {

// ---- payload_layout_kernel: one CTA per (frame, column) item -----------------------------------------------------------
struct LayoutItem {
  const int32_t* offs;   // Utf8: the column's offsets (else null)
  const uint8_t* valid;  // a column with a validity buffer (else null)
  int64_t row, rows;
};

__global__ void __launch_bounds__(256) payload_layout_kernel(const LayoutItem* __restrict__ items, int n, int64_t* __restrict__ out) {
  __shared__ unsigned long long nulls;
  for (int i = blockIdx.x; i < n; i += gridDim.x) {
    const LayoutItem it = items[i];
    if (threadIdx.x == 0) nulls = 0;
    __syncthreads();
    if (it.valid) {
      unsigned long long c = 0;
      for (int64_t r = threadIdx.x; r < it.rows; r += blockDim.x) c += it.valid[it.row + r] == 0;
      for (int d = 16; d; d >>= 1) c += __shfl_xor_sync(0xFFFFFFFFu, c, d);
      if ((threadIdx.x & 31) == 0 && c) atomicAdd(&nulls, c);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      out[3 * i] = it.offs ? it.offs[it.row] : 0;
      out[3 * i + 1] = it.offs ? it.offs[it.row + it.rows] : 0;
      out[3 * i + 2] = int64_t(nulls);
    }
    __syncthreads();
  }
}

// ---- ipc_segment_kernel: one CTA per segment -----------------------------------------------------------------------------
template <typename W>
__device__ __forceinline__ void copy_as(const Seg& g) {
  for (int64_t k = threadIdx.x; k < g.n / int64_t(sizeof(W)); k += blockDim.x) reinterpret_cast<W*>(g.dst)[k] = reinterpret_cast<const W*>(g.src)[k];
}

__global__ void __launch_bounds__(256) ipc_segment_kernel(const Seg* __restrict__ segs, int n_segs) {
  for (int s = blockIdx.x; s < n_segs; s += gridDim.x) {
    const Seg g = segs[s];
    const int64_t n = g.n;
    switch (g.kind) {
      case Seg::kCopy: {
        const uintptr_t a = reinterpret_cast<uintptr_t>(g.src) | reinterpret_cast<uintptr_t>(g.dst) | uintptr_t(n);
        if ((a & 15) == 0) copy_as<uint4>(g);
        else if ((a & 7) == 0) copy_as<uint64_t>(g);
        else if ((a & 3) == 0) copy_as<uint32_t>(g);
        else copy_as<uint8_t>(g);
        break;
      }
      case Seg::kOffsets: {
        int32_t* d = reinterpret_cast<int32_t*>(g.dst);
        if ((reinterpret_cast<uintptr_t>(g.src) & 3) == 0) {
          for (int64_t r = threadIdx.x; r < n; r += blockDim.x) d[r] = reinterpret_cast<const int32_t*>(g.src)[r] + g.arg;
        } else {  // a decoded body is byte-addressed: its offsets need not be word-aligned
          for (int64_t r = threadIdx.x; r < n; r += blockDim.x) {
            const uint8_t* w = g.src + 4 * r;
            d[r] = int32_t(uint32_t(w[0]) | (uint32_t(w[1]) << 8) | (uint32_t(w[2]) << 16) | (uint32_t(w[3]) << 24)) + g.arg;
          }
        }
        break;
      }
      case Seg::kBitsToBytes:
        for (int64_t r = threadIdx.x; r < n; r += blockDim.x) g.dst[r] = (g.src[r >> 3] >> (r & 7)) & 1;
        break;
      case Seg::kBytesToBits:
        for (int64_t k = threadIdx.x; k < (n + 7) / 8; k += blockDim.x) {
          uint32_t v = 0;
          for (int j = 0; j < 8 && 8 * k + j < n; ++j) v |= uint32_t(g.src[8 * k + j] != 0) << j;
          g.dst[k] = uint8_t(v);
        }
        break;
      case Seg::kFill:
        for (int64_t r = threadIdx.x; r < n; r += blockDim.x) g.dst[r] = uint8_t(g.arg);
        break;
      default:
        if (threadIdx.x == 0) *reinterpret_cast<int32_t*>(g.dst) = g.arg;
    }
  }
}

int64_t pad8(int64_t x) { return (x + 7) & ~int64_t(7); }
int64_t align16(int64_t x) { return (x + 15) & ~int64_t(15); }

}  // namespace

void add_segs(std::vector<Seg>& segs, int kind, const uint8_t* src, uint8_t* dst, int64_t n, int32_t arg) {
  if (kind == Seg::kSetI32) {
    segs.push_back({nullptr, dst, 0, kind, arg});
    return;
  }
  // 64 KiB of bytes or rows, 16 Ki words: a multiple of 8 rows, so bitmaps split on byte boundaries
  const int64_t unit = kind == Seg::kOffsets ? 4 : 1, chunk = (int64_t(64) << 10) / unit;
  for (int64_t k = 0; k < n; k += chunk)
    segs.push_back({src ? src + (kind == Seg::kBitsToBytes ? k / 8 : k * unit) : nullptr, dst + (kind == Seg::kBytesToBits ? k / 8 : k * unit),
                    std::min(chunk, n - k), kind, arg});
}

void launch_segments(const CtxPtr& ctx, const std::vector<Seg>& segs, const char* stage) {
  BufferPtr d_segs = alloc(ctx, segs.size() * sizeof(Seg));
  ctx->h2d_bytes.fetch_add(int64_t(segs.size() * sizeof(Seg)), std::memory_order_relaxed);
  if (!segs.empty()) FG_CUDA(cudaMemcpyAsync(d_segs->ptr, segs.data(), segs.size() * sizeof(Seg), cudaMemcpyHostToDevice, ctx->stream));
  {
    LaunchTimer lt(ctx, stage);
    const int grid = int(std::min<size_t>(std::max<size_t>(segs.size(), 1), size_t(ctx->sm_count) * 16));
    ipc_segment_kernel<<<grid, 256, 0, ctx->stream>>>(d_segs->as<Seg>(), int(segs.size()));
  }
  count_launch(ctx);
  FG_CUDA(cudaGetLastError());
  // the segment list is pageable host memory the copy above has already consumed; d_segs is released in stream order
}

PackedFrames pack_frames(const CtxPtr& ctx, const Table& t, const std::vector<std::pair<int64_t, int64_t>>& row_ranges) {
  const size_t n_cols = t.cols.size(), nf = row_ranges.size();

  // ---- layout: Utf8 extents and null counts of every non-empty (frame, column), one read-back ----
  std::vector<LayoutItem> items;
  std::vector<int32_t> item_of(nf * n_cols, -1);
  for (size_t f = 0; f < nf; ++f) {
    if (row_ranges[f].second == 0) continue;  // an empty frame reads nothing on the device
    for (size_t i = 0; i < n_cols; ++i) {
      const Column& c = t.cols[i];
      const bool utf8 = c.dtype == FLOCKGPU_UTF8, some_null = !c.all_null && c.validity;
      if (!utf8 && !some_null) continue;
      item_of[f * n_cols + i] = int32_t(items.size());
      items.push_back({utf8 ? c.offs() : nullptr, some_null ? c.valid() : nullptr, row_ranges[f].first, row_ranges[f].second});
    }
  }
  std::vector<int64_t> lay(items.size() * 3);
  if (!items.empty()) {
    BufferPtr d_items = alloc(ctx, items.size() * sizeof(LayoutItem));
    BufferPtr d_lay = alloc(ctx, lay.size() * 8);
    FG_CUDA(cudaMemcpyAsync(d_items->ptr, items.data(), items.size() * sizeof(LayoutItem), cudaMemcpyHostToDevice, ctx->stream));
    {
      LaunchTimer lt(ctx, "payload_layout_kernel");
      const int grid = int(std::min<size_t>(items.size(), size_t(ctx->sm_count) * 16));
      payload_layout_kernel<<<grid, 256, 0, ctx->stream>>>(d_items->as<LayoutItem>(), int(items.size()), d_lay->as<int64_t>());
    }
    count_launch(ctx);
    FG_CUDA(cudaGetLastError());
    FG_CUDA(cudaMemcpyAsync(lay.data(), d_lay->ptr, lay.size() * 8, cudaMemcpyDeviceToHost, ctx->stream));
    FG_CUDA(cudaStreamSynchronize(ctx->stream));
  }

  // ---- host: body layouts, headers, segments (their destinations are offsets until the bodies are allocated) ----
  PackedFrames P;
  P.body_at.resize(nf);
  P.body_len.resize(nf);
  P.headers.resize(nf);
  std::vector<Seg> segs;
  int64_t packed = 0;
  for (size_t f = 0; f < nf; ++f) {
    const int64_t rb = row_ranges[f].first, rc = row_ranges[f].second;
    std::vector<std::pair<int64_t, int64_t>> nodes, buffers;
    int64_t len = 0;
    auto dst = [&] { return reinterpret_cast<uint8_t*>(packed + len); };
    for (size_t i = 0; i < n_cols; ++i) {
      const Column& c = t.cols[i];
      const int it = item_of[f * n_cols + i];
      const int64_t* L = it >= 0 ? &lay[size_t(it) * 3] : nullptr;  // first offset, last offset, null count
      const bool all_null = c.all_null && rc > 0, some_null = !c.all_null && c.validity && rc > 0;
      nodes.emplace_back(rc, all_null ? rc : some_null ? L[2] : 0);
      const int64_t vbytes = (all_null || some_null) ? (rc + 7) / 8 : 0;  // validity: empty when there is no NULL
      buffers.emplace_back(len, vbytes);
      if (some_null) add_segs(segs, Seg::kBytesToBits, c.valid() + rb, dst(), rc);
      len += pad8(vbytes);
      if (c.dtype == FLOCKGPU_UTF8) {
        // offsets rebased to 0 (Arrow IPC does not require it, arrow-rs and pyarrow both write them rebased, and
        // readers of older versions expect it)
        const int32_t first = L ? int32_t(L[0]) : 0, last = L ? int32_t(L[1]) : 0;
        buffers.emplace_back(len, (rc + 1) * 4);
        if (rc > 0) add_segs(segs, Seg::kOffsets, reinterpret_cast<const uint8_t*>(c.offs() + rb), dst(), rc + 1, -first);
        len += pad8((rc + 1) * 4);
        buffers.emplace_back(len, int64_t(last - first));
        add_segs(segs, Seg::kCopy, static_cast<const uint8_t*>(c.values()) + first, dst(), last - first);
        len += pad8(int64_t(last - first));
      } else {
        buffers.emplace_back(len, rc * c.width());
        if (!c.all_null) add_segs(segs, Seg::kCopy, static_cast<const uint8_t*>(c.values()) + rb * c.width(), dst(), rc * c.width());
        len += pad8(rc * c.width());
      }
    }
    P.body_at[f] = packed;
    P.body_len[f] = len;
    P.headers[f] = build_record_batch_message(rc, nodes, buffers, len);
    packed += align16(len);
  }
  P.bodies = alloc(ctx, size_t(std::max<int64_t>(packed, 16)));
  uint8_t* bodies = P.bodies->as<uint8_t>();
  for (Seg& s : segs) s.dst = bodies + reinterpret_cast<int64_t>(s.dst);
  FG_CUDA(cudaMemsetAsync(bodies, 0, size_t(packed), ctx->stream));
  launch_segments(ctx, segs, "payload_pack_kernel");
  return P;
}

}  // namespace fg

using namespace fg;

extern "C" {

int flockgpu_table_import_ipc(flockgpu_ctx* ctx, const struct ArrowSchema* schema, const uint8_t* const* headers, const int64_t* header_lens,
                              const uint8_t* const* bodies, const int64_t* body_lens, int32_t n_frames, const int32_t* projection, int32_t n_projection,
                              flockgpu_table** out) {
  return guarded([&] {
    FG_CHECK(out, FLOCKGPU_ERR_INVALID, "table_import_ipc: null out pointer");
    // the frames are checked before the context is even looked at: a malformed payload is an INVALID error whatever
    // the state of the device (and CPU-only CI can exercise the checks: tests/test_host.py)
    const IpcFrames view = view_ipc_frames(schema, headers, header_lens, bodies, body_lens, n_frames);
    auto c = core_of(ctx);
    std::lock_guard<std::recursive_mutex> g(c->mu);
    FG_CUDA(cudaSetDevice(c->device));
    *out = wrap_table(import_batches(c, schema, view.tops.data(), n_frames, projection, n_projection, c->feed_zero_copy));
  });
}

int flockgpu_table_export_ipc(flockgpu_ctx* ctx, const flockgpu_table* table, int64_t row_begin, int64_t row_count, uint8_t** out_header, int64_t* out_header_len,
                              uint8_t** out_body, int64_t* out_body_len) {
  return guarded([&] {
    auto c = core_of(ctx);
    FG_CHECK(table && table->table && out_header && out_header_len && out_body && out_body_len, FLOCKGPU_ERR_INVALID, "table_export_ipc: null argument");
    std::lock_guard<std::recursive_mutex> g(c->mu);
    FG_CUDA(cudaSetDevice(c->device));
    const Table& t = *table->table;
    t.dense();
    if (row_count < 0) row_count = t.num_rows - row_begin;
    FG_CHECK(row_begin >= 0 && row_begin + row_count <= t.num_rows, FLOCKGPU_ERR_INVALID, "table_export_ipc: rows [%lld, %lld) outside table of %lld rows",
             (long long)row_begin, (long long)(row_begin + row_count), (long long)t.num_rows);
    const PackedFrames P = pack_frames(c, t, {{row_begin, row_count}});
    const int64_t body_len = P.body_len[0];
    std::unique_ptr<uint8_t, void (*)(void*)> body(static_cast<uint8_t*>(malloc(size_t(body_len ? body_len : 8))), free);
    FG_CHECK(body, FLOCKGPU_ERR_INVALID, "table_export_ipc: out of host memory (%lld bytes)", (long long)body_len);
    c->d2h_bytes.fetch_add(body_len, std::memory_order_relaxed);
    FG_CUDA(cudaMemcpyAsync(body.get(), P.bodies->ptr, size_t(body_len), cudaMemcpyDeviceToHost, c->stream));
    FG_CUDA(cudaStreamSynchronize(c->stream));
    const std::vector<uint8_t>& header = P.headers[0];
    uint8_t* h = static_cast<uint8_t*>(malloc(header.size()));
    FG_CHECK(h, FLOCKGPU_ERR_INVALID, "table_export_ipc: out of host memory");
    memcpy(h, header.data(), header.size());
    *out_header = h;
    *out_header_len = int64_t(header.size());
    *out_body = body.release();
    *out_body_len = body_len;
  });
}

void flockgpu_ipc_free(uint8_t* block) { free(block); }

}  // extern "C"
