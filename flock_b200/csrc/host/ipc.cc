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
// page-locked bodies included).  Export: the inverse; the body is filled by device-to-host copies straight into its
// final place and the flatbuffer header is written by hand.  Encoding::None only: zstd frames are decoded by zstd.cu
// and encoded by zstd_enc.cu (which reuses build_record_batch_message); lz4 / snappy / zlib are not restated
// (DESIGN.md section 7).
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

}  // namespace

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

// Everything about frame `f` that its header alone decides, against the schema and a body of `body_len` bytes: field
// count, batch and field lengths, null counts, and every buffer extent.  The Utf8 offsets live in the body; the caller
// checks them (check_utf8_extent).
void check_frame_layout(const ArrowSchema* schema, int f, const FrameLayout& L, int64_t body_len) {
  const int64_t n_fields = schema->n_children;
  FG_CHECK(int64_t(L.nodes.size()) == n_fields, FLOCKGPU_ERR_INVALID, "table_import_ipc: frame %d describes %zu fields, the schema has %lld", f, L.nodes.size(),
           (long long)n_fields);
  FG_CHECK(L.length >= 0 && L.length < (int64_t(1) << 31), FLOCKGPU_ERR_INVALID, "table_import_ipc: frame %d: batch length %lld", f, (long long)L.length);
  size_t next = 0;
  for (int64_t c = 0; c < n_fields; ++c) {
    const char* fmt = schema->children[c]->format;
    const int dt = dtype_from_format(fmt);
    FG_CHECK(dt >= 0, FLOCKGPU_ERR_UNSUPPORTED, "table_import_ipc: column \"%s\" has unsupported Arrow format \"%s\"", schema->children[c]->name, fmt ? fmt : "");
    const size_t want = dt == FLOCKGPU_UTF8 ? 3 : 2;
    FG_CHECK(next + want <= L.buffers.size(), FLOCKGPU_ERR_INVALID, "table_import_ipc: frame %d lists too few buffers", f);
    const int64_t length = L.nodes[size_t(c)].first, null_count = L.nodes[size_t(c)].second;
    FG_CHECK(length == L.length, FLOCKGPU_ERR_INVALID, "table_import_ipc: frame %d: field length %lld differs from the batch length %lld", f,
             (long long)length, (long long)L.length);
    FG_CHECK(null_count >= 0 && null_count <= length, FLOCKGPU_ERR_INVALID, "table_import_ipc: frame %d: null count %lld of %lld rows", f,
             (long long)null_count, (long long)length);
    for (size_t b = 0; b < want; ++b) {
      const auto& ext = L.buffers[next + b];
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
    next += want;
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
  IpcFrames out;
  for (int f = 0; f < n_frames; ++f) {
    FG_CHECK(body_lens[f] >= 0 && (body_lens[f] == 0 || bodies[f]), FLOCKGPU_ERR_INVALID, "table_import_ipc: frame %d has no body", f);
    const FrameLayout L = parse_record_batch_message(headers[f], header_lens[f]);
    check_frame_layout(schema, f, L, body_lens[f]);
    auto fr = std::make_unique<IpcFrame>();
    fr->kids.resize(size_t(n_fields));
    fr->bufs.resize(size_t(n_fields));
    size_t next = 0;
    for (int64_t c = 0; c < n_fields; ++c) {
      const int dt = dtype_from_format(schema->children[c]->format);
      const size_t want = dt == FLOCKGPU_UTF8 ? 3 : 2;
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
      if (dt == FLOCKGPU_UTF8 && a.length > 0) {
        const auto& offs = L.buffers[next + 1];
        int32_t first, last;
        memcpy(&first, bodies[f] + offs.first, 4);
        memcpy(&last, bodies[f] + offs.first + a.length * 4, 4);
        check_utf8_extent(f, schema->children[c]->name, first, last, L.buffers[next + 2].second);
      }
      next += want;
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

// One frame for rows [row_begin, row_begin + row_count) of `t`.  The two blocks are malloc'ed (flockgpu_ipc_free).
void export_ipc_frame(const CtxPtr& ctx, const Table& t, int64_t row_begin, int64_t row_count, uint8_t** out_header, int64_t* out_header_len, uint8_t** out_body,
                      int64_t* out_body_len) {
  t.dense();
  if (row_count < 0) row_count = t.num_rows - row_begin;
  FG_CHECK(row_begin >= 0 && row_begin + row_count <= t.num_rows, FLOCKGPU_ERR_INVALID, "table_export_ipc: rows [%lld, %lld) outside table of %lld rows",
           (long long)row_begin, (long long)(row_begin + row_count), (long long)t.num_rows);
  // the Utf8 extents of the row range decide the body layout: one small read-back
  std::vector<int32_t> first(t.cols.size(), 0), last(t.cols.size(), 0);
  {
    std::vector<int32_t> h(t.cols.size() * 2, 0);
    bool any = false;
    for (size_t i = 0; i < t.cols.size(); ++i)
      if (t.cols[i].dtype == FLOCKGPU_UTF8 && row_count > 0) {
        FG_CUDA(cudaMemcpyAsync(&h[2 * i], t.cols[i].offs() + row_begin, 4, cudaMemcpyDeviceToHost, ctx->stream));
        FG_CUDA(cudaMemcpyAsync(&h[2 * i + 1], t.cols[i].offs() + row_begin + row_count, 4, cudaMemcpyDeviceToHost, ctx->stream));
        any = true;
      }
    if (any) FG_CUDA(cudaStreamSynchronize(ctx->stream));
    for (size_t i = 0; i < t.cols.size(); ++i) {
      first[i] = h[2 * i];
      last[i] = h[2 * i + 1];
    }
  }
  auto pad8 = [](int64_t x) { return (x + 7) & ~int64_t(7); };
  std::vector<std::pair<int64_t, int64_t>> nodes, buffers;
  int64_t body_len = 0;
  for (size_t i = 0; i < t.cols.size(); ++i) {
    const Column& c = t.cols[i];
    const bool all_null = c.all_null && row_count > 0;
    const bool some_null = !all_null && c.validity && row_count > 0;
    nodes.emplace_back(row_count, all_null ? row_count : 0);  // (null_count of `some_null` columns is filled in once the bytes are here)
    const int64_t vbytes = (all_null || some_null) ? (row_count + 7) / 8 : 0;  // validity: empty when there is no NULL
    buffers.emplace_back(body_len, vbytes);
    body_len += pad8(vbytes);
    if (c.dtype == FLOCKGPU_UTF8) {
      buffers.emplace_back(body_len, (row_count + 1) * 4);
      body_len += pad8((row_count + 1) * 4);
      buffers.emplace_back(body_len, int64_t(last[i] - first[i]));
      body_len += pad8(int64_t(last[i] - first[i]));
    } else {
      buffers.emplace_back(body_len, row_count * c.width());
      body_len += pad8(row_count * c.width());
    }
  }
  uint8_t* body = static_cast<uint8_t*>(calloc(size_t(body_len ? body_len : 8), 1));
  FG_CHECK(body, FLOCKGPU_ERR_INVALID, "table_export_ipc: out of host memory (%lld bytes)", (long long)body_len);
  std::unique_ptr<uint8_t, void (*)(void*)> guard(body, free);
  std::vector<std::vector<uint8_t>> vbytes_host(t.cols.size());
  size_t b = 0;
  for (size_t i = 0; i < t.cols.size(); ++i) {
    const Column& c = t.cols[i];
    if (c.validity && !c.all_null && row_count > 0) {  // byte per row now, packed into the body's bitmap after the sync
      vbytes_host[i].resize(size_t(row_count));
      ctx->d2h_bytes.fetch_add(row_count, std::memory_order_relaxed);
      FG_CUDA(cudaMemcpyAsync(vbytes_host[i].data(), c.valid() + row_begin, size_t(row_count), cudaMemcpyDeviceToHost, ctx->stream));
    }
    ++b;  // validity: zero (all NULL), absent, or packed below
    if (c.dtype == FLOCKGPU_UTF8) {
      int32_t* off = reinterpret_cast<int32_t*>(body + buffers[b].first);
      if (row_count > 0) {
        ctx->d2h_bytes.fetch_add(buffers[b].second + buffers[b + 1].second, std::memory_order_relaxed);
        FG_CUDA(cudaMemcpyAsync(off, c.offs() + row_begin, size_t(buffers[b].second), cudaMemcpyDeviceToHost, ctx->stream));
        if (buffers[b + 1].second)
          FG_CUDA(cudaMemcpyAsync(body + buffers[b + 1].first, static_cast<const char*>(c.values()) + first[i], size_t(buffers[b + 1].second),
                                  cudaMemcpyDeviceToHost, ctx->stream));
      }
      b += 2;
    } else {
      if (row_count > 0 && !c.all_null) {
        ctx->d2h_bytes.fetch_add(buffers[b].second, std::memory_order_relaxed);
        FG_CUDA(cudaMemcpyAsync(body + buffers[b].first, static_cast<const char*>(c.values()) + row_begin * c.width(), size_t(buffers[b].second),
                                cudaMemcpyDeviceToHost, ctx->stream));
      }
      b += 1;
    }
  }
  FG_CUDA(cudaStreamSynchronize(ctx->stream));
  b = 0;
  for (size_t i = 0; i < t.cols.size(); ++i) {
    if (!vbytes_host[i].empty()) {
      uint8_t* bits = body + buffers[b].first;
      int64_t nulls = 0;
      for (int64_t r = 0; r < row_count; ++r) {
        if (vbytes_host[i][size_t(r)]) bits[r >> 3] |= uint8_t(1u << (r & 7));
        else ++nulls;
      }
      nodes[i].second = nulls;
    }
    b += t.cols[i].dtype == FLOCKGPU_UTF8 ? 3 : 2;
  }
  // Utf8 offsets of a row range start at offsets[row_begin]: rebase them to 0 (Arrow IPC does not require it, arrow-rs
  // and pyarrow both write them rebased, and readers of older versions expect it)
  b = 0;
  for (size_t i = 0; i < t.cols.size(); ++i) {
    const Column& c = t.cols[i];
    if (c.dtype == FLOCKGPU_UTF8) {
      if (first[i] != 0 && row_count > 0) {
        int32_t* off = reinterpret_cast<int32_t*>(body + buffers[b + 1].first);
        for (int64_t r = 0; r <= row_count; ++r) off[r] -= first[i];
      }
      b += 3;
    } else {
      b += 2;
    }
  }
  std::vector<uint8_t> header = build_record_batch_message(row_count, nodes, buffers, body_len);
  uint8_t* h = static_cast<uint8_t*>(malloc(header.size()));
  FG_CHECK(h, FLOCKGPU_ERR_INVALID, "table_export_ipc: out of host memory");
  memcpy(h, header.data(), header.size());
  *out_header = h;
  *out_header_len = int64_t(header.size());
  *out_body = guard.release();
  *out_body_len = body_len;
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
    export_ipc_frame(c, *table->table, row_begin, row_count, out_header, out_header_len, out_body, out_body_len);
  });
}

void flockgpu_ipc_free(uint8_t* block) { free(block); }

}  // extern "C"
