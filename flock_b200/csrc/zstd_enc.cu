// zstd_enc.cu -- device tables -> payload frames (Flock's DataFrames), compressed with zstd on the GPU.
//
// In the reference `to_payload` (flock/src/transmute.rs:178-221) turns every result batch into a DataFrame and runs
// `zstd::block::compress(.., 3)` over its header and body on the CPU (flock/src/encoding.rs:72-74).  Here the bodies
// are laid out, packed and compressed in HBM; only the compressed bytes cross the link.  Frame f holds rows
// [f * rows_per_frame, min((f + 1) * rows_per_frame, rows)); its uncompressed header and body are exactly what
// flockgpu_table_export_ipc returns for that row range, because both come from pack_frames (host/ipc.cc):
//
//   device  payload_layout_kernel  the Utf8 extents and null counts of every (frame, column): one small read-back.
//   host    body layouts and flatbuffer headers.
//   device  ipc_segment_kernel     one launch over a segment list writes every frame's IPC body in HBM (profiled as
//                                  payload_pack_kernel).
//   --- this file ---
//   host    headers compressed with the shared encoder functions (zstd_enc.h), as the import decodes them on the host.
//   device  zstd_compress_kernel   one CTA per 128 KiB block of every body, every block independent (zstd_enc.h).
//           zstd_place_kernel      a scan over the compressed block sizes: each block's place behind its frame header.
//           zstd_gather_kernel     the blocks' pieces into one contiguous buffer.
//   copy    one device-to-host copy of the compressed bytes into page-locked memory.
// A fixed number of launches and host waits per call, whatever the number of frames.
#include <algorithm>
#include <cstring>
#include <memory>
#include <vector>

#include "internal.h"
#include "zstd_enc.h"

namespace fg {

namespace zs = zstd;

namespace {

// ---- host: the same phases, one lane after the other -------------------------------------------------------------------
struct HostEncoder {
  std::unique_ptr<zs::BlockShared> S{new zs::BlockShared};
  std::vector<uint64_t> seqs = std::vector<uint64_t>(size_t(zs::kLanes) * zs::kLaneSeqs);
  std::vector<uint8_t> lits = std::vector<uint8_t>(zs::kMaxBlock);
  std::vector<uint32_t> lstream = std::vector<uint32_t>(zs::kLitStreamCap / 4);
  std::vector<uint8_t> sstream = std::vector<uint8_t>(zs::kSeqStreamCap);
  std::vector<uint8_t> head = std::vector<uint8_t>(zs::kHeadCap), mid = std::vector<uint8_t>(zs::kMidCap);

  void compress(const uint8_t* src, int64_t n, std::vector<uint8_t>* out) {
    static const uint8_t none = 0;
    if (!src) src = &none;
    const int64_t nb = std::max<int64_t>(1, (n + zs::kMaxBlock - 1) / zs::kMaxBlock);
    for (int64_t b = 0; b < nb; ++b) {
      zs::BlockOut O;
      zs::BlockIo io{src, n, b * zs::kMaxBlock, int32_t(std::min<int64_t>(zs::kMaxBlock, n - b * zs::kMaxBlock)), b == 0, b == nb - 1,
                     seqs.data(), lits.data(), lstream.data(), sstream.data(), head.data(), mid.data(), &O};
      zs::BlockShared& s = *S;
      for (int l = 0; l < zs::kLanes; ++l) zs::phase_match(io, s, l);
      zs::phase_scan(io, s);
      for (int l = 0; l < zs::kLanes; ++l) zs::phase_literals(io, s, l);
      for (int l = 0; l < zs::kLanes; ++l) zs::phase_rank(s, l);
      zs::phase_lit_plan(io, s);
      for (int l = 0; l < zs::kLanes; ++l) zs::phase_huf_bits(io, s, l);
      zs::phase_huf_sizes(s);
      if (s.lit_mode == 2) std::fill(lstream.begin(), lstream.begin() + (s.lit_stream_bytes + 3) / 4, 0u);
      for (int l = 0; l < zs::kLanes; ++l) zs::phase_huf_write(io, s, l);
      zs::phase_finish(io, s);
      for (int i = 0; i < 4; ++i)
        if (O.n[i]) out->insert(out->end(), O.p[i], O.p[i] + O.n[i]);
    }
  }
};

}  // namespace

void zstd_compress_host(const uint8_t* src, int64_t n, std::vector<uint8_t>* out) {
  HostEncoder enc;
  enc.compress(src, n, out);
}

namespace {

// ---- zstd_compress_kernel: one CTA per block ------------------------------------------------------------------------------
struct EncBlock {
  int64_t body;  // the body's first byte in the packed bodies
  int64_t body_len, off;
  int32_t len, first, last, pad;
};

// per-block scratch, in bytes (each piece 16-byte aligned)
constexpr size_t kSeqBytes = size_t(zs::kLanes) * zs::kLaneSeqs * 8;
constexpr size_t kScratch = kSeqBytes + zs::kMaxBlock + zs::kLitStreamCap + zs::kSeqStreamCap + zs::kHeadCap + zs::kMidCap;

__device__ __forceinline__ zs::BlockIo block_io(const uint8_t* bodies, const EncBlock& B, uint8_t* scratch, zs::BlockOut* out) {
  uint8_t* s = scratch;
  zs::BlockIo io;
  io.body = bodies + B.body;
  io.body_len = B.body_len;
  io.off = B.off;
  io.len = B.len;
  io.first = B.first;
  io.last = B.last;
  io.seqs = reinterpret_cast<uint64_t*>(s);
  s += kSeqBytes;
  io.lits = s;
  s += zs::kMaxBlock;
  io.lstream = reinterpret_cast<uint32_t*>(s);
  s += zs::kLitStreamCap;
  io.sstream = s;
  s += zs::kSeqStreamCap;
  io.head = s;
  s += zs::kHeadCap;
  io.mid = s;
  io.out = out;
  return io;
}

__global__ void __launch_bounds__(zs::kLanes, 1) zstd_compress_kernel(const uint8_t* __restrict__ bodies, const EncBlock* __restrict__ blocks, uint8_t* scratch,
                                                                  zs::BlockOut* outs) {
  extern __shared__ __align__(16) uint8_t smem[];
  zs::BlockShared& S = *reinterpret_cast<zs::BlockShared*>(smem);
  const int b = blockIdx.x, l = threadIdx.x;
  const EncBlock B = blocks[b];
  const zs::BlockIo io = block_io(bodies, B, scratch + size_t(b) * kScratch, outs + b);
  zs::phase_match(io, S, l);
  __syncthreads();
  if (l == 0) zs::phase_scan(io, S);
  __syncthreads();
  zs::phase_literals(io, S, l);
  __syncthreads();
  zs::phase_rank(S, l);
  __syncthreads();
  if (l == 0) zs::phase_lit_plan(io, S);
  __syncthreads();
  zs::phase_huf_bits(io, S, l);
  __syncthreads();
  if (l == 0) zs::phase_huf_sizes(S);
  __syncthreads();
  if (S.lit_mode == 2) {
    for (int k = l; k < (S.lit_stream_bytes + 3) / 4; k += zs::kLanes) io.lstream[k] = 0;
    __syncthreads();
    zs::phase_huf_write(io, S, l);
    __syncthreads();
  }
  if (l == 0) zs::phase_finish(io, S);
}

// ---- zstd_place_kernel: one CTA, exclusive scan over the block sizes ------------------------------------------------------
constexpr int kPlaceThreads = 1024;

__global__ void __launch_bounds__(kPlaceThreads) zstd_place_kernel(const zs::BlockOut* __restrict__ outs, const int32_t* __restrict__ frame_of, int n_blocks,
                                                                   int64_t* __restrict__ at, int64_t* __restrict__ frame_at, int n_frames) {
  __shared__ int64_t part[kPlaceThreads];
  const int t = threadIdx.x;
  const int per = (n_blocks + kPlaceThreads - 1) / kPlaceThreads;
  const int b0 = min(n_blocks, t * per), b1 = min(n_blocks, b0 + per);
  int64_t sum = 0;
  for (int b = b0; b < b1; ++b) sum += int64_t(outs[b].n[0]) + outs[b].n[1] + outs[b].n[2] + outs[b].n[3];
  part[t] = sum;
  __syncthreads();
  for (int d = 1; d < kPlaceThreads; d <<= 1) {
    const int64_t v = t >= d ? part[t - d] : 0;
    __syncthreads();
    part[t] += v;
    __syncthreads();
  }
  int64_t pos = part[t] - sum;
  for (int b = b0; b < b1; ++b) {
    at[b] = pos;
    if (b == 0 || frame_of[b] != frame_of[b - 1]) frame_at[frame_of[b]] = pos;
    pos += int64_t(outs[b].n[0]) + outs[b].n[1] + outs[b].n[2] + outs[b].n[3];
  }
  if (t == kPlaceThreads - 1) frame_at[n_frames] = part[t];
}

// ---- zstd_gather_kernel: one CTA per block --------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) zstd_gather_kernel(const zs::BlockOut* __restrict__ outs, const int64_t* __restrict__ at, int n_blocks, uint8_t* __restrict__ dst) {
  for (int b = blockIdx.x; b < n_blocks; b += gridDim.x) {
    const zs::BlockOut O = outs[b];
    uint8_t* d = dst + at[b];
    for (int i = 0; i < 4; ++i) {
      const uint8_t* s = O.p[i];
      for (int k = threadIdx.x; k < O.n[i]; k += blockDim.x) d[k] = s[k];
      d += O.n[i];
    }
  }
}

int64_t align16(int64_t x) { return (x + 15) & ~int64_t(15); }

}  // namespace

}  // namespace fg

// The frames of one export: headers on the host, bodies in one page-locked block.
struct flockgpu_payload {
  std::vector<uint8_t> headers;
  void* pinned = nullptr;
  struct Frame {
    int64_t header_at, header_len, body_at, body_len;
  };
  std::vector<Frame> frames;
  ~flockgpu_payload() {
    if (pinned) cudaFreeHost(pinned);
  }
};

namespace fg {

namespace {

constexpr int64_t kMaxZstdBody = 10485760;  // what Flock's receiver decompresses into (flock/src/encoding.rs:92)

void export_payload(const CtxPtr& ctx, const Table& t, int32_t encoding, int64_t rows_per_frame, flockgpu_payload* P) {
  t.dense();
  const int64_t rows = t.num_rows;
  const int n_frames = int(rows == 0 ? 0 : (rows + rows_per_frame - 1) / rows_per_frame);
  FG_CHECK(rows / rows_per_frame < (int64_t(1) << 30), FLOCKGPU_ERR_INVALID, "table_export_payload: %lld frames", (long long)(rows / rows_per_frame));
  if (n_frames == 0) return;
  std::vector<std::pair<int64_t, int64_t>> ranges;
  for (int f = 0; f < n_frames; ++f) ranges.emplace_back(int64_t(f) * rows_per_frame, std::min(rows_per_frame, rows - int64_t(f) * rows_per_frame));
  const PackedFrames B = pack_frames(ctx, t, ranges);
  const std::vector<int64_t>& body_at = B.body_at;
  const std::vector<int64_t>& body_len = B.body_len;
  const uint8_t* bodies = B.bodies->as<uint8_t>();
  const int64_t packed = body_at.back() + align16(body_len.back());
  for (int f = 0; f < n_frames && encoding == FLOCKGPU_ENCODING_ZSTD; ++f) {
    const int64_t rb = ranges[size_t(f)].first, rc = ranges[size_t(f)].second, len = body_len[size_t(f)];
    FG_CHECK(len <= kMaxZstdBody, FLOCKGPU_ERR_INVALID,
             "table_export_payload: frame %d (rows %lld..%lld) has a %lld-byte body; a zstd frame's body must stay within %lld bytes (pick fewer rows per frame)", f,
             (long long)rb, (long long)(rb + rc), (long long)len, (long long)kMaxZstdBody);
  }

  // headers: the flatbuffers themselves, or compressed on the host
  P->frames.resize(size_t(n_frames));
  {
    HostEncoder enc;
    for (int f = 0; f < n_frames; ++f) {
      const std::vector<uint8_t>& h = B.headers[size_t(f)];
      P->frames[size_t(f)].header_at = int64_t(P->headers.size());
      if (encoding == FLOCKGPU_ENCODING_ZSTD) enc.compress(h.data(), int64_t(h.size()), &P->headers);
      else P->headers.insert(P->headers.end(), h.begin(), h.end());
      P->frames[size_t(f)].header_len = int64_t(P->headers.size()) - P->frames[size_t(f)].header_at;
    }
  }

  if (encoding == FLOCKGPU_ENCODING_NONE) {
    FG_CUDA(cudaMallocHost(&P->pinned, size_t(std::max<int64_t>(packed, 16))));
    ctx->d2h_bytes.fetch_add(packed, std::memory_order_relaxed);
    FG_CUDA(cudaMemcpyAsync(P->pinned, bodies, size_t(packed), cudaMemcpyDeviceToHost, ctx->stream));
    FG_CUDA(cudaStreamSynchronize(ctx->stream));
    for (int f = 0; f < n_frames; ++f) {
      P->frames[size_t(f)].body_at = body_at[size_t(f)];
      P->frames[size_t(f)].body_len = body_len[size_t(f)];
    }
    return;
  }

  // ---- compression: every block of every body ----
  std::vector<EncBlock> blocks;
  std::vector<int32_t> frame_of;
  for (int f = 0; f < n_frames; ++f) {
    const int64_t len = body_len[size_t(f)];
    const int64_t nb = std::max<int64_t>(1, (len + zs::kMaxBlock - 1) / zs::kMaxBlock);
    for (int64_t b = 0; b < nb; ++b) {
      blocks.push_back({body_at[size_t(f)], len, b * zs::kMaxBlock, int32_t(std::min<int64_t>(zs::kMaxBlock, len - b * zs::kMaxBlock)), b == 0, b == nb - 1, 0});
      frame_of.push_back(f);
    }
  }
  const int n_blocks = int(blocks.size());
  const size_t o_frame_of = align16(int64_t(blocks.size() * sizeof(EncBlock)));
  std::vector<uint8_t> desc(o_frame_of + frame_of.size() * 4);
  memcpy(desc.data(), blocks.data(), blocks.size() * sizeof(EncBlock));
  memcpy(desc.data() + o_frame_of, frame_of.data(), frame_of.size() * 4);
  BufferPtr d_desc = alloc(ctx, desc.size());
  ctx->h2d_bytes.fetch_add(int64_t(desc.size()), std::memory_order_relaxed);
  FG_CUDA(cudaMemcpyAsync(d_desc->ptr, desc.data(), desc.size(), cudaMemcpyHostToDevice, ctx->stream));
  BufferPtr d_scratch = alloc(ctx, size_t(n_blocks) * kScratch);
  BufferPtr d_outs = alloc(ctx, size_t(n_blocks) * sizeof(zs::BlockOut));
  BufferPtr d_at = alloc(ctx, size_t(n_blocks + n_frames + 1) * 8);
  int64_t* d_block_at = d_at->as<int64_t>();
  int64_t* d_frame_at = d_block_at + n_blocks;
  FG_CUDA(cudaFuncSetAttribute(zstd_compress_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(sizeof(zs::BlockShared))));
  {
    LaunchTimer lt(ctx, "zstd_compress_kernel");
    zstd_compress_kernel<<<n_blocks, zs::kLanes, sizeof(zs::BlockShared), ctx->stream>>>(bodies, reinterpret_cast<const EncBlock*>(d_desc->ptr), d_scratch->as<uint8_t>(),
                                                                                       d_outs->as<zs::BlockOut>());
  }
  count_launch(ctx);
  FG_CUDA(cudaGetLastError());
  {
    LaunchTimer lt(ctx, "zstd_place_kernel");
    zstd_place_kernel<<<1, kPlaceThreads, 0, ctx->stream>>>(d_outs->as<zs::BlockOut>(), reinterpret_cast<const int32_t*>(d_desc->as<uint8_t>() + o_frame_of), n_blocks,
                                                           d_block_at, d_frame_at, n_frames);
  }
  count_launch(ctx);
  FG_CUDA(cudaGetLastError());
  int64_t worst = 0;
  for (int f = 0; f < n_frames; ++f) worst += zs::kFrameHeaderMax + body_len[size_t(f)] + 3 * ((body_len[size_t(f)] + zs::kMaxBlock - 1) / zs::kMaxBlock + 1);
  BufferPtr d_out = alloc(ctx, size_t(worst));
  {
    LaunchTimer lt(ctx, "zstd_gather_kernel");
    const int grid = std::min(n_blocks, ctx->sm_count * 16);
    zstd_gather_kernel<<<grid, 256, 0, ctx->stream>>>(d_outs->as<zs::BlockOut>(), d_block_at, n_blocks, d_out->as<uint8_t>());
  }
  count_launch(ctx);
  FG_CUDA(cudaGetLastError());
  std::vector<int64_t> frame_at(size_t(n_frames) + 1);
  FG_CUDA(cudaMemcpyAsync(frame_at.data(), d_frame_at, frame_at.size() * 8, cudaMemcpyDeviceToHost, ctx->stream));
  FG_CUDA(cudaStreamSynchronize(ctx->stream));
  const int64_t total = frame_at[size_t(n_frames)];
  FG_CHECK(total >= 0 && total <= worst, FLOCKGPU_ERR_INVALID, "table_export_payload: compressed size %lld outside [0, %lld]", (long long)total, (long long)worst);
  FG_CUDA(cudaMallocHost(&P->pinned, size_t(std::max<int64_t>(total, 16))));
  ctx->d2h_bytes.fetch_add(total + int64_t(frame_at.size() * 8), std::memory_order_relaxed);
  FG_CUDA(cudaMemcpyAsync(P->pinned, d_out->ptr, size_t(total), cudaMemcpyDeviceToHost, ctx->stream));
  FG_CUDA(cudaStreamSynchronize(ctx->stream));
  for (int f = 0; f < n_frames; ++f) {
    P->frames[size_t(f)].body_at = frame_at[size_t(f)];
    P->frames[size_t(f)].body_len = frame_at[size_t(f) + 1] - frame_at[size_t(f)];
  }
}

}  // namespace

}  // namespace fg

using namespace fg;

extern "C" {

int flockgpu_table_export_payload(flockgpu_ctx* ctx, const flockgpu_table* table, int32_t encoding, int64_t rows_per_frame, flockgpu_payload** out) {
  return guarded([&] {
    FG_CHECK(out, FLOCKGPU_ERR_INVALID, "table_export_payload: null out pointer");
    *out = nullptr;
    FG_CHECK(encoding >= FLOCKGPU_ENCODING_SNAPPY && encoding <= FLOCKGPU_ENCODING_NONE, FLOCKGPU_ERR_INVALID, "table_export_payload: unknown encoding %d", int(encoding));
    FG_CHECK(encoding == FLOCKGPU_ENCODING_ZSTD || encoding == FLOCKGPU_ENCODING_NONE, FLOCKGPU_ERR_UNSUPPORTED,
             "table_export_payload: %s payloads are not encoded on the GPU (zstd and none are)",
             encoding == FLOCKGPU_ENCODING_SNAPPY ? "snappy" : encoding == FLOCKGPU_ENCODING_LZ4 ? "lz4" : "zlib");
    FG_CHECK(rows_per_frame > 0, FLOCKGPU_ERR_INVALID, "table_export_payload: rows_per_frame %lld must be positive", (long long)rows_per_frame);
    FG_CHECK(table && table->table, FLOCKGPU_ERR_INVALID, "table_export_payload: null table");
    auto c = core_of(ctx);
    std::unique_ptr<flockgpu_payload> p(new flockgpu_payload);
    std::lock_guard<std::recursive_mutex> g(c->mu);
    FG_CUDA(cudaSetDevice(c->device));
    export_payload(c, deref(table), encoding, rows_per_frame, p.get());
    *out = p.release();
  });
}

int32_t flockgpu_payload_num_frames(const flockgpu_payload* p) { return p ? int32_t(p->frames.size()) : 0; }

int flockgpu_payload_frame(const flockgpu_payload* p, int32_t i, const uint8_t** header, int64_t* header_len, const uint8_t** body, int64_t* body_len) {
  return guarded([&] {
    FG_CHECK(p && header && header_len && body && body_len, FLOCKGPU_ERR_INVALID, "payload_frame: null argument");
    FG_CHECK(i >= 0 && size_t(i) < p->frames.size(), FLOCKGPU_ERR_INVALID, "payload_frame: frame %d of %zu", int(i), p->frames.size());
    const flockgpu_payload::Frame& f = p->frames[size_t(i)];
    *header = p->headers.data() + f.header_at;
    *header_len = f.header_len;
    *body = static_cast<const uint8_t*>(p->pinned) + f.body_at;
    *body_len = f.body_len;
  });
}

void flockgpu_payload_free(flockgpu_payload* p) { delete p; }

}  // extern "C"
