// zstd.cu -- payload frames compressed with zstd (Flock's default Encoding::Zstd) -> device tables.
//
// In the reference every DataFrame { header, body } of a payload is `zstd::block::compress(.., 3)`ed by `to_payload`
// (flock/src/transmute.rs:178-221) and decompressed by libzstd on the CPU in `Payload::to_record_batch`
// (flock/src/runtime/payload.rs:161-192) before anything reads it.  Here the bodies go to HBM compressed and are decoded
// there (RFC 8878; the decoder pieces are zstd_dec.h):
//
//   host      decode each ~100-byte header (zstd_decode_host), read the flatbuffer, check every buffer extent against
//             the header's bodyLength; walk every body's frames and blocks (magic, reserved bits, dictionary ids, block
//             sizes, content sizes) and read each compressed block's literals- and sequences-section headers into the
//             block table, including WHICH block's Huffman / FSE tables a block reuses.  All of this before the
//             context is looked at.  The body bytes themselves are never decoded on the host.
//   copy      the compressed bodies to HBM through the page-locked staging of import_batches (upload_host_pieces).
//   device    zstd_entropy_kernel     one warp per compressed block of every body: Huffman table + 1 or 4 literal
//                                     streams, the LL / OF / ML tables, the sequences -> (ll, ml, offset value).
//             zstd_execute_kernel     one warp per body: blocks in order, repeat offsets resolved in frame order,
//                                     literals and matches copied into the decoded body (DESIGN.md section 3, K11).
//             ipc_segment_kernel      one launch over a segment list: the projected columns from the decoded bodies
//                                     (host/ipc.cc, shared with the export's pack; profiled as payload_assemble_kernel).
//   A fixed number of launches per import, whatever the number of frames.  Errors found on the device are recorded
//   per body (first one wins) and read back with the sync the import performs anyway: FLOCKGPU_ERR_INVALID naming
//   the frame, never a fault.
#include <algorithm>
#include <cstring>
#include <vector>

#include "internal.h"
#include "zstd_dec.h"

namespace fg {

namespace zs = zstd;

namespace {

// ---- host: serial decoder (headers, self test) -----------------------------------------------------------------------------
struct HostTables {
  zs::HufEntry huf[2048];
  int huf_bits = 0;
  bool have_huf = false;
  zs::FseEntry t[3][512];
  int log[3] = {0, 0, 0};
  bool have[3] = {false, false, false};
};

int decode_block_host(const uint8_t* b, int64_t n, HostTables& T, uint32_t* rep, std::vector<uint8_t>& out, size_t frame_start, int64_t max_out,
                      std::vector<uint8_t>& lits, std::vector<zs::Seq>& seqs) {
  zs::LitHeader lh;
  int e = zs::lit_header(b, n, &lh);
  if (e) return e;
  lits.resize(size_t(lh.regen));
  const uint8_t* lp = b + lh.hdr;
  if (lh.type == 0) {
    if (lh.regen) memcpy(lits.data(), lp, size_t(lh.regen));
  } else if (lh.type == 1) {
    memset(lits.data(), lp[0], size_t(lh.regen));
  } else {
    int64_t tree = 0;
    if (lh.type == 2) {
      if ((e = zs::huf_read_table(lp, lh.comp, T.huf, &T.huf_bits, &tree))) return e;
      T.have_huf = true;
    } else if (!T.have_huf) {
      return zs::Z_NO_TABLE;
    }
    if ((e = zs::huf_decode_literals(T.huf, T.huf_bits, lp + tree, lh.comp - tree, lh.streams, lits.data(), lh.regen, 0, 1))) return e;
  }
  const int64_t so = lh.hdr + int64_t(lh.comp);
  zs::SeqHeader sh;
  if ((e = zs::seq_header(b + so, n - so, &sh))) return e;
  const size_t nseq = size_t(sh.nseq);
  if (nseq) {
    const uint8_t* tp = b + so + sh.hdr;
    const int64_t tn = n - so - sh.hdr;
    int64_t end = 0;
    for (int k = 0; k < 3; ++k) {
      if (zs::seq_mode(sh.modes, k) == 3) {
        if (!T.have[k]) return zs::Z_NO_TABLE;
        continue;
      }
      if ((e = zs::seq_tables(tp, tn, sh.modes, k, T.t[k], &T.log[k], &end))) return e;
      T.have[k] = true;
    }
    if ((e = zs::seq_tables(tp, tn, sh.modes, -1, nullptr, nullptr, &end))) return e;
    seqs.resize(nseq);
    if ((e = zs::seq_decode(tp + end, tn - end, T.t[0], T.log[0], T.t[1], T.log[1], T.t[2], T.log[2], sh.nseq, seqs.data()))) return e;
  }
  const size_t block_start = out.size();
  size_t at = 0;
  for (size_t i = 0; i < nseq; ++i) {
    const zs::Seq& q = seqs[i];
    if (q.ll > lits.size() - at) return zs::Z_COUNTS;
    if (int64_t(out.size()) + int64_t(q.ll) + int64_t(q.ml) > max_out) return zs::Z_OVERFLOW;
    out.insert(out.end(), lits.begin() + int64_t(at), lits.begin() + int64_t(at + q.ll));
    at += q.ll;
    uint32_t off;
    if (!zs::resolve_offset(rep, q.of, q.ll, &off) || off > out.size() - frame_start) return zs::Z_BAD_OFFSET;
    const size_t from = out.size() - off;
    for (uint32_t k = 0; k < q.ml; ++k) {
      const uint8_t c = out[from + k];
      out.push_back(c);
    }
  }
  if (int64_t(out.size() + lits.size() - at) > max_out) return zs::Z_OVERFLOW;
  out.insert(out.end(), lits.begin() + int64_t(at), lits.end());
  return out.size() - block_start > size_t(zs::kMaxBlock) ? zs::Z_BAD_BLOCK : zs::Z_OK;
}

}  // namespace

int zstd_decode_host(const uint8_t* src, int64_t n, int64_t max_out, std::vector<uint8_t>* out) {
  if (!src || n <= 0) return zs::Z_TRUNCATED;
  auto T = std::make_unique<HostTables>();
  std::vector<uint8_t> lits;
  std::vector<zs::Seq> seqs;
  int64_t at = 0;
  while (at < n) {
    if (n - at < 4) return zs::Z_TRUNCATED;
    const uint32_t magic = zs::rd_le(src + at, 4);
    if (zs::is_skippable(magic)) {
      if (n - at < 8) return zs::Z_TRUNCATED;
      const int64_t size = zs::rd_le(src + at + 4, 4);
      if (size > n - at - 8) return zs::Z_TRUNCATED;
      at += 8 + size;
      continue;
    }
    zs::FrameHeader fh;
    int e = zs::frame_header(src + at, n - at, &fh);
    if (e) return e;
    at += fh.hdr;
    *T = HostTables();
    uint32_t rep[3] = {1, 4, 8};
    const size_t frame_start = out->size();
    for (;;) {
      zs::BlockHeader bh;
      if ((e = zs::block_header(src + at, n - at, &bh))) return e;
      at += 3;
      if (bh.type == 0 || bh.type == 1) {
        if (int64_t(out->size()) + bh.size > max_out) return zs::Z_OVERFLOW;
        if (bh.type == 0) out->insert(out->end(), src + at, src + at + bh.size);
        else out->insert(out->end(), size_t(bh.size), src[at]);
      } else if ((e = decode_block_host(src + at, bh.size, *T, rep, *out, frame_start, max_out, lits, seqs))) {
        return e;
      }
      at += bh.src;
      if (bh.last) break;
    }
    if (fh.content_size >= 0 && int64_t(out->size() - frame_start) != fh.content_size) return zs::Z_SIZE;
    if (fh.checksum) {  // Content_Checksum: present, not verified (RFC 8878 3.1.1 lets a decoder skip it)
      if (n - at < 4) return zs::Z_TRUNCATED;
      at += 4;
    }
  }
  return zs::Z_OK;
}

namespace {

// ---- the block table -------------------------------------------------------------------------------------------------------
struct ZBlock {
  int64_t src;      // block content in the compressed buffer
  int64_t lit_out;  // regenerated literals in the literal scratch
  int64_t seq_out;  // first sequence in the sequence scratch
  int64_t fcs;      // first block of a zstd frame: its Frame_Content_Size (-1 absent); other blocks: -2
  int32_t size, src_len;
  int32_t body, index;  // payload frame, block number inside its body
  int32_t type;         // 0 raw, 1 RLE, 2 compressed
  int32_t lit_hdr, lit_type, lit_streams, lit_regen, lit_comp;
  int32_t seq_at, nseq, modes;  // seq_at: the table descriptions, relative to `src`
  int32_t huf_src;              // block whose Huffman tree this block's literals use (itself or an earlier one)
  int32_t tab_src[3];           // block whose LL / OF / ML table this block uses
};

struct ZBody {
  int64_t out, len;  // decoded body in the decoded scratch, its bodyLength
  int32_t first_block, n_blocks;
  int32_t ext_first, ext_n;  // Utf8 offset words to read back once decoded
};

constexpr unsigned kFull = 0xFFFFFFFFu;
constexpr int kEntropyWarps = 4;

__device__ __forceinline__ void record(uint32_t* err, int body, int code, int block) {
  atomicCAS(err + body, 0u, uint32_t(code) | (uint32_t(block) << 8));
}

// ---- zstd_entropy_kernel: one warp per compressed block ------------------------------------------------------------------
struct WarpTables {
  zs::HufEntry huf[2048];
  zs::FseEntry t[3][512];
};

__global__ void __launch_bounds__(32 * kEntropyWarps) zstd_entropy_kernel(const uint8_t* __restrict__ src, const ZBlock* __restrict__ blocks, int n_blocks,
                                                                          uint8_t* __restrict__ lits, zs::Seq* __restrict__ seqs, int32_t* __restrict__ regen,
                                                                          uint32_t* __restrict__ err) {
  __shared__ WarpTables tabs[kEntropyWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int b = blockIdx.x * kEntropyWarps + warp;
  if (b >= n_blocks) return;
  const ZBlock B = blocks[b];
  if (B.type != 2) {
    if (lane == 0) regen[b] = B.size;
    return;
  }
  WarpTables& T = tabs[warp];
  const uint8_t* p = src + B.src;
  uint8_t* L = lits + B.lit_out;
  const uint8_t* lp = p + B.lit_hdr;
  int e = zs::Z_OK;
  if (B.lit_type == 0) {
    for (int k = lane; k < B.lit_regen; k += 32) L[k] = lp[k];
  } else if (B.lit_type == 1) {
    const uint8_t v = lp[0];
    for (int k = lane; k < B.lit_regen; k += 32) L[k] = v;
  } else {
    int bits = 0, tree = 0;
    if (lane == 0) {
      const ZBlock& H = blocks[B.huf_src];
      int64_t used = 0;
      e = zs::huf_read_table(src + H.src + H.lit_hdr, H.lit_comp, T.huf, &bits, &used);
      tree = B.huf_src == b ? int(used) : 0;
    }
    e = __shfl_sync(kFull, e, 0);
    bits = __shfl_sync(kFull, bits, 0);
    tree = __shfl_sync(kFull, tree, 0);
    __syncwarp();
    if (!e && lane < B.lit_streams) e = zs::huf_decode_literals(T.huf, bits, lp + tree, B.lit_comp - tree, B.lit_streams, L, B.lit_regen, lane, 32);
  }
  e = __reduce_max_sync(kFull, e);
  unsigned long long sum_ll = 0, sum_ml = 0;
  if (!e && B.nseq > 0) {
    if (lane == 0) {
      const uint8_t* tp = p + B.seq_at;
      const int64_t tn = B.src_len - B.seq_at;
      int64_t end = 0, unused = 0;
      int logs[3] = {0, 0, 0};
      e = zs::seq_tables(tp, tn, uint8_t(B.modes), -1, nullptr, nullptr, &end);
      for (int k = 0; k < 3 && !e; ++k) {
        const ZBlock& R = blocks[B.tab_src[k]];
        e = zs::seq_tables(src + R.src + R.seq_at, R.src_len - R.seq_at, uint8_t(R.modes), k, T.t[k], &logs[k], &unused);
      }
      if (!e) e = zs::seq_decode(tp + end, tn - end, T.t[0], logs[0], T.t[1], logs[1], T.t[2], logs[2], B.nseq, seqs + B.seq_out);
    }
    e = __shfl_sync(kFull, e, 0);
    __syncwarp();
    if (!e) {
      for (int i = lane; i < B.nseq; i += 32) {
        const zs::Seq q = seqs[B.seq_out + i];
        sum_ll += q.ll;
        sum_ml += q.ml;
      }
      for (int d = 16; d; d >>= 1) {
        sum_ll += __shfl_xor_sync(kFull, sum_ll, d);
        sum_ml += __shfl_xor_sync(kFull, sum_ml, d);
      }
      if (sum_ll > (unsigned long long)B.lit_regen) e = zs::Z_COUNTS;
      else if (B.lit_regen + sum_ml > (unsigned long long)zs::kMaxBlock) e = zs::Z_BAD_BLOCK;
    }
  }
  if (lane == 0) {
    if (e) record(err, B.body, e, B.index);
    regen[b] = e ? 0 : int32_t(B.lit_regen + sum_ml);
  }
}

// ---- zstd_execute_kernel: one warp per body ------------------------------------------------------------------------------------
// n bytes from s to d, 8 at a time; d - s >= 8 or the ranges do not overlap (a match copies forward over its own output)
__device__ __forceinline__ void copy_fwd8(uint8_t* d, const uint8_t* s, uint32_t n) {
  uint32_t k = 0;
  for (; k + 8 <= n; k += 8) {
    uint8_t v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = s[k + i];
#pragma unroll
    for (int i = 0; i < 8; ++i) d[k + i] = v[i];
  }
  for (; k < n; ++k) d[k] = s[k];
}

__device__ __forceinline__ void copy_match(uint8_t* d, uint32_t off, uint32_t n) {
  const uint8_t* s = d - off;
  if (off >= 8) {
    copy_fwd8(d, s, n);
  } else {
    for (uint32_t k = 0; k < n; ++k) d[k] = s[k];
  }
}

// The sequences of one compressed block, 32 at a time (one per lane).  `base` = the block's first output byte, `reach` =
// bytes of its zstd frame before it.  The warp resolves the group's repeat offsets in order, writes every literal run,
// then copies matches in rounds: a match goes as soon as every byte it reads is final, i.e. it is the earliest match
// still pending or its source ends before that one's destination.
__device__ int exec_block(const ZBlock& B, const uint8_t* __restrict__ L, const zs::Seq* __restrict__ S, uint8_t* base, int64_t reach, uint32_t* rep, int lane) {
  uint32_t litpos = 0, opos = 0;
  for (int g = 0; g < B.nseq; g += 32) {
    const int cnt = min(32, B.nseq - g);
    const bool valid = lane < cnt;
    zs::Seq q = valid ? S[g + lane] : zs::Seq{0, 0, 0};
    uint32_t off = 0;
    bool bad = false;
    for (int j = 0; j < cnt; ++j) {
      const uint32_t ov = __shfl_sync(kFull, q.of, j), ll = __shfl_sync(kFull, q.ll, j);
      uint32_t o;
      const bool ok = zs::resolve_offset(rep, ov, ll, &o);
      if (lane == j) {
        off = o;
        bad = !ok;
      }
    }
    uint32_t t = q.ll + q.ml, l = q.ll;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t a = __shfl_up_sync(kFull, t, d), c = __shfl_up_sync(kFull, l, d);
      if (lane >= d) {
        t += a;
        l += c;
      }
    }
    const uint32_t tot = __shfl_sync(kFull, t, 31), totl = __shfl_sync(kFull, l, 31);
    const uint32_t dst = opos + t - (q.ll + q.ml), lsrc = litpos + l - q.ll;
    const uint32_t mstart = dst + q.ll;
    bad = bad || (valid && int64_t(off) > reach + int64_t(mstart));
    if (__any_sync(kFull, bad)) return zs::Z_BAD_OFFSET;
    copy_fwd8(base + dst, L + lsrc, q.ll);
    __syncwarp();
    bool done = !valid;
    while (!__all_sync(kFull, done)) {
      const uint32_t w = __reduce_min_sync(kFull, done ? 0xFFFFFFFFu : mstart);
      const bool ready = !done && (mstart == w || int64_t(mstart) - int64_t(off) + int64_t(q.ml) <= int64_t(w));
      if (ready) copy_match(base + mstart, off, q.ml);
      done = done || ready;
      __syncwarp();
    }
    opos += tot;
    litpos += totl;
  }
  for (uint32_t k = lane; k < uint32_t(B.lit_regen) - litpos; k += 32) base[opos + k] = L[litpos + k];
  return zs::Z_OK;
}

__global__ void __launch_bounds__(32) zstd_execute_kernel(const uint8_t* __restrict__ src, const ZBlock* __restrict__ blocks, const ZBody* __restrict__ bodies,
                                                          int n_bodies, const uint8_t* __restrict__ lits, const zs::Seq* __restrict__ seqs,
                                                          const int32_t* __restrict__ regen, uint8_t* dec, uint32_t* err, const int64_t* __restrict__ ext_req,
                                                          int32_t* __restrict__ ext_out) {
  const int f = blockIdx.x, lane = threadIdx.x;
  if (f >= n_bodies) return;
  const ZBody Bd = bodies[f];
  if (*reinterpret_cast<volatile uint32_t*>(err + f)) return;  // an entropy error: nothing of this body is decoded
  uint8_t* out = dec + Bd.out;
  int64_t pos = 0, frame_start = 0, fcs = -1;
  uint32_t rep[3] = {1, 4, 8};
  int code = zs::Z_OK, i = 0;
  for (; i < Bd.n_blocks; ++i) {
    const int b = Bd.first_block + i;
    const ZBlock B = blocks[b];
    if (B.fcs != -2) {  // a new zstd frame: fresh repeat offsets, matches reach no further back than here
      if (fcs >= 0 && pos - frame_start != fcs) {
        code = zs::Z_SIZE;
        break;
      }
      frame_start = pos;
      fcs = B.fcs;
      rep[0] = 1;
      rep[1] = 4;
      rep[2] = 8;
    }
    const int64_t r = regen[b];
    if (r > Bd.len - pos) {
      code = zs::Z_OVERFLOW;
      break;
    }
    if (B.type == 0) {
      for (int64_t k = lane; k < r; k += 32) out[pos + k] = src[B.src + k];
    } else if (B.type == 1) {
      const uint8_t v = src[B.src];
      for (int64_t k = lane; k < r; k += 32) out[pos + k] = v;
    } else if ((code = exec_block(B, lits + B.lit_out, seqs + B.seq_out, out + pos, pos - frame_start, rep, lane))) {
      break;
    }
    pos += r;
    __syncwarp();
  }
  if (!code && fcs >= 0 && pos - frame_start != fcs) code = zs::Z_SIZE;
  if (!code && pos != Bd.len) code = zs::Z_SIZE;
  if (code) {
    if (lane == 0) record(err, f, code, i);
    return;
  }
  __syncwarp();
  for (int k = lane; k < Bd.ext_n; k += 32) {
    const uint8_t* w = dec + ext_req[Bd.ext_first + k];
    ext_out[Bd.ext_first + k] = int32_t(uint32_t(w[0]) | (uint32_t(w[1]) << 8) | (uint32_t(w[2]) << 16) | (uint32_t(w[3]) << 24));
  }
}

// ---- host orchestration ------------------------------------------------------------------------------------------------------
[[noreturn]] void body_error(int f, int code, int64_t at) {
  fail(code == zs::Z_DICTIONARY ? FLOCKGPU_ERR_UNSUPPORTED : FLOCKGPU_ERR_INVALID, "table_import_payload: frame %d: zstd body at byte %lld: %s", f, (long long)at,
       zs::error_name(code));
}

// Walks every zstd frame of one compressed body: frame and block headers, and the section headers of compressed blocks,
// into `blocks`.  Nothing past a header is decoded here.
void walk_body(int f, const uint8_t* p, int64_t n, int64_t body_len, int64_t src_base, std::vector<ZBlock>& blocks, int64_t& lit_total, int64_t& seq_total) {
  if (n <= 0) body_error(f, zs::Z_TRUNCATED, 0);
  const int32_t first = int32_t(blocks.size());
  int64_t at = 0, known = 0;
  bool all_known = true;
  int frames = 0;
  while (at < n) {
    if (n - at < 4) body_error(f, zs::Z_TRUNCATED, at);
    const uint32_t magic = zs::rd_le(p + at, 4);
    if (zs::is_skippable(magic)) {
      if (n - at < 8 || int64_t(zs::rd_le(p + at + 4, 4)) > n - at - 8) body_error(f, zs::Z_TRUNCATED, at);
      at += 8 + int64_t(zs::rd_le(p + at + 4, 4));
      continue;
    }
    zs::FrameHeader fh;
    if (int e = zs::frame_header(p + at, n - at, &fh)) body_error(f, e, at);
    if (fh.content_size >= 0) {
      known += fh.content_size;
      if (known > body_len) body_error(f, zs::Z_SIZE, at);
    } else {
      all_known = false;
    }
    at += fh.hdr;
    int32_t last_huf = -1, last_tab[3] = {-1, -1, -1};
    bool first_block = true;
    for (;;) {
      zs::BlockHeader bh;
      if (int e = zs::block_header(p + at, n - at, &bh)) body_error(f, e, at);
      ZBlock B;
      memset(&B, 0, sizeof B);
      const int32_t self = int32_t(blocks.size());
      B.src = src_base + at + 3;
      B.size = bh.size;
      B.src_len = bh.src;
      B.body = f;
      B.index = self - first;
      B.type = bh.type;
      B.fcs = first_block ? fh.content_size : -2;
      B.huf_src = B.tab_src[0] = B.tab_src[1] = B.tab_src[2] = self;
      first_block = false;
      if (bh.type == 2) {
        const uint8_t* c = p + at + 3;
        zs::LitHeader lh;
        if (int e = zs::lit_header(c, bh.size, &lh)) body_error(f, e, at);
        B.lit_hdr = lh.hdr;
        B.lit_type = lh.type;
        B.lit_streams = lh.streams;
        B.lit_regen = lh.regen;
        B.lit_comp = lh.comp;
        if (lh.type == 2) last_huf = self;
        if (lh.type == 3) {
          if (last_huf < 0) body_error(f, zs::Z_NO_TABLE, at);
          B.huf_src = last_huf;
        }
        const int64_t so = lh.hdr + int64_t(lh.comp);
        zs::SeqHeader sh;
        if (int e = zs::seq_header(c + so, bh.size - so, &sh)) body_error(f, e, at);
        B.nseq = sh.nseq;
        B.modes = sh.modes;
        B.seq_at = int32_t(so + sh.hdr);
        if (sh.nseq > 0)
          for (int k = 0; k < 3; ++k) {
            if (zs::seq_mode(sh.modes, k) == 3) {
              if (last_tab[k] < 0) body_error(f, zs::Z_NO_TABLE, at);
              B.tab_src[k] = last_tab[k];
            } else {
              last_tab[k] = self;
            }
          }
        B.lit_out = lit_total;
        B.seq_out = seq_total;
        lit_total += lh.regen;
        seq_total += sh.nseq;
      }
      blocks.push_back(B);
      at += 3 + bh.src;
      if (bh.last) break;
    }
    if (fh.checksum) {
      if (n - at < 4) body_error(f, zs::Z_TRUNCATED, at);
      at += 4;
    }
    ++frames;
  }
  if (!frames) body_error(f, zs::Z_TRUNCATED, at);
  if (all_known && known != body_len) body_error(f, zs::Z_SIZE, 0);
}

int64_t align16(int64_t x) { return (x + 15) & ~int64_t(15); }

// `off` bytes into a device buffer, as a T*.
template <typename T>
T* at_offset(const BufferPtr& b, size_t off) {
  return reinterpret_cast<T*>(static_cast<char*>(b->ptr) + off);
}

}  // namespace

TablePtr import_payload_zstd(flockgpu_ctx* handle, const ArrowSchema* schema, const uint8_t* const* headers, const int64_t* header_lens,
                             const uint8_t* const* bodies, const int64_t* body_lens, int n_frames, const int* projection, int n_projection) {
  FG_CHECK(schema && schema->format && !strcmp(schema->format, "+s"), FLOCKGPU_ERR_INVALID, "table_import_payload: schema must be a struct (\"+s\")");
  FG_CHECK(n_frames >= 0 && (n_frames == 0 || (headers && header_lens && bodies && body_lens)), FLOCKGPU_ERR_INVALID, "table_import_payload: bad frame list");
  // ---- host: headers, checks, block table (no device, no context) ----
  std::vector<FrameLayout> layouts;
  std::vector<ZBlock> blocks;
  std::vector<ZBody> zb(static_cast<size_t>(n_frames));
  std::vector<int64_t> ext_req;
  std::vector<std::pair<int, int>> ext_col;  // (frame, column) of each pair of ext_req words
  int64_t lit_total = 0, seq_total = 0, src_total = 0, out_total = 0;
  const int64_t n_fields = schema->n_children;
  const std::vector<size_t> first_buf = field_buffers(schema);
  for (int f = 0; f < n_frames; ++f) {
    FG_CHECK(header_lens[f] >= 0 && (header_lens[f] == 0 || headers[f]), FLOCKGPU_ERR_INVALID, "table_import_payload: frame %d has no header", f);
    FG_CHECK(body_lens[f] >= 0 && (body_lens[f] == 0 || bodies[f]), FLOCKGPU_ERR_INVALID, "table_import_payload: frame %d has no body", f);
    std::vector<uint8_t> header;
    const int e = zstd_decode_host(headers[f], header_lens[f], int64_t(1) << 24, &header);
    FG_CHECK(!e, e == zs::Z_DICTIONARY ? FLOCKGPU_ERR_UNSUPPORTED : FLOCKGPU_ERR_INVALID, "table_import_payload: frame %d: the header does not decode: %s", f,
             zs::error_name(e));
    layouts.push_back(parse_record_batch_message(header.data(), int64_t(header.size())));
    const FrameLayout& L = layouts.back();
    FG_CHECK(L.body_length >= 0, FLOCKGPU_ERR_INVALID, "table_import_payload: frame %d: the header declares no bodyLength", f);
    check_frame_layout(schema, f, L, L.body_length);
    ZBody& Bd = zb[size_t(f)];
    Bd.first_block = int32_t(blocks.size());
    walk_body(f, bodies[f], body_lens[f], L.body_length, src_total, blocks, lit_total, seq_total);
    Bd.n_blocks = int32_t(blocks.size()) - Bd.first_block;
    Bd.out = out_total;
    Bd.len = L.body_length;
    Bd.ext_first = int32_t(ext_req.size());
    for (int64_t c = 0; c < n_fields; ++c)
      if (dtype_from_format(schema->children[c]->format) == FLOCKGPU_UTF8 && L.length > 0) {
        const int64_t offs = Bd.out + L.buffers[first_buf[size_t(c)] + 1].first;
        ext_req.push_back(offs);
        ext_req.push_back(offs + L.length * 4);
        ext_col.emplace_back(f, int(c));
      }
    Bd.ext_n = int32_t(ext_req.size()) - Bd.ext_first;
    src_total += body_lens[f];
    out_total += align16(L.body_length);
  }
  FG_CHECK(blocks.size() < (size_t(1) << 31) && seq_total < (int64_t(1) << 31), FLOCKGPU_ERR_UNSUPPORTED, "table_import_payload: too many blocks in one call");
  std::vector<int> proj;
  if (projection) proj.assign(projection, projection + n_projection);
  else
    for (int i = 0; i < n_fields; ++i) proj.push_back(i);
  int64_t total = 0;
  for (const FrameLayout& L : layouts) total += L.length;
  FG_CHECK(total < (int64_t(1) << 32) - 1, FLOCKGPU_ERR_UNSUPPORTED, "table_import: more than 2^32-2 rows in one relation");
  for (int p : proj) {
    FG_CHECK(p >= 0 && p < n_fields, FLOCKGPU_ERR_INVALID, "table_import: projection index %d out of range", p);
    FG_CHECK(schema->children[p]->dictionary == nullptr, FLOCKGPU_ERR_UNSUPPORTED, "table_import: dictionary-encoded column \"%s\"", schema->children[p]->name);
  }

  // ---- device ----
  const CtxPtr ctx = core_of(handle);
  std::lock_guard<std::recursive_mutex> g(ctx->mu);
  FG_CUDA(cudaSetDevice(ctx->device));
  // compressed bodies, back to back
  BufferPtr d_src = alloc(ctx, size_t(src_total));
  {
    std::vector<HostPiece> pieces;
    size_t off = 0;
    for (int f = 0; f < n_frames; ++f) {
      if (body_lens[f] == 0) continue;
      pieces.push_back({static_cast<char*>(d_src->ptr) + off, reinterpret_cast<const char*>(bodies[f]), size_t(body_lens[f]), off});
      off += size_t(body_lens[f]);
    }
    upload_host_pieces(ctx, pieces, off);
  }
  // descriptors: blocks | bodies | ext requests, one copy
  const size_t n_blocks = blocks.size(), n_ext = ext_req.size();
  const size_t o_bodies = align16(int64_t(n_blocks * sizeof(ZBlock))), o_ext = o_bodies + align16(int64_t(zb.size() * sizeof(ZBody)));
  const size_t desc_bytes = o_ext + n_ext * sizeof(int64_t);
  std::vector<uint8_t> desc(desc_bytes ? desc_bytes : 1);
  if (n_blocks) memcpy(desc.data(), blocks.data(), n_blocks * sizeof(ZBlock));
  if (!zb.empty()) memcpy(desc.data() + o_bodies, zb.data(), zb.size() * sizeof(ZBody));
  if (n_ext) memcpy(desc.data() + o_ext, ext_req.data(), n_ext * sizeof(int64_t));
  BufferPtr d_desc = alloc(ctx, desc.size());
  ctx->h2d_bytes.fetch_add(int64_t(desc.size()), std::memory_order_relaxed);
  FG_CUDA(cudaMemcpyAsync(d_desc->ptr, desc.data(), desc.size(), cudaMemcpyHostToDevice, ctx->stream));
  // scratch: decoded bodies, literals, sequences, block sizes, and the words read back (errors | Utf8 extents)
  BufferPtr d_dec = alloc(ctx, size_t(out_total));
  BufferPtr d_lits = alloc(ctx, size_t(lit_total));
  BufferPtr d_seqs = alloc(ctx, size_t(seq_total) * sizeof(zs::Seq));
  BufferPtr d_regen = alloc(ctx, n_blocks * 4);
  const size_t stat_words = size_t(n_frames) + n_ext;
  BufferPtr d_stat = alloc(ctx, stat_words * 4);
  if (stat_words) FG_CUDA(cudaMemsetAsync(d_stat->ptr, 0, stat_words * 4, ctx->stream));
  const uint8_t* src = static_cast<const uint8_t*>(d_src->ptr);
  const ZBlock* d_blocks = at_offset<const ZBlock>(d_desc, 0);
  const ZBody* d_bodies = at_offset<const ZBody>(d_desc, o_bodies);
  const int64_t* d_ext = at_offset<const int64_t>(d_desc, o_ext);
  uint32_t* d_err = d_stat->as<uint32_t>();
  int32_t* d_ext_out = reinterpret_cast<int32_t*>(d_err + n_frames);
  {
    LaunchTimer lt(ctx, "zstd_entropy_kernel");
    const int grid = std::max<int>(1, int((n_blocks + kEntropyWarps - 1) / kEntropyWarps));
    zstd_entropy_kernel<<<grid, 32 * kEntropyWarps, 0, ctx->stream>>>(src, d_blocks, int(n_blocks), d_lits->as<uint8_t>(), d_seqs->as<zs::Seq>(),
                                                                       d_regen->as<int32_t>(), d_err);
  }
  count_launch(ctx);
  FG_CUDA(cudaGetLastError());
  {
    LaunchTimer lt(ctx, "zstd_execute_kernel");
    zstd_execute_kernel<<<std::max(1, n_frames), 32, 0, ctx->stream>>>(src, d_blocks, d_bodies, n_frames, d_lits->as<uint8_t>(), d_seqs->as<zs::Seq>(),
                                                                       d_regen->as<int32_t>(), d_dec->as<uint8_t>(), d_err, d_ext, d_ext_out);
  }
  count_launch(ctx);
  FG_CUDA(cudaGetLastError());
  std::vector<uint32_t> stat(stat_words);
  if (stat_words) FG_CUDA(cudaMemcpyAsync(stat.data(), d_stat->ptr, stat_words * 4, cudaMemcpyDeviceToHost, ctx->stream));
  FG_CUDA(cudaStreamSynchronize(ctx->stream));
  for (int f = 0; f < n_frames; ++f) {
    const uint32_t w = stat[size_t(f)];
    FG_CHECK(!w, FLOCKGPU_ERR_INVALID, "table_import_payload: frame %d: zstd body does not decode (block %u): %s", f, w >> 8, zs::error_name(int(w & 255)));
  }
  std::vector<int32_t> ext(n_ext);
  if (n_ext) memcpy(ext.data(), stat.data() + n_frames, n_ext * 4);
  // first / last offset of every non-empty Utf8 column of every frame, as import_ipc checks them
  std::vector<std::vector<std::pair<int32_t, int32_t>>> extent(size_t(n_frames), std::vector<std::pair<int32_t, int32_t>>(size_t(n_fields), {0, 0}));
  for (size_t k = 0; k < ext_col.size(); ++k) {
    const int f = ext_col[k].first, c = ext_col[k].second;
    check_utf8_extent(f, schema->children[c]->name, ext[2 * k], ext[2 * k + 1], layouts[size_t(f)].buffers[first_buf[size_t(c)] + 2].second);
    extent[size_t(f)][size_t(c)] = {ext[2 * k], ext[2 * k + 1]};
  }

  // ---- the table: segments of every projected column, one launch ----
  auto t = std::make_shared<Table>();
  t->ctx = ctx;
  t->num_rows = total;
  t->metadata = copy_metadata(schema->metadata);
  std::vector<Seg> segs;
  const uint8_t* dec = d_dec->as<uint8_t>();
  for (int p : proj) {
    const ArrowSchema* cs = schema->children[p];
    const int dt = dtype_from_format(cs->format);
    Column col;
    col.dtype = dt;
    col.name = cs->name ? cs->name : "";
    col.format = cs->format;
    col.nullable = (cs->flags & ARROW_FLAG_NULLABLE) != 0;
    col.length = total;
    const size_t fb = first_buf[size_t(p)];
    bool has_null = false;
    for (const FrameLayout& L : layouts) has_null = has_null || L.nodes[size_t(p)].second > 0;
    if (has_null) col.validity = alloc(ctx, size_t(total));
    if (dt == FLOCKGPU_UTF8) {
      int64_t bytes = 0;
      for (int f = 0; f < n_frames; ++f) bytes += extent[size_t(f)][size_t(p)].second - extent[size_t(f)][size_t(p)].first;
      FG_CHECK(bytes < (int64_t(1) << 31), FLOCKGPU_ERR_UNSUPPORTED, "table_import: Utf8 column \"%s\" holds %lld bytes; at most 2^31-1 per relation", col.name.c_str(),
               (long long)bytes);
      col.offsets = alloc(ctx, size_t(total + 1) * 4);
      col.data = alloc(ctx, size_t(bytes));
      col.values_bytes = bytes;
    } else {
      col.data = alloc(ctx, size_t(total) * dtype_width(dt));
    }
    int64_t row = 0, byte = 0;
    for (int f = 0; f < n_frames; ++f) {
      const FrameLayout& L = layouts[size_t(f)];
      const uint8_t* body = dec + zb[size_t(f)].out;
      const int64_t len = L.length;
      if (len == 0) continue;
      if (has_null) {
        if (L.nodes[size_t(p)].second > 0) add_segs(segs, Seg::kBitsToBytes, body + L.buffers[fb].first, col.validity->as<uint8_t>() + row, len);
        else add_segs(segs, Seg::kFill, nullptr, col.validity->as<uint8_t>() + row, len, 1);
      }
      if (dt == FLOCKGPU_UTF8) {
        const auto ex = extent[size_t(f)][size_t(p)];
        add_segs(segs, Seg::kOffsets, body + L.buffers[fb + 1].first, reinterpret_cast<uint8_t*>(col.offsets->as<int32_t>() + row), len, int32_t(byte - ex.first));
        add_segs(segs, Seg::kCopy, body + L.buffers[fb + 2].first + ex.first, static_cast<uint8_t*>(col.data->ptr) + byte, ex.second - ex.first);
        byte += ex.second - ex.first;
      } else {
        const int w = dtype_width(dt);
        add_segs(segs, Seg::kCopy, body + L.buffers[fb + 1].first, static_cast<uint8_t*>(col.data->ptr) + row * w, len * w);
      }
      row += len;
    }
    if (dt == FLOCKGPU_UTF8) add_segs(segs, Seg::kSetI32, nullptr, reinterpret_cast<uint8_t*>(col.offsets->as<int32_t>() + total), 1, int32_t(byte));
    t->cols.push_back(std::move(col));
  }
  launch_segments(ctx, segs, "payload_assemble_kernel");  // the scratch buffers are released in stream order after the launch
  return t;
}

}  // namespace fg

using namespace fg;

extern "C" {

int flockgpu_table_import_payload(flockgpu_ctx* ctx, const struct ArrowSchema* schema, int32_t encoding, const uint8_t* const* headers,
                                  const int64_t* header_lens, const uint8_t* const* bodies, const int64_t* body_lens, int32_t n_frames,
                                  const int32_t* projection, int32_t n_projection, flockgpu_table** out) {
  if (encoding == FLOCKGPU_ENCODING_NONE)
    return flockgpu_table_import_ipc(ctx, schema, headers, header_lens, bodies, body_lens, n_frames, projection, n_projection, out);
  return guarded([&] {
    FG_CHECK(out, FLOCKGPU_ERR_INVALID, "table_import_payload: null out pointer");
    FG_CHECK(encoding >= FLOCKGPU_ENCODING_SNAPPY && encoding <= FLOCKGPU_ENCODING_NONE, FLOCKGPU_ERR_INVALID, "table_import_payload: unknown encoding %d",
             int(encoding));
    FG_CHECK(encoding == FLOCKGPU_ENCODING_ZSTD, FLOCKGPU_ERR_UNSUPPORTED, "table_import_payload: %s payloads are not decoded on the GPU (zstd and none are)",
             encoding == FLOCKGPU_ENCODING_SNAPPY ? "snappy" : encoding == FLOCKGPU_ENCODING_LZ4 ? "lz4" : "zlib");
    *out = wrap_table(import_payload_zstd(ctx, schema, headers, header_lens, bodies, body_lens, n_frames, projection, n_projection));
  });
}

}  // extern "C"
