// zstd_dec.h -- the pieces of a Zstandard decoder (RFC 8878), shared by the device kernels (zstd.cu) and the host.
//
// Everything here is __host__ __device__: the payload-import kernels decode the blocks of compressed bodies with it, the
// host decodes the ~100-byte compressed IPC headers with it (and walks the bodies to build the block table), and the
// CPU-only self test (flockgpu_selftest_zstd_decompress) runs the same functions serially so that CPU CI checks the
// decoder byte for byte against another implementation.  Written from the RFC; section numbers below refer to it.
//
// Every read is bounded by the range the caller hands in: a bitstream that runs past its start, a table description
// that runs past its section, a count that disagrees with its header is an error code (Z_*), never an access outside.
#pragma once

#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define ZHD __host__ __device__ __forceinline__
#else
#define ZHD inline
#endif

namespace fg {
namespace zstd {

enum : int {
  Z_OK = 0,
  Z_TRUNCATED = 1,    // a header, section or stream runs past the bytes that hold it
  Z_BAD_FSE = 2,      // FSE table description (4.1.1)
  Z_BAD_HUFFMAN = 3,  // Huffman tree description (4.2.1)
  Z_BAD_LITERALS = 4, // literal streams do not decode to their declared size
  Z_BAD_SEQUENCES = 5,// sequence bitstream does not end where its last sequence does
  Z_BAD_OFFSET = 6,   // a match reaches before the start of its frame, or a zero offset
  Z_OVERFLOW = 7,     // more output than the frame / body / block declares
  Z_RESERVED = 8,     // a reserved field is set
  Z_BAD_BLOCK = 9,    // block type 3 or a block larger than 128 KiB
  Z_NO_TABLE = 10,    // treeless literals or Repeat_Mode with no earlier table in the frame
  Z_BAD_MAGIC = 11,
  Z_DICTIONARY = 12,  // a Dictionary_ID other than 0
  Z_SIZE = 13,        // decoded size differs from Frame_Content_Size or from the declared body length
  Z_COUNTS = 14,      // the sequences consume more literals than the literal section holds
};

ZHD const char* error_name(int e) {
  switch (e) {
    case Z_OK: return "ok";
    case Z_TRUNCATED: return "truncated";
    case Z_BAD_FSE: return "corrupt FSE table description";
    case Z_BAD_HUFFMAN: return "corrupt Huffman tree description";
    case Z_BAD_LITERALS: return "literal streams do not decode to their declared size";
    case Z_BAD_SEQUENCES: return "corrupt sequence bitstream";
    case Z_BAD_OFFSET: return "match offset reaches before the start of its frame";
    case Z_OVERFLOW: return "more output than declared";
    case Z_RESERVED: return "reserved bit set";
    case Z_BAD_BLOCK: return "bad block type or size";
    case Z_NO_TABLE: return "table reused before one was defined in the frame";
    case Z_BAD_MAGIC: return "bad frame magic";
    case Z_DICTIONARY: return "frame needs a dictionary";
    case Z_SIZE: return "decoded size differs from the declared size";
    case Z_COUNTS: return "sequences use more literals than the block holds";
    default: return "corrupt data";
  }
}

constexpr uint32_t kMagic = 0xFD2FB528u;
constexpr int32_t kMaxBlock = 128 * 1024;  // Block_Maximum_Size (3.1.1.2.3) and the largest regenerated block
constexpr int kMaxHufBits = 11;            // Max_Number_of_Bits (4.2.1)
constexpr int kLL = 0, kOF = 1, kML = 2;   // order of the table descriptions in a sequences section (3.1.1.3.2.1)

ZHD int highbit(uint32_t v) {  // index of the highest set bit, v > 0
#if defined(__CUDA_ARCH__)
  return 31 - __clz(v);
#else
  return 31 - __builtin_clz(v);
#endif
}

ZHD uint32_t rd_le(const uint8_t* p, int n) {
  uint32_t v = 0;
  for (int i = 0; i < n; ++i) v |= uint32_t(p[i]) << (8 * i);
  return v;
}

// ---- constants (3.1.1.3.2.1.1 code tables, 3.1.1.3.2.2 default distributions) ----------------------------------------------
#define ZD_LL_BASE 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536
#define ZD_LL_BITS 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16
#define ZD_ML_BASE                                                                                                                          \
  3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 19, 20, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32, 33, 34, 35, 37, 39, 41, 43, \
      47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195, 16387, 32771, 65539
#define ZD_ML_BITS \
  0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16
#define ZD_LL_DEFAULT 4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1
#define ZD_ML_DEFAULT                                                                                                                      \
  1, 4, 3, 2, 2, 2, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, \
      -1, -1, -1, -1, -1, -1
#define ZD_OF_DEFAULT 1, 1, 1, 1, 1, 1, 2, 2, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, -1, -1, -1, -1, -1

#if defined(__CUDACC__)
static __constant__ uint32_t d_ll_base[36] = {ZD_LL_BASE};
static __constant__ uint8_t d_ll_bits[36] = {ZD_LL_BITS};
static __constant__ uint32_t d_ml_base[53] = {ZD_ML_BASE};
static __constant__ uint8_t d_ml_bits[53] = {ZD_ML_BITS};
static __constant__ int16_t d_ll_def[36] = {ZD_LL_DEFAULT};
static __constant__ int16_t d_ml_def[53] = {ZD_ML_DEFAULT};
static __constant__ int16_t d_of_def[29] = {ZD_OF_DEFAULT};
#endif
static const uint32_t h_ll_base[36] = {ZD_LL_BASE};
static const uint8_t h_ll_bits[36] = {ZD_LL_BITS};
static const uint32_t h_ml_base[53] = {ZD_ML_BASE};
static const uint8_t h_ml_bits[53] = {ZD_ML_BITS};
static const int16_t h_ll_def[36] = {ZD_LL_DEFAULT};
static const int16_t h_ml_def[53] = {ZD_ML_DEFAULT};
static const int16_t h_of_def[29] = {ZD_OF_DEFAULT};

#if defined(__CUDA_ARCH__)
#define ZD_TAB(name) d_##name
#else
#define ZD_TAB(name) h_##name
#endif

// ---- bit readers ---------------------------------------------------------------------------------------------------------
// Forward little-endian bits (FSE table descriptions).  Reads past the end give zero bits and set `over`.
struct FwdBits {
  const uint8_t* p;
  int64_t n;
  int64_t pos = 0;  // bits consumed
  ZHD uint32_t peek(int nb) const {
    uint64_t v = 0;
    const int64_t b = pos >> 3;
    for (int i = 0; i < 5; ++i)
      if (b + i < n) v |= uint64_t(p[b + i]) << (8 * i);
    return uint32_t(v >> (pos & 7)) & ((1u << nb) - 1);
  }
  ZHD void skip(int nb) { pos += nb; }
  ZHD uint32_t read(int nb) {
    const uint32_t v = peek(nb);
    pos += nb;
    return v;
  }
  ZHD bool over() const { return pos > n * 8; }
};

// Backward bitstream (4.1): bits are consumed from the end towards the start, the highest set bit of the last byte is
// the end mark.  `pos` = bits still unread; it may go negative, the missing bits then read as zero (4.2.1.1 and the
// last state update of a Huffman-weight stream rely on that) -- the caller decides whether that is an error.
struct BitIn {
  const uint8_t* p = nullptr;
  int64_t n = 0;
  int64_t pos = 0;
  int64_t lo = 1;     // cache holds bits [lo, lo + 64); lo is a multiple of 8
  uint64_t cache = 0;
  ZHD int init(const uint8_t* s, int64_t len) {
    p = s;
    n = len;
    if (len < 1) return Z_TRUNCATED;
    const uint8_t last = s[len - 1];
    if (!last) return Z_TRUNCATED;  // no end mark
    pos = (len - 1) * 8 + highbit(last);
    lo = 1;  // not a multiple of 8: forces the first refill
    return Z_OK;
  }
  ZHD void refill() {
    lo = ((pos + 7) & ~int64_t(7)) - 64;
    const int64_t b = lo >> 3;
    uint64_t v = 0;
    if (b >= 0 && b + 8 <= n) {
      for (int i = 0; i < 8; ++i) v |= uint64_t(p[b + i]) << (8 * i);
    } else {
      for (int i = 0; i < 8; ++i)
        if (b + i >= 0 && b + i < n) v |= uint64_t(p[b + i]) << (8 * i);
    }
    cache = v;
  }
  // bits [pos - nb, pos) as an integer (bit pos - 1 is its most significant bit); nb <= 32
  ZHD uint32_t peek(int nb) {
    if (nb == 0) return 0;
    if ((lo & 7) || pos - nb < lo || pos > lo + 64) refill();
    return uint32_t(cache >> (pos - nb - lo)) & uint32_t((uint64_t(1) << nb) - 1);
  }
  ZHD uint32_t read(int nb) {
    const uint32_t v = peek(nb);
    pos -= nb;
    return v;
  }
};

// ---- FSE (4.1.1) -----------------------------------------------------------------------------------------------------------
struct FseEntry {
  uint16_t base;  // baseline of the next state
  uint8_t nb;     // bits to read for the next state
  uint8_t sym;
};

// Normalised counts of an FSE table description.  `*used` = bytes of the description.
ZHD int fse_read_counts(const uint8_t* src, int64_t n, int max_sym, int max_log, int16_t* norm, int* nsym, int* alog, int64_t* used) {
  if (n < 1) return Z_TRUNCATED;
  FwdBits br{src, n};
  const int al = int(br.read(4)) + 5;
  if (al > max_log) return Z_BAD_FSE;
  int remaining = 1 << al, s = 0;
  while (remaining > 0) {
    if (s > max_sym) return Z_BAD_FSE;
    const int bits = highbit(uint32_t(remaining + 1)) + 1;
    uint32_t val = br.peek(bits);
    const uint32_t lower = (1u << (bits - 1)) - 1;
    const uint32_t threshold = (1u << bits) - 1 - uint32_t(remaining + 1);
    if ((val & lower) < threshold) {
      br.skip(bits - 1);
      val &= lower;
    } else {
      br.skip(bits);
      if (val > lower) val -= threshold;
    }
    const int proba = int(val) - 1;
    remaining -= proba < 0 ? -proba : proba;
    norm[s++] = int16_t(proba);
    if (proba == 0) {
      for (;;) {
        const int rep = int(br.read(2));
        for (int i = 0; i < rep; ++i) {
          if (s > max_sym) return Z_BAD_FSE;
          norm[s++] = 0;
        }
        if (rep != 3 || br.over()) break;
      }
    }
    if (br.over()) return Z_TRUNCATED;
  }
  if (remaining != 0) return Z_BAD_FSE;
  *nsym = s;
  *alog = al;
  *used = (br.pos + 7) >> 3;
  return Z_OK;
}

// Decoding table from normalised counts (symbols [0, nsym), nsym <= 64).
ZHD int fse_build(const int16_t* norm, int nsym, int alog, FseEntry* t) {
  const int size = 1 << alog;
  int high = size - 1;
  uint16_t next[64];
  for (int s = 0; s < nsym; ++s) {
    if (norm[s] == -1) {
      if (high < 0) return Z_BAD_FSE;
      t[high--].sym = uint8_t(s);
      next[s] = 1;
    } else {
      next[s] = uint16_t(norm[s]);
    }
  }
  const int step = (size >> 1) + (size >> 3) + 3, mask = size - 1;
  int pos = 0;
  for (int s = 0; s < nsym; ++s)
    for (int i = 0; i < norm[s]; ++i) {
      t[pos].sym = uint8_t(s);
      do {
        pos = (pos + step) & mask;
      } while (pos > high);
    }
  if (pos != 0) return Z_BAD_FSE;
  for (int i = 0; i < size; ++i) {
    const int s = t[i].sym;
    const uint32_t x = next[s]++;
    const int nb = alog - highbit(x);
    t[i].nb = uint8_t(nb);
    t[i].base = uint16_t((x << nb) - uint32_t(size));
  }
  return Z_OK;
}

// ---- Huffman (4.2) ---------------------------------------------------------------------------------------------------------
struct HufEntry {
  uint8_t sym;
  uint8_t nb;
};

// Huffman tree description at src[0, n) -> decoding table of 1 << *bits entries (<= 2048).  `*used` = description bytes.
ZHD int huf_read_table(const uint8_t* src, int64_t n, HufEntry* table, int* bits, int64_t* used) {
  if (n < 1) return Z_TRUNCATED;
  uint8_t w[260];
  int nw = 0;
  const int hb = src[0];
  if (hb < 128) {  // FSE-compressed weights, two interleaved states
    if (1 + hb > n || hb < 1) return Z_TRUNCATED;
    int16_t norm[16];
    int nsym, alog;
    int64_t u;
    int e = fse_read_counts(src + 1, hb, 15, 6, norm, &nsym, &alog, &u);
    if (e) return e == Z_TRUNCATED ? Z_BAD_HUFFMAN : e;
    if (u >= hb) return Z_BAD_HUFFMAN;
    FseEntry ft[64];
    if (fse_build(norm, nsym, alog, ft)) return Z_BAD_HUFFMAN;
    BitIn br;
    if (br.init(src + 1 + u, hb - u)) return Z_BAD_HUFFMAN;
    uint32_t s1 = br.read(alog), s2 = br.read(alog);
    if (br.pos < 0) return Z_BAD_HUFFMAN;
    for (;;) {
      if (nw > 253) return Z_BAD_HUFFMAN;
      w[nw++] = ft[s1].sym;
      s1 = ft[s1].base + br.read(ft[s1].nb);
      if (br.pos < 0) {
        w[nw++] = ft[s2].sym;
        break;
      }
      w[nw++] = ft[s2].sym;
      s2 = ft[s2].base + br.read(ft[s2].nb);
      if (br.pos < 0) {
        w[nw++] = ft[s1].sym;
        break;
      }
    }
    *used = 1 + hb;
  } else {  // direct: 4 bits per weight
    nw = hb - 127;
    const int bytes = (nw + 1) / 2;
    if (1 + bytes > n) return Z_TRUNCATED;
    for (int i = 0; i < nw; ++i) w[i] = uint8_t(i & 1 ? src[1 + i / 2] & 15 : src[1 + i / 2] >> 4);
    *used = 1 + bytes;
  }
  if (nw > 255) return Z_BAD_HUFFMAN;
  uint32_t total = 0;
  for (int i = 0; i < nw; ++i) {
    if (w[i] > kMaxHufBits) return Z_BAD_HUFFMAN;
    if (w[i]) total += 1u << (w[i] - 1);
  }
  if (total == 0) return Z_BAD_HUFFMAN;
  const int maxb = highbit(total) + 1;
  if (maxb > kMaxHufBits) return Z_BAD_HUFFMAN;
  const uint32_t rest = (1u << maxb) - total;
  if (rest == 0 || (rest & (rest - 1))) return Z_BAD_HUFFMAN;
  w[nw++] = uint8_t(highbit(rest) + 1);
  // canonical codes: longer codes first, symbols in order inside one length
  uint32_t rank_count[kMaxHufBits + 2] = {0}, rank_idx[kMaxHufBits + 2];
  for (int s = 0; s < nw; ++s)
    if (w[s]) rank_count[maxb + 1 - w[s]]++;
  rank_idx[maxb] = 0;
  for (int i = maxb; i >= 1; --i) rank_idx[i - 1] = rank_idx[i] + rank_count[i] * (1u << (maxb - i));
  for (int s = 0; s < nw; ++s) {
    if (!w[s]) continue;
    const int nb = maxb + 1 - w[s];
    const uint32_t len = 1u << (maxb - nb);
    for (uint32_t k = 0; k < len; ++k) table[rank_idx[nb] + k] = HufEntry{uint8_t(s), uint8_t(nb)};
    rank_idx[nb] += len;
  }
  *bits = maxb;
  return Z_OK;
}

// One Huffman-coded stream -> exactly `count` bytes; the stream must end exactly at its start.
ZHD int huf_decode_stream(const HufEntry* t, int bits, const uint8_t* src, int64_t n, uint8_t* dst, int64_t count) {
  BitIn br;
  if (br.init(src, n)) return Z_BAD_LITERALS;
  for (int64_t i = 0; i < count; ++i) {
    const HufEntry e = t[br.peek(bits)];
    if (e.nb > br.pos) return Z_BAD_LITERALS;
    br.pos -= e.nb;
    dst[i] = e.sym;
  }
  return br.pos == 0 ? Z_OK : Z_BAD_LITERALS;
}

// The 1 or 4 streams of a literal section (src = the streams, after any tree description).  Streams k = first, first +
// step, ... < 4 are decoded by this caller (the host passes 0, 1; a warp passes lane, 32).
ZHD int huf_decode_literals(const HufEntry* t, int bits, const uint8_t* src, int64_t n, int streams, uint8_t* dst, int64_t regen, int first, int step) {
  if (streams == 1) return first == 0 ? huf_decode_stream(t, bits, src, n, dst, regen) : Z_OK;
  if (n < 6) return Z_TRUNCATED;
  const int64_t s1 = rd_le(src, 2), s2 = rd_le(src + 2, 2), s3 = rd_le(src + 4, 2);
  const int64_t s4 = n - 6 - s1 - s2 - s3;
  if (s4 < 1) return Z_TRUNCATED;
  const int64_t seg = (regen + 3) / 4;
  if (3 * seg > regen) return Z_BAD_LITERALS;
  int e = Z_OK;
  const int64_t begin[4] = {6, 6 + s1, 6 + s1 + s2, 6 + s1 + s2 + s3}, len[4] = {s1, s2, s3, s4};
  for (int k = first; k < 4 && !e; k += step) e = huf_decode_stream(t, bits, src + begin[k], len[k], dst + k * seg, k < 3 ? seg : regen - 3 * seg);
  return e;
}

// ---- sections of a compressed block (3.1.1.3) ---------------------------------------------------------------------------------
struct LitHeader {
  int type;     // 0 raw, 1 RLE, 2 compressed, 3 treeless
  int streams;  // 1 or 4
  int hdr;      // header bytes
  int32_t regen, comp;  // regenerated bytes; bytes after the header (raw: regen, RLE: 1, else tree + streams)
};

ZHD int lit_header(const uint8_t* p, int64_t n, LitHeader* h) {
  if (n < 1) return Z_TRUNCATED;
  const uint32_t b0 = p[0];
  h->type = int(b0 & 3);
  const int sf = int(b0 >> 2) & 3;
  if (h->type < 2) {
    h->streams = 1;
    h->hdr = sf == 1 ? 2 : sf == 3 ? 3 : 1;
    if (n < h->hdr) return Z_TRUNCATED;
    h->regen = sf == 1 ? int32_t((b0 >> 4) + (uint32_t(p[1]) << 4)) : sf == 3 ? int32_t((b0 >> 4) + (uint32_t(p[1]) << 4) + (uint32_t(p[2]) << 12)) : int32_t(b0 >> 3);
    h->comp = h->type == 0 ? h->regen : 1;
  } else {
    h->streams = sf == 0 ? 1 : 4;
    h->hdr = sf < 2 ? 3 : sf == 2 ? 4 : 5;
    if (n < h->hdr) return Z_TRUNCATED;
    uint64_t v = 0;
    for (int i = 0; i < h->hdr; ++i) v |= uint64_t(p[i]) << (8 * i);
    const int sb = sf < 2 ? 10 : sf == 2 ? 14 : 18;
    h->regen = int32_t((v >> 4) & ((1u << sb) - 1));
    h->comp = int32_t((v >> (4 + sb)) & ((1u << sb) - 1));
  }
  if (h->regen > kMaxBlock) return Z_BAD_LITERALS;
  if (int64_t(h->hdr) + h->comp > n) return Z_TRUNCATED;
  return Z_OK;
}

struct SeqHeader {
  int32_t nseq;
  int hdr;        // bytes of Number_of_Sequences + the modes byte
  uint8_t modes;  // Symbol_Compression_Modes
};

ZHD int seq_header(const uint8_t* p, int64_t n, SeqHeader* h) {
  if (n < 1) return Z_TRUNCATED;
  const int b0 = p[0];
  h->modes = 0;
  if (b0 == 0) {
    h->nseq = 0;
    h->hdr = 1;
    return n == 1 ? Z_OK : Z_BAD_SEQUENCES;  // nothing may follow an empty sequences section
  }
  if (b0 < 128) {
    h->nseq = b0;
    h->hdr = 2;
  } else if (b0 < 255) {
    if (n < 2) return Z_TRUNCATED;
    h->nseq = ((b0 - 128) << 8) + p[1];
    h->hdr = 3;
  } else {
    if (n < 3) return Z_TRUNCATED;
    h->nseq = p[1] + (p[2] << 8) + 0x7F00;
    h->hdr = 4;
  }
  if (n < h->hdr) return Z_TRUNCATED;
  h->modes = p[h->hdr - 1];
  if (h->modes & 3) return Z_RESERVED;
  return Z_OK;
}

ZHD int seq_mode(uint8_t modes, int which) { return (modes >> (6 - 2 * which)) & 3; }

// Walks the three table descriptions at p[0, n) (after the modes byte).  Builds table `which` (kLL / kOF / kML; -1 =
// none) into `out` unless its mode is Repeat (Z_NO_TABLE: the caller takes the table of the block it was defined in).
// `*end` = bytes of all three descriptions, i.e. where the sequence bitstream starts.
ZHD int seq_tables(const uint8_t* p, int64_t n, uint8_t modes, int which, FseEntry* out, int* log, int64_t* end) {
  int64_t at = 0;
  for (int k = 0; k < 3; ++k) {
    const int mode = seq_mode(modes, k);
    const int max_sym = k == kLL ? 35 : k == kOF ? 31 : 52, max_log = k == kOF ? 8 : 9;
    const bool want = k == which;
    if (mode == 0) {
      if (want) {
        const int16_t* def = k == kLL ? ZD_TAB(ll_def) : k == kOF ? ZD_TAB(of_def) : ZD_TAB(ml_def);
        int16_t norm[53];
        const int nsym = k == kLL ? 36 : k == kOF ? 29 : 53;
        for (int s = 0; s < nsym; ++s) norm[s] = def[s];
        *log = k == kOF ? 5 : 6;
        if (fse_build(norm, nsym, *log, out)) return Z_BAD_FSE;
      }
    } else if (mode == 1) {
      if (at >= n) return Z_TRUNCATED;
      const int sym = p[at++];
      if (sym > max_sym) return Z_BAD_FSE;
      if (want) {
        out[0] = FseEntry{0, 0, uint8_t(sym)};
        *log = 0;
      }
    } else if (mode == 2) {
      int16_t norm[53];
      int nsym, alog;
      int64_t used;
      const int e = fse_read_counts(p + at, n - at, max_sym, max_log, norm, &nsym, &alog, &used);
      if (e) return e;
      if (want) {
        if (fse_build(norm, nsym, alog, out)) return Z_BAD_FSE;
        *log = alog;
      }
      at += used;
    } else if (want) {
      return Z_NO_TABLE;
    }
  }
  if (at > n) return Z_TRUNCATED;
  *end = at;
  return Z_OK;
}

struct Seq {
  uint32_t ll, ml, of;  // literal length, match length, Offset_Value (3.1.1.5: 1..3 repeat codes, > 3 offset + 3)
};

// The sequence bitstream p[0, n) -> nseq sequences.  The stream must end exactly with the last sequence.
ZHD int seq_decode(const uint8_t* p, int64_t n, const FseEntry* tl, int ll_log, const FseEntry* to, int of_log, const FseEntry* tm, int ml_log, int32_t nseq,
                   Seq* out) {
  BitIn br;
  if (br.init(p, n)) return Z_BAD_SEQUENCES;
  uint32_t sl = br.read(ll_log), so = br.read(of_log), sm = br.read(ml_log);
  if (br.pos < 0) return Z_BAD_SEQUENCES;
  for (int32_t i = 0; i < nseq; ++i) {
    const FseEntry el = tl[sl], eo = to[so], em = tm[sm];
    if (el.sym > 35 || em.sym > 52 || eo.sym > 31) return Z_BAD_SEQUENCES;
    Seq q;
    q.of = (1u << eo.sym) + br.read(eo.sym);
    q.ml = ZD_TAB(ml_base)[em.sym] + br.read(ZD_TAB(ml_bits)[em.sym]);
    q.ll = ZD_TAB(ll_base)[el.sym] + br.read(ZD_TAB(ll_bits)[el.sym]);
    if (i + 1 < nseq) {
      sl = el.base + br.read(el.nb);
      sm = em.base + br.read(em.nb);
      so = eo.base + br.read(eo.nb);
    }
    if (br.pos < 0) return Z_BAD_SEQUENCES;
    out[i] = q;
  }
  return br.pos == 0 ? Z_OK : Z_BAD_SEQUENCES;
}

// Offset_Value -> offset, updating the three repeat offsets (3.1.1.5).  false: the offset would be 0.
ZHD bool resolve_offset(uint32_t* rep, uint32_t ov, uint32_t ll, uint32_t* off) {
  if (ov > 3) {
    *off = ov - 3;
    rep[2] = rep[1];
    rep[1] = rep[0];
    rep[0] = *off;
    return true;
  }
  const uint32_t idx = ov - 1 + (ll == 0 ? 1 : 0);
  if (idx == 0) {
    *off = rep[0];
  } else if (idx == 3) {
    *off = rep[0] - 1;
    if (*off == 0) return false;
    rep[2] = rep[1];
    rep[1] = rep[0];
    rep[0] = *off;
  } else {
    *off = rep[idx];
    if (idx == 2) rep[2] = rep[1];
    rep[1] = rep[0];
    rep[0] = *off;
  }
  return true;
}

// ---- frames and blocks (3.1.1) ----------------------------------------------------------------------------------------------
struct FrameHeader {
  int64_t content_size;  // -1: not present
  int hdr;               // bytes including the magic number
  bool checksum;
};

// One frame header at p[0, n); p starts with the zstd magic.  Skippable frames are the caller's business.
ZHD int frame_header(const uint8_t* p, int64_t n, FrameHeader* h) {
  if (n < 5) return Z_TRUNCATED;
  if (rd_le(p, 4) != kMagic) return Z_BAD_MAGIC;
  const uint32_t d = p[4];
  const int fcs_flag = int(d >> 6), single = int(d >> 5) & 1, did_flag = int(d & 3);
  if (d & 8) return Z_RESERVED;
  h->checksum = (d >> 2) & 1;
  const int did_bytes = did_flag == 0 ? 0 : did_flag == 1 ? 1 : did_flag == 2 ? 2 : 4;
  const int fcs_bytes = fcs_flag == 0 ? single : fcs_flag == 1 ? 2 : fcs_flag == 2 ? 4 : 8;
  h->hdr = 5 + (single ? 0 : 1) + did_bytes + fcs_bytes;
  if (n < h->hdr) return Z_TRUNCATED;
  int at = 5 + (single ? 0 : 1);
  if (did_bytes) {
    uint32_t did = rd_le(p + at, did_bytes);
    if (did != 0) return Z_DICTIONARY;
    at += did_bytes;
  }
  if (fcs_bytes == 0) {
    h->content_size = -1;
  } else if (fcs_bytes == 8) {
    const uint64_t v = uint64_t(rd_le(p + at, 4)) | (uint64_t(rd_le(p + at + 4, 4)) << 32);
    h->content_size = v > (uint64_t(1) << 62) ? (int64_t(1) << 62) : int64_t(v);
  } else {
    h->content_size = int64_t(rd_le(p + at, fcs_bytes)) + (fcs_bytes == 2 ? 256 : 0);
  }
  return Z_OK;
}

ZHD bool is_skippable(uint32_t magic) { return (magic & 0xFFFFFFF0u) == 0x184D2A50u; }

struct BlockHeader {
  bool last;
  int type;      // 0 raw, 1 RLE, 2 compressed
  int32_t size;  // Block_Size: content bytes (raw, compressed) or the repeat count (RLE)
  int32_t src;   // content bytes that follow the header (RLE: 1)
};

ZHD int block_header(const uint8_t* p, int64_t n, BlockHeader* h) {
  if (n < 3) return Z_TRUNCATED;
  const uint32_t v = rd_le(p, 3);
  h->last = v & 1;
  h->type = int(v >> 1) & 3;
  h->size = int32_t(v >> 3);
  if (h->type == 3 || h->size > kMaxBlock) return Z_BAD_BLOCK;
  h->src = h->type == 1 ? 1 : h->size;
  if (3 + int64_t(h->src) > n) return Z_TRUNCATED;
  return Z_OK;
}

}  // namespace zstd
}  // namespace fg
