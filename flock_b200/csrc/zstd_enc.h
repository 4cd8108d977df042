// zstd_enc.h -- the pieces of a Zstandard encoder (RFC 8878), shared by the export kernels (zstd_enc.cu) and the host.
//
// Everything here is __host__ __device__: the payload-export kernel compresses every 128 KiB block of every IPC body
// with it, one CTA per block; the host compresses the ~100-500-byte IPC headers with it; and the CPU-only self test
// (flockgpu_selftest_zstd_compress) runs the very same phases serially, so that CPU CI can check the GPU's bytes.
// Written from the RFC; the decoder side (zstd_dec.h) supplies the constants and the table builders.
//
// One block is compressed in phases.  Each phase is a function of (block state, lane); a CTA runs the lanes of a
// phase in parallel and synchronises between phases, the host runs them one after the other.  Nothing a phase
// produces depends on the order its lanes run in: lanes own disjoint inputs and outputs, and the only shared writes
// are commutative (histogram additions, ORs of disjoint bits).  So the device and the host produce the same bytes.
//
//   match     lane l owns bytes [l * kSpan, (l + 1) * kSpan) of the block.  A private hash table, seeded with the
//             kSeed bytes before that range (in the previous lane's range or the previous block), finds matches
//             greedily; a match never runs past the lane's range end, and may start anywhere earlier in the body.
//   literals  the bytes no match covers, compacted (a scan over the lanes) and counted.
//   literal   Raw, RLE or Huffman (1 stream up to 1023 literals, 4 above), whichever is smallest; Huffman codes are
//   section   limited to 11 bits, the tree is described with FSE-compressed weights or 4-bit weights.
//   sequences LL / OF / ML codes each take Predefined, RLE or FSE_Compressed, by estimated cost.  Offsets are always
//             written as Offset_Value = offset + 3: no repeat codes, so no block depends on an earlier one.
//   block     Compressed when that is smaller than the block itself, else RLE_Block (one repeated byte) or Raw_Block.
#pragma once

#include "zstd_dec.h"

namespace fg {
namespace zstd {

constexpr int kLanes = 128;                   // lanes of one block (threads of the compress kernel)
constexpr int kSpan = kMaxBlock / kLanes;     // bytes a lane owns: 1 KiB
constexpr int kSeed = 1024;                   // bytes before a lane's range that seed its hash table
constexpr int kHashLog = 8;                   // entries of a lane's hash table: 256 x u16
constexpr int kMinMatch = 4;
constexpr int kLaneSeqs = kSpan / kMinMatch;  // a lane's sequences: each covers >= kMinMatch of its bytes
constexpr int kHeadCap = 512;                 // frame header + block header + literals header + tree + jump table
constexpr int kMidCap = 512;                  // sequences header + three table descriptions
constexpr int kLitStreamCap = kMaxBlock + 64; // Huffman streams (only used when smaller than the literals)
constexpr int kSeqStreamCap = kMaxBlock;      // sequence bitstream (longer: the block is stored raw)
constexpr int kFrameHeaderMax = 14;

#if defined(__CUDA_ARCH__)
#define ZATOMIC_ADD(p, v) atomicAdd((p), (v))
#define ZATOMIC_OR(p, v) atomicOr((p), (v))
#else
#define ZATOMIC_ADD(p, v) (*(p) += (v))
#define ZATOMIC_OR(p, v) (*(p) |= (v))
#endif

ZHD uint32_t ld32(const uint8_t* p) { return uint32_t(p[0]) | (uint32_t(p[1]) << 8) | (uint32_t(p[2]) << 16) | (uint32_t(p[3]) << 24); }
ZHD uint32_t hash4(uint32_t v) { return (v * 2654435761u) >> (32 - kHashLog); }

// (literal length, match length, Offset_Value) of one sequence in one word; ll and ml < 2^18, Offset_Value < 2^28
ZHD uint64_t pack_seq(uint32_t ll, uint32_t ml, uint32_t ov) { return uint64_t(ll) | (uint64_t(ml) << 18) | (uint64_t(ov) << 36); }
ZHD uint32_t seq_ll(uint64_t s) { return uint32_t(s & 0x3FFFF); }
ZHD uint32_t seq_ml(uint64_t s) { return uint32_t((s >> 18) & 0x3FFFF); }
ZHD uint32_t seq_ov(uint64_t s) { return uint32_t(s >> 36); }

// ---- codes of a sequence (3.1.1.3.2.1.1) ------------------------------------------------------------------------------------
ZHD int ll_code(uint32_t ll) {
  if (ll < 16) return int(ll);
  if (ll >= 64) return highbit(ll) + 19;
  int c = 24;
  while (ll < ZD_TAB(ll_base)[c]) --c;
  return c;
}
ZHD int ml_code(uint32_t ml) {
  if (ml < 35) return int(ml) - 3;
  if (ml >= 131) return highbit(ml - 3) + 36;
  int c = 42;
  while (ml < ZD_TAB(ml_base)[c]) --c;
  return c;
}
ZHD int of_code(uint32_t ov) { return highbit(ov); }

// ---- bit writers ------------------------------------------------------------------------------------------------------------------
// Forward little-endian bits into dst[0, cap); writes past cap are dropped and set `over`.
struct BitOut {
  uint8_t* p;
  int64_t cap;
  int64_t at = 0;  // bytes written
  uint64_t acc = 0;
  int n = 0;  // bits in acc
  bool over = false;
  ZHD void put(uint32_t v, int nb) {  // nb <= 32
    if (nb == 0) return;
    acc |= uint64_t(v & uint32_t((uint64_t(1) << nb) - 1)) << n;
    n += nb;
    while (n >= 8) {
      if (at < cap) p[at] = uint8_t(acc);
      else over = true;
      ++at;
      acc >>= 8;
      n -= 8;
    }
  }
  ZHD int64_t flush() {  // pad to a byte with zero bits; returns the bytes written
    if (n > 0) put(0, 8 - n);
    return at;
  }
  ZHD int64_t close() {  // the end mark of a backward bitstream (4.1), then pad
    put(1, 1);
    return flush();
  }
};

// ORs the low nb bits of v into bit position `bit` of a zeroed little-endian word array (disjoint bits per caller).
ZHD void or_bits(uint32_t* words, uint64_t bit, uint32_t v, int nb) {
  if (nb == 0) return;
  const uint64_t x = uint64_t(v & uint32_t((uint64_t(1) << nb) - 1)) << (bit & 31);
  uint32_t* w = words + (bit >> 5);
  if (uint32_t(x)) ZATOMIC_OR(w, uint32_t(x));
  if (uint32_t(x >> 32)) ZATOMIC_OR(w + 1, uint32_t(x >> 32));
}

// ---- FSE (4.1.1) ------------------------------------------------------------------------------------------------------------------
// Normalised counts summing to 1 << log from the counts of symbols [0, nsym); every present symbol gets >= 1.
// (1 << log) >= 2 * present symbols is the caller's business.
ZHD void fse_normalize(const uint32_t* cnt, int nsym, uint32_t total, int log, int16_t* norm) {
  const int target = 1 << log;
  int sum = 0, big = -1;
  for (int s = 0; s < nsym; ++s) {
    int v = 0;
    if (cnt[s]) {
      v = int((uint64_t(cnt[s]) << log) / total);
      if (v < 1) v = 1;
      if (big < 0 || cnt[s] > cnt[big]) big = s;
    }
    norm[s] = int16_t(v);
    sum += v;
  }
  while (sum > target) {  // take one from the largest, again and again
    int m = 0;
    for (int s = 1; s < nsym; ++s)
      if (norm[s] > norm[m]) m = s;
    --norm[m];
    --sum;
  }
  norm[big] = int16_t(norm[big] + (target - sum));
}

// Table description (4.1.1) of norm[0, nsym) at accuracy `log`; returns its bytes, or -1 when cap is too small.
ZHD int fse_write_counts(const int16_t* norm, int nsym, int log, uint8_t* dst, int cap) {
  while (nsym > 0 && norm[nsym - 1] == 0) --nsym;
  BitOut bo{dst, cap};
  bo.put(uint32_t(log - 5), 4);
  int remaining = 1 << log;
  for (int s = 0; s < nsym && remaining > 0;) {
    const int proba = norm[s];
    const uint32_t val = uint32_t(proba + 1);
    const int bits = highbit(uint32_t(remaining + 1)) + 1;
    const uint32_t lower = (1u << (bits - 1)) - 1;
    const uint32_t threshold = (1u << bits) - 1 - uint32_t(remaining + 1);
    if (val < threshold) bo.put(val, bits - 1);
    else if (val <= lower) bo.put(val, bits);
    else bo.put(val + threshold, bits);
    remaining -= proba < 0 ? -proba : proba;
    ++s;
    if (proba == 0) {
      int z = 0;
      while (s < nsym && norm[s] == 0) {
        ++z;
        ++s;
      }
      while (z >= 3) {
        bo.put(3, 2);
        z -= 3;
      }
      bo.put(uint32_t(z), 2);
    }
  }
  const int64_t n = bo.flush();
  return bo.over ? -1 : int(n);
}

// Encoder view of an FSE decoding table: the decoding table itself plus, per symbol, its states in table order.
// The k-th state of symbol s (in table order) has x = n_s + k in the decoder's construction (zstd_dec.h fse_build).
struct FseEnc {
  FseEntry dt[512];
  uint16_t states[512];
  uint16_t first[64];
  int16_t n[64];  // normalised count, -1 ("less than 1") counted as 1
  int log;
};

// From normalised counts (log 0: RLE of symbol `rle`).  Z_OK or Z_BAD_FSE.
ZHD int fse_enc_build(const int16_t* norm, int nsym, int log, int rle, FseEnc* E) {
  E->log = log;
  if (log == 0) {
    E->dt[0] = FseEntry{0, 0, uint8_t(rle)};
    for (int s = 0; s < 64; ++s) E->n[s] = 0;
    E->n[rle] = 1;
    E->first[rle] = 0;
    E->states[0] = 0;
    return Z_OK;
  }
  if (fse_build(norm, nsym, log, E->dt)) return Z_BAD_FSE;
  uint16_t fill[64];
  int at = 0;
  for (int s = 0; s < 64; ++s) {
    E->n[s] = s < nsym ? (norm[s] < 0 ? int16_t(1) : norm[s]) : int16_t(0);
    E->first[s] = uint16_t(at);
    fill[s] = uint16_t(at);
    at += E->n[s];
  }
  for (int i = 0; i < (1 << log); ++i) E->states[fill[E->dt[i].sym]++] = uint16_t(i);
  return Z_OK;
}

// The state that decodes `sym` and whose update reaches `next`; *bits / *nb = the update bits.
ZHD uint32_t fse_prev_state(const FseEnc& E, int sym, uint32_t next, uint32_t* bits, int* nb) {
  const int L = E.log, n = E.n[sym], h = highbit(uint32_t(n));
  const uint32_t y = next + (1u << L);
  uint32_t x = y >> (L - h);
  if (int(x) < n) x = y >> (L - h - 1);
  const uint32_t st = E.states[E.first[sym] + (x - uint32_t(n))];
  *nb = E.dt[st].nb;
  *bits = next - E.dt[st].base;
  return st;
}

// Bits per symbol of a distribution in 1/256 bit, and what coding `cnt` with it costs.
ZHD uint32_t log2_fp(uint32_t x) {  // x >= 1: 256 * log2(x), linear between powers of two
  const int h = highbit(x);
  return uint32_t(h) * 256 + ((x << 8 >> h) - 256);
}
ZHD uint64_t fse_cost(const uint32_t* cnt, int nsym, const int16_t* norm, int log) {
  uint64_t c = 0;
  for (int s = 0; s < nsym; ++s) {
    if (!cnt[s]) continue;
    if (norm[s] == 0) return ~uint64_t(0) >> 2;
    const uint32_t p = norm[s] < 0 ? 1u : uint32_t(norm[s]);
    c += uint64_t(cnt[s]) * (uint64_t(log) * 256 - log2_fp(p));
  }
  return c;
}

// ---- Huffman (4.2) -------------------------------------------------------------------------------------------------------------
struct HufEnc {
  uint16_t code[256];
  uint8_t len[256];
  int maxb;
  int nw;  // weights described: symbols [0, nw); symbol nw is the last one, its weight implied
};

// Position of symbol s when the present symbols are sorted by (count, symbol): what each lane computes for its symbols.
ZHD int huf_rank(const uint32_t* cnt, int s) {
  int r = 0;
  for (int t = 0; t < 256; ++t) r += cnt[t] && (cnt[t] < cnt[s] || (cnt[t] == cnt[s] && t < s));
  return r;
}

// Code lengths <= kMaxHufBits from counts (>= 2 present symbols) and `sorted` = present symbols by (count, symbol).
ZHD void huf_lengths(const uint32_t* cnt, const uint8_t* sorted, int n, uint8_t* len) {
  // two-queue Huffman over the sorted leaves; ties prefer the leaf
  uint32_t iw[256];
  int16_t lpar[256], ipar[256];
  int i = 0, j = 0;
  for (int k = 0; k < n - 1; ++k) {
    uint32_t w = 0;
    for (int take = 0; take < 2; ++take) {
      const bool leaf = i < n && (j >= k || cnt[sorted[i]] <= iw[j]);
      if (leaf) {
        w += cnt[sorted[i]];
        lpar[i++] = int16_t(k);
      } else {
        w += iw[j];
        ipar[j++] = int16_t(k);
      }
    }
    iw[k] = w;
  }
  uint8_t depth[256];
  depth[n - 2] = 0;
  for (int k = n - 3; k >= 0; --k) depth[k] = uint8_t(depth[ipar[k]] + 1);
  for (int s = 0; s < 256; ++s) len[s] = 0;
  int over = 0;
  for (int q = 0; q < n; ++q) {
    int d = depth[lpar[q]] + 1;
    if (d > kMaxHufBits) {
      d = kMaxHufBits;
      over = 1;
    }
    len[sorted[q]] = uint8_t(d);
  }
  if (!over) return;
  // Kraft sum in units of 2^-11: lengthen the longest codes below the limit until it fits, then shorten the longest
  // codes while the sum stays <= 1 (the decoder needs a complete code)
  int32_t k = 0;
  for (int q = 0; q < n; ++q) k += 1 << (kMaxHufBits - len[sorted[q]]);
  const int32_t one = 1 << kMaxHufBits;
  while (k > one) {
    int best = -1;
    for (int q = 0; q < n; ++q) {  // ascending count: the first longest one is the rarest
      const int l = len[sorted[q]];
      if (l < kMaxHufBits && (best < 0 || l > len[sorted[best]])) best = q;
    }
    k -= 1 << (kMaxHufBits - len[sorted[best]] - 1);
    ++len[sorted[best]];
  }
  while (k < one) {
    int best = -1;
    for (int q = n - 1; q >= 0; --q) {  // descending count: the first longest one that fits is the commonest
      const int l = len[sorted[q]];
      if ((1 << (kMaxHufBits - l)) <= one - k && (best < 0 || l > len[sorted[best]])) best = q;
    }
    k += 1 << (kMaxHufBits - len[sorted[best]]);
    --len[sorted[best]];
  }
}

// Canonical codes exactly as the decoder's table (zstd_dec.h huf_read_table) assigns them.
ZHD void huf_codes(HufEnc* H) {
  int maxb = 0, last = 0;
  for (int s = 0; s < 256; ++s)
    if (H->len[s]) {
      if (H->len[s] > maxb) maxb = H->len[s];
      last = s;
    }
  H->maxb = maxb;
  H->nw = last;
  uint32_t rank_count[kMaxHufBits + 2] = {0}, rank_idx[kMaxHufBits + 2];
  for (int s = 0; s < 256; ++s)
    if (H->len[s]) rank_count[H->len[s]]++;
  rank_idx[maxb] = 0;
  for (int i = maxb; i >= 1; --i) rank_idx[i - 1] = rank_idx[i] + rank_count[i] * (1u << (maxb - i));
  for (int s = 0; s < 256; ++s) {
    const int nb = H->len[s];
    if (!nb) continue;
    H->code[s] = uint16_t(rank_idx[nb] >> (maxb - nb));
    rank_idx[nb] += 1u << (maxb - nb);
  }
}

// Tree description (4.2.1): FSE-compressed weights when that works and is smaller, else 4-bit weights when there are
// at most 128 of them.  Returns its bytes, or -1 when neither form applies.  `E` is scratch for the weights' table.
ZHD int huf_write_tree(const HufEnc& H, uint8_t* dst, int cap, FseEnc& E) {
  uint8_t w[256];
  const int N = H.nw;
  for (int s = 0; s < N; ++s) w[s] = H.len[s] ? uint8_t(H.maxb + 1 - H.len[s]) : uint8_t(0);
  int best = -1;
  if (N >= 2) {  // FSE: two interleaved states over one table of accuracy 6
    uint32_t cnt[16] = {0};
    int distinct = 0;
    for (int s = 0; s < N; ++s) distinct += cnt[w[s]]++ == 0;
    if (distinct >= 2) {
      int16_t norm[16];
      const int log = 6;
      fse_normalize(cnt, 16, uint32_t(N), log, norm);
      int nsym = 16;
      while (norm[nsym - 1] == 0) --nsym;
      fse_enc_build(norm, nsym, log, 0, &E);
      uint8_t tmp[160];
      int d = fse_write_counts(norm, nsym, log, tmp + 1, 127);
      if (d > 0) {
        BitOut bo{tmp + 1 + d, int64_t(127 - d)};
        uint32_t st[2];
        // the chain of weight N-2 ends with an update that reads past the stream's start (it needs nb >= 1: the
        // symbol's first state has it, its count being < 64), the chain of weight N-1 ends without one
        st[(N - 1) & 1] = E.states[E.first[w[N - 1]]];
        st[(N - 2) & 1] = E.states[E.first[w[N - 2]]];
        for (int k = N - 3; k >= 0; --k) {
          uint32_t bits;
          int nb;
          st[k & 1] = fse_prev_state(E, w[k], st[k & 1], &bits, &nb);
          bo.put(bits, nb);
        }
        bo.put(st[1], log);
        bo.put(st[0], log);
        const int64_t total = d + bo.close();
        if (!bo.over && total < 128) {
          tmp[0] = uint8_t(total);
          best = int(total) + 1;
          if (best <= cap)
            for (int i = 0; i < best; ++i) dst[i] = tmp[i];
          else
            best = -1;
        }
      }
    }
  }
  if (N <= 128) {
    const int direct = 1 + (N + 1) / 2;
    if ((best < 0 || direct < best) && direct <= cap) {
      dst[0] = uint8_t(127 + N);
      for (int i = 0; i < (N + 1) / 2; ++i) dst[1 + i] = uint8_t((w[2 * i] << 4) | (2 * i + 1 < N ? w[2 * i + 1] : 0));
      best = direct;
    }
  }
  return best;
}

// ---- headers -------------------------------------------------------------------------------------------------------------------
ZHD int frame_header_write(int64_t content_size, uint8_t* dst) {  // Single_Segment, no checksum, no dictionary
  dst[0] = 0x28;
  dst[1] = 0xB5;
  dst[2] = 0x2F;
  dst[3] = 0xFD;
  int flag, bytes;
  uint64_t v = uint64_t(content_size);
  if (content_size < 256) flag = 0, bytes = 1;
  else if (content_size < 65536 + 256) flag = 1, bytes = 2, v -= 256;
  else if (content_size < (int64_t(1) << 32)) flag = 2, bytes = 4;
  else flag = 3, bytes = 8;
  dst[4] = uint8_t((flag << 6) | (1 << 5));
  for (int i = 0; i < bytes; ++i) dst[5 + i] = uint8_t(v >> (8 * i));
  return 5 + bytes;
}
ZHD void block_header_write(uint8_t* dst, bool last, int type, uint32_t size) {
  const uint32_t v = (last ? 1u : 0u) | (uint32_t(type) << 1) | (size << 3);
  dst[0] = uint8_t(v);
  dst[1] = uint8_t(v >> 8);
  dst[2] = uint8_t(v >> 16);
}
// Raw / RLE literals section header; returns its bytes
ZHD int lit_header_raw(uint8_t* dst, int type, uint32_t regen) {
  if (regen < 32) {
    dst[0] = uint8_t(type | (regen << 3));
    return 1;
  }
  if (regen < 4096) {
    dst[0] = uint8_t(type | (1 << 2) | ((regen & 15) << 4));
    dst[1] = uint8_t(regen >> 4);
    return 2;
  }
  dst[0] = uint8_t(type | (3 << 2) | ((regen & 15) << 4));
  dst[1] = uint8_t(regen >> 4);
  dst[2] = uint8_t(regen >> 12);
  return 3;
}
// Compressed literals section header (Literals_Block_Type 2); returns its bytes
ZHD int lit_header_huf(uint8_t* dst, int streams, uint32_t regen, uint32_t comp) {
  const uint32_t m = regen > comp ? regen : comp;
  const int sf = streams == 1 ? 0 : m < 1024 ? 1 : m < 16384 ? 2 : 3;
  const int hdr = sf < 2 ? 3 : sf == 2 ? 4 : 5, sb = sf < 2 ? 10 : sf == 2 ? 14 : 18;
  const uint64_t v = 2u | (uint64_t(sf) << 2) | (uint64_t(regen) << 4) | (uint64_t(comp) << (4 + sb));
  for (int i = 0; i < hdr; ++i) dst[i] = uint8_t(v >> (8 * i));
  return hdr;
}
ZHD int seq_count_write(uint8_t* dst, int32_t nseq) {
  if (nseq < 128) {
    dst[0] = uint8_t(nseq);
    return 1;
  }
  if (nseq < 0x7F00) {
    dst[0] = uint8_t((nseq >> 8) + 128);
    dst[1] = uint8_t(nseq);
    return 2;
  }
  dst[0] = 255;
  dst[1] = uint8_t(nseq - 0x7F00);
  dst[2] = uint8_t((nseq - 0x7F00) >> 8);
  return 3;
}

// ---- one block ------------------------------------------------------------------------------------------------------------------
struct LaneOut {
  int32_t nseq, nlit, tail;  // sequences, literal bytes, literals after the last sequence (all of them when nseq = 0)
};

// Where the block's output is: up to four pieces, concatenated (head | literal streams | mid | sequence stream), or
// head | the block's own bytes for a Raw_Block.
struct BlockOut {
  const uint8_t* p[4];
  int32_t n[4];
};

// Global (device) / heap (host) memory of one block's compression.
struct BlockIo {
  const uint8_t* body;  // the body (= zstd frame content) the block belongs to
  int64_t body_len, off;
  int32_t len;
  bool first, last;
  uint64_t* seqs;      // [kLanes * kLaneSeqs]
  uint8_t* lits;       // [kMaxBlock]
  uint32_t* lstream;   // [kLitStreamCap / 4]
  uint8_t* sstream;    // [kSeqStreamCap]
  uint8_t* head;       // [kHeadCap]
  uint8_t* mid;        // [kMidCap]
  BlockOut* out;
};

// Shared (per CTA) state of one block's compression.
struct BlockShared {
  uint16_t table[kLanes][1 << kHashLog];
  LaneOut lane[kLanes];
  int32_t lit_at[kLanes], carry[kLanes];
  uint32_t hist[256];
  uint8_t sorted[256];
  uint32_t chunk_bits[kLanes];
  uint32_t shist[3][64];
  HufEnc huf;
  FseEnc fse[3];
  int32_t nlit, nseq, last_lits;
  int32_t lit_mode;  // 0 raw, 1 RLE, 2 Huffman
  int32_t streams, tree_len, lit_stream_bytes;
  int32_t stream_bytes[4];
  int32_t all_same;
};

// phase 1, lane l: greedy matches over the lane's range.
ZHD void phase_match(const BlockIo& io, BlockShared& S, int l) {
  const uint8_t* body = io.body;
  const int64_t a = io.off + int64_t(l) * kSpan;
  const int64_t b = a + kSpan < io.off + io.len ? a + kSpan : io.off + io.len;
  LaneOut o{0, 0, 0};
  if (a >= b) {
    S.lane[l] = o;
    return;
  }
  uint16_t* T = S.table[l];
  for (int i = 0; i < (1 << kHashLog); ++i) T[i] = 0;
  const int64_t w0 = a > kSeed ? a - kSeed : 0;
  for (int64_t q = w0; q + 4 <= a; ++q) T[hash4(ld32(body + q))] = uint16_t(q - w0 + 1);
  uint64_t* seqs = io.seqs + int64_t(l) * kLaneSeqs;
  int64_t p = a, anchor = a;
  int n = 0;
  while (p + kMinMatch <= b) {
    const uint32_t v = ld32(body + p);
    const uint32_t h = hash4(v);
    const int64_t c = int64_t(T[h]) - 1 + w0;
    const bool hit = T[h] != 0 && ld32(body + c) == v;
    T[h] = uint16_t(p - w0 + 1);
    if (!hit) {
      p += 1 + ((p - anchor) >> 6);  // skip faster through bytes that keep missing
      continue;
    }
    int64_t s = p, q = c, len = 4;
    while (s + len < b && body[q + len] == body[s + len]) ++len;
    while (s > anchor && q > 0 && body[s - 1] == body[q - 1]) {
      --s;
      --q;
      ++len;
    }
    seqs[n++] = pack_seq(uint32_t(s - anchor), uint32_t(len), uint32_t(s - q + 3));
    o.nlit += int32_t(s - anchor);
    p = s + len;
    anchor = p;
  }
  o.nseq = n;
  o.tail = int32_t(b - anchor);
  o.nlit += o.tail;
  S.lane[l] = o;
}

// phase 2, one lane: literal offsets, literal-length carries between lanes, totals; whether the block is one byte.
ZHD void phase_scan(const BlockIo& io, BlockShared& S) {
  int32_t at = 0, seqs = 0, carry = 0;
  for (int l = 0; l < kLanes; ++l) {
    S.lit_at[l] = at;
    S.carry[l] = carry;
    at += S.lane[l].nlit;
    seqs += S.lane[l].nseq;
    carry = S.lane[l].nseq ? S.lane[l].tail : carry + S.lane[l].tail;
  }
  S.nlit = at;
  S.nseq = seqs;
  S.last_lits = carry;
  S.all_same = io.len > 0;
  S.lit_mode = 0;
  S.streams = 1;
  S.tree_len = 0;
  S.lit_stream_bytes = 0;
  for (int i = 0; i < 256; ++i) S.hist[i] = 0;
  for (int k = 0; k < 3; ++k)
    for (int i = 0; i < 64; ++i) S.shist[k][i] = 0;
}

// phase 3, lane l: the lane's literals into place, the literal histogram, the sequence-code histograms, and whether
// the lane's bytes all equal the block's first.
ZHD void phase_literals(const BlockIo& io, BlockShared& S, int l) {
  const int64_t a = io.off + int64_t(l) * kSpan;
  const int64_t b = a + kSpan < io.off + io.len ? a + kSpan : io.off + io.len;
  if (a >= b) return;
  const uint8_t* body = io.body;
  const uint64_t* seqs = io.seqs + int64_t(l) * kLaneSeqs;
  uint8_t* out = io.lits + S.lit_at[l];
  int64_t p = a;
  const uint8_t b0 = body[io.off];
  bool same = true;
  for (int i = 0; i < S.lane[l].nseq; ++i) {
    const uint64_t q = seqs[i];
    const uint32_t ll = seq_ll(q), ml = seq_ml(q);
    for (uint32_t k = 0; k < ll; ++k) {
      const uint8_t c = body[p + k];
      *out++ = c;
      ZATOMIC_ADD(&S.hist[c], 1u);
      same = same && c == b0;
    }
    for (uint32_t k = 0; k < ml && same; ++k) same = body[p + ll + k] == b0;
    ZATOMIC_ADD(&S.shist[kLL][ll_code(ll + (i == 0 ? uint32_t(S.carry[l]) : 0u))], 1u);
    ZATOMIC_ADD(&S.shist[kML][ml_code(ml)], 1u);
    ZATOMIC_ADD(&S.shist[kOF][of_code(seq_ov(q))], 1u);
    p += ll + ml;
  }
  for (; p < b; ++p) {
    const uint8_t c = body[p];
    *out++ = c;
    ZATOMIC_ADD(&S.hist[c], 1u);
    same = same && c == b0;
  }
  if (!same) S.all_same = 0;  // benign race: every writer writes 0
}

// phase 4, lane l: ranks of the literal symbols (l and l + kLanes).
ZHD void phase_rank(BlockShared& S, int l) {
  for (int s = l; s < 256; s += kLanes)
    if (S.hist[s]) S.sorted[huf_rank(S.hist, s)] = uint8_t(s);
}

// phase 5, one lane: the literal section's form, the Huffman code and tree, the stream split.
ZHD void phase_lit_plan(const BlockIo& io, BlockShared& S) {
  int present = 0;
  for (int s = 0; s < 256; ++s) present += S.hist[s] != 0;
  if (S.nlit == 0 || present < 2) {
    S.lit_mode = S.nlit > 1 ? 1 : 0;
    return;
  }
  HufEnc& H = S.huf;
  huf_lengths(S.hist, S.sorted, present, H.len);
  huf_codes(&H);
  // parked at the end of head, moved in phase 7; the LL table's space is free until then
  S.tree_len = huf_write_tree(H, io.head + kHeadCap - 160, 160, S.fse[kLL]);
  if (S.tree_len < 0) return;
  S.streams = S.nlit <= 1023 ? 1 : 4;
  uint64_t total = 0;
  for (int s = 0; s < 256; ++s) total += uint64_t(S.hist[s]) * H.len[s];
  // stream bytes are only known after the bits per stream are summed; this bound decides whether Huffman can win
  const int64_t est = S.tree_len + int64_t((total + 7) / 8) + (S.streams == 4 ? 6 + 4 : 1) + 5;
  if (est >= int64_t(S.nlit) + 3) return;
  S.lit_mode = 2;
}

// The literal range of stream k and of lane t's chunk inside it (streams of 4: lanes [k * 32, k * 32 + 32)).
ZHD void lit_chunk(const BlockShared& S, int l, int32_t* s_begin, int32_t* s_end, int32_t* c_begin, int32_t* c_end, int* k, int* t, int* per) {
  const int ns = S.streams;
  *per = kLanes / ns;
  *k = l / *per;
  *t = l % *per;
  const int32_t seg = ns == 1 ? S.nlit : (S.nlit + 3) / 4;
  *s_begin = *k * seg;
  *s_end = *k == ns - 1 ? S.nlit : *s_begin + seg;
  const int32_t m = *s_end - *s_begin, chunk = (m + *per - 1) / *per;
  *c_begin = *s_begin + *t * chunk < *s_end ? *s_begin + *t * chunk : *s_end;
  *c_end = *c_begin + chunk < *s_end ? *c_begin + chunk : *s_end;
}

// phase 6a, lane l: bits of the lane's chunk of its Huffman stream.
ZHD void phase_huf_bits(const BlockIo& io, BlockShared& S, int l) {
  if (S.lit_mode != 2) return;
  int32_t sb, se, cb, ce;
  int k, t, per;
  lit_chunk(S, l, &sb, &se, &cb, &ce, &k, &t, &per);
  uint32_t bits = 0;
  for (int32_t i = cb; i < ce; ++i) bits += S.huf.len[io.lits[i]];
  S.chunk_bits[l] = bits;
}

// phase 6b, one lane: stream sizes (each ends with its end mark), whether Huffman still wins; zeroes nothing.
ZHD void phase_huf_sizes(BlockShared& S) {
  if (S.lit_mode != 2) return;
  const int per = kLanes / S.streams;
  int32_t total = 0;
  for (int k = 0; k < S.streams; ++k) {
    uint32_t bits = 0;
    for (int t = 0; t < per; ++t) bits += S.chunk_bits[k * per + t];
    S.stream_bytes[k] = int32_t(bits / 8 + 1);
    total += S.stream_bytes[k];
  }
  const int32_t comp = S.tree_len + (S.streams == 4 ? 6 : 0) + total;
  const int hdr = comp < 1024 && S.nlit < 1024 ? 3 : (comp < 16384 && S.nlit < 16384 ? 4 : 5);
  bool fits = S.streams == 1 ? comp <= 1023 : true;
  for (int k = 0; k < 3 && S.streams == 4; ++k) fits = fits && S.stream_bytes[k] < 65536;
  const int32_t raw = S.nlit + (S.nlit < 32 ? 1 : S.nlit < 4096 ? 2 : 3);
  if (!fits || comp + hdr >= raw) {
    S.lit_mode = 0;
    return;
  }
  S.lit_stream_bytes = total;
}

// phase 6c, lane l: the lane's chunk of its stream, ORed into the zeroed stream words.  Symbol i of a stream of m sits
// at bit sum(len[i+1 .. m)): the stream is written from its last symbol, the decoder reads it from its first.
ZHD void phase_huf_write(const BlockIo& io, BlockShared& S, int l) {
  if (S.lit_mode != 2) return;
  int32_t sb, se, cb, ce;
  int k, t, per;
  lit_chunk(S, l, &sb, &se, &cb, &ce, &k, &t, &per);
  uint64_t bit = 0;
  for (int j = 0; j < k; ++j) bit += uint64_t(S.stream_bytes[j]) * 8;
  for (int u = t + 1; u < per; ++u) bit += S.chunk_bits[k * per + u];
  for (int32_t i = ce - 1; i >= cb; --i) {
    const uint8_t c = io.lits[i];
    or_bits(io.lstream, bit, S.huf.code[c], S.huf.len[c]);
    bit += S.huf.len[c];
  }
  if (t == 0) {  // end mark after the stream's last bit
    uint64_t end = 0;
    for (int j = 0; j < k; ++j) end += uint64_t(S.stream_bytes[j]) * 8;
    for (int u = 0; u < per; ++u) end += S.chunk_bits[k * per + u];
    or_bits(io.lstream, end, 1, 1);
  }
}

// Mode and table of one of LL / OF / ML by estimated cost; writes the description (if any) at d.  Returns the mode.
ZHD int seq_table_plan(const uint32_t* cnt, int which, int32_t nseq, FseEnc* E, uint8_t* d, int cap, int* dlen) {
  const int max_sym = which == kLL ? 35 : which == kOF ? 31 : 52, max_log = which == kOF ? 8 : 9;
  const int16_t* def = which == kLL ? ZD_TAB(ll_def) : which == kOF ? ZD_TAB(of_def) : ZD_TAB(ml_def);
  const int def_n = which == kLL ? 36 : which == kOF ? 29 : 53, def_log = which == kOF ? 5 : 6;
  int present = 0, only = 0, top = 0;
  for (int s = 0; s <= max_sym; ++s)
    if (cnt[s]) {
      ++present;
      only = s;
      top = s;
    }
  *dlen = 0;
  if (present == 1) {  // RLE: one byte, no bits per symbol
    d[0] = uint8_t(only);
    *dlen = 1;
    fse_enc_build(nullptr, 0, 0, only, E);
    return 1;
  }
  int16_t pre[53];
  for (int s = 0; s < def_n; ++s) pre[s] = def[s];
  const uint64_t pre_cost = top < def_n ? fse_cost(cnt, top + 1, pre, def_log) : ~uint64_t(0) >> 1;
  int log = highbit(uint32_t(nseq)) + 1;
  if (log < 5) log = 5;
  while ((1 << log) < 2 * present) ++log;
  if (log > max_log) log = max_log;
  int16_t norm[53];
  fse_normalize(cnt, top + 1, uint32_t(nseq), log, norm);
  const int w = fse_write_counts(norm, top + 1, log, d, cap);
  const uint64_t fse_c = w < 0 ? ~uint64_t(0) >> 1 : fse_cost(cnt, top + 1, norm, log) + uint64_t(w) * 8 * 256;
  if (fse_c < pre_cost) {
    *dlen = w;
    fse_enc_build(norm, top + 1, log, 0, E);
    return 2;
  }
  fse_enc_build(pre, def_n, def_log, 0, E);
  return 0;
}

// phase 7, one lane: the sequences section (tables by cost, the bitstream from the last sequence to the first), the
// literals section header, the block's form and its pieces.
ZHD void phase_finish(const BlockIo& io, BlockShared& S) {
  uint8_t* head = io.head;
  int h = io.first ? frame_header_write(io.body_len, head) : 0;
  const int bh = h;
  h += 3;
  BlockOut& O = *io.out;
  for (int i = 0; i < 4; ++i) {
    O.p[i] = nullptr;
    O.n[i] = 0;
  }
  if (io.len == 0) {
    block_header_write(head + bh, true, 0, 0);
    O.p[0] = head;
    O.n[0] = h;
    return;
  }
  if (S.all_same && io.len > 1) {
    block_header_write(head + bh, io.last, 1, uint32_t(io.len));
    head[h++] = io.body[io.off];
    O.p[0] = head;
    O.n[0] = h;
    return;
  }
  // literals section
  int64_t lit_bytes;
  if (S.lit_mode == 2) {
    const int32_t comp = S.tree_len + (S.streams == 4 ? 6 : 0) + S.lit_stream_bytes;
    h += lit_header_huf(head + h, S.streams, uint32_t(S.nlit), uint32_t(comp));
    const uint8_t* tree = io.head + kHeadCap - 160;
    for (int i = 0; i < S.tree_len; ++i) head[h + i] = tree[i];
    h += S.tree_len;
    if (S.streams == 4)
      for (int k = 0; k < 3; ++k) {
        head[h++] = uint8_t(S.stream_bytes[k]);
        head[h++] = uint8_t(S.stream_bytes[k] >> 8);
      }
    lit_bytes = S.lit_stream_bytes;
  } else if (S.lit_mode == 1) {
    h += lit_header_raw(head + h, 1, uint32_t(S.nlit));
    head[h++] = io.lits[0];
    lit_bytes = 0;
  } else {
    h += lit_header_raw(head + h, 0, uint32_t(S.nlit));
    lit_bytes = S.nlit;
  }
  // sequences section
  uint8_t* mid = io.mid;
  int m = seq_count_write(mid, S.nseq);
  int64_t seq_bytes = 0;
  bool ok = true;
  if (S.nseq > 0) {
    const int modes_at = m++;
    int mode[3];
    for (int k = 0; k < 3; ++k) {
      int dlen = 0;
      mode[k] = seq_table_plan(S.shist[k], k, S.nseq, &S.fse[k], mid + m, kMidCap - m, &dlen);
      m += dlen;
    }
    mid[modes_at] = uint8_t((mode[kLL] << 6) | (mode[kOF] << 4) | (mode[kML] << 2));
    BitOut bo{io.sstream, kSeqStreamCap};
    uint32_t st[3] = {0, 0, 0};
    bool started = false;
    for (int l = kLanes - 1; l >= 0; --l) {
      const uint64_t* seqs = io.seqs + int64_t(l) * kLaneSeqs;
      for (int i = S.lane[l].nseq - 1; i >= 0; --i) {
        const uint64_t q = seqs[i];
        const uint32_t ll = seq_ll(q) + (i == 0 ? uint32_t(S.carry[l]) : 0u), ml = seq_ml(q), ov = seq_ov(q);
        const int lc = ll_code(ll), mc = ml_code(ml), oc = of_code(ov);
        if (!started) {
          st[kLL] = S.fse[kLL].states[S.fse[kLL].first[lc]];
          st[kML] = S.fse[kML].states[S.fse[kML].first[mc]];
          st[kOF] = S.fse[kOF].states[S.fse[kOF].first[oc]];
          started = true;
        } else {
          uint32_t bl, bm, bf;
          int nl, nm, nf;
          st[kLL] = fse_prev_state(S.fse[kLL], lc, st[kLL], &bl, &nl);
          st[kML] = fse_prev_state(S.fse[kML], mc, st[kML], &bm, &nm);
          st[kOF] = fse_prev_state(S.fse[kOF], oc, st[kOF], &bf, &nf);
          bo.put(bf, nf);
          bo.put(bm, nm);
          bo.put(bl, nl);
        }
        bo.put(ll - ZD_TAB(ll_base)[lc], ZD_TAB(ll_bits)[lc]);
        bo.put(ml - ZD_TAB(ml_base)[mc], ZD_TAB(ml_bits)[mc]);
        bo.put(ov - (1u << oc), oc);
      }
    }
    bo.put(st[kML], S.fse[kML].log);
    bo.put(st[kOF], S.fse[kOF].log);
    bo.put(st[kLL], S.fse[kLL].log);
    seq_bytes = bo.close();
    ok = !bo.over;
  }
  const int64_t content = int64_t(h - bh - 3) + lit_bytes + m + seq_bytes;
  if (!ok || content >= io.len) {  // Raw_Block
    h = bh + 3;
    block_header_write(head + bh, io.last, 0, uint32_t(io.len));
    O.p[0] = head;
    O.n[0] = h;
    O.p[1] = io.body + io.off;
    O.n[1] = io.len;
    return;
  }
  block_header_write(head + bh, io.last, 2, uint32_t(content));
  O.p[0] = head;
  O.n[0] = h;
  O.p[1] = S.lit_mode == 0 ? io.lits : reinterpret_cast<const uint8_t*>(io.lstream);
  O.n[1] = int32_t(lit_bytes);
  O.p[2] = mid;
  O.n[2] = m;
  O.p[3] = io.sstream;
  O.n[3] = int32_t(seq_bytes);
}

}  // namespace zstd
}  // namespace fg
