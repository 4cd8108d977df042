// ndjson.cu -- newline-delimited JSON events -> a device table: the parse step in front of the hot path.
//
// Reference: `event_bytes_to_batch(events, schema, batch_size)` (flock/src/transmute.rs:255-266) runs arrow's
// schema-driven `json::Reader` over the serde_json lines of the NEXMark generator (one flat object per event, e.g.
// {"auction":1000,"bidder":1001,"price":5000,"b_date_time":1436918400000}; call sites flock/src/datasource/nexmark/
// nexmark.rs:181-203 -- q1's stated purpose is "parse speed").  Semantics restated here: fields are found BY NAME (any
// order), fields the schema does not list are skipped (nested values included), integers must be JSON integers in
// range, strings are unescaped (\" \\ \/ \b \f \n \r \t \uXXXX with surrogate pairs) and arrive as UTF-8.  Without
// validity bitmaps on this path a missing field or a JSON null is an error, like any malformed line.
//
//   ndjson_lines_kernel   positions of the '\n' bytes: single-pass stable compaction (compact.cuh), 64 bytes per thread
//   ndjson_parse_kernel   one thread per line, twice: pass 0 writes the fixed-width values and the unescaped LENGTH of
//                         every string, pass 1 (after the exclusive scans that turn lengths into Arrow offsets) the
//                         string bytes
#include <algorithm>

#include "compact.cuh"
#include "device_utils.cuh"
#include "expr_program.h"
#include "internal.h"

namespace fg {

constexpr int NJ_MAX_COLS = MAX_IN_COLS;
constexpr int NJ_NAME_POOL = 512;

struct NdLinesArgs {
  CompactScratch sc;
  const uint8_t* data;
  int64_t n_bytes;
  uint32_t* nl_pos;  // byte index of every '\n', ascending
};

__global__ void __launch_bounds__(CP_THREADS) ndjson_lines_kernel(const __grid_constant__ NdLinesArgs a) {
  constexpr int E = 4, I = 64, G = I / E, TILE = CP_THREADS * I;
  __shared__ CompactSmem<E, I> sm;
  const int tid = threadIdx.x;
  long long tile;
  for (int it = 0; (tile = cp_next_tile(sm, a.sc, it)) >= 0; ++it) {
    const int64_t tile_base = tile * TILE;
    unsigned long long bits = 0;
#pragma unroll
    for (int g = 0; g < G; ++g) {
      const int64_t b0 = tile_base + (int64_t(g) * CP_THREADS + tid) * E;
      unsigned w = 0;
      if (b0 + 3 < a.n_bytes) {
        w = *reinterpret_cast<const unsigned*>(a.data + b0);  // the buffer is 4-byte aligned (own allocation)
      } else {
        for (int e = 0; e < 4; ++e)
          if (b0 + e < a.n_bytes) w |= unsigned(a.data[b0 + e]) << (8 * e);
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) bits |= (unsigned long long)(b0 + e < a.n_bytes && ((w >> (8 * e)) & 0xffu) == '\n') << (g * E + e);
    }
    unsigned lane_prefix[G];
    cp_rank_tile<E, I>(sm, a.sc, tile, bits, lane_prefix);
    if (bits && sm.tile_total) {
      unsigned long long m = bits;
      while (m) {
        const int k = __ffsll((long long)m) - 1;
        m &= m - 1;
        a.nl_pos[cp_position<E, I>(sm, bits, k, lane_prefix)] = uint32_t(tile_base + cp_item_index<E>(k, tid));
      }
    }
    __syncthreads();
  }
}

struct NdParseArgs {
  const uint8_t* data;
  int64_t n_bytes, n_rows;
  const uint32_t* nl_pos;  // [n_newlines]; row r spans (nl_pos[r - 1], nl_pos[r]) -- or up to n_bytes for an unterminated last line
  int64_t n_newlines;
  int32_t n_cols, pass;
  int32_t dtype[NJ_MAX_COLS];
  int32_t name_off[NJ_MAX_COLS], name_len[NJ_MAX_COLS];
  char names[NJ_NAME_POOL];
  void* values[NJ_MAX_COLS];     // fixed width: value array; Utf8: value bytes (pass 1)
  int32_t* offsets[NJ_MAX_COLS];  // Utf8: pass 0 writes the LENGTH of row r to offsets[r]; pass 1 reads the scanned offsets
  unsigned long long* error;      // first bad line + 1 (atomicMin), ~0 = none;  error[1] = reason of that line
};

enum NdError : int { ND_SYNTAX = 1, ND_MISSING = 2, ND_NULL = 3, ND_TYPE = 4, ND_RANGE = 5, ND_DUPLICATE = 6, ND_FLOAT = 7 };

struct Cursor {
  const uint8_t* p;
  const uint8_t* end;
  __device__ __forceinline__ void ws() {
    while (p < end && (*p == ' ' || *p == '\t' || *p == '\r')) ++p;
  }
  __device__ __forceinline__ bool eat(uint8_t c) {
    ws();
    if (p < end && *p == c) {
      ++p;
      return true;
    }
    return false;
  }
};

__device__ __forceinline__ int hex_val(uint8_t c) {
  if (c >= '0' && c <= '9') return c - '0';
  if (c >= 'a' && c <= 'f') return c - 'a' + 10;
  if (c >= 'A' && c <= 'F') return c - 'A' + 10;
  return -1;
}

// Reads a JSON string (the cursor stands behind the opening quote); writes the unescaped bytes to `out` when it is not
// NULL; returns the unescaped length or -1 on malformed input.  The cursor ends behind the closing quote.
__device__ int read_string(Cursor& c, uint8_t* out) {
  int n = 0;
  auto emit = [&](unsigned b) {
    if (out) out[n] = uint8_t(b);
    ++n;
  };
  auto emit_cp = [&](unsigned cp) {
    if (cp < 0x80) {
      emit(cp);
    } else if (cp < 0x800) {
      emit(0xC0 | (cp >> 6));
      emit(0x80 | (cp & 0x3F));
    } else if (cp < 0x10000) {
      emit(0xE0 | (cp >> 12));
      emit(0x80 | ((cp >> 6) & 0x3F));
      emit(0x80 | (cp & 0x3F));
    } else {
      emit(0xF0 | (cp >> 18));
      emit(0x80 | ((cp >> 12) & 0x3F));
      emit(0x80 | ((cp >> 6) & 0x3F));
      emit(0x80 | (cp & 0x3F));
    }
  };
  while (c.p < c.end) {
    const uint8_t ch = *c.p++;
    if (ch == '"') return n;
    if (ch != '\\') {
      emit(ch);
      continue;
    }
    if (c.p >= c.end) return -1;
    const uint8_t e = *c.p++;
    switch (e) {
      case '"': emit('"'); break;
      case '\\': emit('\\'); break;
      case '/': emit('/'); break;
      case 'b': emit('\b'); break;
      case 'f': emit('\f'); break;
      case 'n': emit('\n'); break;
      case 'r': emit('\r'); break;
      case 't': emit('\t'); break;
      case 'u': {
        auto hex4 = [&](unsigned* v) {
          if (c.end - c.p < 4) return false;
          unsigned x = 0;
          for (int i = 0; i < 4; ++i) {
            const int h = hex_val(c.p[i]);
            if (h < 0) return false;
            x = x * 16 + unsigned(h);
          }
          c.p += 4;
          *v = x;
          return true;
        };
        unsigned cp;
        if (!hex4(&cp)) return -1;
        if (cp >= 0xD800 && cp < 0xDC00) {  // high surrogate: a low one must follow
          unsigned lo;
          if (c.end - c.p < 6 || c.p[0] != '\\' || c.p[1] != 'u') return -1;
          c.p += 2;
          if (!hex4(&lo) || lo < 0xDC00 || lo >= 0xE000) return -1;
          cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00);
        } else if (cp >= 0xDC00 && cp < 0xE000) {
          return -1;
        }
        emit_cp(cp);
        break;
      }
      default: return -1;
    }
  }
  return -1;  // no closing quote on this line
}

// Skips one JSON value of any shape (nested containers included).  Returns false on malformed input.
__device__ bool skip_value(Cursor& c) {
  int depth = 0;
  while (true) {
    c.ws();
    if (c.p >= c.end) return false;
    const uint8_t ch = *c.p;
    if (ch == '"') {
      ++c.p;
      if (read_string(c, nullptr) < 0) return false;
    } else if (ch == '{' || ch == '[') {
      ++depth;
      ++c.p;
      continue;
    } else if (ch == '}' || ch == ']') {
      if (depth == 0) return false;
      --depth;
      ++c.p;
    } else if (ch == ',' || ch == ':') {
      if (depth == 0) return false;
      ++c.p;
      continue;
    } else {
      // number / true / false / null: up to the next structural character
      while (c.p < c.end && *c.p != ',' && *c.p != '}' && *c.p != ']' && *c.p != ':' && *c.p != ' ' && *c.p != '\t' && *c.p != '\r') ++c.p;
    }
    if (depth == 0) return true;
  }
}

// A JSON integer into [lo, hi] (as signed 64-bit; UInt64 columns pass hi = -1 and are range-checked as unsigned).
__device__ int read_integer(Cursor& c, bool is_unsigned64, long long lo, long long hi, unsigned long long* out) {
  c.ws();
  bool neg = false;
  if (c.p < c.end && *c.p == '-') {
    neg = true;
    ++c.p;
  }
  if (c.p >= c.end || *c.p < '0' || *c.p > '9') return (c.p < c.end && (*c.p == 'n')) ? ND_NULL : ND_TYPE;
  unsigned long long v = 0;
  int digits = 0;
  while (c.p < c.end && *c.p >= '0' && *c.p <= '9') {
    const unsigned d = *c.p - '0';
    if (v > (~0ull - d) / 10) return ND_RANGE;
    v = v * 10 + d;
    ++c.p;
    ++digits;
  }
  if (c.p < c.end && (*c.p == '.' || *c.p == 'e' || *c.p == 'E')) return ND_TYPE;  // not an integer literal
  if (is_unsigned64) {
    if (neg && v != 0) return ND_RANGE;
    *out = v;
    return 0;
  }
  if (neg) {
    if (v > 0x8000000000000000ull) return ND_RANGE;
    const long long s = v == 0x8000000000000000ull ? (long long)0x8000000000000000ull : -(long long)v;
    if (s < lo) return ND_RANGE;
    *out = (unsigned long long)s;
  } else {
    if (v > (unsigned long long)hi) return ND_RANGE;
    *out = v;
  }
  return 0;
}

// A JSON number into a double, exactly, for the inputs where one IEEE operation suffices (<= 15 significant digits and
// a decimal exponent within +-22: mantissa and power of ten are both exact doubles); anything longer is refused.
__device__ int read_double(Cursor& c, double* out) {
  c.ws();
  bool neg = false;
  if (c.p < c.end && *c.p == '-') {
    neg = true;
    ++c.p;
  }
  if (c.p >= c.end || !((*c.p >= '0' && *c.p <= '9'))) return (c.p < c.end && *c.p == 'n') ? ND_NULL : ND_TYPE;
  unsigned long long m = 0;
  int sig = 0, exp10 = 0;
  bool seen_nonzero = false;
  while (c.p < c.end && *c.p >= '0' && *c.p <= '9') {
    if (*c.p != '0') seen_nonzero = true;
    if (seen_nonzero) ++sig;
    if (sig > 15) return ND_FLOAT;
    m = m * 10 + unsigned(*c.p - '0');
    ++c.p;
  }
  if (c.p < c.end && *c.p == '.') {
    ++c.p;
    if (c.p >= c.end || *c.p < '0' || *c.p > '9') return ND_SYNTAX;
    while (c.p < c.end && *c.p >= '0' && *c.p <= '9') {
      if (*c.p != '0') seen_nonzero = true;
      if (seen_nonzero) ++sig;
      if (sig > 15) return ND_FLOAT;
      m = m * 10 + unsigned(*c.p - '0');
      --exp10;
      ++c.p;
    }
  }
  if (c.p < c.end && (*c.p == 'e' || *c.p == 'E')) {
    ++c.p;
    bool eneg = false;
    if (c.p < c.end && (*c.p == '+' || *c.p == '-')) {
      eneg = *c.p == '-';
      ++c.p;
    }
    if (c.p >= c.end || *c.p < '0' || *c.p > '9') return ND_SYNTAX;
    int e = 0;
    while (c.p < c.end && *c.p >= '0' && *c.p <= '9') {
      if (e < 10000) e = e * 10 + (*c.p - '0');
      ++c.p;
    }
    exp10 += eneg ? -e : e;
  }
  if (m == 0) {
    *out = neg ? -0.0 : 0.0;
    return 0;
  }
  if (exp10 < -22 || exp10 > 22) return ND_FLOAT;
  const double p10[23] = {1e0, 1e1, 1e2, 1e3, 1e4, 1e5, 1e6, 1e7, 1e8, 1e9, 1e10, 1e11, 1e12, 1e13, 1e14, 1e15, 1e16, 1e17, 1e18, 1e19, 1e20, 1e21, 1e22};
  double v = __ull2double_rn(m);
  v = exp10 >= 0 ? __dmul_rn(v, p10[exp10]) : __ddiv_rn(v, p10[-exp10]);
  *out = neg ? -v : v;
  return 0;
}

__global__ void __launch_bounds__(128) ndjson_parse_kernel(const __grid_constant__ NdParseArgs a) {
  for (int64_t row = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; row < a.n_rows; row += int64_t(gridDim.x) * blockDim.x) {
    const int64_t begin = row == 0 ? 0 : int64_t(a.nl_pos[row - 1]) + 1;
    const int64_t end = row < a.n_newlines ? int64_t(a.nl_pos[row]) : a.n_bytes;
    Cursor c{a.data + begin, a.data + end};
    int err = 0;
    unsigned seen = 0;
    if (!c.eat('{')) err = ND_SYNTAX;
    bool first = true;
    while (!err) {
      if (c.eat('}')) break;
      if (!first && !c.eat(',')) {
        err = ND_SYNTAX;
        break;
      }
      first = false;
      if (!c.eat('"')) {
        err = ND_SYNTAX;
        break;
      }
      // the key: compared with the schema's names while it is read (keys with escapes match nothing and are skipped)
      const uint8_t* k0 = c.p;
      if (read_string(c, nullptr) < 0) {
        err = ND_SYNTAX;
        break;
      }
      const int klen = int(c.p - 1 - k0);
      int col = -1;
      for (int i = 0; i < a.n_cols && col < 0; ++i) {
        if (a.name_len[i] != klen) continue;
        bool same = true;
        for (int b = 0; b < klen && same; ++b) same = uint8_t(a.names[a.name_off[i] + b]) == k0[b];
        if (same) col = i;
      }
      if (!c.eat(':')) {
        err = ND_SYNTAX;
        break;
      }
      if (col < 0) {
        if (!skip_value(c)) err = ND_SYNTAX;
        continue;
      }
      if (seen & (1u << col)) {
        err = ND_DUPLICATE;
        break;
      }
      seen |= 1u << col;
      const int dt = a.dtype[col];
      if (dt == FLOCKGPU_UTF8) {
        c.ws();
        if (c.p >= c.end || *c.p != '"') {
          err = (c.p < c.end && *c.p == 'n') ? ND_NULL : ND_TYPE;
          break;
        }
        ++c.p;
        uint8_t* dst = a.pass == 1 ? static_cast<uint8_t*>(a.values[col]) + a.offsets[col][row] : nullptr;
        const int n = read_string(c, dst);
        if (n < 0) {
          err = ND_SYNTAX;
          break;
        }
        if (a.pass == 0) a.offsets[col][row] = n;
      } else if (dt == FLOCKGPU_FLOAT64) {
        double v = 0;
        err = read_double(c, &v);
        if (!err && a.pass == 0) static_cast<double*>(a.values[col])[row] = v;
      } else {
        unsigned long long v = 0;
        const bool u64 = dt == FLOCKGPU_UINT64;
        const long long lo = dt == FLOCKGPU_INT32 ? -2147483648ll : dt == FLOCKGPU_UINT32 ? 0ll : (long long)0x8000000000000000ull;
        const long long hi = dt == FLOCKGPU_INT32 ? 2147483647ll : dt == FLOCKGPU_UINT32 ? 4294967295ll : 0x7fffffffffffffffll;
        err = read_integer(c, u64, lo, hi, &v);
        if (!err && a.pass == 0) {
          if (dt == FLOCKGPU_INT32 || dt == FLOCKGPU_UINT32) static_cast<uint32_t*>(a.values[col])[row] = uint32_t(v);
          else static_cast<unsigned long long*>(a.values[col])[row] = v;
        }
      }
    }
    if (!err) {
      c.ws();
      if (c.p != c.end) err = ND_SYNTAX;                                     // trailing bytes behind the object
      else if (seen != (a.n_cols >= 32 ? ~0u : (1u << a.n_cols) - 1u)) err = ND_MISSING;
    }
    if (err && a.pass == 0) {
      // make sure pass 1 finds sane lengths even on bad lines (the host raises before it would run anyway)
      for (int i = 0; i < a.n_cols; ++i)
        if (a.dtype[i] == FLOCKGPU_UTF8 && !(seen & (1u << i))) a.offsets[i][row] = 0;
      const unsigned long long tag = (unsigned long long)(row + 1);
      if (atomicMin(a.error, tag) > tag) a.error[1] = (unsigned long long)err;  // racy only between bad lines: any reason of a bad line will do
    }
  }
}

// in place: lengths -> exclusive offsets, offsets[n] = total (the grid-wide prefix of compact.cuh over tiles of 2048 rows)
constexpr int NS_ITEMS = 8;
constexpr int NS_TILE = CP_THREADS * NS_ITEMS;
struct NdScanArgs {
  CompactScratch sc;  // sc.out_count receives the total
  int32_t* off;
  int64_t n;
};

__global__ void __launch_bounds__(CP_THREADS) ndjson_offsets_kernel(const __grid_constant__ NdScanArgs a) {
  __shared__ CompactSmem<1, 16> sm;
  __shared__ unsigned long long s_warp[CP_WARPS];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  long long tile;
  for (int it = 0; (tile = cp_next_tile(sm, a.sc, it)) >= 0; ++it) {
    const int64_t i0 = tile * NS_TILE + int64_t(tid) * NS_ITEMS;
    unsigned len[NS_ITEMS];
    unsigned long long local = 0;
#pragma unroll
    for (int k = 0; k < NS_ITEMS; ++k) {
      len[k] = i0 + k < a.n ? unsigned(a.off[i0 + k]) : 0u;
      local += len[k];
    }
    const unsigned long long incl = warp_inclusive_sum(local);
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    unsigned long long warp_base = 0, tile_total = 0;
#pragma unroll
    for (int w = 0; w < CP_WARPS; ++w) {
      const unsigned long long v = s_warp[w];
      if (w < warp) warp_base += v;
      tile_total += v;
    }
    if (a.sc.single_wave) cp_grid_prefix(sm, a.sc, tile, tile_total);
    else cp_block_lookback(sm, a.sc, tile, tile_total);
    unsigned long long run = sm.excl + warp_base + (incl - local);
#pragma unroll
    for (int k = 0; k < NS_ITEMS; ++k) {
      if (i0 + k < a.n) a.off[i0 + k] = int32_t(run);
      run += len[k];
    }
    if (tile == a.sc.num_tiles - 1 && tid == 0) a.off[a.n] = int32_t(sm.excl + tile_total);
    __syncthreads();
  }
}

static const char* nd_reason(unsigned long long r) {
  switch (int(r)) {
    case ND_MISSING: return "a field of the schema is missing";
    case ND_NULL: return "null value (no validity bitmaps on this path)";
    case ND_TYPE: return "value of the wrong JSON type";
    case ND_RANGE: return "integer out of range for the column type";
    case ND_DUPLICATE: return "duplicate key";
    case ND_FLOAT: return "number with more than 15 significant digits or an exponent beyond +-22 (not exactly representable by one IEEE operation)";
    default: return "malformed JSON";
  }
}

TablePtr import_ndjson(const CtxPtr& ctx, const ArrowSchema* schema, const uint8_t* data, int64_t n_bytes) {
  FG_CHECK(schema && schema->format && !strcmp(schema->format, "+s"), FLOCKGPU_ERR_INVALID, "table_import_ndjson: schema must be a struct (\"+s\")");
  FG_CHECK(n_bytes >= 0 && (n_bytes == 0 || data), FLOCKGPU_ERR_INVALID, "table_import_ndjson: bad buffer");
  FG_CHECK(n_bytes < (int64_t(1) << 32) - 1, FLOCKGPU_ERR_UNSUPPORTED, "table_import_ndjson: more than 4 GiB of text in one call");
  const int n_cols = int(schema->n_children);
  FG_CHECK(n_cols >= 1 && n_cols <= std::min(NJ_MAX_COLS, 31), FLOCKGPU_ERR_UNSUPPORTED, "table_import_ndjson: 1..%d columns", std::min(NJ_MAX_COLS, 31));
  NdParseArgs pa{};
  pa.n_cols = n_cols;
  int pool = 0;
  auto t = std::make_shared<Table>();
  t->ctx = ctx;
  for (int c = 0; c < n_cols; ++c) {
    const ArrowSchema* cs = schema->children[c];
    const int dt = dtype_from_format(cs->format);
    // Date32 in NDJSON (date strings) is not parsed
    FG_CHECK(dt >= 0 && dt != FLOCKGPU_BOOL && dt != FLOCKGPU_DATE32, FLOCKGPU_ERR_UNSUPPORTED, "table_import_ndjson: column \"%s\" has unsupported Arrow format \"%s\"", cs->name ? cs->name : "",
             cs->format ? cs->format : "");
    const int len = int(strlen(cs->name ? cs->name : ""));
    FG_CHECK(pool + len <= NJ_NAME_POOL, FLOCKGPU_ERR_UNSUPPORTED, "table_import_ndjson: field names exceed %d bytes", NJ_NAME_POOL);
    memcpy(pa.names + pool, cs->name ? cs->name : "", size_t(len));
    pa.name_off[c] = pool;
    pa.name_len[c] = len;
    pa.dtype[c] = dt;
    pool += len;
    Column col;
    col.dtype = dt;
    col.name = cs->name ? cs->name : "";
    col.format = cs->format;
    col.nullable = (cs->flags & ARROW_FLAG_NULLABLE) != 0;
    t->cols.push_back(std::move(col));
  }
  if (schema->metadata) {
    // raw Arrow metadata block: int32 n, then n x (int32 klen, key, int32 vlen, value)
    const char* p = schema->metadata;
    int32_t n;
    memcpy(&n, p, 4);
    p += 4;
    for (int32_t i = 0; i < n; ++i)
      for (int k = 0; k < 2; ++k) {
        int32_t l;
        memcpy(&l, p, 4);
        p += 4 + l;
      }
    t->metadata.assign(schema->metadata, size_t(p - schema->metadata));
  }
  // ---- text to HBM (pageable or page-locked source: one copy)
  BufferPtr text = alloc(ctx, size_t(n_bytes) + 16);
  if (n_bytes) {
    ctx->h2d_bytes.fetch_add(n_bytes, std::memory_order_relaxed);
    FG_CUDA(cudaMemcpyAsync(text->ptr, data, size_t(n_bytes), cudaMemcpyHostToDevice, ctx->stream));
  }
  // ---- line ends
  BufferPtr nl = alloc(ctx, size_t(n_bytes) * 4 + 16);  // worst case: every byte is a newline
  unsigned long long n_newlines = 0;
  if (n_bytes) {
    NdLinesArgs la{};
    la.data = text->as<uint8_t>();
    la.n_bytes = n_bytes;
    la.nl_pos = nl->as<uint32_t>();
    const long long tiles = (n_bytes + CP_THREADS * 64 - 1) / (CP_THREADS * 64);
    la.sc = prepare_compact(ctx, tiles, resident_ctas(ctx, reinterpret_cast<const void*>(ndjson_lines_kernel), CP_THREADS), ctx->d_scalars + 13);
    {
      LaunchTimer lt(ctx, "ndjson_lines_kernel");
      launch_compact(ctx, ndjson_lines_kernel, la.sc, la);
    }
    FG_CUDA(cudaGetLastError());
    count_launch(ctx);
    read_scalars(ctx, 13, 1, &n_newlines);  // also: the host buffer has been consumed (inputs are borrowed for the call)
  }
  // rows: one per newline, plus an unterminated last line if the text does not end in '\n'
  bool open_tail = false;
  if (n_bytes) {
    uint8_t last = 0;
    memcpy(&last, data + n_bytes - 1, 1);
    open_tail = last != '\n';
  }
  const int64_t n_rows = int64_t(n_newlines) + (open_tail ? 1 : 0);
  t->num_rows = n_rows;
  for (int c = 0; c < n_cols; ++c) {
    Column& col = t->cols[size_t(c)];
    col.length = n_rows;
    if (col.dtype == FLOCKGPU_UTF8) {
      col.offsets = alloc(ctx, size_t(n_rows + 1) * 4);
      pa.offsets[c] = col.offsets->as<int32_t>();
      if (n_rows == 0) FG_CUDA(cudaMemsetAsync(col.offsets->ptr, 0, 4, ctx->stream));
    } else {
      col.data = alloc(ctx, size_t(n_rows) * col.width());
      pa.values[c] = col.data->ptr;
    }
  }
  if (n_rows == 0) {
    for (Column& col : t->cols)
      if (col.dtype == FLOCKGPU_UTF8) col.data = alloc(ctx, 0);
    return t;
  }
  pa.data = text->as<uint8_t>();
  pa.n_bytes = n_bytes;
  pa.n_rows = n_rows;
  pa.nl_pos = nl->as<uint32_t>();
  pa.n_newlines = int64_t(n_newlines);
  pa.error = ctx->d_scalars + 14;  // [14] first bad line + 1, [15] its reason
  FG_CUDA(cudaMemsetAsync(pa.error, 0xff, 8, ctx->stream));
  FG_CUDA(cudaMemsetAsync(pa.error + 1, 0, 8, ctx->stream));
  const int grid = int(std::max<int64_t>(1, std::min<int64_t>((n_rows + 127) / 128, int64_t(ctx->sm_count) * 16)));
  pa.pass = 0;
  {
    LaunchTimer lt(ctx, "ndjson_parse_kernel");
    ndjson_parse_kernel<<<grid, 128, 0, ctx->stream>>>(pa);
  }
  FG_CUDA(cudaGetLastError());
  count_launch(ctx);
  // ---- string lengths -> offsets
  std::vector<int> utf8;
  for (int c = 0; c < n_cols; ++c)
    if (t->cols[size_t(c)].dtype == FLOCKGPU_UTF8) utf8.push_back(c);
  FG_CHECK(utf8.size() <= 16, FLOCKGPU_ERR_UNSUPPORTED, "table_import_ndjson: more than 16 Utf8 columns");
  for (size_t u = 0; u < utf8.size(); ++u) {
    NdScanArgs sa{};
    sa.off = pa.offsets[utf8[u]];
    sa.n = n_rows;
    const long long tiles = (n_rows + NS_TILE - 1) / NS_TILE;
    sa.sc = prepare_compact(ctx, tiles, resident_ctas(ctx, reinterpret_cast<const void*>(ndjson_offsets_kernel), CP_THREADS), ctx->d_scalars + 16 + u);
    {
      LaunchTimer lt(ctx, "ndjson_offsets_kernel");
      launch_compact(ctx, ndjson_offsets_kernel, sa.sc, sa);
    }
    FG_CUDA(cudaGetLastError());
    count_launch(ctx);
  }
  unsigned long long st[18] = {};
  read_scalars(ctx, 14, 2 + int(utf8.size()), st);
  if (st[0] != ~0ull)
    fail(FLOCKGPU_ERR_EXECUTION, "table_import_ndjson: line %llu: %s", st[0], nd_reason(st[1]));
  if (!utf8.empty()) {
    for (size_t u = 0; u < utf8.size(); ++u) {
      Column& col = t->cols[size_t(utf8[u])];
      FG_CHECK(st[2 + u] < (1ull << 31), FLOCKGPU_ERR_UNSUPPORTED, "table_import_ndjson: Utf8 column \"%s\" exceeds 2^31-1 bytes", col.name.c_str());
      col.values_bytes = int64_t(st[2 + u]);
      col.data = alloc(ctx, size_t(st[2 + u]));
      pa.values[utf8[u]] = col.data->ptr;
    }
    pa.pass = 1;
    {
      LaunchTimer lt(ctx, "ndjson_parse_kernel");
      ndjson_parse_kernel<<<grid, 128, 0, ctx->stream>>>(pa);
    }
    FG_CUDA(cudaGetLastError());
    count_launch(ctx);
  }
  return t;
}

}  // namespace fg

using namespace fg;

extern "C" int flockgpu_table_import_ndjson(flockgpu_ctx* ctx, const struct ArrowSchema* schema, const uint8_t* data, int64_t n_bytes, flockgpu_table** out) {
  return guarded([&] {
    auto c = core_of(ctx);
    FG_CHECK(out, FLOCKGPU_ERR_INVALID, "table_import_ndjson: null out pointer");
    std::lock_guard<std::recursive_mutex> g(c->mu);
    FG_CUDA(cudaSetDevice(c->device));
    TablePtr t = import_ndjson(c, schema, data, n_bytes);
    FG_CUDA(cudaStreamSynchronize(c->stream));  // `text` and `nl` are released in stream order; the caller's buffer was consumed earlier
    *out = wrap_table(t);
  });
}
