// selftest.cc -- host-side checks of the expression COMPILER (expr_compile.cc) without a GPU.
//
// flockgpu_selftest_* run the very same term/chain programs the kernels interpret (expr_program.h is
// __host__ __device__) over HOST Arrow buffers, one row at a time.  They exist so that `pytest -m "not
// gpu"` can verify the lowering of DataFusion expressions on a CPU-only box.  They are NOT an execution
// path: no operator, plan node or Python wrapper calls them, and they handle one expression, not plans.
#include "expr_compile.h"
#include "internal.h"
#include "pred_i32.h"
#include "zstd_dec.h"

using namespace fg;

namespace {

struct HostBatch {
  std::vector<ColInfo> infos;
  std::vector<ColRef> refs;
  std::vector<std::vector<uint8_t>> validity;  // byte per row, like Column::validity on the device (reserved up front: refs point into it)
  int64_t rows = 0;
};

HostBatch view_batch(const ArrowSchema* schema, const ArrowArray* batch) {
  FG_CHECK(schema && batch && schema->format && !strcmp(schema->format, "+s"), FLOCKGPU_ERR_INVALID, "selftest: need a struct batch");
  HostBatch hb;
  hb.rows = batch->length;
  hb.validity.reserve(size_t(schema->n_children));
  for (int64_t c = 0; c < schema->n_children; ++c) {
    const ArrowSchema* cs = schema->children[c];
    const ArrowArray* a = batch->children[c];
    int dt = dtype_from_format(cs->format);
    FG_CHECK(dt >= 0, FLOCKGPU_ERR_UNSUPPORTED, "selftest: unsupported column format %s", cs->format);
    ColInfo info{dt, cs->name ? cs->name : "", cs->format};
    ColRef r{};
    r.dtype = dt;
    int64_t off = batch->offset + a->offset;
    if (a->null_count != 0 && a->buffers[0]) {  // the bitmap as the import path expands it: one byte per row
      const uint8_t* bits = static_cast<const uint8_t*>(a->buffers[0]);
      std::vector<uint8_t> v(size_t(std::max<int64_t>(hb.rows, 1)));
      bool any_null = false;
      for (int64_t i = 0; i < hb.rows; ++i) {
        v[size_t(i)] = (bits[(off + i) >> 3] >> ((off + i) & 7)) & 1u;
        any_null |= !v[size_t(i)];
      }
      if (any_null) {
        hb.validity.push_back(std::move(v));
        r.validity = hb.validity.back().data();
        info.has_nulls = true;
      }
    }
    hb.infos.push_back(info);
    if (dt == FLOCKGPU_UTF8) {
      r.offsets = static_cast<const int32_t*>(a->buffers[1]) + off;
      r.data = a->buffers[2];
    } else {
      r.data = static_cast<const char*>(a->buffers[1]) + off * dtype_width(dt);
    }
    hb.refs.push_back(r);
  }
  return hb;
}

}  // namespace

extern "C" {

// Evaluates `predicate` over a host record batch with the device interpreter compiled for the host.
// out_mask[rows] receives 0/1; *out_fast_kind (may be NULL) the specialised kernel shape that would run
// on the GPU (0 = generic interpreter, 1 = i32 % m CMP c, 2 = i32 CMP c).
int flockgpu_selftest_eval_predicate(const struct ArrowSchema* schema, const struct ArrowArray* batch, const flockgpu_expr* predicate,
                                     uint8_t* out_mask, int32_t* out_fast_kind) {
  return guarded([&] {
    HostBatch hb = view_batch(schema, batch);
    CompiledPredicate cp = compile_predicate(tokens_to_expr(predicate), hb.infos);
    if (out_fast_kind) *out_fast_kind = cp.fast.kind;
    int err = 0;
    for (int64_t r = 0; r < hb.rows; ++r) {
      int64_t rows[1] = {r};
      out_mask[r] = uint8_t(eval_predicate<1>(cp.prog, hb.refs.data(), rows, &err) & 1u);
    }
    FG_CHECK(!err, FLOCKGPU_ERR_EXECUTION, "Divide by zero");
  });
}

// Evaluates a value expression; `out` must hold rows * 8 bytes (4-byte types are written packed).
// *out_dtype receives the flockgpu_dtype of the result, *out_passthrough 1 if it is a plain column.  Compiled as a
// pure projection compiles it: what this accepts, a ProjectionExec over the same columns runs in the chain form.
int flockgpu_selftest_eval_value(const struct ArrowSchema* schema, const struct ArrowArray* batch, const flockgpu_expr* expr, void* out,
                                 int32_t* out_dtype, int32_t* out_passthrough) {
  return guarded([&] {
    HostBatch hb = view_batch(schema, batch);
    CompiledValue cv = compile_value(tokens_to_expr(expr), hb.infos, PROJECT_MAX_NULL_INPUTS);
    if (out_dtype) *out_dtype = cv.dtype;
    if (out_passthrough) *out_passthrough = cv.passthrough ? 1 : 0;
    if (cv.passthrough) return;
    int err = 0;
    for (int64_t r = 0; r < hb.rows; ++r) {
      int64_t rows[1] = {r};
      Val acc[1];
      eval_chain<1>(cv.chain, hb.refs.data(), rows, acc, &err);
      store_val(out, cv.dtype, r, acc[0]);
    }
    FG_CHECK(!err, FLOCKGPU_ERR_EXECUTION, "Divide by zero");
  });
}

// The tree form: all of `exprs` as ONE register program (or exprs[0] as a predicate), run by eval_tree compiled for the
// host with a private register file.
int flockgpu_selftest_eval_tree(const struct ArrowSchema* schema, const struct ArrowArray* batch, const flockgpu_expr* exprs, int32_t n_exprs,
                                int32_t predicate, void* const* out_values, uint8_t* const* out_valid, int32_t* out_dtypes,
                                int32_t* out_passthrough, int32_t* out_n_instr) {
  return guarded([&] {
    FG_CHECK(exprs && n_exprs >= 1 && out_values && (!predicate || n_exprs == 1), FLOCKGPU_ERR_INVALID, "selftest_eval_tree: bad arguments");
    HostBatch hb = view_batch(schema, batch);
    std::vector<Expr> es;
    for (int i = 0; i < n_exprs; ++i) es.push_back(tokens_to_expr(&exprs[i]));
    const CompiledTree ct = predicate ? compile_tree_predicate(es[0], hb.infos) : compile_tree_values(es, hb.infos);
    if (out_n_instr) *out_n_instr = ct.prog.n_instr;
    std::vector<TreeOut> outs(TREE_MAX_OUTS);
    if (!predicate) {
      FG_CHECK(out_valid && out_dtypes && out_passthrough, FLOCKGPU_ERR_INVALID, "selftest_eval_tree: bad arguments");
      for (int i = 0; i < n_exprs; ++i) {
        const TreeRoot& r = ct.roots[size_t(i)];
        out_dtypes[i] = r.dtype;
        out_passthrough[i] = r.passthrough ? 1 : 0;
        if (r.passthrough) continue;
        memset(out_valid[i], 1, size_t(hb.rows));
        outs[size_t(r.out)] = TreeOut{out_values[i], r.may_be_null ? out_valid[i] : nullptr, r.dtype, 0};
      }
    }
    Val reg_val[TREE_REGS];
    uint8_t reg_flag[TREE_REGS];
    const TreeRegs<1, 1> regs{reg_val, reg_flag};
    int err = 0;
    for (int64_t r = 0; r < hb.rows; ++r) {
      int64_t rows[1] = {r};
      const unsigned keep = eval_tree<1>(ct.prog, hb.refs.data(), outs.data(), rows, false, regs, &err);
      if (predicate) static_cast<uint8_t*>(out_values[0])[r] = uint8_t(keep & 1u);
    }
    FG_CHECK(!err, FLOCKGPU_ERR_EXECUTION, "Divide by zero");
  });
}

}  // extern "C"

// The vectorised predicate `CAST(x AS Int64) [% modulus] cmp rhs` (modulus = 0: no `%`) exactly as the filter kernel
// evaluates it: same constants (pred_i32_consts), same per-row test (pred_i32_test), on the host.  out_mode receives the
// arithmetic shape chosen (0 affine range test, 1 Lemire fastmod, 2 rotate test for even moduli).
int flockgpu_selftest_pred_i32(int64_t modulus, int32_t cmp, int64_t rhs, const int32_t* x, int64_t n, uint8_t* out_keep, int32_t* out_mode) {
  return guarded([&] {
    FG_CHECK(x && out_keep && n >= 0 && modulus >= 0 && modulus < (int64_t(1) << 31), FLOCKGPU_ERR_INVALID, "selftest_pred_i32: bad arguments");
    PredI32Consts k;
    const int mode = pred_i32_consts(modulus, cmp, rhs, &k);
    if (out_mode) *out_mode = mode;
    for (int64_t i = 0; i < n; ++i)
      out_keep[i] = mode == 0 ? pred_i32_test<0>(k, x[i]) : mode == 1 ? pred_i32_test<1>(k, x[i]) : pred_i32_test<2>(k, x[i]);
  });
}

// The zstd decoder of the payload import (zstd_dec.h) run serially on the host: what CPU CI compares byte for byte with
// another implementation.
int flockgpu_selftest_zstd_decompress(const uint8_t* src, int64_t src_len, uint8_t* dst, int64_t capacity, int64_t* out_len) {
  return guarded([&] {
    FG_CHECK(src_len >= 0 && (src || src_len == 0) && capacity >= 0 && (dst || capacity == 0) && out_len, FLOCKGPU_ERR_INVALID,
             "selftest_zstd_decompress: bad arguments");
    std::vector<uint8_t> out;
    const int e = zstd_decode_host(src, src_len, capacity, &out);
    FG_CHECK(!e, e == zstd::Z_DICTIONARY ? FLOCKGPU_ERR_UNSUPPORTED : FLOCKGPU_ERR_INVALID, "selftest_zstd_decompress: %s", zstd::error_name(e));
    if (!out.empty()) memcpy(dst, out.data(), out.size());
    *out_len = int64_t(out.size());
  });
}

// The zstd encoder of the payload export (zstd_enc.h) run serially on the host: the bytes the GPU gives for the same
// input, which CPU CI decompresses with another implementation.
int flockgpu_selftest_zstd_compress(const uint8_t* src, int64_t src_len, uint8_t* dst, int64_t capacity, int64_t* out_len) {
  return guarded([&] {
    FG_CHECK(src_len >= 0 && (src || src_len == 0) && capacity >= 0 && (dst || capacity == 0) && out_len, FLOCKGPU_ERR_INVALID,
             "selftest_zstd_compress: bad arguments");
    std::vector<uint8_t> out;
    zstd_compress_host(src, src_len, &out);
    FG_CHECK(int64_t(out.size()) <= capacity, FLOCKGPU_ERR_INVALID, "selftest_zstd_compress: %zu compressed bytes, capacity %lld", out.size(), (long long)capacity);
    memcpy(dst, out.data(), out.size());
    *out_len = int64_t(out.size());
  });
}
