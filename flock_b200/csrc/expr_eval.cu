// expr_eval.cu -- evaluates the computed values of an operator that the chain form cannot express: one launch of
// expr_eval_kernel runs ONE register program (expr_tree.h) with several roots over all rows.
//
// Replaces, per batch, PhysicalExpr::evaluate of every aggregate argument, group / sort key and projection of the
// reference's plans (DataFusion 6 evaluates each expression vector-at-a-time and materialises every intermediate
// array; here the intermediates live in the register file and only the roots are written).
//
// A thread takes four consecutive rows: 16-byte loads of the 4- and 8-byte input columns, 16-byte stores of the
// results, one 4-byte store of their validity bytes.  Traffic = each input column the program reads, once, plus the
// outputs written: the kernel is bound by HBM as long as the program is short.
#include <algorithm>

#include "expr_compile.h"
#include "internal.h"

namespace fg {

constexpr int EV_THREADS = 128;
constexpr int EV_ROWS = 4;

struct EvalArgs {
  int64_t n_rows;
  int* err_flag;
  ColRef cols[MAX_IN_COLS];
  TreeOut outs[TREE_MAX_OUTS];
  TreeProgram prog;
};

__global__ void __launch_bounds__(EV_THREADS) expr_eval_kernel(const __grid_constant__ EvalArgs a) {
  // the register file: [register][row][thread]
  __shared__ Val reg_val[TREE_REGS * EV_ROWS * EV_THREADS];
  __shared__ uint8_t reg_flag[TREE_REGS * EV_ROWS * EV_THREADS];
  const TreeRegs<EV_ROWS, EV_THREADS> regs{reg_val + threadIdx.x, reg_flag + threadIdx.x};
  int err = 0;
  const int64_t stride = int64_t(gridDim.x) * EV_THREADS * EV_ROWS;
  for (int64_t base = (int64_t(blockIdx.x) * EV_THREADS + threadIdx.x) * EV_ROWS; base < a.n_rows; base += stride) {
    int64_t rows[EV_ROWS];
#pragma unroll
    for (int j = 0; j < EV_ROWS; ++j) rows[j] = base + j < a.n_rows ? base + j : -1;
    eval_tree<EV_ROWS>(a.prog, a.cols, a.outs, rows, base + EV_ROWS <= a.n_rows, regs, &err);
  }
  if (err) *a.err_flag = 1;
}

std::vector<Column> eval_exprs(const CtxPtr& ctx, const Table& in, const std::vector<Expr>& exprs, const std::vector<std::string>& names) {
  in.dense();
  const std::vector<ColInfo> infos = col_infos(in);
  const CompiledTree ct = compile_tree_values(exprs, infos);
  auto args = std::make_unique<EvalArgs>();
  memset(args.get(), 0, sizeof(EvalArgs));
  args->n_rows = in.num_rows;
  args->err_flag = reinterpret_cast<int*>(ctx->d_scalars + 8);
  args->prog = ct.prog;
  filter_colrefs(in, args->cols);
  std::vector<Column> out;
  for (size_t i = 0; i < exprs.size(); ++i) {
    const TreeRoot& r = ct.roots[i];
    Column c;
    if (r.passthrough) {
      c = in.cols[r.src_col];  // shares the input's buffers
    } else {
      c.dtype = r.dtype;
      c.format = r.format;
      c.length = in.num_rows;
      c.data = alloc(ctx, size_t(in.num_rows) * dtype_width(r.dtype));
      if (r.may_be_null) {
        c.validity = alloc(ctx, size_t(std::max<int64_t>(in.num_rows, 1)));
        c.nullable = true;
      }
      TreeOut& o = args->outs[r.out];
      o.dst = c.data->ptr;
      o.validity = c.validity ? c.validity->as<uint8_t>() : nullptr;
      o.dtype = r.dtype;
    }
    c.name = i < names.size() && !names[i].empty() ? names[i] : (r.passthrough ? c.name : expr_to_string(exprs[i], infos));
    out.push_back(std::move(c));
  }
  if (ct.n_outs == 0 || in.num_rows == 0) return out;
  if (ct.may_fail) FG_CUDA(cudaMemsetAsync(args->err_flag, 0, sizeof(int), ctx->stream));
  const int64_t per_block = int64_t(EV_THREADS) * EV_ROWS;
  const int resident = resident_ctas(ctx, reinterpret_cast<const void*>(&expr_eval_kernel), EV_THREADS);
  const int grid = int(std::min<int64_t>((in.num_rows + per_block - 1) / per_block, int64_t(std::max(resident, 1))));
  {
    LaunchTimer lt(ctx, "expr_eval_kernel");
    expr_eval_kernel<<<grid, EV_THREADS, 0, ctx->stream>>>(*args);
  }
  FG_CUDA(cudaGetLastError());
  count_launch(ctx);
  if (ct.may_fail) {
    unsigned long long flag = 0;
    read_scalars(ctx, 8, 1, &flag);
    FG_CHECK((flag & 0xffffffffull) == 0, FLOCKGPU_ERR_EXECUTION, "Divide by zero");
  }
  return out;
}

}  // namespace fg
