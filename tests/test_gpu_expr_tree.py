"""The tree form of the expression program on the GPU: `filter_compact_kernel<PredTree>` and `expr_eval_kernel`
(csrc/expr_tree.h, csrc/expr_eval.cu) through flockgpu_filter_project and through plans whose aggregates and sorts
take expressions.  The judges are numpy / Arrow compute restatements; tests/test_expr_tree_host.py ties the same
interpreter to a row-at-a-time reference."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import flock_b200 as fb
from flock_b200 import _ffi, col, lit, case, plans

pytestmark = pytest.mark.gpu

SHIPMODES = ["MAIL", "SHIP", "AIR", "RAIL", "TRUCK", "FOB", "REG AIR"]


def relation(n, seed=0, nulls=True):
    rng = np.random.default_rng(seed)
    mask = lambda k: (rng.integers(0, k, n) == 0) if nulls and n else None
    return pa.RecordBatch.from_arrays([
        pa.array(rng.integers(-50, 50, n).astype(np.int32), mask=mask(5)),
        pa.array(rng.integers(-(1 << 40), 1 << 40, n)),
        pa.array(np.round(rng.uniform(900, 100000, n), 2), mask=mask(9)),
        pa.array(rng.integers(0, 11, n) / 100.0),
        pa.array(rng.integers(0, 9, n) / 100.0),
        pa.array([SHIPMODES[k] for k in rng.integers(0, 7, n)], pa.string(), mask=mask(11)),
        pa.array(rng.integers(0, 5, n).astype(np.int32)),
    ], names=["a", "l", "price", "disc", "tax", "mode", "k"])


def launches(ctx, fn):
    ctx.profile_begin()
    out = fn()
    prof = ctx.profile_end()
    return out, {k: v["launches"] for k, v in prof.items()}


@pytest.mark.parametrize("compact_mode", [0, 1])
@pytest.mark.parametrize("n", [0, 1, 65_536, 1_000_003])
@pytest.mark.parametrize("nulls", [False, True])
def test_tree_filter_is_one_launch_and_keeps_the_right_rows(gpu_ctx, n, nulls, compact_mode):
    b = relation(n, seed=n % 97 + nulls, nulls=nulls)
    A, P, M = b.column(0), b.column(2), b.column(5)
    pred = col(5).isin(["MAIL", "SHIP"]) & ((col(0) > 3) | col(2).is_null() | (case([(col(6) == 0, col(1))], otherwise=-col(1)) > 0))
    L, K = b.column(1), b.column(6)
    want_mask = pc.and_kleene(pc.is_in(M, value_set=pa.array(["MAIL", "SHIP"])),
                              pc.or_kleene(pc.or_kleene(pc.greater(A, 3), pc.is_null(P)),
                                           pc.greater(pc.if_else(pc.equal(K, 0), L, pc.negate(L)), 0)))
    want = b.filter(pc.fill_null(want_mask, False))
    gpu_ctx.set_option("compact_mode", compact_mode)
    try:
        t = gpu_ctx.import_batches([b])
        out, prof = launches(gpu_ctx, lambda: gpu_ctx.filter_project(t, pred).to_batch())
    finally:
        gpu_ctx.set_option("compact_mode", 0)
    assert out.num_rows == want.num_rows
    for i in range(b.num_columns):                                 # fixed-width, Utf8 and nullable pass-through columns, in input order
        assert out.column(i).equals(want.column(i)), i
    if n:
        assert prof.get("filter_compact_kernel") == 1 and "expr_eval_kernel" not in prof


@pytest.mark.parametrize("n", [0, 1, 65_536, 1_000_003])
@pytest.mark.parametrize("nulls", [False, True])
def test_tree_projection_is_one_launch_and_bit_exact(gpu_ctx, n, nulls):
    b = relation(n, seed=3 + n % 89, nulls=nulls)
    price, disc, tax = (b.column(i) for i in (2, 3, 4))
    exprs = [col(2) * (1.0 - col(3)) * (1.0 + col(4)),                                       # TPC-H q1's charge
             col(2) * (1.0 - col(3)),
             case([((col(5) == "MAIL") | (col(5) == "SHIP"), lit(1))], otherwise=lit(0)),    # TPC-H q12's CASE
             -col(0),
             col(5),
             col(1) + 1]                                                                     # a chain: keeps its own kernel
    t = gpu_ctx.import_batches([b])
    out, prof = launches(gpu_ctx, lambda: gpu_ctx.filter_project(t, None, exprs, ["charge", "disc_price", "hi", "neg", "mode", "l1"]).to_batch())
    disc_price = pc.multiply(price, pc.subtract(1.0, disc))
    want = [pc.multiply(disc_price, pc.add(1.0, tax)), disc_price,
            pc.if_else(pc.fill_null(pc.or_kleene(pc.equal(b.column(5), "MAIL"), pc.equal(b.column(5), "SHIP")), False), 1, 0),
            pc.negate(b.column(0)), b.column(5), pc.add(b.column(1), 1)]
    assert out.num_rows == n
    for i, w in enumerate(want):
        g = out.column(i)
        assert g.type == w.type, (i, g.type, w.type)
        assert g.null_count == w.null_count
        if pa.types.is_floating(w.type):                           # computed Float64 columns are bit-exact: one rounding per node
            gv, wv = (np.asarray(x.fill_null(0.0)).view(np.int64) for x in (g, w))
            assert np.array_equal(gv, wv) and np.array_equal(np.asarray(g.is_null()), np.asarray(w.is_null())), i
        else:
            assert g.equals(w), i
    if n:
        assert prof.get("expr_eval_kernel") == 1 and prof.get("project_generic_kernel") == 1


def test_filter_with_tree_projection_and_division_by_zero(gpu_ctx):
    b = relation(200_000, seed=11)
    t = gpu_ctx.import_batches([b])
    # the quotient is only taken where the divisor is not zero; rows with k = 0 are dropped by the filter besides
    safe = case([(col(6) != 0, col(1) / col(6).cast("int64"))], otherwise=lit(-1))
    out = gpu_ctx.filter_project(t, col(5).isin(["AIR"]) & (col(6) > 0), [safe, col(5)], ["q", "mode"]).to_batch()
    keep = pc.fill_null(pc.and_kleene(pc.equal(b.column(5), "AIR"), pc.greater(b.column(6), 0)), False)
    kept = b.filter(keep)
    l, k = np.asarray(kept.column(1)), np.asarray(kept.column(6)).astype(np.int64)
    assert np.array_equal(np.asarray(out.column(0)), (np.abs(l) // k) * np.sign(l))     # truncated division
    assert out.column(1).equals(kept.column(5))
    # a division by zero in a row that is evaluated is an execution error, and the context stays usable
    with pytest.raises(fb.FlockGpuError, match="Divide by zero") as info:
        gpu_ctx.filter_project(t, None, [case([(col(6) >= 0, col(1) / col(6).cast("int64"))], otherwise=lit(-1))], ["q"]).to_batch()
    assert info.value.code == _ffi.ERR_EXECUTION
    with pytest.raises(fb.FlockGpuError, match="Divide by zero"):
        gpu_ctx.filter_project(t, (col(1) + col(1)) % (col(6) - 2).cast("int64") * (col(1) - col(1) + 1) == 0).to_batch()
    assert gpu_ctx.filter_project(t, col(6).isin([1, 2])).num_rows == int(np.isin(np.asarray(b.column(6)), [1, 2]).sum())


def test_old_forms_keep_their_kernels(gpu_ctx):
    b = relation(100_000, seed=5, nulls=False)
    t = gpu_ctx.import_batches([b])
    _, prof = launches(gpu_ctx, lambda: gpu_ctx.filter_project(t, None, [(col(1) - 3) * 2], ["x"]).to_batch())
    assert prof.get("project_generic_kernel") == 1 and "expr_eval_kernel" not in prof
    _, prof = launches(gpu_ctx, lambda: gpu_ctx.filter_project(t, (col(5) == "MAIL") | (col(5) == "SHIP"), [col(1)], ["l"]).to_batch())
    assert prof.get("filter_compact_kernel") == 1 and "expr_eval_kernel" not in prof


# ---- expressions inside plan nodes ---------------------------------------------------------------------------------
def _column(b, name):
    return plans.column(name, b.schema.names.index(name))


def _q1_like(b):
    """SELECT k + 1 (computed group key), SUM(price * (1 - disc)), SUM(price * (1 - disc) * (1 + tax)),
    SUM(CASE WHEN mode = 'MAIL' OR mode = 'SHIP' THEN 1 ELSE 0 END), COUNT(*) GROUP BY k + 1"""
    f = lambda v: plans.literal("Float64", v)
    disc_price = plans.binary(_column(b, "price"), "Multiply", plans.binary(f(1.0), "Minus", _column(b, "disc")))
    charge = plans.binary(disc_price, "Multiply", plans.binary(f(1.0), "Plus", _column(b, "tax")))
    hi = plans.case_expr([(plans.binary(plans.binary(_column(b, "mode"), "Eq", plans.literal("Utf8", "MAIL")), "Or",
                                        plans.binary(_column(b, "mode"), "Eq", plans.literal("Utf8", "SHIP"))), plans.literal("Int64", 1))],
                         plans.literal("Int64", 0))
    key = plans.binary(plans.cast(_column(b, "k"), "Int64"), "Plus", plans.literal("Int64", 1))
    aggs = [plans.aggregate_expr("sum", "SUM(disc_price)", disc_price, "Float64"), plans.aggregate_expr("sum", "SUM(charge)", charge, "Float64"),
            plans.aggregate_expr("sum", "SUM(hi)", hi, "Int64"), plans.aggregate_expr("count", "COUNT(UInt8(1))", plans.literal("UInt8", 1), "UInt64")]
    scan = plans.memory_exec(b.schema, None)
    partial = plans.hash_aggregate_exec("Partial", [(key, "k1")], aggs, scan)
    return partial, aggs


def _q1_like_numpy(b):
    price = np.asarray(b.column("price").fill_null(np.nan))
    disc, tax, k = np.asarray(b.column("disc")), np.asarray(b.column("tax")), np.asarray(b.column("k")).astype(np.int64) + 1
    dp = price * (1.0 - disc)
    ch = dp * (1.0 + tax)
    hi = np.asarray(pc.fill_null(pc.is_in(b.column("mode"), value_set=pa.array(["MAIL", "SHIP"])), False)).astype(np.int64)
    out = {}
    for g in np.unique(k):
        m = k == g
        out[int(g)] = (np.nansum(dp[m]), np.nansum(ch[m]), int(hi[m].sum()), int(m.sum()))
    return out


def test_aggregate_over_expressions_single_and_staged(gpu_ctx):
    b = relation(300_000, seed=21)
    partial, aggs = _q1_like(b)
    final_single = plans.hash_aggregate_exec("FinalPartitioned", [(plans.column("k1", 0), "k1")], aggs,
                                             plans.coalesce_batches_exec(plans.repartition_hash(partial, [plans.column("k1", 0)])))
    ec = fb.ExecutionContext(gpu_ctx, final_single)
    s = ec.plan_str()
    assert "gby=[CAST(k@6 AS Int64) + 1 as k1]" in s and "SUM(charge)" in s
    ec.feed_data_sources([[[b]]])
    gpu_ctx.profile_begin()
    single = ec.execute()[0][0]
    prof = gpu_ctx.profile_end()
    assert prof["expr_eval_kernel"]["launches"] == 1               # four computed entries, one launch
    want = _q1_like_numpy(b)

    def check(batch):
        rows = {r["k1"]: r for r in batch.to_pylist()}
        assert sorted(rows) == sorted(want)
        for g, (dp, ch, hi, cnt) in want.items():
            r = rows[g]
            assert r["SUM(hi)"] == hi and r["COUNT(UInt8(1))"] == cnt                     # keys, counts and CASE sums exactly
            n = cnt
            assert abs(r["SUM(disc_price)"] - dp) <= n * np.finfo(np.float64).eps * abs(dp)   # summation-order bound
            assert abs(r["SUM(charge)"] - ch) <= n * np.finfo(np.float64).eps * abs(ch)
    check(single)
    # staged: the Partial plan on its own, its state columns fed to a Final plan
    stage0 = fb.ExecutionContext(gpu_ctx, partial)
    stage0.feed_data_sources([[[b]]])
    states = stage0.execute()[0]
    final = plans.hash_aggregate_exec("Final", [(plans.column("k1", 0), "k1")], aggs, plans.memory_exec(states[0].schema, None))
    stage1 = fb.ExecutionContext(gpu_ctx, final)
    stage1.feed_data_sources([[states]])
    check(stage1.execute()[0][0])


def test_sort_on_an_expression(gpu_ctx):
    b = relation(50_000, seed=31, nulls=False).select(["a", "l", "k"])
    key = plans.binary(plans.binary(plans.cast(plans.column("a", 0), "Int64"), "Multiply", plans.cast(plans.column("k", 2), "Int64")), "Minus",
                       plans.binary(plans.column("l", 1), "Modulo", plans.literal("Int64", 1000)))
    ec = fb.ExecutionContext(gpu_ctx, plans.sort_exec([(key, True, False)], plans.memory_exec(b.schema, None)))
    assert "SortExec: [CAST(a@0 AS Int64) * CAST(k@2 AS Int64) - l@1 % 1000 DESC]" in ec.plan_str()
    ec.feed_data_sources([[[b]]])
    out = ec.execute()[0][0]
    assert out.schema.names == ["a", "l", "k"]                     # the computed key is not part of the output
    a, l, k = (np.asarray(out.column(i)).astype(np.int64) for i in range(3))
    keys = a * k - np.fmod(l, 1000)
    assert np.all(np.diff(keys) <= 0)
    assert sorted(np.asarray(out.column(1)).tolist()) == sorted(np.asarray(b.column(1)).tolist())
