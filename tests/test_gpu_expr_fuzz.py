"""The expression programs on the GPU against two judges, over edge values, at every tile shape and tail.

Every result of a kernel is compared (a) with the host build of the same program (`selftest_eval_tree`,
`selftest_eval_value`, `selftest_eval_predicate`) over every row, bit for bit: Float64 by bits (NaN as "is NaN"),
validity exactly, "Divide by zero" raised or not; this sees what exists only on the device (16-byte loads and stores,
the shared-memory register file, the CUDA conversion intrinsics, the error flag of a grid).  And (b), through (a), with
`ref_eval`, the row-at-a-time reference of tests/test_expr_tree_host.py: the host results the GPU is held to equal the
reference over a fixed sample of rows (the first and last 8, 4 either side of every multiple of 1024 up to 8192, the
edge blocks, 2000 random rows); this sees what the two builds share.

The relation (`edge_relation`) draws ~30 % of every column from its edge pool and repeats one edge block at the start,
in the middle and in the last rows.  The trees come from `random_tree(..., edges=True)`; each runs alone, with the
others in one projection, as a predicate under both compaction modes and as a predicate with a tree projection."""
import functools

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import flock_b200 as fb
from flock_b200 import _ffi, col, lit, case, plans
from test_expr_tree_host import (DivideByZero, EDGE_BLOCK, I32_MAX, I32_MIN, I64_MAX, I64_MIN, edge_relation, random_tree, ref_eval,
                                 run_tree, same)

pytestmark = pytest.mark.gpu

SEEDS = [42, 7, 1234]
SMALL = [0, 1, 3, 4, 5, 1023, 1025, 8191, 8193]


@functools.lru_cache(None)
def large_rows():
    """From here the filter takes 16 rows per thread (PredTreeT<16>, PredGenericT<16>): the size rule of filter_project."""
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * 4 * 256 * 16


def rows_of(size):
    return size if isinstance(size, int) else large_rows() + (1 if size == "large+1" else -1)


@functools.lru_cache(2)
def relation(n, seed, nulls):
    return edge_relation(n, seed, nulls)


def sample_rows(n, seed):
    rng = np.random.default_rng(seed)
    s = set(range(min(8, n))) | set(range(max(n - 8, 0), n))
    for m in range(1024, 8193, 1024):
        s |= set(range(max(m - 4, 0), min(m + 4, n)))
    for start in {0, (n // 2) & ~3, max(n - EDGE_BLOCK, 0)}:
        s |= set(range(start, min(start + EDGE_BLOCK, n)))
    if n:
        s |= set(rng.integers(0, n, 2000).tolist())
    return np.array(sorted(s), dtype=np.int64)


def feeds(ctx, b):
    """The relation as one batch and as ragged batches (1, 3, 1000, ... rows)."""
    yield ctx.import_batches([b])
    n = b.num_rows
    if n > 1:
        cuts = sorted({0, n} | {c for c in (1, 4, 1004, n // 3, n - 2) if 0 < c < n})
        yield ctx.import_batches([b.slice(s, e - s) for s, e in zip(cuts, cuts[1:])])


def profiled(ctx, fn):
    ctx.profile_begin()
    try:
        out = fn()
    finally:
        prof = ctx.profile_end()
    return out, {k: v["launches"] for k, v in prof.items()}


def column_np(arr):
    """(values, valid) of a fixed-width column as numpy, values in the storage type."""
    arr = arr.combine_chunks() if isinstance(arr, pa.ChunkedArray) else arr
    dt = {pa.int32(): np.int32, pa.uint32(): np.uint32, pa.date32(): np.int32, pa.uint64(): np.uint64, pa.float64(): np.float64}.get(arr.type, np.int64)
    vals = np.frombuffer(arr.buffers()[1], dt, len(arr) + arr.offset)[arr.offset:] if len(arr) else np.zeros(0, dt)
    return vals, ~arr.is_null().to_numpy(zero_copy_only=False)


def assert_bits(gv, gvalid, hv, hvalid, what):
    assert len(gv) == len(hv), what
    assert np.array_equal(gvalid, hvalid), (what, np.flatnonzero(gvalid != hvalid)[:8])
    if gv.dtype == np.float64:
        ok = (gv.view(np.int64) == hv.view(np.int64)) | (np.isnan(gv) & np.isnan(hv))
    else:
        ok = gv == hv
    bad = np.flatnonzero(~ok & hvalid)
    assert len(bad) == 0, (what, bad[:8], gv[bad[:4]], hv[bad[:4]])


def assert_same_rows(out, want, what):
    """Every pass-through column exactly: same rows, in input order, same bits, same NULLs."""
    assert out.num_rows == want.num_rows, what
    for i, f in enumerate(want.schema):
        assert_same_column(out.column(i), want.column(i), (what, f.name))


def assert_same_column(g, w, what):
    assert g.type == w.type, what
    if w.type == pa.string():
        assert g.equals(w), what
    else:
        assert_bits(*column_np(g), *column_np(w), what)


def raises_div0(fn):
    with pytest.raises(fb.FlockGpuError, match="Divide by zero") as info:
        fn()
    assert info.value.code == _ffi.ERR_EXECUTION


def chain_compiles(b, e, predicate):
    """A filter or pure projection over `b` runs `e` in the term / chain form (when it cannot, the operators take the
    tree form).  The whole of `b`: which columns have NULLs decides it."""
    try:
        (fb.selftest_eval_predicate if predicate else fb.selftest_eval_value)(b, e)
        return True
    except fb.FlockGpuError as err:
        return err.code != _ffi.ERR_UNSUPPORTED


def draw_trees(rng, b, count, kind_of):
    """`count` trees the compiler takes, each with its host result over `b`; trees over the register or instruction
    budget are refused by name and counted."""
    out, refused = [], 0
    while len(out) < count:
        kind = kind_of(len(out))
        e = random_tree(rng, int(rng.integers(2, 6)), kind, edges=True)
        status, res = run_tree(b, e, kind)
        if status == "refused":
            refused += 1
            continue
        out.append((e, kind, status, res))
    assert refused <= count, refused
    return out


def reference_on(bs, e):
    try:
        return ref_eval(e, bs)
    except DivideByZero:
        return None


@pytest.mark.parametrize("size", SMALL + ["large-1", "large+1"])
@pytest.mark.parametrize("seed", SEEDS)
def test_random_trees_in_every_role(gpu_ctx, seed, size):
    n = rows_of(size)
    large = not isinstance(size, int)
    b = relation(n, seed + n, [0, 7, -1][(seed + n) % 3])
    sample = sample_rows(n, seed)
    bs = b.take(sample)
    rng = np.random.default_rng(seed * 7919 + n)
    count = 4 if large else 10
    values = draw_trees(rng, b, count, lambda k: ("int", "float")[k % 2])
    preds = draw_trees(rng, b, count, lambda k: "bool")

    # judge (b) for the host results the GPU is compared with below: on the sample, host and reference agree
    for e, kind, status, res in values + preds:
        want = reference_on(bs, e)
        if status == "raised":
            continue                                       # (the zero divisor may lie outside the sample)
        assert want is not None, e.tokens
        if kind == "bool":
            assert list(res[sample]) == [w is True for w in want], e.tokens
        elif res[0] is not None:
            same(res[0][sample], res[1][sample], want, res[2])

    # ---- a projection of one tree, and of all of them in one program
    tree_only = []
    for e, kind, status, res in values:
        chain = chain_compiles(b, e, False)
        for t in feeds(gpu_ctx, b):
            if status == "raised":
                raises_div0(lambda: gpu_ctx.filter_project(t, None, [e], ["v"]).to_batch())
                continue
            out, prof = profiled(gpu_ctx, lambda: gpu_ctx.filter_project(t, None, [e], ["v"]).to_batch())
            if res[0] is None:
                assert_same_column(out.column(0), b.column(e.tokens[0][2]), e.tokens)   # a plain column passes through
                continue
            assert_bits(*column_np(out.column(0)), res[0], res[1], e.tokens)
            if n:
                chain_kernels = sum(prof.get(k, 0) for k in ("project_generic_kernel", "project_i32_to_f64_mul_kernel"))
                assert (chain_kernels == 1 and "expr_eval_kernel" not in prof) if chain else (chain_kernels == 0 and prof.get("expr_eval_kernel") == 1), \
                    (chain, e.tokens, prof)
        if status == "ok" and res[0] is not None and not chain:
            tree_only.append((e, res))
    for k in range(0, len(tree_only), 4):
        group = tree_only[k:k + 4]
        for t in feeds(gpu_ctx, b):
            try:
                out, prof = profiled(gpu_ctx, lambda: gpu_ctx.filter_project(t, None, [e for e, _ in group]).to_batch())
            except fb.FlockGpuError as err:                # the roots together exceed the program's budget
                assert err.code == _ffi.ERR_UNSUPPORTED and ("registers" in err.message or "instructions" in err.message), err
                continue
            for i, (e, res) in enumerate(group):
                assert_bits(*column_np(out.column(i)), res[0], res[1], e.tokens)
            if n:
                assert prof.get("expr_eval_kernel") == 1, prof  # several roots, one launch

    # ---- predicates, alone (all columns pass through) and with a tree projection (survivors first, then the tree)
    project = [e for e, _ in tree_only[:2]] or [-col(1) * case([(col(0) > 0, col(6))], otherwise=lit(2))]
    for e, kind, status, res in preds:
        want_rows = None if status == "raised" else b.filter(pa.array(res))
        for mode in (0, 1):
            gpu_ctx.set_option("compact_mode", mode)
            try:
                for t in feeds(gpu_ctx, b):
                    if want_rows is None:
                        raises_div0(lambda: gpu_ctx.filter_project(t, e).to_batch())
                        continue
                    out, prof = profiled(gpu_ctx, lambda: gpu_ctx.filter_project(t, e).to_batch())
                    assert_same_rows(out, want_rows, (mode, e.tokens))
                    if n:
                        assert prof.get("filter_compact_kernel") == 1 and "expr_eval_kernel" not in prof, prof
            finally:
                gpu_ctx.set_option("compact_mode", 0)
        if want_rows is None:
            continue
        v = project[len(want_rows) % len(project)]
        status_v, res_v = run_tree(want_rows, v, "int")
        for t in feeds(gpu_ctx, b):
            if status_v == "raised":
                raises_div0(lambda: gpu_ctx.filter_project(t, e, [v, col(5), col(10)]).to_batch())
                continue
            out = gpu_ctx.filter_project(t, e, [v, col(5), col(10)]).to_batch()
            assert_bits(*column_np(out.column(0)), res_v[0], res_v[1], (e.tokens, v.tokens))
            assert out.column(1).equals(want_rows.column(5)) and out.column(2).equals(want_rows.column(10))


# ---- the chain and term forms over the same relation --------------------------------------------------------------------
CHAIN_VALUES = [0.908 * col(0).cast("float64"), (col(1) + 5) * 3, col(1) * 3 - lit(I64_MIN), (col(1) + lit(I64_MAX)) / col(6).cast("int64"),
                col(1) % col(6).cast("int64"), lit(I64_MIN) / col(6).cast("int64"), col(0) * col(6), col(0) + lit(I32_MAX, "int32"),
                col(2) + lit(1 << 63, "uint64"), col(8).cast("int64") * 7, col(3) * 2.5 - col(1).cast("float64"), col(2).cast("float64") / col(3)]
CHAIN_PREDS = [(col(5) == "MAIL") | (col(5) == "SHIP"), (col(1) + 5) * 3 > col(0).cast("int64"), col(3) < 0.1, (col(1) - lit(I64_MIN)) % 7 == 0,
               col(2) > lit((1 << 63) + 1, "uint64"), ~(col(3) >= col(7))]
I32_PREDS = [getattr(col(0).cast("int64") % m, op)(c) for m in (1, 7, 123, (1 << 31) - 1) for c in (I32_MIN, -1, 0) for op in ("__eq__", "__lt__", "__ge__")]


@pytest.mark.parametrize("size", [1, 5, 1025, 8193, "large-1", "large+1"])
def test_chain_and_term_forms(gpu_ctx, size):
    n = rows_of(size)
    b = relation(n, 99 + n, 0)
    sample = sample_rows(n, 5)
    bs = b.take(sample)
    t = gpu_ctx.import_batches([b])
    for e in CHAIN_VALUES:
        host, dt = fb.selftest_eval_value(b, e)
        same(host[sample], np.ones(len(sample), bool), ref_eval(e, bs), dt)
        out, prof = profiled(gpu_ctx, lambda: gpu_ctx.filter_project(t, None, [e], ["v"]).to_batch())
        assert_bits(*column_np(out.column(0)), host, np.ones(n, bool), e.tokens)
        assert "expr_eval_kernel" not in prof and prof.get("project_generic_kernel", prof.get("project_i32_to_f64_mul_kernel")) == 1, (e.tokens, prof)
    for e, vectorised in [(e, False) for e in CHAIN_PREDS] + [(e, True) for e in I32_PREDS[(n % 3)::3]]:
        mask, fast = fb.selftest_eval_predicate(b, e)
        assert list(mask[sample]) == [w is True for w in ref_eval(e, bs)], e.tokens
        assert (fast != 0) == vectorised, e.tokens                 # CAST(i32 AS Int64) [% m] CMP c: the vectorised PredI32
        for mode in (0, 1):
            gpu_ctx.set_option("compact_mode", mode)
            try:
                out, prof = profiled(gpu_ctx, lambda: gpu_ctx.filter_project(t, e, [col(10), col(0), col(5), 0.5 * col(1).cast("float64")]).to_batch())
            finally:
                gpu_ctx.set_option("compact_mode", 0)
            assert np.array_equal(column_np(out.column(0))[0], np.flatnonzero(mask)), (mode, e.tokens)
            kept = b.filter(pa.array(mask))
            assert out.column(1).equals(kept.column(0)) and out.column(2).equals(kept.column(5))
            assert_bits(*column_np(out.column(3)), 0.5 * column_np(kept.column(1))[0].astype(np.float64), np.ones(len(kept), bool), e.tokens)
            assert prof.get("filter_compact_kernel") == 1 and "expr_eval_kernel" not in prof, prof


def test_lossy_casts_take_the_tree_form(gpu_ctx):
    """A CAST that can give NULL is refused by the chain and term forms, which have no NULLs of their own: projections
    and filters evaluate it in the tree form, NULL where the target type cannot hold the value."""
    b = relation(8193, 3, 7)
    t = gpu_ctx.import_batches([b])
    for e in ((col(3) * 2.5).cast("int64"), col(3).cast("uint64") + 1, col(1).cast("int32"), col(2).cast("int64") - col(1)):
        assert not chain_compiles(b, e, False) and not chain_compiles(b, e > 0, True), e.tokens
        (v, valid, _), = fb.selftest_eval_tree(b, [e])[0]
        assert not valid.all()                                         # some value of the edge relation does not fit
        out, prof = profiled(gpu_ctx, lambda: gpu_ctx.filter_project(t, None, [e]).to_batch())
        assert_bits(*column_np(out.column(0)), v, valid, e.tokens)
        assert prof.get("expr_eval_kernel") == 1 and "project_generic_kernel" not in prof, prof
        p = e > 0
        mask, _ = fb.selftest_eval_tree(b, p, predicate=True)
        out = gpu_ctx.filter_project(t, p, [col(10), e]).to_batch()
        assert np.array_equal(column_np(out.column(0))[0], np.flatnonzero(mask)), p.tokens
        assert_bits(*column_np(out.column(1)), v[mask], valid[mask], p.tokens)


# ---- page-locked batches read in place: densified before a tree or generic predicate -----------------------------------
def test_host_resident_batches_are_densified(gpu_ctx):
    n = 5 * 8192 + 77
    b = relation(n, 11, 0)
    pinned = [gpu_ctx.pinned_copy(b.take(np.arange(s, min(s + 8192, n)))) for s in range(0, n, 8192)]   # buffers of their own
    C = lambda name: plans.column(name, b.schema.names.index(name))
    i64 = lambda v: plans.literal("Int64", v)
    # CASE WHEN a > 0 THEN l ELSE -1 END > 0 (tree form); s = 'MAIL' OR l > 0 (term form)
    tree_pred = plans.binary(plans.case_expr([(plans.binary(C("a"), "Gt", plans.literal("Int32", 0)), C("l"))], i64(-1)), "Gt", i64(0))
    term_pred = plans.binary(plans.binary(C("s"), "Eq", plans.literal("Utf8", "MAIL")), "Or", plans.binary(C("l"), "Gt", i64(0)))
    value = plans.case_expr([(plans.binary(C("z"), "Lt", plans.literal("Int32", 0)), plans.binary(C("l"), "Divide", plans.cast(C("z"), "Int64")))], i64(7))
    E_preds = [case([(col(0) > 0, col(1))], otherwise=lit(-1)) > 0, (col(5) == "MAIL") | (col(1) > 0)]
    E_value = case([(col(6) < 0, col(1) / col(6).cast("int64"))], otherwise=lit(7))
    gpu_ctx.set_option("feed_zero_copy", 1)
    try:
        for pred, e in zip((tree_pred, term_pred), E_preds):
            ec = fb.ExecutionContext(gpu_ctx, plans.projection_exec([(C("rid"), "rid"), (value, "v"), (C("s"), "s")],
                                                                     plans.filter_exec(pred, plans.memory_exec(b.schema, None))))
            ec.feed_data_sources([fb.HostRelation(pinned)])
            got = pa.Table.from_batches(ec.execute()[0])
            ec.close()
            mask, _ = fb.selftest_eval_tree(b, e, predicate=True)
            kept = b.filter(pa.array(mask))
            (v, valid, _), = fb.selftest_eval_tree(kept, [E_value])[0]
            assert np.array_equal(got["rid"].to_numpy(), np.flatnonzero(mask))
            assert_bits(*column_np(got["v"]), v, valid, "v")
            assert got["s"].combine_chunks().equals(kept.column(5))
    finally:
        gpu_ctx.set_option("feed_zero_copy", 0)


# ---- division by zero: raised exactly where the reference raises, and the context stays usable -------------------------
def divisor_relation(n, zero_at, drop=(), null=()):
    rng = np.random.default_rng(n)
    z = rng.choice([3, -1, 7, I32_MIN], n).astype(np.int32)
    z[list(zero_at)] = 0
    k = np.ones(n, np.int32)
    k[list(drop)] = 0
    mask = np.zeros(n, bool)
    mask[list(null)] = True
    return pa.RecordBatch.from_arrays([pa.array(rng.integers(-(1 << 62), 1 << 62, n)), pa.array(z, mask=mask if len(null) else None), pa.array(k),
                                       pa.array(np.arange(n))], names=["l", "z", "k", "rid"])


QUOTIENT = col(0) / col(1).cast("int64")                                      # chain form
GUARDED = case([(col(2) != 0, col(0) / col(1).cast("int64"))], otherwise=lit(-1))   # tree form: the CASE skips k = 0
TREE_QUOTIENT = case([(col(2) >= 0, col(0) % col(1))], otherwise=lit(-1))      # tree form, Int64 % Int32


@pytest.mark.parametrize("where", ["last row", "last tile", "dropped row", "under a NULL", "untaken branch"])
def test_division_by_zero_placement(gpu_ctx, where):
    n = 8193 if where != "last tile" else large_rows() + 1
    r = {"last row": n - 1, "last tile": n - 100}.get(where, n // 2 + 1)
    b = divisor_relation(n, [r], drop=[r] if where in ("dropped row", "untaken branch") else (), null=[r] if where == "under a NULL" else ())
    t = gpu_ctx.import_batches([b])
    sample = sample_rows(n, 1)
    for e in (QUOTIENT, GUARDED, TREE_QUOTIENT):
        raises = reference_on(b.take([r]), e) is None
        assert reference_on(b.take(sample[sample != r]), e) is not None
        if where == "dropped row":
            # filter first: the row with the zero divisor is gone before the value is computed
            out = gpu_ctx.filter_project(t, col(2) != 0, [e, col(3)]).to_batch()
            kept = b.filter(pc.not_equal(b.column(2), 0))
            (v, valid, _), = fb.selftest_eval_tree(kept, [e])[0]
            assert_bits(*column_np(out.column(0)), v, valid, where)
            continue
        if raises:
            raises_div0(lambda: gpu_ctx.filter_project(t, None, [e]).to_batch())
            raises_div0(lambda: gpu_ctx.filter_project(t, e > 0).to_batch())
        else:
            (v, valid, _), = fb.selftest_eval_tree(b, [e])[0]
            assert_bits(*column_np(gpu_ctx.filter_project(t, None, [e]).to_batch().column(0)), v, valid, where)
            mask, _ = fb.selftest_eval_tree(b, e > 0, predicate=True)
            assert gpu_ctx.filter_project(t, e > 0).num_rows == int(mask.sum())
        # the next call on the same context is right
        safe = case([(col(1) != 0, col(0) / col(1).cast("int64"))], otherwise=lit(0))
        (v, valid, _), = fb.selftest_eval_tree(b, [safe])[0]
        assert_bits(*column_np(gpu_ctx.filter_project(t, None, [safe]).to_batch().column(0)), v, valid, "after")
    assert where not in ("last row", "last tile") or raises


def test_a_null_divisor_raises_nothing(gpu_ctx):
    """Regression: a division that the chain or term form can express, over a column with NULLs, used to divide in the
    NULL rows too and raise "Divide by zero" for the 0 stored under a NULL.  It is NULL there (the tree form)."""
    n = 5000
    zeros_under_nulls = pa.array(np.where(np.arange(n) % 3 == 0, 5, 0).astype(np.int32), mask=np.arange(n) % 3 != 0)
    only_nulls = pa.array(np.zeros(n, np.int32), mask=np.ones(n, bool))
    b = pa.RecordBatch.from_arrays([pa.array(np.arange(n) - 2500), zeros_under_nulls, only_nulls], names=["l", "z", "n"])
    t = gpu_ctx.import_batches([b])
    for e in (col(0) / col(1).cast("int64"), col(0) % col(2), col(0) + col(2), case([(col(2) > 1, col(0))], otherwise=lit(3))):
        (v, valid, _), = fb.selftest_eval_tree(b, [e])[0]
        assert_bits(*column_np(gpu_ctx.filter_project(t, None, [e]).to_batch().column(0)), v, valid, e.tokens)
    for p in (col(0) / col(1).cast("int64") > 0, (col(0) % col(2) == 0) | (col(0) > 2000)):
        mask, _ = fb.selftest_eval_tree(b, p, predicate=True)
        out = gpu_ctx.filter_project(t, p, [col(0)]).to_batch()
        assert np.array_equal(column_np(out.column(0))[0], np.asarray(b.column(0))[mask]), p.tokens
