"""HashJoinExec { join_type: Semi / Anti } on the GPU (`-m gpu`), against `ref_semi`, a plain set-of-keys reference.

Semantics: the output is the left input's rows, each at most once, in left order, with the left schema.  Semi keeps a
left row when some right row has an equal key tuple, Anti keeps exactly the others.  Key equality is the inner join's
(test_gpu_join_edges): a tuple with a NULL or NaN component matches nothing, so such a left row is never in Semi and
always in Anti; Float64 components compare by bits otherwise.  Unlike key types are refused.

The joins run as plans over two memory_exec leaves.  The smaller side is hashed: with the left side hashed,
`semi_mark_kernel` marks the slots the right rows find before `semi_select_kernel` runs; with the right side hashed only
`semi_select_kernel` runs.  Each test names the orientation it expects and checks it in the launch profile."""
import numpy as np
import pyarrow as pa
import pytest

import flock_b200 as fb
from flock_b200 import plans
from test_gpu_join_edges import (ERR_UNSUPPORTED, KEY_KINDS, MULTI_KINDS, REFUSED, comparable, key_tuples, make_array, narrow, rb,
                                 side)

pytestmark = pytest.mark.gpu

SEMI_KERNELS = ("join_build_kernel", "semi_mark_kernel", "semi_select_kernel")


def ref_semi(left, right, lkeys, rkeys, anti: bool) -> pa.Table:
    present = {k for k in key_tuples(right, rkeys) if k is not None}
    keep = [i for i, k in enumerate(key_tuples(left, lkeys)) if (k is not None and k in present) != anti]
    return pa.Table.from_batches([left]).take(pa.array(keep, pa.int64()))


def cut(b: pa.RecordBatch, start: int, n: int) -> pa.RecordBatch:
    """Rows [start, start + n) of b as fresh arrays (no slice offset)."""
    return b.take(pa.array(np.arange(start, start + n), pa.int64()))


def semi_plan(left, right, lkeys, rkeys, join_type: str) -> dict:
    on = [(plans.column(left.schema.names[a], a), plans.column(right.schema.names[b], b)) for a, b in zip(lkeys, rkeys)]
    return plans.hash_join_exec(plans.memory_exec(left.schema, None), plans.memory_exec(right.schema, None), on, join_type=join_type)


def gpu_semi(ctx, left, right, lkeys, rkeys, join_type):
    """(result as Arrow, {kernel: launches} of the execution)."""
    ec = fb.ExecutionContext(ctx, semi_plan(left, right, lkeys, rkeys, join_type))
    try:
        ec.feed_data_sources([[[left]], [[right]]])
        ctx.profile_begin()
        try:
            got = ec.execute_device().to_arrow()
        finally:
            prof = ctx.profile_end()
        ec.clean_data_sources()
    finally:
        ec.close()
    return got, {k: v["launches"] for k, v in prof.items()}


def check_semi(ctx, left, right, lkeys, rkeys, orientation=None):
    """Semi and Anti equal ref_semi row for row (Float64 by bits), and together they are the left input.
    `orientation`: "left" / "right" = the side the profile must show hashed."""
    n = {}
    for jt in ("Semi", "Anti"):
        got, ran = gpu_semi(ctx, left, right, lkeys, rkeys, jt)
        want = ref_semi(left, right, lkeys, rkeys, jt == "Anti")
        assert got.schema.names == left.schema.names and [f.type for f in got.schema] == [f.type for f in left.schema]
        assert got.num_rows == want.num_rows, (jt, got.num_rows, want.num_rows)
        for name in left.schema.names:
            assert comparable(got[name]).equals(comparable(want[name])), (jt, name)
        path = [k for k in SEMI_KERNELS if ran.get(k)]
        assert "join_count_scan_kernel" not in ran and "join_emit_kernel" not in ran, ran
        if orientation == "left":
            assert path == list(SEMI_KERNELS), ran
        elif orientation == "right":
            assert path == ["join_build_kernel", "semi_select_kernel"], ran
        n[jt] = got.num_rows
    assert n["Semi"] + n["Anti"] == left.num_rows
    return n


@pytest.mark.parametrize("kind", list(KEY_KINDS))
def test_single_key_edges(gpu_ctx, kind):
    """One key column of every type the inner join has (KW 4, KW 8, row keys for Utf8), edge values many times over;
    NULL keys on the left, then on the right; each side hashed in turn."""
    rng = np.random.default_rng(len(kind) * 11)
    l, lk = side([kind], 5000, rng, "l_", null_every=[4], edge_share=0.3)
    r, rk = side([kind], 3000, rng, "r_", keys_first=False, edge_share=0.3)
    n = check_semi(gpu_ctx, l, r, lk, rk, orientation="right")
    assert n["Semi"] > 0 and n["Anti"] > 0
    l2, lk2 = side([kind], 2000, rng, "l_", edge_share=0.3)
    r2, rk2 = side([kind], 6000, rng, "r_", null_every=[3], keys_first=False, edge_share=0.3)
    n = check_semi(gpu_ctx, l2, r2, lk2, rk2, orientation="left")
    assert n["Semi"] > 0 and n["Anti"] > 0


def test_float_key_rules(gpu_ctx):
    """NaN (any payload) meets nothing, -0.0 does not meet +0.0, +inf meets +inf, subnormals meet themselves: on either side
    hashed."""
    nan2 = float(np.array([0x7FF0000000000001], np.uint64).view(np.float64)[0])
    lv = [0.0, -0.0, np.inf, np.nan, nan2, 5e-324, -np.inf, 1.5, -5e-324]
    rv = [-0.0, np.nan, nan2, np.inf, 5e-324, -1.5]
    l = rb(a=pa.array(lv), x=pa.array(np.arange(len(lv))))
    r = rb(b=pa.array(rv), y=pa.array(np.arange(len(rv))))
    for left, right, lk, rk, orient in ((l, r, [0], [0], "right"), (cut(l, 0, 5), r, [0], [0], "left")):
        check_semi(gpu_ctx, left, right, lk, rk, orientation=orient)
    got, _ = gpu_semi(gpu_ctx, l, r, [0], [0], "Semi")
    assert got["x"].to_pylist() == [1, 2, 5]
    got, _ = gpu_semi(gpu_ctx, l, r, [0], [0], "Anti")
    assert got["x"].to_pylist() == [0, 3, 4, 6, 7, 8]


@pytest.mark.parametrize("kinds", MULTI_KINDS[:6], ids=lambda k: "-".join(k))
def test_multi_key_edges(gpu_ctx, kinds):
    """Two packed 4-byte columns and row keys; a NULL in any component of a key skips it; each side hashed in turn."""
    rng = np.random.default_rng(len(kinds) + 40)
    l, lk = side(kinds, 4000, rng, "l_", null_every=[5 + 2 * i for i in range(len(kinds))], filler=narrow(4000, rng, kinds), edge_share=0.3)
    r, rk = side(kinds, 6000, rng, "r_", keys_first=False, filler=narrow(6000, rng, kinds), edge_share=0.3)
    n = check_semi(gpu_ctx, l, r, lk, rk, orientation="left")
    assert n["Semi"] > 100 and n["Anti"] > 100
    check_semi(gpu_ctx, r, l, rk, lk, orientation="right")


def test_empty_and_one_row_sides(gpu_ctx):
    """An empty right side: Anti is the whole left input, Semi nothing; an empty left side: an empty table with the left
    schema; one-row sides, matching and not."""
    rng = np.random.default_rng(3)
    l, lk = side(["int64"], 1000, rng, "l_", null_every=[7], filler=[np.arange(1000)], edge_share=0.0)
    r, rk = side(["int64"], 1000, rng, "r_", keys_first=False, filler=[np.arange(1000) * 2], edge_share=0.0)
    assert check_semi(gpu_ctx, l, cut(r, 0, 0), lk, rk) == {"Semi": 0, "Anti": 1000}
    assert check_semi(gpu_ctx, cut(l, 0, 0), r, lk, rk) == {"Semi": 0, "Anti": 0}
    assert check_semi(gpu_ctx, cut(l, 10, 1), r, lk, rk, orientation="left") == {"Semi": 1, "Anti": 0}       # key 10
    assert check_semi(gpu_ctx, cut(l, 11, 1), r, lk, rk, orientation="left") == {"Semi": 0, "Anti": 1}       # key 11
    assert check_semi(gpu_ctx, l, cut(r, 5, 1), lk, rk, orientation="right") == {"Semi": 1, "Anti": 999}     # key 10
    assert check_semi(gpu_ctx, cut(l, 14, 1), r, lk, rk) == {"Semi": 0, "Anti": 1}                           # NULL over key 14


def test_all_match_and_no_match(gpu_ctx):
    rng = np.random.default_rng(4)
    for n_l, n_r in ((3000, 50_000), (50_000, 3000)):
        keys = rng.permutation(1 << 20)[:max(n_l, n_r)]
        l, lk = side(["int32"], n_l, rng, "l_", filler=[keys[:n_l]], edge_share=0.0)
        same = rng.choice(keys[:n_l], n_r)
        r, rk = side(["int32"], n_r, rng, "r_", keys_first=False, filler=[same], edge_share=0.0)
        orient = "left" if n_l <= n_r else "right"
        if n_l <= n_r:
            assert check_semi(gpu_ctx, l, r, lk, rk, orientation=orient) == {"Semi": n_l, "Anti": 0}
        r2, rk2 = side(["int32"], n_r, rng, "r_", keys_first=False, filler=[keys[:n_r] + (1 << 21)], edge_share=0.0)
        assert check_semi(gpu_ctx, l, r2, lk, rk2, orientation=orient) == {"Semi": 0, "Anti": n_l}


def test_duplicated_keys(gpu_ctx):
    """3000 rows of one key on each side next to singletons: the left rows appear once each, never once per right
    duplicate."""
    rng = np.random.default_rng(12)
    n = 3000 + 20_000
    lk = np.concatenate([np.full(3000, -7, np.int64), np.arange(20_000, dtype=np.int64) * 3 + 1])
    rk = np.concatenate([np.full(3000, -7, np.int64), np.arange(20_000, dtype=np.int64) * 2 + 1])
    rng.shuffle(lk)
    l, _ = side(["int64"], n, rng, "l_", filler=[lk], edge_share=0.0)
    r, _ = side(["int64"], n, rng, "r_", filler=[rk], edge_share=0.0, keys_first=False)
    rki = [r.schema.names.index("r_k0")]
    n_semi = 3000 + len(np.intersect1d(lk[lk != -7], rk[rk != -7]))
    assert check_semi(gpu_ctx, l, r, [0], rki, orientation="left")["Semi"] == n_semi
    assert check_semi(gpu_ctx, l, cut(r, 0, n - 1), [0], rki, orientation="right")["Semi"] <= n_semi


@pytest.mark.parametrize("n_left,n_right", [(1_000_000, 30_000), (60_000, 4_000_000)])
def test_large_sides(gpu_ctx, n_left, n_right):
    """Sizes of TPC-H SF 1 (q4: ~57 K orders against ~3.8 M lineitems hashes the left side), under both grid-prefix
    protocols of the compaction."""
    rng = np.random.default_rng(n_left)
    l, lk = side(["int32"], n_left, rng, "l_", null_every=[9], filler=[rng.integers(0, 2 * n_left, n_left)], edge_share=0.0, with_payload=False)
    r, rk = side(["int32"], n_right, rng, "r_", filler=[rng.integers(0, 2 * n_left, n_right)], edge_share=0.0, keys_first=False, with_payload=False)
    for mode in (0, 1):
        gpu_ctx.set_option("compact_mode", mode)
        try:
            check_semi(gpu_ctx, l, r, lk, rk, orientation="right" if n_right < n_left else "left")
        finally:
            gpu_ctx.set_option("compact_mode", 0)


@pytest.mark.parametrize("types", REFUSED, ids=lambda t: "%s-%s" % t)
def test_refusals_then_the_context_still_joins(gpu_ctx, types):
    """Unlike key types are refused with the inner join's message, either way round; the context then runs the same
    join of like types."""
    lt, rt = types
    l = rb(a=make_array(lt, [1, 2, 3]), id=pa.array([1, 2, 3]))
    r = rb(b=make_array(rt, [1, 2, 3, 3]))
    for jt in ("Semi", "Anti"):
        for a, b in ((l, r), (r, l)):
            with pytest.raises(fb.FlockGpuError) as info:
                gpu_semi(gpu_ctx, a, b, [0], [0], jt)
            assert info.value.code == ERR_UNSUPPORTED and "key types differ" in str(info.value)
    assert check_semi(gpu_ctx, l, rb(b=make_array(lt, [1, 3, 3, 9])), [0], [0]) == {"Semi": 2, "Anti": 1}


def test_all_null_key_column(gpu_ctx):
    """A key column with no valid value on either side matches nothing."""
    l = rb(a=pa.array([None, None, None], pa.int64()), id=pa.array([0, 1, 2]))
    r = rb(b=pa.array([1, 2], pa.int64()))
    assert check_semi(gpu_ctx, l, r, [0], [0]) == {"Semi": 0, "Anti": 3}
    assert check_semi(gpu_ctx, r, l, [0], [0]) == {"Semi": 0, "Anti": 2}
