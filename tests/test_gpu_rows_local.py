"""agg_rows_local_kernel (`-m gpu`): the CTA-local pre-aggregation for row (Utf8 / wide / nullable) group keys.  Where it
is taken is read from the launch profile: TPC-H q1 at SF 1 takes it, q3 does not, nor does any NEXMark or YSB plan; on
synthetic inputs of 2^18 rows and more its results equal numpy's with few groups, with ~3 000 groups (table flushes),
with NULL keys, with (Utf8, Date32) keys, and through Partial states then Final."""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import flock_b200 as fb
from flock_b200 import nexgen, plans, tpchgen
from test_gpu_value_edges import avg_ok, sum_ok
from test_nexmark_more_host import more_events
from test_ysb_host import ysb_inputs

pytestmark = pytest.mark.gpu
LOCAL = "agg_rows_local_kernel"


@pytest.fixture(scope="module")
def ctx():
    with fb.Context(0) as c:
        yield c


def profiled(ctx, fn):
    ctx.profile_begin()
    out = fn()
    prof = ctx.profile_end()
    return out, prof.get(LOCAL, {}).get("launches", 0), prof


def run_plan(ctx, plan, sources):
    ec = fb.ExecutionContext(ctx, plan)
    ec.feed_data_sources(sources)
    ctx.profile_begin()
    out = pa.Table.from_batches(ec.execute()[0])
    prof = ctx.profile_end()
    ec.clean_data_sources()
    ec.close()
    return out, prof.get(LOCAL, {}).get("launches", 0)


def tpch_sources(q, T):
    return [[T[t].to_batches()] for t in plans.TPCH_SOURCES[q]]


def test_taken_for_q1_not_for_q3_at_sf1(ctx):
    cols = {"lineitem": tpchgen.schema("lineitem").names, "orders": tpchgen.schema("orders").names, "customer": tpchgen.schema("customer").names}
    T = tpchgen.generate(1.0, 42, columns=cols)
    _, l1 = run_plan(ctx, plans.tpch_q1(), tpch_sources("q1", T))
    _, l3 = run_plan(ctx, plans.tpch_q3(), tpch_sources("q3", T))
    assert l1 == 1 and l3 == 0


def test_never_in_nexmark_or_ysb(ctx):
    ev = nexgen.generate(300_000, seed=42, batch_rows=65536)
    for q, f in plans.QUERIES.items():
        assert run_plan(ctx, f(), [[ev[r]] for r in plans.SOURCES[q]])[1] == 0, q
    mev = more_events(300_000, 42, 65536)
    for q, f in plans.MORE_QUERIES.items():
        assert run_plan(ctx, f(), [[mev[r]] for r in plans.MORE_SOURCES[q]])[1] == 0, q
    yi = ysb_inputs(1_000_000, 42, batch_rows=65536)
    assert run_plan(ctx, plans.ysb(), [[yi[r]] for r in plans.YSB_SOURCES["ysb"]])[1] == 0


def _check_groups(out: pa.Table, keys: list[np.ndarray], x: np.ndarray, key_names: list[str]):
    """out: keys..., SUM(x), MIN(x), MAX(x), COUNT(*), AVG(x) -- against numpy per group."""
    got = {}
    cols = [out.column(i).to_pylist() for i in range(out.num_columns)]
    for r in zip(*cols):
        got[tuple(r[:len(keys)])] = r[len(keys):]
    want_keys = list(zip(*[k.tolist() for k in keys]))
    groups = {}
    for i, k in enumerate(want_keys):
        groups.setdefault(k, []).append(i)
    assert len(got) == len(groups)
    for k, idx in groups.items():
        xs = x[idx]
        s, mn, mx, c, avg = got[k]
        assert c == len(idx) and mn == xs.min() and mx == xs.max() and sum_ok(s, xs)
        assert avg_ok(avg, xs)


AGGS = [("sum", -2, "s"), ("min", -2, "mn"), ("max", -2, "mx"), ("count", -1, "c"), ("avg", -2, "a")]


def _aggs(xcol):
    return [(f, xcol if c == -2 else c, nm) for f, c, nm in AGGS]


@pytest.mark.parametrize("n_groups", [4, 3000])
def test_utf8_keys(ctx, n_groups):
    rng = np.random.default_rng(n_groups)
    n = 1 << 19
    names = np.array([f"group-{i:05d}" for i in range(n_groups)], dtype=object)
    k = names[rng.integers(0, n_groups, n)]
    x = rng.normal(size=n) * 1000
    t = ctx.import_batches([pa.record_batch([pa.array(k, pa.utf8()), pa.array(x)], ["k", "x"])])
    out, launches, _ = profiled(ctx, lambda: ctx.hash_aggregate(t, [0], _aggs(1)).to_arrow())
    assert launches == 1
    _check_groups(out, [k], x, ["k"])


def test_null_and_two_column_keys(ctx):
    rng = np.random.default_rng(3)
    n = 300_000
    s = np.array(["A", "N", "R"], dtype=object)[rng.integers(0, 3, n)]
    svalid = rng.random(n) > 0.1
    d = rng.integers(9000, 9010, n).astype(np.int32)
    x = rng.integers(-1000, 1000, n).astype(np.float64)
    sa = pa.array([v if ok else None for v, ok in zip(s, svalid)], pa.utf8())
    t = ctx.import_batches([pa.record_batch([sa, pa.array(d, pa.date32()), pa.array(x)], ["s", "d", "x"])])
    out, launches, _ = profiled(ctx, lambda: ctx.hash_aggregate(t, [0, 1], _aggs(2)).to_arrow())
    assert launches == 1 and out.schema.field(1).type == pa.date32()
    out = out.set_column(1, "d", out.column(1).cast(pa.int32()))
    _check_groups(out, [np.array([v if ok else None for v, ok in zip(s, svalid)], dtype=object), d], x, ["s", "d"])


def test_partial_then_final(ctx):
    rng = np.random.default_rng(4)
    n = 1 << 19
    k = np.array(["x", "yy", "zzz", "wwww", "v"], dtype=object)[rng.integers(0, 5, n)]
    x = rng.normal(size=n)
    t = ctx.import_batches([pa.record_batch([pa.array(k, pa.utf8()), pa.array(x)], ["k", "x"])])
    halves = [ctx.import_batches([pa.record_batch([pa.array(k[i::2], pa.utf8()), pa.array(x[i::2])], ["k", "x"])]) for i in range(2)]
    aggs = [("sum", 1, "s"), ("min", 1, "mn"), ("max", 1, "mx"), ("count", -1, "c"), ("avg", 1, "a")]
    parts, launches, _ = profiled(ctx, lambda: [ctx.hash_aggregate(h, [0], aggs, mode="partial") for h in halves])
    assert launches == 2
    states = ctx.concat(parts)
    final = ctx.hash_aggregate(states, [0], [("sum", 1, "s"), ("min", 2, "mn"), ("max", 3, "mx"), ("count", 4, "c"), ("avg", 5, "a")], mode="final").to_arrow()
    _check_groups(final, [k], x, ["k"])
    single = ctx.hash_aggregate(t, [0], aggs).to_arrow()
    assert sorted(single.column(0).to_pylist()) == sorted(final.column(0).to_pylist())


def test_mostly_distinct_keys_stay_on_the_direct_insert(ctx):
    n = 1 << 19
    k = np.array([f"key-{i}" for i in range(n)], dtype=object)
    t = ctx.import_batches([pa.record_batch([pa.array(k, pa.utf8()), pa.array(np.ones(n))], ["k", "x"])])
    out, launches, prof = profiled(ctx, lambda: ctx.hash_aggregate(t, [0], [("sum", 1, "s")]).to_arrow())
    assert launches == 0 and prof.get("agg_insert_rows_kernel", {}).get("launches", 0) == 1 and out.num_rows == n
