"""TPC-H q7, q8 and q9 on the GPU (`-m gpu`), date_part on the device, and joins and projections over more than 16
columns.

- q7, q8 and q9 through flock_context_unmarshal / feed / execute against sqlite3 at SF 0.01 for three seeds and on
  Flock's `.tbl` fixtures, and against the pyarrow restatement at SF 1.  The ORDER BY is checked on the GPU's own output;
  every SUM is held to the error bound of a Float64 sum in any order, 2 (m - 1) u sum|x|, never to a relative bound (q9's
  amounts change sign), and q8's ratio to the bounds of its numerator and denominator.
- date_part on the device equals the host build of the same register program bit for bit over an edge relation (the
  first and last days of years around 0, 1970 and 2000, INT32 / INT64 extremes, the last unit of a day) as a
  projection, a predicate under both compaction modes, a group key and a sort key, at the tile and size edges, fed as
  one batch, as ragged batches and page-locked in place.
- A NEXMark-flavoured EXTRACT(HOUR FROM b_date_time) count, and a YSB-shaped plan whose fact filter holds date_part.
- A hash join with a 20-column side and a ProjectionExec over a 24-column join output that reads two columns of the same
  name, against pyarrow."""
import collections
import functools

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import flock_b200 as fb
from flock_b200 import case, col, lit, nexgen, plans, tpchgen, ysbgen
from test_tpch_host import SEEDS, fixture_tables, sqlite_db
from test_tpch_more_host import ARROW_MORE, N_OUT, UNITS, arrow_rows, assert_within_bounds, days_from_civil, edge_values, sqlite_more

pytestmark = pytest.mark.gpu

QUERIES = list(plans.TPCH_MORE_QUERIES)


def run_gpu(ctx, q: str, T: dict[str, pa.Table]) -> pa.Table:
    ec = fb.ExecutionContext(ctx, plans.TPCH_MORE_QUERIES[q]())
    ec.feed_data_sources([[T[t].to_batches() or [pa.RecordBatch.from_pylist([], schema=T[t].schema)]] for t in plans.TPCH_MORE_SOURCES[q]])
    out = pa.Table.from_batches(ec.execute()[0])
    ec.clean_data_sources()
    ec.close()
    return out


OUT_SCHEMA = {"q7": [("supp_nation", pa.utf8()), ("cust_nation", pa.utf8()), ("l_year", pa.int32()), ("revenue", pa.float64())],
              "q8": [("o_year", pa.int32()), ("mkt_share", pa.float64())],
              "q9": [("nation", pa.utf8()), ("o_year", pa.int32()), ("sum_profit", pa.float64())]}
ORDER = {"q7": [(0, False), (1, False), (2, False)], "q8": [(0, False)], "q9": [(0, False), (1, True)]}


def checked_rows(q: str, got: pa.Table) -> list[tuple]:
    assert [(f.name, f.type) for f in got.schema] == OUT_SCHEMA[q]
    rows = [tuple(r.values()) for r in got.to_pylist()]
    for a, b in zip(rows, rows[1:]):
        for i, desc in ORDER[q]:
            if a[i] != b[i]:
                assert (a[i] > b[i]) if desc else (a[i] < b[i]), (q, a, b)
                break
        else:
            raise AssertionError((q, "two rows with one group key", a, b))
    return rows


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("q", QUERIES)
def test_query_matches_sqlite(gpu_ctx, q, seed):
    T = tpchgen.generate(0.01, seed)
    rows = checked_rows(q, run_gpu(gpu_ctx, q, T))
    want = ARROW_MORE[q](T)
    sql = sqlite_more(sqlite_db(T), q)
    assert [r[:N_OUT[q] - 1] for r in rows] == [tuple(r[:N_OUT[q] - 1]) for r in sql]
    assert_within_bounds(q, rows, want)      # and sqlite's values lie in the same intervals (test_tpch_more_host)
    assert_within_bounds(q, sql, want)
    assert rows or q != "q9"


@pytest.mark.parametrize("q", QUERIES)
def test_tbl_fixtures(gpu_ctx, q):
    T = fixture_tables()
    rows = checked_rows(q, run_gpu(gpu_ctx, q, T))
    assert rows == sqlite_more(sqlite_db(T), q) == arrow_rows(q, ARROW_MORE[q](T)) == []


@functools.lru_cache(1)
def sf1():
    return tpchgen.generate(1.0, 42)


@pytest.mark.parametrize("q", QUERIES)
def test_sf1_matches_arrow(gpu_ctx, q):
    T = sf1()
    rows = checked_rows(q, run_gpu(gpu_ctx, q, T))
    assert rows
    assert_within_bounds(q, rows, ARROW_MORE[q](T))


# ---- date_part on the device against the host build ----------------------------------------------------------------------
@functools.lru_cache(None)
def large_rows():
    """From here the filter takes 16 rows per thread (PredTreeT<16>): the size rule of filter_project."""
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * 4 * 256 * 16


SIZES = [0, 1, 3, 4, 5, 8193, "large-1", "large+1"]


def rows_of(size):
    return size if isinstance(size, int) else large_rows() + (1 if size == "large+1" else -1)


@functools.lru_cache(2)
def date_relation(n: int) -> pa.RecordBatch:
    """Date32 and Timestamp s / ms / us / ns (no timezone), half edge values and half ordinary instants, 10 % NULL; and a
    row id.  The edge block repeats at the start, in the middle and in the last rows."""
    rng = np.random.default_rng(n)
    arrays, names = [], []
    for unit, per_day in UNITS.items():
        pool = np.array(edge_values(unit), np.int64)
        v = np.where(rng.random(n) < 0.5, pool[rng.integers(0, len(pool), n)],
                     rng.integers(days_from_civil(1900, 1, 1), days_from_civil(2100, 1, 1), n) * per_day + rng.integers(0, per_day, n))
        for start in {0, (n // 2) & ~3, max(n - len(pool), 0)}:
            m = min(len(pool), n - start)
            v[start:start + m] = pool[:m]
        mask = rng.random(n) < 0.1
        if unit == "date32":
            arrays.append(pa.array(v.astype(np.int32), pa.int32(), mask=mask).cast(pa.date32()))
        else:
            arrays.append(pa.array(v, pa.int64(), mask=mask).cast(pa.timestamp(unit)))
        names.append("t_" + unit)
    arrays.append(pa.array(np.arange(n, dtype=np.int64)))
    names.append("rid")
    return pa.record_batch(arrays, names)


EXTRACTS = [col(i).extract(f) for i in range(5) for f in ("year", "hour")]
PREDICATES = [(col(0).extract("year") >= 2000) | (col(2).extract("hour") == 23), col(4).extract("year") < col(1).extract("year"),
              case([(col(3).extract("hour") > 11, lit(1))], lit(0)) == 1]


def feeds(ctx, b):
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


def int32_bits(a) -> tuple[np.ndarray, np.ndarray]:
    """(values, valid) of an Int32 column as stored, the slots under NULLs included."""
    a = a.combine_chunks() if isinstance(a, pa.ChunkedArray) else a
    vals = np.frombuffer(a.buffers()[1], np.int32, len(a) + a.offset)[a.offset:] if len(a) else np.zeros(0, np.int32)
    return vals, ~a.is_null().to_numpy(zero_copy_only=False)


def assert_column(got, vals, valid, what):
    """Bit for bit: the validity, and every stored value (the host build and the kernels both store 0 under a NULL)."""
    gv, gvalid = int32_bits(got)
    assert np.array_equal(gvalid, valid), what
    assert np.array_equal(gv, vals), (what, np.flatnonzero(gv != vals)[:8])


def count_plan(schema: pa.Schema, key: dict, name: str) -> dict:
    count = plans.aggregate_expr("count", "COUNT(UInt8(1))", plans.literal("UInt8", 1), "UInt64")
    partial = plans.hash_aggregate_exec("Partial", [(key, name)], [count], plans.memory_exec(schema, None))
    shuffled = plans.coalesce_batches_exec(plans.repartition_hash(partial, [plans.column(name, 0)]))
    return plans.hash_aggregate_exec("FinalPartitioned", [(plans.column(name, 0), name)], [count], shuffled)


def run_plan(ctx, plan, sources):
    ec = fb.ExecutionContext(ctx, plan)
    ec.feed_data_sources(sources)
    out, prof = profiled(ctx, lambda: pa.Table.from_batches(ec.execute()[0]))
    ec.clean_data_sources()
    ec.close()
    return out, prof


@pytest.mark.parametrize("size", SIZES)
def test_date_part_on_the_device_equals_the_host_build(gpu_ctx, size):
    n = rows_of(size)
    b = date_relation(n)
    host, _ = fb.selftest_eval_tree(b, EXTRACTS)
    for t in feeds(gpu_ctx, b):
        out, prof = profiled(gpu_ctx, lambda: gpu_ctx.filter_project(t, None, EXTRACTS).to_batch())
        for i, (v, valid, dt) in enumerate(host):
            assert dt == fb.INT32 and out.schema.field(i).type == pa.int32()
            assert_column(out.column(i), v, valid, (size, i))
        if n:
            assert prof.get("expr_eval_kernel") == 1 and "project_generic_kernel" not in prof, prof
    for p in PREDICATES:
        mask, _ = fb.selftest_eval_tree(b, p, predicate=True)
        for mode in (0, 1):
            gpu_ctx.set_option("compact_mode", mode)
            try:
                for t in feeds(gpu_ctx, b):
                    out, prof = profiled(gpu_ctx, lambda: gpu_ctx.filter_project(t, p, [col(5), EXTRACTS[1]]).to_batch())
                    assert np.array_equal(out.column(0).to_numpy(), np.flatnonzero(mask)), (size, mode, p.tokens)
                    v, valid, _ = host[1]
                    assert_column(out.column(1), v[mask], valid[mask], (size, mode, p.tokens))
                    if n:
                        assert prof.get("filter_compact_kernel") == 1, prof
            finally:
                gpu_ctx.set_option("compact_mode", 0)
    # a group key and a sort key, through the plan reader
    key = plans.date_part("YEAR", plans.column("t_ms", 2))
    got, prof = run_plan(gpu_ctx, count_plan(b.schema, key, "y"), [[[b]]])
    v, valid, _ = host[4]
    want = collections.Counter(int(x) if ok else None for x, ok in zip(v, valid))
    assert dict(zip(got.column("y").to_pylist(), got.column(1).to_pylist())) == want, size
    if n:
        assert prof.get("expr_eval_kernel") == 1, prof
    # sort keys take no NULLs: HOUR of a Timestamp(Microsecond) column without them, descending, then the row id
    plain = pa.record_batch([pc.fill_null(b.column(3), pa.scalar(0, pa.timestamp("us"))), b.column(5)], ["t_us", "rid"])
    sort = plans.sort_exec([(plans.date_part("hour", plans.column("t_us", 0)), True, False), (plans.column("rid", 1), False, False)],
                           plans.memory_exec(plain.schema, None))
    got, prof = run_plan(gpu_ctx, sort, [[[plain]]])
    (v, valid, _), = fb.selftest_eval_tree(plain, [col(0).extract("hour")])[0]
    assert valid.all()
    assert np.array_equal(got.column("rid").to_numpy(), np.lexsort((np.arange(n), -v.astype(np.int64)))), size
    assert got.schema.names == ["t_us", "rid"]
    if n:
        assert prof.get("expr_eval_kernel") == 1, prof


def test_date_part_over_page_locked_batches(gpu_ctx):
    n = 5 * 8192 + 77
    b = date_relation(n)
    pinned = [gpu_ctx.pinned_copy(b.take(np.arange(s, min(s + 8192, n)))) for s in range(0, n, 8192)]   # buffers of their own
    C = lambda name: plans.column(name, b.schema.names.index(name))
    pred = plans.binary(plans.date_part("YEAR", C("t_date32")), "GtEq", plans.literal("Int32", 2000))
    plan = plans.projection_exec([(C("rid"), "rid"), (plans.date_part("HOUR", C("t_ns")), "h")],
                                 plans.filter_exec(pred, plans.memory_exec(b.schema, None)))
    gpu_ctx.set_option("feed_zero_copy", 1)
    try:
        ec = fb.ExecutionContext(gpu_ctx, plan)
        ec.feed_data_sources([fb.HostRelation(pinned)])
        got = pa.Table.from_batches(ec.execute()[0])
        ec.close()
    finally:
        gpu_ctx.set_option("feed_zero_copy", 0)
    mask, _ = fb.selftest_eval_tree(b, col(0).extract("year") >= lit(2000, "int32"), predicate=True)
    (v, valid, _), = fb.selftest_eval_tree(b, [col(4).extract("hour")])[0]
    assert np.array_equal(got["rid"].to_numpy(), np.flatnonzero(mask))
    assert_column(got["h"], v[mask], valid[mask], "h")


def test_nexmark_hour_count(gpu_ctx):
    """SELECT EXTRACT(HOUR FROM b_date_time), COUNT(*) FROM bid GROUP BY 1 over Timestamp(Millisecond) bids."""
    bids = nexgen.bids(300_000, seed=42)
    ts = bids.column("b_date_time").cast(pa.int64()).to_numpy()
    key = plans.date_part("HOUR", plans.column("b_date_time", 3))
    got, _ = run_plan(gpu_ctx, count_plan(bids.schema, key, "h"), [[nexgen.split_batches(bids)]])
    hours, counts = np.unique((ts // 3_600_000) % 24, return_counts=True)
    assert got.schema.field("h").type == pa.int32()
    assert dict(zip(got.column("h").to_pylist(), got.column(1).to_pylist())) == dict(zip(hours.tolist(), counts.tolist()))


def test_ysb_with_date_part_in_the_fact_filter(gpu_ctx):
    """The one-pass join count interprets the term form, which has no date_part: the filter runs first, on its own."""
    camp = ysbgen.campaigns(100, 10, 7)
    ev = ysbgen.ad_events(200_000, camp, 7, columns=["ad_id", "event_type", "event_time"])
    ms = ev.column("event_time").cast(pa.int64()).to_numpy()
    sec = int(np.median((ms // 1000) % 60))
    n = 8
    scan = plans.repartition_rr(plans.memory_exec(plans.AD_EVENT, [2, 4, 5]), n)   # ad_id 0, event_type 1, event_time 2
    # event_type = 'view' AND EXTRACT(HOUR FROM event_time) >= 0 AND the first `sec` seconds of every minute
    pred = plans.binary(plans.binary(plans.column("event_type", 1), "Eq", plans.literal("Utf8", "view")), "And",
                        plans.binary(plans.date_part("HOUR", plans.column("event_time", 2)), "GtEq", plans.literal("Int32", 0)))
    pred = plans.binary(pred, "And", plans.binary(plans.binary(plans.cast(plans.column("event_time", 2), "Int64"), "Modulo", plans.literal("Int64", 60_000)),
                                                  "Lt", plans.literal("Int64", sec * 1000)))
    events = plans.coalesce_batches_exec(plans.repartition_hash(plans.coalesce_batches_exec(plans.filter_exec(pred, scan)), [plans.column("ad_id", 0)], n))
    camps = plans.coalesce_batches_exec(plans.repartition_hash(plans.repartition_rr(plans.memory_exec(plans.CAMPAIGN, [0, 1]), n),
                                                               [plans.column("c_ad_id", 0)], n))
    join = plans.hash_join_exec(events, camps, [(plans.column("ad_id", 0), plans.column("c_ad_id", 0))])
    plan = plans.two_phase_aggregate([("campaign_id", 4)], [plans._ysb_count()], plans.coalesce_batches_exec(join), n)
    got, prof = run_plan(gpu_ctx, plan, [[[ev]], [[camp]]])
    keep = pc.and_(pc.equal(ev.column("event_type"), "view"), pa.array(ms % 60_000 < sec * 1000))
    views = pa.Table.from_batches([ev]).filter(keep)
    assert 0 < views.num_rows < ev.num_rows
    j = views.join(pa.Table.from_batches([camp]), "ad_id", "c_ad_id", join_type="inner")
    want = collections.Counter(j.column("campaign_id").to_pylist())
    assert dict(zip(got.column("campaign_id").to_pylist(), got.column(plans.YSB_COUNT).to_pylist())) == want
    assert prof.get("dim_count_kernel") == 1 and prof.get("filter_compact_kernel", 0) >= 1 and "join_build_kernel" not in prof, sorted(prof)


# ---- more than 16 columns --------------------------------------------------------------------------------------------------
def wide_side(n: int, n_cols: int, keys: int, seed: int, prefix: str) -> pa.RecordBatch:
    """An id, an Int32 key, a Utf8 column called `name`, and columns of Int32 / Int64 / Float64 / Utf8 / Date32 with NULLs."""
    rng = np.random.default_rng(seed)
    arrays = [pa.array(np.arange(n, dtype=np.int64)), pa.array(rng.integers(0, keys, n).astype(np.int32)),
              pa.array([f"{prefix}{i % 97}" for i in range(n)], pa.utf8(), mask=rng.random(n) < 0.1)]
    names = [prefix + "id", "key", "name"]
    for c in range(n_cols - 3):
        mask = rng.random(n) < 0.2
        kind = c % 5
        if kind == 0:
            a = pa.array(rng.integers(-1 << 31, 1 << 31, n).astype(np.int32), mask=mask)
        elif kind == 1:
            a = pa.array(rng.integers(-1 << 62, 1 << 62, n), mask=mask)
        elif kind == 2:
            a = pa.array(rng.standard_normal(n), mask=mask)
        elif kind == 3:
            a = pa.array([("x" * (i % 5)) + str(i) for i in range(n)], pa.utf8(), mask=mask)
        else:
            a = pa.array(rng.integers(-20000, 20000, n).astype(np.int32), mask=mask).cast(pa.date32())
        arrays.append(a)
        names.append(f"{prefix}{c}")
    return pa.record_batch(arrays, names)


def joined(left: pa.RecordBatch, right: pa.RecordBatch) -> pa.Table:
    """left ++ right of every pair with equal keys, ordered by (left id, right id)."""
    lt, rt = pa.Table.from_batches([left]), pa.Table.from_batches([right])
    pairs = lt.select(["lid", "key"]).join(rt.select(["rid", "key"]).rename_columns(["rid", "rkey"]), "key", "rkey", join_type="inner")
    pairs = pairs.sort_by([("lid", "ascending"), ("rid", "ascending")])
    l, r = lt.take(pairs["lid"]), rt.take(pairs["rid"])
    return pa.table(l.columns + r.columns, names=l.column_names + r.column_names)


@pytest.mark.parametrize("left_rows, right_rows", [(5000, 3000), (3000, 5000)])
def test_hash_join_with_a_20_column_side(gpu_ctx, left_rows, right_rows):
    left = wide_side(left_rows, 20, 1000, 1, "l")
    right = wide_side(right_rows, 4, 1000, 2, "r")
    got = gpu_ctx.hash_join(gpu_ctx.import_batches([left]), gpu_ctx.import_batches([right]), [1], [1]).to_arrow()
    assert got.num_columns == 24
    got = got.sort_by([("lid", "ascending"), ("rid", "ascending")])
    want = joined(left, right)
    assert got.num_rows == want.num_rows > 0
    for i in range(24):
        assert got.column(i).combine_chunks().equals(want.column(i).combine_chunks()), want.column_names[i]


def test_projection_over_a_24_column_join_reads_two_columns_named_alike(gpu_ctx):
    left = wide_side(4000, 20, 500, 3, "l")
    right = wide_side(2500, 4, 500, 4, "r")
    ls, rs = left.schema, right.schema
    join = plans.hash_join_exec(plans.memory_exec(ls, None), plans.memory_exec(rs, None), [(plans.column("key", 1), plans.column("key", 1))])
    # left: lid 0, key 1, name 2, l0 3, l1 4 (Int64) ...; right: rid 20, key 21, name 22, r0 23
    plan = plans.projection_exec([(plans.column("name", 2), "a"), (plans.column("name", 22), "b"), (plans.column("lid", 0), "lid"),
                                  (plans.binary(plans.column("l1", 4), "Minus", plans.literal("Int64", 7)), "c"),
                                  (plans.column("rid", 20), "rid")], join)
    got, _ = run_plan(gpu_ctx, plan, [[[left]], [[right]]])
    got = got.sort_by([("lid", "ascending"), ("rid", "ascending")])
    want = joined(left, right)
    assert got.column_names == ["a", "b", "lid", "c", "rid"] and got.num_rows == want.num_rows > 0
    assert got["a"].combine_chunks().equals(want.column(2).combine_chunks())
    assert got["b"].combine_chunks().equals(want.column(22).combine_chunks())
    assert got["c"].combine_chunks().equals(pc.subtract(want.column(4), 7).combine_chunks())
