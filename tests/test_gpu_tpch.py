"""TPC-H q1, q3, q5, q6, q10, q12 and q14 on the GPU (`-m gpu`): every query through flock_context_unmarshal / feed /
execute against sqlite3 running Flock's own query text at SF 0.01 for three seeds and on Flock's `.tbl` fixtures, q1,
q6, q12 and q14 at SF 1 against the pyarrow restatement, the ORDER BY checked on the GPU's own output, and Date32
columns through IPC, zstd payloads, sort, join and partition."""
import datetime

import numpy as np
import pyarrow as pa
import pytest

import flock_b200 as fb
from flock_b200 import plans, tpchgen
from test_tpch_host import ARROW, SEEDS, fixture_tables, rows_close, sqlite_db, sqlite_query

pytestmark = pytest.mark.gpu

QUERIES = list(plans.TPCH_QUERIES)


@pytest.fixture(scope="module")
def ctx():
    with fb.Context(0) as c:
        yield c


def run_gpu(ctx, q: str, T: dict[str, pa.Table]) -> pa.Table:
    ec = fb.ExecutionContext(ctx, plans.TPCH_QUERIES[q]())
    ec.feed_data_sources([[T[t].to_batches() or [pa.RecordBatch.from_pylist([], schema=T[t].schema)]] for t in plans.TPCH_SOURCES[q]])
    out = pa.Table.from_batches(ec.execute()[0])
    ec.clean_data_sources()
    ec.close()
    return out


def _plain(v):
    return v.isoformat() if isinstance(v, datetime.date) else v


def rows_of(t: pa.Table) -> list[tuple]:
    return [tuple(_plain(v) for v in r.values()) for r in t.to_pylist()]


def _canon(rows):
    return sorted(rows, key=lambda r: tuple((0, round(x, 2)) if isinstance(x, float) else (1, x) for x in r))


ORDER = {"q1": [(0, False), (1, False)], "q3": [(1, True), (2, False)], "q5": [(1, True)], "q10": [(2, True)], "q12": [(0, False)]}


def check_order(q: str, rows: list[tuple]):
    for a, b in zip(rows, rows[1:]):
        for i, desc in ORDER.get(q, []):
            if a[i] != b[i]:
                assert (a[i] > b[i]) if desc else (a[i] < b[i]), (q, a, b)
                break


# Float64 SUM / AVG in any order: |error| <= gamma_(m-1) * sum|x| (test_gpu_value_edges.sum_tolerance).  Every TPC-H
# addend here is positive, so sum|x| is the value itself and the bound is relative, (m - 1) * u, m = the lines summed.
def check(q: str, got: pa.Table, want: list[tuple], addends: int):
    rows = rows_of(got)
    check_order(q, rows)
    k = max(addends - 1, 1) * 2.0 ** -53
    # the result and the reference each within the bound of two sums and two more roundings (q14's 100 * a / b)
    rel = 4 * (k / (1 - k) + 2 * 2.0 ** -53)
    assert rows_close(_canon(rows), _canon(want), rel=rel), (q, rows[:5], want[:5])


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("q", QUERIES)
def test_query_matches_sqlite(ctx, q, seed):
    T = tpchgen.generate(0.01, seed)
    check(q, run_gpu(ctx, q, T), sqlite_query(sqlite_db(T), q), T["lineitem"].num_rows)


# On the 10-row fixtures no line passes q6's or q14's filter: their SUMs are NULL, and a projection over an all-NULL
# column is refused by filter_project (a limit of the projection, not of these queries)
@pytest.mark.parametrize("q", [q for q in QUERIES if q not in ("q6", "q14")])
def test_tbl_fixtures(ctx, q):
    T = fixture_tables()
    check(q, run_gpu(ctx, q, T), sqlite_query(sqlite_db(T), q), T["lineitem"].num_rows)


@pytest.mark.parametrize("q", ["q1", "q6", "q12", "q14"])
def test_sf1_matches_arrow(ctx, q):
    T = tpchgen.generate(1.0, 42, columns={t: tpchgen.schema(t).names for t in plans.TPCH_SOURCES[q]})
    check(q, run_gpu(ctx, q, T), [tuple(_plain(v) for v in r) for r in ARROW[q](T)], T["lineitem"].num_rows)


def test_q1_output_schema(ctx):
    out = run_gpu(ctx, "q1", tpchgen.generate(0.01, 42, columns={"lineitem": tpchgen.schema("lineitem").names}))
    assert out.schema.names == ["l_returnflag", "l_linestatus", "sum_qty", "sum_base_price", "sum_disc_price", "sum_charge", "avg_qty",
                                "avg_price", "avg_disc", "count_order"]
    assert out.schema.field("count_order").type == pa.uint64() and out.schema.field("avg_disc").type == pa.float64()


def test_date32_round_trips(ctx):
    rng = np.random.default_rng(5)
    n = 100_003
    days = rng.integers(-1000, 20000, n).astype(np.int32)
    b = pa.record_batch([pa.array(days, pa.date32()), pa.array(np.arange(n, dtype=np.int64))], ["d", "i"])
    t = ctx.import_batches([b])
    assert t.to_arrow().column("d").combine_chunks().equals(b.column("d"))
    h, body = t.to_ipc()
    assert ctx.import_ipc(b.schema, [(h, body)]).to_arrow().equals(pa.Table.from_batches([b]))
    frames = t.to_payload("zstd", rows_per_frame=30000)
    assert ctx.import_payload(b.schema, frames).to_arrow().equals(pa.Table.from_batches([b]))
    s = ctx.sort(t, [0], [True]).to_arrow()
    assert s.column("d").to_numpy().astype("datetime64[D]").astype(np.int64).tolist() == sorted(days.tolist(), reverse=True)
    dim = pa.record_batch([pa.array(np.unique(days)[:50], pa.date32()), pa.array(np.arange(50, dtype=np.int32))], ["k", "v"])
    j = ctx.hash_join(ctx.import_batches([dim]), t, [0], [0]).to_arrow()
    want = int(np.isin(days, np.unique(days)[:50]).sum())
    assert j.num_rows == want and j.schema.field("k").type == pa.date32()
    assert all(a == b for a, b in zip(j.column("k").to_pylist(), j.column("d").to_pylist()))
    parts = ctx.hash_partition(t, [0], 4)
    got = pa.concat_tables([p.to_arrow() for p in parts])
    assert sorted(got.column("i").to_pylist()) == list(range(n))
    for p in parts:   # equal dates meet in one partition
        others = set().union(*[set(q.to_arrow().column("d").to_pylist()) for q in parts if q is not p])
        assert not (set(p.to_arrow().column("d").to_pylist()) & others)


def test_date32_group_and_minmax(ctx):
    rng = np.random.default_rng(9)
    n = 300_000
    days = rng.integers(9000, 9100, n).astype(np.int32)
    vals = rng.integers(0, 1 << 20, n).astype(np.int32)
    b = pa.record_batch([pa.array(days, pa.date32()), pa.array(vals, pa.date32())], ["d", "v"])
    out = ctx.hash_aggregate(ctx.import_batches([b]), [0], [("min", 1, "mn"), ("max", 1, "mx"), ("count", -1, "n")]).to_arrow()
    assert out.schema.field(0).type == pa.date32() and out.schema.field(1).type == pa.date32()
    got = {r[0]: r[1:] for r in zip(*[c.cast(pa.int32()).to_pylist() if pa.types.is_date32(c.type) else c.to_pylist() for c in out.columns])}
    for d in np.unique(days)[:20]:
        m = days == d
        assert got[int(d)] == (int(vals[m].min()), int(vals[m].max()), int(m.sum()))
    with pytest.raises(fb.FlockGpuError) as e:
        ctx.hash_aggregate(ctx.import_batches([b]), [0], [("sum", 1, "s")])
    assert "Date32" in str(e.value)


def test_ndjson_refuses_date32(ctx):
    """NDJSON has no Date32 parser: the import refuses the schema before any kernel runs."""
    schema = pa.schema([("d", pa.date32()), ("i", pa.int64())])
    launches = ctx.kernel_launches
    with pytest.raises(fb.FlockGpuError) as e:
        ctx.import_ndjson(schema, b'{"d": 10471, "i": 1}\n')
    assert e.value.code == -2 and ctx.kernel_launches == launches
