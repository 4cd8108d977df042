"""TPC-H q4, q16, q18 and q21 on the GPU (`-m gpu`): their EXISTS, IN and NOT IN subqueries run as Semi / Anti hash joins.

Each query goes through flock_context_unmarshal / feed / execute and must equal sqlite3 running Flock's text
(test_tpch_subquery_host) at SF 0.01 for three seeds, with the planted complaint suppliers and heavy orders, and on
Flock's `.tbl` fixtures; at SF 1, q4 and q18 must equal the pyarrow restatements.  Rows are compared in the order the
GPU gives them, since every ORDER BY here covers the whole group key; Float64 sums to a relative 1e-9."""
import functools

import pyarrow as pa
import pytest

import flock_b200 as fb
from flock_b200 import plans, tpchgen
from test_tpch_host import SEEDS, fixture_tables, rows_close
from test_tpch_subquery_host import ARROW_SUBQUERY, planted, sqlite_indexed, sqlite_subquery

pytestmark = pytest.mark.gpu

QUERIES = list(plans.TPCH_SUBQUERY_QUERIES)


def run_gpu(ctx, q: str, T: dict[str, pa.Table], make=None) -> list[tuple]:
    ec = fb.ExecutionContext(ctx, (make or plans.TPCH_SUBQUERY_QUERIES[q])())
    ec.feed_data_sources([[T[t].to_batches() or [pa.RecordBatch.from_pylist([], schema=T[t].schema)]] for t in plans.TPCH_SUBQUERY_SOURCES[q]])
    out = ec.execute_device().to_arrow()
    ec.clean_data_sources()
    ec.close()
    # sqlite3 holds dates as ISO strings
    return [tuple(v.isoformat() if hasattr(v, "isoformat") else v for v in r.values()) for r in out.to_pylist()]


@pytest.mark.parametrize("seed", SEEDS)
@pytest.mark.parametrize("q", QUERIES)
def test_query_matches_sqlite(gpu_ctx, q, seed):
    T = planted(tpchgen.generate(0.01, seed))
    got = run_gpu(gpu_ctx, q, T)
    assert got and rows_close(got, sqlite_subquery(sqlite_indexed(T), q))


@pytest.mark.parametrize("seed", SEEDS)
def test_q16_without_anti_differs(gpu_ctx, seed):
    """The Anti join removes rows: q16 planned without it answers differently."""
    T = planted(tpchgen.generate(0.01, seed))
    with_anti = run_gpu(gpu_ctx, "q16", T)
    without = run_gpu(gpu_ctx, "q16", T, make=lambda: plans.tpch_q16(anti=False))      # the supplier source feeds no leaf
    assert without != with_anti and sum(r[3] for r in without) > sum(r[3] for r in with_anti)


@pytest.mark.parametrize("q", QUERIES)
def test_tbl_fixtures(gpu_ctx, q):
    T = fixture_tables()
    assert rows_close(run_gpu(gpu_ctx, q, T), sqlite_subquery(sqlite_indexed(T), q))


@functools.lru_cache(1)
def sf1():
    return planted(tpchgen.generate(1.0, 42))


@pytest.mark.parametrize("q", ["q4", "q18"])
def test_sf1_matches_arrow(gpu_ctx, q):
    T = sf1()
    got = run_gpu(gpu_ctx, q, T)
    assert got and rows_close(got, ARROW_SUBQUERY[q](T))


@pytest.mark.parametrize("q", ["q4", "q18"])
def test_semi_equals_distinct_inner_rewrite(gpu_ctx, q):
    """The Semi plan and the DISTINCT + inner join plan of the same query agree on the GPU at SF 0.01."""
    T = planted(tpchgen.generate(0.01, 7))
    make = {"q4": lambda: plans.tpch_q4(as_inner=True), "q18": lambda: plans.tpch_q18(as_inner=True)}[q]
    assert rows_close(run_gpu(gpu_ctx, q, T), run_gpu(gpu_ctx, q, T, make=make))
