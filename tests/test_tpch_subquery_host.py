"""TPC-H q4, q16, q18 and q21 without a GPU: the plans' shapes and Semi / Anti join types, and CPU references that agree.

The references: sqlite3 runs Flock's query texts (tests/golden/tpch/queries/qN.sql) as they are, with two rewrites:
`DATE 'x'` becomes `'x'` (dates are ISO strings, as in test_tpch_host), and q4's one interval sum
`DATE '1993-07-01' + interval '3' month` becomes `'1993-10-01'`, the value the plan builder folds it to.  A pyarrow
restatement with `pc.is_in` covers q4 and q18.

The generator plants no supplier comment that q16's NOT IN looks for and no order heavy enough for q18's
SUM(l_quantity) > 300, so `planted()` adds both here, leaving tpchgen's own output as it is."""
import re

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import flock_b200 as fb
from flock_b200 import _ffi, plans, tpchgen
from test_tpch_host import SEEDS, _d, fixture_tables, query_sql, rows_close, sqlite_db

QUERIES = list(plans.TPCH_SUBQUERY_QUERIES)
# the join type of each Semi / Anti join of the query, outermost first (plan_str's order)
JOIN_TYPES = {"q4": ["Semi"], "q16": ["Anti"], "q18": ["Semi"], "q21": ["Anti", "Semi"]}


def sqlite_indexed(T: dict[str, pa.Table]):
    """sqlite_db with an index on the correlation key of q4's and q21's subqueries, which are otherwise a scan of
    lineitem per outer row."""
    db = sqlite_db(T)
    db.execute("CREATE INDEX lineitem_orderkey ON lineitem (l_orderkey)")
    return db


def sqlite_subquery(db, q: str) -> list[tuple]:
    sql = re.sub(r"DATE\s+'1993-07-01'\s*\+\s*interval\s+'3'\s+month", "'1993-10-01'", query_sql(q), flags=re.IGNORECASE)
    sql = re.sub(r"DATE\s+'([0-9-]+)'", r"'\1'", sql, flags=re.IGNORECASE)
    return db.execute(sql).fetchall()


def planted(T: dict[str, pa.Table]) -> dict[str, pa.Table]:
    """T with every 13th supplier's comment holding "Customer ... Complaints" (q16), and the lines of the first five
    orders with seven lines at quantity 50, 350 in all (q18)."""
    T = dict(T)
    su = T["supplier"]
    keys = su["s_suppkey"].to_numpy()
    comments = [f"{c[:20]} Customer slow Complaints {c[20:40]}" if k % 13 == 5 else c for k, c in zip(keys, su["s_comment"].to_pylist())]
    T["supplier"] = su.set_column(su.schema.get_field_index("s_comment"), "s_comment", pa.array(comments, pa.utf8()))
    li = T["lineitem"]
    ok = li["l_orderkey"].to_numpy()
    u, counts = np.unique(ok, return_counts=True)
    heavy = u[counts == 7][:5]
    q = np.where(np.isin(ok, heavy), 50.0, li["l_quantity"].to_numpy())
    T["lineitem"] = li.set_column(li.schema.get_field_index("l_quantity"), "l_quantity", pa.array(q, pa.float64()))
    return T


# ---- pyarrow restatements (from the SQL text) ----------------------------------------------------------------------------
def arrow_q4(T) -> list[tuple]:
    od = T["orders"]
    od = od.filter(pc.and_(pc.greater_equal(od["o_orderdate"], _d("1993-07-01")), pc.less(od["o_orderdate"], _d("1993-10-01"))))
    li = T["lineitem"]
    late = li.filter(pc.less(li["l_commitdate"], li["l_receiptdate"]))["l_orderkey"]
    od = od.filter(pc.is_in(od["o_orderkey"], late.unique()))
    g = od.group_by("o_orderpriority").aggregate([("o_orderkey", "count")]).sort_by("o_orderpriority")
    return list(zip(g["o_orderpriority"].to_pylist(), g["o_orderkey_count"].to_pylist()))


def arrow_q18(T) -> list[tuple]:
    li = T["lineitem"]
    sums = li.group_by("l_orderkey").aggregate([("l_quantity", "sum")])
    big = sums.filter(pc.greater(sums["l_quantity_sum"], 300.0))["l_orderkey"]
    od = T["orders"].filter(pc.is_in(T["orders"]["o_orderkey"], big))
    j = T["customer"].join(od, "c_custkey", "o_custkey", join_type="inner")
    j = j.join(li.select(["l_orderkey", "l_quantity"]), "o_orderkey", "l_orderkey", join_type="inner")
    g = j.group_by(["c_name", "c_custkey", "o_orderkey", "o_orderdate", "o_totalprice"]).aggregate([("l_quantity", "sum")])
    g = g.sort_by([("o_totalprice", "descending"), ("o_orderdate", "ascending")])
    rows = zip(*[g[c].to_pylist() for c in ("c_name", "c_custkey", "o_orderkey", "o_orderdate", "o_totalprice", "l_quantity_sum")])
    return [(a, b, c, d.isoformat(), e, f) for a, b, c, d, e, f in rows]


ARROW_SUBQUERY = {"q4": arrow_q4, "q18": arrow_q18}


@pytest.fixture(scope="module", params=SEEDS)
def sf001(request):
    return request.param, planted(tpchgen.generate(0.01, request.param))


# ---- plan shapes ----------------------------------------------------------------------------------------------------------
def _joins(p: dict, out=None) -> list[str]:
    out = [] if out is None else out
    if p["execution_plan"] == "hash_join_exec":
        out.append(p["join_type"])
    for k in ("input", "left", "right"):
        if k in p:
            _joins(p[k], out)
    return out


@pytest.mark.parametrize("q", QUERIES)
def test_plan_shape_and_join_types(q):
    p = plans.TPCH_SUBQUERY_QUERIES[q]()
    s = fb.ExecutionContext(None, p).plan_str(0)
    assert s.count("MemoryExec") == len(plans.TPCH_SUBQUERY_SOURCES[q])
    assert s.splitlines()[0].startswith("SortExec: [")
    shown = re.findall(r"join_type=(\w+)", s)
    assert [t for t in shown if t != "Inner"] == JOIN_TYPES[q]
    assert [t for t in _joins(p) if t != "Inner"] == JOIN_TYPES[q]
    if q == "q16":
        assert "HashJoinExec: mode=Partitioned, join_type=Anti, on=[(ps_suppkey, s_suppkey)]" in s
    if q == "q4":
        assert "HashJoinExec: mode=Partitioned, join_type=Semi, on=[(o_orderkey, l_orderkey)]" in s


def test_comparison_plans():
    """q4 and q18 planned as DISTINCT + inner join (the benchmark's comparison) have no Semi join, q16 without its Anti
    has no Anti join, and each keeps its sources."""
    for make, n_src in ((lambda: plans.tpch_q4(as_inner=True), 2), (lambda: plans.tpch_q18(as_inner=True), 4)):
        s = fb.ExecutionContext(None, make()).plan_str(0)
        assert "join_type=Semi" not in s and s.count("MemoryExec") == n_src
    s = fb.ExecutionContext(None, plans.tpch_q16(anti=False)).plan_str(0)
    assert "join_type=Anti" not in s and s.count("MemoryExec") == 2


@pytest.mark.parametrize("jt", ["Left", "Right", "Full", "Bogus"])
def test_other_join_types_refused(jt):
    p = plans.tpch_q4()
    node = p
    while node["execution_plan"] != "hash_join_exec":
        node = node["input"]
    node["join_type"] = jt
    with pytest.raises(fb.FlockGpuError) as info:
        fb.ExecutionContext(None, p)
    assert info.value.code == _ffi.ERR_UNSUPPORTED and jt in info.value.message


def test_existing_query_sets_unchanged():
    assert list(plans.TPCH_QUERIES) == ["q1", "q3", "q5", "q6", "q10", "q12", "q14"]
    assert list(plans.TPCH_MORE_QUERIES) == ["q7", "q8", "q9"]
    assert all(j == "Inner" for make in (*plans.TPCH_QUERIES.values(), *plans.TPCH_MORE_QUERIES.values()) for j in _joins(make()))


# ---- the references agree ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("q", QUERIES)
def test_sqlite_answers_are_not_empty(sf001, q):
    _, T = sf001
    got = sqlite_subquery(sqlite_indexed(T), q)
    assert got and got[0][0] is not None


@pytest.mark.parametrize("q", ["q4", "q18"])
def test_sqlite_equals_arrow(sf001, q):
    _, T = sf001
    assert rows_close(sqlite_subquery(sqlite_indexed(T), q), ARROW_SUBQUERY[q](T))


def test_planting_leaves_the_generator_alone():
    a, b = tpchgen.generate(0.01, 42), tpchgen.generate(0.01, 42)
    planted(a)
    assert all(a[t].equals(b[t]) for t in tpchgen.TABLES)
    assert not any("Customer" in c and "Complaints" in c for c in a["supplier"]["s_comment"].to_pylist())


def test_q16_anti_removes_rows(sf001):
    """The NOT IN matters at every seed: q16 without it (same text, the subquery dropped) answers differently."""
    _, T = sf001
    db = sqlite_indexed(T)
    without = re.sub(r"AND\s+ps_suppkey\s+NOT\s+IN\s*\(SELECT.*?'%Customer%Complaints%'\)", "", query_sql("q16"), flags=re.S)
    assert "NOT IN" not in without
    assert db.execute(without).fetchall() != sqlite_subquery(db, "q16")


def test_tbl_fixtures_answer():
    """Flock's 10-row fixtures: every query runs under sqlite3; q4 and q18 agree with pyarrow."""
    T = fixture_tables()
    for q in QUERIES:
        sqlite_subquery(sqlite_indexed(T), q)
    for q in ("q4", "q18"):
        assert rows_close(sqlite_subquery(sqlite_indexed(T), q), ARROW_SUBQUERY[q](T))
