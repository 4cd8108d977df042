"""TPC-H q1, q3, q5, q6, q10, q12 and q14 without a GPU: the generator's invariants, the plans' shapes, Date32 and LIKE
through the kernels' own expression interpreter run on the host, and two independent CPU references that agree.

The references: sqlite3 runs the query texts of Flock (tests/golden/tpch/queries/qN.sql) as they are, with dates as
ISO strings (`DATE 'x'` rewritten to `'x'`) and a case-sensitive LIKE; a pyarrow restatement written from the SQL
text covers the single-join queries q1, q6, q12 and q14.  Flock's own 10-row `.tbl` fixtures (tests/golden/tpch/)
parse with Flock's schemas."""
import datetime
import math
import re
import sqlite3
from pathlib import Path

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import flock_b200 as fb
from flock_b200 import col, lit, plans, tpchgen

GOLDEN = Path(__file__).parent / "golden" / "tpch"
SEEDS = [42, 7, 1234]
QUERIES = list(plans.TPCH_QUERIES)


def query_sql(q: str) -> str:
    return (GOLDEN / "queries" / f"{q}.sql").read_text()


# ---- sqlite3: the query texts themselves ----------------------------------------------------------------------------------
def sqlite_db(tables: dict[str, pa.Table]) -> sqlite3.Connection:
    db = sqlite3.connect(":memory:")
    db.execute("PRAGMA case_sensitive_like = ON")
    for name, t in tables.items():
        cols = []
        for f in t.schema:
            a = t.column(f.name)
            if pa.types.is_date32(f.type):
                a = pc.strftime(a.cast(pa.timestamp("s")), "%Y-%m-%d")
            cols.append(a.to_pylist())
        db.execute(f"CREATE TABLE {name} ({', '.join(t.schema.names)})")
        db.executemany(f"INSERT INTO {name} VALUES ({', '.join('?' * len(cols))})", list(zip(*cols)))
    return db


def sqlite_query(db: sqlite3.Connection, q: str) -> list[tuple]:
    sql = re.sub(r"DATE\s+'([0-9-]+)'", r"'\1'", query_sql(q), flags=re.IGNORECASE)
    return db.execute(sql).fetchall()


# ---- pyarrow restatements (from the SQL text) ----------------------------------------------------------------------------
def _d(iso: str) -> pa.Scalar:
    return pa.scalar(datetime.date.fromisoformat(iso), pa.date32())


def _rev(t):
    return pc.multiply(t["l_extendedprice"], pc.subtract(1.0, t["l_discount"]))


def arrow_q1(T) -> list[tuple]:
    li = T["lineitem"].filter(pc.less_equal(T["lineitem"]["l_shipdate"], _d("1998-09-02")))
    dp = _rev(li)
    li = li.append_column("dp", dp).append_column("ch", pc.multiply(dp, pc.add(1.0, li["l_tax"])))
    g = li.group_by(["l_returnflag", "l_linestatus"]).aggregate(
        [("l_quantity", "sum"), ("l_extendedprice", "sum"), ("dp", "sum"), ("ch", "sum"), ("l_quantity", "mean"),
         ("l_extendedprice", "mean"), ("l_discount", "mean"), ("l_quantity", "count")])
    g = g.sort_by([("l_returnflag", "ascending"), ("l_linestatus", "ascending")])
    names = ["l_returnflag", "l_linestatus", "l_quantity_sum", "l_extendedprice_sum", "dp_sum", "ch_sum", "l_quantity_mean",
             "l_extendedprice_mean", "l_discount_mean", "l_quantity_count"]
    return list(zip(*[g[n].to_pylist() for n in names]))


def arrow_q6(T) -> list[tuple]:
    li = T["lineitem"]
    m = pc.and_(pc.and_(pc.greater_equal(li["l_shipdate"], _d("1994-01-01")), pc.less(li["l_shipdate"], _d("1995-01-01"))),
                pc.and_(pc.and_(pc.greater_equal(li["l_discount"], 0.06 - 0.01), pc.less_equal(li["l_discount"], 0.06 + 0.01)),
                        pc.less(li["l_quantity"], 24.0)))
    li = li.filter(m)
    return [(pc.sum(pc.multiply(li["l_extendedprice"], li["l_discount"])).as_py(),)]


def arrow_q12(T) -> list[tuple]:
    li = T["lineitem"]
    m = pc.and_(pc.and_(pc.is_in(li["l_shipmode"], pa.array(["MAIL", "SHIP"])), pc.less(li["l_commitdate"], li["l_receiptdate"])),
                pc.and_(pc.less(li["l_shipdate"], li["l_commitdate"]),
                        pc.and_(pc.greater_equal(li["l_receiptdate"], _d("1994-01-01")), pc.less(li["l_receiptdate"], _d("1995-01-01")))))
    j = li.filter(m).join(T["orders"], "l_orderkey", "o_orderkey", join_type="inner")
    high = pc.is_in(j["o_orderpriority"], pa.array(["1-URGENT", "2-HIGH"]))
    j = j.append_column("hi", pc.cast(high, pa.int64())).append_column("lo", pc.cast(pc.invert(high), pa.int64()))
    g = j.group_by("l_shipmode").aggregate([("hi", "sum"), ("lo", "sum")]).sort_by("l_shipmode")
    return list(zip(g["l_shipmode"].to_pylist(), g["hi_sum"].to_pylist(), g["lo_sum"].to_pylist()))


def arrow_q14(T) -> list[tuple]:
    li = T["lineitem"]
    li = li.filter(pc.and_(pc.greater_equal(li["l_shipdate"], _d("1995-09-01")), pc.less(li["l_shipdate"], _d("1995-10-01"))))
    j = li.join(T["part"], "l_partkey", "p_partkey", join_type="inner")
    rev = _rev(j)
    promo = pc.if_else(pc.match_like(j["p_type"], "PROMO%"), rev, 0.0)
    total = pc.sum(rev).as_py()
    return [(None if total is None else 100.0 * pc.sum(promo).as_py() / total,)]


ARROW = {"q1": arrow_q1, "q6": arrow_q6, "q12": arrow_q12, "q14": arrow_q14}


def rows_close(got: list[tuple], want: list[tuple], rel: float = 1e-9) -> bool:
    """Equal rows; floats within a relative bound (sums in another order)."""
    if len(got) != len(want):
        return False
    for g, w in zip(got, want):
        if len(g) != len(w):
            return False
        for a, b in zip(g, w):
            if isinstance(a, float) or isinstance(b, float):
                if a is None or b is None:
                    if a is not b:
                        return False
                elif not math.isclose(a, b, rel_tol=rel, abs_tol=0.0):
                    return False
            elif a != b:
                return False
    return True


@pytest.fixture(scope="module", params=SEEDS)
def sf001(request):
    return request.param, tpchgen.generate(0.01, request.param)


# ---- generator invariants ------------------------------------------------------------------------------------------------
def test_generator_invariants(sf001):
    seed, T = sf001
    card = tpchgen.cardinalities(0.01)
    for t in ("part", "supplier", "customer", "orders", "nation", "region"):
        assert T[t].num_rows == card[t]
    for t, sch in tpchgen.SCHEMAS.items():
        assert T[t].schema.names == sch.names and T[t].schema.types == sch.types
    od, li, pt = T["orders"], T["lineitem"], T["part"]
    ok = od["o_orderkey"].to_numpy()
    assert np.all(((ok - 1) % 32) < 8) and np.all(np.diff(ok) > 0)
    assert np.all(od["o_custkey"].to_numpy() % 3 != 0)
    d = lambda c: li[c].cast(pa.int32()).to_numpy()
    odate = od["o_orderdate"].cast(pa.int32()).to_numpy()
    assert odate.min() >= tpchgen.STARTDATE and odate.max() <= tpchgen.ENDDATE - 151
    order_date = dict(zip(ok.tolist(), odate.tolist()))
    lo = np.array([order_date[k] for k in li["l_orderkey"].to_pylist()])
    ship, commit, receipt = d("l_shipdate"), d("l_commitdate"), d("l_receiptdate")
    assert np.all((ship - lo >= 1) & (ship - lo <= 121)) and np.all((commit - lo >= 30) & (commit - lo <= 90))
    assert np.all((receipt - ship >= 1) & (receipt - ship <= 30))
    status = np.array(li["l_linestatus"].to_pylist())
    assert np.array_equal(status == "O", ship > tpchgen.CURRENTDATE)
    flag = np.array(li["l_returnflag"].to_pylist())
    assert np.all((flag == "N") == (receipt > tpchgen.CURRENTDATE)) and set(flag[receipt <= tpchgen.CURRENTDATE]) <= {"R", "A"}
    q = li["l_quantity"].to_numpy()
    assert q.min() >= 1 and q.max() <= 50 and np.all(q == np.round(q))
    disc, tax = li["l_discount"].to_numpy(), li["l_tax"].to_numpy()
    assert disc.min() >= 0 and disc.max() <= 0.10 + 1e-12 and tax.min() >= 0 and tax.max() <= 0.08 + 1e-12
    pk = pt["p_partkey"].to_numpy()
    assert np.array_equal(np.round(pt["p_retailprice"].to_numpy() * 100), tpchgen.retailprice_cents(pk))
    lp = li["l_partkey"].to_numpy().astype(np.int64)
    assert np.allclose(li["l_extendedprice"].to_numpy(), q * tpchgen.retailprice_cents(lp) / 100.0)
    # every line's supplier is one of its part's four partsupp suppliers
    ps = set(zip(T["partsupp"]["ps_partkey"].to_pylist(), T["partsupp"]["ps_suppkey"].to_pylist()))
    assert all(pair in ps for pair in zip(lp.tolist(), li["l_suppkey"].to_pylist()))
    assert set(T["customer"]["c_mktsegment"].to_pylist()) <= set(tpchgen.SEGMENTS)
    assert set(od["o_orderpriority"].to_pylist()) <= set(tpchgen.PRIORITIES)
    assert set(li["l_shipmode"].to_pylist()) <= set(tpchgen.SHIPMODES)
    assert all(t.startswith(("STANDARD", "SMALL", "MEDIUM", "LARGE", "ECONOMY", "PROMO")) for t in pt["p_type"].to_pylist()[:200])
    # O_ORDERSTATUS from the lines
    lines = li.group_by("l_orderkey").aggregate([("l_linestatus", "distinct")])
    statuses = dict(zip(lines["l_orderkey"].to_pylist(), lines["l_linestatus_distinct"].to_pylist()))
    for k, s in list(zip(ok.tolist(), od["o_orderstatus"].to_pylist()))[:500]:
        assert s == ("P" if len(statuses[k]) == 2 else "F" if statuses[k] == ["F"] else "O")
    assert [r for _, r in tpchgen.NATIONS] == T["nation"]["n_regionkey"].to_pylist() and len(tpchgen.REGIONS) == 5


def test_generator_is_seeded_and_projects():
    a = tpchgen.generate(0.002, 7, columns={"lineitem": ["l_shipdate", "l_quantity"]})
    b = tpchgen.generate(0.002, 7)
    assert list(a) == ["lineitem"] and a["lineitem"].schema.names == ["l_shipdate", "l_quantity"]
    assert a["lineitem"].equals(b["lineitem"].select(["l_shipdate", "l_quantity"]))
    assert not tpchgen.generate(0.002, 8)["lineitem"].equals(b["lineitem"])


# ---- plan shapes ----------------------------------------------------------------------------------------------------------
def _nodes(p: dict, out=None) -> list[str]:
    out = [] if out is None else out
    out.append(p["execution_plan"])
    for k in ("input", "left", "right"):
        if k in p:
            _nodes(p[k], out)
    return out


@pytest.mark.parametrize("q", QUERIES)
def test_plan_shape(q):
    p = plans.TPCH_QUERIES[q]()
    kinds = _nodes(p)
    assert kinds.count("memory_exec") == len(plans.TPCH_SOURCES[q])
    assert kinds.count("hash_join_exec") == len(plans.TPCH_SOURCES[q]) - 1
    assert kinds[0] == ("projection_exec" if q in ("q6", "q14") else "sort_exec")
    aggs = [k for k in kinds if k == "hash_aggregate_exec"]
    assert len(aggs) == 2


def test_q6_between_is_float_literal_arithmetic():
    # 0.06 + 0.01 is 0.06999999999999999 in binary64: a discount of exactly 0.07 is outside q6's BETWEEN (sqlite agrees)
    assert 0.06 + 0.01 < 0.07
    db = sqlite3.connect(":memory:")
    assert db.execute("SELECT 0.07 BETWEEN .06 - 0.01 AND .06 + 0.01, 0.05 BETWEEN .06 - 0.01 AND .06 + 0.01").fetchone() == (0, 1)


# ---- Date32 and LIKE through the kernels' interpreter on the host -------------------------------------------------------
def test_date32_predicate_has_the_int32_kind():
    days = pa.array([0, 10470, 10471, 10472, -5, 20000], pa.date32())
    ints = pa.array([0, 10470, 10471, 10472, -5, 20000], pa.int32())
    for cmp in ("__le__", "__lt__", "__gt__", "__ge__", "__eq__", "__ne__"):
        dm, dk = fb.selftest_eval_predicate(pa.record_batch([days], ["d"]), getattr(col(0), cmp)(lit(10471, "date32")))
        im, ik = fb.selftest_eval_predicate(pa.record_batch([ints], ["d"]), getattr(col(0), cmp)(lit(10471, "int32")))
        assert dk == ik == 2 and list(dm) == list(im)


def test_date32_tree_values_and_refusals():
    days = pa.array([1, None, 10471, -3], pa.date32())
    b = pa.record_batch([days, pa.array([1, 2, 3, 4], pa.int32())], ["d", "i"])
    (res, _) = fb.selftest_eval_tree(b, [fb.case([(col(1) > 2, col(0))], lit(7, "date32"))])
    vals, valid, dt = res[0]
    assert dt == fb.DATE32 and list(valid) == [True, True, True, True] and vals.tolist() == [7, 7, 10471, -3]
    mask, _ = fb.selftest_eval_tree(b, col(0).isin([lit(1, "date32"), lit(-3, "date32")]), predicate=True)
    assert list(mask) == [True, False, False, True]
    for bad in (col(0) + 1, col(0).cast("int32"), -col(0), col(0) < lit(3, "int32")):
        with pytest.raises(fb.FlockGpuError) as e:
            fb.selftest_eval_tree(b, [bad])
        assert e.value.code == -2 and "Date32" in str(e.value)


LIKE_STRINGS = ["", "a", "ab", "abc", "PROMO BRUSHED TIN", "STANDARD PROMO", "promo x", "é", "aé", "éa", "日本語", "a%b", "a_b",
                "xxabxxab", "abab", None]
LIKE_PATTERNS = ["%", "", "_", "__", "a%", "%a", "%b%", "a_c", "_%_", "PROMO%", "%PROMO%", "%o_", "é", "_a", "a_", "%é%",
                 "日_語", "___", "%ab", "ab%ab", "%a%b%"]


@pytest.mark.parametrize("negated", [False, True])
def test_like_matches_arrow(negated):
    s = pa.array(LIKE_STRINGS, pa.utf8())
    b = pa.record_batch([s], ["s"])
    for p in LIKE_PATTERNS:
        (res, _) = fb.selftest_eval_tree(b, [fb.case([(col(0).like(p, negated), lit(1))], lit(0))])
        vals, valid, _ = res[0]
        want = pc.match_like(s, p)
        if negated:
            want = pc.invert(want)
        want = [0 if w is None else int(w) for w in want.to_pylist()]   # CASE: a NULL condition falls through to 0
        assert vals.tolist() == want, p
        mask, _ = fb.selftest_eval_tree(b, col(0).like(p, negated), predicate=True)
        assert [bool(w) for w in want] == list(mask), p


def test_like_refusals():
    b = pa.record_batch([pa.array(["a"]), pa.array([1], pa.int32())], ["s", "i"])
    with pytest.raises(fb.FlockGpuError) as e:
        fb.selftest_eval_tree(b, col(1).like("1%"), predicate=True)
    assert e.value.code == -2
    with pytest.raises(fb.FlockGpuError) as e:
        fb.selftest_eval_tree(b, fb.E(col(0).tokens + col(0).tokens + [(fb.OP_LIKE, 0, 0, 0, 0.0, None)]), predicate=True)
    assert e.value.code == -2 and "pattern" in str(e.value)
    mask, _ = fb.selftest_eval_tree(b, col(0).like(None), predicate=True)
    assert list(mask) == [False]


# ---- two independent CPU references agree -----------------------------------------------------------------------------------
@pytest.mark.parametrize("q", ["q1", "q6", "q12", "q14"])
def test_sqlite_equals_arrow(sf001, q):
    _, T = sf001
    assert rows_close(sqlite_query(sqlite_db(T), q), ARROW[q](T))


@pytest.mark.parametrize("q", QUERIES)
def test_sqlite_answers_are_not_empty(sf001, q):
    _, T = sf001
    got = sqlite_query(sqlite_db(T), q)
    assert got and got[0][0] is not None


# ---- Flock's .tbl fixtures ----------------------------------------------------------------------------------------------------
def read_tbl(table: str) -> pa.Table:
    """Flock's '|'-separated fixtures (trailing '|') with Flock's schemas."""
    sch = tpchgen.schema(table)
    files = sorted(GOLDEN.glob(f"{table}_*.tbl")) or [GOLDEN / f"{table}.tbl"]
    rows = [line.rstrip("\n").split("|")[:len(sch)] for f in files for line in f.read_text().splitlines() if line]
    cols = []
    for i, f in enumerate(sch):
        vals = [r[i] for r in rows]
        if pa.types.is_int32(f.type):
            cols.append(pa.array([int(v) for v in vals], pa.int32()))
        elif pa.types.is_float64(f.type):
            cols.append(pa.array([float(v) for v in vals], pa.float64()))
        elif pa.types.is_date32(f.type):
            cols.append(pa.array([datetime.date.fromisoformat(v) for v in vals], pa.date32()))
        else:
            cols.append(pa.array(vals, pa.utf8()))
    return pa.table(cols, schema=sch)


def fixture_tables() -> dict[str, pa.Table]:
    return {t: read_tbl(t) for t in tpchgen.TABLES}


def test_tbl_fixtures_parse():
    T = fixture_tables()
    assert {t: T[t].num_rows for t in T} == {"part": 10, "supplier": 10, "partsupp": 10, "customer": 10, "orders": 10,
                                             "lineitem": 20, "nation": 10, "region": 5}
    assert T["lineitem"]["l_shipdate"][0].as_py() == datetime.date(1996, 3, 13)
    # known answers of the fixtures, pinned: q1's three groups; no fixture line passes q6's filter (SUM over no row)
    q1 = [("A", "F", 54.0, 79781.76, 74994.8544, 80244.494208, 27.0, 39890.88, 0.06, 2),
          ("N", "O", 366.0, 453111.46, 423755.3792, 441189.380304, 26.142857142857142, 32365.104285714286, 0.07, 14),
          ("R", "F", 188.0, 201709.04, 185862.78, 185862.78, 47.0, 50427.26, 0.08, 4)]
    for got in (sqlite_query(sqlite_db(T), "q1"), arrow_q1(T)):
        assert rows_close(got, q1, rel=1e-12)
    assert sqlite_query(sqlite_db(T), "q6") == [(None,)] and arrow_q6(T) == [(None,)]

