"""TPC-H q7, q8 and q9 without a GPU: EXTRACT / date_part through the kernels' own register-program interpreter run on
the host against a pure-integer reference, its refusals, the plan reader's scalar function, the generator's P_NAME, the
plans' shapes, and two independent CPU references that agree.

The references: sqlite3 runs Flock's query texts (tests/golden/tpch/queries/q7.sql ...) with `DATE 'x'` written as
`'x'` and `EXTRACT(YEAR FROM c)` as `CAST(strftime('%Y', c) AS INTEGER)` (sqlite has no EXTRACT); a pyarrow
restatement of each query is written from the SQL text.  The date_part reference is itself checked against `datetime`,
numpy's datetime64 and pyarrow's temporal kernels."""
import datetime
import hashlib
import json
import math
import re

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import flock_b200 as fb
from flock_b200 import col, lit, case, plans, tpchgen
from test_tpch_host import GOLDEN, SEEDS, fixture_tables, sqlite_db

QUERIES = list(plans.TPCH_MORE_QUERIES)
I32_MIN, I32_MAX = -(1 << 31), (1 << 31) - 1
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


# ---- the date_part reference: Python integers, floor division ------------------------------------------------------------
UNITS = {"date32": 1, "s": 86400, "ms": 86400 * 10**3, "us": 86400 * 10**6, "ns": 86400 * 10**9}   # units per day


def days_from_civil(y: int, m: int, d: int) -> int:
    y -= m <= 2
    era = y // 400
    yoe = y - era * 400
    doy = (153 * (m + (-3 if m > 2 else 9)) + 2) // 5 + d - 1
    return era * 146097 + yoe * 365 + yoe // 4 - yoe // 100 + doy - 719468


def year_of_day(day: int) -> int:
    """The proleptic Gregorian year holding `day`, by counting 400-year eras and then years: independent of the
    closed form the kernels use."""
    era, rest = divmod(day - days_from_civil(0, 1, 1), 146097)
    y = era * 400
    while True:
        n = 366 if (y % 4 == 0 and (y % 100 != 0 or y % 400 == 0)) else 365
        if rest < n:
            return y
        rest -= n
        y += 1


def ref_date_part(field: str, unit: str, v):
    if v is None:
        return None
    day, rem = divmod(v, UNITS[unit])
    if field == "hour":
        return rem // (UNITS[unit] // 24) if unit != "date32" else 0
    y = year_of_day(day)
    return y if I32_MIN <= y <= I32_MAX else None


def edge_days() -> list[int]:
    days = [I32_MIN, I32_MAX, days_from_civil(2000, 2, 29), days_from_civil(2400, 2, 29), -1, 0, 1,
            days_from_civil(0, 1, 1) - 1, days_from_civil(0, 1, 1), days_from_civil(0, 1, 1) + 1]
    for y in (-1, 0, 1900, 1969, 1970, 2000, 2100):
        days += [days_from_civil(y, 1, 1), days_from_civil(y, 12, 31)]
    return days


def edge_values(unit: str) -> list[int]:
    per_day = UNITS[unit]
    if unit == "date32":
        return edge_days()
    vals = [I64_MIN, I64_MIN + 1, I64_MAX, -1, 0, 1, per_day * days_from_civil(0, 1, 1) - 1, per_day * days_from_civil(0, 1, 1),
            per_day * days_from_civil(0, 1, 1) + 1]
    for d in edge_days():
        for off in (0, per_day // 24 * 23, per_day - 1):   # hours 0 and 23, the last unit of the day
            vals.append(d * per_day + off)
    return [v for v in vals if I64_MIN <= v <= I64_MAX]


def edge_batch(unit: str, nullable: bool) -> pa.RecordBatch:
    vals = edge_values(unit)
    mask = [nullable and i % 3 == 1 for i in range(len(vals))]
    typ = pa.date32() if unit == "date32" else pa.timestamp(unit)
    data = pa.array(vals, pa.int32() if unit == "date32" else pa.int64(), mask=np.array(mask)).cast(typ) if nullable else \
        pa.array(vals, pa.int32() if unit == "date32" else pa.int64()).cast(typ)
    ints = pa.array(np.arange(len(vals), dtype=np.int32) % 7 + 1995)
    return pa.record_batch([data, ints], ["t", "i"])


def column_ints(b: pa.RecordBatch, i: int = 0) -> list:
    a = b.column(i)
    return a.cast(pa.int32() if pa.types.is_date32(a.type) else pa.int64()).to_pylist()


# ---- the reference checked against datetime, numpy and pyarrow ------------------------------------------------------------
def test_reference_against_datetime():
    rng = np.random.default_rng(1)
    epoch = datetime.date(1970, 1, 1).toordinal()
    lo, hi = datetime.date(1, 1, 1).toordinal() - epoch, datetime.date(9999, 12, 31).toordinal() - epoch
    for d in [lo, hi] + rng.integers(lo, hi + 1, 3000).tolist() + [x for x in edge_days() if lo <= x <= hi]:
        assert year_of_day(d) == datetime.date.fromordinal(d + epoch).year, d
        assert days_from_civil(*datetime.date.fromordinal(d + epoch).timetuple()[:3]) == d


@pytest.mark.parametrize("unit", list(UNITS))
def test_reference_against_numpy(unit):
    """numpy's datetime64 casts to a coarser unit by floor division (NaT = INT64_MIN aside).  Its hours need the start of
    the day in the value's own unit, which INT64_MIN + 1 s, ms and us do not have."""
    vals = [v for v in edge_values(unit) if v != I64_MIN]
    np_unit = "D" if unit == "date32" else unit
    a = np.array(vals, np.int64).astype(f"datetime64[{np_unit}]")
    years = a.astype("datetime64[Y]").astype(np.int64) + 1970
    hours = (a.astype("datetime64[h]") - a.astype("datetime64[D]")).astype(np.int64)
    for v, y, h in zip(vals, years.tolist(), hours.tolist()):
        assert ref_date_part("year", unit, v) == (y if I32_MIN <= y <= I32_MAX else None), (unit, v)
        if v // UNITS[unit] * UNITS[unit] >= I64_MIN:
            assert ref_date_part("hour", unit, v) == h, (unit, v)


@pytest.mark.parametrize("unit", list(UNITS))
def test_reference_against_arrow(unit):
    rng = np.random.default_rng(2)
    per_day = UNITS[unit]
    days = rng.integers(days_from_civil(1700, 1, 1), days_from_civil(2250, 1, 1), 2000)
    vals = (days * per_day + rng.integers(0, per_day, 2000)).tolist()
    a = pa.array(vals, pa.int32() if unit == "date32" else pa.int64()).cast(pa.date32() if unit == "date32" else pa.timestamp(unit))
    assert pc.year(a).to_pylist() == [ref_date_part("year", unit, v) for v in vals]
    if unit != "date32":
        assert pc.hour(a).to_pylist() == [ref_date_part("hour", unit, v) for v in vals]


# ---- date_part through the host build of the kernels' interpreter ---------------------------------------------------------
@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("unit", list(UNITS))
def test_date_part_matches_the_reference(unit, nullable):
    b = edge_batch(unit, nullable)
    vals = column_ints(b)
    (year, hour, upper), n_instr = fb.selftest_eval_tree(b, [col(0).extract("year"), col(0).extract("hour"), col(0).extract("YEAR")])
    for (v, valid, dt), field in ((year, "year"), (hour, "hour"), (upper, "year")):
        assert dt == fb.INT32
        want = [ref_date_part(field, unit, x) for x in vals]
        assert list(valid) == [w is not None for w in want], (unit, field)
        assert [int(x) if ok else None for x, ok in zip(v, valid)] == want, (unit, field)
    assert n_instr == 1 + 2 + 3   # one load, two date_parts ("year" and "YEAR" are one node), three stores


def test_date_part_roles():
    b = edge_batch("date32", True)
    vals = column_ints(b)
    ints = b.column(1).to_pylist()
    years = [ref_date_part("year", "date32", v) for v in vals]
    mask, _ = fb.selftest_eval_tree(b, col(0).extract("year") == col(1), predicate=True)
    assert list(mask) == [y is not None and y == i for y, i in zip(years, ints)]
    mask, _ = fb.selftest_eval_tree(b, col(0).extract("year") >= lit(1970, "int32"), predicate=True)
    assert list(mask) == [y is not None and y >= 1970 for y in years]
    (c, a, m), _ = fb.selftest_eval_tree(b, [case([(col(0).extract("year") < 1970, lit(1))], lit(0)),
                                              col(0).extract("year") + 1, col(0).extract("year").cast("int64") * col(1).cast("int64")])
    assert c[0].tolist() == [1 if y is not None and y < 1970 else 0 for y in years]
    assert [int(x) if ok else None for x, ok in zip(*a[:2])] == [None if y is None else y + 1 for y in years]
    assert [int(x) if ok else None for x, ok in zip(*m[:2])] == [None if y is None else y * i for y, i in zip(years, ints)]


def refused(fn):
    with pytest.raises(fb.FlockGpuError) as e:
        fn()
    assert e.value.code == -2, str(e.value)
    return str(e.value)


def test_date_part_refusals():
    d = pa.record_batch([pa.array([1], pa.date32())], ["d"])
    assert "field 3" in refused(lambda: fb.selftest_eval_tree(d, [col(0).extract(3)]))
    tz = pa.record_batch([pa.array([1], pa.int64()).cast(pa.timestamp("ns", "UTC"))], ["t"])
    assert plans.TS_NS_UTC == plans.data_type_json(tz.schema.field(0).type)
    assert "UTC" in refused(lambda: fb.selftest_eval_tree(tz, [col(0).extract("year")]))
    for typ, name in ((pa.int64(), "Int64"), (pa.utf8(), "Utf8")):
        b = pa.record_batch([pa.array([1 if typ == pa.int64() else "1"], typ)], ["x"])
        assert name in refused(lambda: fb.selftest_eval_tree(b, [col(0).extract("year")]))
    assert "Timestamp" in refused(lambda: fb.selftest_eval_tree(d, [lit(5, "timestamp").extract("year")]))


# ---- the plan reader ------------------------------------------------------------------------------------------------------
def _plan_with(expr: dict) -> dict:
    sch = pa.schema([("d", pa.date32()), ("t", pa.timestamp("ms"))])
    return plans.projection_exec([(expr, "y")], plans.memory_exec(sch, None))


def test_plan_refusals():
    d = plans.column("d", 0)
    month = plans.date_part("MONTH", d)
    assert "MONTH" in refused(lambda: fb.ExecutionContext(None, _plan_with(month)))
    non_literal = dict(plans.date_part("YEAR", d), args=[plans.column("t", 1), d])
    assert "date_part" in refused(lambda: fb.ExecutionContext(None, _plan_with(non_literal)))
    other = {"physical_expr": "scalar_function_expr", "fun": "ToTimestamp", "name": "to_timestamp", "args": [d], "return_type": "Int64"}
    assert "ToTimestamp" in refused(lambda: fb.ExecutionContext(None, _plan_with(other)))
    by_name = {"physical_expr": "scalar_function", "name": "upper", "args": [d]}
    assert "upper" in refused(lambda: fb.ExecutionContext(None, _plan_with(by_name)))


def test_plan_str_and_unmarshal():
    for tag, extra in (("scalar_function_expr", {}), ("scalar_function", {}), ("scalar_function_expr", {"fun": None, "name": "datepart"})):
        e = dict(plans.date_part("year", plans.column("t", 1)), physical_expr=tag, **extra)
        if e.get("fun") is None:
            e.pop("fun")
        ec = fb.ExecutionContext(None, _plan_with(e))
        assert "date_part(year, t@1) as y" in ec.plan_str(0)
        ec.close()
    ec = fb.ExecutionContext(None, json.dumps(plans.tpch_q7()))
    s = ec.plan_str(0)
    ec.close()
    assert "date_part(YEAR, l_shipdate@6) as l_year" in s and "n_name@12 as supp_nation, n_name@14 as cust_nation" in s


# ---- the generator: P_NAME, and every other column as it was ----------------------------------------------------------------
# sha256 over each table's columns but p_name (column_digest), computed before P_NAME changed: SF 0.01, seed 42
TABLE_DIGESTS = {
    "region": "e36a871a27cb102f3aaf46618a08a20d",
    "nation": "d47924212c292e073fdaf0371a33b694",
    "part": "c4e5c2fff47bf230e7adb2092acf6ef5",
    "supplier": "8497306832ad5c4cfaa64f6063ee146d",
    "partsupp": "5f2324b3b0345ea0a4dc7e58ff363ff2",
    "customer": "fd6d4bbe6135c12d67d6928edab3c4f0",
    "lineitem": "34889262c9e7440dc21d1edad0afb759",
    "orders": "af0519a4fc3b10b2aba7bd8dce58cc0f",
}


def column_digest(a) -> str:
    a = a.combine_chunks() if isinstance(a, pa.ChunkedArray) else a
    if pa.types.is_string(a.type):
        data = "\x00".join(a.to_pylist()).encode()
    else:
        data = (a.cast(pa.int32()) if pa.types.is_date32(a.type) else a).to_numpy(zero_copy_only=False).tobytes()
    return hashlib.sha256(data).hexdigest()[:16]


def test_generator_keeps_every_other_column():
    T = tpchgen.generate(0.01, 42)
    for t, tab in T.items():
        h = hashlib.sha256()
        for n in tab.schema.names:
            if n != "p_name":
                h.update(n.encode() + column_digest(tab[n]).encode())
        assert h.hexdigest()[:32] == TABLE_DIGESTS[t], t


@pytest.mark.parametrize("seed", SEEDS)
def test_part_names(seed):
    assert len(tpchgen.COLORS) == 92 == len(set(tpchgen.COLORS)) and "green" in tpchgen.COLORS
    names = tpchgen.generate(0.01, seed, columns={"part": ["p_name"]})["part"]["p_name"].to_pylist()
    words = [n.split(" ") for n in names]
    assert all(len(w) == 5 == len(set(w)) and set(w) <= set(tpchgen.COLORS) for w in words)
    assert sum("green" in w for w in words) > 0
    assert names == tpchgen.generate(0.01, seed)["part"]["p_name"].to_pylist()


# ---- plan shapes ----------------------------------------------------------------------------------------------------------
def _walk(p: dict):
    yield p
    for k in ("input", "left", "right"):
        if k in p:
            yield from _walk(p[k])


SORT_KEYS = {"q7": [("supp_nation", False), ("cust_nation", False), ("l_year", False)], "q8": [("o_year", False)],
             "q9": [("nation", False), ("o_year", True)]}
SUBQUERY = {"q7": ["supp_nation", "cust_nation", "l_year", "volume"], "q8": ["o_year", "volume", "nation"], "q9": ["nation", "o_year", "amount"]}


@pytest.mark.parametrize("q", QUERIES)
def test_plan_shape(q):
    p = plans.TPCH_MORE_QUERIES[q]()
    kinds = [n["execution_plan"] for n in _walk(p)]
    assert kinds.count("memory_exec") == len(plans.TPCH_MORE_SOURCES[q])
    assert kinds.count("hash_join_exec") == len(plans.TPCH_MORE_SOURCES[q]) - 1
    assert kinds[0] == "sort_exec" and kinds.count("hash_aggregate_exec") == 2
    assert [(k["expr"]["name"], k["options"]["descending"]) for k in p["expr"]] == SORT_KEYS[q]
    partial = next(n for n in _walk(p) if n["execution_plan"] == "hash_aggregate_exec" and n["mode"] == "Partial")
    sub = partial["input"]
    assert sub["execution_plan"] == "projection_exec" and [nm for _, nm in sub["expr"]] == SUBQUERY[q]
    assert kinds.count("filter_exec") == {"q7": 2, "q8": 3, "q9": 1}[q]


# ---- two independent references ---------------------------------------------------------------------------------------------
def sqlite_more(db, q: str) -> list[tuple]:
    sql = (GOLDEN / "queries" / f"{q}.sql").read_text()
    sql = re.sub(r"DATE\s+'([0-9-]+)'", r"'\1'", sql, flags=re.IGNORECASE)
    sql = re.sub(r"extract\s*\(\s*year\s+from\s+(\w+)\s*\)", r"CAST(strftime('%Y', \1) AS INTEGER)", sql, flags=re.IGNORECASE)
    return db.execute(sql).fetchall()


def _d(iso: str) -> pa.Scalar:
    return pa.scalar(datetime.date.fromisoformat(iso), pa.date32())


def _between(a, lo, hi):
    return pc.and_(pc.greater_equal(a, _d(lo)), pc.less_equal(a, _d(hi)))


def _rev(t):
    return pc.multiply(t["l_extendedprice"], pc.subtract(1.0, t["l_discount"]))


def _nation(T, cols, names):
    return T["nation"].select(cols).rename_columns(names)


def _grouped(t: pa.Table, keys: list[str], sums: list[str]) -> pa.Table:
    """SUM of each of `sums` per group, with the sum of magnitudes (`x_abs`) and the addend count (`n`)."""
    for s in sums:
        t = t.append_column(s + "_abs", pc.abs(t[s]))
    g = t.group_by(keys).aggregate([(s, "sum") for s in sums] + [(s + "_abs", "sum") for s in sums] + [(sums[0], "count")])
    return g.rename_columns([c[:-4] if c.endswith("_sum") else "n" if c.endswith("_count") else c for c in g.column_names])


def arrow_q7(T) -> pa.Table:
    li = T["lineitem"].filter(_between(T["lineitem"]["l_shipdate"], "1995-01-01", "1996-12-31"))
    j = li.join(T["supplier"].select(["s_suppkey", "s_nationkey"]), "l_suppkey", "s_suppkey", join_type="inner")
    j = j.join(T["orders"].select(["o_orderkey", "o_custkey"]), "l_orderkey", "o_orderkey", join_type="inner")
    j = j.join(T["customer"].select(["c_custkey", "c_nationkey"]), "o_custkey", "c_custkey", join_type="inner")
    j = j.join(_nation(T, ["n_nationkey", "n_name"], ["n1", "supp_nation"]), "s_nationkey", "n1", join_type="inner")
    j = j.join(_nation(T, ["n_nationkey", "n_name"], ["n2", "cust_nation"]), "c_nationkey", "n2", join_type="inner")
    s, c = j["supp_nation"], j["cust_nation"]
    j = j.filter(pc.or_(pc.and_(pc.equal(s, "FRANCE"), pc.equal(c, "GERMANY")), pc.and_(pc.equal(s, "GERMANY"), pc.equal(c, "FRANCE"))))
    j = j.append_column("l_year", pc.year(j["l_shipdate"])).append_column("volume", _rev(j))
    g = _grouped(j, ["supp_nation", "cust_nation", "l_year"], ["volume"])
    g = g.sort_by([("supp_nation", "ascending"), ("cust_nation", "ascending"), ("l_year", "ascending")])
    return g.select(["supp_nation", "cust_nation", "l_year", "volume", "volume_abs", "n"])


def arrow_q8(T) -> pa.Table:
    pt = T["part"].filter(pc.equal(T["part"]["p_type"], "ECONOMY ANODIZED STEEL")).select(["p_partkey"])
    od = T["orders"].filter(_between(T["orders"]["o_orderdate"], "1995-01-01", "1996-12-31")).select(["o_orderkey", "o_custkey", "o_orderdate"])
    re_ = T["region"].filter(pc.equal(T["region"]["r_name"], "AMERICA")).select(["r_regionkey"])
    j = T["lineitem"].select(["l_orderkey", "l_partkey", "l_suppkey", "l_extendedprice", "l_discount"])
    j = j.join(pt, "l_partkey", "p_partkey", join_type="inner")
    j = j.join(T["supplier"].select(["s_suppkey", "s_nationkey"]), "l_suppkey", "s_suppkey", join_type="inner")
    j = j.join(od, "l_orderkey", "o_orderkey", join_type="inner")
    j = j.join(T["customer"].select(["c_custkey", "c_nationkey"]), "o_custkey", "c_custkey", join_type="inner")
    j = j.join(_nation(T, ["n_nationkey", "n_regionkey"], ["n1", "n1_region"]), "c_nationkey", "n1", join_type="inner")
    j = j.join(re_, "n1_region", "r_regionkey", join_type="inner")
    j = j.join(_nation(T, ["n_nationkey", "n_name"], ["n2", "nation"]), "s_nationkey", "n2", join_type="inner")
    vol = _rev(j)
    j = j.append_column("o_year", pc.year(j["o_orderdate"])).append_column("volume", vol)
    j = j.append_column("brazil", pc.if_else(pc.equal(j["nation"], "BRAZIL"), vol, 0.0))
    g = _grouped(j, ["o_year"], ["brazil", "volume"]).sort_by("o_year")
    g = g.append_column("mkt_share", pc.divide(g["brazil"], g["volume"]))
    return g.select(["o_year", "mkt_share", "brazil", "volume", "brazil_abs", "volume_abs", "n"])


def arrow_q9(T) -> pa.Table:
    pt = T["part"].filter(pc.match_like(T["part"]["p_name"], "%green%")).select(["p_partkey"])
    j = T["lineitem"].select(["l_orderkey", "l_partkey", "l_suppkey", "l_quantity", "l_extendedprice", "l_discount"])
    j = j.join(pt, "l_partkey", "p_partkey", join_type="inner")
    j = j.join(T["supplier"].select(["s_suppkey", "s_nationkey"]), "l_suppkey", "s_suppkey", join_type="inner")
    j = j.join(T["partsupp"].select(["ps_partkey", "ps_suppkey", "ps_supplycost"]), ["l_suppkey", "l_partkey"], ["ps_suppkey", "ps_partkey"],
               join_type="inner")
    j = j.join(T["orders"].select(["o_orderkey", "o_orderdate"]), "l_orderkey", "o_orderkey", join_type="inner")
    j = j.join(_nation(T, ["n_nationkey", "n_name"], ["n", "nation"]), "s_nationkey", "n", join_type="inner")
    amount = pc.subtract(_rev(j), pc.multiply(j["ps_supplycost"], j["l_quantity"]))
    j = j.append_column("o_year", pc.year(j["o_orderdate"])).append_column("amount", amount)
    g = _grouped(j, ["nation", "o_year"], ["amount"]).sort_by([("nation", "ascending"), ("o_year", "descending")])
    return g.select(["nation", "o_year", "amount", "amount_abs", "n"])


ARROW_MORE = {"q7": arrow_q7, "q8": arrow_q8, "q9": arrow_q9}
N_OUT = {"q7": 4, "q8": 2, "q9": 3}   # the query's own columns; the rest are the error-bound terms


def arrow_rows(q: str, t: pa.Table) -> list[tuple]:
    return [tuple(r[:N_OUT[q]]) for r in zip(*[c.to_pylist() for c in t.columns])] if t.num_rows else []


def sum_bound(abs_sum: float, n: int) -> float:
    """|a - b| for two Float64 sums of the same n addends in any order: each within (n - 1) u sum|x| of the exact sum
    (u = 2^-53), plus a few roundings of the products the addends are."""
    u = 2.0 ** -53
    return 2 * (max(n - 1, 1) + 4) * u * abs_sum


def value_interval(q: str, r: dict) -> tuple[float, float]:
    """Where any evaluation order puts the group's value: each SUM within sum_bound of the restatement's; q8's ratio
    within the bounds of its numerator and denominator, and the division's rounding."""
    if q == "q8":
        num, den = r["brazil"], r["volume"]
        en, ed = sum_bound(r["brazil_abs"], r["n"]), sum_bound(r["volume_abs"], r["n"])
        lo = (num - en) / (den + ed) if num - en >= 0 else (num - en) / (den - ed)
        hi = (num + en) / (den - ed)
        return lo - abs(lo) * 2.0 ** -51, hi + abs(hi) * 2.0 ** -51
    v = r["volume" if q == "q7" else "amount"]
    e = sum_bound(r["volume_abs" if q == "q7" else "amount_abs"], r["n"])
    return v - e, v + e


def assert_within_bounds(q: str, got: list[tuple], want: pa.Table):
    """Per group: the restatement's keys exactly, and a value within value_interval."""
    assert len(got) == want.num_rows, (q, len(got), want.num_rows)
    for g, r in zip(got, want.to_pylist()):
        keys = list(r.values())[:N_OUT[q] - 1]
        assert list(g[:len(keys)]) == keys, (q, g, r)
        lo, hi = value_interval(q, r)
        assert lo <= g[N_OUT[q] - 1] <= hi, (q, g, r)


@pytest.fixture(scope="module", params=SEEDS)
def sf001(request):
    return request.param, tpchgen.generate(0.01, request.param)


@pytest.mark.parametrize("q", QUERIES)
def test_sqlite_equals_arrow(sf001, q):
    seed, T = sf001
    got = sqlite_more(sqlite_db(T), q)
    want = ARROW_MORE[q](T)
    assert_within_bounds(q, got, want)
    if q == "q9":
        assert got, seed                                    # P_NAME holds "green": q9 is not empty


@pytest.mark.parametrize("q", QUERIES)
def test_tbl_fixtures_are_empty(q):
    T = fixture_tables()
    assert sqlite_more(sqlite_db(T), q) == [] and ARROW_MORE[q](T).num_rows == 0


def test_sum_bound_holds_for_negative_addends():
    """q9's amounts change sign: a relative bound on the result would not hold, the bound on sum|x| does."""
    x = np.array([1e16, 1.0, -1e16, 3.0, -2.5])
    exact = math.fsum(x)
    for perm in ([0, 1, 2, 3, 4], [1, 3, 4, 0, 2], [0, 2, 1, 3, 4]):
        s = 0.0
        for i in perm:
            s += x[i]
        assert abs(s - exact) <= sum_bound(float(np.abs(x).sum()), len(x))
