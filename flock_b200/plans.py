"""NEXMark physical plans in the reference's own serde-JSON plan format.

The reference serialises ``Arc<dyn ExecutionPlan>`` with typetag tags ("execution_plan": "filter_exec",
"physical_expr": "binary_expr", ...; fixtures flock/src/tests/data/plan/{simple_select,aggregate,join}.json)
and ships the string in the Lambda environment (flock/src/runtime/context.rs:366-398).  No Rust
toolchain exists here, so these builders write the same JSON by hand, following the physical plans the
reference's own tests print (flock/src/distributed_plan/planner.rs:86-255) and SURVEY.md Appendix B.
Both the GPU executor (flock_b200.ExecutionContext) and the CPU oracle execute exactly this JSON.
"""
from __future__ import annotations

import pyarrow as pa

from . import nexgen, tpchgen, ysbgen

TARGET_PARTITIONS = 8     # flock/src/configs/flock.toml:113
TARGET_BATCH_SIZE = 4096  # CoalesceBatchesExec default seen in every plan dump


# ---- data types / schema ---------------------------------------------------------------------------
def data_type_json(t: pa.DataType):
    if pa.types.is_int32(t): return "Int32"
    if pa.types.is_uint32(t): return "UInt32"
    if pa.types.is_int64(t): return "Int64"
    if pa.types.is_uint64(t): return "UInt64"
    if pa.types.is_float64(t): return "Float64"
    if pa.types.is_string(t): return "Utf8"
    if pa.types.is_date32(t): return "Date32"
    if pa.types.is_timestamp(t):
        unit = {"s": "Second", "ms": "Millisecond", "us": "Microsecond", "ns": "Nanosecond"}[t.unit]
        return {"Timestamp": [unit, t.tz]}
    raise TypeError(f"unsupported type {t}")


def schema_json(schema: pa.Schema) -> dict:
    md = {k.decode(): v.decode() for k, v in (schema.metadata or {}).items()}
    return {"fields": [{"name": f.name, "data_type": data_type_json(f.type), "nullable": f.nullable,
                        "dict_id": 0, "dict_is_ordered": False} for f in schema],
            "metadata": md}


# ---- physical expressions ----------------------------------------------------------------------------
def column(name: str, index: int) -> dict:
    return {"physical_expr": "column", "name": name, "index": index}


def literal(type_name: str, value) -> dict:
    return {"physical_expr": "literal", "value": {type_name: value}}


def binary(left: dict, op: str, right: dict) -> dict:
    return {"physical_expr": "binary_expr", "left": left, "op": op, "right": right}


def cast(expr: dict, type_json) -> dict:
    return {"physical_expr": "cast_expr", "expr": expr, "cast_type": type_json}


def try_cast(expr: dict, type_json) -> dict:
    return {"physical_expr": "try_cast_expr", "expr": expr, "cast_type": type_json}


# The reference's fixtures serialise no CASE, IN list, IS NULL or unary minus: the tags below follow the snake-cased
# struct names like the tags the fixtures do show (binary_expr, try_cast_expr), with DataFusion 6's field names.
def case_expr(when_then: list[tuple[dict, dict]], else_expr: dict | None = None, expr: dict | None = None) -> dict:
    """CaseExpr { expr, when_then_expr, else_expr }: CASE [expr] WHEN w THEN t ... [ELSE else_expr] END."""
    return {"physical_expr": "case_expr", "expr": expr, "when_then_expr": [[w, t] for w, t in when_then], "else_expr": else_expr}


def in_list(expr: dict, values: list[dict], negated: bool = False) -> dict:
    """InListExpr { expr, list, negated }."""
    return {"physical_expr": "in_list_expr", "expr": expr, "list": values, "negated": negated}


def is_null(arg: dict) -> dict:
    return {"physical_expr": "is_null_expr", "arg": arg}


def is_not_null(arg: dict) -> dict:
    return {"physical_expr": "is_not_null_expr", "arg": arg}


def negative(arg: dict) -> dict:
    return {"physical_expr": "negative_expr", "arg": arg}


def date_part(field: str, expr: dict) -> dict:
    """SQL's EXTRACT(field FROM expr) as DataFusion 6 plans it: ScalarFunctionExpr date_part(Utf8(field), expr) -> Int32.
    No fixture of the reference serialises a scalar function; the tag and fields follow the struct's as above."""
    return {"physical_expr": "scalar_function_expr", "fun": "DatePart", "name": "date_part", "args": [literal("Utf8", field), expr],
            "return_type": "Int32"}


# ---- execution plans -------------------------------------------------------------------------------------
def memory_exec(schema: pa.Schema, projection: list[int] | None) -> dict:
    return {"execution_plan": "memory_exec", "schema": schema_json(schema), "projection": projection}


def projection_exec(exprs: list[tuple[dict, str]], input: dict) -> dict:
    return {"execution_plan": "projection_exec", "expr": [[e, n] for e, n in exprs], "input": input}


def filter_exec(predicate: dict, input: dict) -> dict:
    return {"execution_plan": "filter_exec", "predicate": predicate, "input": input}


def coalesce_batches_exec(input: dict, target_batch_size: int = TARGET_BATCH_SIZE) -> dict:
    return {"execution_plan": "coalesce_batches_exec", "input": input, "target_batch_size": target_batch_size}


def coalesce_partitions_exec(input: dict) -> dict:
    return {"execution_plan": "coalesce_partitions_exec", "input": input}


def repartition_rr(input: dict, n: int = TARGET_PARTITIONS) -> dict:
    return {"execution_plan": "repartition_exec", "input": input, "partitioning": {"RoundRobinBatch": n}}


def repartition_hash(input: dict, exprs: list[dict], n: int = TARGET_PARTITIONS) -> dict:
    return {"execution_plan": "repartition_exec", "input": input, "partitioning": {"Hash": [exprs, n]}}


def aggregate_expr(func: str, name: str, expr: dict, data_type) -> dict:
    return {"aggregate_expr": func, "name": name, "expr": expr, "data_type": data_type, "nullable": True}


def hash_aggregate_exec(mode: str, group_expr: list[tuple[dict, str]], aggr_expr: list[dict], input: dict) -> dict:
    return {"execution_plan": "hash_aggregate_exec", "mode": mode, "group_expr": [[e, n] for e, n in group_expr],
            "aggr_expr": aggr_expr, "input": input}


def hash_join_exec(left: dict, right: dict, on: list[tuple[dict, dict]], mode: str = "Partitioned", join_type: str = "Inner") -> dict:
    """join_type "Inner": left ++ right columns; "Semi" / "Anti": the left rows with / without an equal key on the right,
    left columns only (DataFusion 6's JoinType variant names)."""
    return {"execution_plan": "hash_join_exec", "join_type": join_type, "mode": mode, "left": left, "right": right,
            "on": [[{"name": l["name"], "index": l["index"]}, {"name": r["name"], "index": r["index"]}] for l, r in on]}


def sort_exec(exprs: list[tuple[dict, bool, bool]], input: dict) -> dict:
    """flock/src/tests/data/plan/join.json: {"expr": [{"expr": column, "options": {"descending", "nulls_first"}}]}."""
    return {"execution_plan": "sort_exec", "input": input,
            "expr": [{"expr": e, "options": {"descending": desc, "nulls_first": nf}} for e, desc, nf in exprs]}


def global_limit_exec(input: dict, limit: int) -> dict:
    return {"execution_plan": "global_limit_exec", "input": input, "limit": limit}


def row_number_window(name: str, partition_by: list[dict], order_by: list[tuple[dict, bool, bool]], input: dict) -> dict:
    """WindowAggExec with one ROW_NUMBER() (the only window function NEXMark q6 uses).  No fixture of the reference
    serialises this node; the layout follows DataFusion 6's WindowAggExec { input, window_expr } and its
    BuiltInWindowExpr { fun, name, partition_by, order_by } fields."""
    return {"execution_plan": "window_agg_exec", "input": input,
            "window_expr": [{"window_expr": "built_in_window_expr", "fun": "RowNumber", "name": name, "partition_by": partition_by,
                             "order_by": [{"expr": e, "options": {"descending": desc, "nulls_first": nf}} for e, desc, nf in order_by]}]}


def two_phase_aggregate(group: list[tuple[str, int]], aggrs: list[dict], input: dict, n: int = TARGET_PARTITIONS) -> dict:
    """Partial -> RepartitionExec(Hash[group]) -> CoalesceBatches -> FinalPartitioned (stage.rs:597-601);
    without group columns: Partial -> CoalescePartitions -> Final (stage.rs:535-537)."""
    gexpr = [(column(nm, ix), nm) for nm, ix in group]
    partial = hash_aggregate_exec("Partial", gexpr, aggrs, input)
    if not group:
        return hash_aggregate_exec("Final", [], aggrs, coalesce_partitions_exec(partial))
    gfinal = [(column(nm, i), nm) for i, (nm, _) in enumerate(group)]
    shuffled = coalesce_batches_exec(repartition_hash(partial, [column(nm, i) for i, (nm, _) in enumerate(group)], n))
    return hash_aggregate_exec("FinalPartitioned", gfinal, aggrs, shuffled)


# ---- NEXMark q1..q8 (benchmarks/src/nexmark/query/qN.sql) -------------------------------------------------
BID, AUCTION, PERSON = nexgen.bid_schema(), nexgen.auction_schema(), nexgen.person_schema()
TS_MS = {"Timestamp": ["Millisecond", None]}


def q1(n: int = TARGET_PARTITIONS) -> dict:
    """planner.rs:90-92  SELECT auction, bidder, 0.908 * price AS price, b_date_time FROM bid"""
    scan = repartition_rr(memory_exec(BID, [0, 1, 2, 3]), n)
    return projection_exec([
        (column("auction", 0), "auction"), (column("bidder", 1), "bidder"),
        (binary(literal("Float64", 0.908), "Multiply", cast(column("price", 2), "Float64")), "price"),
        (column("b_date_time", 3), "b_date_time")], scan)


def q2(n: int = TARGET_PARTITIONS) -> dict:
    """planner.rs:120-124  SELECT auction, price FROM bid WHERE auction % 123 = 0"""
    scan = repartition_rr(memory_exec(BID, [0, 2]), n)
    pred = binary(binary(cast(column("auction", 0), "Int64"), "Modulo", literal("Int64", 123)), "Eq", literal("Int64", 0))
    return projection_exec([(column("auction", 0), "auction"), (column("price", 1), "price")],
                           coalesce_batches_exec(filter_exec(pred, scan)))


def q3_stage0(n: int = TARGET_PARTITIONS) -> list[dict]:
    """planner.rs:151-163: the two shuffle stages (auction side, person side)."""
    a_scan = repartition_rr(memory_exec(AUCTION, [0, 7, 8]), n)
    a_pred = binary(cast(column("category", 2), "Int64"), "Eq", literal("Int64", 10))
    a = coalesce_batches_exec(repartition_hash(coalesce_batches_exec(filter_exec(a_pred, a_scan)), [column("seller", 1)], n))
    p_scan = repartition_rr(memory_exec(PERSON, [0, 1, 4, 5]), n)
    st = column("state", 3)
    p_pred = binary(binary(binary(st, "Eq", literal("Utf8", "or")), "Or", binary(st, "Eq", literal("Utf8", "id"))),
                    "Or", binary(st, "Eq", literal("Utf8", "ca")))
    p = coalesce_batches_exec(repartition_hash(coalesce_batches_exec(filter_exec(p_pred, p_scan)), [column("p_id", 0)], n))
    return [a, p]


def q3(n: int = TARGET_PARTITIONS) -> dict:
    """planner.rs:151-171 as ONE plan (centralized mode runs the whole plan in one worker,
    benchmarks/src/nexmark/main.rs:209-214): auction JOIN person ON seller = p_id."""
    a, p = q3_stage0(n)
    join = hash_join_exec(a, p, [(column("seller", 1), column("p_id", 0))])
    return projection_exec([(column("name", 4), "name"), (column("city", 5), "city"), (column("state", 6), "state"),
                            (column("a_id", 0), "a_id")], coalesce_batches_exec(join))


def _count_by_auction(n: int) -> dict:
    scan = repartition_rr(memory_exec(BID, [0]), n)
    cnt = aggregate_expr("count", "COUNT(UInt8(1))", literal("UInt8", 1), "UInt64")
    return two_phase_aggregate([("auction", 0)], [cnt], scan, n)


def q5(n: int = TARGET_PARTITIONS) -> dict:
    """SURVEY.md Appendix B (types q5_plan.fmt): AuctionBids JOIN MaxBids ON num = maxn.  The COUNT-by-auction
    subtree appears twice, exactly as DataFusion 6 plans it (no common-subexpression elimination)."""
    left = projection_exec([(column("auction", 0), "auction"), (column("COUNT(UInt8(1))", 1), "num")], _count_by_auction(n))
    nums = projection_exec([(column("COUNT(UInt8(1))", 1), "num")], _count_by_auction(n))
    mx = aggregate_expr("max", "MAX(CountBids.num)", column("num", 0), "UInt64")
    right = projection_exec([(column("MAX(CountBids.num)", 0), "maxn")], two_phase_aggregate([], [mx], nums, n))
    lsh = coalesce_batches_exec(repartition_hash(left, [column("num", 1)], n))
    rsh = coalesce_batches_exec(repartition_hash(right, [column("maxn", 0)], n))
    join = hash_join_exec(lsh, rsh, [(column("num", 1), column("maxn", 0))])
    return projection_exec([(column("auction", 0), "auction"), (column("num", 1), "num")], coalesce_batches_exec(join))


def q8(n: int = TARGET_PARTITIONS) -> dict:
    """SURVEY.md Appendix B (q8_plan.fmt): P(p_id, name GROUP BY) JOIN A(seller GROUP BY) ON p_id = seller."""
    p_scan = repartition_rr(memory_exec(PERSON, [0, 1]), n)
    P = two_phase_aggregate([("p_id", 0), ("name", 1)], [], p_scan, n)
    a_scan = repartition_rr(memory_exec(AUCTION, [7]), n)
    A = two_phase_aggregate([("seller", 0)], [], a_scan, n)
    lsh = coalesce_batches_exec(repartition_hash(P, [column("p_id", 0)], n))
    rsh = coalesce_batches_exec(repartition_hash(A, [column("seller", 0)], n))
    join = hash_join_exec(lsh, rsh, [(column("p_id", 0), column("seller", 0))])
    return projection_exec([(column("p_id", 0), "p_id"), (column("name", 1), "name")], coalesce_batches_exec(join))


def q4(n: int = TARGET_PARTITIONS) -> dict:
    """benchmarks/src/nexmark/query/q4.sql, types q4_plan.fmt:
       SELECT category, AVG(final) FROM (SELECT MAX(price) AS final, category FROM auction JOIN bid ON a_id = auction
       WHERE b_date_time BETWEEN a_date_time AND expires GROUP BY a_id, category) GROUP BY category.
    Physical shape as DataFusion 6 builds it: Hash-repartitioned Partitioned join, Filter (BETWEEN = two comparisons),
    two two-phase aggregates."""
    a_scan = repartition_rr(memory_exec(AUCTION, [0, 5, 6, 8]), n)     # a_id, a_date_time, expires, category
    b_scan = repartition_rr(memory_exec(BID, [0, 2, 3]), n)            # auction, price, b_date_time
    lsh = coalesce_batches_exec(repartition_hash(a_scan, [column("a_id", 0)], n))
    rsh = coalesce_batches_exec(repartition_hash(b_scan, [column("auction", 0)], n))
    join = coalesce_batches_exec(hash_join_exec(lsh, rsh, [(column("a_id", 0), column("auction", 0))]))
    # a_id 0, a_date_time 1, expires 2, category 3, auction 4, price 5, b_date_time 6
    between = binary(binary(column("b_date_time", 6), "GtEq", column("a_date_time", 1)), "And",
                     binary(column("b_date_time", 6), "LtEq", column("expires", 2)))
    filt = coalesce_batches_exec(filter_exec(between, join))
    mx = aggregate_expr("max", "MAX(bid.price)", column("price", 5), "Int32")
    inner = two_phase_aggregate([("a_id", 0), ("category", 3)], [mx], filt, n)           # a_id, category, MAX(bid.price)
    q = projection_exec([(column("MAX(bid.price)", 2), "final"), (column("category", 1), "category")], inner)
    avg = aggregate_expr("avg", "AVG(Q.final)", column("final", 0), "Float64")
    outer = two_phase_aggregate([("category", 1)], [avg], q, n)
    return projection_exec([(column("category", 0), "category"), (column("AVG(Q.final)", 1), "AVG(Q.final)")], outer)


def q7(n: int = TARGET_PARTITIONS) -> dict:
    """benchmarks/src/nexmark/query/q7.sql, types q7_plan.fmt:
       SELECT auction, price, bidder, b_date_time FROM bid JOIN (SELECT MAX(price) AS maxprice FROM bid) ON price = maxprice."""
    bid = repartition_rr(memory_exec(BID, [0, 1, 2, 3]), n)
    mx = aggregate_expr("max", "MAX(bid.price)", column("price", 2), "Int32")
    b1 = projection_exec([(column("MAX(bid.price)", 0), "maxprice")],
                         two_phase_aggregate([], [mx], repartition_rr(memory_exec(BID, [0, 1, 2, 3]), n), n))
    lsh = coalesce_batches_exec(repartition_hash(bid, [column("price", 2)], n))
    rsh = coalesce_batches_exec(repartition_hash(b1, [column("maxprice", 0)], n))
    join = hash_join_exec(lsh, rsh, [(column("price", 2), column("maxprice", 0))])
    return projection_exec([(column("auction", 0), "auction"), (column("price", 2), "price"), (column("bidder", 1), "bidder"),
                            (column("b_date_time", 3), "b_date_time")], coalesce_batches_exec(join))


def q6(n: int = TARGET_PARTITIONS) -> dict:
    """benchmarks/src/nexmark/query/q6.sql, types q6_plan.fmt: average selling price of each seller's last ten closed
    auctions.  SortExec + WindowAggExec(ROW_NUMBER) on top of q4's join and BETWEEN filter (SURVEY section 8f rank 3)."""
    a_scan = repartition_rr(memory_exec(AUCTION, [0, 5, 6, 7]), n)     # a_id, a_date_time, expires, seller
    b_scan = repartition_rr(memory_exec(BID, [0, 2, 3]), n)            # auction, price, b_date_time
    lsh = coalesce_batches_exec(repartition_hash(a_scan, [column("a_id", 0)], n))
    rsh = coalesce_batches_exec(repartition_hash(b_scan, [column("auction", 0)], n))
    join = coalesce_batches_exec(hash_join_exec(lsh, rsh, [(column("a_id", 0), column("auction", 0))]))
    # a_id 0, a_date_time 1, expires 2, seller 3, auction 4, price 5, b_date_time 6
    between = binary(binary(column("b_date_time", 6), "GtEq", column("a_date_time", 1)), "And",
                     binary(column("b_date_time", 6), "LtEq", column("expires", 2)))
    filt = coalesce_partitions_exec(coalesce_batches_exec(filter_exec(between, join)))
    w1_name = "ROW_NUMBER() PARTITION BY [#auction.a_id] ORDER BY [#bid.price DESC NULLS FIRST]"
    w1 = row_number_window(w1_name, [column("a_id", 0)], [(column("price", 5), True, True)],
                           sort_exec([(column("a_id", 0), False, False), (column("price", 5), True, True)], filt))
    # window column first: rn 0, a_id 1, a_date_time 2, expires 3, seller 4, auction 5, price 6, b_date_time 7
    winners = coalesce_batches_exec(filter_exec(binary(column(w1_name, 0), "Eq", literal("UInt64", 1)), w1))
    q = projection_exec([(column("seller", 4), "seller"), (column("a_id", 1), "a_id"), (column("price", 6), "price"),
                         (column("b_date_time", 7), "b_date_time"), (column(w1_name, 0), "price_rank")], winners)
    q_sorted = sort_exec([(column("a_id", 1), False, False), (column("price", 2), True, True)], q)       # ORDER BY a_id, price DESC of subquery Q
    q2 = projection_exec([(column("seller", 0), "seller"), (column("price", 2), "price"), (column("b_date_time", 3), "b_date_time"),
                          (column("price_rank", 4), "price_rank")], q_sorted)
    w2_name = "ROW_NUMBER() PARTITION BY [#Q.seller] ORDER BY [#Q.b_date_time DESC NULLS FIRST]"
    w2 = row_number_window(w2_name, [column("seller", 0)], [(column("b_date_time", 2), True, True)],
                           sort_exec([(column("seller", 0), False, False), (column("b_date_time", 2), True, True)], q2))
    # rn 0, seller 1, price 2, b_date_time 3, price_rank 4
    last10 = coalesce_batches_exec(filter_exec(binary(column(w2_name, 0), "LtEq", literal("UInt64", 10)), w2))
    r = projection_exec([(column("seller", 1), "seller"), (column("price", 2), "price"), (column(w2_name, 0), "time_rank")], last10)
    avg = aggregate_expr("avg", "AVG(R.price)", column("price", 1), "Float64")
    outer = two_phase_aggregate([("seller", 0)], [avg], repartition_rr(r, n), n)
    return projection_exec([(column("seller", 0), "seller"), (column("AVG(R.price)", 1), "AVG(R.price)")], outer)


# ---- NEXMark q0 / q10, q9, q12, q13 ----------------------------------------------------------------------------------
BID_PTIME, SIDE_INPUT = nexgen.bid_ptime_schema(), nexgen.side_input_schema()
TS_NS_UTC = {"Timestamp": ["Nanosecond", "UTC"]}


def q10(n: int = TARGET_PARTITIONS) -> dict:
    """benchmarks/src/nexmark/query/q10.sql (q0.sql is the same query):  SELECT auction, bidder, price, b_date_time FROM bid"""
    scan = repartition_rr(memory_exec(BID, [0, 1, 2, 3]), n)
    return projection_exec([(column("auction", 0), "auction"), (column("bidder", 1), "bidder"), (column("price", 2), "price"),
                            (column("b_date_time", 3), "b_date_time")], scan)


q0 = q10


def q9(n: int = TARGET_PARTITIONS) -> dict:
    """benchmarks/src/nexmark/query/q9.sql, types q9_plan.fmt:
       SELECT auction, bidder, price, b_date_time FROM bid JOIN (SELECT a_id AS id, MAX(price) AS final FROM auction
       JOIN bid ON a_id = auction WHERE b_date_time BETWEEN a_date_time AND expires GROUP BY a_id) AS Q
       ON auction = id AND price = final.
    The inner part is q4's join and BETWEEN filter grouped by a_id alone; the outer join is Partitioned on the key pair,
    both sides Hash-repartitioned on it.  The BETWEEN filter applies to the subquery only: the outer join keeps every
    bid at its auction's top price, in the auction's lifetime or not."""
    a_scan = repartition_rr(memory_exec(AUCTION, [0, 5, 6]), n)        # a_id, a_date_time, expires
    b_scan = repartition_rr(memory_exec(BID, [0, 1, 2, 3]), n)         # auction, bidder, price, b_date_time
    lsh = coalesce_batches_exec(repartition_hash(a_scan, [column("a_id", 0)], n))
    rsh = coalesce_batches_exec(repartition_hash(b_scan, [column("auction", 0)], n))
    join = coalesce_batches_exec(hash_join_exec(lsh, rsh, [(column("a_id", 0), column("auction", 0))]))
    # a_id 0, a_date_time 1, expires 2, auction 3, bidder 4, price 5, b_date_time 6
    between = binary(binary(column("b_date_time", 6), "GtEq", column("a_date_time", 1)), "And",
                     binary(column("b_date_time", 6), "LtEq", column("expires", 2)))
    filt = coalesce_batches_exec(filter_exec(between, join))
    mx = aggregate_expr("max", "MAX(bid.price)", column("price", 5), "Int32")
    inner = two_phase_aggregate([("a_id", 0)], [mx], filt, n)                              # a_id, MAX(bid.price)
    q = projection_exec([(column("a_id", 0), "id"), (column("MAX(bid.price)", 1), "final")], inner)
    bid = repartition_rr(memory_exec(BID, [0, 1, 2, 3]), n)
    lsh2 = coalesce_batches_exec(repartition_hash(bid, [column("auction", 0), column("price", 2)], n))
    rsh2 = coalesce_batches_exec(repartition_hash(q, [column("id", 0), column("final", 1)], n))
    outer = hash_join_exec(lsh2, rsh2, [(column("auction", 0), column("id", 0)), (column("price", 2), column("final", 1))])
    return projection_exec([(column("auction", 0), "auction"), (column("bidder", 1), "bidder"), (column("price", 2), "price"),
                            (column("b_date_time", 3), "b_date_time")], coalesce_batches_exec(outer))


def q12(n: int = TARGET_PARTITIONS) -> dict:
    """benchmarks/src/nexmark/query/q12.sql, types q12_plan.fmt: SELECT bidder, COUNT(*) AS bid_count, MIN(p_time) AS
    start_time, MAX(p_time) AS end_time FROM bid GROUP BY bidder, over bids that carry a processing time p_time."""
    scan = repartition_rr(memory_exec(BID_PTIME, [1, 4]), n)          # bidder, p_time
    cnt = aggregate_expr("count", "COUNT(UInt8(1))", literal("UInt8", 1), "UInt64")
    mn = aggregate_expr("min", "MIN(bid.p_time)", column("p_time", 1), TS_NS_UTC)
    mx = aggregate_expr("max", "MAX(bid.p_time)", column("p_time", 1), TS_NS_UTC)
    agg = two_phase_aggregate([("bidder", 0)], [cnt, mn, mx], scan, n)
    return projection_exec([(column("bidder", 0), "bidder"), (column("COUNT(UInt8(1))", 1), "bid_count"),
                            (column("MIN(bid.p_time)", 2), "start_time"), (column("MAX(bid.p_time)", 3), "end_time")], agg)


def q13(n: int = TARGET_PARTITIONS) -> dict:
    """benchmarks/src/nexmark/query/q13.sql, types q13_plan.fmt:
       SELECT auction, bidder, price, b_date_time, value FROM bid JOIN side_input ON auction = key"""
    bid = repartition_rr(memory_exec(BID, [0, 1, 2, 3]), n)
    side = repartition_rr(memory_exec(SIDE_INPUT, [0, 1]), n)
    lsh = coalesce_batches_exec(repartition_hash(bid, [column("auction", 0)], n))
    rsh = coalesce_batches_exec(repartition_hash(side, [column("key", 0)], n))
    join = hash_join_exec(lsh, rsh, [(column("auction", 0), column("key", 0))])
    # auction 0, bidder 1, price 2, b_date_time 3, key 4, value 5
    return projection_exec([(column("auction", 0), "auction"), (column("bidder", 1), "bidder"), (column("price", 2), "price"),
                            (column("b_date_time", 3), "b_date_time"), (column("value", 5), "value")], coalesce_batches_exec(join))


QUERIES = {"q1": q1, "q2": q2, "q3": q3, "q4": q4, "q5": q5, "q6": q6, "q7": q7, "q8": q8}
GPU_QUERIES = list(QUERIES)
# relations each query feeds, in feed order (flock/src/datasource/nexmark/nexmark.rs:181-203); q5 scans bid
# twice, and feed_data_sources hands one source to one leaf (context.rs:293-303), so bid is fed twice.
SOURCES = {"q1": ["bid"], "q2": ["bid"], "q3": ["auction", "person"], "q4": ["auction", "bid"], "q5": ["bid", "bid"],
           "q6": ["auction", "bid"], "q7": ["bid", "bid"], "q8": ["person", "auction"]}
# q9 / q10 / q12 / q13: kept apart from QUERIES, whose every entry the existing suites and bench.py iterate.
# "bid_ptime" is nexgen.bids_ptime, "side_input" nexgen.side_input.
MORE_QUERIES = {"q9": q9, "q10": q10, "q12": q12, "q13": q13}
MORE_SOURCES = {"q9": ["auction", "bid", "bid"], "q10": ["bid"], "q12": ["bid_ptime"], "q13": ["bid", "side_input"]}


# ---- YSB, the Yahoo Streaming Benchmark (benchmarks/src/ysb/ysb.sql) --------------------------------------------------
AD_EVENT, CAMPAIGN = ysbgen.ad_event_schema(), ysbgen.campaign_schema()
YSB_COUNT = "COUNT(UInt8(1))"


def _ysb_count() -> dict:
    return aggregate_expr("count", YSB_COUNT, literal("UInt8", 1), "UInt64")


def ysb_stage0(n: int = TARGET_PARTITIONS) -> list[dict]:
    """planner.rs:315-327: the two shuffling plans, the viewed events by ad_id and the campaigns by c_ad_id."""
    scan = repartition_rr(memory_exec(AD_EVENT, [2, 4]), n)                               # ad_id, event_type
    views = coalesce_batches_exec(filter_exec(binary(column("event_type", 1), "Eq", literal("Utf8", "view")), scan))
    events = coalesce_batches_exec(repartition_hash(views, [column("ad_id", 0)], n))
    camps = coalesce_batches_exec(repartition_hash(repartition_rr(memory_exec(CAMPAIGN, [0, 1]), n), [column("c_ad_id", 0)], n))
    return [events, camps]


def _ysb_partial(events: dict, camps: dict) -> dict:
    # ad_id 0, event_type 1, c_ad_id 2, campaign_id 3
    join = coalesce_batches_exec(hash_join_exec(events, camps, [(column("ad_id", 0), column("c_ad_id", 0))]))
    return hash_aggregate_exec("Partial", [(column("campaign_id", 3), "campaign_id")], [_ysb_count()], join)


def _ysb_final(input: dict) -> dict:
    final = hash_aggregate_exec("FinalPartitioned", [(column("campaign_id", 0), "campaign_id")], [_ysb_count()], input)
    return projection_exec([(column("campaign_id", 0), "campaign_id"), (column(YSB_COUNT, 1), YSB_COUNT)], final)


def ysb_stages(n: int = TARGET_PARTITIONS) -> list[list[dict]]:
    """planner.rs:315-345: the query stages a distributed run hands to its functions, in order.  Stage 1 reads the
    outputs of stage 0 (viewed events, campaigns), stage 2 the output of stage 1 (campaign_id and the COUNT state)."""
    views = pa.schema([AD_EVENT.field("ad_id"), AD_EVENT.field("event_type")], metadata=AD_EVENT.metadata)
    partial = _ysb_partial(memory_exec(views, None), memory_exec(CAMPAIGN, None))
    stage1 = coalesce_batches_exec(repartition_hash(partial, [column("campaign_id", 0)], n))
    states = pa.schema([pa.field("campaign_id", pa.utf8(), False), pa.field(YSB_COUNT + "[count]", pa.uint64(), True)], metadata=AD_EVENT.metadata)
    return [ysb_stage0(n), [stage1], [_ysb_final(memory_exec(states, None))]]


def ysb(n: int = TARGET_PARTITIONS) -> dict:
    """SELECT campaign_id, COUNT(*) FROM ad_event INNER JOIN campaign ON ad_id = c_ad_id WHERE event_type = 'view'
       GROUP BY campaign_id
    as ONE plan, the three stages of planner.rs:315-345 stacked (centralized mode runs the whole plan in one worker)."""
    events, camps = ysb_stage0(n)
    shuffled = coalesce_batches_exec(repartition_hash(_ysb_partial(events, camps), [column("campaign_id", 0)], n))
    return _ysb_final(shuffled)


YSB_QUERIES = {"ysb": ysb}
YSB_SOURCES = {"ysb": ["ad_event", "campaign"]}


# ---- TPC-H (flock/src/datasource/tpch/queries/qN.sql) over Flock's schemas (flock/src/datasource/tpch/mod.rs) -----------
# The reference ships no TPC-H plan dump, so the shape is DataFusion 6's usual one and unverified: MemoryExec
# projections -> FilterExec -> Hash repartitions -> Partitioned inner joins in FROM order (keys from the WHERE
# equalities) -> Partial / FinalPartitioned aggregate -> ProjectionExec -> SortExec.  DATE 'YYYY-MM-DD' is written as
# CAST('YYYY-MM-DD' AS Date32), the form before constant folding; the plan reader folds it to a Date32 literal.
class _Rel:
    """A plan node and the names of its output columns, so that expressions can refer to columns by name."""

    def __init__(self, plan: dict, names: list[str]):
        self.plan, self.names = plan, names

    def c(self, name: str) -> dict:
        return column(name, self.names.index(name))


def _tpch_scan(table: str, cols: list[str], n: int) -> _Rel:
    sch = tpchgen.schema(table)
    return _Rel(repartition_rr(memory_exec(sch, [sch.get_field_index(c) for c in cols]), n), cols)


def _date(iso: str) -> dict:
    return cast(literal("Utf8", iso), "Date32")


def _f64(x) -> dict:
    return cast(literal("Int64", x), "Float64")


def _filter(r: _Rel, pred) -> _Rel:
    return _Rel(coalesce_batches_exec(filter_exec(pred(r), r.plan)), r.names)


def _and(*terms: dict) -> dict:
    out = terms[0]
    for t in terms[1:]:
        out = binary(out, "And", t)
    return out


def _join(left: _Rel, right: _Rel, on: list[tuple[str, str]], n: int) -> _Rel:
    lsh = coalesce_batches_exec(repartition_hash(left.plan, [left.c(a) for a, _ in on], n))
    rsh = coalesce_batches_exec(repartition_hash(right.plan, [right.c(b) for _, b in on], n))
    return _Rel(coalesce_batches_exec(hash_join_exec(lsh, rsh, [(left.c(a), right.c(b)) for a, b in on])), left.names + right.names)


def _revenue(r: _Rel) -> dict:
    return binary(r.c("l_extendedprice"), "Multiply", binary(_f64(1), "Minus", r.c("l_discount")))


def _grouped(r: _Rel, group: list[str], aggrs: list[dict], n: int) -> _Rel:
    out = two_phase_aggregate([(g, r.names.index(g)) for g in group], aggrs, r.plan, n)
    return _Rel(out, group + [a["name"] for a in aggrs])


def _project_sort(r: _Rel, exprs: list[tuple[dict, str]], order: list[tuple[str, bool]]) -> dict:
    proj = _Rel(projection_exec(exprs, r.plan), [nm for _, nm in exprs])
    return sort_exec([(proj.c(nm), desc, False) for nm, desc in order], proj.plan)


def _sum(name: str, e: dict, dt="Float64") -> dict:
    return aggregate_expr("sum", name, e, dt)


def tpch_q1(n: int = TARGET_PARTITIONS) -> dict:
    li = _tpch_scan("lineitem", ["l_quantity", "l_extendedprice", "l_discount", "l_tax", "l_returnflag", "l_linestatus", "l_shipdate"], n)
    li = _filter(li, lambda r: binary(r.c("l_shipdate"), "LtEq", _date("1998-09-02")))
    disc_price = _revenue(li)
    charge = binary(disc_price, "Multiply", binary(_f64(1), "Plus", li.c("l_tax")))
    aggrs = [_sum("SUM(lineitem.l_quantity)", li.c("l_quantity")), _sum("SUM(lineitem.l_extendedprice)", li.c("l_extendedprice")),
             _sum("SUM(lineitem.l_extendedprice * Int64(1) - lineitem.l_discount)", disc_price),
             _sum("SUM(lineitem.l_extendedprice * Int64(1) - lineitem.l_discount * Int64(1) + lineitem.l_tax)", charge),
             aggregate_expr("avg", "AVG(lineitem.l_quantity)", li.c("l_quantity"), "Float64"),
             aggregate_expr("avg", "AVG(lineitem.l_extendedprice)", li.c("l_extendedprice"), "Float64"),
             aggregate_expr("avg", "AVG(lineitem.l_discount)", li.c("l_discount"), "Float64"),
             aggregate_expr("count", "COUNT(UInt8(1))", literal("UInt8", 1), "UInt64")]
    g = _grouped(li, ["l_returnflag", "l_linestatus"], aggrs, n)
    outs = ["sum_qty", "sum_base_price", "sum_disc_price", "sum_charge", "avg_qty", "avg_price", "avg_disc", "count_order"]
    return _project_sort(g, [(g.c("l_returnflag"), "l_returnflag"), (g.c("l_linestatus"), "l_linestatus")] +
                         [(g.c(a["name"]), o) for a, o in zip(aggrs, outs)], [("l_returnflag", False), ("l_linestatus", False)])


def tpch_q3(n: int = TARGET_PARTITIONS) -> dict:
    cu = _filter(_tpch_scan("customer", ["c_custkey", "c_mktsegment"], n), lambda r: binary(r.c("c_mktsegment"), "Eq", literal("Utf8", "BUILDING")))
    od = _filter(_tpch_scan("orders", ["o_orderkey", "o_custkey", "o_orderdate", "o_shippriority"], n),
                 lambda r: binary(r.c("o_orderdate"), "Lt", _date("1995-03-15")))
    li = _filter(_tpch_scan("lineitem", ["l_orderkey", "l_extendedprice", "l_discount", "l_shipdate"], n),
                 lambda r: binary(r.c("l_shipdate"), "Gt", _date("1995-03-15")))
    j = _join(_join(cu, od, [("c_custkey", "o_custkey")], n), li, [("o_orderkey", "l_orderkey")], n)
    rev = _sum("SUM(lineitem.l_extendedprice * Int64(1) - lineitem.l_discount)", _revenue(j))
    g = _grouped(j, ["l_orderkey", "o_orderdate", "o_shippriority"], [rev], n)
    return _project_sort(g, [(g.c("l_orderkey"), "l_orderkey"), (g.c(rev["name"]), "revenue"), (g.c("o_orderdate"), "o_orderdate"),
                             (g.c("o_shippriority"), "o_shippriority")], [("revenue", True), ("o_orderdate", False)])


def tpch_q5(n: int = TARGET_PARTITIONS) -> dict:
    cu = _tpch_scan("customer", ["c_custkey", "c_nationkey"], n)
    od = _filter(_tpch_scan("orders", ["o_orderkey", "o_custkey", "o_orderdate"], n),
                 lambda r: _and(binary(r.c("o_orderdate"), "GtEq", _date("1994-01-01")), binary(r.c("o_orderdate"), "Lt", _date("1995-01-01"))))
    li = _tpch_scan("lineitem", ["l_orderkey", "l_suppkey", "l_extendedprice", "l_discount"], n)
    su = _tpch_scan("supplier", ["s_suppkey", "s_nationkey"], n)
    na = _tpch_scan("nation", ["n_nationkey", "n_name", "n_regionkey"], n)
    re = _filter(_tpch_scan("region", ["r_regionkey", "r_name"], n), lambda r: binary(r.c("r_name"), "Eq", literal("Utf8", "ASIA")))
    j = _join(cu, od, [("c_custkey", "o_custkey")], n)
    j = _join(j, li, [("o_orderkey", "l_orderkey")], n)
    j = _join(j, su, [("l_suppkey", "s_suppkey"), ("c_nationkey", "s_nationkey")], n)
    j = _join(j, na, [("s_nationkey", "n_nationkey")], n)
    j = _join(j, re, [("n_regionkey", "r_regionkey")], n)
    rev = _sum("SUM(lineitem.l_extendedprice * Int64(1) - lineitem.l_discount)", _revenue(j))
    g = _grouped(j, ["n_name"], [rev], n)
    return _project_sort(g, [(g.c("n_name"), "n_name"), (g.c(rev["name"]), "revenue")], [("revenue", True)])


def tpch_q6(n: int = TARGET_PARTITIONS) -> dict:
    li = _tpch_scan("lineitem", ["l_quantity", "l_extendedprice", "l_discount", "l_shipdate"], n)
    # BETWEEN .06 - 0.01 AND .06 + 0.01 stays Float64 literal arithmetic: 0.06 + 0.01 = 0.06999999999999999 < 0.07
    lo = binary(literal("Float64", 0.06), "Minus", literal("Float64", 0.01))
    hi = binary(literal("Float64", 0.06), "Plus", literal("Float64", 0.01))
    li = _filter(li, lambda r: _and(binary(r.c("l_shipdate"), "GtEq", _date("1994-01-01")), binary(r.c("l_shipdate"), "Lt", _date("1995-01-01")),
                                    binary(r.c("l_discount"), "GtEq", lo), binary(r.c("l_discount"), "LtEq", hi),
                                    binary(r.c("l_quantity"), "Lt", _f64(24))))
    rev = _sum("SUM(lineitem.l_extendedprice * lineitem.l_discount)", binary(li.c("l_extendedprice"), "Multiply", li.c("l_discount")))
    g = _grouped(li, [], [rev], n)
    return projection_exec([(g.c(rev["name"]), "revenue")], g.plan)


def tpch_q10(n: int = TARGET_PARTITIONS) -> dict:
    cu = _tpch_scan("customer", ["c_custkey", "c_name", "c_address", "c_nationkey", "c_phone", "c_acctbal", "c_comment"], n)
    od = _filter(_tpch_scan("orders", ["o_orderkey", "o_custkey", "o_orderdate"], n),
                 lambda r: _and(binary(r.c("o_orderdate"), "GtEq", _date("1993-10-01")), binary(r.c("o_orderdate"), "Lt", _date("1994-01-01"))))
    li = _filter(_tpch_scan("lineitem", ["l_orderkey", "l_extendedprice", "l_discount", "l_returnflag"], n),
                 lambda r: binary(r.c("l_returnflag"), "Eq", literal("Utf8", "R")))
    na = _tpch_scan("nation", ["n_nationkey", "n_name"], n)
    j = _join(cu, od, [("c_custkey", "o_custkey")], n)
    j = _join(j, li, [("o_orderkey", "l_orderkey")], n)
    j = _join(j, na, [("c_nationkey", "n_nationkey")], n)
    rev = _sum("SUM(lineitem.l_extendedprice * Int64(1) - lineitem.l_discount)", _revenue(j))
    group = ["c_custkey", "c_name", "c_acctbal", "c_phone", "n_name", "c_address", "c_comment"]
    g = _grouped(j, group, [rev], n)
    return _project_sort(g, [(g.c("c_custkey"), "c_custkey"), (g.c("c_name"), "c_name"), (g.c(rev["name"]), "revenue"),
                             (g.c("c_acctbal"), "c_acctbal"), (g.c("n_name"), "n_name"), (g.c("c_address"), "c_address"),
                             (g.c("c_phone"), "c_phone"), (g.c("c_comment"), "c_comment")], [("revenue", True)])


def tpch_q12(n: int = TARGET_PARTITIONS) -> dict:
    li = _filter(_tpch_scan("lineitem", ["l_orderkey", "l_shipdate", "l_commitdate", "l_receiptdate", "l_shipmode"], n),
                 lambda r: _and(in_list(r.c("l_shipmode"), [literal("Utf8", "MAIL"), literal("Utf8", "SHIP")]),
                                binary(r.c("l_commitdate"), "Lt", r.c("l_receiptdate")), binary(r.c("l_shipdate"), "Lt", r.c("l_commitdate")),
                                binary(r.c("l_receiptdate"), "GtEq", _date("1994-01-01")), binary(r.c("l_receiptdate"), "Lt", _date("1995-01-01"))))
    od = _tpch_scan("orders", ["o_orderkey", "o_orderpriority"], n)
    j = _join(li, od, [("l_orderkey", "o_orderkey")], n)
    pr = j.c("o_orderpriority")
    urgent, high = literal("Utf8", "1-URGENT"), literal("Utf8", "2-HIGH")
    hi = case_expr([(binary(binary(pr, "Eq", urgent), "Or", binary(pr, "Eq", high)), literal("Int64", 1))], literal("Int64", 0))
    lo = case_expr([(binary(binary(pr, "NotEq", urgent), "And", binary(pr, "NotEq", high)), literal("Int64", 1))], literal("Int64", 0))
    aggrs = [_sum("SUM(CASE WHEN orders.o_orderpriority = Utf8(\"1-URGENT\") OR orders.o_orderpriority = Utf8(\"2-HIGH\") THEN Int64(1) ELSE Int64(0) END)", hi, "Int64"),
             _sum("SUM(CASE WHEN orders.o_orderpriority != Utf8(\"1-URGENT\") AND orders.o_orderpriority != Utf8(\"2-HIGH\") THEN Int64(1) ELSE Int64(0) END)", lo, "Int64")]
    g = _grouped(j, ["l_shipmode"], aggrs, n)
    return _project_sort(g, [(g.c("l_shipmode"), "l_shipmode"), (g.c(aggrs[0]["name"]), "high_line_count"), (g.c(aggrs[1]["name"]), "low_line_count")],
                         [("l_shipmode", False)])


def tpch_q14(n: int = TARGET_PARTITIONS) -> dict:
    li = _filter(_tpch_scan("lineitem", ["l_partkey", "l_extendedprice", "l_discount", "l_shipdate"], n),
                 lambda r: _and(binary(r.c("l_shipdate"), "GtEq", _date("1995-09-01")), binary(r.c("l_shipdate"), "Lt", _date("1995-10-01"))))
    pt = _tpch_scan("part", ["p_partkey", "p_type"], n)
    j = _join(li, pt, [("l_partkey", "p_partkey")], n)
    promo = case_expr([(binary(j.c("p_type"), "Like", literal("Utf8", "PROMO%")), _revenue(j))], _f64(0))
    aggrs = [_sum("SUM(CASE WHEN part.p_type LIKE Utf8(\"PROMO%\") THEN lineitem.l_extendedprice * Int64(1) - lineitem.l_discount ELSE Int64(0) END)", promo),
             _sum("SUM(lineitem.l_extendedprice * Int64(1) - lineitem.l_discount)", _revenue(j))]
    g = _grouped(j, [], aggrs, n)
    share = binary(binary(literal("Float64", 100.0), "Multiply", g.c(aggrs[0]["name"])), "Divide", g.c(aggrs[1]["name"]))
    return projection_exec([(share, "promo_revenue")], g.plan)


TPCH_QUERIES = {"q1": tpch_q1, "q3": tpch_q3, "q5": tpch_q5, "q6": tpch_q6, "q10": tpch_q10, "q12": tpch_q12, "q14": tpch_q14}
# the table each MemoryExec leaf scans, in leaf (feed) order
TPCH_SOURCES = {"q1": ["lineitem"], "q3": ["customer", "orders", "lineitem"],
                "q5": ["customer", "orders", "lineitem", "supplier", "nation", "region"], "q6": ["lineitem"],
                "q10": ["customer", "orders", "lineitem", "nation"], "q12": ["lineitem", "orders"], "q14": ["lineitem", "part"]}


# ---- TPC-H q7, q8 and q9: EXTRACT(YEAR ...) and joins of up to 20 columns -------------------------------------------------
# Shape unverified, like the queries above.  q8 and q9 list part and supplier first with no key between them, which
# DataFusion 6's FROM-order planner would join as a cross join; the plans here join in FROM order except that part
# follows lineitem, the first relation it has a key with.  BETWEEN is written as >= AND <=.
def _between(e: dict, lo: str, hi: str) -> dict:
    return _and(binary(e, "GtEq", _date(lo)), binary(e, "LtEq", _date(hi)))


def _subquery(r: _Rel, exprs: list[tuple[dict, str]]) -> _Rel:
    return _Rel(projection_exec(exprs, r.plan), [nm for _, nm in exprs])


def tpch_q7(n: int = TARGET_PARTITIONS) -> dict:
    su = _tpch_scan("supplier", ["s_suppkey", "s_nationkey"], n)
    li = _filter(_tpch_scan("lineitem", ["l_orderkey", "l_suppkey", "l_extendedprice", "l_discount", "l_shipdate"], n),
                 lambda r: _between(r.c("l_shipdate"), "1995-01-01", "1996-12-31"))
    od = _tpch_scan("orders", ["o_orderkey", "o_custkey"], n)
    cu = _tpch_scan("customer", ["c_custkey", "c_nationkey"], n)
    n1 = _tpch_scan("nation", ["n_nationkey", "n_name"], n)
    n2 = _tpch_scan("nation", ["n_nationkey", "n_name"], n)
    j = _join(su, li, [("s_suppkey", "l_suppkey")], n)
    j = _join(j, od, [("l_orderkey", "o_orderkey")], n)
    j = _join(j, cu, [("o_custkey", "c_custkey")], n)
    j = _join(j, n1, [("s_nationkey", "n_nationkey")], n)
    j = _join(j, n2, [("c_nationkey", "n_nationkey")], n)
    # two columns are named n_name: n1's comes first, n2's is the last
    sn, cn = column("n_name", j.names.index("n_name")), column("n_name", len(j.names) - 1)
    fr, de = literal("Utf8", "FRANCE"), literal("Utf8", "GERMANY")
    j = _Rel(coalesce_batches_exec(filter_exec(binary(_and(binary(sn, "Eq", fr), binary(cn, "Eq", de)), "Or",
                                                      _and(binary(sn, "Eq", de), binary(cn, "Eq", fr))), j.plan)), j.names)
    shipping = _subquery(j, [(sn, "supp_nation"), (cn, "cust_nation"), (date_part("YEAR", j.c("l_shipdate")), "l_year"),
                             (_revenue(j), "volume")])
    rev = _sum("SUM(shipping.volume)", shipping.c("volume"))
    g = _grouped(shipping, ["supp_nation", "cust_nation", "l_year"], [rev], n)
    return _project_sort(g, [(g.c("supp_nation"), "supp_nation"), (g.c("cust_nation"), "cust_nation"), (g.c("l_year"), "l_year"),
                             (g.c(rev["name"]), "revenue")], [("supp_nation", False), ("cust_nation", False), ("l_year", False)])


def tpch_q8(n: int = TARGET_PARTITIONS) -> dict:
    su = _tpch_scan("supplier", ["s_suppkey", "s_nationkey"], n)
    li = _tpch_scan("lineitem", ["l_orderkey", "l_partkey", "l_suppkey", "l_extendedprice", "l_discount"], n)
    pt = _filter(_tpch_scan("part", ["p_partkey", "p_type"], n), lambda r: binary(r.c("p_type"), "Eq", literal("Utf8", "ECONOMY ANODIZED STEEL")))
    od = _filter(_tpch_scan("orders", ["o_orderkey", "o_custkey", "o_orderdate"], n),
                 lambda r: _between(r.c("o_orderdate"), "1995-01-01", "1996-12-31"))
    cu = _tpch_scan("customer", ["c_custkey", "c_nationkey"], n)
    n1 = _tpch_scan("nation", ["n_nationkey", "n_regionkey"], n)
    n2 = _tpch_scan("nation", ["n_nationkey", "n_name"], n)
    re = _filter(_tpch_scan("region", ["r_regionkey", "r_name"], n), lambda r: binary(r.c("r_name"), "Eq", literal("Utf8", "AMERICA")))
    j = _join(su, li, [("s_suppkey", "l_suppkey")], n)
    j = _join(j, pt, [("l_partkey", "p_partkey")], n)
    j = _join(j, od, [("l_orderkey", "o_orderkey")], n)
    j = _join(j, cu, [("o_custkey", "c_custkey")], n)
    j = _join(j, n1, [("c_nationkey", "n_nationkey")], n)
    j = _join(j, n2, [("s_nationkey", "n_nationkey")], n)
    j = _join(j, re, [("n_regionkey", "r_regionkey")], n)
    nations = _subquery(j, [(date_part("YEAR", j.c("o_orderdate")), "o_year"), (_revenue(j), "volume"), (j.c("n_name"), "nation")])
    brazil = case_expr([(binary(nations.c("nation"), "Eq", literal("Utf8", "BRAZIL")), nations.c("volume"))], _f64(0))
    aggrs = [_sum("SUM(CASE WHEN all_nations.nation = Utf8(\"BRAZIL\") THEN all_nations.volume ELSE Int64(0) END)", brazil),
             _sum("SUM(all_nations.volume)", nations.c("volume"))]
    g = _grouped(nations, ["o_year"], aggrs, n)
    share = binary(g.c(aggrs[0]["name"]), "Divide", g.c(aggrs[1]["name"]))
    return _project_sort(g, [(g.c("o_year"), "o_year"), (share, "mkt_share")], [("o_year", False)])


def tpch_q9(n: int = TARGET_PARTITIONS) -> dict:
    su = _tpch_scan("supplier", ["s_suppkey", "s_nationkey"], n)
    li = _tpch_scan("lineitem", ["l_orderkey", "l_partkey", "l_suppkey", "l_quantity", "l_extendedprice", "l_discount"], n)
    pt = _filter(_tpch_scan("part", ["p_partkey", "p_name"], n), lambda r: binary(r.c("p_name"), "Like", literal("Utf8", "%green%")))
    ps = _tpch_scan("partsupp", ["ps_partkey", "ps_suppkey", "ps_supplycost"], n)
    od = _tpch_scan("orders", ["o_orderkey", "o_orderdate"], n)
    na = _tpch_scan("nation", ["n_nationkey", "n_name"], n)
    j = _join(su, li, [("s_suppkey", "l_suppkey")], n)
    j = _join(j, pt, [("l_partkey", "p_partkey")], n)
    j = _join(j, ps, [("l_suppkey", "ps_suppkey"), ("l_partkey", "ps_partkey")], n)
    j = _join(j, od, [("l_orderkey", "o_orderkey")], n)
    j = _join(j, na, [("s_nationkey", "n_nationkey")], n)
    amount = binary(_revenue(j), "Minus", binary(j.c("ps_supplycost"), "Multiply", j.c("l_quantity")))
    profit = _subquery(j, [(j.c("n_name"), "nation"), (date_part("YEAR", j.c("o_orderdate")), "o_year"), (amount, "amount")])
    total = _sum("SUM(profit.amount)", profit.c("amount"))
    g = _grouped(profit, ["nation", "o_year"], [total], n)
    return _project_sort(g, [(g.c("nation"), "nation"), (g.c("o_year"), "o_year"), (g.c(total["name"]), "sum_profit")],
                         [("nation", False), ("o_year", True)])


# q7 / q8 / q9: kept apart from TPCH_QUERIES, whose every entry the existing suites iterate and run through sqlite3,
# which has no EXTRACT.  nation is scanned twice by q7 and q8, and each scan is fed its own copy.
TPCH_MORE_QUERIES = {"q7": tpch_q7, "q8": tpch_q8, "q9": tpch_q9}
TPCH_MORE_SOURCES = {"q7": ["supplier", "lineitem", "orders", "customer", "nation", "nation"],
                     "q8": ["supplier", "lineitem", "part", "orders", "customer", "nation", "nation", "region"],
                     "q9": ["supplier", "lineitem", "part", "partsupp", "orders", "nation"]}


# ---- TPC-H q4, q16, q18 and q21: EXISTS, IN and NOT IN subqueries as Semi / Anti hash joins ----------------------------------
# Shape unverified, like the queries above.  A subquery becomes the right input of a Partitioned Semi (EXISTS, IN) or Anti
# (NOT EXISTS, NOT IN) join on its correlation key; the join keeps the left input's columns.  q21's correlated
# conditions have no key equality (l2.l_suppkey <> l1.l_suppkey), and DataFusion 6's HashJoinExec has no join filter,
# so they are decorrelated into per-order counts: another supplier on the order exists iff the order has at least two
# distinct suppliers, and no other late supplier exists iff the order's one late supplier is l1's own (l1 is late).
# COUNT(DISTINCT x) is DataFusion's single-distinct rewrite: group by (keys, x), then COUNT(*) grouped by the keys.
def _semi(left: _Rel, right: _Rel, on: list[tuple[str, str]], n: int, join_type: str = "Semi", as_inner: bool = False) -> _Rel:
    """left Semi / Anti right.  `as_inner` plans a Semi join the way it is written without one, for comparison:
    DISTINCT over the right keys, then an inner join (left ++ the right keys)."""
    if as_inner:
        assert join_type == "Semi"
        keys = _grouped(right, [b for _, b in on], [], n)
        return _join(left, keys, on, n)
    lsh = coalesce_batches_exec(repartition_hash(left.plan, [left.c(a) for a, _ in on], n))
    rsh = coalesce_batches_exec(repartition_hash(right.plan, [right.c(b) for _, b in on], n))
    return _Rel(coalesce_batches_exec(hash_join_exec(lsh, rsh, [(left.c(a), right.c(b)) for a, b in on], join_type=join_type)), left.names)


def _count(name: str) -> dict:
    return aggregate_expr("count", name, literal("UInt8", 1), "UInt64")


def tpch_q4(n: int = TARGET_PARTITIONS, as_inner: bool = False) -> dict:
    # DATE '1993-07-01' + interval '3' month, folded
    od = _filter(_tpch_scan("orders", ["o_orderkey", "o_orderdate", "o_orderpriority"], n),
                 lambda r: _and(binary(r.c("o_orderdate"), "GtEq", _date("1993-07-01")), binary(r.c("o_orderdate"), "Lt", _date("1993-10-01"))))
    li = _filter(_tpch_scan("lineitem", ["l_orderkey", "l_commitdate", "l_receiptdate"], n),
                 lambda r: binary(r.c("l_commitdate"), "Lt", r.c("l_receiptdate")))
    j = _semi(od, li, [("o_orderkey", "l_orderkey")], n, as_inner=as_inner)
    cnt = _count("COUNT(UInt8(1))")
    g = _grouped(j, ["o_orderpriority"], [cnt], n)
    return _project_sort(g, [(g.c("o_orderpriority"), "o_orderpriority"), (g.c(cnt["name"]), "order_count")], [("o_orderpriority", False)])


def tpch_q16(n: int = TARGET_PARTITIONS, anti: bool = True) -> dict:
    """`anti=False` leaves out the NOT IN (supplier complaints) join."""
    ps = _tpch_scan("partsupp", ["ps_partkey", "ps_suppkey"], n)
    sizes = [literal("Int32", s) for s in (49, 14, 23, 45, 19, 3, 36, 9)]
    pt = _filter(_tpch_scan("part", ["p_partkey", "p_brand", "p_type", "p_size"], n),
                 lambda r: _and(binary(r.c("p_brand"), "NotEq", literal("Utf8", "Brand#45")),
                                binary(r.c("p_type"), "NotLike", literal("Utf8", "MEDIUM POLISHED%")), in_list(r.c("p_size"), sizes)))
    j = _join(ps, pt, [("ps_partkey", "p_partkey")], n)
    if anti:
        su = _filter(_tpch_scan("supplier", ["s_suppkey", "s_comment"], n),
                     lambda r: binary(r.c("s_comment"), "Like", literal("Utf8", "%Customer%Complaints%")))
        j = _semi(j, su, [("ps_suppkey", "s_suppkey")], n, "Anti")
    pairs = _grouped(j, ["p_brand", "p_type", "p_size", "ps_suppkey"], [], n)
    cnt = _count("COUNT(DISTINCT partsupp.ps_suppkey)")
    g = _grouped(pairs, ["p_brand", "p_type", "p_size"], [cnt], n)
    return _project_sort(g, [(g.c("p_brand"), "p_brand"), (g.c("p_type"), "p_type"), (g.c("p_size"), "p_size"), (g.c(cnt["name"]), "supplier_cnt")],
                         [("supplier_cnt", True), ("p_brand", False), ("p_type", False), ("p_size", False)])


def tpch_q18(n: int = TARGET_PARTITIONS, as_inner: bool = False) -> dict:
    qty = _sum("SUM(lineitem.l_quantity)", column("l_quantity", 1))
    big = _grouped(_tpch_scan("lineitem", ["l_orderkey", "l_quantity"], n), ["l_orderkey"], [qty], n)
    big = _filter(big, lambda r: binary(r.c(qty["name"]), "Gt", _f64(300)))
    cu = _tpch_scan("customer", ["c_custkey", "c_name"], n)
    od = _tpch_scan("orders", ["o_orderkey", "o_custkey", "o_totalprice", "o_orderdate"], n)
    li = _tpch_scan("lineitem", ["l_orderkey", "l_quantity"], n)
    od = _semi(od, big, [("o_orderkey", "l_orderkey")], n, as_inner=as_inner)
    if as_inner:  # drop the DISTINCT keys: the joins below name l_orderkey / l_quantity of the second lineitem scan
        od = _subquery(od, [(od.c(c), c) for c in ("o_orderkey", "o_custkey", "o_totalprice", "o_orderdate")])
    j = _join(cu, od, [("c_custkey", "o_custkey")], n)
    j = _join(j, li, [("o_orderkey", "l_orderkey")], n)
    total = _sum("SUM(lineitem.l_quantity)", j.c("l_quantity"))
    g = _grouped(j, ["c_name", "c_custkey", "o_orderkey", "o_orderdate", "o_totalprice"], [total], n)
    return _project_sort(g, [(g.c(c), c) for c in ("c_name", "c_custkey", "o_orderkey", "o_orderdate", "o_totalprice")] +
                         [(g.c(total["name"]), "SUM(lineitem.l_quantity)")], [("o_totalprice", True), ("o_orderdate", False)])


def _orders_with_suppliers(li: _Rel, name: str, n: int) -> _Rel:
    """The l_orderkey of orders with more than one distinct l_suppkey among the lines of `li`."""
    pairs = _grouped(li, ["l_orderkey", "l_suppkey"], [], n)
    g = _grouped(pairs, ["l_orderkey"], [_count(name)], n)
    return _filter(g, lambda r: binary(r.c(name), "Gt", literal("UInt64", 1)))


def tpch_q21(n: int = TARGET_PARTITIONS) -> dict:
    late = lambda r: binary(r.c("l_receiptdate"), "Gt", r.c("l_commitdate"))
    su = _tpch_scan("supplier", ["s_suppkey", "s_name", "s_nationkey"], n)
    l1 = _filter(_tpch_scan("lineitem", ["l_orderkey", "l_suppkey", "l_commitdate", "l_receiptdate"], n), late)
    l2 = _tpch_scan("lineitem", ["l_orderkey", "l_suppkey"], n)
    l3 = _filter(_tpch_scan("lineitem", ["l_orderkey", "l_suppkey", "l_commitdate", "l_receiptdate"], n), late)
    od = _filter(_tpch_scan("orders", ["o_orderkey", "o_orderstatus"], n), lambda r: binary(r.c("o_orderstatus"), "Eq", literal("Utf8", "F")))
    na = _filter(_tpch_scan("nation", ["n_nationkey", "n_name"], n), lambda r: binary(r.c("n_name"), "Eq", literal("Utf8", "SAUDI ARABIA")))
    l1 = _semi(l1, _orders_with_suppliers(l2, "COUNT(DISTINCT l2.l_suppkey)", n), [("l_orderkey", "l_orderkey")], n, "Semi")
    l1 = _semi(l1, _orders_with_suppliers(l3, "COUNT(DISTINCT l3.l_suppkey)", n), [("l_orderkey", "l_orderkey")], n, "Anti")
    j = _join(su, l1, [("s_suppkey", "l_suppkey")], n)
    j = _join(j, od, [("l_orderkey", "o_orderkey")], n)
    j = _join(j, na, [("s_nationkey", "n_nationkey")], n)
    cnt = _count("COUNT(UInt8(1))")
    g = _grouped(j, ["s_name"], [cnt], n)
    return _project_sort(g, [(g.c("s_name"), "s_name"), (g.c(cnt["name"]), "numwait")], [("numwait", True), ("s_name", False)])


# Kept apart from TPCH_QUERIES and TPCH_MORE_QUERIES, whose entries the existing suites and tools iterate.
TPCH_SUBQUERY_QUERIES = {"q4": tpch_q4, "q16": tpch_q16, "q18": tpch_q18, "q21": tpch_q21}
TPCH_SUBQUERY_SOURCES = {"q4": ["orders", "lineitem"], "q16": ["partsupp", "part", "supplier"],
                         "q18": ["lineitem", "customer", "orders", "lineitem"],
                         "q21": ["supplier", "lineitem", "lineitem", "lineitem", "orders", "nation"]}
