"""NEXMark q9, q10 (= q0), q12 and q13 without a GPU (`-m "not gpu"`): the plans' shapes, the CPU oracle against an
independent restatement of each query on Arrow C++ compute / Acero (below, written from the SQL text like
oracle/acero_ref.py) at three seeds and two partition counts, the committed golden vectors
(tests/golden/nexmark_more_golden.json, written by tests/golden/make_golden_more.py), and the generator's additions
(bids with a processing time, the synthetic side input).  The helpers here also serve tests/test_gpu_nexmark_more.py."""
import hashlib
import json
from pathlib import Path

import numpy as np
import pyarrow as pa
import pytest

import pyarrow.compute as pc

import flock_b200 as fb
import oracle
from flock_b200 import nexgen, plans

GOLDEN_MORE = Path(__file__).parent / "golden" / "nexmark_more_golden.json"


def more_events(n_events: int, seed: int, batch_rows: int = 8192) -> dict:
    """The relations q9 / q10 / q12 / q13 read for the first `n_events` events."""
    ev = nexgen.generate(n_events, seed=seed, batch_rows=batch_rows, relations=("auction", "bid"))
    _, n_a, n_b = nexgen.relation_counts(n_events)
    ev["bid_ptime"] = nexgen.split_batches(nexgen.bids_ptime(n_b, seed), batch_rows)
    ev["side_input"] = nexgen.split_batches(nexgen.side_input(n_a, seed), batch_rows)
    return ev


def more_sources(query: str, ev: dict) -> list:
    return [[ev[r]] for r in plans.MORE_SOURCES[query]]


# ---- the second restatement: Arrow C++ compute / Acero, from the SQL text (benchmarks/src/nexmark/query/qN.sql) ---------
def _table(batches) -> pa.Table:
    return pa.Table.from_batches(list(batches)).combine_chunks()


def acero_q10(bid) -> pa.Table:
    """SELECT auction, bidder, price, b_date_time FROM bid  (q0.sql: SELECT * FROM bid)"""
    return _table(bid).select(["auction", "bidder", "price", "b_date_time"])


def acero_q9(auction, bid, outer=None) -> pa.Table:
    """SELECT auction, bidder, price, b_date_time FROM bid JOIN (SELECT a_id AS id, MAX(price) AS final FROM auction
       JOIN bid ON a_id = auction WHERE b_date_time BETWEEN a_date_time AND expires GROUP BY a_id) AS Q
       ON auction = id AND price = final
    The BETWEEN belongs to the subquery: the outer join takes every bid at the top price, whenever it was placed.
    `outer`: the bids of the outer scan when they differ from the subquery's (Acero's join matches no NULL key)."""
    a = _table(auction).select(["a_id", "a_date_time", "expires"])
    b = _table(bid)
    j = a.join(b.select(["auction", "price", "b_date_time"]), keys="a_id", right_keys="auction", join_type="inner")
    ts = j["b_date_time"]
    j = j.filter(pc.and_(pc.greater_equal(ts, j["a_date_time"]), pc.less_equal(ts, j["expires"])))
    q = j.group_by("a_id").aggregate([("price", "max")]).rename_columns(["id", "final"])
    o = b if outer is None else _table(outer)
    return o.join(q, keys=["auction", "price"], right_keys=["id", "final"], join_type="inner").select(["auction", "bidder", "price", "b_date_time"])


def acero_q12(bid_ptime) -> pa.Table:
    """SELECT bidder, COUNT(*) AS bid_count, MIN(p_time) AS start_time, MAX(p_time) AS end_time FROM bid GROUP BY bidder"""
    g = _table(bid_ptime).group_by("bidder").aggregate([([], "count_all"), ("p_time", "min"), ("p_time", "max")])
    return pa.table({"bidder": g["bidder"], "bid_count": pc.cast(g["count_all"], pa.uint64()), "start_time": g["p_time_min"],
                     "end_time": g["p_time_max"]})


def acero_q13(bid, side_input) -> pa.Table:
    """SELECT auction, bidder, price, b_date_time, value FROM bid JOIN side_input ON auction = key"""
    j = _table(bid).join(_table(side_input), keys="auction", right_keys="key", join_type="inner")
    return j.select(["auction", "bidder", "price", "b_date_time", "value"])


ACERO = {"q9": acero_q9, "q10": acero_q10, "q12": acero_q12, "q13": acero_q13}


def acero(query: str, ev: dict) -> pa.Table:
    return ACERO[query](*[ev[r] for r in dict.fromkeys(plans.MORE_SOURCES[query])])


def with_null_keys(batches, seed: int, fraction: float = 0.1) -> list:
    """The bids with `auction` and `price` nullable and about `fraction` of each set to NULL."""
    t = _table(batches)
    rng = np.random.default_rng(seed)
    masks = {c: rng.random(t.num_rows) < fraction for c in ("auction", "price")}
    schema = pa.schema([f.with_nullable(f.name in masks) for f in t.schema], metadata=t.schema.metadata)
    cols = [pa.array(t[f.name].to_numpy(), f.type, mask=masks[f.name]) if f.name in masks else t[f.name].combine_chunks() for f in schema]
    return nexgen.split_batches(pa.RecordBatch.from_arrays(cols, schema=schema), 8192)


def without_null_keys(batches) -> list:
    """The rows of `batches` whose auction and price are both set: in an inner join on (auction, price) the others match
    nothing, so q9 over these rows is q9 over all of them.  (The CPU oracle refuses NULL inputs.)"""
    t = _table(batches)
    return nexgen.split_batches(t.filter(pc.and_(pc.is_valid(t["auction"]), pc.is_valid(t["price"]))).to_batches()[0], 8192)


def digest(t: pa.Table) -> str:
    return hashlib.sha256(json.dumps(t.to_pylist(), default=str, sort_keys=True).encode()).hexdigest()


def q9_numpy(auction: pa.Table, bid: pa.Table) -> pa.Table:
    """q9 from the SQL with numpy: each auction's MAX(price) over the bids inside its lifetime, then every bid (in the
    lifetime or not) whose (auction, price) is (a_id, that MAX); NULL auction or price matches nothing."""
    a_id = auction["a_id"].to_numpy().astype(np.int64)
    lo, size = int(a_id.min()), int(a_id.max() - a_id.min() + 1)
    start = np.zeros(size, np.int64)
    end = np.zeros(size, np.int64)
    known = np.zeros(size, bool)
    start[a_id - lo] = auction["a_date_time"].cast(pa.int64()).to_numpy()
    end[a_id - lo] = auction["expires"].cast(pa.int64()).to_numpy()
    known[a_id - lo] = True
    valid = bid["auction"].is_valid().to_numpy(zero_copy_only=False) & bid["price"].is_valid().to_numpy(zero_copy_only=False)
    auc = bid["auction"].fill_null(0).to_numpy().astype(np.int64)
    price = bid["price"].fill_null(0).to_numpy().astype(np.int64)
    ts = bid["b_date_time"].cast(pa.int64()).to_numpy()
    idx = auc - lo
    inside = valid & (idx >= 0) & (idx < size)
    inside[inside] &= known[idx[inside]]
    life = inside.copy()
    life[inside] &= (ts[inside] >= start[idx[inside]]) & (ts[inside] <= end[idx[inside]])
    final = np.full(size, np.iinfo(np.int64).min)
    np.maximum.at(final, idx[life], price[life])
    keep = inside.copy()
    keep[inside] &= price[inside] == final[idx[inside]]
    return bid.select(["auction", "bidder", "price", "b_date_time"]).filter(pa.array(keep))


def q9_edge_bids(ev: dict) -> tuple[list, dict]:
    """The bids of `ev` plus bids that reach q9's corners: ties at an auction's top price (in its lifetime), bids at the
    top price placed before the auction opened (outside its lifetime: they set no MAX but match it), bids for auction
    ids below and above every generated id.  Returns the batches and the (auction, bidder, price) of the ties and of
    the early bids."""
    a = pa.Table.from_batches(ev["auction"]).combine_chunks()
    b = pa.Table.from_batches(ev["bid"]).combine_chunks()
    top = q9_numpy(a, b).slice(0, 20)
    auc, bidder, price = (top[c].to_numpy().astype(np.int64) for c in ("auction", "bidder", "price"))
    ts = top["b_date_time"].cast(pa.int64()).to_numpy()
    opens = dict(zip(a["a_id"].to_pylist(), a["a_date_time"].cast(pa.int64()).to_pylist()))
    lo, hi = int(a["a_id"].to_numpy().min()), int(a["a_id"].to_numpy().max())
    t0 = int(b["b_date_time"].cast(pa.int64())[0].as_py())
    new = {"auction": np.concatenate([auc[:10], auc[10:], [lo - 7, lo - 1, hi + 1, hi + 5000]]),
           "bidder": np.concatenate([bidder[:10] + 1, bidder[10:] + 2, np.arange(1000, 1004)]),
           "price": np.concatenate([price, [100] * 4]),
           "b_date_time": np.concatenate([ts[:10], [opens[int(x)] - 1 for x in auc[10:]], [t0] * 4])}
    add = pa.RecordBatch.from_arrays([pa.array(new[f.name].astype(np.int64)).cast(f.type) for f in b.schema], schema=b.schema)
    whole = pa.Table.from_batches([*ev["bid"], add]).combine_chunks().to_batches()[0]
    rows = list(zip(*(new[c].tolist() for c in ("auction", "bidder", "price"))))
    return nexgen.split_batches(whole, 8192), {"ties": rows[:10], "before_open": rows[10:20], "outside": rows[20:]}


# ---- plan shapes -----------------------------------------------------------------------------------------------------
def test_plan_shapes():
    s9 = fb.ExecutionContext(None, plans.q9()).plan_str()
    assert "join_type=Inner, on=[(auction, id), (price, final)]" in s9
    assert "join_type=Inner, on=[(a_id, auction)]" in s9
    assert s9.count("FilterExec: b_date_time@6 >= a_date_time@1 AND b_date_time@6 <= expires@2") == 1
    assert "RepartitionExec: partitioning=Hash([auction@0, price@2], 8)" in s9 and "RepartitionExec: partitioning=Hash([id@0, final@1], 8)" in s9
    assert "HashAggregateExec: mode=FinalPartitioned, gby=[a_id@0 as a_id], aggr=[MAX(bid.price)]" in s9
    assert "ProjectionExec: expr=[a_id@0 as id, MAX(bid.price)@1 as final]" in s9
    assert s9.splitlines()[0] == "ProjectionExec: expr=[auction@0 as auction, bidder@1 as bidder, price@2 as price, b_date_time@3 as b_date_time]"
    s10 = fb.ExecutionContext(None, plans.q10()).plan_str().splitlines()
    assert s10 == ["ProjectionExec: expr=[auction@0 as auction, bidder@1 as bidder, price@2 as price, b_date_time@3 as b_date_time]",
                   "  RepartitionExec: partitioning=RoundRobinBatch(8)", "    MemoryExec: partitions=0, gpu_resident_rows=0"]
    assert plans.q0 is plans.q10
    s12 = fb.ExecutionContext(None, plans.q12()).plan_str()
    assert "aggr=[COUNT(UInt8(1)), MIN(bid.p_time), MAX(bid.p_time)]" in s12 and "gby=[bidder@0 as bidder]" in s12
    assert "COUNT(UInt8(1))@1 as bid_count, MIN(bid.p_time)@2 as start_time, MAX(bid.p_time)@3 as end_time" in s12
    s13 = fb.ExecutionContext(None, plans.q13()).plan_str()
    assert "join_type=Inner, on=[(auction, key)]" in s13 and "value@5 as value" in s13
    # q12 scans bidder and p_time (nanoseconds in UTC) of the bid relation with processing time
    leaf = plans.q12()["input"]["input"]["input"]["input"]["input"]["input"]
    assert leaf["projection"] == [1, 4] and leaf["schema"]["fields"][4]["data_type"] == {"Timestamp": ["Nanosecond", "UTC"]}


# ---- the two oracles agree ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [42, 7, 1234])
@pytest.mark.parametrize("query", ["q9", "q10", "q12", "q13"])
def test_oracle_matches_acero_more(query, seed):
    ev = more_events(60_000, seed)
    want = acero(query, ev)
    assert want.num_rows > 0
    for n in (1, 8):
        oracle.assert_tables_equal(oracle.execute_plan(plans.MORE_QUERIES[query](n), more_sources(query, ev)), want)


def test_q9_edges_in_both_oracles():
    ev = more_events(60_000, 42)
    bids, added = q9_edge_bids(ev)
    ev = {**ev, "bid": bids}
    got = oracle.execute_plan(plans.q9(), more_sources("q9", ev))
    oracle.assert_tables_equal(got, acero("q9", ev))
    want = q9_numpy(pa.Table.from_batches(ev["auction"]), pa.Table.from_batches(bids))
    oracle.assert_tables_equal(got, want)
    rows = set(zip(*[got[c].to_pylist() for c in ("auction", "bidder", "price")]))
    assert set(added["ties"]) <= rows and set(added["before_open"]) <= rows and not set(added["outside"]) & rows
    auctions_won = set(got["auction"].to_pylist())
    a_ids = set(pa.Table.from_batches(ev["auction"])["a_id"].to_pylist())
    assert a_ids - auctions_won                                                  # some auctions have no in-lifetime bid


def test_q9_null_keys_match_nothing():
    """A nullable outer bid relation (the first bid source feeds the outer join): NULL auction or price never joins.
    Acero over the NULLs, the oracle over the rows that can match, and numpy agree."""
    ev = more_events(30_000, 7)
    nullable = with_null_keys(ev["bid"], 3)
    got = oracle.execute_plan(plans.q9(), [[ev["auction"]], [without_null_keys(nullable)], [ev["bid"]]])
    oracle.assert_tables_equal(got, acero_q9(ev["auction"], ev["bid"], outer=nullable))
    inner_final = q9_numpy(_table(ev["auction"]), _table(ev["bid"]))
    keep = set(zip(inner_final["auction"].to_pylist(), inner_final["price"].to_pylist()))
    nb = _table(nullable)
    expect = [i for i, (a, p) in enumerate(zip(nb["auction"].to_pylist(), nb["price"].to_pylist())) if a is not None and p is not None and (a, p) in keep]
    assert got.num_rows == len(expect) and got.num_rows > 0 and len(expect) < inner_final.num_rows
    assert sorted(zip(got["auction"].to_pylist(), got["bidder"].to_pylist())) == sorted((nb["auction"][i].as_py(), nb["bidder"][i].as_py()) for i in expect)


def test_golden_vectors_more_reproduce():
    g = json.loads(GOLDEN_MORE.read_text())
    ev = more_events(g["n_events"], g["seed"], g["batch_rows"])
    for query, want in g["queries"].items():
        got = oracle.canonical(oracle.execute_plan(plans.MORE_QUERIES[query](), more_sources(query, ev)))
        assert got.num_rows == want["num_rows"] and got.schema.names == want["columns"], query
        assert digest(got) == want["digest"], query


# ---- generator additions ---------------------------------------------------------------------------------------------------
def test_nexgen_more_is_deterministic_and_typed():
    p1, p2 = nexgen.bids_ptime(50_000, seed=5), nexgen.bids_ptime(50_000, seed=5)
    assert p1.equals(p2) and not p1.equals(nexgen.bids_ptime(50_000, seed=6))
    assert p1.schema.equals(nexgen.bid_ptime_schema(), check_metadata=True)
    assert p1.schema.field("p_time").type == pa.timestamp("ns", tz="UTC") and not p1.schema.field("p_time").nullable
    assert p1.select(["auction", "bidder", "price", "b_date_time"]).equals(nexgen.bids(50_000, seed=5))
    t = p1["p_time"].cast(pa.int64()).to_numpy()
    assert np.all(np.diff(t) >= 0) and np.unique(t).size < t.size                   # monotone, with repeats
    assert nexgen.bids_ptime(10, 5, first_bid=40)["p_time"].equals(p1["p_time"].slice(40, 10))
    s1, s2 = nexgen.side_input(20_000, seed=5), nexgen.side_input(20_000, seed=5)
    assert s1.equals(s2) and not s1.equals(nexgen.side_input(20_000, seed=6))
    assert s1.schema.equals(nexgen.side_input_schema(), check_metadata=True) and s1.schema.metadata == {b"name": b"side_input"}
    assert [(f.name, f.type, f.nullable) for f in s1.schema] == [("key", pa.int32(), False), ("value", pa.int32(), False)]
    keys = s1["key"].to_numpy()
    ids = np.arange(nexgen.FIRST_AUCTION_ID, nexgen.FIRST_AUCTION_ID + 20_000)
    assert np.all(np.diff(keys) > 0) and np.isin(keys, ids).all() and 0.8 * ids.size < keys.size < 0.95 * ids.size
