"""The Yahoo Streaming Benchmark query without a GPU (`-m "not gpu"`): the generator's distributions, the plans' shapes
against the reference's three stages, the CPU oracle against an independent Acero restatement of the SQL (whole plan
and stage by stage, 1 and 8 partitions, three seeds) and the committed golden vector (tests/golden/ysb_golden.json,
written by tests/golden/make_golden_ysb.py).  The helpers here also serve tests/test_gpu_ysb.py."""
import hashlib
import json
import re
from pathlib import Path

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import flock_b200 as fb
import oracle
from flock_b200 import plans, ysbgen

GOLDEN_YSB = Path(__file__).parent / "golden" / "ysb_golden.json"
UUID_V4 = re.compile(r"^[0-9a-f]{8}-[0-9a-f]{4}-4[0-9a-f]{3}-[89ab][0-9a-f]{3}-[0-9a-f]{12}$")
COUNT = "COUNT(UInt8(1))"


def ysb_inputs(n_events: int, seed: int, n_campaigns: int = 100, ads: int = 10, batch_rows: int = 8192, columns=None) -> dict:
    camp = ysbgen.campaigns(n_campaigns, ads, seed)
    ev = ysbgen.ad_events(n_events, camp, seed, columns=columns)
    return {"ad_event": _split(ev, batch_rows), "campaign": [camp]}


def _split(batch: pa.RecordBatch, rows: int) -> list:
    return [batch.slice(i, rows) for i in range(0, batch.num_rows, rows)] or [batch]


def ysb_sources(inputs: dict) -> list:
    return [[inputs[r]] for r in plans.YSB_SOURCES["ysb"]]


def _table(batches) -> pa.Table:
    return pa.Table.from_batches(list(batches)).combine_chunks()


def acero_ysb(ad_event, campaign) -> pa.Table:
    """SELECT campaign_id, COUNT(*) FROM ad_event INNER JOIN campaign ON ad_id = c_ad_id WHERE event_type = 'view'
       GROUP BY campaign_id   (benchmarks/src/ysb/ysb.sql)"""
    e = _table(ad_event)
    views = e.filter(pc.equal(e["event_type"], "view")).select(["ad_id", "event_type"])
    j = views.join(_table(campaign), keys="ad_id", right_keys="c_ad_id", join_type="inner")
    g = j.group_by("campaign_id").aggregate([([], "count_all")])
    return pa.table({"campaign_id": g["campaign_id"], COUNT: pc.cast(g["count_all"], pa.uint64())})


def oracle_stages(inputs: dict, n: int) -> pa.Table:
    """The three stages one after another (launcher/aws/mod.rs:680-844): every stage's partitions feed the next."""
    s0, s1, s2 = plans.ysb_stages(n)
    ex = oracle.PlanExecutor(s0)
    ex.feed_data_sources(ysb_sources(inputs))
    views, camps = ex.execute_partitioned()
    ex = oracle.PlanExecutor(s1)
    ex.feed_data_sources([views, camps])
    (states,) = ex.execute_partitioned()
    ex = oracle.PlanExecutor(s2)
    ex.feed_data_sources([states])
    return pa.Table.from_batches([b for b in ex.execute()[0] if b.num_rows])


def digest(t: pa.Table) -> str:
    return hashlib.sha256(json.dumps(t.to_pylist(), default=str, sort_keys=True).encode()).hexdigest()


# ---- generator ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [42, 7, 1234])
def test_ysbgen_distributions(seed):
    camp = ysbgen.campaigns(100, 10, seed)
    assert camp.schema.equals(ysbgen.campaign_schema(), check_metadata=True) and camp.schema.metadata == {b"name": b"ysb_campaigns"}
    assert camp.num_rows == 1000 and camp["c_ad_id"].null_count == 0 and camp["campaign_id"].null_count == 0
    ads, cids = camp["c_ad_id"].to_pylist(), camp["campaign_id"].to_pylist()
    assert all(UUID_V4.match(s) for s in ads + cids)
    assert len(set(ads)) == 1000 and len(set(cids)) == 100 and all(cids.count(c) == 10 for c in set(cids))
    n = 60_000
    ev = ysbgen.ad_events(n, camp, seed)
    assert ev.schema.equals(ysbgen.ad_event_schema(), check_metadata=True) and ev.schema.metadata == {b"name": b"ysb_ad_events"}
    assert all(not f.nullable for f in ev.schema)
    assert all(UUID_V4.match(s) for s in ev["user_id"].to_pylist()[:2000] + ev["page_id"].to_pylist()[:2000])
    assert set(ev["ad_id"].to_pylist()) <= set(ads)
    assert set(ev["ip_address"].to_pylist()) == {"0.0.0.0"}
    t = ev["event_time"].cast(pa.int64()).to_numpy()
    assert t[0] == 1 and np.all(np.diff(t) == 1)                       # 1000 events per second: one per millisecond

    def uniform(values, k):                                              # chi-square against the uniform mix, 1e-6 level
        counts = np.unique(np.asarray(values), return_counts=True)[1]
        assert counts.size == k
        exp = len(values) / k
        chi2 = ((counts - exp) ** 2 / exp).sum()
        assert chi2 < k + 8 * np.sqrt(2 * k), chi2
    uniform(ev["ad_id"].to_pylist(), 1000)
    uniform(ev["ad_type"].to_pylist(), 5)
    uniform(ev["event_type"].to_pylist(), 3)
    assert set(ev["ad_type"].to_pylist()) == set(ysbgen.AD_TYPES) and set(ev["event_type"].to_pylist()) == set(ysbgen.EVENT_TYPES)


def test_ysbgen_is_deterministic_and_restricts_columns():
    camp = ysbgen.campaigns(10, 10, 5)
    assert camp.equals(ysbgen.campaigns(10, 10, 5)) and not camp.equals(ysbgen.campaigns(10, 10, 6))
    full = ysbgen.ad_events(5000, camp, 5)
    assert full.equals(ysbgen.ad_events(5000, camp, 5)) and not full.equals(ysbgen.ad_events(5000, camp, 6))
    part = ysbgen.ad_events(5000, camp, 5, columns=["ad_id", "event_type"])
    assert part.schema.names == ["ad_id", "event_type"] and part.schema.metadata == full.schema.metadata
    assert part.equals(full.select(["ad_id", "event_type"]))
    fast = ysbgen.ad_events(4000, camp, 5, columns=["event_time"], events_per_second=4000)
    assert fast["event_time"].cast(pa.int64()).to_numpy()[[0, 3, 4, 3999]].tolist() == [1, 1, 2, 1000]


def test_to_ndjson_is_serde_json_of_adevent():
    camp = ysbgen.campaigns(2, 3, 9)
    ev = ysbgen.ad_events(50, camp, 9)
    text = ysbgen.to_ndjson(ev)
    lines = text.decode().split("\n")
    assert lines[-1] == "" and len(lines) == 51
    first = json.loads(lines[0])
    assert list(first) == ["user_id", "page_id", "ad_id", "ad_type", "event_type", "event_time", "ip_address"]
    assert lines[0].startswith('{"user_id":"') and '"event_time":1,' in lines[0] and " " not in lines[0]
    back = [json.loads(x) for x in lines[:-1]]
    for name in ("ad_id", "event_type", "user_id"):
        assert [r[name] for r in back] == ev[name].to_pylist()
    assert [r["event_time"] for r in back] == ev["event_time"].cast(pa.int64()).to_pylist()
    assert ysbgen.to_ndjson(ev.slice(0, 0)) == b""


# ---- plan shapes: planner.rs:315-345 ---------------------------------------------------------------------------------------
def test_plan_shapes():
    s0 = [fb.ExecutionContext(None, p).plan_str().splitlines() for p in plans.ysb_stages()[0]]
    assert s0[0] == ["CoalesceBatchesExec: target_batch_size=4096", "  RepartitionExec: partitioning=Hash([ad_id@0], 8)",
                     "    CoalesceBatchesExec: target_batch_size=4096", "      FilterExec: event_type@1 = view",
                     "        RepartitionExec: partitioning=RoundRobinBatch(8)", "          MemoryExec: partitions=0, gpu_resident_rows=0"]
    assert s0[1] == ["CoalesceBatchesExec: target_batch_size=4096", "  RepartitionExec: partitioning=Hash([c_ad_id@0], 8)",
                     "    RepartitionExec: partitioning=RoundRobinBatch(8)", "      MemoryExec: partitions=0, gpu_resident_rows=0"]
    (s1,), (s2,) = plans.ysb_stages()[1:]
    assert fb.ExecutionContext(None, s1).plan_str().splitlines() == [
        "CoalesceBatchesExec: target_batch_size=4096", "  RepartitionExec: partitioning=Hash([campaign_id@0], 8)",
        f"    HashAggregateExec: mode=Partial, gby=[campaign_id@3 as campaign_id], aggr=[{COUNT}]",
        "      CoalesceBatchesExec: target_batch_size=4096", "        HashJoinExec: mode=Partitioned, join_type=Inner, on=[(ad_id, c_ad_id)]",
        "          MemoryExec: partitions=0, gpu_resident_rows=0", "          MemoryExec: partitions=0, gpu_resident_rows=0"]
    assert fb.ExecutionContext(None, s2).plan_str().splitlines() == [
        f"ProjectionExec: expr=[campaign_id@0 as campaign_id, {COUNT}@1 as {COUNT}]",
        f"  HashAggregateExec: mode=FinalPartitioned, gby=[campaign_id@0 as campaign_id], aggr=[{COUNT}]",
        "    MemoryExec: partitions=0, gpu_resident_rows=0"]
    assert fb.ExecutionContext(None, plans.ysb_stages()[0]).is_shuffling() and fb.ExecutionContext(None, s1).is_shuffling()
    assert not fb.ExecutionContext(None, s2).is_shuffling()
    whole = fb.ExecutionContext(None, plans.ysb()).plan_str()
    for line in s0[0] + s0[1] + fb.ExecutionContext(None, s1).plan_str().splitlines()[:5]:
        assert line.strip() in whole
    scan = plans.ysb()["input"]["input"]["input"]["input"]["input"]["input"]["left"]["input"]["input"]["input"]["input"]["input"]
    assert scan["execution_plan"] == "memory_exec" and scan["projection"] == [2, 4]        # ad_id, event_type
    assert plans.YSB_QUERIES == {"ysb": plans.ysb} and plans.YSB_SOURCES == {"ysb": ["ad_event", "campaign"]}


# ---- the two oracles agree ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [42, 7, 1234])
def test_oracle_matches_acero_ysb(seed):
    inputs = ysb_inputs(40_000, seed)
    want = acero_ysb(inputs["ad_event"], inputs["campaign"])
    assert want.num_rows == 100 and pc.sum(want[COUNT]).as_py() == pc.sum(pc.equal(_table(inputs["ad_event"])["event_type"], "view")).as_py()
    for n in (1, 8):
        oracle.assert_tables_equal(oracle.execute_plan(plans.ysb(n), ysb_sources(inputs)), want)
        oracle.assert_tables_equal(oracle_stages(inputs, n), want)


def test_oracle_matches_acero_on_duplicate_and_missing_keys():
    """A dimension with a duplicated ad id (its events count twice, once per campaign) and ads that no event names."""
    camp = ysbgen.campaigns(20, 5, 3)
    ev = ysbgen.ad_events(20_000, camp, 3, columns=["ad_id", "event_type"])
    dup = pa.RecordBatch.from_pydict({"c_ad_id": [camp["c_ad_id"][0].as_py(), "unused-ad"], "campaign_id": ["extra", "never"]},
                                     schema=ysbgen.campaign_schema())
    inputs = {"ad_event": _split(ev, 4096), "campaign": [camp, dup]}
    want = acero_ysb(inputs["ad_event"], inputs["campaign"])
    assert "extra" in want["campaign_id"].to_pylist() and "never" not in want["campaign_id"].to_pylist()
    for n in (1, 8):
        oracle.assert_tables_equal(oracle.execute_plan(plans.ysb(n), ysb_sources(inputs)), want)
        oracle.assert_tables_equal(oracle_stages(inputs, n), want)


def test_golden_vector_ysb_reproduces():
    g = json.loads(GOLDEN_YSB.read_text())
    inputs = ysb_inputs(g["n_events"], g["seed"], g["n_campaigns"], g["ads"], g["batch_rows"])
    got = oracle.canonical(oracle.execute_plan(plans.ysb(), ysb_sources(inputs)))
    assert got.num_rows == g["num_rows"] and got.schema.names == g["columns"]
    assert digest(got) == g["digest"]
    assert sum(got[COUNT].to_pylist()) == g["views"]
