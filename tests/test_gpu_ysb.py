"""The Yahoo Streaming Benchmark query on the GPU (`-m gpu`): through flock_context_unmarshal / feed / execute against the
CPU oracle at three seeds, at 10 M events against numpy, stage by stage against the whole plan, from NDJSON text, and
the corners of the one-pass join count (dim_count_kernel): duplicate and NULL keys, keys one byte apart, empty inputs,
the dimension on either side, an Int32 key, no filter, event filters the term form refuses, and dimensions of D_MAX and
D_MAX + 1 rows.  The kernels that
ran are read from the launch profile."""
import collections

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import flock_b200 as fb
import oracle
from flock_b200 import nexgen, plans, ysbgen
from test_ysb_host import COUNT, _split, acero_ysb, ysb_inputs, ysb_sources

pytestmark = pytest.mark.gpu

D_MAX = 4096
JOIN_KERNELS = ("join_build_kernel", "join_count_scan_kernel", "join_emit_kernel", "join_one_kernel")


def run_gpu(ctx, plan, sources):
    ec = fb.ExecutionContext(ctx, plan)
    ec.feed_data_sources(sources)
    ctx.profile_begin()
    out = pa.Table.from_batches(ec.execute()[0])
    prof = ctx.profile_end()
    ec.clean_data_sources()
    ec.close()
    return out, prof


def launches(prof, name):
    return prof.get(name, {}).get("launches", 0)


def assert_fused(prof):
    assert launches(prof, "dim_count_kernel") == 1, sorted(prof)
    assert all(launches(prof, k) == 0 for k in JOIN_KERNELS), sorted(prof)
    assert launches(prof, "filter_compact_kernel") <= 1, sorted(prof)      # the selection of the counted dimension rows


def assert_schema(got):
    assert got.schema.names[-1] == COUNT and got.schema.field(COUNT).type == pa.uint64()


# ---- plans beside the reference's: the same query in other shapes ------------------------------------------------------
def star_plan(dim_left: bool = False, with_filter: bool = True, n: int = 8, pred: dict | None = None) -> dict:
    """ysb with the dimension on either side of the join, with or without the event filter (event_type = 'view', or
    `pred` over ad_id 0 and event_type 1)."""
    scan = plans.repartition_rr(plans.memory_exec(plans.AD_EVENT, [2, 4]), n)
    if with_filter:
        pred = pred or plans.binary(plans.column("event_type", 1), "Eq", plans.literal("Utf8", "view"))
        scan = plans.coalesce_batches_exec(plans.filter_exec(pred, scan))
    events = plans.coalesce_batches_exec(plans.repartition_hash(scan, [plans.column("ad_id", 0)], n))
    camps = plans.coalesce_batches_exec(plans.repartition_hash(plans.repartition_rr(plans.memory_exec(plans.CAMPAIGN, [0, 1]), n), [plans.column("c_ad_id", 0)], n))
    if dim_left:   # c_ad_id 0, campaign_id 1, ad_id 2, event_type 3
        join, group = plans.hash_join_exec(camps, events, [(plans.column("c_ad_id", 0), plans.column("ad_id", 0))]), ("campaign_id", 1)
    else:
        join, group = plans.hash_join_exec(events, camps, [(plans.column("ad_id", 0), plans.column("c_ad_id", 0))]), ("campaign_id", 3)
    return plans.two_phase_aggregate([group], [plans._ysb_count()], plans.coalesce_batches_exec(join), n)


def bids_by_value_plan(n: int = 8) -> dict:
    """SELECT value, COUNT(*) FROM bid JOIN side_input ON auction = key GROUP BY value: an Int32 key."""
    bid = plans.coalesce_batches_exec(plans.repartition_hash(plans.repartition_rr(plans.memory_exec(plans.BID, [0]), n), [plans.column("auction", 0)], n))
    side = plans.coalesce_batches_exec(plans.repartition_hash(plans.repartition_rr(plans.memory_exec(plans.SIDE_INPUT, [0, 1]), n), [plans.column("key", 0)], n))
    join = plans.hash_join_exec(bid, side, [(plans.column("auction", 0), plans.column("key", 0))])   # auction 0, key 1, value 2
    return plans.two_phase_aggregate([("value", 2)], [plans._ysb_count()], plans.coalesce_batches_exec(join), n)


# ---- the query ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [42, 7, 1234])
def test_ysb_matches_oracle(gpu_ctx, seed):
    inputs = ysb_inputs(120_000, seed)
    got, prof = run_gpu(gpu_ctx, plans.ysb(), ysb_sources(inputs))
    want = oracle.execute_plan(plans.ysb(), ysb_sources(inputs))
    assert want.num_rows == 100
    oracle.assert_tables_equal(got, want)
    assert_fused(prof)
    assert [(f.name, f.type, f.nullable) for f in got.schema] == [("campaign_id", pa.utf8(), False), (COUNT, pa.uint64(), True)]


def test_ysb_10m_events_against_numpy(gpu_ctx):
    camp = ysbgen.campaigns(100, 10, 42)
    ev = ysbgen.ad_events(10_000_000, camp, 42, columns=["ad_id", "event_type"])
    got, prof = run_gpu(gpu_ctx, plans.ysb(), [[_split(ev, 65536)], [[camp]]])
    ad = pc.index_in(ev["ad_id"], value_set=camp["c_ad_id"]).to_numpy()
    views = pc.equal(ev["event_type"], "view").to_numpy(zero_copy_only=False)
    cids = camp["campaign_id"].to_pylist()
    campaign_of_ad = np.unique(np.array(cids), return_inverse=True)[1]
    names = np.unique(np.array(cids))
    want = np.bincount(campaign_of_ad[ad[views]], minlength=names.size)
    assert want.sum() > 3_000_000
    order = np.argsort(np.array(got["campaign_id"].to_pylist()))
    assert np.array_equal(np.array(got["campaign_id"].to_pylist())[order], names)
    assert np.array_equal(got[COUNT].to_numpy()[order], want.astype(np.uint64))
    assert_fused(prof)
    # no launch of the generic path over the events: the compaction and gathers that ran select and group the 1 000
    # counted dimension rows -- 5 000 events launch exactly the same kernels
    _, small = run_gpu(gpu_ctx, plans.ysb(), [[[ev.slice(0, 5000)]], [[camp]]])
    assert {k: v["launches"] for k, v in prof.items()} == {k: v["launches"] for k, v in small.items()}


def test_ysb_stages_one_after_another_equal_the_whole_plan(gpu_ctx):
    inputs = ysb_inputs(200_000, 7)
    whole, _ = run_gpu(gpu_ctx, plans.ysb(), ysb_sources(inputs))
    s0, s1, s2 = plans.ysb_stages()
    ec0 = fb.ExecutionContext(gpu_ctx, s0)
    ec0.feed_data_sources(ysb_sources(inputs))
    views, camps = ec0.execute_device(0), ec0.execute_device(1)
    assert views.num_rows == pc.sum(pc.equal(_table_of(inputs["ad_event"])["event_type"], "view")).as_py()
    ec1 = fb.ExecutionContext(gpu_ctx, s1[0])
    ec1.feed_tables([views, camps])
    gpu_ctx.profile_begin()
    states = ec1.execute_device(0)
    prof = gpu_ctx.profile_end()
    assert_fused(prof)                                   # stage 1: the Partial form of the one-pass count
    assert states.schema.names == ["campaign_id", COUNT + "[count]"]
    ec2 = fb.ExecutionContext(gpu_ctx, s2[0])
    ec2.feed_tables([states])
    staged = ec2.execute_device(0).to_arrow()
    oracle.assert_tables_equal(staged, whole)            # sorted compare, launcher/aws/mod.rs:680-844
    oracle.assert_tables_equal(staged, acero_ysb(inputs["ad_event"], inputs["campaign"]))
    for e in (ec0, ec1, ec2):
        e.close()


def _table_of(batches):
    return pa.Table.from_batches(batches)


def test_ysb_from_ndjson_text(gpu_ctx):
    camp = ysbgen.campaigns(100, 10, 1234)
    ev = ysbgen.ad_events(30_000, camp, 1234)
    text = ysbgen.to_ndjson(ev)
    events = gpu_ctx.import_ndjson(ysbgen.ad_event_schema(), text)
    assert events.num_rows == ev.num_rows
    ec = fb.ExecutionContext(gpu_ctx, plans.ysb())
    ec.feed_tables([events, gpu_ctx.import_batches([camp])])
    got = ec.execute_device(0).to_arrow()
    ec.close()
    oracle.assert_tables_equal(got, oracle.execute_plan(plans.ysb(), [[[ev]], [[camp]]]))


# ---- corners ----------------------------------------------------------------------------------------------------------------
def test_duplicate_dimension_keys_count_once_per_dimension_row(gpu_ctx):
    camp = ysbgen.campaigns(20, 5, 3)
    ev = ysbgen.ad_events(50_000, camp, 3, columns=["ad_id", "event_type"])
    a0, a1 = camp["c_ad_id"][0].as_py(), camp["c_ad_id"][7].as_py()
    extra = pa.RecordBatch.from_pydict({"c_ad_id": [a0, a0, a1, "unused-ad"], "campaign_id": ["extra", "extra", "other", "never"]}, schema=ysbgen.campaign_schema())
    src = [[_split(ev, 8192)], [[camp, extra]]]
    got, prof = run_gpu(gpu_ctx, plans.ysb(), src)
    assert_fused(prof)
    want = oracle.execute_plan(plans.ysb(), src)
    oracle.assert_tables_equal(got, want)
    counts = dict(zip(got["campaign_id"].to_pylist(), got[COUNT].to_pylist()))
    evt = pa.Table.from_batches([ev])
    v0 = pc.sum(pc.and_(pc.equal(evt["ad_id"], a0), pc.equal(evt["event_type"], "view"))).as_py()
    assert counts["extra"] == 2 * v0 and "never" not in counts


def _nullable(batch, masks: dict) -> pa.RecordBatch:
    schema = pa.schema([f.with_nullable(True) for f in batch.schema], metadata=batch.schema.metadata)
    cols = [pa.array(batch[f.name].to_pylist(), f.type, mask=masks[f.name]) if f.name in masks else batch[f.name] for f in batch.schema]
    return pa.RecordBatch.from_arrays(cols, schema=schema)


def test_null_keys_event_types_and_group_values(gpu_ctx):
    camp = ysbgen.campaigns(30, 10, 11)
    ev = ysbgen.ad_events(40_000, camp, 11, columns=["ad_id", "event_type"])
    rng = np.random.default_rng(11)
    ev_n = _nullable(ev, {"ad_id": rng.random(ev.num_rows) < 0.05, "event_type": rng.random(ev.num_rows) < 0.05})
    key_null = np.zeros(camp.num_rows, bool)
    key_null[[3, 150]] = True                                            # NULL dimension keys match nothing
    group_null = np.zeros(camp.num_rows, bool)
    group_null[20:30] = True                                             # campaign 2 has a NULL id: a group of its own
    camp_n = _nullable(camp, {"c_ad_id": key_null, "campaign_id": group_null})
    src = [[_split(ev_n, 8192)], [[camp_n]]]
    got, prof = run_gpu(gpu_ctx, plans.ysb(), src)
    assert_fused(prof)
    want = acero_ysb([ev_n], [camp_n])                                    # the CPU oracle refuses NULL inputs
    assert None in want["campaign_id"].to_pylist()
    oracle.assert_tables_equal(got, want)
    assert got.schema.field("campaign_id").nullable


def test_keys_one_byte_apart_and_the_empty_string(gpu_ctx):
    keys = ["", "a", "ab", "abc", "abd", "abcd", "b" * 200, "b" * 199 + "c", ysbgen.campaigns(1, 1, 5)["c_ad_id"][0].as_py()]
    camp = pa.RecordBatch.from_pydict({"c_ad_id": keys, "campaign_id": [f"c{i % 4}" for i in range(len(keys))]}, schema=ysbgen.campaign_schema())
    probes = keys + ["abe", "ab ", "b" * 201, "B", "aé", "abcde"]
    rng = np.random.default_rng(5)
    idx = rng.integers(0, len(probes), 30_000)
    types = np.array(ysbgen.EVENT_TYPES)[rng.integers(0, 3, idx.size)]
    schema = pa.schema([plans.AD_EVENT.field("ad_id"), plans.AD_EVENT.field("event_type")], metadata=plans.AD_EVENT.metadata)
    ev = pa.RecordBatch.from_arrays([pa.array(np.array(probes, dtype=object)[idx].tolist()), pa.array(types.tolist())], schema=schema)
    src = [[_split(ev, 4096)], [[camp]]]
    got, prof = run_gpu(gpu_ctx, plans.ysb(), src)
    assert_fused(prof)
    oracle.assert_tables_equal(got, oracle.execute_plan(plans.ysb(), src))
    oracle.assert_tables_equal(got, acero_ysb([ev], [camp]))


def test_empty_fact_empty_dimension_and_nothing_viewed(gpu_ctx):
    camp = ysbgen.campaigns(10, 10, 2)
    ev = ysbgen.ad_events(20_000, camp, 2, columns=["ad_id", "event_type"])
    no_views = ev.filter(pc.not_equal(ev["event_type"], "view"))
    for src in ([[[ev.slice(0, 0)]], [[camp]]], [[[ev]], [[camp.slice(0, 0)]]], [[_split(no_views, 4096)], [[camp]]]):
        got, prof = run_gpu(gpu_ctx, plans.ysb(), src)
        assert got.num_rows == 0
        assert [(f.name, f.type, f.nullable) for f in got.schema] == [("campaign_id", pa.utf8(), False), (COUNT, pa.uint64(), True)]
        assert all(launches(prof, k) == 0 for k in JOIN_KERNELS), sorted(prof)


@pytest.mark.parametrize("dim_left", [False, True])
@pytest.mark.parametrize("with_filter", [True, False])
def test_dimension_on_either_side_with_and_without_filter(gpu_ctx, dim_left, with_filter):
    inputs = ysb_inputs(80_000, 42)
    plan = star_plan(dim_left, with_filter)
    src = ysb_sources(inputs) if not dim_left else [[inputs["campaign"]], [inputs["ad_event"]]]
    got, prof = run_gpu(gpu_ctx, plan, src)
    assert_fused(prof)
    want = oracle.execute_plan(plan, src)
    assert want.num_rows == 100
    oracle.assert_tables_equal(got, want)
    if not with_filter:
        assert sum(got[COUNT].to_pylist()) == 80_000


@pytest.mark.parametrize("kind", ["in_list", "like", "is_not_null"])
def test_fact_filter_the_term_form_refuses_runs_first(gpu_ctx, kind):
    """An event filter the term form cannot evaluate runs as its own filter, in the tree form, before the one-pass count."""
    camp = ysbgen.campaigns(100, 10, 13)
    ev = ysbgen.ad_events(100_000, camp, 13, columns=["ad_id", "event_type"])
    etype, utf8 = plans.column("event_type", 1), lambda s: plans.literal("Utf8", s)
    if kind == "in_list":
        pred, keep = plans.in_list(etype, [utf8("view"), utf8("click")]), pc.is_in(ev["event_type"], value_set=pa.array(["view", "click"]))
    elif kind == "like":
        pred, keep = plans.binary(etype, "Like", utf8("%e%")), pc.match_like(ev["event_type"], "%e%")
    else:
        ev = _nullable(ev, {"event_type": np.random.default_rng(13).random(ev.num_rows) < 0.3})
        pred, keep = plans.is_not_null(etype), pc.is_valid(ev["event_type"])
    got, prof = run_gpu(gpu_ctx, star_plan(pred=pred), [[_split(ev, 8192)], [[camp]]])
    kept = pa.Table.from_batches([ev]).filter(keep)
    assert 0 < kept.num_rows < ev.num_rows
    want = collections.Counter(kept.join(pa.Table.from_batches([camp]), "ad_id", "c_ad_id", join_type="inner")["campaign_id"].to_pylist())
    assert dict(zip(got["campaign_id"].to_pylist(), got[COUNT].to_pylist())) == want
    assert launches(prof, "dim_count_kernel") == 1 and all(launches(prof, k) == 0 for k in JOIN_KERNELS), sorted(prof)


def test_int32_key_bids_by_side_input_value(gpu_ctx):
    bids = nexgen.split_batches(nexgen.bids(300_000, seed=7), 65536)
    side = nexgen.side_input(3000, seed=7)
    assert side.num_rows <= D_MAX
    src = [[bids], [[side]]]
    got, prof = run_gpu(gpu_ctx, bids_by_value_plan(), src)
    assert_fused(prof)
    want = oracle.execute_plan(bids_by_value_plan(), src)
    assert want.num_rows > 0
    oracle.assert_tables_equal(got, want)


def test_dimension_of_d_max_rows_and_one_more(gpu_ctx):
    camp = ysbgen.campaigns(1024, 4, 9)
    assert camp.num_rows == D_MAX
    ev = ysbgen.ad_events(200_000, camp, 9, columns=["ad_id", "event_type"])
    one_more = pa.RecordBatch.from_pydict({"c_ad_id": ["no-event-names-this-ad"], "campaign_id": ["late"]}, schema=ysbgen.campaign_schema())
    at_max, prof_max = run_gpu(gpu_ctx, plans.ysb(), [[_split(ev, 65536)], [[camp]]])
    over, prof_over = run_gpu(gpu_ctx, plans.ysb(), [[_split(ev, 65536)], [[camp, one_more]]])
    assert_fused(prof_max)
    assert launches(prof_over, "dim_count_kernel") == 0 and launches(prof_over, "join_build_kernel") == 1, sorted(prof_over)
    oracle.assert_tables_equal(at_max, over)
    assert at_max.schema == over.schema
    oracle.assert_tables_equal(at_max, oracle.execute_plan(plans.ysb(), [[_split(ev, 65536)], [[camp]]]))


@pytest.mark.parametrize("query", ["q1", "q2", "q3", "q4", "q5", "q6", "q7", "q8", "q9", "q10", "q12", "q13"])
def test_nexmark_profiles_have_no_dim_count(gpu_ctx, query):
    from test_nexmark_more_host import more_events
    ev = more_events(60_000, 42)
    ev["person"] = nexgen.generate(60_000, seed=42, batch_rows=8192, relations=("person",))["person"]
    table, sources = (plans.QUERIES, plans.SOURCES) if query in plans.QUERIES else (plans.MORE_QUERIES, plans.MORE_SOURCES)
    _, prof = run_gpu(gpu_ctx, table[query](), [[ev[r]] for r in sources[query]])
    assert launches(prof, "dim_count_kernel") == 0 and launches(prof, "dim_count_build_kernel") == 0, sorted(prof)
