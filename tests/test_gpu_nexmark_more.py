"""NEXMark q9, q10, q12 and q13 on the GPU (`-m gpu`): through flock_context_unmarshal / feed / execute against the CPU
oracle at three seeds, at full size against independent numpy statements of the SQL, and q9's outer join answered
from the direct-address (a_id, MAX(price)) table: the kernels that ran are read from the launch profile, and the
corners of the join (ties, bids outside their auction's lifetime or the table's range, NULL keys, empty relations, a
table that another consumer materialised first, a table that is open-addressed) are compared with the oracle."""
import numpy as np
import pyarrow as pa
import pytest

import flock_b200 as fb
import oracle
from flock_b200 import nexgen, plans
from test_nexmark_more_host import acero_q9, more_events, more_sources, q9_edge_bids, q9_numpy, with_null_keys, without_null_keys

pytestmark = pytest.mark.gpu

OUTER_JOIN_KERNELS = ("join_build_kernel", "join_count_scan_kernel", "join_emit_kernel")


def run_gpu(ctx, plan, sources, profile=False):
    ec = fb.ExecutionContext(ctx, plan)
    ec.feed_data_sources(sources)
    if profile:
        ctx.profile_begin()
    out = pa.Table.from_batches(ec.execute()[0])
    prof = ctx.profile_end() if profile else None
    ec.clean_data_sources()
    ec.close()
    return (out, prof) if profile else out


def assert_matches_oracle(got, plan, sources):
    want = oracle.execute_plan(plan, sources)
    if want.num_columns == 0:          # the oracle collects no batch at all from an empty relation
        assert got.num_rows == 0
        return
    oracle.assert_tables_equal(got, want)


def launches(prof, name):
    return prof.get(name, {}).get("launches", 0)


@pytest.mark.parametrize("seed", [42, 7, 1234])
@pytest.mark.parametrize("query", ["q9", "q10", "q12", "q13"])
def test_more_queries_match_oracle(gpu_ctx, query, seed):
    ev = more_events(120_000, seed)
    got = run_gpu(gpu_ctx, plans.MORE_QUERIES[query](), more_sources(query, ev))
    want = oracle.execute_plan(plans.MORE_QUERIES[query](), more_sources(query, ev))
    assert want.num_rows > 0
    oracle.assert_tables_equal(got, want)
    if query == "q12":
        assert got.schema.field("start_time").type == pa.timestamp("ns", tz="UTC")
        assert got.schema.field("end_time").type == pa.timestamp("ns", tz="UTC")


# ---- full size against numpy ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def events_10m():
    return nexgen.generate(10_000_000, seed=42, relations=("auction", "bid"))


def test_q9_10m_events_table_path(gpu_ctx, events_10m):
    ev = events_10m
    src = [[ev[r]] for r in plans.MORE_SOURCES["q9"]]
    got, prof = run_gpu(gpu_ctx, plans.q9(), src, profile=True)
    want = q9_numpy(pa.Table.from_batches(ev["auction"]), pa.Table.from_batches(ev["bid"]))
    assert want.num_rows > 100_000
    oracle.assert_tables_equal(got, want)
    # the outer join is one selection over the bids: the join kernels ran once, for the inner join only
    assert launches(prof, "group_match_kernel") == 1, sorted(prof)
    assert all(launches(prof, k) == 1 for k in OUTER_JOIN_KERNELS), sorted(prof)
    # ... and the whole query launches fewer kernels than the generic path: materialised (id, final) rows + hash_join
    tables = {r: gpu_ctx.import_batches(ev[r]) for r in ("auction", "bid")}
    ec = fb.ExecutionContext(gpu_ctx, plans.q9())
    ec.feed_tables([tables[r] for r in plans.MORE_SOURCES["q9"]])
    n0 = gpu_ctx.kernel_launches
    ec.execute_device(0).to_arrow()
    table_path = gpu_ctx.kernel_launches - n0
    inner = fb.ExecutionContext(gpu_ctx, plans.q9()["input"]["input"]["right"]["input"]["input"])
    inner.feed_tables([tables["auction"], tables["bid"]])
    n0 = gpu_ctx.kernel_launches
    gpu_ctx.profile_begin()
    q = inner.execute_device(0)
    assert q.num_rows > 0                # the (id, final) rows are written out: the join sees rows, not the table
    generic = gpu_ctx.hash_join(tables["bid"], q, [0, 2], [0, 1])
    generic_prof = gpu_ctx.profile_end()
    generic_out = gpu_ctx.filter_project(generic, projections=[fb.col(i) for i in range(4)], names=["auction", "bidder", "price", "b_date_time"]).to_arrow()
    generic_path = gpu_ctx.kernel_launches - n0
    assert all(launches(generic_prof, k) == 2 for k in OUTER_JOIN_KERNELS), sorted(generic_prof)
    assert table_path < generic_path, (table_path, generic_path)
    oracle.assert_tables_equal(generic_out, got)
    ec.close()
    inner.close()


def test_q12_10m_bids(gpu_ctx):
    b = nexgen.bids_ptime(10_000_000, seed=42)
    got = run_gpu(gpu_ctx, plans.q12(), [[nexgen.split_batches(b)]])
    bidder = b["bidder"].to_numpy()
    t = b["p_time"].cast(pa.int64()).to_numpy()
    keys, inv, cnt = np.unique(bidder, return_inverse=True, return_counts=True)
    lo = np.full(keys.size, np.iinfo(np.int64).max)
    hi = np.full(keys.size, np.iinfo(np.int64).min)
    np.minimum.at(lo, inv, t)
    np.maximum.at(hi, inv, t)
    assert got.schema.field("start_time").type == pa.timestamp("ns", tz="UTC") and got.schema.names == ["bidder", "bid_count", "start_time", "end_time"]
    order = np.argsort(got["bidder"].to_numpy(), kind="stable")
    assert np.array_equal(got["bidder"].to_numpy()[order], keys)
    assert np.array_equal(got["bid_count"].to_numpy()[order], cnt.astype(np.uint64))
    assert np.array_equal(got["start_time"].cast(pa.int64()).to_numpy()[order], lo)
    assert np.array_equal(got["end_time"].cast(pa.int64()).to_numpy()[order], hi)
    assert np.any(lo != hi)


def test_q13_10m_bids(gpu_ctx):
    bids = nexgen.split_batches(nexgen.bids(10_000_000, seed=42))
    n_a = nexgen.relation_counts(10_000_000 * 50 // 46)[1]
    side = nexgen.side_input(n_a, seed=42)
    got = run_gpu(gpu_ctx, plans.q13(), [[bids], [nexgen.split_batches(side)]])
    b = pa.Table.from_batches(bids)
    auc = b["auction"].to_numpy()
    keys, values = side["key"].to_numpy(), side["value"].to_numpy()
    pos = np.clip(np.searchsorted(keys, auc), 0, keys.size - 1)
    hit = keys[pos] == auc
    assert 0 < hit.sum() < auc.size
    want = b.filter(pa.array(hit)).append_column("value", pa.array(values[pos[hit]]))
    oracle.assert_tables_equal(got, want)


# ---- q9's corners, on the table path (600 K events: the inner join keeps ~385 K rows, enough for level 1 and a
# direct-address table) ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def events_600k():
    return more_events(600_000, 42)


def test_q9_ties_early_bids_and_ids_outside_the_table(gpu_ctx, events_600k):
    bids, added = q9_edge_bids(events_600k)
    src = [[events_600k["auction"]], [bids], [bids]]
    got, prof = run_gpu(gpu_ctx, plans.q9(), src, profile=True)
    assert launches(prof, "group_match_kernel") == 1, sorted(prof)
    assert_matches_oracle(got, plans.q9(), src)
    rows = set(zip(*[got[c].to_pylist() for c in ("auction", "bidder", "price")]))
    assert set(added["ties"]) <= rows and set(added["before_open"]) <= rows and not set(added["outside"]) & rows
    assert set(pa.Table.from_batches(events_600k["auction"])["a_id"].to_pylist()) - set(got["auction"].to_pylist())  # auctions nobody won


def test_q9_null_keys_on_the_probe_side(gpu_ctx, events_600k):
    outer = with_null_keys(events_600k["bid"], 11, 0.05)
    src = [[events_600k["auction"]], [outer], [events_600k["bid"]]]      # the first bid source feeds the outer join
    got, prof = run_gpu(gpu_ctx, plans.q9(), src, profile=True)
    assert launches(prof, "group_match_kernel") == 1, sorted(prof)
    assert got.num_rows > 0 and got["auction"].null_count == 0 and got["price"].null_count == 0
    # the oracle refuses NULLs: it runs over the rows that can match (an inner join drops the others), Acero over all
    assert_matches_oracle(got, plans.q9(), [[events_600k["auction"]], [without_null_keys(outer)], [events_600k["bid"]]])
    oracle.assert_tables_equal(got, acero_q9(events_600k["auction"], events_600k["bid"], outer=outer))


def test_q9_empty_bid_relations(gpu_ctx, events_600k):
    empty = [events_600k["bid"][0].slice(0, 0)]
    for src in ([[events_600k["auction"]], [empty], [events_600k["bid"]]],      # empty probe side, table path
                [[events_600k["auction"]], [empty], [empty]]):                  # no bid at all
        got = run_gpu(gpu_ctx, plans.q9(), src)
        assert got.num_rows == 0 and got.schema.names == ["auction", "bidder", "price", "b_date_time"]
        assert_matches_oracle(got, plans.q9(), src)


def test_q9_table_materialised_before_the_join(gpu_ctx, events_600k):
    tables = {r: gpu_ctx.import_batches(events_600k[r]) for r in ("auction", "bid")}
    inner_plan = plans.q9()["input"]["input"]["right"]["input"]["input"]
    inner = fb.ExecutionContext(gpu_ctx, inner_plan)
    inner.feed_tables([tables["auction"], tables["bid"]])
    q = inner.execute_device(0)
    rows = q.to_arrow()                  # another consumer writes the rows out first: the emit path's rows
    oracle.assert_tables_equal(rows, oracle.execute_plan(inner_plan, [[events_600k["auction"]], [events_600k["bid"]]]))
    gpu_ctx.profile_begin()
    joined = gpu_ctx.hash_join(tables["bid"], q, [0, 2], [0, 1]).to_arrow()
    prof = gpu_ctx.profile_end()
    assert launches(prof, "group_match_kernel") == 0 and launches(prof, "join_build_kernel") == 1, sorted(prof)
    want = q9_numpy(pa.Table.from_batches(events_600k["auction"]), pa.Table.from_batches(events_600k["bid"]))
    assert joined.schema.names == ["auction", "bidder", "price", "b_date_time", "id", "final"]
    oracle.assert_tables_equal(joined.select([0, 1, 2, 3]), want)
    assert joined["id"].equals(joined["auction"]) and joined["final"].equals(joined["price"])
    # the same join while the table is still a table: same rows, same schema and nullability
    q2 = inner.execute_device(0)
    table_joined = gpu_ctx.hash_join(tables["bid"], q2, [0, 2], [0, 1])
    assert [(f.name, f.type, f.nullable) for f in table_joined.schema] == [(f.name, f.type, f.nullable) for f in joined.schema]
    oracle.assert_tables_equal(table_joined.to_arrow(), joined, sort=False)    # both in probe-row order
    inner.close()


def test_q9_spread_ids_take_the_open_addressed_table(gpu_ctx, events_600k):
    """Auction ids 1000 apart: the level-2 table of MAX(price) is open-addressed, the join takes the generic path."""
    def spread(batches, col):
        out = []
        for b in batches:
            i = b.schema.get_field_index(col)
            out.append(b.set_column(i, b.schema.field(i), pa.array(b[col].to_numpy() * 1000, pa.int32())))
        return out
    src = [[spread(events_600k["auction"], "a_id")], [spread(events_600k["bid"], "auction")], [spread(events_600k["bid"], "auction")]]
    got, prof = run_gpu(gpu_ctx, plans.q9(), src, profile=True)
    assert launches(prof, "group_match_kernel") == 0 and launches(prof, "agg_emit_dense_kernel") == 0, sorted(prof)
    assert launches(prof, "join_build_kernel") == 2, sorted(prof)
    assert got.num_rows > 0
    assert_matches_oracle(got, plans.q9(), src)
