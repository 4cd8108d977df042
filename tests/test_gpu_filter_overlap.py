"""Back-to-back PredI32 filters over independent resident relations overlap: each launch may start while the one before
it drains (programmatic dependent launch).  Results must stay exact, and only launches whose inputs are older than the
previous filter's outputs may overlap: never a chained filter, nor a filter next to another kind of kernel."""
import numpy as np
import pyarrow as pa
import pytest

import flock_b200 as fb
from flock_b200 import col, nexgen, plans

pytestmark = pytest.mark.gpu

TILE_ROWS = 256 * 32
Q2 = col(0).cast("int64") % 123 == 0


def _relation(n, seed):
    return nexgen.bids(n, seed=seed, columns=["auction", "price"])


def _expect(b, modulus=123):
    au, pr = b["auction"].to_numpy(), b["price"].to_numpy()
    keep = np.fmod(au.astype(np.int64), modulus) == 0
    return au[keep], pr[keep]


def _check(got, b, modulus=123):
    au, pr = _expect(b, modulus)
    assert got.num_rows == len(au)
    t = got.to_arrow()
    assert np.array_equal(t["auction"].to_numpy(), au)
    assert np.array_equal(t["price"].to_numpy(), pr)


def test_ring_of_relations(gpu_ctx):
    """The bench loop: q2 over a ring of four resident relations, no synchronisation between the steps."""
    rels = [_relation(1_000_000 + 7919 * r, seed=100 + r) for r in range(4)]
    resident = [gpu_ctx.import_batches(nexgen.split_batches(b)) for b in rels]
    ec = fb.ExecutionContext(gpu_ctx, plans.q2())
    K = 24
    outs = []
    for i in range(K):
        ec.feed_tables([resident[i % 4]])
        outs.append(ec.execute_device(0))
        if i == 0:
            o0 = gpu_ctx.overlapped_launches
    assert gpu_ctx.overlapped_launches - o0 == K - 1
    for i, out in enumerate(outs):
        _check(out, rels[i % 4])
    ec.close()


def test_chained_filters_do_not_overlap(gpu_ctx):
    """A filter over the output of the filter just before it waits for that filter to complete."""
    b = _relation(2_000_000, seed=7)
    t = gpu_ctx.import_batches(nexgen.split_batches(b))
    first = gpu_ctx.filter_project(t, col(0).cast("int64") % 3 == 0)
    o0 = gpu_ctx.overlapped_launches
    second = gpu_ctx.filter_project(first, col(0).cast("int64") % 5 == 0)   # the same kernel instantiation
    assert gpu_ctx.overlapped_launches == o0
    au, pr = b["auction"].to_numpy(), b["price"].to_numpy()
    keep = np.fmod(au.astype(np.int64), 15) == 0
    got = second.to_arrow()
    assert np.array_equal(got["auction"].to_numpy(), au[keep])
    assert np.array_equal(got["price"].to_numpy(), pr[keep])


def test_block_reuse(gpu_ctx):
    """The input of a running filter is released at once; the next filter's outputs may take its blocks."""
    rels = [_relation(1_500_000, seed=200 + r) for r in range(6)]
    keep = gpu_ctx.import_batches(nexgen.split_batches(_relation(1_500_000, seed=199)))
    outs = []
    o0 = gpu_ctx.overlapped_launches
    for r, b in enumerate(rels):
        t = gpu_ctx.import_batches([b])   # one batch: the column is one block of the same size class as the outputs
        outs.append(gpu_ctx.filter_project(t, Q2))
        t.release()                       # dropped while its filter may still run
        outs.append(gpu_ctx.filter_project(keep, Q2))
    # each filter over `keep` follows the filter over a relation imported behind the one before: it may overlap
    assert gpu_ctx.overlapped_launches - o0 >= len(rels) - 1
    kb = _relation(1_500_000, seed=199)
    for r, b in enumerate(rels):
        _check(outs[2 * r], b)
        _check(outs[2 * r + 1], kb)


def test_mixed_neighbours_do_not_overlap(gpu_ctx):
    """A filter next to an aggregate that consumes its output, or after a sort that produces its input."""
    b = _relation(1_000_000, seed=11)
    t = gpu_ctx.import_batches(nexgen.split_batches(b))
    o0 = gpu_ctx.overlapped_launches
    f1 = gpu_ctx.filter_project(t, Q2)
    agg = gpu_ctx.hash_aggregate(f1, [0], [("count", -1, "n")], "single")
    f2 = gpu_ctx.filter_project(t, Q2)
    s = gpu_ctx.sort(t, [1])
    f3 = gpu_ctx.filter_project(s, Q2)
    assert gpu_ctx.overlapped_launches == o0
    _check(f1, b)
    _check(f2, b)
    au, pr = _expect(b)
    counts = dict(zip(*np.unique(au, return_counts=True)))
    a = agg.to_arrow()
    assert {int(k): int(v) for k, v in zip(a.column(0).to_numpy(), a.column(1).to_numpy())} == {int(k): int(v) for k, v in counts.items()}
    order = np.argsort(b["price"].to_numpy(), kind="stable")
    sa, sp = b["auction"].to_numpy()[order], b["price"].to_numpy()[order]
    k = np.fmod(sa.astype(np.int64), 123) == 0
    got = f3.to_arrow()
    assert sorted(zip(got["auction"].to_numpy(), got["price"].to_numpy())) == sorted(zip(sa[k], sp[k]))


def test_row_counts_early_and_late(gpu_ctx):
    rels = [_relation(800_000 + 1000 * r, seed=300 + r) for r in range(2)]
    resident = [gpu_ctx.import_batches(nexgen.split_batches(b)) for b in rels]
    # read immediately after each launch
    for i in range(6):
        out = gpu_ctx.filter_project(resident[i % 2], Q2)
        assert out.num_rows == len(_expect(rels[i % 2])[0])
    # read long after a run of launches that overlap
    outs = [gpu_ctx.filter_project(resident[i % 2], Q2) for i in range(8)]
    gpu_ctx.synchronize()
    for i, out in enumerate(outs):
        assert out.num_rows == len(_expect(rels[i % 2])[0])


def _boundary_sizes():
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    sizes = {1, 3, 4095, 4097, TILE_ROWS - 1, TILE_ROWS, TILE_ROWS + 1, 5 * TILE_ROWS + 17}
    for per_sm in range(1, 6):
        g = sms * per_sm * TILE_ROWS
        sizes |= {g - 1, g, g + 1, 2 * g, 2 * g + 3, int(2.5 * g) + 123}
    return sorted(sizes)


def test_overlap_at_round_boundaries(gpu_ctx):
    """Two relations of each round-boundary size alternated, several launches each, compared after the whole run."""
    rng = np.random.default_rng(9)
    for n in _boundary_sizes():
        pair = []
        for s in range(2):
            v = rng.integers(0, 1 << 20, n).astype(np.int32)
            v[rng.integers(0, n, max(n // 50, 1))] = 7 * 1001
            pair.append(pa.RecordBatch.from_arrays([pa.array(v), pa.array(np.arange(n, dtype=np.int64) + s)], names=["auction", "price"]))
        res = [gpu_ctx.import_batches([b]) for b in pair]
        o0 = gpu_ctx.overlapped_launches
        outs = [gpu_ctx.filter_project(res[i % 2], col(0).cast("int64") % 7 == 0) for i in range(6)]
        assert gpu_ctx.overlapped_launches - o0 >= 5, n
        for i, out in enumerate(outs):
            b = pair[i % 2]
            au, pr = b["auction"].to_numpy(), b["price"].to_numpy()
            keep = np.fmod(au.astype(np.int64), 7) == 0
            t = out.to_arrow()
            assert np.array_equal(t["auction"].to_numpy(), au[keep]), n
            assert np.array_equal(t["price"].to_numpy(), pr[keep]), n
