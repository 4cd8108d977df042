"""The vectorised filter (PredI32) walks cooperative rounds of 8 Ki-row tiles: tile t runs in round t // grid, where the
grid is the kernel's resident CTAs.  Relation sizes at and around the round boundaries, checked against the oracle."""
import numpy as np
import pyarrow as pa
import pytest

import oracle
from flock_b200 import col

pytestmark = pytest.mark.gpu

TILE_ROWS = 256 * 32


def _sizes():
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    sizes = {1, 3, 4095, 4097, TILE_ROWS - 1, TILE_ROWS, TILE_ROWS + 1, 5 * TILE_ROWS + 17}
    # the grid is sms x (resident CTAs per SM), which depends on the build's register count: cover every plausible one
    for per_sm in range(1, 6):
        g = sms * per_sm * TILE_ROWS
        sizes |= {g - 1, g, g + 1, 2 * g, 2 * g + 3, int(2.5 * g) + 123}
    return sorted(sizes)


def _oracle_filter(b, pred):
    import ctypes as C
    cols = oracle.Cols(b)
    toks, _ = oracle._ctoks(pred.tokens)
    mask = np.zeros(max(b.num_rows, 1), np.uint8)
    oracle._check(oracle.lib().orc_eval_predicate(cols.arr, b.num_columns, C.c_int64(b.num_rows), toks, len(toks), mask.ctypes.data_as(C.c_void_p)), "pred")
    return b.filter(pa.array(mask[:b.num_rows].astype(bool)))


def test_filter_rounds_at_boundaries(gpu_ctx):
    sizes = _sizes()
    rng = np.random.default_rng(5)
    n_max = sizes[-1]
    v = rng.integers(0, 1 << 20, n_max).astype(np.int32)
    v[rng.integers(0, n_max, n_max // 50)] = 7 * 1001      # a hot value: long runs of survivors in some threads
    ids = np.arange(n_max, dtype=np.int64)
    for n in sizes:
        b = pa.RecordBatch.from_arrays([pa.array(v[:n]), pa.array(ids[:n])], names=["v", "i"])
        t = gpu_ctx.import_batches([b])
        for pred in (col(0).cast("int64") % 7 == 0, col(0) < 1000):
            got = gpu_ctx.filter_project(t, pred).to_batch()
            want = _oracle_filter(b, pred)
            assert got.num_rows == want.num_rows, n
            assert got.equals(want), n
        # a computed output: the kernel with the expression interpreter, which keeps fewer CTAs resident (more rounds)
        got = gpu_ctx.filter_project(t, col(0).cast("int64") % 7 == 0, [col(1) - col(0).cast("int64"), col(0)], ["d", "v"]).to_batch()
        keep = np.fmod(v[:n].astype(np.int64), 7) == 0
        assert np.array_equal(got["d"].to_numpy(), ids[:n][keep] - v[:n][keep].astype(np.int64)), n
        assert np.array_equal(got["v"].to_numpy(), v[:n][keep]), n
