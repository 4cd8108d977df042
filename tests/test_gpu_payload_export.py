"""flockgpu_table_export_payload on the GPU: a table in HBM becomes a payload's DataFrames, each body packed and
zstd-compressed on the device.  Every frame decompresses (pyarrow / libzstd) to what to_ipc gives for its row range,
pyarrow's IPC reader reads every uncompressed frame as the table's rows, every zstd body is byte for byte the host
self test's output for that uncompressed body, the import takes the frames back to the same table, and only
compressed bytes cross the link."""
import numpy as np
import pyarrow as pa
import pytest

import flock_b200 as fb
import oracle
from flock_b200 import _ffi, nexgen, plans
from conftest import sources_for

pytestmark = pytest.mark.gpu

KERNELS = ("payload_pack_kernel", "zstd_compress_kernel", "zstd_place_kernel", "zstd_gather_kernel")
MAX_BODY = 10 << 20


def _unz(data: bytes) -> bytes:
    return pa.Codec("zstd").decompress(data, decompressed_size=_content_size(data), asbytes=True)


def _content_size(frame: bytes) -> int:
    d = frame[4]
    assert (d >> 5) & 1 and not (d >> 2) & 1 and not d & 3       # Single_Segment, no checksum, no dictionary
    nb = (1, 2, 4, 8)[d >> 6]
    return int.from_bytes(frame[5:5 + nb], "little") + (256 if nb == 2 else 0)


def _read(header: bytes, body: bytes, schema: pa.Schema) -> pa.RecordBatch:
    msg = pa.ipc.read_message(pa.py_buffer(b"\xff\xff\xff\xff" + len(header).to_bytes(4, "little") + header + body))
    return pa.ipc.read_record_batch(msg, schema)


def _same(a: fb.Table, b: fb.Table) -> None:
    ta, tb = a.to_arrow(), b.to_arrow()
    assert ta.schema == tb.schema
    assert ta.equals(tb)
    for ca, cb in zip(ta.columns, tb.columns):
        assert ca.null_count == cb.null_count


@pytest.fixture(scope="module")
def bids_153():
    return nexgen.bids_chunked(10_000_000)


def test_q2_bids_153_frames(gpu_ctx, bids_153):
    t = gpu_ctx.import_batches(bids_153)
    rows = t.num_rows
    gpu_ctx.profile_begin()
    before, d2h = gpu_ctx.kernel_launches, gpu_ctx.bytes_moved()[1]
    zs = t.to_payload("zstd", 65536)
    launches_153 = gpu_ctx.kernel_launches - before
    d2h = gpu_ctx.bytes_moved()[1] - d2h
    prof = gpu_ctx.profile_end()
    assert len(zs) == 153
    for k in KERNELS:
        assert prof.get(k, {}).get("launches") == 1, prof
    # only compressed bytes crossed the link (plus one size word per frame)
    assert d2h <= sum(len(b) for _, b in zs) + 16 * len(zs) + 64, d2h
    plain = t.to_payload("none", 65536)
    assert len(plain) == 153
    table = pa.Table.from_batches(bids_153)
    for f, ((zh, zb), (h, b)) in enumerate(zip(zs, plain)):
        n = min(65536, rows - f * 65536)
        assert _unz(zh) == h and _unz(zb) == b, f
        assert (h, b) == t.to_ipc(f * 65536, n), f
        assert _read(h, b, table.schema).equals(table.slice(f * 65536, n).combine_chunks().to_batches()[0]), f
        assert zb == fb.selftest_zstd_compress(b), f                   # the GPU's bytes are the host encoder's
        assert len(zb) < len(b) // 2, f
    assert t.to_payload("zstd", 65536) == zs                           # the same bytes on every call
    one = gpu_ctx.import_batches(bids_153[:1])
    before = gpu_ctx.kernel_launches
    assert len(one.to_payload("zstd", 65536)) == 1
    assert gpu_ctx.kernel_launches - before == launches_153             # launches do not grow with the frame count
    _same(gpu_ctx.import_payload(table.schema, zs), t)


def _all_types_batch(n: int, rng) -> pa.RecordBatch:
    mask = rng.random(n) < 0.3
    strs = ["" if i % 5 == 0 else "v%d-%s" % (i, "x" * (i % 13)) for i in range(n)]
    return pa.RecordBatch.from_arrays([
        pa.array(rng.integers(-2**31, 2**31, n, dtype=np.int64).astype(np.int32)),
        pa.array(rng.integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32), mask=~mask),
        pa.array(rng.integers(-2**62, 2**62, n), mask=mask),
        pa.array(rng.integers(0, 2**63, n, dtype=np.uint64) * 2),
        pa.array(rng.standard_normal(n), mask=np.ones(n, bool)),
        pa.array(rng.integers(0, 2**40, n), pa.timestamp("ms")),
        pa.array(strs, pa.utf8(), mask=np.arange(n) % 7 == 3),
        pa.array(strs[::-1], pa.utf8()),
        pa.array([""] * n, pa.utf8()),
        pa.array([None] * n, pa.utf8()),
    ], names=["i32", "u32", "i64", "u64", "f64_all_null", "ts", "s_null", "s", "s_empty", "s_all_null"])


def _round_trip(ctx, t: fb.Table, rows_per_frame: int) -> None:
    zs = t.to_payload("zstd", rows_per_frame)
    assert len(zs) == -(-t.num_rows // rows_per_frame)
    plain = t.to_payload("none", rows_per_frame)
    table = t.to_arrow()
    for f, ((zh, zb), (h, b)) in enumerate(zip(zs, plain)):
        n = min(rows_per_frame, t.num_rows - f * rows_per_frame)
        assert _unz(zh) == h and _unz(zb) == b and zb == fb.selftest_zstd_compress(b), (rows_per_frame, f)
        assert (h, b) == t.to_ipc(f * rows_per_frame, n)
        got, want = _read(h, b, table.schema), table.slice(f * rows_per_frame, n)
        assert pa.Table.from_batches([got]).equals(want), (rows_per_frame, f)
        assert [c.null_count for c in got.columns] == [c.null_count for c in want.columns], (rows_per_frame, f)
    schema = table.schema
    back = ctx.import_payload(schema, zs)
    _same(back, t)
    _same(ctx.import_payload(schema, plain, encoding="none"), t)


def test_round_trip_every_column_type_with_nulls(gpu_ctx):
    rng = np.random.default_rng(5)
    t = gpu_ctx.import_batches([_all_types_batch(10_007, rng)])
    # validity crosses the link as bitmaps, not a byte per row: the body plus the layout read-back (24 B per column that
    # is Utf8 or has NULLs)
    laid_out = sum(1 for c in t.to_arrow().columns if c.null_count or pa.types.is_string(c.type))
    d2h = gpu_ctx.bytes_moved()[1]
    _, body = t.to_ipc()
    d2h = gpu_ctx.bytes_moved()[1] - d2h
    assert d2h <= len(body) + 24 * laid_out, (d2h, len(body))
    for rows_per_frame in (1, 7, 4096, 65536, 20_000):
        if rows_per_frame == 1:
            _round_trip(gpu_ctx, gpu_ctx.import_batches([_all_types_batch(40, rng)]), 1)
        else:
            _round_trip(gpu_ctx, t, rows_per_frame)
    _round_trip(gpu_ctx, gpu_ctx.import_batches([_all_types_batch(1, rng)]), 65536)
    empty = gpu_ctx.import_batches([_all_types_batch(0, rng)])
    assert empty.to_payload("zstd") == [] and empty.to_payload("none") == []


def test_utf8_frames_at_the_10_mib_limit(gpu_ctx):
    # 1000 rows of L bytes: body = 4008 offset bytes + 1000 * L value bytes
    under = gpu_ctx.import_batches([pa.record_batch([pa.array(["a" * 7 + "%05d" % i + "z" * 10469 for i in range(1000)])], names=["s"])])
    zs = under.to_payload("zstd", 1000)
    assert len(zs) == 1 and len(_unz(zs[0][1])) == 4008 + 1000 * 10481 <= MAX_BODY
    _same(gpu_ctx.import_payload(under.to_arrow().schema, zs), under)
    over = gpu_ctx.import_batches([pa.record_batch([pa.array(["s%d" % i for i in range(1000)] + ["b" * 10482] * 1000)], names=["s"])])
    with pytest.raises(fb.FlockGpuError) as info:
        over.to_payload("zstd", 1000)
    assert info.value.code == _ffi.ERR_INVALID and "frame 1" in info.value.message
    assert len(over.to_payload("none", 1000)) == 2                   # NONE has no such limit
    assert len(over.to_payload("zstd", 500)) == 4                    # and the context is still usable


def test_query_results_exported_and_decompressed_match_the_oracle(gpu_ctx, events_small):
    for q in ("q2", "q3", "q8"):
        tables = [gpu_ctx.import_batches(events_small[rel]) for rel in plans.SOURCES[q]]
        ec = fb.ExecutionContext(gpu_ctx, plans.QUERIES[q]())
        ec.feed_tables(tables)
        res = ec.execute_device(0)
        schema = res.to_arrow().schema
        frames = res.to_payload("zstd", 1000)
        batches = [_read(_unz(h), _unz(b), schema) for h, b in frames]
        got = pa.Table.from_batches(batches, schema=schema)
        ec.close()
        oracle.assert_tables_equal(got, oracle.execute_plan(plans.QUERIES[q](), sources_for(q, events_small)))


def test_utf8_export_profile_and_traffic(gpu_ctx, events_small):
    t = gpu_ctx.import_batches(events_small["person"])
    gpu_ctx.profile_begin()
    d2h = gpu_ctx.bytes_moved()[1]
    zs = t.to_payload("zstd", 4096)
    d2h = gpu_ctx.bytes_moved()[1] - d2h
    prof = gpu_ctx.profile_end()
    for k in KERNELS + ("payload_layout_kernel",):
        assert prof.get(k, {}).get("launches") == 1, prof
    n_cols = t.to_arrow().num_columns
    assert d2h <= sum(len(b) for _, b in zs) + (16 + 24 * n_cols) * len(zs) + 64, d2h
    _same(gpu_ctx.import_payload(t.to_arrow().schema, zs), t)


def test_errors_leave_the_context_usable(gpu_ctx):
    t = gpu_ctx.import_batches([pa.record_batch([pa.array(np.arange(100, dtype=np.int32))], names=["a"])])
    for enc, code in (("snappy", _ffi.ERR_UNSUPPORTED), ("lz4", _ffi.ERR_UNSUPPORTED), ("zlib", _ffi.ERR_UNSUPPORTED), (99, _ffi.ERR_INVALID)):
        with pytest.raises(fb.FlockGpuError) as info:
            t.to_payload(enc)
        assert info.value.code == code
        assert len(t.to_payload("zstd", 30)) == 4
    with pytest.raises(fb.FlockGpuError) as info:
        t.to_payload("zstd", 0)
    assert info.value.code == _ffi.ERR_INVALID
    frames = t.to_payload("zstd", 30)
    _same(gpu_ctx.import_payload(t.to_arrow().schema, frames), t)
