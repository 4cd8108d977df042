"""flockgpu_table_import_payload on the GPU: payload frames as Flock sends them (header and body each zstd-compressed,
level 3 by default) decode on the device into the same table import_ipc and import_batches give for the uncompressed
data, and queries over those tables give the oracle's results."""
import numpy as np
import pyarrow as pa
import pytest

import flock_b200 as fb
import oracle
from flock_b200 import _ffi, nexgen, plans
from conftest import sources_for

pytestmark = pytest.mark.gpu

KERNELS = ("zstd_entropy_kernel", "zstd_execute_kernel", "payload_assemble_kernel")


def _ipc(batch: pa.RecordBatch) -> tuple[bytes, bytes]:
    m = pa.ipc.read_message(batch.serialize())
    return m.metadata.to_pybytes(), m.body.to_pybytes()


def _z(data: bytes, level: int = 3) -> bytes:
    return pa.Codec("zstd", compression_level=level).compress(data, asbytes=True)


def _payload(batches, level=3):
    """(plain frames, zstd frames); `level` may be a list, one per frame."""
    plain = [_ipc(b) for b in batches]
    levels = level if isinstance(level, list) else [level] * len(plain)
    return plain, [(_z(h, L), _z(b, L)) for (h, b), L in zip(plain, levels)]


def _same(a: fb.Table, b: fb.Table) -> None:
    ta, tb = a.to_arrow(), b.to_arrow()
    assert ta.schema == tb.schema
    assert ta.equals(tb)
    for ca, cb in zip(ta.columns, tb.columns):
        assert ca.null_count == cb.null_count


def _check_all_three(ctx, schema, batches, projection=None, level=3):
    plain, packed = _payload(batches, level)
    got = ctx.import_payload(schema, packed, projection)
    _same(got, ctx.import_ipc(schema, plain, projection))
    _same(got, ctx.import_batches(batches, projection, schema=schema))
    return got


@pytest.fixture(scope="module")
def bids_153():
    return nexgen.bids_chunked(10_000_000)


def test_q2_bid_frames(gpu_ctx, bids_153):
    assert len(bids_153) == 153
    schema = bids_153[0].schema
    plain, packed = _payload(bids_153)
    gpu_ctx.profile_begin()
    before = gpu_ctx.kernel_launches
    got = gpu_ctx.import_payload(schema, packed)
    launches_153 = gpu_ctx.kernel_launches - before
    prof = gpu_ctx.profile_end()
    for k in KERNELS:
        assert prof.get(k, {}).get("launches") == 1, prof
    _same(got, gpu_ctx.import_ipc(schema, plain))
    _same(got, gpu_ctx.import_batches(bids_153))
    before = gpu_ctx.kernel_launches
    one = gpu_ctx.import_payload(schema, packed[:1])
    assert gpu_ctx.kernel_launches - before == launches_153          # launches do not grow with the frame count
    _same(one, gpu_ctx.import_batches(bids_153[:1]))
    # q2 over the decoded relation: the result of the uncompressed import
    outs = []
    for t in (got, gpu_ctx.import_batches(bids_153)):
        ec = fb.ExecutionContext(gpu_ctx, plans.q2())
        ec.feed_tables([t])
        outs.append(ec.execute_device(0).to_arrow())
        ec.close()
    assert outs[0].equals(outs[1]) and outs[0].num_rows > 0


def test_q3_person_and_auction_frames_with_projections(gpu_ctx, events_small):
    for rel in ("person", "auction"):
        batches = events_small[rel]
        schema = batches[0].schema
        _check_all_three(gpu_ctx, schema, batches)
        _check_all_three(gpu_ctx, schema, batches, projection=[0, 3, 1])
        _check_all_three(gpu_ctx, schema, batches, projection=[len(schema) - 1])


def _all_types_batch(n: int, start: int, rng) -> pa.RecordBatch:
    mask = rng.random(n) < 0.3
    strs = ["" if i % 5 == 0 else "v%d-%s" % (start + i, "x" * (i % 13)) for i in range(n)]
    return pa.RecordBatch.from_arrays([
        pa.array(rng.integers(-2**31, 2**31, n, dtype=np.int64).astype(np.int32)),
        pa.array(rng.integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32)),
        pa.array(rng.integers(-2**62, 2**62, n), mask=mask),
        pa.array(rng.integers(0, 2**63, n, dtype=np.uint64) * 2),
        pa.array(rng.standard_normal(n), mask=~mask if n % 2 else None),
        pa.array(rng.integers(0, 2**40, n), pa.timestamp("ms")),
        pa.array(strs, pa.utf8(), mask=np.arange(n) % 7 == 3),
        pa.array(strs[::-1], pa.utf8()),
    ], names=["i32", "u32", "i64", "u64", "f64", "ts", "s_null", "s"])


def test_all_column_types_nulls_at_odd_offsets_and_empty_frames(gpu_ctx):
    rng = np.random.default_rng(5)
    sizes = [1001, 0, 77, 3, 0, 4099, 1, 250]
    batches, start = [], 0
    for n in sizes:
        batches.append(_all_types_batch(n, start, rng))
        start += n
    schema = batches[0].schema
    got = _check_all_three(gpu_ctx, schema, batches)
    assert got.num_rows == sum(sizes)
    _check_all_three(gpu_ctx, schema, batches, projection=[6, 2, 7])
    # mixed levels in one call, including the fast negative levels and the slow high ones
    _check_all_three(gpu_ctx, schema, batches, level=[-5, 1, 3, 9, 19, 22, 3, -1])
    # only empty frames, and no frame at all
    empty = [b.slice(0, 0) for b in batches[:3]]
    _check_all_three(gpu_ctx, schema, empty)
    none = gpu_ctx.import_payload(schema, [])
    assert none.num_rows == 0 and none.to_arrow().schema == schema


def test_query_results_over_decoded_tables_match_the_oracle(gpu_ctx, events_small):
    for q in ("q2", "q3", "q8"):
        tables = []
        for rel in plans.SOURCES[q]:
            batches = events_small[rel]
            tables.append(gpu_ctx.import_payload(batches[0].schema, _payload(batches)[1]))
        ec = fb.ExecutionContext(gpu_ctx, plans.QUERIES[q]())
        ec.feed_tables(tables)
        got = ec.execute_device(0).to_arrow()
        ec.close()
        oracle.assert_tables_equal(got, oracle.execute_plan(plans.QUERIES[q](), sources_for(q, events_small)))


def test_round_trip_through_to_ipc(gpu_ctx):
    rng = np.random.default_rng(9)
    t = gpu_ctx.import_batches([_all_types_batch(5000, 0, rng)])
    frames = [t.to_ipc(0, 1234), t.to_ipc(1234, 0), t.to_ipc(1234)]
    back = gpu_ctx.import_payload(t.schema, [(_z(h), _z(b)) for h, b in frames])
    _same(back, t)


def test_other_encodings(gpu_ctx, events_small):
    batches = events_small["person"][:3]
    schema = batches[0].schema
    plain = [_ipc(b) for b in batches]
    _same(gpu_ctx.import_payload(schema, plain, encoding="none"), gpu_ctx.import_ipc(schema, plain))
    for enc in ("lz4", "snappy", "zlib"):
        with pytest.raises(fb.FlockGpuError) as info:
            gpu_ctx.import_payload(schema, plain, encoding=enc)
        assert info.value.code == _ffi.ERR_UNSUPPORTED


def _one_sequence_frame(of_code: int, of_bits: int, nbits: int) -> bytes:
    """A zstd frame of one compressed block, built by hand: 4 raw literals "abcd", then one sequence (ll 4, ml 4) whose
    LL / OF / ML tables are all RLE, so the bitstream holds only the offset's extra bits.  8 bytes declared."""
    content = bytes([4 << 3]) + b"abcd"                          # raw literals section, 4 bytes
    content += bytes([1, 0b01010100, 4, of_code, 1])             # 1 sequence; LL, OF, ML tables RLE: LL 4, OF code, ML code 1 (= 4)
    content += bytes([(1 << nbits) | of_bits])                   # end mark above the offset's extra bits
    header = 1 | (2 << 1) | (len(content) << 3)                  # last block, compressed
    return (0xFD2FB528).to_bytes(4, "little") + bytes([0x20, 8]) + header.to_bytes(3, "little") + content


def test_a_match_before_the_frame_start_is_an_error_from_the_device(gpu_ctx):
    header, body = _ipc(pa.record_batch([pa.array([1684234849], pa.int32())], names=["a"]))
    assert body == b"abcd" + bytes(4)
    good = _one_sequence_frame(2, 3, 2)                          # Offset_Value 4 + 3 = 7: offset 4
    bad = _one_sequence_frame(7, 0, 7)                           # Offset_Value 128: offset 125, 4 bytes produced
    assert fb.selftest_zstd_decompress(good, 64) == b"abcdabcd"
    with pytest.raises(fb.FlockGpuError) as info:
        fb.selftest_zstd_decompress(bad, 64)
    assert "offset" in info.value.message
    schema = pa.schema([pa.field("a", pa.int32())])
    with pytest.raises(fb.FlockGpuError) as info:
        gpu_ctx.import_payload(schema, [(_z(header), good), (_z(header), bad)])
    assert info.value.code == _ffi.ERR_INVALID and "frame 1" in info.value.message and "offset" in info.value.message
    t = gpu_ctx.import_payload(schema, [(_z(header), good)])   # the context is still usable
    assert t.to_arrow()["a"].to_pylist() == [int.from_bytes(b"abcd", "little")]
