"""The zstd decoder of the payload import (csrc/zstd_dec.h), on the CPU (no `gpu` mark).

flockgpu_selftest_zstd_decompress runs the decoder functions the GPU kernels use, serially on the host, and must give back
pyarrow's (libzstd's) input byte for byte.  A frame walker below checks that the corpus really reaches every block type,
every literal type, 1- and 4-stream Huffman literals and all four sequence-table modes.  The payload checks that run
before a device is involved are exercised through flockgpu_table_import_payload with a NULL context."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pytest

import flock_b200 as fb
from flock_b200 import _ffi, nexgen

LEVELS = (-5, 1, 3, 9, 19, 22)


def _ipc(batch: pa.RecordBatch) -> tuple[bytes, bytes]:
    m = pa.ipc.read_message(batch.serialize())
    return m.metadata.to_pybytes(), m.body.to_pybytes()


def _compress(data: bytes, level: int = 3) -> bytes:
    return pa.Codec("zstd", compression_level=level).compress(data, asbytes=True)


def _streamed(data: bytes, pieces: int = 5) -> bytes:
    """A streaming frame: no content size, a Window_Descriptor, flushed mid-stream."""
    sink = pa.BufferOutputStream()
    s = pa.CompressedOutputStream(sink, "zstd")
    step = max(1, len(data) // pieces)
    for i in range(0, len(data), step):
        s.write(data[i:i + step])
        s.flush()
    s.close()
    return sink.getvalue().to_pybytes()


def _corpus() -> dict[str, bytes]:
    rng = np.random.default_rng(11)
    c = {
        "bid": _ipc(nexgen.bids(30_000, seed=3))[1],
        "auction": _ipc(nexgen.auctions(6_000, seed=3))[1],
        "person": _ipc(nexgen.persons(4_000, seed=3))[1],
        "random": rng.bytes(200_000),
        "zeros": bytes(300_000),
        "runs": b"".join(bytes([int(b)]) * int(n) for b, n in zip(rng.integers(0, 4, 4000), rng.integers(1, 200, 4000))),
        "period1": b"q" * 70_000,
        "period3": b"abc" * 30_000 + rng.bytes(100) + b"xyz" * 10_000,
        "text": b" ".join(b"token%d" % int(v) for v in rng.zipf(1.3, 60_000) % 5000),
        "big_mixed": rng.bytes(50_000) + bytes(100_000) + _ipc(nexgen.bids(20_000, seed=5))[1],
    }
    for n in range(0, 65):
        c[f"small{n}"] = bytes(rng.integers(0, 3, n, dtype=np.uint8))
    return c


CORPUS = _corpus()


def _decode(frame: bytes, capacity: int) -> bytes:
    return fb.selftest_zstd_decompress(frame, capacity)


# ---- a small frame walker: what the corpus covers ------------------------------------------------------------------------
def _walk(data: bytes) -> list[dict]:
    """Every block of every frame: {"block": 0 raw | 1 RLE | 2 compressed, "lit": 0..3, "streams": 1 | 4, "modes": (LL, OF, ML)}."""
    out, at = [], 0
    while at < len(data):
        magic = int.from_bytes(data[at:at + 4], "little")
        if magic & 0xFFFFFFF0 == 0x184D2A50:
            at += 8 + int.from_bytes(data[at + 4:at + 8], "little")
            continue
        assert magic == 0xFD2FB528
        d = data[at + 4]
        single = (d >> 5) & 1
        at += 5 + (0 if single else 1) + (0, 1, 2, 4)[d & 3] + (single, 2, 4, 8)[d >> 6]
        while True:
            v = int.from_bytes(data[at:at + 3], "little")
            last, bt, size = v & 1, (v >> 1) & 3, v >> 3
            at += 3
            info = {"block": bt}
            if bt == 2:
                b0 = data[at]
                lt, sf = b0 & 3, (b0 >> 2) & 3
                info["lit"] = lt
                if lt < 2:
                    lh = {0: 1, 1: 2, 2: 1, 3: 3}[sf]
                    regen = b0 >> 3 if lh == 1 else (b0 >> 4) + (data[at + 1] << 4) + ((data[at + 2] << 12) if lh == 3 else 0)
                    comp = regen if lt == 0 else 1
                else:
                    info["streams"] = 1 if sf == 0 else 4
                    lh = 3 if sf < 2 else 4 if sf == 2 else 5
                    sb = 10 if sf < 2 else 14 if sf == 2 else 18
                    comp = (int.from_bytes(data[at:at + lh], "little") >> (4 + sb)) & ((1 << sb) - 1)
                so = at + lh + comp
                if data[so]:
                    modes = data[so + (1 if data[so] < 128 else 2 if data[so] < 255 else 3)]
                    info["modes"] = ((modes >> 6) & 3, (modes >> 4) & 3, (modes >> 2) & 3)
            at += 1 if bt == 1 else size
            out.append(info)
            if last:
                break
        if (d >> 2) & 1:
            at += 4
    return out


def test_decoder_returns_pyarrows_input_and_the_corpus_covers_every_coding():
    seen = {"block": set(), "lit": set(), "streams": set(), "mode": set()}
    n_frames = 0
    for name, data in CORPUS.items():
        frames = [_compress(data, L) for L in LEVELS] + [_streamed(data)]
        for i, frame in enumerate(frames):
            got = _decode(frame, len(data))
            assert got == data, (name, LEVELS[i] if i < len(LEVELS) else "stream")
            n_frames += 1
            for b in _walk(frame):
                seen["block"].add(b["block"])
                if "lit" in b:
                    seen["lit"].add(b["lit"])
                if "streams" in b:
                    seen["streams"].add(b["streams"])
                for m in b.get("modes", ()):
                    seen["mode"].add(m)
    assert seen["block"] == {0, 1, 2}, seen                 # raw, RLE, compressed blocks
    assert seen["lit"] == {0, 1, 2, 3}, seen                # raw, RLE, Huffman, treeless literals
    assert seen["streams"] == {1, 4}, seen                  # 1- and 4-stream Huffman literals
    assert seen["mode"] == {0, 1, 2, 3}, seen               # predefined, RLE, FSE-compressed, repeat tables
    assert n_frames == len(CORPUS) * (len(LEVELS) + 1)


def test_streaming_frames_carry_no_content_size():
    frame = _streamed(CORPUS["bid"])
    d = frame[4]
    assert not (d >> 5) & 1 and d >> 6 == 0               # a Window_Descriptor, no Frame_Content_Size
    assert _decode(frame, len(CORPUS["bid"])) == CORPUS["bid"]


def _with_checksum_flag(frame: bytes) -> bytes:
    """The frame with Content_Checksum_flag set and 4 checksum bytes appended (not verified, RFC 8878 3.1.1)."""
    assert not (frame[4] >> 2) & 1
    return frame[:4] + bytes([frame[4] | 4]) + frame[5:] + b"\x12\x34\x56\x78"


def _with_dictionary_id(frame: bytes, did: int = 7) -> bytes:
    d = frame[4]
    assert d & 3 == 0
    single = (d >> 5) & 1
    cut = 5 + (0 if single else 1)
    return frame[:4] + bytes([d | 3]) + frame[5:cut] + did.to_bytes(4, "little") + frame[cut:]


def test_concatenated_skippable_and_checksummed_frames_decode():
    a, b = CORPUS["text"], CORPUS["auction"]
    skippable = (0x184D2A53).to_bytes(4, "little") + (5).to_bytes(4, "little") + b"hello"
    stream = _compress(a, 3) + skippable + _with_checksum_flag(_compress(b, 1)) + _streamed(a[:5000])
    assert _decode(stream, 10 << 20) == a + b + a[:5000]
    with pytest.raises(fb.FlockGpuError) as info:
        _decode(_with_dictionary_id(_compress(a)), 10 << 20)
    assert info.value.code == _ffi.ERR_UNSUPPORTED and "dictionary" in info.value.message


def test_output_beyond_the_capacity_is_an_error():
    data = CORPUS["period1"]
    with pytest.raises(fb.FlockGpuError) as info:
        _decode(_compress(data), len(data) - 1)
    assert info.value.code == _ffi.ERR_INVALID


SMALL = b"flock payload " * 20 + bytes(range(40)) * 3 + b"flock payload " * 5


def test_every_truncation_of_a_small_frame_is_invalid():
    frame = _compress(SMALL, 3)
    assert _decode(frame, 4096) == SMALL
    assert any(b["block"] == 2 and b.get("modes") for b in _walk(frame))
    for n in range(len(frame)):
        with pytest.raises(fb.FlockGpuError) as info:
            _decode(frame[:n], 4096)
        assert info.value.code == _ffi.ERR_INVALID, n


def test_every_flipped_byte_is_invalid_or_decodes_to_the_declared_length():
    frame = _compress(SMALL, 3)
    outcomes = {"invalid": 0, "ok": 0}
    for i in range(len(frame)):
        for mask in (0x01, 0x80, 0xFF):
            bad = bytearray(frame)
            bad[i] ^= mask
            try:
                got = _decode(bytes(bad), 4096)
            except fb.FlockGpuError as e:
                assert e.code in (_ffi.ERR_INVALID, _ffi.ERR_UNSUPPORTED), (i, mask, e)
                outcomes["invalid"] += 1
                continue
            assert len(got) == len(SMALL), (i, mask)          # a flipped literal may decode to other bytes
            outcomes["ok"] += 1
    assert outcomes["invalid"] > 0


# ---- payload checks before any device: a NULL context --------------------------------------------------------------------
def _import_payload_without_a_device(schema: pa.Schema, frames, encoding: int = fb.ENCODING_ZSTD) -> tuple[int, str]:
    keep = [(pa.py_buffer(h), pa.py_buffer(b)) for h, b in frames]
    n = len(keep)
    hp = (C.c_void_p * max(n, 1))(*[h.address for h, _ in keep])
    hl = (C.c_int64 * max(n, 1))(*[h.size for h, _ in keep])
    bp = (C.c_void_p * max(n, 1))(*[b.address for _, b in keep])
    bl = (C.c_int64 * max(n, 1))(*[b.size for _, b in keep])
    c_schema = _ffi.ArrowSchema()
    schema._export_to_c(C.addressof(c_schema))
    out = C.c_void_p()
    try:
        rc = _ffi.lib.flockgpu_table_import_payload(None, C.byref(c_schema), encoding, hp, hl, bp, bl, n, None, 0, C.byref(out))
    finally:
        if c_schema.release:
            C.CFUNCTYPE(None, C.c_void_p)(c_schema.release)(C.addressof(c_schema))
    assert rc != 0
    return rc, _ffi.lib.flockgpu_last_error().decode()


def test_payload_frames_are_validated_before_a_device_is_involved():
    b = pa.RecordBatch.from_arrays([pa.array(np.arange(3000, dtype=np.int32)), pa.array(["s%d" % (i % 17) for i in range(3000)]),
                                    pa.array(np.arange(3000, dtype=np.int64), mask=np.arange(3000) % 3 == 0)], names=["a", "s", "v"])
    header, body = _ipc(b)
    zh, zbody = _compress(header), _compress(body)
    ok = (_ffi.ERR_INVALID, "null context handle")
    assert _import_payload_without_a_device(b.schema, [(zh, zbody)]) == ok
    assert _import_payload_without_a_device(b.schema, [(zh, _streamed(body)), (zh, zbody + _compress(b""))]) == ok
    # bad magic, a reserved bit, a truncated body, a last block missing, trailing bytes
    rc, msg = _import_payload_without_a_device(b.schema, [(zh, b"\x00" + zbody[1:])])
    assert rc == _ffi.ERR_INVALID and "magic" in msg
    rc, msg = _import_payload_without_a_device(b.schema, [(zh, zbody[:4] + bytes([zbody[4] | 8]) + zbody[5:])])
    assert rc == _ffi.ERR_INVALID and "reserved" in msg
    rc, msg = _import_payload_without_a_device(b.schema, [(zh, zbody[:len(zbody) // 2])])
    assert rc == _ffi.ERR_INVALID and "truncated" in msg
    rc, msg = _import_payload_without_a_device(b.schema, [(zh, zbody + b"\x01\x02")])
    assert rc == _ffi.ERR_INVALID and "frame 0" in msg
    # a content size that differs from the header's bodyLength
    rc, msg = _import_payload_without_a_device(b.schema, [(zh, _compress(body + bytes(8)))])
    assert rc == _ffi.ERR_INVALID and "declared size" in msg
    # a Dictionary_ID
    rc, msg = _import_payload_without_a_device(b.schema, [(zh, _with_dictionary_id(zbody))])
    assert rc == _ffi.ERR_UNSUPPORTED and "dictionary" in msg
    # a header frame that does not decode, and one whose flatbuffer is wrong
    rc, msg = _import_payload_without_a_device(b.schema, [(zh[:-3], zbody)])
    assert rc == _ffi.ERR_INVALID and "header does not decode" in msg
    rc, msg = _import_payload_without_a_device(b.schema, [(_compress(b"\xff" * 64), zbody)])
    assert rc == _ffi.ERR_INVALID and "IPC header" in msg
    # the second frame is named
    rc, msg = _import_payload_without_a_device(b.schema, [(zh, zbody), (zh, zbody[:-1])])
    assert rc == _ffi.ERR_INVALID and "frame 1" in msg


def test_other_encodings():
    b = pa.RecordBatch.from_arrays([pa.array(np.arange(10, dtype=np.int32))], names=["a"])
    header, body = _ipc(b)
    for enc in (fb.ENCODING_SNAPPY, fb.ENCODING_LZ4, fb.ENCODING_ZLIB):
        rc, msg = _import_payload_without_a_device(b.schema, [(header, body)], enc)
        assert rc == _ffi.ERR_UNSUPPORTED and "not decoded on the GPU" in msg
    for enc in (-1, 5, 99):
        rc, msg = _import_payload_without_a_device(b.schema, [(header, body)], enc)
        assert rc == _ffi.ERR_INVALID and "unknown encoding" in msg
    # NONE is import_ipc: its checks pass, then the NULL context is refused
    assert _import_payload_without_a_device(b.schema, [(header, body)], fb.ENCODING_NONE) == (_ffi.ERR_INVALID, "null context handle")
