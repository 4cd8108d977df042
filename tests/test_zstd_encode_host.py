"""The zstd encoder of the payload export (csrc/zstd_enc.h), on the CPU (no `gpu` mark).

flockgpu_selftest_zstd_compress runs the encoder phases the GPU kernel runs, serially on the host; the export's zstd
bodies are byte for byte what it returns for the uncompressed bodies (tests/test_gpu_payload_export.py checks that), so
what is checked here holds for the GPU's output.  Every frame must decompress to its input with pyarrow (libzstd) and
with the import's own decoder.  A frame walker checks that the corpus reaches every block type, raw and Huffman
literals, predefined and FSE-compressed sequence tables and a match reaching into an earlier block; compressed sizes
must beat libzstd's fastest level on the bodies a payload carries."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pytest

import flock_b200 as fb
from flock_b200 import _ffi, nexgen

BLOCK = 128 << 10


def _body(batch: pa.RecordBatch) -> bytes:
    return pa.ipc.read_message(batch.serialize()).body.to_pybytes()


def _libzstd(data: bytes, level: int) -> bytes:
    return pa.Codec("zstd", compression_level=level).compress(data, asbytes=True)


def _pa_decompress(frame: bytes, n: int) -> bytes:
    return pa.Codec("zstd").decompress(frame, decompressed_size=n, asbytes=True) if n else b""


def _corpus() -> dict[str, bytes]:
    rng = np.random.default_rng(21)
    c = {
        "bid": _body(nexgen.bids(30_000, seed=3)),
        "auction": _body(nexgen.auctions(6_000, seed=3)),
        "person": _body(nexgen.persons(4_000, seed=3)),
        "random": rng.bytes(200_000),
        "zeros": bytes(300_000),
        "runs": b"".join(bytes([int(b)]) * int(n) for b, n in zip(rng.integers(0, 4, 4000), rng.integers(1, 200, 4000))),
        "period1": b"q" * 70_000,
        "period3": b"abc" * 30_000 + rng.bytes(100) + b"xyz" * 10_000,
        "text": b" ".join(b"token%d" % int(v) for v in rng.zipf(1.3, 60_000) % 5000),
        "block-1": rng.bytes(BLOCK - 1),
        "block": bytes(rng.integers(0, 16, BLOCK, dtype=np.uint8)),
        "block+1": b"flock " * (BLOCK // 6) + rng.bytes(BLOCK + 1 - 6 * (BLOCK // 6)),
        # block 1 starts with the last 512 bytes of block 0 and is random otherwise: only a match into block 0 shrinks it
        "earlier_block": (lambda r: r + r[-512:] + rng.bytes(BLOCK - 512))(rng.bytes(BLOCK)),
        "multi_3M": rng.bytes(1 << 20) + _body(nexgen.bids(60_000, seed=7)) + bytes(500_000),
        "multi_10M": (_body(nexgen.persons(60_000, seed=9)) * 3)[:10 << 20],
    }
    for n in range(0, 65):
        c[f"small{n}"] = bytes(rng.integers(0, 3, n, dtype=np.uint8))
    return c


CORPUS = _corpus()
ENCODED = {name: fb.selftest_zstd_compress(data) for name, data in CORPUS.items()}


# ---- a small frame walker ----------------------------------------------------------------------------------------------------
def _walk(data: bytes) -> tuple[dict, list[dict]]:
    """(frame header fields, every block): {"block": 0 raw | 1 RLE | 2 compressed, "lit": 0..3, "streams": 1 | 4,
    "modes": (LL, OF, ML)}.  One frame, which must end exactly at the end of `data`."""
    assert int.from_bytes(data[:4], "little") == 0xFD2FB528
    d = data[4]
    single, fcs_flag = (d >> 5) & 1, d >> 6
    fcs_bytes = (single, 2, 4, 8)[fcs_flag]
    at = 5 + (0 if single else 1) + (0, 1, 2, 4)[d & 3]
    fcs = int.from_bytes(data[at:at + fcs_bytes], "little") + (256 if fcs_bytes == 2 else 0)
    at += fcs_bytes
    frame = {"single": single, "checksum": (d >> 2) & 1, "dict": d & 3, "fcs": fcs, "header": at}
    blocks = []
    while True:
        v = int.from_bytes(data[at:at + 3], "little")
        last, bt, size = v & 1, (v >> 1) & 3, v >> 3
        at += 3
        info = {"block": bt, "size": size}
        if bt == 2:
            b0 = data[at]
            lt, sf = b0 & 3, (b0 >> 2) & 3
            info["lit"] = lt
            if lt < 2:
                lh = {0: 1, 1: 2, 2: 1, 3: 3}[sf]
                comp = 0
            else:
                info["streams"] = 1 if sf == 0 else 4
                lh = 3 if sf < 2 else 4 if sf == 2 else 5
                sb = 10 if sf < 2 else 14 if sf == 2 else 18
                comp = (int.from_bytes(data[at:at + lh], "little") >> (4 + sb)) & ((1 << sb) - 1)
            if lt == 0:
                regen = b0 >> 3 if lh == 1 else (b0 >> 4) + (data[at + 1] << 4) + ((data[at + 2] << 12) if lh == 3 else 0)
                comp = regen
            elif lt == 1:
                comp = 1
            so = at + lh + comp
            if data[so]:
                modes = data[so + (1 if data[so] < 128 else 2 if data[so] < 255 else 3)]
                info["modes"] = ((modes >> 6) & 3, (modes >> 4) & 3, (modes >> 2) & 3)
        at += 1 if bt == 1 else size
        blocks.append(info)
        if last:
            break
    assert at == len(data), "trailing bytes after the frame"
    return frame, blocks


def test_every_frame_decodes_to_its_input_with_pyarrow_and_with_the_import_decoder():
    for name, data in CORPUS.items():
        z = ENCODED[name]
        assert _pa_decompress(z, len(data)) == data, name
        assert fb.selftest_zstd_decompress(z, len(data)) == data, name


def test_frame_header_and_coverage():
    seen = {"block": set(), "lit": set(), "streams": set(), "mode": set()}
    for name, data in CORPUS.items():
        frame, blocks = _walk(ENCODED[name])
        # Single_Segment with Frame_Content_Size = the input's length, no checksum, no dictionary
        assert frame["single"] == 1 and frame["fcs"] == len(data) and frame["checksum"] == 0 and frame["dict"] == 0, name
        assert len(blocks) == max(1, -(-len(data) // BLOCK)), name
        for b in blocks:
            seen["block"].add(b["block"])
            if "lit" in b:
                seen["lit"].add(b["lit"])
            if "streams" in b:
                seen["streams"].add(b["streams"])
            for m in b.get("modes", ()):
                seen["mode"].add(m)
            assert b.get("modes", (0, 0, 0))[0] != 3 and 3 not in b.get("modes", ()), name   # no Repeat_Mode
            assert b.get("lit") != 3, name                                                     # no treeless literals
    assert seen["block"] == {0, 1, 2}, seen           # raw, RLE and compressed blocks
    assert {0, 2} <= seen["lit"], seen                # raw and Huffman literals
    assert seen["streams"] == {1, 4}, seen            # 1- and 4-stream Huffman literals
    assert {0, 2} <= seen["mode"], seen               # predefined and FSE-compressed sequence tables


def test_a_match_reaches_into_an_earlier_block():
    _, blocks = _walk(ENCODED["earlier_block"])
    assert [b["block"] for b in blocks] == [0, 2]    # block 0 is random (raw); block 1 shrinks only through block 0
    _, alone = _walk(fb.selftest_zstd_compress(CORPUS["earlier_block"][BLOCK:]))
    assert [b["block"] for b in alone] == [0]


def test_incompressible_input_stays_within_the_header_plus_three_bytes_per_block():
    rng = np.random.default_rng(4)
    for n in (0, 1, 100, BLOCK - 1, BLOCK, BLOCK + 1, 3 * BLOCK + 17, 1 << 20):
        data = rng.bytes(n)
        z = fb.selftest_zstd_compress(data)
        frame, blocks = _walk(z)
        assert len(z) <= frame["header"] + len(data) + 3 * max(1, -(-n // BLOCK)), n
        assert _pa_decompress(z, n) == data


def test_the_same_input_gives_the_same_bytes():
    for name in ("bid", "text", "multi_3M"):
        assert fb.selftest_zstd_compress(CORPUS[name]) == ENCODED[name]


def _ratio_bodies() -> dict[str, bytes]:
    bids = nexgen.bids(2_000_000, seed=42)
    keep = pa.array(np.asarray(bids["auction"]) % 123 == 0)      # q2: SELECT auction, price FROM bid WHERE auction % 123 = 0
    q2 = pa.RecordBatch.from_arrays([bids["auction"].filter(keep), bids["price"].filter(keep)], names=["auction", "price"])
    persons = nexgen.persons(65_536, seed=42)
    return {
        "bid 64Ki": _body(nexgen.bids(65_536, seed=42)),
        "auction 16Ki": _body(nexgen.auctions(16_384, seed=42)),
        "person 16Ki": _body(nexgen.persons(16_384, seed=42)),
        "q2 result": _body(q2),
        "(p_id, name) 64Ki": _body(pa.RecordBatch.from_arrays([persons["p_id"], persons["name"]], names=["p_id", "name"])),
    }


def test_compressed_sizes_beat_libzstds_fastest_level_on_payload_bodies(capsys):
    lines = []
    for name, data in _ratio_bodies().items():
        z = fb.selftest_zstd_compress(data)
        assert _pa_decompress(z, len(data)) == data, name
        ref = {level: len(_libzstd(data, level)) for level in (-1, 1, 3)}
        assert len(z) <= ref[-1], (name, len(z), ref)
        lines.append(f"{name:20s} {len(data):9d} B  ratio {len(data) / len(z):.2f}  (libzstd -1 / 1 / 3: "
                     + " / ".join(f"{len(data) / ref[level]:.2f}" for level in (-1, 1, 3)) + ")")
    with capsys.disabled():
        print("\n" + "\n".join(lines))


# ---- argument checks that need no device ---------------------------------------------------------------------------------------
def _export_without_a_device(table, encoding: int, rows_per_frame: int = 1024) -> tuple[int, str]:
    out = C.c_void_p()
    rc = _ffi.lib.flockgpu_table_export_payload(None, table, encoding, rows_per_frame, C.byref(out))
    assert rc != 0 and not out.value
    return rc, _ffi.lib.flockgpu_last_error().decode()


def test_export_arguments_are_checked_before_a_device_is_involved():
    for enc in (-1, 5, 99):
        rc, msg = _export_without_a_device(None, enc)
        assert rc == _ffi.ERR_INVALID and "unknown encoding" in msg
    for enc in (fb.ENCODING_SNAPPY, fb.ENCODING_LZ4, fb.ENCODING_ZLIB):
        rc, msg = _export_without_a_device(None, enc)
        assert rc == _ffi.ERR_UNSUPPORTED and "not encoded on the GPU" in msg
    for enc in (fb.ENCODING_ZSTD, fb.ENCODING_NONE):
        rc, msg = _export_without_a_device(None, enc)
        assert rc == _ffi.ERR_INVALID and "null table" in msg
    assert _ffi.lib.flockgpu_payload_num_frames(None) == 0
    _ffi.lib.flockgpu_payload_free(None)


def test_selftest_capacity():
    with pytest.raises(fb.FlockGpuError) as info:
        z = C.create_string_buffer(4)
        n = C.c_int64()
        fb.check(_ffi.lib.flockgpu_selftest_zstd_compress(C.c_char_p(b"abcdefgh" * 100), 800, z, 4, C.byref(n)))
    assert info.value.code == _ffi.ERR_INVALID
