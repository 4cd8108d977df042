"""Payload decode, end to end: q2's 10 M bids as 153 level-3 zstd DataFrames from pageable host memory.

    python tools/payload_bench.py [--steps 7] [--rows 10000000] [--level 3]

Per step, each followed by the q2 execute (results checked equal across the three):
  (a) gpu     Context.import_payload(zstd): compressed bodies to HBM, decoded there (per-kernel split from the profile)
  (b) cpu     what Flock does today: pyarrow zstd decompress of every frame on all host cores, then import_ipc
  (c) plain   import_ipc of frames that are already decompressed (the floor: no decode at all)
(a) and (b) alternate step by step; medians are reported.  Prints the card name and its power limit: both are part of
every number."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import pyarrow as pa  # noqa: E402

import flock_b200 as fb  # noqa: E402
from flock_b200 import nexgen, plans  # noqa: E402

KERNELS = ("zstd_entropy_kernel", "zstd_execute_kernel", "payload_assemble_kernel")


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:  # the numbers still print; the line says why the card is unknown
        return f"unknown ({e})"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--level", type=int, default=3)
    ap.add_argument("--threads", type=int, default=os.cpu_count())
    args = ap.parse_args()
    print(f"card: {card()}; host cores: {os.cpu_count()}")

    batches = nexgen.bids_chunked(args.rows)
    schema = batches[0].schema
    codec = pa.Codec("zstd", compression_level=args.level)
    plain = []
    for b in batches:
        m = pa.ipc.read_message(b.serialize())
        plain.append((m.metadata.to_pybytes(), m.body.to_pybytes()))
    packed = [(codec.compress(h, asbytes=True), codec.compress(b, asbytes=True)) for h, b in plain]
    raw_bytes = sum(len(b) for _, b in plain)
    wire_bytes = sum(len(h) + len(b) for h, b in packed)
    print(f"{len(packed)} frames: {raw_bytes / 1e6:.1f} MB decoded, {wire_bytes / 1e6:.1f} MB compressed (ratio {raw_bytes / wire_bytes:.2f})")
    pool = ThreadPoolExecutor(args.threads)

    def _dec(data: bytes) -> bytes:
        # sized by the frame's Frame_Content_Size, as the reference's zstd::block::decompress sizes its buffer
        return codec.decompress(data, decompressed_size=_content_size(data), asbytes=True)

    def cpu_decompress(frames):
        return list(pool.map(lambda hb: (_dec(hb[0]), _dec(hb[1])), frames))

    with fb.Context(0) as ctx:
        ec = fb.ExecutionContext(ctx, plans.q2())

        def run_q2(t):
            ec.feed_tables([t])
            out = ec.execute_device(0)
            ctx.synchronize()
            return out

        legs = {"gpu": [], "cpu": [], "plain": []}
        split = {k: [] for k in KERNELS}
        results = {}
        for step in range(args.steps + 1):
            for leg in ("gpu", "cpu", "plain") if step % 2 == 0 else ("cpu", "gpu", "plain"):
                if leg == "gpu":
                    ctx.profile_begin()
                t0 = time.perf_counter()
                if leg == "gpu":
                    t = ctx.import_payload(schema, packed)
                elif leg == "cpu":
                    t = ctx.import_ipc(schema, cpu_decompress(packed))
                else:
                    t = ctx.import_ipc(schema, plain)
                out = run_q2(t)
                dt = time.perf_counter() - t0
                if leg == "gpu":
                    prof = ctx.profile_end()
                if step == 0:
                    results[leg] = out.to_arrow()
                    continue                                     # the first step warms up every leg
                legs[leg].append(dt * 1e3)
                if leg == "gpu":
                    for k in KERNELS:
                        split[k].append(prof.get(k, {}).get("ms", float("nan")))
                del t, out
        ok = results["gpu"].equals(results["cpu"]) and results["gpu"].equals(results["plain"])
        ec.close()
    med = {k: statistics.median(v) for k, v in legs.items()}
    for leg, label in (("gpu", "(a) import_payload(zstd) + q2"), ("cpu", "(b) CPU zstd + import_ipc + q2"), ("plain", "(c) import_ipc(uncompressed) + q2")):
        print(f"{label:40s} median {med[leg]:8.2f} ms   [{min(legs[leg]):.2f} .. {max(legs[leg]):.2f}]")
    for k in KERNELS:
        ms = statistics.median(split[k])
        print(f"    {k:28s} {ms:8.3f} ms   {raw_bytes / (ms * 1e-3) / 1e9:8.1f} GB/s decoded")
    print(f"q2 results equal across (a), (b), (c): {ok}")
    print(json.dumps({"card": card(), "frames": len(packed), "decoded_mb": raw_bytes / 1e6, "wire_mb": wire_bytes / 1e6,
                      "median_ms": med, "kernel_ms": {k: statistics.median(v) for k, v in split.items()}, "results_equal": ok}))
    if not ok:
        sys.exit(1)


def _content_size(frame: bytes) -> int:
    d = frame[4]
    single, fcs_flag = (d >> 5) & 1, d >> 6
    at = 5 + (0 if single else 1) + (0, 1, 2, 4)[d & 3]
    n = (single, 2, 4, 8)[fcs_flag]
    if n == 0:
        raise ValueError("frame without a content size")
    v = int.from_bytes(frame[at:at + n], "little")
    return v + 256 if n == 2 else v


if __name__ == "__main__":
    main()
