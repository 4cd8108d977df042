"""Payload encode, end to end: an HBM table -> zstd DataFrames in host memory (the mirror of tools/payload_bench.py).

    python tools/payload_export_bench.py [--steps 7] [--rows-per-frame 65536] [--out FILE]

Two workloads: q2's 10 M bids (153 frames of 65,536 rows) and 20 M persons (p_id, name), the shape of q8's shuffle.
Per step, on each workload:
  (a) gpu     Table.to_payload("zstd"): bodies packed and compressed on the device, compressed bytes copied out
  (b) cpu3    what Flock does today: to_ipc per frame, then pyarrow zstd level 3 of every header and body on all host cores
  (c) cpu1    the same at level 1
  (d) none    Table.to_payload("none"): the packed bodies, uncompressed
The legs rotate step by step; medians are reported, with the compressed bytes, the ratios, the device-to-host bytes
and the per-kernel split of (a) from the profile.  Prints the card name and its power limit: both are part of every
number."""
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
from flock_b200 import nexgen  # noqa: E402

KERNELS = ("payload_layout_kernel", "payload_pack_kernel", "zstd_compress_kernel", "zstd_place_kernel", "zstd_gather_kernel")


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as e:  # the numbers still print; the line says why the card is unknown
        return f"unknown ({e})"


def workloads() -> dict[str, list[pa.RecordBatch]]:
    persons = []
    for start in range(0, 20_000_000, 4_000_000):
        p = nexgen.persons(4_000_000, seed=42, first_person=start, columns=["p_id", "name"])
        persons.append(pa.RecordBatch.from_arrays([p["p_id"], p["name"]], names=["p_id", "name"]))
    return {"bids 10M": nexgen.bids_chunked(10_000_000), "persons 20M (p_id, name)": persons}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--rows-per-frame", type=int, default=65536)
    ap.add_argument("--threads", type=int, default=os.cpu_count())
    ap.add_argument("--out", type=str, default="")
    args = ap.parse_args()
    rpf = args.rows_per_frame
    print(f"card: {card()}; host cores: {os.cpu_count()}")
    pool = ThreadPoolExecutor(args.threads)
    codecs = {L: pa.Codec("zstd", compression_level=L) for L in (1, 3)}
    report = {"card": card(), "host_cores": os.cpu_count(), "rows_per_frame": rpf, "workloads": {}}

    with fb.Context(0) as ctx:
        for name, batches in workloads().items():
            t = ctx.import_batches(batches)
            n_frames = -(-t.num_rows // rpf)

            def cpu(level):
                frames = [t.to_ipc(f * rpf, min(rpf, t.num_rows - f * rpf)) for f in range(n_frames)]
                c = codecs[level]
                return list(pool.map(lambda hb: (c.compress(hb[0], asbytes=True), c.compress(hb[1], asbytes=True)), frames))

            legs = {"gpu": lambda: t.to_payload("zstd", rpf), "cpu3": lambda: cpu(3), "cpu1": lambda: cpu(1), "none": lambda: t.to_payload("none", rpf)}
            times = {k: [] for k in legs}
            split = {k: [] for k in KERNELS}
            d2h = {}
            sizes = {}
            order = list(legs)
            for step in range(args.steps + 1):
                for leg in order[step % len(order):] + order[:step % len(order)]:
                    if leg == "gpu":
                        ctx.profile_begin()
                    moved = ctx.bytes_moved()[1]
                    t0 = time.perf_counter()
                    frames = legs[leg]()
                    dt = time.perf_counter() - t0
                    d2h[leg] = ctx.bytes_moved()[1] - moved
                    if leg == "gpu":
                        prof = ctx.profile_end()
                    if step == 0:
                        sizes[leg] = sum(len(h) + len(b) for h, b in frames)
                        continue                                     # the first step warms up every leg
                    times[leg].append(dt * 1e3)
                    if leg == "gpu":
                        for k in KERNELS:
                            split[k].append(prof.get(k, {}).get("ms", 0.0))
                    del frames
            raw = sizes["none"]
            med = {k: statistics.median(v) for k, v in times.items()}
            kms = {k: statistics.median(v) for k, v in split.items()}
            print(f"\n{name}: {n_frames} frames, {raw / 1e6:.1f} MB uncompressed")
            for leg, label in (("gpu", "(a) to_payload(zstd)"), ("cpu3", "(b) to_ipc + CPU zstd -3"), ("cpu1", "(c) to_ipc + CPU zstd -1"),
                               ("none", "(d) to_payload(none)")):
                print(f"  {label:28s} median {med[leg]:9.2f} ms [{min(times[leg]):.2f} .. {max(times[leg]):.2f}]   "
                      f"{sizes[leg] / 1e6:8.2f} MB (ratio {raw / sizes[leg]:.2f})   D2H {d2h[leg] / 1e6:8.2f} MB")
            for k in KERNELS:
                print(f"    {k:28s} {kms[k]:8.3f} ms")
            report["workloads"][name] = {"frames": n_frames, "uncompressed_bytes": raw, "bytes": sizes, "median_ms": med, "d2h_bytes": d2h,
                                         "kernel_ms": kms}
    print(json.dumps(report))
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(report, indent=1))


if __name__ == "__main__":
    main()
