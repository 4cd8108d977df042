#!/usr/bin/env python
"""tools/nexmark_q9_q13_bench.py -- NEXMark q9, q10, q12 and q13 through the GPU executor, one JSON line each.

    python tools/nexmark_q9_q13_bench.py [--queries q9,q10,q12,q13] [--reps 20] [--scale 1.0]

Sizes: q9 over 10 M events (600 K auctions, 9.2 M bids), q12 and q13 over 10 M bids, q10 over one 64 Ki-row batch.
Per query: the device time of one plan execution with its relations resident in HBM and the L2 flushed before each
repetition (CUDA events on the context stream around execute + row count; median and best of --reps), events/s
(input rows / time), and the algorithmic bytes: every input column the plan scans read once plus every output
column written once.  For q9 the same call also times the generic path on the same inputs -- the (id, final) rows
written out, then hash_join on the two keys through the op-level veneer -- and checks that both outputs are equal.
The card's name and power limit are read in the same run and printed beside the figures.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import pyarrow as pa    # noqa: E402

import flock_b200 as fb                   # noqa: E402
import oracle                             # noqa: E402
from flock_b200 import nexgen, plans      # noqa: E402

BATCH = 65536


def card() -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (r.stdout.splitlines()[0].split(",") + ["?"])[:2] if r.returncode == 0 and r.stdout else ("unknown", "unknown")
    return {"gpu": name.strip(), "power_limit": power.strip()}


def inputs(q: str, scale: float, seed: int) -> dict:
    """relation name -> 64 Ki-row batches."""
    if q == "q9":
        return nexgen.generate(int(10_000_000 * scale), seed=seed, batch_rows=BATCH, relations=("auction", "bid"))
    if q == "q10":
        return {"bid": [nexgen.bids(BATCH, seed=seed)]}
    n = int(10_000_000 * scale)
    if q == "q12":
        return {"bid_ptime": nexgen.split_batches(nexgen.bids_ptime(n, seed), BATCH)}
    n_a = nexgen.relation_counts(n * 50 // 46)[1]                      # the auctions of the window those bids belong to
    return {"bid": nexgen.split_batches(nexgen.bids(n, seed=seed), BATCH),
            "side_input": nexgen.split_batches(nexgen.side_input(n_a, seed), BATCH)}


def scanned_bytes(plan: dict, tables: dict) -> int:
    """Bytes of every column the plan's leaves scan (each leaf read once)."""
    total, stack = 0, [plan]
    while stack:
        p = stack.pop()
        kids = [p[k] for k in ("input", "left", "right") if k in p]
        stack += kids
        if p.get("execution_plan") == "memory_exec":
            names = [f["name"] for f in p["schema"]["fields"]]
            want = [names[i] for i in p["projection"]]
            for t in tables.values():
                if set(want) <= set(t.schema.names):
                    total += sum(pa.Table.from_batches(t.to_batches()).column(c).nbytes for c in want)
                    break
    return total


def time_reps(ctx, fn, reps: int) -> list[float]:
    fn()                                   # warm-up: module loads, allocator, first-touch of the pools
    ms = []
    for _ in range(reps):
        ctx.synchronize()
        ctx.flush_l2()
        ctx.timer_start(0)
        fn()
        ctx.timer_stop(0)
        ms.append(ctx.timer_ms(0))
    return ms


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", default="q9,q10,q12,q13")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--seed", type=int, default=42)
    args = ap.parse_args()
    hw = card()
    with fb.Context(0) as ctx:
        for q in args.queries.split(","):
            rel = inputs(q, args.scale, args.seed)
            dev = {r: ctx.import_batches(b) for r, b in rel.items()}
            plan = plans.MORE_QUERIES[q]()
            ec = fb.ExecutionContext(ctx, plan)
            ec.feed_tables([dev[r] for r in plans.MORE_SOURCES[q]])
            result = {}

            def run():
                t = ec.execute_device(0)
                result["rows"] = t.num_rows        # waits for the row count: a deferred result is written out here
                result["table"] = t
            ms = time_reps(ctx, run, args.reps)
            out = result["table"].to_arrow()
            in_rows = sum(b.num_rows for r in dict.fromkeys(plans.MORE_SOURCES[q]) for b in rel[r])
            events = int(10_000_000 * args.scale) if q == "q9" else in_rows
            alg_bytes = scanned_bytes(plan, {r: pa.Table.from_batches(b) for r, b in rel.items()}) + out.nbytes
            line = {"query": q, **hw, "input_rows": in_rows, "events": events, "output_rows": out.num_rows, "reps": args.reps,
                    "ms_median": statistics.median(ms), "ms_best": min(ms), "events_per_s": events / (statistics.median(ms) / 1e3),
                    "algorithmic_bytes": alg_bytes, "gb_per_s_median": alg_bytes / (statistics.median(ms) / 1e3) / 1e9}
            if q == "q9":
                # the generic path on the same inputs: the aggregate's rows written out, then the two-key hash join
                inner = fb.ExecutionContext(ctx, plan["input"]["input"]["right"]["input"]["input"])
                inner.feed_tables([dev["auction"], dev["bid"]])
                gen = {}

                def run_generic():
                    t = inner.execute_device(0)
                    t.num_rows                      # (id, final) rows written out: the join sees rows, not the table
                    j = ctx.hash_join(dev["bid"], t, [0, 2], [0, 1])
                    gen["rows"] = j.num_rows
                    gen["table"] = j
                gms = time_reps(ctx, run_generic, args.reps)
                g = gen["table"].to_arrow().select([0, 1, 2, 3])
                oracle.assert_tables_equal(g, out)
                line.update({"generic_ms_median": statistics.median(gms), "generic_ms_best": min(gms),
                             "generic_events_per_s": events / (statistics.median(gms) / 1e3), "outputs_equal": True})
                inner.close()
            ec.close()
            print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
