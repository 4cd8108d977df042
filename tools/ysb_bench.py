#!/usr/bin/env python
"""tools/ysb_bench.py -- the Yahoo Streaming Benchmark query on one GPU, one JSON line per measurement.

    python tools/ysb_bench.py [--events 10000000] [--reps 20]

Inputs: --events ad events (ad_id, event_type) in 64 Ki-row batches over 100 campaigns x 10 ads, resident in HBM.
Device time of one execution (CUDA events on the context stream around execute + row count), the L2 flushed before
each repetition, median and best of --reps:
  (a) `ysb` through ExecutionContext: the one-pass join count (dim_count_kernel);
  (b) the generic path on the same inputs, composed from the operators: filter_project -> hash_join -> hash_aggregate
      (the same rows asserted);
  (c) a dimension over D_MAX (100 x 100 ads), where the plan takes the generic path by itself;
  (d) the CPU plan interpreter (oracle/) with one thread per host core, once.
The card's name and power limit are read in the same run and printed beside the figures.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import pyarrow as pa    # noqa: E402

import flock_b200 as fb                   # noqa: E402
import oracle                             # noqa: E402
from flock_b200 import plans, ysbgen      # noqa: E402

BATCH = 65536
COUNT = plans.YSB_COUNT


def card() -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (r.stdout.splitlines()[0].split(",") + ["?"])[:2] if r.returncode == 0 and r.stdout else ("unknown", "unknown")
    return {"gpu": name.strip(), "power_limit": power.strip()}


def time_reps(ctx, fn, reps: int) -> list[float]:
    fn()                                   # warm-up
    ms = []
    for _ in range(reps):
        ctx.synchronize()
        ctx.flush_l2()
        ctx.timer_start(0)
        fn()
        ctx.timer_stop(0)
        ms.append(ctx.timer_ms(0))
    return ms


def batches(b: pa.RecordBatch) -> list:
    return [b.slice(i, BATCH) for i in range(0, b.num_rows, BATCH)]


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--events", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--seed", type=int, default=42)
    ap.add_argument("--skip-cpu", action="store_true")
    args = ap.parse_args()
    hw = card()
    camp = ysbgen.campaigns(100, 10, args.seed)
    wide = ysbgen.campaigns(100, 100, args.seed)
    ev = ysbgen.ad_events(args.events, camp, args.seed, columns=["ad_id", "event_type"])
    ev_wide = ysbgen.ad_events(args.events, wide, args.seed, columns=["ad_id", "event_type"])
    base = {**hw, "events": args.events, "reps": args.reps}
    with fb.Context(0) as ctx:
        def through_plan(events, dim, label):
            dev_e, dev_c = ctx.import_batches(batches(events)), ctx.import_batches([dim])
            ec = fb.ExecutionContext(ctx, plans.ysb())
            ec.feed_tables([dev_e, dev_c])
            res = {}

            def run():
                t = ec.execute_device(0)
                res["rows"] = t.num_rows
                res["table"] = t
            ms = time_reps(ctx, run, args.reps)
            ctx.profile_begin()
            run()
            prof = ctx.profile_end()
            out = res["table"].to_arrow()
            ec.close()
            print(json.dumps({"path": label, **base, "dimension_rows": dim.num_rows, "output_rows": out.num_rows,
                              "ms_median": statistics.median(ms), "ms_best": min(ms),
                              "events_per_s": args.events / (statistics.median(ms) / 1e3),
                              "dim_count_kernel": prof.get("dim_count_kernel", {}).get("launches", 0)}), flush=True)
            return out, dev_e, dev_c

        fused, dev_e, dev_c = through_plan(ev, camp, "(a) ysb plan, one-pass join count")

        # (b) the generic operators on the same inputs: filter, Utf8 join, gather, group-by
        res = {}

        def generic():
            views = ctx.filter_project(dev_e, fb.col(1) == fb.lit("view"))
            j = ctx.hash_join(views, dev_c, [0], [0])                  # ad_id 0, event_type 1, c_ad_id 2, campaign_id 3
            g = ctx.hash_aggregate(j, [3], [("count", -1, COUNT)])
            res["rows"] = g.num_rows
            res["table"] = g
        gms = time_reps(ctx, generic, args.reps)
        g = res["table"].to_arrow()
        oracle.assert_tables_equal(g, fused)
        print(json.dumps({"path": "(b) generic filter_project -> hash_join -> hash_aggregate", **base, "dimension_rows": camp.num_rows,
                          "output_rows": g.num_rows, "ms_median": statistics.median(gms), "ms_best": min(gms),
                          "events_per_s": args.events / (statistics.median(gms) / 1e3), "outputs_equal": True}), flush=True)

        over, _, _ = through_plan(ev_wide, wide, "(c) ysb plan, dimension over D_MAX (generic path)")

    if not args.skip_cpu:
        cores = os.cpu_count()
        t0 = time.perf_counter()
        cpu = oracle.execute_plan(plans.ysb(cores), [[batches(ev)], [[camp]]], threads=cores)
        secs = time.perf_counter() - t0
        oracle.assert_tables_equal(cpu, fused)
        print(json.dumps({"path": "(d) CPU plan interpreter", "host_cores": cores, "events": args.events, "ms": secs * 1e3,
                          "events_per_s": args.events / secs, "outputs_equal": True}), flush=True)


if __name__ == "__main__":
    main()
