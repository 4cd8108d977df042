"""TPC-H q4, q16, q18 and q21 end to end at SF 1 (generator data with tests/test_tpch_subquery_host.py's planted complaint
suppliers and heavy orders): each plan fed once (device-resident), then executed 20 times with the L2 flushed before
each execution; whole-query device time (CUDA events around the execution) median / best, and the per-kernel profile of
one more execution with the Semi / Anti kernels' share of the kernel time (semi_mark_kernel + semi_select_kernel; the
table build is join_build_kernel, shared with the inner join and listed apart).

q4 and q18 also run planned as DISTINCT(right keys) + inner join ("q4_inner", "q18_inner"), alternating with the Semi
plan execution by execution, so both see the same state of the card.  The card's name and power limit are read in the
same run.  One JSON line per query.

    python tools/tpch_subquery_bench.py [--scale S] [--runs R]"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--runs", type=int, default=20)
    args = ap.parse_args()
    import flock_b200 as fb
    from flock_b200 import plans, tpchgen
    from test_tpch_subquery_host import planted

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    T = planted(tpchgen.generate(args.scale, 42))
    variants = {"q4": [("q4", plans.tpch_q4), ("q4_inner", lambda: plans.tpch_q4(as_inner=True))],
                "q16": [("q16", plans.tpch_q16)],
                "q18": [("q18", plans.tpch_q18), ("q18_inner", lambda: plans.tpch_q18(as_inner=True))],
                "q21": [("q21", plans.tpch_q21)]}
    with fb.Context(0) as ctx:
        for q, runs in variants.items():
            ecs = []
            for name, make in runs:
                ec = fb.ExecutionContext(ctx, make())
                ec.feed_data_sources([[T[t].to_batches()] for t in plans.TPCH_SUBQUERY_SOURCES[q]])
                for _ in range(3):
                    ec.execute_device().release()
                ecs.append((name, ec, []))
            rows = {}
            for _ in range(args.runs):
                for name, ec, ms in ecs:
                    ctx.flush_l2(); ctx.synchronize()
                    ctx.timer_start(0); out = ec.execute_device(); ctx.timer_stop(0)
                    ms.append(ctx.timer_ms(0))
                    rows[name] = out.num_rows
                    out.release()
            for name, ec, ms in ecs:
                ctx.flush_l2(); ctx.synchronize()
                ctx.profile_begin(); ec.execute_device().release(); prof = ctx.profile_end()
                ec.clean_data_sources(); ec.close()
                ms.sort()
                kernel_ms = sum(v["ms"] for v in prof.values())
                semi_ms = sum(prof.get(k, {}).get("ms", 0.0) for k in ("semi_mark_kernel", "semi_select_kernel"))
                print(json.dumps({"card": card, "query": name, "scale": args.scale, "rows": rows[name], "ms_median": ms[len(ms) // 2],
                                  "ms_best": ms[0], "kernel_ms": kernel_ms, "semi_anti_share": semi_ms / kernel_ms if kernel_ms else 0.0,
                                  "kernels": {k: prof[k] for k in sorted(prof, key=lambda k: -prof[k]["ms"])}}), flush=True)


if __name__ == "__main__":
    main()
