"""TPC-H q7, q8 and q9 end to end at SF 1: each plan fed once (device-resident), then executed 20 times with the L2
flushed before each execution; whole-query device time (CUDA events around the execution) median / best, and the
per-kernel profile of one more execution with expr_eval_kernel's share of the kernel time.  The card's name and power
limit are read in the same run.

    python tools/tpch_query_bench.py [--scale S] [--tree DIR ...] [--rounds R]

Every --tree is a checkout whose flock_b200 package is imported in its own process; the trees are run alternately,
`--rounds` times, and one JSON line per query and run is printed."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

CHILD = r"""
import json, sys
import pyarrow as pa
sys.path.insert(0, sys.argv[1])
import flock_b200 as fb
from flock_b200 import plans, tpchgen
scale, card = float(sys.argv[2]), sys.argv[3]
T = tpchgen.generate(scale, 42)
with fb.Context(0) as ctx:
    for q, make in plans.TPCH_MORE_QUERIES.items():
        ec = fb.ExecutionContext(ctx, make())
        ec.feed_data_sources([[T[t].to_batches()] for t in plans.TPCH_MORE_SOURCES[q]])
        for _ in range(3):
            ec.execute_device().release()
        ms = []
        for _ in range(20):
            ctx.flush_l2(); ctx.synchronize()
            ctx.timer_start(0); out = ec.execute_device(); ctx.timer_stop(0)
            ms.append(ctx.timer_ms(0))
            rows = out.num_rows
            out.release()
        ctx.flush_l2(); ctx.synchronize()
        ctx.profile_begin(); ec.execute_device().release(); prof = ctx.profile_end()
        ec.clean_data_sources(); ec.close()
        ms.sort()
        kernel_ms = sum(v["ms"] for v in prof.values())
        share = prof.get("expr_eval_kernel", {}).get("ms", 0.0) / kernel_ms if kernel_ms else 0.0
        print(json.dumps({"card": card, "tree": sys.argv[1], "query": q, "scale": scale, "rows": rows, "ms_median": ms[len(ms) // 2],
                          "ms_best": ms[0], "kernel_ms": kernel_ms, "expr_eval_share": share,
                          "kernels": {k: prof[k] for k in sorted(prof, key=lambda k: -prof[k]["ms"])}}), flush=True)
"""


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--tree", action="append", default=[])
    ap.add_argument("--rounds", type=int, default=1)
    args = ap.parse_args()
    trees = args.tree or [str(Path(__file__).resolve().parent.parent)]
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    for _ in range(args.rounds):
        for tree in trees:
            r = subprocess.run([sys.executable, "-c", CHILD, tree, str(args.scale), card], capture_output=True, text=True)
            print(r.stdout.strip() or json.dumps({"card": card, "tree": tree, "error": r.stderr[-2000:]}), flush=True)


if __name__ == "__main__":
    main()
