"""TPC-H q1's grouped aggregate as a micro-workload: `hash_aggregate` over pre-materialised columns shaped like q1's
input after its filter (two one-byte Utf8 keys in 4 groups; four SUMs, an AVG and COUNT(*): seven accumulators unshared, six shared), device-resident,
L2 flushed before each of 20 repetitions, median / best.  The card's name and power limit are read in the same run.

    python tools/tpch_bench.py [--rows N] [--tree DIR ...]

Every --tree is a checkout whose flock_b200 package is imported in its own process (e.g. this commit and its parent);
the trees are run alternately, `--rounds` times, and one JSON line per run is printed."""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

CHILD = r"""
import json, sys
import numpy as np, pyarrow as pa
sys.path.insert(0, sys.argv[1])
import flock_b200 as fb
n = int(sys.argv[2])
rng = np.random.default_rng(42)
flag = np.array(["A", "N", "R"], dtype=object)[rng.integers(0, 3, n)]
status = np.where(flag == "N", np.array(["O", "F"], dtype=object)[rng.integers(0, 2, n)], "F").astype(object)
qty = rng.integers(1, 51, n).astype(np.float64)
price = qty * rng.integers(90000, 200000, n) / 100.0
disc = rng.integers(0, 11, n) / 100.0
tax = rng.integers(0, 9, n) / 100.0
dp = price * (1 - disc)
ch = dp * (1 + tax)
b = pa.record_batch([pa.array(flag, pa.utf8()), pa.array(status, pa.utf8()), pa.array(qty), pa.array(price), pa.array(dp), pa.array(ch),
                     pa.array(disc)], ["l_returnflag", "l_linestatus", "q", "p", "dp", "ch", "d"])
# q1's accumulators that a parent without shared accumulators also runs (at most 8): four SUMs, one AVG, COUNT(*)
aggs = [("sum", 2, "sum_qty"), ("sum", 3, "sum_base_price"), ("sum", 4, "sum_disc_price"), ("sum", 5, "sum_charge"), ("avg", 6, "avg_disc"),
        ("count", -1, "count_order")]
with fb.Context(0) as ctx:
    t = ctx.import_batches([b])
    for _ in range(3):
        ctx.hash_aggregate(t, [0, 1], aggs).release()
    ctx.profile_begin(); out = ctx.hash_aggregate(t, [0, 1], aggs); prof = ctx.profile_end()
    rows = out.to_arrow().num_rows
    ms = []
    for _ in range(20):
        ctx.flush_l2(); ctx.synchronize()
        ctx.timer_start(0); ctx.hash_aggregate(t, [0, 1], aggs).release(); ctx.timer_stop(0)
        ms.append(ctx.timer_ms(0))
ms.sort()
print(json.dumps({"tree": sys.argv[1], "rows": n, "groups": rows, "ms_median": ms[len(ms) // 2], "ms_best": ms[0],
                  "kernels": sorted(prof)}))
"""


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=6_000_000)
    ap.add_argument("--tree", action="append", default=[])
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    trees = args.tree or [str(Path(__file__).resolve().parent.parent)]
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card}))
    for _ in range(args.rounds):
        for tree in trees:
            r = subprocess.run([sys.executable, "-c", CHILD, tree, str(args.rows)], capture_output=True, text=True)
            print(r.stdout.strip() or json.dumps({"tree": tree, "error": r.stderr[-2000:]}), flush=True)


if __name__ == "__main__":
    main()
