#!/usr/bin/env python
"""Debug: per-tile globaltimer stamps of filter_compact_kernel on the q2 workload (FLOCKGPU_TRACE=<file>), per round.

Round r of the cooperative mode is the band of tiles [r * grid, (r + 1) * grid).  Times are microseconds from the first
CTA start.  "wait loads" is how long a tile's verdicts came after the CTA finished its previous tile: about zero when
the tile's loads, issued one round earlier, landed while that round ranked, waited for its prefix and wrote."""
import os, sys
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
out = sys.argv[1] if len(sys.argv) > 1 else "gpurun_out/trace.txt"
os.environ["FLOCKGPU_TRACE"] = out
import numpy as np
import flock_b200 as fb
from flock_b200 import nexgen, plans
ctx = fb.Context(0)
tabs = [ctx.import_batches(nexgen.split_batches(nexgen.bids(10_000_000, seed=s))) for s in (1, 2, 3)]
ec = fb.ExecutionContext(ctx, plans.q2())
for i in range(6):
    ec.feed_tables([tabs[i % 3]])
    n = ec.execute_device(0).num_rows
rows = [l.split() for l in open(out).read().splitlines()]
ntiles, grid, rounds_mode = int(rows[0][0]), int(rows[0][1]), int(rows[0][2])
a = np.array([[int(x) for x in r] for r in rows[1:1 + ntiles]], dtype=np.int64)
t0 = a[:, 0].min()
us = lambda x: (x - t0) / 1e3
def stat(x): return f"min {x.min():7.2f}  p50 {np.median(x):7.2f}  max {x.max():7.2f}"
print("tiles", ntiles, "grid", grid, "cooperative rounds" if rounds_mode else "decoupled look-back", "rows kept", n)
rnd = np.arange(ntiles) // grid if rounds_mode else np.zeros(ntiles, dtype=np.int64)
for r in range(rnd.max() + 1):
    s = a[rnd == r]
    print(f"round {r} ({len(s)} tiles)")
    print("  start        ", stat(us(s[:, 0])))
    print("  verdicts     ", stat(us(s[:, 1])))
    print("  ranked       ", stat(us(s[:, 2])))
    print("  prefix known ", stat(us(s[:, 3])))
    print("  written      ", stat(us(s[:, 4])))
    print("  wait loads   ", stat((s[:, 1] - s[:, 0]) / 1e3))
    print("  rank->offset ", stat((s[:, 3] - s[:, 2]) / 1e3))
    print("  write phase  ", stat((s[:, 4] - s[:, 3]) / 1e3))
end = a[a[:, 5] > 0, 5]
if len(end):
    print("cta end        ", stat(us(end)))
sm = a[:, 7]
print("tiles per SM: min", np.bincount(sm).min(), "max", np.bincount(sm).max())
