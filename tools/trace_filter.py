#!/usr/bin/env python
"""Debug: per-tile globaltimer stamps of filter_compact_kernel on the q2 workload (FLOCKGPU_TRACE=<file>), per round.

The q2 steps run back to back over a ring of three relations, as in bench.py, with no synchronisation between them
(the library writes the stamps of all of them at the next synchronising call).  Round r of the cooperative mode is
the band of tiles [r * grid, (r + 1) * grid).  Times are microseconds from the first CTA start of the last launch.
"wait loads" is how long a tile's verdicts came after the CTA finished its previous tile: about zero when the tile's
loads, issued one round earlier, landed while that round ranked, waited for its prefix and wrote.  "overlap" is, for
each pair of consecutive launches, how long before launch N's last CTA end launch N + 1's first CTA started."""
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
for rep in range(2):            # the first pass loads the module and allocates; its trace is overwritten by the second
    res = []
    for i in range(6):
        ec.feed_tables([tabs[i % 3]])
        res.append(ec.execute_device(0))
    ctx.synchronize()
n = res[-1].num_rows

lines = open(out).read().splitlines()
launches = []   # (tiles, grid, rounds mode, overlapped, stamps)
i = 0
while i < len(lines):
    h = [int(x) for x in lines[i].split()]
    a = np.array([[int(x) for x in r.split()] for r in lines[i + 1:i + 1 + h[0]]], dtype=np.int64)
    launches.append((h[0], h[1], h[2], h[3], a))
    i += 1 + h[0]

print(f"{len(launches)} launches traced")
for k in range(1, len(launches)):
    prev, cur = launches[k - 1][4], launches[k][4]
    prev_end = prev[prev[:, 5] > 0, 5].max()
    lead = (prev_end - cur[:, 0].min()) / 1e3
    started = int((cur[:, 0] < prev_end).sum())
    print(f"launch {k}: {'overlapped' if launches[k][3] else 'serialised'}; first CTA start {lead:6.2f} us before launch {k - 1}'s last CTA end "
          f"({started} tiles started before it)")

ntiles, grid, rounds_mode, _, a = launches[-1]
t0 = a[:, 0].min()
us = lambda x: (x - t0) / 1e3
def stat(x): return f"min {x.min():7.2f}  p50 {np.median(x):7.2f}  max {x.max():7.2f}"
print("last launch: tiles", ntiles, "grid", grid, "cooperative rounds" if rounds_mode else "decoupled look-back", "rows kept", n)
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
