"""Writes tests/golden/ysb_golden.json: the expected YSB output on a small seeded input (100 campaigns x 10 ads,
50 000 events).

The vector is produced by the CPU oracle (oracle/) after it has been cross-checked, in this script, against the
independent Arrow C++ / Acero restatement of the query in tests/test_ysb_host.py, for the whole plan and for its three
stages run one after another.
Run from the repo root:  python tests/golden/make_golden_ysb.py
"""
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import oracle                                # noqa: E402
from flock_b200 import plans                 # noqa: E402
from test_ysb_host import COUNT, acero_ysb, digest, oracle_stages, ysb_inputs, ysb_sources  # noqa: E402

N_EVENTS, SEED, N_CAMPAIGNS, ADS, BATCH_ROWS = 50_000, 42, 100, 10, 8192


def main():
    inputs = ysb_inputs(N_EVENTS, SEED, N_CAMPAIGNS, ADS, BATCH_ROWS)
    got = oracle.execute_plan(plans.ysb(), ysb_sources(inputs))
    oracle.assert_tables_equal(got, acero_ysb(inputs["ad_event"], inputs["campaign"]))     # two implementations agree
    oracle.assert_tables_equal(oracle_stages(inputs, 8), got)                               # and the staged run
    t = oracle.canonical(got)
    out = {"n_events": N_EVENTS, "seed": SEED, "n_campaigns": N_CAMPAIGNS, "ads": ADS, "batch_rows": BATCH_ROWS,
           "num_rows": t.num_rows, "columns": t.schema.names, "views": sum(t[COUNT].to_pylist()),
           "head": json.loads(json.dumps(t.slice(0, 5).to_pylist(), default=str)), "digest": digest(t)}
    path = Path(__file__).parent / "ysb_golden.json"
    path.write_text(json.dumps(out, indent=1) + "\n")
    print("wrote", path, out["num_rows"], "rows,", out["views"], "views")


if __name__ == "__main__":
    main()
