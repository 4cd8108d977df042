"""Writes tests/golden/nexmark_more_golden.json: expected NEXMark q9, q10, q12 and q13 outputs on the small seeded input
of nexmark_golden.json (make_golden.py).

The vectors are produced by the CPU oracle (oracle/) after it has been cross-checked, in this script, against the
independent Arrow C++ / Acero restatement of each query in tests/test_nexmark_more_host.py.
Run from the repo root:  python tests/golden/make_golden_more.py
"""
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import oracle                                # noqa: E402
from flock_b200 import plans                 # noqa: E402
from make_golden import BATCH_ROWS, N_EVENTS, SEED  # noqa: E402
from test_nexmark_more_host import acero, digest, more_events, more_sources  # noqa: E402


def main():
    ev = more_events(N_EVENTS, SEED, BATCH_ROWS)
    out = {"n_events": N_EVENTS, "seed": SEED, "batch_rows": BATCH_ROWS, "queries": {}}
    for q in plans.MORE_QUERIES:
        got = oracle.execute_plan(plans.MORE_QUERIES[q](), more_sources(q, ev))
        oracle.assert_tables_equal(got, acero(q, ev))                       # two implementations agree
        t = oracle.canonical(got)
        out["queries"][q] = {"num_rows": t.num_rows, "columns": t.schema.names,
                             "head": json.loads(json.dumps(t.slice(0, 5).to_pylist(), default=str)), "digest": digest(t)}
    path = Path(__file__).parent / "nexmark_more_golden.json"
    path.write_text(json.dumps(out, indent=1) + "\n")
    print("wrote", path, {q: v["num_rows"] for q, v in out["queries"].items()})


if __name__ == "__main__":
    main()
