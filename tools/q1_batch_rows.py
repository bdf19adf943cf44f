"""Q1 kernel time over freshly generated resident lineitem stores that differ only in their rows per batch.

A compaction after a DELETE leaves batches of a few rows fewer than 200,000 (the live rows of each).  This tool separates the
cost of such ragged batch sizes from everything else a compaction changes: every store is generated on the device in one go,
so its bytes sit in the same kind of slabs whatever the batch size.  One JSON line per store: the best of `--reps` Q1 kernel
times (aggTimeNs), rows, batches.

    python tools/q1_batch_rows.py --sf 100 --rows-per-batch 200000 199760 199000 180000
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from snappydata_b200 import capi, lineitem, plan as P   # noqa: E402

ROWS = {10: 59_986_052, 100: 600_037_902}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=int, default=100, choices=sorted(ROWS))
    ap.add_argument("--rows-per-batch", type=int, nargs="+", default=[200_000, 199_760, 199_000, 180_000])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--run", type=int, default=None, help="label written into every line")
    a = ap.parse_args()
    api = capi.product_api()
    api.check(api.init(0))
    total = ROWS[a.sf]
    for rpb in a.rows_per_batch:
        store = capi.Store(api, lineitem.LINEITEM_SCHEMA)
        store.gen_lineitem(0, total, rpb, 128, 6, lineitem.Q1_COLUMN_MASK)
        p = capi.Plan(api, P.q1_plan())
        lits = p.literal_array(P.Q1_LITERALS)
        best = None
        for _ in range(a.reps + 1):   # the first execution builds the plan's descriptors
            p.execute_store_raw(store, lits, len(P.Q1_LITERALS))
            ms = p.metrics()["aggTimeNs"] / 1e6
            best = ms if best is None else min(best, ms)
        line = ({"run": a.run} if a.run is not None else {}) | {"sf": a.sf, "rows": total, "rows_per_batch": rpb,
                                                                "batches": store.num_batches(), "q1_kernel_ms": round(best, 3)}
        print(json.dumps(line), flush=True)
        p.close()
        store.close()


if __name__ == "__main__":
    main()
