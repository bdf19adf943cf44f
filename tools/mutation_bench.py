"""UPDATE / DELETE speed over a resident lineitem store (sd_plan_update_store / sd_plan_delete_store).

For each scale factor and selectivity: a fresh device-generated store (Q1's seven columns), then
  UPDATE SET l_discount = l_discount + 0.01, l_quantity = l_quantity + 1 WHERE l_shipdate < d0 + k
  DELETE WHERE l_shipdate >= d1 AND l_shipdate < d1 + k
with k ship dates of 2526 chosen for the selectivity.  Per statement: the host clock around the synchronous call, the scan
kernels' time and algorithmic GB/s (the plan's algorithmicBytes over the scan time, against the 3.35 TB/s data sheet), the sort
and merge kernel times, the host install time (sdx_last_mutation_timing), and the Q1 kernel time over the store before and after
(the cost of the overlay path).  After each statement the store is compacted (sd_store_compact, every dirty batch): the
call's host clock, its device phases (materialise + encode, sdx_last_compaction_timing), the bytes it read and wrote, their
algorithmic GB/s over the device time, sd_store_bytes before and after, the store's compressible and total slab bytes
afterwards (sdx_store_memory_info), and the Q1 kernel time over the compacted store.
One JSON line per statement on stdout.

    python tools/mutation_bench.py --sf 10 100 --sel 0.001 0.01 0.1 [--run 2]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from snappydata_b200 import capi, lineitem, plan as P   # noqa: E402
from snappydata_b200.column_format import SqlType as T   # noqa: E402
from snappydata_b200.plan import L_DISCOUNT, L_QUANTITY, L_SHIPDATE, PlanBuilder   # noqa: E402

ROWS_SF10 = 59_986_052
ROWS_SF100 = 600_037_902


def q1_kernel_ms(api, store, reps=3):
    p = capi.Plan(api, P.q1_plan())
    lits = p.literal_array(P.Q1_LITERALS)
    best = None
    for _ in range(reps + 1):   # the first execution builds the plan's descriptors
        p.execute_store_raw(store, lits, 3)
        ms = p.metrics()["aggTimeNs"] / 1e6
        best = ms if best is None else min(best, ms)
    p.close()
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=int, nargs="+", default=[10, 100])
    ap.add_argument("--sel", type=float, nargs="+", default=[0.001, 0.01, 0.1])
    ap.add_argument("--run", type=int, default=None, help="label written into every line (repeated runs in one file)")
    a = ap.parse_args()
    api = capi.product_api()
    api.check(api.init(0))
    b = PlanBuilder()
    disc, qty, ship = b.col(T.DOUBLE, L_DISCOUNT), b.col(T.DOUBLE, L_QUANTITY), b.col(T.DATE, L_SHIPDATE)
    b.filter(ship < b.lit(T.DATE))
    b.update({L_DISCOUNT: disc + b.lit(T.DOUBLE), L_QUANTITY: qty + b.lit(T.DOUBLE)})
    up_desc = b.build()
    b = PlanBuilder()
    ship = b.col(T.DATE, L_SHIPDATE)
    b.filter((ship >= b.lit(T.DATE)) & (ship < b.lit(T.DATE)))
    b.delete()
    del_desc = b.build()
    for sf in a.sf:
        total = ROWS_SF10 if sf == 10 else ROWS_SF100 if sf == 100 else ROWS_SF10 * sf // 10
        for sel in a.sel:
            k = max(1, round(2526 * sel))
            store = capi.Store(api, lineitem.LINEITEM_SCHEMA)
            store.gen_lineitem(0, total, 200_000, 128, 6, lineitem.Q1_COLUMN_MASK)
            q1_before = q1_kernel_ms(api, store)
            for kind, desc, lits in (("update", up_desc, [8036 + k, 0.01, 1.0]), ("delete", del_desc, [9000, 9000 + k])):
                p = capi.Plan(api, desc)
                t = time.perf_counter()
                rows = p.update_store(store, lits) if kind == "update" else p.delete_store(store, lits)
                wall = (time.perf_counter() - t) * 1e3
                tm = capi.last_mutation_timing(api)
                algo = p.metrics()["algorithmicBytes"]
                p.close()
                q1_after = q1_kernel_ms(api, store)
                bytes_before = store.nbytes()
                t = time.perf_counter()
                cc = store.compact(0.0)
                c_wall = (time.perf_counter() - t) * 1e3
                ct = capi.last_compaction_timing(api)
                dev_ms = ct["materialise_ms"] + ct["encode_ms"]
                q1_compacted = q1_kernel_ms(api, store)
                print(json.dumps(({"run": a.run} if a.run is not None else {}) | {"sf": sf, "rows": total, "statement": kind, "selectivity": sel, "ship_dates": k, "rows_changed": rows,
                                  "fraction": rows / total, "statement_ms": round(wall, 3), "scan_ms": round(tm["scan_ms"], 3),
                                  "scan_algorithmic_bytes": algo, "scan_gbps": round(algo / (tm["scan_ms"] * 1e6), 1),
                                  "scan_frac_of_3350": round(algo / (tm["scan_ms"] * 1e6) / 3350.0, 3),
                                  "sort_ms": round(tm["sort_ms"], 3), "merge_ms": round(tm["merge_ms"], 3),
                                  "install_ms": round(tm["install_ms"], 3), "q1_kernel_ms_unmutated": round(q1_before, 3),
                                  "q1_kernel_ms_after": round(q1_after, 3),
                                  "compaction_ms": round(c_wall, 3), "compaction_device_ms": round(dev_ms, 3),
                                  "compaction_materialise_ms": round(ct["materialise_ms"], 3), "compaction_encode_ms": round(ct["encode_ms"], 3),
                                  "compaction_host_ms": round(ct["host_ms"], 3), "batches_rewritten": cc["batches_rewritten"],
                                  "batches_removed": cc["batches_removed"], "rows_purged": cc["rows_purged"],
                                  "compaction_bytes_read": int(ct["bytes_read"]), "compaction_bytes_written": cc["bytes_written"],
                                  "compaction_gbps": round((ct["bytes_read"] + cc["bytes_written"]) / (dev_ms * 1e6), 1) if dev_ms > 0 else None,
                                  "store_bytes_before_compaction": bytes_before, "store_bytes_after_compaction": store.nbytes(),
                                  "q1_kernel_ms_after_compaction": round(q1_compacted, 3),
                                  "store_compressible_bytes": store.memory_info()[0], "store_slab_bytes": store.memory_info()[1]}), flush=True)
            store.close()


if __name__ == "__main__":
    main()
