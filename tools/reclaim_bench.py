"""Device memory of a resident lineitem store under steady writes, with and without sd_store_reclaim.

For each scale factor: a fresh device-generated store (Q1's seven columns), then cycles of
  1 % UPDATE (l_discount += 0.01 over 26 of 2526 ship dates) | 1 % DELETE (26 other ship dates), alternating
  -> sd_store_compact(0) -> sd_store_reclaim(0)
and after the last cycle one sd_store_reclaim(1) that repacks every slab.  Per step: the store's slab and allocated bytes
(sdx_store_memory_info, sd_store_bytes), the reclaim's out[] and timing phases (sdx_last_reclaim_timing), its copy rate as
(read + written bytes) / copy ms, and the Q1 kernel time before the statement, after the compaction and after the reclaim.
The card's name, power limit and SM clock are read in the same run.  One JSON line per step on stdout.

    python tools/reclaim_bench.py --sf 10 100 [--cycles 6]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from snappydata_b200 import capi, lineitem, plan as P   # noqa: E402
from snappydata_b200.column_format import SqlType as T   # noqa: E402
from snappydata_b200.plan import L_DISCOUNT, L_SHIPDATE, PlanBuilder   # noqa: E402

ROWS_SF10 = 59_986_052
ROWS_SF100 = 600_037_902


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, sm, sm_max = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:   # the numbers stay usable without it
        return {"gpu": None, "card_query_error": str(e)}


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


def memory(store):
    comp, slabs = store.memory_info()
    live, kept = store.extent_bytes()
    return {"slab_bytes": slabs, "compressible_slab_bytes": comp, "store_bytes": store.nbytes(), "live_extent_bytes": live,
            "kept_retired_bytes": kept}


def reclaim_line(api, store, fraction):
    t = time.perf_counter()
    r = store.reclaim(fraction)
    wall = (time.perf_counter() - t) * 1e3
    tm = capi.last_reclaim_timing(api)
    rate = 2 * r["bytes_moved"] / (tm["copy_ms"] * 1e6) if tm["copy_ms"] > 0 else None
    return {"reclaim_fraction": fraction, "reclaim_wall_ms": round(wall, 3), **r, **{k: round(v, 3) for k, v in tm.items()},
            "copy_gbps_read_plus_write": round(rate, 1) if rate else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sf", type=int, nargs="+", default=[10, 100])
    ap.add_argument("--cycles", type=int, default=6)
    a = ap.parse_args()
    api = capi.product_api()
    api.check(api.init(0))
    hw = card()
    b = PlanBuilder()
    disc, ship = b.col(T.DOUBLE, L_DISCOUNT), b.col(T.DATE, L_SHIPDATE)
    b.filter((ship >= b.lit(T.DATE)) & (ship < b.lit(T.DATE)))
    b.update({L_DISCOUNT: disc + b.lit(T.DOUBLE)})
    up_desc = b.build()
    b = PlanBuilder()
    ship = b.col(T.DATE, L_SHIPDATE)
    b.filter((ship >= b.lit(T.DATE)) & (ship < b.lit(T.DATE)))
    b.delete()
    del_desc = b.build()
    for sf in a.sf:
        total = ROWS_SF10 if sf == 10 else ROWS_SF100 if sf == 100 else ROWS_SF10 * sf // 10
        store = capi.Store(api, lineitem.LINEITEM_SCHEMA)
        store.gen_lineitem(0, total, 200_000, 128, 6, lineitem.Q1_COLUMN_MASK)
        base = {"sf": sf, "rows": total, **hw}
        print(json.dumps(base | {"step": "fresh", "q1_kernel_ms": round(q1_kernel_ms(api, store), 3)} | memory(store)), flush=True)
        for cycle in range(a.cycles):
            kind = "update" if cycle % 2 == 0 else "delete"
            d0 = 8036 + 60 * cycle   # 26 ship dates of 2526 (~1 %), a different window every cycle
            q1_before = q1_kernel_ms(api, store)
            p = capi.Plan(api, up_desc if kind == "update" else del_desc)
            rows = p.update_store(store, [d0, d0 + 26, 0.01]) if kind == "update" else p.delete_store(store, [d0, d0 + 26])
            p.close()
            t = time.perf_counter()
            cc = store.compact(0.0)
            c_wall = (time.perf_counter() - t) * 1e3
            after_compaction = memory(store)
            q1_compacted = q1_kernel_ms(api, store)
            line = base | {"step": "cycle", "cycle": cycle, "statement": kind, "rows_changed": rows, "q1_kernel_ms_before": round(q1_before, 3),
                           "compaction_ms": round(c_wall, 3), "compaction_bytes_written": cc["bytes_written"],
                           "after_compaction": after_compaction, "q1_kernel_ms_after_compaction": round(q1_compacted, 3)}
            line |= reclaim_line(api, store, 0.0)
            line |= {"after_reclaim": memory(store), "q1_kernel_ms_after_reclaim": round(q1_kernel_ms(api, store), 3)}
            print(json.dumps(line), flush=True)
        line = base | {"step": "repack"} | reclaim_line(api, store, 1.0)
        line |= {"after_reclaim": memory(store), "q1_kernel_ms_after_reclaim": round(q1_kernel_ms(api, store), 3)}
        print(json.dumps(line), flush=True)
        store.close()


if __name__ == "__main__":
    main()
