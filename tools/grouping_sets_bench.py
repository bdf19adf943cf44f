"""Speed of GROUP BY ... WITH ROLLUP / WITH CUBE plans over a resident lineitem store: one scan with the plain GROUP BY's
kernel, then the roll-up kernel (sd_rollup.cu) over its groups.

Plans (one cached plan each, executed over the device-generated store):
  q1            TPC-H Q1 (GROUP BY l_returnflag, l_linestatus)
  q1_rollup     Q1 WITH ROLLUP(l_returnflag, l_linestatus): sets (rf, ls), (rf), ()
  q1_cube       Q1 WITH CUBE: the four sets
  q1_three      the three plain GROUP BY queries ROLLUP replaces, (rf, ls), (rf) and (), run back to back
  hash_cube     CUBE(l_shipdate, l_returnflag, l_linestatus) with SUM(l_quantity), SUM(l_extendedprice), COUNT(*)
  hash_plain    the same aggregates GROUP BY (l_shipdate, l_returnflag, l_linestatus)
  rollup_rate   ROLLUP(l_extendedprice, l_quantity) with COUNT(*), SUM(l_discount) over a --rate-rows store: millions of fine
                groups, for the roll-up kernel's rate in (fine group, set) pairs per second
Per execution: scan kernel ms (CUDA events, sd_plan_metrics aggTimeNs), roll-up ms (CUDA events, sdx_plan_rollup_info),
whole-call ms (host clock around sd_plan_execute_store, which ends with the rows on the host) and the rest of the call
(whole - scan - roll-up: descriptor work, read-backs, emission of the rows).  Best and median of --reps after one warm-up, every
plan twice, interleaved.  The card's name, power limit and SM clock are read by nvidia-smi in the same run.  Writes
profiles/h100_grouping_sets.jsonl and profiles/h100_grouping_sets.md.

    python tools/grouping_sets_bench.py [--rows 600037902] [--rate-rows 6001215] [--reps 5] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from snappydata_b200 import capi, lineitem, plan as P   # noqa: E402
from snappydata_b200.capi import Op, PlanDesc   # noqa: E402
from snappydata_b200.column_format import SqlType as T   # noqa: E402
from snappydata_b200.plan import PlanBuilder   # noqa: E402

ROWS_SF100, ROWS_SF1 = 600_037_902, 6_001_215


def with_sets(d: PlanDesc, masks) -> PlanDesc:
    """d's GROUP BY with the grouping sets `masks` (the set nodes appended last)"""
    first = len(d.exprs_py)
    nodes = [(Op.GROUPING_SET, int(T.INT), m, 0, 0) for m in masks] + [(Op.GROUPING_ID, int(T.INT), first, len(masks), 0)]
    return PlanDesc(d.cols_py, d.exprs_py + nodes, d.filter, d.keys_py + [first + len(masks)], d.aggs_py, d.proj_py,
                    d.literal_types_py)


def present(d: PlanDesc, mask: int) -> PlanDesc:
    """d grouped by the keys present in the set `mask` only"""
    n = len(d.keys_py)
    keys = [k for i, k in enumerate(d.keys_py) if not (mask >> (n - 1 - i)) & 1]
    return PlanDesc(d.cols_py, d.exprs_py, d.filter, keys, d.aggs_py, d.proj_py, d.literal_types_py)


def hash_plan():
    b = PlanBuilder()
    qty, price = b.col(T.DOUBLE, P.L_QUANTITY), b.col(T.DOUBLE, P.L_EXTENDEDPRICE)
    rf, ls, ship = b.col(T.STRING, P.L_RETURNFLAG), b.col(T.STRING, P.L_LINESTATUS), b.col(T.DATE, P.L_SHIPDATE)
    b.group_by(ship, rf, ls)
    b.sum(qty).sum(price).count()
    return b.build()


def rate_plan():
    b = PlanBuilder()
    qty, price, disc = b.col(T.DOUBLE, P.L_QUANTITY), b.col(T.DOUBLE, P.L_EXTENDEDPRICE), b.col(T.DOUBLE, P.L_DISCOUNT)
    b.group_by(price, qty)
    b.count().sum(disc)
    return with_sets(b.build(), [0, 1, 3])


Q1 = P.q1_plan()
PLANS = {   # name -> ([plans run back to back], literals, store)
    "q1": ([Q1], P.Q1_LITERALS, "main"),
    "q1_rollup": ([with_sets(Q1, [0, 1, 3])], P.Q1_LITERALS, "main"),
    "q1_cube": ([with_sets(Q1, [0, 1, 2, 3])], P.Q1_LITERALS, "main"),
    "q1_three": ([present(Q1, m) for m in (0, 1, 3)], P.Q1_LITERALS, "main"),
    "hash_cube": ([with_sets(hash_plan(), list(range(8)))], [], "main"),
    "hash_plain": ([hash_plan()], [], "main"),
    "rollup_rate": ([rate_plan()], [], "rate"),
}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    vals = [v.strip() for v in out.stdout.strip().split(",")]
    return dict(zip(q.split(","), vals)) if len(vals) == 4 else {"nvidia-smi": out.stdout.strip() or out.stderr.strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=ROWS_SF100)
    ap.add_argument("--rate-rows", type=int, default=ROWS_SF1)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles"))
    a = ap.parse_args()
    api = capi.product_api()
    api.check(api.init(0))
    stores = {}
    for name, rows in (("main", a.rows), ("rate", a.rate_rows)):
        s = capi.Store(api, lineitem.LINEITEM_SCHEMA)
        s.gen_lineitem(0, rows, 200_000, 128, 1, lineitem.Q1_COLUMN_MASK)
        stores[name] = (s, rows)
    lines = []
    for rnd in range(2):
        for name, (descs, lits, sname) in PLANS.items():
            store, rows = stores[sname]
            plans = [capi.Plan(api, d) for d in descs]
            arrs = [p.literal_array(lits) for p in plans]
            samples = []
            for i in range(a.reps + 1):
                scan = rollup = whole = 0.0
                out_rows = fine = coarse = launches = 0
                for p, arr in zip(plans, arrs):
                    t0 = time.perf_counter()
                    raw = p.execute_store_raw(store, arr, len(lits))
                    whole += (time.perf_counter() - t0) * 1e3
                    m, r = p.metrics(), p.rollup_info()
                    scan += m["aggTimeNs"] / 1e6
                    rollup += r["ms"]
                    out_rows += m["numOutputRows"]
                    fine, coarse, launches = fine + r["fine"], coarse + r["coarse"], launches + r["launches"]
                if i:
                    samples.append((whole, scan, rollup, out_rows, fine, coarse, launches))
            best = min(samples)
            med = lambda j: statistics.median(s[j] for s in samples)   # noqa: E731
            rec = {"plan": name, "round": rnd, "rows": rows, "kernels": [p.kernel_name() for p in plans],
                   "whole_ms_best": best[0], "whole_ms_median": med(0), "scan_ms_median": med(1), "rollup_ms_median": med(2),
                   "rest_ms_median": med(0) - med(1) - med(2), "output_rows": best[3], "fine_groups": best[4],
                   "coarse_groups": best[5], "rollup_launches": best[6],
                   "rollup_pairs_per_s": (best[4] * _nsets(descs[0]) / (med(2) / 1e3)) if med(2) > 0 else None,
                   "accumulators": sorted({r["accumulator"] for p in plans for r in p.launch_log()}), **card()}
            for p in plans:
                p.close()
            print(json.dumps(rec), flush=True)
            lines.append(rec)
    for s, _ in stores.values():
        s.close()
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "h100_grouping_sets.jsonl"), "w") as f:
        for rec in lines:
            f.write(json.dumps(rec) + "\n")
    with open(os.path.join(a.out, "h100_grouping_sets.md"), "w") as f:
        c = lines[0]
        f.write("# ROLLUP / CUBE over a resident lineitem store\n\n")
        f.write(f"`tools/grouping_sets_bench.py --rows {a.rows} --rate-rows {a.rate_rows} --reps {a.reps}`: {c.get('name')}, power limit "
                f"{c.get('power.limit')}, SM clock {c.get('clocks.sm')} (max {c.get('clocks.max.sm')}) read in the same run.  Scan and "
                "roll-up ms from CUDA events, whole-call ms from the host clock around sd_plan_execute_store (rows on the host when it "
                "returns); rest = whole - scan - roll-up (descriptors, read-backs, row emission), a difference of medians.  Medians "
                "of the executions after one warm-up (whole: best as well); every plan ran twice, interleaved.\n\n")
        f.write("| plan | round | rows | placement | scan ms | roll-up ms | rest ms | whole ms (median) | whole ms (best) | fine groups | "
                "coarse groups | roll-up (group, set) pairs/s |\n|---|---|---|---|---|---|---|---|---|---|---|---|\n")
        for r in lines:
            rate = f"{r['rollup_pairs_per_s'] / 1e6:.0f} M" if r["rollup_pairs_per_s"] else "-"
            f.write(f"| {r['plan']} | {r['round']} | {r['rows']} | {','.join(r['accumulators'])} | {r['scan_ms_median']:.2f} | "
                    f"{r['rollup_ms_median']:.3f} | {r['rest_ms_median']:.2f} | {r['whole_ms_median']:.2f} | {r['whole_ms_best']:.2f} | "
                    f"{r['fine_groups']} | {r['coarse_groups']} | {rate} |\n")


def _nsets(d: PlanDesc) -> int:
    op, _, _, count, _ = d.exprs_py[d.keys_py[-1]]
    return count if op == Op.GROUPING_ID else 0


if __name__ == "__main__":
    main()
