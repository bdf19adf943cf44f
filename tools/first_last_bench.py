"""Speed of FIRST / LAST plans, against Q1 itself.

Plans:
  q1             TPC-H Q1 over a resident SF-100 lineitem store (device-generated)
  q1_first_last  Q1 with FIRST and LAST of l_extendedprice and of l_shipdate added (4 pairs of slots)
  drop_dups      the shape Spark plans for Dataset.dropDuplicates(l_orderkey): GROUP BY l_orderkey with FIRST of four other
                 columns (LONG, DOUBLE, INT, DATE), over an SF-10-sized resident table (60 M rows, 4 rows per order key in
                 key order as lineitem is, 15 M groups: the hash table).  The generator has no l_orderkey, so this table is
                 built on the host from a seed.
q1 and q1_first_last alternate, twice.  Per plan: the kernel time of each execution (CUDA events, sd_plan_metrics aggTimeNs;
best and median of --reps after one warm-up) and the whole call on the host clock (sd_plan_execute_store: scan, then partial-row
emission), so call - kernel is the host's share (row emission dominates at millions of groups).  The card's name, power limit and
SM clock are read by nvidia-smi in the same run.  Writes profiles/h100_first_last.jsonl and profiles/h100_first_last.md.

    python tools/first_last_bench.py [--rows 600037902] [--dd-rows 60000000] [--reps 10] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from snappydata_b200 import capi, lineitem, plan as P   # noqa: E402
from snappydata_b200.column_format import SqlType as T, build_batch   # noqa: E402
from snappydata_b200.plan import PlanBuilder   # noqa: E402

ROWS_SF100 = 600_037_902


def q1_first_last():
    b = PlanBuilder()
    qty, price = b.col(T.DOUBLE, P.L_QUANTITY), b.col(T.DOUBLE, P.L_EXTENDEDPRICE)
    disc, tax = b.col(T.DOUBLE, P.L_DISCOUNT), b.col(T.DOUBLE, P.L_TAX)
    rf, ls, ship = b.col(T.STRING, P.L_RETURNFLAG), b.col(T.STRING, P.L_LINESTATUS), b.col(T.DATE, P.L_SHIPDATE)
    cutoff, one_a, one_b = b.lit(T.DATE), b.lit(T.DOUBLE), b.lit(T.DOUBLE)
    b.filter(ship <= cutoff)
    b.group_by(rf, ls)
    dp = price * (one_a - disc)
    b.sum(qty).sum(price).sum(dp).sum(dp * (one_b + tax)).avg(qty).avg(price).avg(disc).count()
    b.first(price).last(price).first(ship).last(ship)
    return b.build()


DD_SCHEMA = [("l_orderkey", T.LONG, False), ("a", T.LONG, False), ("b", T.DOUBLE, False), ("c", T.INT, False), ("d", T.DATE, False)]


def drop_dups():
    b = PlanBuilder()
    e = [b.col(t, j, nl) for j, (_, t, nl) in enumerate(DD_SCHEMA)]
    b.group_by(e[0])
    for x in e[1:]:
        b.first(x)
    return b.build()


def dd_store(api, rows, per_batch=1_000_000, seed=10):
    st = capi.Store(api, [(t, nl) for _, t, nl in DD_SCHEMA])
    rng = np.random.default_rng(seed)
    for bi, first in enumerate(range(0, rows, per_batch)):
        n = min(per_batch, rows - first)
        data = {"l_orderkey": (np.arange(first, first + n) // 4).astype(np.int64), "a": rng.integers(-10 ** 12, 10 ** 12, n),
                "b": rng.standard_normal(n), "c": rng.integers(-2 ** 31, 2 ** 31, n).astype(np.int32),
                "d": rng.integers(8036, 8036 + 2526, n).astype(np.int32)}
        batch = build_batch(n, DD_SCHEMA, data, {}, batch_id=bi, bucket_id=bi % 8)
        st.put(batch)
    return st


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    vals = [v.strip() for v in out.stdout.strip().split(",")]
    return dict(zip(q.split(","), vals)) if len(vals) == 4 else {"nvidia-smi": out.stdout.strip() or out.stderr.strip()}


def measure(api, name, desc, store, lits, reps, rows):
    p = capi.Plan(api, desc)
    arr = p.literal_array(lits)
    ms, call = [], []
    for i in range(reps + 1):
        t = time.perf_counter()
        out = p.execute_store_raw(store, arr, len(lits))
        dt = (time.perf_counter() - t) * 1e3
        if i:
            ms.append(p.metrics()["aggTimeNs"] / 1e6)
            call.append(dt)
    m = p.metrics()
    rec = {"plan": name, "rows": rows, "kernel": p.kernel_name(), "kernel_ms_best": min(ms), "kernel_ms_median": statistics.median(ms),
           "call_ms_best": min(call), "call_ms_median": statistics.median(call), "groups": m["numOutputRows"],
           "output_bytes": len(out), "rows_per_s": m["rowsScanned"] / (min(ms) / 1e3),
           "accumulators": sorted({r["accumulator"] for r in p.launch_log()}), "launches": m["kernelLaunches"], **card()}
    p.close()
    print(json.dumps(rec), flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=ROWS_SF100)
    ap.add_argument("--dd-rows", type=int, default=60_000_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles"))
    a = ap.parse_args()
    api = capi.product_api()
    api.check(api.init(0))
    lines = []
    store = capi.Store(api, lineitem.LINEITEM_SCHEMA)
    store.gen_lineitem(0, a.rows, 200_000, 128, 1, lineitem.Q1_COLUMN_MASK)
    for rnd in range(2):   # alternated: the spread between rounds is part of the result
        for name, make in (("q1", P.q1_plan), ("q1_first_last", q1_first_last)):
            rec = measure(api, name, make(), store, P.Q1_LITERALS, a.reps, a.rows)
            rec["round"] = rnd
            lines.append(rec)
    store.close()
    st = dd_store(api, a.dd_rows)
    rec = measure(api, "drop_dups", drop_dups(), st, [], max(2, a.reps // 3), a.dd_rows)
    rec["round"] = 0
    lines.append(rec)
    st.close()
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "h100_first_last.jsonl"), "w") as f:
        for rec in lines:
            f.write(json.dumps(rec) + "\n")
    with open(os.path.join(a.out, "h100_first_last.md"), "w") as f:
        c = lines[0]
        f.write("# FIRST / LAST\n\n")
        f.write(f"`tools/first_last_bench.py --rows {a.rows} --dd-rows {a.dd_rows} --reps {a.reps}`: {c.get('name')}, power limit "
                f"{c.get('power.limit')}, SM clock {c.get('clocks.sm')} (max {c.get('clocks.max.sm')}) read in the same run.  Kernel time "
                "from CUDA events (sd_plan_metrics aggTimeNs); call time on the host clock around sd_plan_execute_store (scan + "
                "partial-row emission); best and median of the executions after one warm-up.  q1 and q1_first_last alternate, twice.\n\n")
        f.write("| plan | round | placement | groups | kernel ms best | median | call ms best | median |\n|---|---|---|---|---|---|---|---|\n")
        for r in lines:
            f.write(f"| {r['plan']} | {r['round']} | {','.join(r['accumulators'])} | {r['groups']} | {r['kernel_ms_best']:.2f} | "
                    f"{r['kernel_ms_median']:.2f} | {r['call_ms_best']:.1f} | {r['call_ms_median']:.1f} |\n")


if __name__ == "__main__":
    main()
