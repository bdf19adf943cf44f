"""Speed of COVAR_POP / COVAR_SAMP / CORR plans over a resident SF-100 lineitem store, against Q1 itself.

Plans (one cached plan each, executed over the device-generated store):
  q1            TPC-H Q1
  q1_cov        Q1 with CORR(l_extendedprice, l_discount) and COVAR_SAMP(l_quantity, l_extendedprice) added
  q6_corr       Q6's filter with CORR(l_extendedprice, l_discount)
  hash_covar    GROUP BY l_shipdate (the hash table, 2526 groups) with COVAR_POP(l_extendedprice, l_discount)
  hash_sum      the same group-by with SUM(l_extendedprice), SUM(l_discount) instead: the baseline of hash_covar (same columns
                read, no K lookup)
Per plan: the kernel time of each execution (CUDA events, sd_plan_metrics aggTimeNs; best and median of --reps after one
warm-up), rows/s and algorithmic GB/s (the plan's algorithmicBytes over the kernel time), with the card's name, power limit and
SM clock read by nvidia-smi in the same run.  Writes profiles/h100_covariance.jsonl (one line per plan) and profiles/h100_covariance.md.

    python tools/covariance_bench.py [--rows 600037902] [--reps 10] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from snappydata_b200 import capi, lineitem, plan as P   # noqa: E402
from snappydata_b200.column_format import SqlType as T   # noqa: E402
from snappydata_b200.plan import PlanBuilder   # noqa: E402

ROWS_SF100 = 600_037_902


def q1_like(aggs):
    b = PlanBuilder()
    qty, price = b.col(T.DOUBLE, P.L_QUANTITY), b.col(T.DOUBLE, P.L_EXTENDEDPRICE)
    disc, tax = b.col(T.DOUBLE, P.L_DISCOUNT), b.col(T.DOUBLE, P.L_TAX)
    rf, ls, ship = b.col(T.STRING, P.L_RETURNFLAG), b.col(T.STRING, P.L_LINESTATUS), b.col(T.DATE, P.L_SHIPDATE)
    cutoff, one_a, one_b = b.lit(T.DATE), b.lit(T.DOUBLE), b.lit(T.DOUBLE)
    b.filter(ship <= cutoff)
    b.group_by(rf, ls)
    aggs(b, qty, price, disc, tax, one_a, one_b)
    return b.build()


def q1_cov(b, qty, price, disc, tax, one_a, one_b):
    dp = price * (one_a - disc)
    b.sum(qty).sum(price).sum(dp).sum(dp * (one_b + tax)).avg(qty).avg(price).avg(disc).count()
    b.corr(price, disc).covar_samp(qty, price)


def hash_plan(aggs):
    b = PlanBuilder()
    ship, price, disc = b.col(T.DATE, P.L_SHIPDATE), b.col(T.DOUBLE, P.L_EXTENDEDPRICE), b.col(T.DOUBLE, P.L_DISCOUNT)
    b.group_by(ship)
    aggs(b, price, disc)
    return b.build()


def q6_corr():
    b = PlanBuilder()
    ship, disc = b.col(T.DATE, P.L_SHIPDATE), b.col(T.DOUBLE, P.L_DISCOUNT)
    qty, price = b.col(T.DOUBLE, P.L_QUANTITY), b.col(T.DOUBLE, P.L_EXTENDEDPRICE)
    d0, d1, lo, hi, q = b.lit(T.DATE), b.lit(T.DATE), b.lit(T.DOUBLE), b.lit(T.DOUBLE), b.lit(T.DOUBLE)
    b.filter((ship >= d0) & (ship < d1) & (disc >= lo) & (disc <= hi) & (qty < q))
    b.corr(price, disc)
    return b.build()


PLANS = {"q1": (P.q1_plan, P.Q1_LITERALS), "q1_cov": (lambda: q1_like(q1_cov), P.Q1_LITERALS), "q6_corr": (q6_corr, P.Q6_LITERALS),
         "hash_covar": (lambda: hash_plan(lambda b, price, disc: b.covar_pop(price, disc).count()), []),
         "hash_sum": (lambda: hash_plan(lambda b, price, disc: b.sum(price).sum(disc).count()), [])}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    vals = [v.strip() for v in out.stdout.strip().split(",")]
    return dict(zip(q.split(","), vals)) if len(vals) == 4 else {"nvidia-smi": out.stdout.strip() or out.stderr.strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=ROWS_SF100)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles"))
    a = ap.parse_args()
    api = capi.product_api()
    api.check(api.init(0))
    store = capi.Store(api, lineitem.LINEITEM_SCHEMA)
    store.gen_lineitem(0, a.rows, 200_000, 128, 1, lineitem.Q1_COLUMN_MASK)
    lines = []
    for rnd in range(2):   # every plan twice, interleaved: the spread between rounds is part of the result
        for name, (make, lits) in PLANS.items():
            p = capi.Plan(api, make())
            arr = p.literal_array(lits)
            ms = []
            for i in range(a.reps + 1):
                p.execute_store_raw(store, arr, len(lits))
                if i:
                    ms.append(p.metrics()["aggTimeNs"] / 1e6)
            m = p.metrics()
            rec = {"plan": name, "round": rnd, "rows": a.rows, "kernel": p.kernel_name(), "kernel_ms_best": min(ms),
                   "kernel_ms_median": statistics.median(ms), "rows_per_s": m["rowsScanned"] / (min(ms) / 1e3),
                   "algo_gb_per_s": m["algorithmicBytes"] / (min(ms) / 1e3) / 1e9, "launches": m["kernelLaunches"],
                   "accumulators": sorted({r["accumulator"] for r in p.launch_log()}), **card()}
            p.close()
            print(json.dumps(rec), flush=True)
            lines.append(rec)
    store.close()
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "h100_covariance.jsonl"), "w") as f:
        for rec in lines:
            f.write(json.dumps(rec) + "\n")
    with open(os.path.join(a.out, "h100_covariance.md"), "w") as f:
        c = lines[0]
        f.write("# Covariance and correlation over a resident lineitem store\n\n")
        f.write(f"`tools/covariance_bench.py --rows {a.rows} --reps {a.reps}`: {c.get('name')}, power limit {c.get('power.limit')}, "
                f"SM clock {c.get('clocks.sm')} (max {c.get('clocks.max.sm')}) read in the same run.  Kernel time from CUDA events "
                "(sd_plan_metrics aggTimeNs), best and median of the executions after one warm-up; GB/s = the plan's algorithmic "
                "bytes over the best kernel time.  Every plan ran twice, interleaved (rounds 0 and 1).\n\n")
        f.write("| plan | round | placement | kernel ms best | median | rows/s | algorithmic GB/s |\n|---|---|---|---|---|---|---|\n")
        for r in lines:
            f.write(f"| {r['plan']} | {r['round']} | {','.join(r['accumulators'])} | {r['kernel_ms_best']:.2f} | "
                    f"{r['kernel_ms_median']:.2f} | {r['rows_per_s'] / 1e9:.2f} G | {r['algo_gb_per_s']:.0f} |\n")


if __name__ == "__main__":
    main()
