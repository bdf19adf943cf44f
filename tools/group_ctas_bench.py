"""Q1's dense group-by at one and two CTAs per SM, in one process tree on one GPU.

Diagnostics (Q1 alone, no parity): the shipped kernel, a two-stage ring, and the two diagnostic builds that show where a
tile's time goes -- SD_EXP_SKIP_ROWS (stage -> registers -> sink, no row loop) and SD_EXP_SINK_GROUPS (slots and group
computed, added into registers instead of the private table) -- each under the parent's verbatim ring layout and under the
default layout.  Then alternated pairs of full `bench.py --gpus 1 --dump-outputs` runs, SD_TUNE_RING_LAYOUT=verbatim (the
parent's layout and shape) against the default, with the dumped final rows compared; with --parent, a third leg runs the
bench.py of another built tree (the parent commit's).  Writes <out>/group_ctas.jsonl.

    python tools/group_ctas_bench.py --out /tmp/group_ctas [--pairs 3] [--no-diag] [--no-pairs] [--parent DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KNOBS = ("SD_TUNE_RING_LAYOUT", "SD_TUNE_GROUP_CTAS", "SD_TUNE_NSTAGES", "SD_JIT_DEFINES")

DIAGNOSTICS = [
    ("shipped", {}),
    ("nstages2", {"SD_TUNE_NSTAGES": "2"}),
    ("skip_rows", {"SD_JIT_DEFINES": "-DSD_EXP_SKIP_ROWS=1"}),
    ("sink_groups", {"SD_JIT_DEFINES": "-DSD_EXP_SINK_GROUPS=1"}),
]


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.check_output(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], text=True).strip().splitlines()[0]
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as e:   # (the measurement itself still runs; the record says what is missing)
        return {"error": str(e)}


def run_bench(knobs, args, root=ROOT):
    env = {k: v for k, v in os.environ.items() if k not in KNOBS}
    env.update(knobs)
    cmd = [sys.executable, os.path.join(root, "bench.py"), "--gpus", "1"] + args
    p = subprocess.run(cmd, env=env, cwd=root, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    lines = [l for l in p.stdout.splitlines() if l.startswith("{")]
    if p.returncode or not lines:
        sys.stderr.write(p.stdout[-4000:] + p.stderr[-4000:])
        raise SystemExit(f"bench.py failed ({p.returncode}) with {knobs}")
    return json.loads(lines[-1])


def q1_fields(r):
    return {"q1_value": r["value"], "q1_ms_per_step": r["ms_per_step"], "q1_kernel_ms": r["roofline"]["kernel_ms_per_launch"],
            "kernel": r["roofline"]["kernel"], "clocks": r.get("clocks")}


def compare_rows(a, b):
    """Q1 final rows of two runs: counts identical, every other column within 1e-12 relative (only the summation order differs)."""
    x, y = np.load(a), np.load(b)
    if x.shape != y.shape:
        return {"ok": False, "why": f"shapes {x.shape} vs {y.shape}"}
    rel = np.abs(x - y) / np.maximum(np.abs(x), 1e-300)
    return {"ok": bool(np.all(rel <= 1e-12)), "max_rel": float(rel.max()), "identical": bool(np.array_equal(x, y))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--pairs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-diag", action="store_true")
    ap.add_argument("--no-pairs", action="store_true")
    ap.add_argument("--layouts", default="verbatim,default", help="ring layouts the diagnostics run under")
    ap.add_argument("--parent", default=None, help="a built tree whose bench.py runs as a third leg of every pair")
    ap.add_argument("--phase", default="", help="label written into every record (what tree / build the run measured)")
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    log = open(os.path.join(a.out, "group_ctas.jsonl"), "a")

    def emit(rec):
        log.write(json.dumps({"phase": a.phase, **rec} if a.phase else rec) + "\n")
        log.flush()
    info = gpu_info()
    emit({"gpu": info})
    print("gpu", info, flush=True)
    steps = ["--steps", str(a.steps), "--warmup", str(a.warmup)]
    if not a.no_diag:
        for layout in a.layouts.split(","):
            for tag, knobs in DIAGNOSTICS:
                k = dict(knobs)
                if layout != "default":
                    k["SD_TUNE_RING_LAYOUT"] = layout
                r = run_bench(k, steps + ["--no-also", "--no-parity", "--no-e2e", "--no-cpu"])
                rec = {"diag": tag, "layout": layout, "knobs": k, "gpu": info, **q1_fields(r)}
                emit(rec)
                print("%-12s %-9s kernel %.3f ms, value %.4g rows/s" % (tag, layout, rec["q1_kernel_ms"], rec["q1_value"]), flush=True)
    if not a.no_pairs:
        for i in range(a.pairs):
            for layout in ("verbatim", "default") + (("parent",) if a.parent else ()):
                tag = f"{layout}{i}"
                dump = os.path.abspath(os.path.join(a.out, "dump_" + tag))
                r = run_bench({"SD_TUNE_RING_LAYOUT": "verbatim"} if layout == "verbatim" else {}, steps + ["--dump-outputs", dump],
                              os.path.abspath(a.parent) if layout == "parent" else ROOT)
                parity = {"q1": (r.get("parity_check") or {}).get("ok"), "q6": ((r.get("also") or {}).get("parity_check") or {}).get("ok"),
                          "c4": ((r.get("also_c4") or {}).get("parity_check") or {}).get("ok"),
                          "c5": ((r.get("also_c5") or {}).get("parity_check") or {}).get("ok")}
                rec = {"run": tag, "layout": layout, "gpu": info, **q1_fields(r), "parity_ok": parity,
                       "q6_value": (r.get("also") or {}).get("value"), "c4_value": (r.get("also_c4") or {}).get("value"),
                       "c5_value": (r.get("also_c5") or {}).get("value"), "c4_ms_per_step": (r.get("also_c4") or {}).get("ms_per_step"),
                       "c5_ms_per_step": (r.get("also_c5") or {}).get("ms_per_step"), "e2e": r.get("e2e"), "e2e_plain": r.get("e2e_plain")}
                if layout != "verbatim":
                    ref = os.path.join(a.out, f"dump_verbatim{i}")
                    rec["q1_rows_vs_verbatim"] = compare_rows(os.path.join(ref, "q1_final_rows.npy"), os.path.join(dump, "q1_final_rows.npy"))
                    rec["q6_rows_vs_verbatim"] = compare_rows(os.path.join(ref, "q6_final_rows.npy"), os.path.join(dump, "q6_final_rows.npy"))
                emit(rec)
                print("%-10s Q1 %.4g rows/s kernel %.3f ms | Q6 %.4g | C4 %.4g | C5 %.4g | parity %s %s" % (
                    tag, rec["q1_value"], rec["q1_kernel_ms"], rec["q6_value"] or 0, rec["c4_value"] or 0, rec["c5_value"] or 0, parity,
                    rec.get("q1_rows_vs_verbatim", "")), flush=True)


if __name__ == "__main__":
    main()
