"""Scan images on and off, alternated in one process tree on one GPU: bench.py (Q1 value, Q1 kernel ms, Q6, C4, C5 and
parity) run --repeats times per setting, the dumped Q1 / Q6 final rows compared between settings, and the ingest cost of
the image build (gen_lineitem over SF-10 lineitem).  SD_TUNE_NO_SCAN_IMAGES=1 switches images off for both the build and
the scans.  Writes <out>/scan_images.jsonl and prints a summary.

    python tools/scan_images_bench.py --out /tmp/scan_images [--repeats 3]
"""
import argparse
import filecmp
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.check_output(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], text=True).strip().splitlines()[0]
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as e:   # (the measurement itself still runs; the record says what is missing)
        return {"error": str(e)}


def run_bench(env_off, steps, warmup, dump):
    env = dict(os.environ)
    env.pop("SD_TUNE_NO_SCAN_IMAGES", None)
    if env_off:
        env["SD_TUNE_NO_SCAN_IMAGES"] = "1"
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup), "--dump-outputs", dump]
    p = subprocess.run(cmd, env=env, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    lines = [l for l in p.stdout.splitlines() if l.startswith("{")]
    if p.returncode or not lines:
        sys.stderr.write(p.stdout[-4000:] + p.stderr[-4000:])
        raise SystemExit(f"bench.py failed ({p.returncode})")
    return json.loads(lines[-1])


def ingest_child(rows):
    """gen_lineitem timing in this process (the setting comes from the environment)."""
    import torch
    sys.path.insert(0, ROOT)
    from snappydata_b200 import capi, lineitem
    api = capi.product_api()
    api.check(api.init(0))
    torch.cuda.synchronize()
    out = []
    for _ in range(3):
        st = capi.Store(api, lineitem.LINEITEM_SCHEMA)
        t = time.perf_counter()
        st.gen_lineitem(0, rows, 1 << 20, 128, 1, lineitem.Q1_COLUMN_MASK)
        out.append((time.perf_counter() - t) * 1e3)
        info = st.image_info()
        st.close()
    print(json.dumps({"gen_ms": out, "image_info": info}))


def pick(r):
    extras = {k: r.get(k) for k in r if k.startswith("also") or k.startswith("e2e")}
    return {"q1_value": r["value"], "q1_ms_per_step": r["ms_per_step"], "q1_kernel_ms": r["roofline"]["kernel_ms_per_launch"],
            "roofline": r["roofline"], "parity": r.get("parity_check"), "clocks": r.get("clocks"),
            "extras": extras}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ingest-rows", type=int, default=59_986_052)
    ap.add_argument("--ingest-child", action="store_true")
    a = ap.parse_args()
    if a.ingest_child:
        ingest_child(a.ingest_rows)
        return
    os.makedirs(a.out, exist_ok=True)
    log = open(os.path.join(a.out, "scan_images.jsonl"), "a")
    info = gpu_info()
    log.write(json.dumps({"gpu": info}) + "\n")
    print("gpu", info, flush=True)
    for off in (True, False):   # ingest cost of the build
        env = dict(os.environ)
        env.pop("SD_TUNE_NO_SCAN_IMAGES", None)
        if off:
            env["SD_TUNE_NO_SCAN_IMAGES"] = "1"
        o = subprocess.check_output([sys.executable, os.path.abspath(__file__), "--out", a.out, "--ingest-child", "--ingest-rows",
                                     str(a.ingest_rows)], env=env, cwd=ROOT, text=True)
        rec = {"ingest": "off" if off else "on", **json.loads(o.strip().splitlines()[-1])}
        log.write(json.dumps(rec) + "\n")
        print(rec, flush=True)
    for i in range(a.repeats):
        for off in (True, False):
            tag = ("off" if off else "on") + str(i)
            dump = os.path.join(a.out, "dump_" + tag)
            r = run_bench(off, a.steps, a.warmup, dump)
            rec = {"run": tag, "images": not off, "gpu": info, **pick(r)}
            log.write(json.dumps(rec) + "\n")
            log.flush()
            print(tag, "q1 value %.4g rows/s, kernel %.3f ms, parity %s" % (rec["q1_value"], rec["q1_kernel_ms"], (rec["parity"] or {}).get("ok")), flush=True)
            if i or not off:
                ref = os.path.join(a.out, "dump_off0")
                for name in sorted(os.listdir(ref)):
                    same = filecmp.cmp(os.path.join(ref, name), os.path.join(dump, name), shallow=False)
                    print("  ", name, "identical to off0" if same else "DIFFERS from off0", flush=True)
                    log.write(json.dumps({"run": tag, "dump": name, "identical_to_off0": same}) + "\n")


if __name__ == "__main__":
    main()
