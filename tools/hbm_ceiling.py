"""Measured HBM read ceiling for the Q1 scan's bytes (tools/hbm_ceiling.cu): compiles the probe into a temporary
directory, runs each variant in its own process and samples the SM clock with a read-only `nvidia-smi --query-gpu` loop
beside it (the same query bench.py's ClockSampler makes).  Prints one JSON line per variant and a header line with the
card's name, power limit and maximum clocks.

    python tools/hbm_ceiling.py [--out FILE] [--reps N] [--allocs plain,compressible] [--fills const,random,q1,q1:shipdate,...]

With --allocs or --fills it runs R1 and R2 (4 CTAs/SM) and R3 (3 stages) for every allocation x fill combination instead of the
grid and stage sweep below: whether generic memory compression lowers the DRAM bytes behind the scan's reads.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

# (variant, options): the contiguous read at two grid sizes, the column layout at three, the scan's ring at the stage
# count the Q1 kernel gets today (3) and at the counts more shared memory would allow
RUNS = [("r1", ["--ctas-per-sm", "2"]), ("r1", ["--ctas-per-sm", "4"]),
        ("r2", ["--ctas-per-sm", "2"]), ("r2", ["--ctas-per-sm", "4"]), ("r2", ["--ctas-per-sm", "8"]),
        ("r3", ["--stages", "2"]), ("r3", ["--stages", "3"]), ("r3", ["--stages", "4"]), ("r3", ["--stages", "5"]),
        ("r3lds", ["--stages", "3"]), ("r3lds", ["--stages", "5"])]
COMPRESSION_RUNS = [("r1", ["--ctas-per-sm", "4"]), ("r2", ["--ctas-per-sm", "4"]), ("r3", ["--stages", "3"])]

CLOCK_Q = "clocks.sm,clocks.mem,power.draw,clocks_event_reasons.sw_power_cap"


def smi(query):
    out = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={query}", "--format=csv,noheader,nounits"],
                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, check=True).stdout
    return [x.strip() for x in out.strip().split(",")]


class Sampler:
    def __init__(self):
        self.f = tempfile.NamedTemporaryFile("w+", suffix=".csv", delete=False)
        self.p = subprocess.Popen(["nvidia-smi", "--id=0", f"--query-gpu={CLOCK_Q}", "--format=csv,noheader,nounits", "-lms", "100"],
                                  stdout=self.f, stderr=subprocess.DEVNULL)

    def stop(self):
        time.sleep(0.15)
        self.p.terminate()
        try:
            self.p.wait(timeout=5)
        except subprocess.TimeoutExpired:
            self.p.kill()
            self.p.wait()
        self.f.flush()
        rows = [l.strip().split(", ") for l in open(self.f.name) if l.strip()]
        os.unlink(self.f.name)
        sm, mem, pw, capped = [], [], [], 0
        for r in rows:
            try:
                sm.append(float(r[0]))
                mem.append(float(r[1]))
                pw.append(float(r[2]))
                capped += r[3].strip().lower() == "active"
            except (ValueError, IndexError):
                continue

        def med(v):
            return sorted(v)[len(v) // 2] if v else None
        return {"sm_mhz_median": med(sm), "mem_mhz_median": med(mem), "power_w_median": med(pw),
                "sw_power_cap_samples": capped, "samples": len(sm)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the lines to this file")
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--allocs", default=None, help="comma-separated --alloc values")
    ap.add_argument("--fills", default=None, help="comma-separated --fill values")
    args = ap.parse_args()
    if args.allocs or args.fills:
        runs = [(v, opts + ["--alloc", a, "--fill", f]) for a in (args.allocs or "plain").split(",")
                for f in (args.fills or "const").split(",") for v, opts in COMPRESSION_RUNS]
    else:
        runs = RUNS
    lines = []
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "hbm_ceiling")
        subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-o", exe,
                        os.path.join(HERE, "hbm_ceiling.cu")], check=True)
        name, plimit, maxsm, maxmem = smi("name,power.limit,clocks.max.sm,clocks.max.mem")
        lines.append(json.dumps({"gpu": name, "power_limit_w": float(plimit), "sm_max_mhz": float(maxsm), "mem_max_mhz": float(maxmem)}))
        print(lines[-1], flush=True)
        for variant, opts in runs:
            s = Sampler()
            p = subprocess.run([exe, variant, "--reps", str(args.reps)] + opts, stdout=subprocess.PIPE, text=True)
            clk = s.stop()
            if p.returncode != 0:
                print(f"{variant} {opts} failed with exit code {p.returncode}", file=sys.stderr)
                return p.returncode
            rec = json.loads(p.stdout.strip().splitlines()[-1])
            rec.update(clk)
            lines.append(json.dumps(rec))
            print(lines[-1], flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
