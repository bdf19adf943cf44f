"""SASS evidence for the ahead-of-time scan kernels, from the built library (no GPU needed):
   python tools/sass_evidence.py > sass_scan_kernels.txt"""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "snappydata_b200", "csrc", "libsnappygpu.so")
sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
funcs, cur = {}, None
for ln in sass.splitlines():
    m = re.search(r"Function : (\S+)", ln)
    if m:
        cur = m.group(1)
        funcs[cur] = []
        continue
    m = re.search(r"/\*([0-9a-f]{4,})\*/\s+(.*?);", ln)
    if m and cur:
        funcs[cur].append((int(m.group(1), 16), m.group(2).strip()))


def count(ins, pat):
    return sum(1 for _, s in ins if re.search(pat, s))


print("SASS evidence for the ahead-of-time scan kernels (cuobjdump -sass snappydata_b200/csrc/libsnappygpu.so, sm_90a;")
print("tools/sass_evidence.py).  Per kernel: instruction count, the bulk-copy / mbarrier / shared-memory mnemonics that prove the")
print("cp.async.bulk (TMA unit) ring, the producer's first bulk copy, and the consumer from the full-barrier wait to the stage's release:")
print("stage loads (LDS) -> FENCE.VIEW.ASYNC.S (fence.proxy.async, DESIGN.md section 5) -> WARPSYNC -> @lane0 SYNCS.ARRIVE.")
print("No tensor-core ops (HMMA / HGMMA): the path has no contraction.\n")
for name, ins in funcs.items():
    if "scan_aggregate_kernel" not in name:
        continue
    plan = re.search(r"Plan_[0-9a-f]+", name)
    print("== %s" % (plan.group(0) if plan else name))
    print("   instructions %d; UBLKCP (cp.async.bulk global->shared) %d; SYNCS (mbarrier) %d; FENCE.VIEW.ASYNC %d; LDS.128 %d; LDS.64 %d; LDS (all) %d; STS %d; "
          "DADD %d; DMUL %d; LDG %d; ATOMS/ATOMG/RED %d; MEMBAR %d; HMMA/HGMMA %d" % (
              len(ins), count(ins, r"\bUBLKCP"), count(ins, r"\bSYNCS"), count(ins, r"FENCE\.VIEW\.ASYNC"), count(ins, r"\bLDS\.128"), count(ins, r"\bLDS\.64"),
              count(ins, r"\bLDS\b"), count(ins, r"\bSTS\b"), count(ins, r"\bDADD"), count(ins, r"\bDMUL"), count(ins, r"\bLDG"), count(ins, r"\b(ATOMS|ATOMG|RED)\b"),
              count(ins, r"\bMEMBAR"), count(ins, r"\b(HMMA|HGMMA)")))
    ub = [i for i, (_, s) in enumerate(ins) if s.startswith("UBLKCP") or " UBLKCP" in s]
    if ub:
        print("   -- producer: wait for the stage to be empty, expect-tx, first bulk copy")
        tw = [i for i in range(ub[0]) if "SYNCS.PHASECHK" in ins[i][1]]
        lo = tw[-1] if tw else max(0, ub[0] - 8)
        for a, s in ins[lo:ub[0] + 1]:
            if re.search(r"SYNCS|UBLKCP|BRA|ELECT", s):
                print("      /*%04x*/ %s" % (a, s))
    arr = [i for i, (_, s) in enumerate(ins) if "SYNCS.ARRIVE.TRANS64.A1T0" in s]
    if arr:
        i1 = arr[0]
        tw = [i for i in range(i1) if "SYNCS.PHASECHK" in ins[i][1]]
        i0 = tw[-1] if tw else max(0, i1 - 30)
        print("   -- consumer: full-barrier wait ... stage loads ... proxy fence ... release")
        for a, s in ins[i0:i1 + 1]:
            if re.search(r"SYNCS|LDS|FENCE|WARPSYNC|BAR\.", s):
                print("      /*%04x*/ %s" % (a, s))
    print()
