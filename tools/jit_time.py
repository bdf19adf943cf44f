"""Time the NVRTC compile of a plan's kernel on the host (no GPU needed): python tools/jit_time.py [q1|q6|c1] [0|1 = with per-row paths] [extra nvrtc options...]"""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cuda.bindings import nvrtc
from snappydata_b200 import build, plan as P

def main():
    which = sys.argv[1] if len(sys.argv) > 1 else "q1"
    slow = int(sys.argv[2]) if len(sys.argv) > 2 else 0      # 1: the variant that carries the per-row paths
    extra = sys.argv[3:]
    g = build.generate_plan_source(P.AOT_PLANS[which](), slow_paths=slow)
    csrc = os.path.join(os.path.dirname(build.__file__), "csrc")
    hdrs = [open(os.path.join(csrc, n)).read().encode() for n in ("sd_device.h", "sd_kernels.cuh")]
    src = ('#include "sd_kernels.cuh"\n' + g["source"]).encode()
    err, prog = nvrtc.nvrtcCreateProgram(src, b"plan.cu", 2, hdrs, [b"sd_device.h", b"sd_kernels.cuh"])
    nvrtc.nvrtcAddNameExpression(prog, ("sd::scan_aggregate_kernel<%s>" % g["name"]).encode())
    opts = [b"--gpu-architecture=sm_90a", b"-std=c++17", b"--fmad=false", b"-default-device"] + [e.encode() for e in extra]
    t = time.time()
    (err,) = nvrtc.nvrtcCompileProgram(prog, len(opts), opts)
    dt = time.time() - t
    if int(err) != 0:
        _, n = nvrtc.nvrtcGetProgramLogSize(prog); log = b" " * n; nvrtc.nvrtcGetProgramLog(prog, log); print(log.decode()[-2000:])
    _, n = nvrtc.nvrtcGetCUBINSize(prog)
    print(f"{which} slow_paths={slow}: nvrtc {dt:.2f} s, cubin {n} bytes, opts {[o.decode() for o in opts[3:]]}")

main()
