// sd_jit.cpp -- kernel launch helpers and the NVRTC path for plans that have no ahead-of-time
// compiled kernel.  Mirrors the role Janino plays for the reference (WholeStageCodegen compiles the
// generated class at plan time, caches it per plan: core/SnappySession.scala:2571-2607 plan cache):
// generated PLAN struct + the hand-written kernel template (embedded as text) -> NVRTC -> cubin
// for sm_90a -> CUfunction, cached in the kernel registry by plan signature.
//
// libnvrtc / libcuda are dlopen'ed on first use so that libsnappygpu.so itself loads on a box with no
// driver (the CPU-only build/test container).
#include <cuda.h>
#include <dlfcn.h>
#include <nvrtc.h>
#include <cstdlib>

#include <cstdio>
#include <cstring>
#include <mutex>

#include "sd_host.h"

extern "C" const char sd_embedded_device_h[];
extern "C" const char sd_embedded_kernels_cuh[];

namespace sd {

namespace {

struct Dyn {
  void* nvrtc = nullptr;
  void* cuda = nullptr;
  // nvrtc
  nvrtcResult (*CreateProgram)(nvrtcProgram*, const char*, const char*, int, const char* const*, const char* const*) = nullptr;
  nvrtcResult (*DestroyProgram)(nvrtcProgram*) = nullptr;
  nvrtcResult (*CompileProgram)(nvrtcProgram, int, const char* const*) = nullptr;
  nvrtcResult (*GetProgramLogSize)(nvrtcProgram, size_t*) = nullptr;
  nvrtcResult (*GetProgramLog)(nvrtcProgram, char*) = nullptr;
  nvrtcResult (*GetCUBINSize)(nvrtcProgram, size_t*) = nullptr;
  nvrtcResult (*GetCUBIN)(nvrtcProgram, char*) = nullptr;
  nvrtcResult (*AddNameExpression)(nvrtcProgram, const char*) = nullptr;
  nvrtcResult (*GetLoweredName)(nvrtcProgram, const char*, const char**) = nullptr;
  const char* (*GetErrorString)(nvrtcResult) = nullptr;
  // driver
  CUresult (*ModuleLoadData)(CUmodule*, const void*) = nullptr;
  CUresult (*ModuleGetFunction)(CUfunction*, CUmodule, const char*) = nullptr;
  CUresult (*FuncSetAttribute)(CUfunction, CUfunction_attribute, int) = nullptr;
  CUresult (*FuncGetAttribute)(int*, CUfunction_attribute, CUfunction) = nullptr;
  CUresult (*OccupancyMaxActiveBlocks)(int*, CUfunction, int, size_t) = nullptr;
  CUresult (*LaunchKernel)(CUfunction, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, unsigned, CUstream, void**, void**) = nullptr;
  CUresult (*GetErrorStringDrv)(CUresult, const char**) = nullptr;
  bool ok = false;
  std::string why;
};

Dyn& dyn() {
  static Dyn d;
  static std::once_flag once;
  std::call_once(once, [] {
    const char* nv[] = {"libnvrtc.so.12", "/usr/local/cuda/lib64/libnvrtc.so.12", "libnvrtc.so", "/usr/local/cuda/lib64/libnvrtc.so"};
    for (const char* n : nv) if ((d.nvrtc = dlopen(n, RTLD_NOW | RTLD_GLOBAL))) break;
    if (!d.nvrtc) { d.why = "libnvrtc.so.12 not found (needed to compile a plan without an ahead-of-time kernel)"; return; }
    d.cuda = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
    if (!d.cuda) { d.why = "libcuda.so.1 not found"; return; }
#define NV(sym) *(void**)(&d.sym) = dlsym(d.nvrtc, "nvrtc" #sym); if (!d.sym) { d.why = "nvrtc" #sym " missing"; return; }
    NV(CreateProgram) NV(DestroyProgram) NV(CompileProgram) NV(GetProgramLogSize) NV(GetProgramLog) NV(GetCUBINSize) NV(GetCUBIN)
    NV(AddNameExpression) NV(GetLoweredName) NV(GetErrorString)
#undef NV
#define CUF(field, sym) *(void**)(&d.field) = dlsym(d.cuda, sym); if (!d.field) { d.why = sym " missing"; return; }
    CUF(ModuleLoadData, "cuModuleLoadData") CUF(ModuleGetFunction, "cuModuleGetFunction") CUF(FuncSetAttribute, "cuFuncSetAttribute") CUF(FuncGetAttribute, "cuFuncGetAttribute")
    CUF(OccupancyMaxActiveBlocks, "cuOccupancyMaxActiveBlocksPerMultiprocessor") CUF(LaunchKernel, "cuLaunchKernel")
    CUF(GetErrorStringDrv, "cuGetErrorString")
#undef CUF
    d.ok = true;
  });
  return d;
}

const char* drv_err(CUresult r) {
  const char* s = nullptr;
  if (dyn().GetErrorStringDrv) dyn().GetErrorStringDrv(r, &s);
  return s ? s : "unknown driver error";
}

}  // namespace

int kernel_prepare(const KernelEntry& k, bool two_cta, size_t smem, int* ctas_per_sm) {
  const void* func = two_cta ? k.func2 : k.func;
  void* drv_func = two_cta ? k.drv_func2 : k.drv_func;
  if (func) {
    SD_CUDA(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    // ask for the largest shared-memory carveout so that several CTAs with private group tables fit per SM
    SD_CUDA(cudaFuncSetAttribute(func, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared));
    SD_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(ctas_per_sm, func, kernel_block_threads(k), smem));
    return 0;
  }
  Dyn& d = dyn();
  if (!d.ok || !drv_func) return set_error(SD_ERR_CUDA, "no kernel for this plan: %s", d.why.c_str());
  CUresult r = d.FuncSetAttribute((CUfunction)drv_func, CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES, (int)smem);
  if (r != CUDA_SUCCESS) return set_error(SD_ERR_CUDA, "cuFuncSetAttribute: %s", drv_err(r));
  d.FuncSetAttribute((CUfunction)drv_func, CU_FUNC_ATTRIBUTE_PREFERRED_SHARED_MEMORY_CARVEOUT, 100);
  r = d.OccupancyMaxActiveBlocks(ctas_per_sm, (CUfunction)drv_func, kernel_block_threads(k), smem);
  if (r != CUDA_SUCCESS) return set_error(SD_ERR_CUDA, "cuOccupancyMaxActiveBlocksPerMultiprocessor: %s", drv_err(r));
  return 0;
}

int kernel_local_bytes(const KernelEntry& k, bool two_cta, size_t* bytes) {
  const void* func = two_cta ? k.func2 : k.func;
  void* drv_func = two_cta ? k.drv_func2 : k.drv_func;
  if (func) {
    cudaFuncAttributes a;
    SD_CUDA(cudaFuncGetAttributes(&a, func));
    *bytes = a.localSizeBytes;
    return 0;
  }
  Dyn& d = dyn();
  if (!d.ok || !drv_func) return set_error(SD_ERR_CUDA, "no kernel for this plan: %s", d.why.c_str());
  int v = 0;
  CUresult r = d.FuncGetAttribute(&v, CU_FUNC_ATTRIBUTE_LOCAL_SIZE_BYTES, (CUfunction)drv_func);
  if (r != CUDA_SUCCESS) return set_error(SD_ERR_CUDA, "cuFuncGetAttribute: %s", drv_err(r));
  *bytes = (size_t)v;
  return 0;
}

int kernel_launch(const KernelEntry& k, bool two_cta, int grid, size_t smem, cudaStream_t stream, void** args) {
  const void* func = two_cta ? k.func2 : k.func;
  void* drv_func = two_cta ? k.drv_func2 : k.drv_func;
  if (func) {
    SD_CUDA(cudaLaunchKernel(func, dim3(grid), dim3(kernel_block_threads(k)), args, smem, stream));
    return 0;
  }
  Dyn& d = dyn();
  if (!d.ok || !drv_func) return set_error(SD_ERR_CUDA, "no kernel for this plan: %s", d.why.c_str());
  CUresult r = d.LaunchKernel((CUfunction)drv_func, grid, 1, 1, kernel_block_threads(k), 1, 1, (unsigned)smem, (CUstream)stream, args, nullptr);
  if (r != CUDA_SUCCESS) return set_error(SD_ERR_CUDA, "cuLaunchKernel: %s", drv_err(r));
  return 0;
}

int jit_compile(const PlanSpec& spec, int device, KernelEntry& out) {
  Dyn& d = dyn();
  if (!d.ok) return set_error(SD_ERR_CUDA, "plan %s has no ahead-of-time kernel and NVRTC is unavailable: %s", spec.struct_name.c_str(), d.why.c_str());
  SD_CUDA(cudaSetDevice(device));
  SD_CUDA(cudaFree(0));   // make sure the primary context exists and is current for the driver calls
  std::string src = "#include \"sd_kernels.cuh\"\n" + spec.source;
  const std::string name_expr = "sd::scan_aggregate_kernel<" + spec.struct_name + ">";
  const char* headers[] = {sd_embedded_device_h, sd_embedded_kernels_cuh};
  const char* names[] = {"sd_device.h", "sd_kernels.cuh"};
  nvrtcProgram prog;
  nvrtcResult nr = d.CreateProgram(&prog, src.c_str(), (spec.struct_name + ".cu").c_str(), 2, headers, names);
  if (nr != NVRTC_SUCCESS) return set_error(SD_ERR_CUDA, "nvrtcCreateProgram: %s", d.GetErrorString(nr));
  d.AddNameExpression(prog, name_expr.c_str());
  // a dense group-by's staged-only variant has a second kernel for two CTAs per SM (sd_kernels.cuh TwoCtaKernel)
  const bool two_cta = spec.mode == MODE_GROUPS && !spec.slow_paths && spec.stages > 0 && spec.reg_groups == 0;
  const std::string name_expr2 = "sd::scan_aggregate_kernel_2cta<" + spec.struct_name + ">";
  if (two_cta) d.AddNameExpression(prog, name_expr2.c_str());
  // -lineinfo adds ~50 % to the compile: only when a profile of a JIT kernel is wanted (SD_JIT_LINEINFO=1)
  // -device-int128: 128-bit integers of the wide-DECIMAL helpers in sd_kernels.cuh (nvcc allows them on sm_90a by default)
  std::vector<std::string> optv = {"--gpu-architecture=sm_90a", "-std=c++17", "--fmad=false", "-default-device", "-device-int128"};
  const char* li = getenv("SD_JIT_LINEINFO");
  if (li && atoi(li) > 0) optv.push_back("-lineinfo");
  if (const char* defs = getenv("SD_JIT_DEFINES")) {   // space-separated -DNAME=VALUE switches (experiments; part of the plan signature)
    std::string tok;
    for (const char* q = defs;; q++) {
      if (*q == ' ' || *q == 0) { if (!tok.empty()) optv.push_back(tok); tok.clear(); if (!*q) break; }
      else tok.push_back(*q);
    }
  }
  std::vector<const char*> opts;
  for (const std::string& o : optv) opts.push_back(o.c_str());
  nr = d.CompileProgram(prog, (int)opts.size(), opts.data());
  if (nr != NVRTC_SUCCESS) {
    size_t ls = 0;
    d.GetProgramLogSize(prog, &ls);
    std::string log(ls + 1, '\0');
    d.GetProgramLog(prog, &log[0]);
    d.DestroyProgram(&prog);
    return set_error(SD_ERR_CUDA, "NVRTC compile of %s failed: %.800s", spec.struct_name.c_str(), log.c_str());
  }
  size_t cs = 0;
  d.GetCUBINSize(prog, &cs);
  std::vector<char> cubin(cs);
  d.GetCUBIN(prog, cubin.data());
  const char* lowered = nullptr;
  nr = d.GetLoweredName(prog, name_expr.c_str(), &lowered);
  if (nr != NVRTC_SUCCESS || !lowered) { d.DestroyProgram(&prog); return set_error(SD_ERR_CUDA, "nvrtcGetLoweredName failed"); }
  CUmodule mod;
  CUresult r = d.ModuleLoadData(&mod, cubin.data());
  if (r != CUDA_SUCCESS) { d.DestroyProgram(&prog); return set_error(SD_ERR_CUDA, "cuModuleLoadData: %s", drv_err(r)); }
  CUfunction fn, fn2 = nullptr;
  r = d.ModuleGetFunction(&fn, mod, lowered);
  if (r == CUDA_SUCCESS && two_cta) {
    const char* lowered2 = nullptr;
    nr = d.GetLoweredName(prog, name_expr2.c_str(), &lowered2);
    if (nr != NVRTC_SUCCESS || !lowered2) { d.DestroyProgram(&prog); return set_error(SD_ERR_CUDA, "nvrtcGetLoweredName failed"); }
    r = d.ModuleGetFunction(&fn2, mod, lowered2);
  }
  d.DestroyProgram(&prog);
  if (r != CUDA_SUCCESS) return set_error(SD_ERR_CUDA, "cuModuleGetFunction: %s", drv_err(r));
  out.signature = spec.signature;
  out.func = nullptr;
  out.drv_func = (void*)fn;
  out.func2 = nullptr;
  out.drv_func2 = (void*)fn2;
  out.tile_smem = ((size_t)tile_smem_bytes((int)spec.cols.size(), spec.rpt) + 15) & ~size_t(15);
  out.origin = "jit";
  out.name = spec.struct_name;
  out.staged = spec.stages > 0 ? 1 : 0;
  out.stage_bytes = 0;
  for (int k : spec.kinds) out.stage_bytes += (size_t)THREADS * spec.rpt * kind_stage_width(k) + 128;
  return 0;
}

}  // namespace sd
