// How this engine launches a chain of kernels: the activation codes, the programmatic-dependent-launch (PDL) device
// helpers every kernel of a chain calls, and the host-side launch context (SM count, PDL switch, launch counter,
// first-error capture, owned device allocations) of one policy or GST predictor handle.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

#include "cn_host_util.h"

enum { CN_ACT_NONE = 0, CN_ACT_RELU = 1, CN_ACT_TANH = 2 };

// Programmatic dependent launch (PDL): kernels of a chain are launched with
// cudaLaunchAttributeProgrammaticStreamSerialization; each one lets its successor be scheduled as early as
// possible (launch_dependents) and itself waits for the full completion + memory flush of its predecessor
// (wait) before it touches global memory.  Both are no-ops for a normal launch.
__device__ __forceinline__ void cn_pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void cn_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void cn_pdl_prologue() { cn_pdl_trigger(); cn_pdl_wait(); }
// Device-side counts written by an earlier kernel of the chain: a plain load through a `const __restrict__` pointer is an
// invariant load to the compiler, which schedules it ABOVE griddepcontrol.wait (seen in SASS: LDG.CONSTANT before
// ACQBULK) and so reads the previous step's value.  A volatile asm load stays behind the wait.
// tools/check_pdl_sass.py (tests/test_build_checks.py) scans the built library for this pattern.
__device__ __forceinline__ int cn_ld_after_wait(const int* p) {
  int v;
  asm volatile("ld.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// Launch context of a handle.  launch_k and the tensor-core GEMM (cn_gemm_tc.h) enqueue through it; allocations made
// with palloc belong to it and are released by cn_launch_free.
struct CnLaunchCtx {
  int num_sms = 132;
  bool pdl = false;             // programmatic dependent launch along the kernel chain (CN_PDL=0 disables)
  int64_t launches = 0;
  bool launch_error = false;    // a launch or a GEMM output map failed (cn_last_error has the stage and the reason)
  const char* cur_stage = nullptr;   // stage name of the launches being enqueued (error reports)
  std::vector<void*> allocs;
};

// SM count of `device` and the CN_PDL switch
inline void cn_launch_init(CnLaunchCtx* c, int device) {
  cudaDeviceGetAttribute(&c->num_sms, cudaDevAttrMultiProcessorCount, device);
  const char* pd = getenv("CN_PDL");
  c->pdl = !(pd && pd[0] == '0');
}

inline void cn_launch_free(CnLaunchCtx* c) {
  for (void* q : c->allocs) cudaFree(q);
  c->allocs.clear();
}

// zero-filled device buffer of `count` floats, owned by the context
inline int palloc(CnLaunchCtx* c, float** ptr, size_t count) {
  void* q = nullptr;
  cudaError_t err = cudaMalloc(&q, (count ? count : 4) * sizeof(float));
  if (err != cudaSuccess) return cn_set_error("cudaMalloc(%zu floats): %s", count, cudaGetErrorString(err));
  cudaMemset(q, 0, (count ? count : 4) * sizeof(float));
  c->allocs.push_back(q);
  *ptr = static_cast<float*>(q);
  return 0;
}

// Kernel launch with (optionally) programmatic dependent launch: the kernel may be scheduled before its
// predecessor in the stream has finished; every kernel of the chain calls griddepcontrol.wait before touching
// global memory (cn_pdl_prologue / cn_pdl_wait), so the data dependencies are unchanged.
template <typename... KArgs, typename... Args>
void launch_k(CnLaunchCtx* c, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = c->pdl ? 1 : 0;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
  if (e != cudaSuccess && !c->launch_error) {     // keep the FIRST failure and the stage it happened in
    c->launch_error = true;
    cn_set_error("kernel launch failed in stage '%s' (launch #%lld of this handle): %s",
                 c->cur_stage ? c->cur_stage : "?", (long long)c->launches, cudaGetErrorString(e));
  }
  c->launches += 1;
}
