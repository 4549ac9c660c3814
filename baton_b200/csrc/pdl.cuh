// Programmatic Dependent Launch (PDL) helpers.
//
// A local-SGD step is ~200 small kernels in a dependency chain; at ~1 ms per step the per-node
// launch latency and prologue (barrier init, descriptor prefetch, smem tables) is a
// large share of the time.  Every kernel of this library
//   1. calls griddep_launch_dependents() first thing  -> the NEXT kernel in the stream / captured
//      graph may become resident and run its prologue while this one is still executing, and
//   2. calls griddep_wait() before its first access to global memory -> it only consumes the
//      previous kernel's results once that grid has completed and flushed.
// Launches go through launch_pdl(), which sets cudaLaunchAttributeProgrammaticStreamSerialization
// (captured into CUDA graphs as programmatic dependency edges).  BATON_PDL=0 disables it.
#pragma once
#include <cuda_runtime.h>

#include <cstdlib>
#include <utility>

namespace b200 {

// ---- in-graph kernel timeline (build with -DB200_TRACE: `BATON_BUILD_TRACE=1 python -m baton_b200.build_ext`) ----
// CUDA graphs hide per-kernel timing from CUDA events, and ncu serialises launches with cold caches, so neither
// shows where a captured local-SGD step spends its time.  In a trace build CTA 0 of every kernel stamps
// %globaltimer twice: when it becomes resident (tag < 0, at griddep_launch_dependents) and when its
// dependencies have completed (tag > 0, after griddep_wait).  tag = TU id * 100000 + source line, resolved back
// to the kernel name by baton_b200/utils/trace.py.  The buffer pointer lives in a per-translation-unit
// __device__ variable (no relocatable device code), set through b200_trace_set_<tu>().
#ifndef B200_TU_TAG
#define B200_TU_TAG 0
#endif
#ifdef B200_TRACE
static __device__ unsigned long long* b200_trace_ptr = nullptr;   // [0] = cursor, [1] = capacity, then (t, tag) pairs
__device__ __forceinline__ void trace_stamp(long long tag) {
  if (threadIdx.x == 0 && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) {
    unsigned long long* p = b200_trace_ptr;
    if (p != nullptr) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      const unsigned long long i = atomicAdd(p, 1ull);
      if (i < p[1]) {
        p[2 + 2 * i] = t;
        p[3 + 2 * i] = static_cast<unsigned long long>(tag);
      }
    }
  }
}
// intra-kernel stamp from ANY single thread of CTA (0,0,0) (the caller guarantees one thread executes it)
__device__ __forceinline__ void trace_point(long long tag) {
  if (blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) {
    unsigned long long* p = b200_trace_ptr;
    if (p != nullptr) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      const unsigned long long i = atomicAdd(p, 1ull);
      if (i < p[1]) {
        p[2 + 2 * i] = t;
        p[3 + 2 * i] = static_cast<unsigned long long>(tag);
      }
    }
  }
}
static int b200_trace_set_local(unsigned long long* p) {
  return static_cast<int>(cudaMemcpyToSymbol(b200_trace_ptr, &p, sizeof(p)));
}
#define B200_TRACE_REGISTER(tu) \
  extern "C" int b200_trace_set_##tu(unsigned long long* p) { return b200::b200_trace_set_local(p); }
#else
__device__ __forceinline__ void trace_stamp(long long) {}
__device__ __forceinline__ void trace_point(long long) {}
#define B200_TRACE_REGISTER(tu) \
  extern "C" int b200_trace_set_##tu(unsigned long long*) { return -1; }
#endif

__device__ __forceinline__ void griddep_wait_tagged(long long tag) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  trace_stamp(tag);
}
__device__ __forceinline__ void griddep_launch_dependents_tagged(long long tag) {
  trace_stamp(-tag);
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
// TRACE_POINT(): intra-kernel timeline stamp (trace build only), tag = 5e9 + TU * 100000 + line; the label is the comment
// on the same source line
#define TRACE_POINT() trace_point(5000000000ll + static_cast<long long>(B200_TU_TAG) * 100000 + __LINE__)
#define griddep_wait() griddep_wait_tagged(static_cast<long long>(B200_TU_TAG) * 100000 + __LINE__)
#define griddep_launch_dependents() griddep_launch_dependents_tagged(static_cast<long long>(B200_TU_TAG) * 100000 + __LINE__)

// streaming multiprocessors of the current device (grid caps, one-wave thresholds, co-residency bounds)
inline int device_sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 1;
  }
  return n;
}
// BATON_PDL=0 launches every kernel without the programmatic-serialization attribute.  It selects no separate code:
// it rules PDL in or out as the cause of an ordering race (DESIGN.md section 6), and scripts/microbench.py measures
// the per-node cost with and without it.
inline bool pdl_enabled() {
  static int on = -1;
  if (on < 0) {
    const char* e = std::getenv("BATON_PDL");
    on = (e != nullptr && e[0] == '0') ? 0 : 1;
  }
  return on == 1;
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(std::forward<Args>(args))...);
}

}  // namespace b200
