// Shared helpers for libdvd_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>

#include "../../include/dvd_b200.h"

namespace dvd {

void set_error(const char* fmt, ...);

#define DVD_ARG_CHECK(cond, ...)                 \
  do {                                           \
    if (!(cond)) {                               \
      dvd::set_error(__VA_ARGS__);               \
      return -1;                                 \
    }                                            \
  } while (0)

#define DVD_CUDA_LAUNCH_CHECK(what)                                               \
  do {                                                                            \
    cudaError_t e__ = cudaGetLastError();                                         \
    if (e__ != cudaSuccess) {                                                     \
      dvd::set_error("%s: %s", what, cudaGetErrorString(e__));                    \
      return (int)e__;                                                            \
    }                                                                             \
  } while (0)

#define DVD_CUDA_CALL(expr)                                                       \
  do {                                                                            \
    cudaError_t e__ = (expr);                                                     \
    if (e__ != cudaSuccess) {                                                     \
      dvd::set_error("%s: %s", #expr, cudaGetErrorString(e__));                   \
      return (int)e__;                                                            \
    }                                                                             \
  } while (0)

static inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

int num_sms();

// ---- programmatic dependent launch --------------------------------------------------------------------------------
// Every kernel of the library is launched with cudaLaunchAttributeProgrammaticStreamSerialization (unless DVD_PDL=0) and begins
// with DVD_PDL_ENTER(): griddepcontrol.wait (the preceding grid of the stream has completed and its writes are visible), then
// griddepcontrol.launch_dependents (the NEXT grid may be scheduled as soon as every CTA of this one has passed this point and
// resources free up: its launch latency, CTA start-up, barrier / tensor-memory set-up overlap this grid's tail). Because each
// kernel waits before it triggers, at most two grids of a stream are in flight and completion stays transitive: when a grid's
// wait returns, every earlier grid of the stream has completed. Tensor-core kernels run their set-up BEFORE the wait.
bool pdl_enabled();

template <typename... KArgs, typename... Args>
inline cudaError_t launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem_bytes, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem_bytes;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1u : 0u;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<Args&&>(args)...);
}

// ---- device helpers -------------------------------------------------------------------------
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
#define DVD_PDL_ENTER()            \
  do {                             \
    dvd::pdl_wait();               \
    dvd::pdl_launch_dependents();  \
  } while (0)

// ---- ordered reductions (DESIGN.md 2.11) ----------------------------------------------------------------------------
// The *_ordered entry points do not add partial sums into shared outputs with fp32 atomics, whose order changes from run to
// run: every CTA (or warp) writes its partials into a slab of its own in a caller-supplied workspace, and ordered_sum adds the
// slabs in slab order: dst0[i] += sum_s slab[s * n + i] for i < n0, dst1[i - n0] += ... for n0 <= i < n (dst1 may be null
// when n0 == n).
int launch_ordered_sum(const float* slab, int nslab, long n, float* dst0, long n0, float* dst1, cudaStream_t st);

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// streaming 128-bit load that does not pollute L1 (inputs are touched once per kernel)
__device__ __forceinline__ float4 ldg_stream4(const float* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ float ldg_stream1(const float* p) {
  float r;
  asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
  return r;
}
__device__ __forceinline__ void st_stream4(float* p, float4 v) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y),
               "f"(v.z), "f"(v.w)
               : "memory");
}

}  // namespace dvd
