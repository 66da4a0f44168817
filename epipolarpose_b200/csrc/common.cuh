// Shared helpers for libepb.so (sm_90a).  Error convention: see include/epb.h.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include "../../include/epb.h"

void epb_set_error(const char* fmt, ...);

#define EPB_CHECK_ARG(cond)                                                   \
  do {                                                                        \
    if (!(cond)) {                                                            \
      epb_set_error("%s:%d: invalid argument: %s", __FILE__, __LINE__, #cond); \
      return EPB_EINVAL;                                                      \
    }                                                                         \
  } while (0)

#define EPB_CUDA(call)                                                        \
  do {                                                                        \
    cudaError_t e__ = (call);                                                 \
    if (e__ != cudaSuccess) {                                                 \
      epb_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call,             \
                    cudaGetErrorString(e__));                                 \
      return EPB_ECUDA;                                                       \
    }                                                                         \
  } while (0)

#define EPB_LAUNCH_CHECK() EPB_CUDA(cudaGetLastError())

// per-(purpose, device, stream) internal scratch; see core.cu
enum { EPB_WS_SOFTARGMAX = 1, EPB_WS_HMLOSS = 2, EPB_WS_BNCOEF = 3, EPB_WS_WPLANES = 4,
       EPB_WS_FPAIR = 5, EPB_WS_BNPART = 6, EPB_WS_SABWD = 7, EPB_WS_PATCHINV = 8, EPB_WS_KMEANS = 9 };
int epb_workspace(int kind, size_t bytes, cudaStream_t st, void** out);

static inline cudaStream_t as_stream(epb_stream_t s) { return (cudaStream_t)s; }

constexpr int kNumSMs = 132;  // H100 SXM

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// streaming 128-bit load that does not pollute L1
__device__ __forceinline__ float4 ldg_stream(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
