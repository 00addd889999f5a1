// Shared helpers for libctb200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <stdlib.h>
#include "../../include/ctb200.h"

namespace ctb {

extern thread_local char g_err[512];
extern thread_local int64_t g_launches;

inline int fail(int code, const char* fmt, const char* a = "", long b = 0, long c = 0) {
  snprintf(g_err, sizeof(g_err), fmt, a, b, c);
  return code;
}

#define CT_REQUIRE(cond, msg)                                                      \
  do {                                                                             \
    if (!(cond)) return ctb::fail(CT_ERR_INVALID, "%s: requirement failed: " msg " (%ld,%ld)", \
                                  __func__, 0, 0);                                 \
  } while (0)

#define CT_CUDA_OK(expr)                                                            \
  do {                                                                             \
    cudaError_t _e = (expr);                                                       \
    if (_e != cudaSuccess)                                                         \
      return ctb::fail(CT_ERR_CUDA, "%s: CUDA error %ld at line %ld", cudaGetErrorString(_e), \
                       (long)_e, (long)__LINE__);                                  \
  } while (0)

// SM count of the current device (grid caps of the grid-stride kernels), cached per device
inline int device_sm_count() {
  static thread_local int sms_of[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 64 && sms_of[dev]) return sms_of[dev];
  int sms = 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  if (dev < 64) sms_of[dev] = sms;
  return sms;
}

inline int after_launch() {
  ++g_launches;
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(CT_ERR_CUDA, "kernel launch failed: %s (%ld)", cudaGetErrorString(e), (long)e);
  }
  return CT_OK;
}

// ---- programmatic dependent launch (PDL): a kernel launched with the attribute may start while its predecessor in
// the stream is still running; it must execute pdl_wait() before touching anything the predecessor produces (or
// writing anything the predecessor may still read).  What runs before the wait -- shared-memory carve-up, mbarrier
// init, the halo engine's weight load -- overlaps the predecessor's tail.  pdl_trigger() lets the
// NEXT kernel of the stream do the same with us.  CTB_PDL=0 launches everything stream-serialised (no overlap).
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

inline bool pdl_enabled() {
  static const int on = getenv("CTB_PDL") ? atoi(getenv("CTB_PDL")) : 1;
  return on != 0;
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_kernel(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl,
                                 Args... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = (pdl && pdl_enabled()) ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// ---- element type helpers -----------------------------------------------------------
template <typename T> struct Elem;
template <> struct Elem<float> {
  static __device__ __forceinline__ float ld(const float* p) { return __ldg(p); }
  static __device__ __forceinline__ void st(float* p, float v) { *p = v; }
};
template <> struct Elem<__nv_bfloat16> {
  static __device__ __forceinline__ float ld(const __nv_bfloat16* p) {
    return __bfloat162float(*p);
  }
  static __device__ __forceinline__ void st(__nv_bfloat16* p, float v) {
    *p = __float2bfloat16_rn(v);
  }
};

__device__ __forceinline__ float sigmoidf_ref(float x) {
  // same formula as ATen's CPU/CUDA sigmoid: 1 / (1 + exp(-x)), fp32, IEEE division
  return 1.0f / (1.0f + expf(-x));
}
// Branch-free variant for the tensor-core engines' epilogues (ex2.approx + rcp.approx, ~2 ulp): the IEEE division
// and full-range expf of sigmoidf_ref form a ~130-cycle dependent chain per element that the two epilogue warps
// per scheduler cannot hide (the 80-channel heat-map head spent 13k cycles per 128-pixel tile in it).
__device__ __forceinline__ float sigmoidf_fast(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }

}  // namespace ctb
