// Shared host/device helpers for libpww_b200.so (sm_90a).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/pww_b200.h"

namespace pww {

// Element type of the activations: __half (fp16) or __nv_bfloat16 (bf16).  Every kernel family is instantiated for
// both; the conversions below are the only place the two differ outside the MMA instruction (mma_sm90.cuh).  Both
// are 2-byte types, so copies, strides and shared-memory layouts are the same.
template <typename E> struct Elem;
template <> struct Elem<__half> {
  using E2 = __half2;
  static __device__ __forceinline__ float to_float(__half x) { return __half2float(x); }
  static __device__ __forceinline__ __half from_float(float x) { return __float2half_rn(x); }
  static __device__ __forceinline__ float2 to_float2(__half2 x) { return __half22float2(x); }
  static __device__ __forceinline__ __half2 from_float2(float lo, float hi) { return __floats2half2_rn(lo, hi); }
};
template <> struct Elem<__nv_bfloat16> {
  using E2 = __nv_bfloat162;
  static __device__ __forceinline__ float to_float(__nv_bfloat16 x) { return __bfloat162float(x); }
  static __device__ __forceinline__ __nv_bfloat16 from_float(float x) { return __float2bfloat16_rn(x); }
  static __device__ __forceinline__ float2 to_float2(__nv_bfloat162 x) { return __bfloat1622float2(x); }
  static __device__ __forceinline__ __nv_bfloat162 from_float2(float lo, float hi) { return __floats2bfloat162_rn(lo, hi); }
};

// Per-image partial of the score statistic written by one CTA of the stats kernel.
struct StatPartial {
  double vmax;   // max of the scores seen by the CTA
  double sum;    // sum of the element-type-rounded scores
  double sumsq;  // sum of squares
  double pad;
};

template <typename E>
struct XattnParams {
  const E* q;
  const E* k;
  const E* v;
  E* out;
  int B, H, N, T, D;
  int64_t q_bs, q_rs, k_bs, k_rs, o_bs, o_rs;  // element strides
  const float* wmap;
  int64_t wmap_bs;
  const int32_t* wmap_index;
  const float* stats;
  const float* g_sigma;
  int64_t g_stride;        // image b's G(sigma) is g_sigma[b * g_stride]: 0 = one value for every image
  float scale;
  // stats kernel only
  int stat;
  const int32_t* stat_kind;   // [B] per-image statistic kind, or NULL = `stat` for every image
  float* stats_out;
  unsigned int* counters;  // [B] arrival counters (zero on entry, zero on exit)
  StatPartial* partials;   // [B][grid] partial slots, one per CTA
};

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// x rounded to the nearest value of element type E.
template <typename E>
__device__ __forceinline__ float round_to(float x) { return Elem<E>::to_float(Elem<E>::from_float(x)); }

// Statistic kind of image b: max unless the image's kind (per-image array, else the launch's `stat`) is PWW_STAT_STD.
template <typename E>
__device__ __forceinline__ bool image_is_max(const XattnParams<E>& p, int b) {
  return p.stat_kind != nullptr ? __ldg(p.stat_kind + b) != PWW_STAT_STD : p.stat != PWW_STAT_STD;
}
// G(sigma) of image b.
template <typename E>
__device__ __forceinline__ float image_g(const XattnParams<E>& p, int b) { return __ldg(p.g_sigma + (int64_t)b * p.g_stride); }

// ---- host side of the launchers: per-device state, keyed by the current device (the Python shim makes the tensors'
// device current) ----
constexpr int kMaxDevices = 64;
inline int cur_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return (dev >= 0 && dev < kMaxDevices) ? dev : 0;
}
inline int num_sms() {
  static int n[kMaxDevices] = {0};
  const int dev = cur_device();
  if (!n[dev]) cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev);
  return n[dev];
}
// Lets Kernel take `bytes` of dynamic shared memory; the attribute is set once per device.
template <auto Kernel>
cudaError_t allow_dynamic_smem(uint32_t bytes) {
  static bool done[kMaxDevices] = {false};
  const int dev = cur_device();
  if (done[dev]) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e == cudaSuccess) done[dev] = true;
  return e;
}

// The image order of the host schedule replays: img[0, nb) = the images with a weight map (wmap_index[b] >= 0), then
// img[nb, B) = the others, each in batch order.  Returns nb.  The kernels build the same order with warp ballots.
inline int partition_images(int B, const int* wmap_index, int* img) {
  int nb = 0;
  for (int b = 0; b < B; ++b) if (wmap_index[b] >= 0) img[nb++] = b;
  int nu = 0;
  for (int b = 0; b < B; ++b) if (wmap_index[b] < 0) img[nb + nu++] = b;
  return nb;
}

}  // namespace pww
