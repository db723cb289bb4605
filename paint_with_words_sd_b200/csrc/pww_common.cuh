// Shared host/device helpers for libpww_b200.so (sm_90a).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/pww_b200.h"

namespace pww {

// Per-image partial of the score statistic written by one CTA of the stats kernel.
struct StatPartial {
  double vmax;   // max of fp16-rounded scores seen by the CTA
  double sum;    // sum of fp16-rounded scores
  double sumsq;  // sum of squares
  double pad;
};

struct XattnParams {
  const __half* q;
  const __half* k;
  const __half* v;
  __half* out;
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

__device__ __forceinline__ float round_to_f16(float x) { return __half2float(__float2half_rn(x)); }

// Statistic kind of image b: max unless the image's kind (per-image array, else the launch's `stat`) is PWW_STAT_STD.
__device__ __forceinline__ bool image_is_max(const XattnParams& p, int b) {
  return p.stat_kind != nullptr ? __ldg(p.stat_kind + b) != PWW_STAT_STD : p.stat != PWW_STAT_STD;
}
// G(sigma) of image b.
__device__ __forceinline__ float image_g(const XattnParams& p, int b) { return __ldg(p.g_sigma + (int64_t)b * p.g_stride); }

}  // namespace pww
