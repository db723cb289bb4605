// ControlNet residual injection (pww_control_inject_f16 / _bf16): the 12 skip residuals and the mid residual of a
// ControlNet, each scaled per image, added in place into the UNet's skips and mid-block output in ONE launch.
//
//   dst_k[b] = E( dst_k[b] + E( s[k, b] * res_k[b] ) )      k < n, b < rows
//
// dst_k is [B, elems_k] and res_k [rows, elems_k], both dense; only the first `rows` images of dst_k are touched (rows
// = B / 2 is guess mode: the cond half).  The pointer / size table travels by value in the kernel parameters, so a
// captured CUDA graph carries it.  The arithmetic is fp32 with explicit round-to-nearest intrinsics, so nvcc cannot
// contract the multiply and the add into an FMA: the result is bitwise what torch computes for `skip + (r * s)` with
// the product rounded to E.
#pragma once
#include "pww_common.cuh"

namespace pww {
namespace ctl {

constexpr int kThreads = 256;
constexpr int kMaxLevels = 16;
constexpr int kVec = 8;                  // elements per 16-byte access

struct InjectArgs {
  void* dst[kMaxLevels];
  const void* res[kMaxLevels];
  int64_t vec_per_image[kMaxLevels];     // elems_k / 8
  int64_t off[kMaxLevels + 1];           // prefix offsets in 16-byte vectors: level k owns [off[k], off[k + 1])
  const float* scales;                   // [n, rows] fp32 on the device, or NULL = 1
  int n, rows;
};

template <typename E>
__device__ __forceinline__ unsigned inject_pair(unsigned d, unsigned r, float s) {
  typename Elem<E>::E2 dh, rh;
  memcpy(&dh, &d, 4);
  memcpy(&rh, &r, 4);
  const float2 df = Elem<E>::to_float2(dh), rf = Elem<E>::to_float2(rh);
  // the product is rounded to E before the add, as torch's `r * s` in the element type is
  const float p0 = round_to<E>(__fmul_rn(s, rf.x)), p1 = round_to<E>(__fmul_rn(s, rf.y));
  const typename Elem<E>::E2 o = Elem<E>::from_float2(__fadd_rn(df.x, p0), __fadd_rn(df.y, p1));
  unsigned u;
  memcpy(&u, &o, 4);
  return u;
}

// Grid-stride over every 16-byte vector of every level.  A thread's vector index only grows, so the level it is in is
// found by walking the prefix offsets forward from the level of its previous vector.
template <typename E>
__global__ void __launch_bounds__(kThreads) control_inject_kernel(const InjectArgs a) {
  const int64_t total = a.off[a.n];
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int k = 0;
  for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < total; v += stride) {
    while (v >= a.off[k + 1]) ++k;
    const int64_t local = v - a.off[k], vpi = a.vec_per_image[k];
    const int b = (int)(local / vpi);
    const int64_t j = local - (int64_t)b * vpi;
    const float s = a.scales != nullptr ? __ldg(a.scales + (int64_t)k * a.rows + b) : 1.f;
    uint4* d = reinterpret_cast<uint4*>(a.dst[k]) + (int64_t)b * vpi + j;
    const uint4 r = __ldg(reinterpret_cast<const uint4*>(a.res[k]) + (int64_t)b * vpi + j);
    uint4 x = *d;
    x.x = inject_pair<E>(x.x, r.x, s);
    x.y = inject_pair<E>(x.y, r.y, s);
    x.z = inject_pair<E>(x.z, r.z, s);
    x.w = inject_pair<E>(x.w, r.w, s);
    *d = x;
  }
}

// At most `max_blocks` CTAs: at the SD shapes every thread handles a few vectors.
template <typename E>
cudaError_t launch_inject(const InjectArgs& a, int64_t max_blocks, cudaStream_t s) {
  const int64_t total = a.off[a.n];
  int64_t blocks = (total + kThreads - 1) / kThreads;
  if (blocks > max_blocks) blocks = max_blocks;
  control_inject_kernel<E><<<(unsigned)blocks, kThreads, 0, s>>>(a);
  return cudaGetLastError();
}

}  // namespace ctl
}  // namespace pww
