// Multi-ControlNet residual combine (pww_control_combine_f16 / _bf16): the residuals of several ControlNets, each scaled
// per unit, level and image, summed level by level in unit order in ONE launch.
//
//   out_k[b] = E( ... E( E(s[0,k,b] * r_{0,k}[b]) + E(s[1,k,b] * r_{1,k}[b]) ) ... + E(s[U-1,k,b] * r_{U-1,k}[b]) )
//                                                                                  k < n, b < rows
//
// Every tensor of level k is [rows, elems_k], dense.  out[k] may be the same buffer as any res[u * n + k] (the sampler
// sums in place into the first unit's residuals): each thread reads all its inputs before it writes the one vector
// they share, so the residuals are read with ordinary loads, not the read-only path.  The pointer / size table travels
// by value in the kernel parameters (about 1.7 KB at 10 units), so a captured CUDA graph carries it.  Each product and
// each partial sum is rounded to E with explicit round-to-nearest intrinsics, so nvcc cannot form an FMA: the result is
// bitwise torch's `(r0 * s0).to(E) + (r1 * s1).to(E) + ...` evaluated left to right in E, the order of the reference
// extension's `total_control[k] += control[k] * weight` loop.  The UNet then adds the sum with the single-ControlNet
// inject at scale 1, and E(1 * x) = x.
#pragma once
#include "pww_common.cuh"
#include "control_inject.cuh"

namespace pww {
namespace ctl {

constexpr int kMaxUnits = 10;            // the reference extension's "Multi ControlNet: Max models amount"

struct CombineArgs {
  void* out[kMaxLevels];
  const void* res[kMaxUnits * kMaxLevels];   // unit-major: res[u * n + k]
  int64_t vec_per_image[kMaxLevels];         // elems_k / 8
  int64_t off[kMaxLevels + 1];               // prefix offsets in 16-byte vectors: level k owns [off[k], off[k + 1])
  const float* scales;                       // [units, n, rows] fp32 on the device
  int units, n, rows;
};

// Unit u's contribution to a pair of elements: acc = E(acc + E(s * r)), or E(s * r) for the first unit.
template <typename E>
__device__ __forceinline__ void combine_pair(float2& acc, unsigned r, float s, bool first) {
  typename Elem<E>::E2 rh;
  memcpy(&rh, &r, 4);
  const float2 rf = Elem<E>::to_float2(rh);
  const float p0 = round_to<E>(__fmul_rn(s, rf.x)), p1 = round_to<E>(__fmul_rn(s, rf.y));
  acc.x = first ? p0 : round_to<E>(__fadd_rn(acc.x, p0));
  acc.y = first ? p1 : round_to<E>(__fadd_rn(acc.y, p1));
}

template <typename E>
__device__ __forceinline__ unsigned pack_pair(float2 v) {
  const typename Elem<E>::E2 o = Elem<E>::from_float2(v.x, v.y);   // exact: both halves are already values of E
  unsigned u;
  memcpy(&u, &o, 4);
  return u;
}

// Grid-stride over every 16-byte vector of every level, as control_inject_kernel.
template <typename E>
__global__ void __launch_bounds__(kThreads) control_combine_kernel(const CombineArgs a) {
  const int64_t total = a.off[a.n];
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int k = 0;
  for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < total; v += stride) {
    while (v >= a.off[k + 1]) ++k;
    const int64_t local = v - a.off[k], vpi = a.vec_per_image[k];
    const int b = (int)(local / vpi);             // every tensor of level k is dense, so `local` indexes them all
    float2 acc[4];
    for (int u = 0; u < a.units; ++u) {
      const float s = __ldg(a.scales + ((int64_t)u * a.n + k) * a.rows + b);
      const uint4 r = reinterpret_cast<const uint4*>(a.res[u * a.n + k])[local];
      combine_pair<E>(acc[0], r.x, s, u == 0);
      combine_pair<E>(acc[1], r.y, s, u == 0);
      combine_pair<E>(acc[2], r.z, s, u == 0);
      combine_pair<E>(acc[3], r.w, s, u == 0);
    }
    uint4 o;
    o.x = pack_pair<E>(acc[0]);
    o.y = pack_pair<E>(acc[1]);
    o.z = pack_pair<E>(acc[2]);
    o.w = pack_pair<E>(acc[3]);
    reinterpret_cast<uint4*>(a.out[k])[local] = o;
  }
}

template <typename E>
cudaError_t launch_combine(const CombineArgs& a, int64_t max_blocks, cudaStream_t s) {
  const int64_t total = a.off[a.n];
  int64_t blocks = (total + kThreads - 1) / kThreads;
  if (blocks > max_blocks) blocks = max_blocks;
  control_combine_kernel<E><<<(unsigned)blocks, kThreads, 0, s>>>(a);
  return cudaGetLastError();
}

}  // namespace ctl
}  // namespace pww
