// T2I-Adapter feature add fused into a residual epilogue (pww_adapter_residual_f16 / _bf16).  The last layer of each
// UNet encoder level ends with a residual add (a transformer's `proj + res`, or the level-3 ResNet block's epilogue);
// an adapter's feature for that level is added to its result before the skip is taken, in the same launch:
//
//   s = E( a + b [+ bias_c] )                     every row
//   out = E( s + feat_r )   for r < feat_rows,    out = s otherwise
//
// over [rows, h, w, C] channels-last tensors (feat: [feat_rows, h, w, C]).  fp32 arithmetic, rounded to E after each
// add, so the result is bitwise torch's `(proj + res) + feat` in E, and with a bias the ResNet epilogue followed by
// `+ feat`.  `out` may alias a or b (each thread reads its vector before it writes it), so neither carries __restrict__
// or goes through the read-only cache.
#pragma once
#include "pww_common.cuh"

namespace pww {
namespace adp {

constexpr int kThreads = 256;

template <typename E>
__global__ void __launch_bounds__(kThreads) adapter_residual_kernel(const E* a, const E* b,
                                                                    const float* __restrict__ bias,
                                                                    const E* __restrict__ feat, E* out,
                                                                    long long total_vec, long long feat_vec, int nvec) {
  using X = Elem<E>;
  using E2 = typename X::E2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total_vec;
       i += (long long)gridDim.x * blockDim.x) {
    const uint4 av = reinterpret_cast<const uint4*>(a)[i];
    const uint4 bv = reinterpret_cast<const uint4*>(b)[i];
    float bb[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (bias != nullptr) {
      const int v = (int)(i % nvec);
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(bias) + 2 * v);
      const float4 b1 = __ldg(reinterpret_cast<const float4*>(bias) + 2 * v + 1);
      bb[0] = b0.x; bb[1] = b0.y; bb[2] = b0.z; bb[3] = b0.w;
      bb[4] = b1.x; bb[5] = b1.y; bb[6] = b1.z; bb[7] = b1.w;
    }
    const E2* ah = reinterpret_cast<const E2*>(&av);
    const E2* bh = reinterpret_cast<const E2*>(&bv);
    __align__(16) E2 o[4];
    if (bias != nullptr) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 fa = X::to_float2(ah[k]), fb = X::to_float2(bh[k]);
        o[k] = X::from_float2(__fadd_rn(__fadd_rn(fa.x, fb.x), bb[2 * k]),
                              __fadd_rn(__fadd_rn(fa.y, fb.y), bb[2 * k + 1]));
      }
    } else {
      // no bias term at all: adding 0.f would turn a -0 sum into +0, which torch's two-operand add does not
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 fa = X::to_float2(ah[k]), fb = X::to_float2(bh[k]);
        o[k] = X::from_float2(__fadd_rn(fa.x, fb.x), __fadd_rn(fa.y, fb.y));
      }
    }
    if (i < feat_vec) {
      const uint4 fv = __ldg(reinterpret_cast<const uint4*>(feat) + i);
      const E2* fh = reinterpret_cast<const E2*>(&fv);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 fs = X::to_float2(o[k]), ff = X::to_float2(fh[k]);
        o[k] = X::from_float2(__fadd_rn(fs.x, ff.x), __fadd_rn(fs.y, ff.y));
      }
    }
    reinterpret_cast<uint4*>(out)[i] = *reinterpret_cast<const uint4*>(o);
  }
}

// Grid-stride, at most `max_blocks` CTAs of 256 threads, one 16-byte vector (8 channels) per thread and iteration.
template <typename E>
cudaError_t launch(const void* a, const void* b, const float* bias, const void* feat, void* out, long long total_vec,
                   long long feat_vec, int nvec, long long max_blocks, cudaStream_t s) {
  long long blocks = (total_vec + kThreads - 1) / kThreads;
  if (blocks > max_blocks) blocks = max_blocks;
  adapter_residual_kernel<E><<<(unsigned)blocks, kThreads, 0, s>>>((const E*)a, (const E*)b, bias, (const E*)feat,
                                                                    (E*)out, total_vec, feat_vec, nvec);
  return cudaGetLastError();
}

}  // namespace adp
}  // namespace pww
