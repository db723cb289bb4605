// Memory-bound fused ops of the UNet that CALLS the attention path (SURVEY.md 8f-1): GroupNorm(+per-channel add)(+SiLU)
// and GEGLU on channels-last activations of element type E (fp16 or bf16).  Each replaces 3-6 eager PyTorch launches
// and, together with channels-last convolutions, removes every NCHW<->NHWC conversion from the step.  Both are HBM-bound
// streaming kernels: 16-byte vector loads/stores, one pass for statistics + one pass to apply, deterministic reductions.
// Arithmetic is fp32 in both types; only the loads' conversion and the stores' rounding depend on E.
#pragma once
#include "pww_common.cuh"

namespace pww {
namespace uops {

template <typename E>
struct GnParams {
  const E* x;      // [B, HW, C] channels-last activations
  const E* add;    // [B, C] (row stride add_bs) or nullptr: per-image per-channel value added BEFORE normalisation
  long long add_bs;
  const E* gamma;  // [C]
  const E* beta;   // [C]
  E* y;            // [B, HW, C]
  float* partial;       // [B, chunks, G, 2] (sum, sumsq) scratch
  float* stats;         // [B, G, 2] (mean, rstd), written by the last stats block of each image
  unsigned int* counters;  // [B] arrival counters (zero on entry, zero on exit)
  int B, HW, C, G, chunks, rows_per_chunk, silu;
  float eps;
};

// pass 1: per (image, row chunk) partial sums per group.  block = nvec * rpp threads (nvec = C/8 vectors per row)
template <typename E>
__global__ void gn_stats_kernel(GnParams<E> p) {
  using X = Elem<E>;
  using E2 = typename X::E2;
  extern __shared__ float sm[];                 // [rpp][C][2] staging for the cross-row reduction, then [G][2]
  const int nvec = p.C >> 3;
  const int rpp = blockDim.x / nvec;
  const int v = threadIdx.x % nvec, rl = threadIdx.x / nvec;
  const int b = blockIdx.y, chunk = blockIdx.x;
  const int r0 = chunk * p.rows_per_chunk, r1 = min(p.HW, r0 + p.rows_per_chunk);
  float s[8], q[8], a[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { s[i] = 0.f; q[i] = 0.f; a[i] = 0.f; }
  if (p.add) {
    const uint4 av = *reinterpret_cast<const uint4*>(p.add + (size_t)b * p.add_bs + v * 8);
    const E2* ah = reinterpret_cast<const E2*>(&av);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float2 f = X::to_float2(ah[i]); a[2 * i] = f.x; a[2 * i + 1] = f.y; }
  }
  const E* xb = p.x + (size_t)b * p.HW * p.C;
  // 4 independent 16-byte loads in flight per thread
  for (int r = r0 + rl; r < r1; r += 4 * rpp) {
    uint4 xv[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int rr = r + u * rpp;
      xv[u] = rr < r1 ? __ldg(reinterpret_cast<const uint4*>(xb + (size_t)rr * p.C) + v) : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (r + u * rpp < r1) {
        const E2* xh = reinterpret_cast<const E2*>(&xv[u]);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          float2 f = X::to_float2(xh[i]);
          const float x0 = f.x + a[2 * i], x1 = f.y + a[2 * i + 1];
          s[2 * i] += x0; q[2 * i] = fmaf(x0, x0, q[2 * i]);
          s[2 * i + 1] += x1; q[2 * i + 1] = fmaf(x1, x1, q[2 * i + 1]);
        }
      }
    }
  }
  // per-thread channel sums -> shared [rl][c]
  float* ss = sm;
  float* sq = sm + rpp * p.C;
#pragma unroll
  for (int i = 0; i < 8; ++i) { ss[rl * p.C + v * 8 + i] = s[i]; sq[rl * p.C + v * 8 + i] = q[i]; }
  __syncthreads();
  // one thread per group reduces its channels over all row lanes in a fixed order
  const int cg = p.C / p.G;
  for (int g = threadIdx.x; g < p.G; g += blockDim.x) {
    float ts = 0.f, tq = 0.f;
    for (int r = 0; r < rpp; ++r)
      for (int c = g * cg; c < (g + 1) * cg; ++c) { ts += ss[r * p.C + c]; tq += sq[r * p.C + c]; }
    float* out = p.partial + (((size_t)b * p.chunks + chunk) * p.G + g) * 2;
    out[0] = ts; out[1] = tq;
  }
  // the last block of this image reduces the chunk partials in a fixed order -> (mean, rstd) per group
  __shared__ int is_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = (atomicAdd(&p.counters[b], 1u) == (unsigned)p.chunks - 1u) ? 1 : 0;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  // only FULL warps finalise (blockDim.x = nvec * rpp need not be a multiple of 32: a trailing partial warp would
  // alias warp 0's groups and shuffle with lanes that do not exist)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  for (int g = warp; warp < nwarps && g < p.G; g += nwarps) {
    const float* pp = p.partial + ((size_t)b * p.chunks * p.G + g) * 2;
    float ts = 0.f, tq = 0.f;
    for (int c = lane; c < p.chunks; c += 32) { ts += __ldcg(pp + (size_t)c * p.G * 2); tq += __ldcg(pp + (size_t)c * p.G * 2 + 1); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      ts += __shfl_xor_sync(0xffffffffu, ts, o);
      tq += __shfl_xor_sync(0xffffffffu, tq, o);
    }
    if (lane == 0) {
      const float n = (float)p.HW * (float)cg;
      const float mean = ts / n;
      float var = tq / n - mean * mean;
      var = var < 0.f ? 0.f : var;
      p.stats[((size_t)b * p.G + g) * 2] = mean;
      p.stats[((size_t)b * p.G + g) * 2 + 1] = rsqrtf(var + p.eps);
    }
  }
  if (threadIdx.x == 0) p.counters[b] = 0u;
}

// pass 2: y = act((x + add - mean) * rstd * gamma + beta).  grid (row chunks, B); block = nvec * rpp threads: a thread
// keeps ONE 8-channel vector column, so its scale/shift live in registers and the row loop is pure streaming.
template <typename E>
__global__ void gn_apply_kernel(GnParams<E> p, int rows_per_block) {
  using X = Elem<E>;
  using E2 = typename X::E2;
  const int nvec = p.C >> 3;
  const int rpp = blockDim.x / nvec;
  const int v = threadIdx.x % nvec, rl = threadIdx.x / nvec;
  const int b = blockIdx.y;
  const int cg = p.C / p.G;
  float sc[8], sh[8];
  {
    const uint4 gv = __ldg(reinterpret_cast<const uint4*>(p.gamma) + v);
    const uint4 bv = __ldg(reinterpret_cast<const uint4*>(p.beta) + v);
    uint4 av = make_uint4(0, 0, 0, 0);
    if (p.add) av = __ldg(reinterpret_cast<const uint4*>(p.add + (size_t)b * p.add_bs) + v);
    const E* gh = reinterpret_cast<const E*>(&gv);
    const E* bh = reinterpret_cast<const E*>(&bv);
    const E* ah = reinterpret_cast<const E*>(&av);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int g = (v * 8 + i) / cg;
      const float mean = __ldg(p.stats + ((size_t)b * p.G + g) * 2), rstd = __ldg(p.stats + ((size_t)b * p.G + g) * 2 + 1);
      sc[i] = rstd * X::to_float(gh[i]);
      sh[i] = X::to_float(bh[i]) + (X::to_float(ah[i]) - mean) * sc[i];
    }
  }
  const int r0 = blockIdx.x * rows_per_block, r1 = min(p.HW, r0 + rows_per_block);
  const E* xb = p.x + (size_t)b * p.HW * p.C;
  E* yb = p.y + (size_t)b * p.HW * p.C;
  for (int r = r0 + rl; r < r1; r += rpp) {
    const uint4 xv = __ldg(reinterpret_cast<const uint4*>(xb + (size_t)r * p.C) + v);
    const E2* xh = reinterpret_cast<const E2*>(&xv);
    __align__(16) E2 o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = X::to_float2(xh[k]);
      float y0 = fmaf(f.x, sc[2 * k], sh[2 * k]);
      float y1 = fmaf(f.y, sc[2 * k + 1], sh[2 * k + 1]);
      if (p.silu) {
        y0 = __fdividef(y0, 1.f + __expf(-y0));
        y1 = __fdividef(y1, 1.f + __expf(-y1));
      }
      o[k] = X::from_float2(y0, y1);
    }
    reinterpret_cast<uint4*>(yb + (size_t)r * p.C)[v] = *reinterpret_cast<const uint4*>(o);
  }
}

// GEGLU: out[m, i] = in[m, i] * gelu(in[m, I + i])   (exact erf GELU, like torch.nn.functional.gelu)
template <typename E>
__global__ void geglu_kernel(const E* __restrict__ in, E* __restrict__ out, long long M, int I) {
  using X = Elem<E>;
  using E2 = typename X::E2;
  const int nvec = I >> 3;
  const long long total = M * nvec;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long m = i / nvec;
    const int v = (int)(i % nvec);
    const uint4 av = __ldg(reinterpret_cast<const uint4*>(in + m * 2 * I) + v);
    const uint4 gv = __ldg(reinterpret_cast<const uint4*>(in + m * 2 * I + I) + v);
    const E2* ah = reinterpret_cast<const E2*>(&av);
    const E2* gh = reinterpret_cast<const E2*>(&gv);
    __align__(16) E2 o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 a = X::to_float2(ah[k]), g = X::to_float2(gh[k]);
      const float g0 = 0.5f * g.x * (1.f + erff(g.x * 0.70710678118654752f));
      const float g1 = 0.5f * g.y * (1.f + erff(g.y * 0.70710678118654752f));
      o[k] = X::from_float2(a.x * g0, a.y * g1);
    }
    reinterpret_cast<uint4*>(out + m * I)[v] = *reinterpret_cast<const uint4*>(o);
  }
}

// Fused residual add + LayerNorm over the last dim: s = x (+ res); sum_out = s (optional); y = LN(s) * gamma + beta.
// One warp per row; a lane keeps its 16-byte vectors of the row in registers (C <= 2048), two-pass mean/variance.
template <typename E, int VPL>   // vectors per lane
__global__ void add_layernorm_kernel(const E* __restrict__ x, const E* __restrict__ res,
                                     const E* __restrict__ gamma, const E* __restrict__ beta,
                                     E* __restrict__ sum_out, E* __restrict__ y, long long M, int C, float eps) {
  using X = Elem<E>;
  using E2 = typename X::E2;
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= M) return;
  const int nvec = C >> 3;
  float v[VPL][8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      const uint4 xv = __ldg(reinterpret_cast<const uint4*>(x + row * C) + vi);
      const E2* xh = reinterpret_cast<const E2*>(&xv);
      uint4 rv = make_uint4(0, 0, 0, 0);
      if (res) rv = __ldg(reinterpret_cast<const uint4*>(res + row * C) + vi);
      const E2* rh = reinterpret_cast<const E2*>(&rv);
      __align__(16) E2 so[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 a = X::to_float2(xh[k]), b = X::to_float2(rh[k]);
        // the residual stream is E in the eager model too: round the sum once, then normalise the rounded value
        so[k] = X::from_float2(a.x + b.x, a.y + b.y);
        const float2 f = X::to_float2(so[k]);
        v[i][2 * k] = f.x; v[i][2 * k + 1] = f.y;
        sum += f.x + f.y;
      }
      if (sum_out) reinterpret_cast<uint4*>(sum_out + row * C)[vi] = *reinterpret_cast<const uint4*>(so);
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) v[i][k] = 0.f;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / (float)C;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    if (lane + i * 32 < nvec) {
#pragma unroll
      for (int k = 0; k < 8; ++k) { const float d = v[i][k] - mean; sq = fmaf(d, d, sq); }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = rsqrtf(sq / (float)C + eps);
#pragma unroll
  for (int i = 0; i < VPL; ++i) {
    const int vi = lane + i * 32;
    if (vi < nvec) {
      const uint4 gv = __ldg(reinterpret_cast<const uint4*>(gamma) + vi);
      const uint4 bv = __ldg(reinterpret_cast<const uint4*>(beta) + vi);
      const E2* gh = reinterpret_cast<const E2*>(&gv);
      const E2* bh = reinterpret_cast<const E2*>(&bv);
      __align__(16) E2 o[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 g = X::to_float2(gh[k]), b = X::to_float2(bh[k]);
        o[k] = X::from_float2((v[i][2 * k] - mean) * rstd * g.x + b.x, (v[i][2 * k + 1] - mean) * rstd * g.y + b.y);
      }
      reinterpret_cast<uint4*>(y + row * C)[vi] = *reinterpret_cast<const uint4*>(o);
    }
  }
}

// ResNet-block epilogue: out[r, c] = E(a[r, c] + h[r, c] + bias[c]) over [rows, C] channels-last activations, with
// a = the block input (identity) or the bias-free shortcut conv output, h = the bias-free conv2 output and bias the fp32
// sum of conv2's and the shortcut's biases.  fp32 arithmetic, one rounding.  `out` may alias `h` (each thread reads its
// vector before it writes it), so neither carries __restrict__ or goes through the read-only cache.
template <typename E>
__global__ void resnet_residual_kernel(const E* a, const E* h, const float* __restrict__ bias, E* out,
                                       long long total_vec, int nvec) {
  using X = Elem<E>;
  using E2 = typename X::E2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total_vec;
       i += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(i % nvec);
    const uint4 av = reinterpret_cast<const uint4*>(a)[i];
    const uint4 hv = reinterpret_cast<const uint4*>(h)[i];
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(bias) + 2 * v);
    const float4 b1 = __ldg(reinterpret_cast<const float4*>(bias) + 2 * v + 1);
    const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
    const E2* ah = reinterpret_cast<const E2*>(&av);
    const E2* hh = reinterpret_cast<const E2*>(&hv);
    __align__(16) E2 o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 fa = X::to_float2(ah[k]), fh = X::to_float2(hh[k]);
      o[k] = X::from_float2(fa.x + fh.x + bb[2 * k], fa.y + fh.y + bb[2 * k + 1]);
    }
    reinterpret_cast<uint4*>(out)[i] = *reinterpret_cast<const uint4*>(o);
  }
}

inline int gn_chunks(int HW) {
  int rows = HW >= 4096 ? 64 : (HW >= 1024 ? 32 : 16);   // enough blocks to fill the SMs, few enough to finalise fast
  int c = (HW + rows - 1) / rows;
  return c < 1 ? 1 : (c > 512 ? 512 : c);
}

}  // namespace uops
}  // namespace pww
