// Memory-bound fused ops of the UNet that CALLS the attention path (SURVEY.md 8f-1): GroupNorm(+per-channel add)(+SiLU)
// and GEGLU on channels-last activations of element type E (fp16 or bf16).  Each replaces 3-6 eager PyTorch launches
// and, together with channels-last convolutions, removes every NCHW<->NHWC conversion from the step.  Both are HBM-bound
// streaming kernels: 16-byte vector loads/stores, one pass for statistics + one pass to apply, deterministic reductions.
// Arithmetic is fp32 in both types; only the loads' conversion and the stores' rounding depend on E.
#pragma once
#include "pww_common.cuh"

namespace pww {
namespace uops {

// GroupNorm.  Both passes split an image into channel slices (whole groups AND whole 16-byte vectors: a multiple of
// lcm(8, C/G) channels) and row chunks; a thread keeps one 8-channel vector column of its slice.  The split is a
// function of (HW, C, G) only (gn_split), so batching never changes a result.
template <typename E>
struct GnParams {
  const E* x;      // [B, HW, C] channels-last activations
  const E* add;    // [B, C] (row stride add_bs) or nullptr: per-image per-channel value added BEFORE normalisation
  long long add_bs;
  const E* gamma;  // [C]
  const E* beta;   // [C]
  E* y;            // [B, HW, C]
  float2* partial; // [B, G, chunks]: (sum, sum of squares) of x + add - shift over one row chunk
  int HW, C, G, sv, chunks, rows_per_chunk, silu;   // sv: vectors per channel slice
  float eps;
};

// The value the sums of group g (first channel c) of image b are taken about: the group's first element.  Shifted
// sums keep E[d^2] - E[d]^2 accurate when |mean| >> std, where fp32 E[x^2] - mean^2 cancels.
template <typename E>
__device__ __forceinline__ float gn_shift(const GnParams<E>& p, int b, int c) {
  float s = Elem<E>::to_float(p.x[(size_t)b * p.HW * p.C + c]);
  if (p.add) s += Elem<E>::to_float(p.add[(size_t)b * p.add_bs + c]);
  return s;
}

// 16-byte vectors of rows r, r + rpp, r + 2 rpp, r + 3 rpp of one column (zero at and past r1): four loads in flight.
__device__ __forceinline__ void gn_load4(uint4 (&xv)[4], const uint4* col, int stride_vec, int r, int rpp, int r1) {
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int rr = r + u * rpp;
    xv[u] = rr < r1 ? __ldg(col + (size_t)rr * stride_vec) : make_uint4(0, 0, 0, 0);
  }
}

// pass 1: grid (row chunk, channel slice, image).  Per-thread column sums -> shared memory -> one warp per group
// reduces its rpp x C/G values (lanes in a fixed stride, then a shuffle tree) -> partial[b, g, chunk].
template <typename E>
__global__ void __launch_bounds__(1024) gn_stats_kernel(GnParams<E> p) {
  using X = Elem<E>;
  using E2 = typename X::E2;
  // let the apply pass (launched as a programmatic dependent) start its prologue; it waits for this grid's
  // completion before it reads the partials
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  extern __shared__ float sm[];   // [64] group shifts, then [2][rpp][sv * 8] per-thread channel sums
  const int cg = p.C / p.G, sv = p.sv, rpp = blockDim.x / sv, b = blockIdx.z;
  const int v0 = blockIdx.y * sv, nv = min(sv, (p.C >> 3) - v0);   // the last slice may be narrower
  const int c0 = v0 * 8, ng = nv * 8 / cg;
  const int v = threadIdx.x % sv, rl = threadIdx.x / sv;
  const bool lane_on = rl < rpp && v < nv;
  const int r0 = blockIdx.x * p.rows_per_chunk;
  const int r1 = lane_on ? min(p.HW, r0 + p.rows_per_chunk) : r0;
  const uint4* col = reinterpret_cast<const uint4*>(p.x + (size_t)b * p.HW * p.C + c0) + v;
  const int stride_vec = p.C >> 3;
  uint4 xv[4];
  gn_load4(xv, col, stride_vec, r0 + rl, rpp, r1);
  float* s_shift = sm;
  float* ss = sm + 64;
  float* sq = ss + rpp * sv * 8;
  if (threadIdx.x < ng) s_shift[threadIdx.x] = gn_shift(p, b, c0 + threadIdx.x * cg);
  float o[8], s[8], q[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { o[i] = 0.f; s[i] = 0.f; q[i] = 0.f; }
  if (p.add && lane_on) {
    const uint4 av = __ldg(reinterpret_cast<const uint4*>(p.add + (size_t)b * p.add_bs + c0) + v);
    const E2* ah = reinterpret_cast<const E2*>(&av);
#pragma unroll
    for (int i = 0; i < 4; ++i) { const float2 f = X::to_float2(ah[i]); o[2 * i] = f.x; o[2 * i + 1] = f.y; }
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i] -= s_shift[(v * 8 + i) / cg];   // < 64 for every thread: sv * 8 / cg <= G
  for (int r = r0 + rl; r < r1; r += 4 * rpp) {
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (r + u * rpp < r1) {
        const E2* xh = reinterpret_cast<const E2*>(&xv[u]);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = X::to_float2(xh[i]);
          const float d0 = f.x + o[2 * i], d1 = f.y + o[2 * i + 1];
          s[2 * i] += d0; q[2 * i] = fmaf(d0, d0, q[2 * i]);
          s[2 * i + 1] += d1; q[2 * i + 1] = fmaf(d1, d1, q[2 * i + 1]);
        }
      }
    }
    if (r + 4 * rpp < r1) gn_load4(xv, col, stride_vec, r + 4 * rpp, rpp, r1);
  }
  const int w8 = sv * 8;
  if (lane_on) {
#pragma unroll
    for (int i = 0; i < 8; ++i) { ss[rl * w8 + v * 8 + i] = s[i]; sq[rl * w8 + v * 8 + i] = q[i]; }
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5, n = rpp * cg;
  for (int lg = warp; lg < ng; lg += nwarps) {
    float ts = 0.f, tq = 0.f;
    for (int j = lane; j < n; j += 32) {
      const int r = j / cg, c = lg * cg + (j - r * cg);
      ts += ss[r * w8 + c]; tq += sq[r * w8 + c];
    }
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) {
      ts += __shfl_xor_sync(0xffffffffu, ts, m);
      tq += __shfl_xor_sync(0xffffffffu, tq, m);
    }
    if (lane == 0) p.partial[((size_t)b * p.G + c0 / cg + lg) * p.chunks + blockIdx.x] = make_float2(ts, tq);
  }
}

// pass 2: y = act((x + add - mean) * rstd * gamma + beta).  grid (row blocks, channel slice, image), the stats pass's
// block shape, rows_per_block <= 4 rpp.  Launched as a programmatic dependent of the stats grid: a thread first
// loads its (up to) four rows of one column, all in flight, and its gamma / beta / add, which overlaps the stats
// grid's tail; after the grid-dependency wait, segments of L lanes (one per group of the slice) fold the group's chunk
// partials in a fixed order (every block of the slice computes the same bits); then it writes its rows.
template <typename E>
__global__ void __launch_bounds__(1024) gn_apply_kernel(GnParams<E> p, int rows_per_block) {
  using X = Elem<E>;
  using E2 = typename X::E2;
  __shared__ float3 s_stat[64];   // (shift, E[d], rstd) of the slice's groups: mean = shift + E[d]
  const int cg = p.C / p.G, sv = p.sv, rpp = blockDim.x / sv, b = blockIdx.z;
  const int v0 = blockIdx.y * sv, nv = min(sv, (p.C >> 3) - v0);
  const int c0 = v0 * 8, ng = nv * 8 / cg;
  const int v = threadIdx.x % sv, rl = threadIdx.x / sv;
  const bool lane_on = rl < rpp && v < nv;
  const int r0 = blockIdx.x * rows_per_block;
  const int r1 = lane_on ? min(p.HW, r0 + rows_per_block) : r0;
  const int stride_vec = p.C >> 3;
  const uint4* __restrict__ xcol = reinterpret_cast<const uint4*>(p.x + (size_t)b * p.HW * p.C + c0) + v;
  uint4* __restrict__ ycol = reinterpret_cast<uint4*>(p.y + (size_t)b * p.HW * p.C + c0) + v;
  uint4 xv[4];
  gn_load4(xv, xcol, stride_vec, r0 + rl, rpp, r1);
  float sc[8], sh[8];
  uint4 gv = make_uint4(0, 0, 0, 0), bv = gv, av = gv;
  if (lane_on) {
    gv = __ldg(reinterpret_cast<const uint4*>(p.gamma + c0) + v);
    bv = __ldg(reinterpret_cast<const uint4*>(p.beta + c0) + v);
    if (p.add) av = __ldg(reinterpret_cast<const uint4*>(p.add + (size_t)b * p.add_bs + c0) + v);
  }
  {
    // L lanes per group: a power of two with ng * L <= blockDim.x (>= 4, as ng <= 64), so a segment never
    // straddles a warp; every load of the fold is issued before the first add
    int L = 32;
    while (ng * L > (int)blockDim.x) L >>= 1;
    const int lg = threadIdx.x / L, j = threadIdx.x % L, g = c0 / cg + lg;
    float ts = 0.f, tq = 0.f, shift = 0.f;
    if (lg < ng && j == 0) shift = gn_shift(p, b, g * cg);
    // everything above reads only this GroupNorm's inputs; the partials are the statistics grid's output
    asm volatile("griddepcontrol.wait;" ::: "memory");
    if (lg < ng) {
      const float2* pp = p.partial + ((size_t)b * p.G + g) * p.chunks;
#pragma unroll 4
      for (int c = j; c < p.chunks; c += L) { const float2 t = pp[c]; ts += t.x; tq += t.y; }
    }
    for (int m = L >> 1; m > 0; m >>= 1) {
      ts += __shfl_xor_sync(0xffffffffu, ts, m);
      tq += __shfl_xor_sync(0xffffffffu, tq, m);
    }
    if (lg < ng && j == 0) {
      const float n = (float)p.HW * (float)cg;
      const float dm = ts / n;
      float var = tq / n - dm * dm;
      var = var < 0.f ? 0.f : var;
      s_stat[lg] = make_float3(shift, dm, rsqrtf(var + p.eps));
    }
  }
  __syncthreads();
  {
    const E* gh = reinterpret_cast<const E*>(&gv);
    const E* bh = reinterpret_cast<const E*>(&bv);
    const E* ah = reinterpret_cast<const E*>(&av);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      // add - mean as (add - shift) - E[d]: no fp32 rounding of the mean itself, which would err by 2^-24 |mean| where
      // |add| >> std and rstd multiplies that by up to 1 / sqrt(eps)
      const float3 st = s_stat[(v * 8 + i) / cg];
      sc[i] = st.z * X::to_float(gh[i]);
      sh[i] = X::to_float(bh[i]) + ((X::to_float(ah[i]) - st.x) - st.y) * sc[i];
    }
  }
  const int r = r0 + rl;
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    if (r + u * rpp >= r1) break;
    const E2* xh = reinterpret_cast<const E2*>(&xv[u]);
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
    ycol[(size_t)(r + u * rpp) * stride_vec] = *reinterpret_cast<const uint4*>(o);
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

// GroupNorm's work split over one image: a function of (HW, C, G) only.
constexpr int kGnMaxChunks = 64;             // row chunks of the statistics pass, at most (and at most HW)
constexpr int kGnStatBlocksPerImage = 128;   // two images fill the H100's 132 SMs about twice
struct GnSplit {
  int sv;              // vectors per channel slice: whole lcm(8, C/G)-channel units, about 32 vectors
  int slices;          // channel slices (the last may be narrower)
  int threads, rpp;    // threads per block (a multiple of 32, >= 256) and row lanes: threads / sv
  int chunks, rows_per_chunk;
};
inline GnSplit gn_split(int HW, int C, int G) {
  GnSplit s;
  const int cg = C / G, nvec = C >> 3;
  int gcd = cg, t = 8;
  while (t) { const int r = gcd % t; gcd = t; t = r; }
  const int uv = cg / gcd;                          // vectors per unit: lcm(8, cg) / 8
  const int nunits = nvec / uv, want = (nvec + 31) / 32;
  const int per_slice = (nunits + want - 1) / want;
  s.sv = per_slice * uv;
  s.slices = (nunits + per_slice - 1) / per_slice;
  s.threads = s.sv > 256 ? (s.sv + 31) / 32 * 32 : 256;
  s.rpp = s.threads / s.sv;
  int chunks = (kGnStatBlocksPerImage + s.slices - 1) / s.slices;
  const int most = (HW + s.rpp - 1) / s.rpp;
  chunks = chunks < most ? chunks : most;
  chunks = chunks < kGnMaxChunks ? chunks : kGnMaxChunks;
  s.rows_per_chunk = (HW + chunks - 1) / chunks;
  s.chunks = (HW + s.rows_per_chunk - 1) / s.rows_per_chunk;
  return s;
}
}  // namespace uops
}  // namespace pww
