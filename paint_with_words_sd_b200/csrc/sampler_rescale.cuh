// Guidance rescale inside the sampler update (pww_sampler_update_rescale): diffusers' `rescale_noise_cfg` (Lin et al.
// 2023, "Common Diffusion Noise Schedules and Sample Steps are Flawed", section 3.4), per image i with phi_i in [0, 1]:
//   cfg   = out_u + g_i (out_c - out_u)                          (as in pww_sampler_update)
//   k_i   = phi_i std(out_c) / std(cfg) + (1 - phi_i)            unbiased std over the 4 h w values of image i
//   out'  = k_i cfg,  then pww_sampler_update's step form on out'
// The std needs the whole image before any of its latents can be updated, so an image is one thread-block cluster of
// up to 8 CTAs (the portable size) of 512 threads: 4096 threads, one 4-pixel group each up to 128x128 latents.  The
// group a thread owns first stays in registers over the three passes (the mean, the sum of squared deviations, the
// update); further groups of larger latents are recomputed from the UNet output (L2-resident at these sizes).
// Every partial is folded in a fixed order (a shuffle tree per warp, the warps in order, the CTAs in rank order through
// distributed shared memory), and the cluster size and the thread -> pixel map depend only on h and w: an image gets
// the same bits alone, in any batch and at any position.
#pragma once
#include <cooperative_groups.h>

#include "sampler_step.cuh"

namespace pww {
namespace smp {

constexpr int kRescaleThreads = 512;
constexpr int kRescaleMaxCluster = 8;

struct RescaleArgs {
  const float* phi;                     // [m] guidance rescale per image
  float* stats;                         // [m, 3] (std_cond, std_cfg, k), or NULL
};

template <int PX>
__device__ __forceinline__ void add_values(const float (&c)[4][PX], const float (&f)[4][PX], float2& s) {
#pragma unroll
  for (int ch = 0; ch < 4; ++ch)
#pragma unroll
    for (int j = 0; j < PX; ++j) {
      s.x = __fadd_rn(s.x, c[ch][j]);
      s.y = __fadd_rn(s.y, f[ch][j]);
    }
}

template <int PX>
__device__ __forceinline__ void add_squared_deviations(const float (&c)[4][PX], const float (&f)[4][PX], float2 mean,
                                                       float2& s) {
#pragma unroll
  for (int ch = 0; ch < 4; ++ch)
#pragma unroll
    for (int j = 0; j < PX; ++j) {
      const float dc = __fsub_rn(c[ch][j], mean.x), df = __fsub_rn(f[ch][j], mean.y);
      s.x = __fadd_rn(s.x, __fmul_rn(dc, dc));
      s.y = __fadd_rn(s.y, __fmul_rn(df, df));
    }
}

// The cluster-wide sum of every thread's v, the same bits in every thread.  `slot` is this CTA's partial: the other
// CTAs read it after the cluster barrier here, so it is not rewritten, and the CTA does not exit, before a later one.
__device__ __forceinline__ float2 cluster_sum(float2 v, float2* warp_part, float2* slot,
                                              const cooperative_groups::cluster_group& cl) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    v.x = __fadd_rn(v.x, __shfl_xor_sync(0xffffffffu, v.x, o));
    v.y = __fadd_rn(v.y, __shfl_xor_sync(0xffffffffu, v.y, o));
  }
  if ((threadIdx.x & 31) == 0) warp_part[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    float2 t = warp_part[0];
    for (int w = 1; w < kRescaleThreads / 32; ++w) {
      t.x = __fadd_rn(t.x, warp_part[w].x);
      t.y = __fadd_rn(t.y, warp_part[w].y);
    }
    *slot = t;
  }
  cl.sync();
  float2 t = *cl.map_shared_rank(slot, 0);
  for (unsigned r = 1; r < cl.num_blocks(); ++r) {
    const float2 p = *cl.map_shared_rank(slot, r);
    t.x = __fadd_rn(t.x, p.x);
    t.y = __fadd_rn(t.y, p.y);
  }
  return t;
}

// out' = k cfg (phi == 0: cfg itself, k never applied), then step_form on the 4 channels of pixels
// p0 .. p0 + PX - 1 of image i.
template <int PX, bool BLEND>
__device__ __forceinline__ void rescaled_update(const UpdateArgs& a, const BlendArgs& bl, int i, int p0,
                                                float (&eg)[4][PX], float phi, float k) {
  if (phi != 0.f) {
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
      for (int j = 0; j < PX; ++j) eg[c][j] = __fmul_rn(k, eg[c][j]);
  }
  step_form<PX, BLEND>(a, bl, i, p0, a.m, a.h * a.w, eg);
}

// One cluster per image; thread t of CTA rank r owns the PX-pixel groups r * 512 + t + k * (cluster size * 512).
// `bl` is read only by the BLEND instances.
template <typename T, int PX, bool CL, bool BLEND>
__global__ void __launch_bounds__(kRescaleThreads, 1) sampler_update_rescale_kernel(const UpdateArgs a,
                                                                                    const RescaleArgs r,
                                                                                    const BlendArgs bl) {
  namespace cg = cooperative_groups;
  const cg::cluster_group cl = cg::this_cluster();
  __shared__ float2 warp_part[kRescaleThreads / 32];
  __shared__ float2 slots[2];
  const int cs = (int)cl.num_blocks();
  const int i = (int)(blockIdx.x / cs);
  const int hw = a.h * a.w, groups = hw / PX, stride = cs * kRescaleThreads;
  const int g0 = (int)cl.block_rank() * kRescaleThreads + (int)threadIdx.x;
  const bool own = g0 < groups;
  const float n = (float)(4 * hw);
  float c0[4][PX], f0[4][PX];

  // pass 1: the means of out_c and cfg
  float2 s = make_float2(0.f, 0.f);
  if (own) {
    cond_and_cfg<T, PX, CL>(a, i, g0 * PX, c0, f0);
    add_values<PX>(c0, f0, s);
  }
  for (int g = g0 + stride; g < groups; g += stride) {
    float c[4][PX], f[4][PX];
    cond_and_cfg<T, PX, CL>(a, i, g * PX, c, f);
    add_values<PX>(c, f, s);
  }
  const float2 sum = cluster_sum(s, warp_part, &slots[0], cl);
  const float2 mean = make_float2(__fdiv_rn(sum.x, n), __fdiv_rn(sum.y, n));

  // pass 2: the sums of squared deviations from them
  float2 d = make_float2(0.f, 0.f);
  if (own) add_squared_deviations<PX>(c0, f0, mean, d);
  for (int g = g0 + stride; g < groups; g += stride) {
    float c[4][PX], f[4][PX];
    cond_and_cfg<T, PX, CL>(a, i, g * PX, c, f);
    add_squared_deviations<PX>(c, f, mean, d);
  }
  const float2 ss = cluster_sum(d, warp_part, &slots[1], cl);
  const float std_c = __fsqrt_rn(__fdiv_rn(ss.x, __fsub_rn(n, 1.f)));
  const float std_f = __fsqrt_rn(__fdiv_rn(ss.y, __fsub_rn(n, 1.f)));
  const float phi = __ldg(r.phi + i);
  const float k = __fadd_rn(__fmul_rn(phi, __fdiv_rn(std_c, std_f)), __fsub_rn(1.f, phi));
  if (r.stats != nullptr && cl.block_rank() == 0 && threadIdx.x == 0) {
    r.stats[3 * i + 0] = std_c;
    r.stats[3 * i + 1] = std_f;
    r.stats[3 * i + 2] = phi == 0.f ? 1.f : k;
  }

  // pass 3: the update
  if (own) rescaled_update<PX, BLEND>(a, bl, i, g0 * PX, f0, phi, k);
  for (int g = g0 + stride; g < groups; g += stride) {
    float c[4][PX], f[4][PX];
    cond_and_cfg<T, PX, CL>(a, i, g * PX, c, f);
    rescaled_update<PX, BLEND>(a, bl, i, g * PX, f, phi, k);
  }
  cl.sync();      // the other CTAs have read slots[1]
}

// CTAs per image: the smallest power of two (at most 8) whose threads cover the image's PX-pixel groups once.
inline int rescale_cluster_size(int64_t groups) {
  int cs = 1;
  while (cs < kRescaleMaxCluster && (int64_t)cs * kRescaleThreads < groups) cs *= 2;
  return cs;
}

template <typename T, int PX, bool CL, bool BLEND>
cudaError_t launch_rescale_instance(const UpdateArgs& a, const RescaleArgs& r, const BlendArgs& bl, cudaStream_t s) {
  const int cs = rescale_cluster_size((int64_t)a.h * a.w / PX);
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)(a.m * cs));
  cfg.blockDim = dim3(kRescaleThreads);
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cs;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, sampler_update_rescale_kernel<T, PX, CL, BLEND>, a, r, bl);
}

template <typename T, bool BLEND>
cudaError_t launch_update_rescale(const UpdateArgs& a, const RescaleArgs& r, const BlendArgs& bl, bool px4, bool cl,
                                  cudaStream_t s) {
  return with_layout(px4, cl, [&](auto px, auto c) { return launch_rescale_instance<T, px, c, BLEND>(a, r, bl, s); });
}

}  // namespace smp
}  // namespace pww
