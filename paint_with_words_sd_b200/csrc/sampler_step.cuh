// The sampler step around the UNet (pww_sampler_input / pww_sampler_update): the scaled, CFG-doubled UNet input, and
// the CFG combine + one linear step form that LMS, Euler, Euler ancestral and DPM++ 2M fill with their own coefficients.
//
// Every scalar that changes per step is read from device memory (a captured CUDA graph replays with new values), and
// all arithmetic is fp32 with explicit round-to-nearest intrinsics in the order of the step form, so nvcc cannot
// contract a multiply and an add into an FMA:
//   eps    = eps_u + g_i (eps_c - eps_u)
//   q      = a x + b eps                          (a == 0: q = b eps)
//   x_next = alpha x + (beta0 q + beta1 h1 + ...)  (alpha == 1: x + (...))   [+ gamma z when gamma != 0 and z exists]
// The BLEND instances (pww_sampler_update_masked) then put the area outside the mask M back on the init latents'
// noise path at the next sigma (masked img2img):
//   x_next = M x_next + (1 - M) (init + z0 sigma')
#pragma once
#include <type_traits>

#include "pww_common.cuh"

namespace pww {
namespace smp {

constexpr int kThreads = 256;

// form[] columns (pipeline.FORM_COLUMNS): alpha, a, b, gamma, history slot, noise row
struct UpdateArgs {
  const void* eps;                      // [2m, 4, h, w] UNet output: cond rows 0..m-1, uncond rows m..2m-1
  int64_t e_sn, e_sc, e_sh, e_sw;       // its element strides
  float* lat;                           // [m, 4, h, w] fp32, updated in place
  float* hist;                          // [nh, m, 4, h, w] ring of step-form entries
  const float* noise;                   // [n, m, 4, h, w] per-step noise rows, or NULL
  const float* gscale;                  // [m] guidance scale per image
  const float* beta;                    // [4]
  const float* form;                    // [6]
  int m, h, w, nh;
};

// The masked instances' extra inputs.  A separate kernel parameter after the existing ones, not UpdateArgs fields, so
// the parameter offsets, and with them the code, of the unmasked instances stay as they are.
struct BlendArgs {
  const float* init;                    // [m, 4, h, w] the init image's latents
  const float* noise0;                  // [m, 4, h, w] the noise that made the start latents init + sigma0 noise0
  const float* mask;                    // [m, 1, h, w] in [0, 1], 1 = repaint
  const float* sigma_next;              // [1] the next step's sigma (0 after the last step)
};

struct InputArgs {
  const float* lat;                     // [m, 4, h, w] fp32
  const float* scale;                   // [1] 1/sqrt(sigma^2 + 1)
  const float* extra;                   // [m, C - 4, h, w] fp32 (inpaint mask + masked-image latents), or NULL
  void* out;                            // [2m, C, h, w] contiguous, UNet dtype
  int m, C, hw;
};

// T = float, __half or __nv_bfloat16 (the UNet's dtype)
template <typename T>
__device__ __forceinline__ float to_f(T v) {
  if constexpr (sizeof(T) == 4) return v;
  else return Elem<T>::to_float(v);
}

// Two 2-byte elements packed in one 32-bit word.
template <typename T>
__device__ __forceinline__ float2 pair_to_f2(unsigned u) {
  typename Elem<T>::E2 h;
  memcpy(&h, &u, sizeof(h));
  return Elem<T>::to_float2(h);
}

// PX consecutive fp32 values (PX = 4: one 16-byte access).
template <int PX>
__device__ __forceinline__ void load_px(const float* p, float (&v)[PX]) {
  if constexpr (PX == 4) {
    const float4 t = *reinterpret_cast<const float4*>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  } else {
    v[0] = *p;
  }
}
template <int PX>
__device__ __forceinline__ void store_px(float* p, const float (&v)[PX]) {
  if constexpr (PX == 4) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  } else {
    *p = v[0];
  }
}

// e[c][j] = channel c of pixel p0 + j of one image's eps, whose rows are w pixels wide.  CL: channels-last packed rows
// (pixel p's 4 channels at 4p .. 4p+3), read with 8- or 16-byte accesses; otherwise one strided load per element, with
// the channel, row and column strides sc, sh and sw.
template <typename T, int PX, bool CL>
__device__ __forceinline__ void load_eps(const T* base, int64_t sc, int64_t sh, int64_t sw, int w, int p0,
                                         float (&e)[4][PX]) {
  if constexpr (CL && sizeof(T) == 4) {
    const float4* s = reinterpret_cast<const float4*>(base + (int64_t)p0 * 4);
#pragma unroll
    for (int j = 0; j < PX; ++j) {
      const float4 t = __ldg(s + j);
      e[0][j] = t.x; e[1][j] = t.y; e[2][j] = t.z; e[3][j] = t.w;
    }
  } else if constexpr (CL && PX == 4) {
    const uint4* s = reinterpret_cast<const uint4*>(base + (int64_t)p0 * 4);
#pragma unroll
    for (int k = 0; k < 2; ++k) {                 // one 16-byte access = two pixels
      const uint4 t = __ldg(s + k);
      const float2 a0 = pair_to_f2<T>(t.x), a1 = pair_to_f2<T>(t.y), b0 = pair_to_f2<T>(t.z), b1 = pair_to_f2<T>(t.w);
      e[0][2 * k] = a0.x; e[1][2 * k] = a0.y; e[2][2 * k] = a1.x; e[3][2 * k] = a1.y;
      e[0][2 * k + 1] = b0.x; e[1][2 * k + 1] = b0.y; e[2][2 * k + 1] = b1.x; e[3][2 * k + 1] = b1.y;
    }
  } else if constexpr (CL) {                      // 2-byte types, one pixel: one 8-byte access
    const uint2 t = __ldg(reinterpret_cast<const uint2*>(base + (int64_t)p0 * 4));
    const float2 a0 = pair_to_f2<T>(t.x), a1 = pair_to_f2<T>(t.y);
    e[0][0] = a0.x; e[1][0] = a0.y; e[2][0] = a1.x; e[3][0] = a1.y;
  } else {
#pragma unroll
    for (int j = 0; j < PX; ++j) {
      const int p = p0 + j, y = p / w, x = p - y * w;
      const T* px = base + y * sh + x * sw;
#pragma unroll
      for (int c = 0; c < 4; ++c) e[c][j] = to_f(px[c * sc]);
    }
  }
}

// The CFG combine of one value: eps_u + g (eps_c - eps_u).
__device__ __forceinline__ float cfg(float g, float ec, float eu) {
  return __fadd_rn(eu, __fmul_rn(g, __fsub_rn(ec, eu)));
}

// c = eps_c and f = the guided eps of image i at pixels p0 .. p0 + PX - 1.
template <typename T, int PX, bool CL>
__device__ __forceinline__ void cond_and_cfg(const UpdateArgs& a, int i, int p0, float (&c)[4][PX],
                                             float (&f)[4][PX]) {
  const T* eps = static_cast<const T*>(a.eps);
  const float g = __ldg(a.gscale + i);
  load_eps<T, PX, CL>(eps + (int64_t)i * a.e_sn, a.e_sc, a.e_sh, a.e_sw, a.w, p0, c);
  load_eps<T, PX, CL>(eps + (int64_t)(i + a.m) * a.e_sn, a.e_sc, a.e_sh, a.e_sw, a.w, p0, f);
#pragma unroll
  for (int ch = 0; ch < 4; ++ch)
#pragma unroll
    for (int j = 0; j < PX; ++j) f[ch][j] = cfg(g, c[ch][j], f[ch][j]);
}

// The masked instances' epilogue on one channel's PX values x of the step's result, at element offset `off`:
//   x = M x + (1 - M) (init + z0 sigma')         mk: the pixels' mask values, sn: sigma'
// For M == 1 this is x + 0 = x, for M == 0 it is 0 + (init + z0 sigma') (finite x and init + z0 sigma').
template <int PX>
__device__ __forceinline__ void blend_px(const BlendArgs& bl, int64_t off, const float (&mk)[PX], float sn,
                                         float (&x)[PX]) {
  float x0[PX], z0[PX];
  load_px<PX>(bl.init + off, x0);
  load_px<PX>(bl.noise0 + off, z0);
#pragma unroll
  for (int j = 0; j < PX; ++j)
    x[j] = __fadd_rn(__fmul_rn(mk[j], x[j]), __fmul_rn(__fsub_rn(1.f, mk[j]), __fadd_rn(x0[j], __fmul_rn(z0[j], sn))));
}

// The step form, shared by the plain, rescale and panorama updates, on the guided eps eg of image i at pixels
// p0 .. p0 + PX - 1 (m images of hw pixels in a history entry / noise row): writes the history entry, then the latents,
// with the BLEND instances' mask blend before the store.  `bl` is read only by the BLEND instances.
template <int PX, bool BLEND>
__device__ __forceinline__ void step_form(const UpdateArgs& a, const BlendArgs& bl, int i, int p0, int m, int hw,
                                          const float (&eg)[4][PX]) {
  float mk[PX], sn = 0.f;
  if constexpr (BLEND) {
    load_px<PX>(bl.mask + (int64_t)i * hw + p0, mk);
    sn = __ldg(bl.sigma_next);
  }
  const float alpha = __ldg(a.form + 0), ca = __ldg(a.form + 1), cb = __ldg(a.form + 2), gamma = __ldg(a.form + 3);
  const int slot = (int)__ldg(a.form + 4), row = (int)__ldg(a.form + 5);
  const float b0 = __ldg(a.beta + 0);
  const bool with_noise = a.noise != nullptr && gamma != 0.f;
  const int64_t entry = (int64_t)m * 4 * hw;   // elements of one history entry / noise row
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const int64_t off = ((int64_t)i * 4 + c) * hw + p0;
    float x[PX], q[PX], s[PX];
    load_px<PX>(a.lat + off, x);
#pragma unroll
    for (int j = 0; j < PX; ++j) {
      const float e = eg[c][j];
      q[j] = ca == 0.f ? __fmul_rn(cb, e) : __fadd_rn(__fmul_rn(ca, x[j]), __fmul_rn(cb, e));
      s[j] = __fmul_rn(b0, q[j]);
    }
    store_px<PX>(a.hist + slot * entry + off, q);
    for (int k = 1; k < a.nh; ++k) {
      const float bk = __ldg(a.beta + k);
      float hk[PX];
      load_px<PX>(a.hist + ((slot - k + a.nh) % a.nh) * entry + off, hk);
#pragma unroll
      for (int j = 0; j < PX; ++j) s[j] = __fadd_rn(s[j], __fmul_rn(bk, hk[j]));
    }
#pragma unroll
    for (int j = 0; j < PX; ++j) x[j] = alpha == 1.f ? __fadd_rn(x[j], s[j]) : __fadd_rn(__fmul_rn(alpha, x[j]), s[j]);
    if (with_noise) {
      float z[PX];
      load_px<PX>(a.noise + row * entry + off, z);
#pragma unroll
      for (int j = 0; j < PX; ++j) x[j] = __fadd_rn(x[j], __fmul_rn(gamma, z[j]));
    }
    if constexpr (BLEND) blend_px<PX>(bl, off, mk, sn, x);
    store_px<PX>(a.lat + off, x);
  }
}

// One thread per (image, PX consecutive pixels), all 4 channels.  `bl` is read only by the BLEND instances.
template <typename T, int PX, bool CL, bool BLEND>
__global__ void __launch_bounds__(kThreads) sampler_update_kernel(const UpdateArgs a, const BlendArgs bl) {
  const int hw = a.h * a.w, groups = hw / PX;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)a.m * groups) return;
  const int i = (int)(idx / groups);
  const int p0 = (int)(idx - (int64_t)i * groups) * PX;
  float ec[4][PX], eg[4][PX];
  cond_and_cfg<T, PX, CL>(a, i, p0, ec, eg);
  step_form<PX, BLEND>(a, bl, i, p0, a.m, hw, eg);
}

template <typename T, int PX>
__device__ __forceinline__ void store_out(T* p, const float (&v)[PX]) {
  if constexpr (sizeof(T) == 4) {
    store_px<PX>(p, v);
  } else if constexpr (PX == 4) {
    const typename Elem<T>::E2 lo = Elem<T>::from_float2(v[0], v[1]), hi = Elem<T>::from_float2(v[2], v[3]);
    uint2 u;
    memcpy(&u.x, &lo, 4);
    memcpy(&u.y, &hi, 4);
    *reinterpret_cast<uint2*>(p) = u;
  } else {
    *p = Elem<T>::from_float(v[0]);
  }
}

// One thread per (image, channel, PX consecutive pixels); writes the value to the cond row i and the uncond row m + i.
template <typename T, int PX>
__global__ void __launch_bounds__(kThreads) sampler_input_kernel(const InputArgs a) {
  const int groups = a.hw / PX;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)a.m * a.C * groups) return;
  const int ic = (int)(idx / groups);
  const int i = ic / a.C, c = ic - i * a.C;
  const int p0 = (int)(idx - (int64_t)ic * groups) * PX;
  float v[PX];
  if (c < 4) {
    load_px<PX>(a.lat + ((int64_t)i * 4 + c) * a.hw + p0, v);
    const float s = __ldg(a.scale);
#pragma unroll
    for (int j = 0; j < PX; ++j) v[j] = __fmul_rn(v[j], s);
  } else {
    load_px<PX>(a.extra + ((int64_t)i * (a.C - 4) + (c - 4)) * a.hw + p0, v);
  }
  T* out = static_cast<T*>(a.out);
  store_out<T, PX>(out + ((int64_t)i * a.C + c) * a.hw + p0, v);
  store_out<T, PX>(out + ((int64_t)(i + a.m) * a.C + c) * a.hw + p0, v);
}

inline unsigned blocks_for(int64_t threads) { return (unsigned)((threads + kThreads - 1) / kThreads); }

// f(integral_constant<int, PX>{}, bool_constant<CL>{}) for the update kernels' layout: PX = 4 or 1 pixels per thread,
// CL = channels-last packed eps rows or strided.
template <typename F>
cudaError_t with_layout(bool px4, bool cl, F&& f) {
  using P1 = std::integral_constant<int, 1>;
  using P4 = std::integral_constant<int, 4>;
  if (px4) return cl ? f(P4{}, std::true_type{}) : f(P4{}, std::false_type{});
  return cl ? f(P1{}, std::true_type{}) : f(P1{}, std::false_type{});
}

template <typename T, bool BLEND>
cudaError_t launch_update(const UpdateArgs& a, const BlendArgs& bl, bool px4, bool cl, cudaStream_t s) {
  return with_layout(px4, cl, [&](auto px, auto c) {
    sampler_update_kernel<T, px, c, BLEND><<<blocks_for(a.m * (int64_t)a.h * a.w / px), kThreads, 0, s>>>(a, bl);
    return cudaGetLastError();
  });
}

template <typename T>
cudaError_t launch_input(const InputArgs& a, bool px4, cudaStream_t s) {
  const int64_t n = (int64_t)a.m * a.C * a.hw;
  if (px4) sampler_input_kernel<T, 4><<<blocks_for(n / 4), kThreads, 0, s>>>(a);
  else sampler_input_kernel<T, 1><<<blocks_for(n), kThreads, 0, s>>>(a);
  return cudaGetLastError();
}

}  // namespace smp
}  // namespace pww
