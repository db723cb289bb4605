// The canvas side of a MultiDiffusion step (pww_window_input / pww_window_update): overlapping window x window
// crops of one canvas latent [1, 4, H, W] go through the UNet as a batch, and every canvas value averages the guided
// outputs of the windows that cover it before the sampler's step form runs on the canvas.
//
// Window v = iy * n_cols + ix has its origin at (rows[iy], cols[ix]).  A column start with cols[ix] + window > W
// wraps: window column x reads canvas column (cols[ix] + x) mod W (circular panoramas).  Rows never wrap.
//
// The update's arithmetic, fp32 with explicit round-to-nearest intrinsics, per canvas value with the covering
// windows v1 < v2 < ... < vc:
//   g_v = eps_u,v + gs (eps_c,v - eps_u,v)        cfg's ops, at the window-local position
//   E   = g_v1;  E = E + g_v2;  ...;  E = E + g_vc
//   e   = E / c
// then step_form on (x, e) with m = 1.  One thread owns each canvas value, so the result does not depend on how the
// windows are split into chunks.
#pragma once
#include "sampler_step.cuh"

namespace pww {
namespace smp {

constexpr int kMaxWindowChunks = 64;

struct WindowInputArgs {
  const float* lat;                     // [1, 4, H, W] fp32 canvas
  const float* scale;                   // [1] 1/sqrt(sigma^2 + 1)
  const int* rows;                      // [n_rows] window row starts
  const int* cols;                      // [n_cols] window column starts
  void* out;                            // [2n, 4, window, window] contiguous, UNet dtype
  int n_cols, first, n, window, H, W;
};

struct WindowArgs {
  const int* rows;                      // [n_rows]
  const int* cols;                      // [n_cols]
  int n_rows, n_cols, window;
  int per_chunk, views;                 // windows per chunk (the last chunk may hold fewer), windows in all
  int64_t e_sn, e_sc, e_sh, e_sw;       // the window outputs' element strides
};

// The UNet outputs of the chunks: chunk k's [2 n_k, 4, window, window] holds its windows' cond rows, then their
// uncond rows.  Passed by value, so a captured CUDA graph carries the table.
struct WindowOutputs {
  const void* eps[kMaxWindowChunks];
};

// One thread per (window, channel, PX consecutive window pixels); writes the value to rows j and n + j.
template <typename T, int PX>
__global__ void __launch_bounds__(kThreads) window_input_kernel(const WindowInputArgs a) {
  const int ww = a.window * a.window, groups = ww / PX;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)a.n * 4 * groups) return;
  const int jc = (int)(idx / groups);
  const int j = jc >> 2, c = jc & 3;
  const int q = (int)(idx - (int64_t)jc * groups) * PX;
  const int ly = q / a.window, lx = q - ly * a.window;
  const int view = a.first + j;
  const int iy = view / a.n_cols, ix = view - iy * a.n_cols;
  const int y = __ldg(a.rows + iy) + ly, x0 = __ldg(a.cols + ix) + lx;
  const float* src = a.lat + ((int64_t)c * a.H + y) * a.W;
  const float s = __ldg(a.scale);
  float v[PX];
#pragma unroll
  for (int k = 0; k < PX; ++k) {
    int x = x0 + k;
    if (x >= a.W) x -= a.W;                       // start < W and window <= W: one wrap at most
    v[k] = __fmul_rn(__ldg(src + x), s);
  }
  T* out = static_cast<T*>(a.out);
  store_out<T, PX>(out + ((int64_t)j * 4 + c) * ww + q, v);
  store_out<T, PX>(out + ((int64_t)(j + a.n) * 4 + c) * ww + q, v);
}

// One thread per PX consecutive canvas pixels of one row, all 4 channels.  `a` describes the canvas (m = 1, h = H,
// w = W, the latents, history, noise, guidance scale and step rows).
template <typename T, int PX, bool CL>
__global__ void __launch_bounds__(kThreads) window_update_kernel(const UpdateArgs a, const WindowArgs v,
                                                                  const WindowOutputs t) {
  const int hw = a.h * a.w, groups = hw / PX;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= groups) return;
  const int p0 = idx * PX, y = p0 / a.w, x0 = p0 - y * a.w;
  const float g = __ldg(a.gscale);
  float eg[4][PX];
#pragma unroll
  for (int j = 0; j < PX; ++j) {
    float e[4] = {0.f, 0.f, 0.f, 0.f};
    int cnt = 0;
    for (int iy = 0; iy < v.n_rows; ++iy) {
      const int ly = y - __ldg(v.rows + iy);
      if (ly < 0 || ly >= v.window) continue;
      for (int ix = 0; ix < v.n_cols; ++ix) {
        int lx = x0 + j - __ldg(v.cols + ix);
        if (lx < 0) lx += a.w;
        if (lx >= v.window) continue;
        const int view = iy * v.n_cols + ix, chunk = view / v.per_chunk, k = view - chunk * v.per_chunk;
        const int n = min(v.per_chunk, v.views - chunk * v.per_chunk);
        const T* base = static_cast<const T*>(t.eps[chunk]);
        float ec[4][1], eu[4][1];
        load_eps<T, 1, CL>(base + (int64_t)k * v.e_sn, v.e_sc, v.e_sh, v.e_sw, v.window, ly * v.window + lx, ec);
        load_eps<T, 1, CL>(base + (int64_t)(k + n) * v.e_sn, v.e_sc, v.e_sh, v.e_sw, v.window, ly * v.window + lx, eu);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const float gv = cfg(g, ec[c][0], eu[c][0]);
          e[c] = cnt == 0 ? gv : __fadd_rn(e[c], gv);
        }
        ++cnt;
      }
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) eg[c][j] = __fdiv_rn(e[c], (float)cnt);
  }
  step_form<PX, false>(a, BlendArgs{}, 0, p0, 1, hw, eg);
}

template <typename T>
cudaError_t launch_window_input(const WindowInputArgs& a, bool px4, cudaStream_t s) {
  const int64_t n = (int64_t)a.n * 4 * a.window * a.window;
  if (px4) window_input_kernel<T, 4><<<blocks_for(n / 4), kThreads, 0, s>>>(a);
  else window_input_kernel<T, 1><<<blocks_for(n), kThreads, 0, s>>>(a);
  return cudaGetLastError();
}

template <typename T>
cudaError_t launch_window_update(const UpdateArgs& a, const WindowArgs& v, const WindowOutputs& t, bool px4, bool cl,
                                 cudaStream_t s) {
  return with_layout(px4, cl, [&](auto px, auto c) {
    window_update_kernel<T, px, c><<<blocks_for((int64_t)a.h * a.w / px), kThreads, 0, s>>>(a, v, t);
    return cudaGetLastError();
  });
}

}  // namespace smp
}  // namespace pww
