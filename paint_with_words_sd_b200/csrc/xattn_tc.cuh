// Paint-with-Words cross-attention on Hopper tensor cores (sm_90a), keys T <= 80 or 2 / 3 CLIP chunks (T = 154, 231):
// the two-launch pair that takes the reference's dense [N, T] fp32 weight map (maps with more than 10 distinct columns
// cannot be packed for the one-launch kernel of xattn_fused2.cuh).  KC = chunks of the key sequence: each chunk is one
// 80-row K / V tile of the stage, and the softmax streams over them (xattn_core.cuh).
//
// Fused region of the reference's inj_forward (paint_with_words.py:87-118), per image b / head h / 128-row tile:
//     statistics kernel:  per-image max / (sum, sumsq) of E(Q_h K_h^T) over all heads, rows and tokens (E = fp16 / bf16)
//     forward kernel:     S = Q_h K_h^T;  P = softmax(scale * (S + g[b] * M_b * w[b]));  O = P V_h
// The statistic kind and g are one value for the launch or one per image (XattnParams::stat_kind, g_stride).
// with the warp-level MMA tiles of xattn_core.cuh.  Work unit = (image, row tile, head); every CTA of the persistent grid
// owns a contiguous range of units and double-buffers them: the cp.async copies of unit i + 1 are in flight while unit i
// is computed.  The forward kernel walks its range in the FwdWalk order, which pairs one image with a weight map and one
// without and alternates their heads, so that every CTA gets the same mix of biased and unbiased units.
#pragma once
#include <cuda.h>
#include <stdio.h>
#include <stdlib.h>

#include "mma_sm90.cuh"
#include "pww_common.cuh"
#include "xattn_core.cuh"

namespace pww {
namespace tc {

constexpr int kBM = core::kBM;   // query rows per tile
constexpr int kTP = core::kTP;   // padded key count
constexpr int kThreads = core::kThreads;
constexpr int kMaxBatch = 256;   // images per launch (the C ABI splits larger batches)
constexpr int kMaxLocal = 4;     // images one CTA's unit range can touch: B/132 + 2 <= 4 for B <= 256

template <int D, int KC = 1>
struct Cfg {
  using T_ = core::Tile<D>;
  static constexpr uint32_t STAGE = T_::QBYTES + 2 * KC * T_::KBYTES;   // Q | K chunks | V chunks of one unit
  // two stages (the copies of unit i + 1 overlap unit i) where they fit; one at the long contexts of head dim 160
  static constexpr int NST = (2 * STAGE <= 232448 - 8192) ? 2 : 1;
  static constexpr uint32_t SMEM = NST * STAGE;
  static_assert(SMEM <= 232448 - 8192, "shared memory budget (dynamic + static tables)");
};

template <typename E>
struct TcParams {
  XattnParams<E> x;
  int tiles;        // row tiles per image
  int units;        // B * tiles * H
};

// Walks consecutive units without a div/mod per step.
struct UnitIter {
  int b, tile, h, tiles, H;
  __device__ __forceinline__ UnitIter(int u, int tiles_, int H_) : tiles(tiles_), H(H_) {
    h = u % H_;
    const int t = u / H_;
    tile = t % tiles_;
    b = t / tiles_;
  }
  __device__ __forceinline__ void next() {
    if (++h == H) {
      h = 0;
      if (++tile == tiles) { tile = 0; ++b; }
    }
  }
};
// Forward-kernel unit order.  Units are tile-major; inside a row tile the images are visited in groups:
//   * pair group: one biased image A (has a weight map) and one unbiased image U (classifier-free guidance puts as many
//     of each in the batch).  2H units, head h = j/2, in the order  U A | A U | U A | ...  so that biased and unbiased
//     units alternate at the finest grain: every CTA's contiguous range gets the same mix, whatever the image order in
//     the batch, and all H heads of A read its row tile of the map while it is in L2.
//   * solo group: an image without a partner (all-biased or all-unbiased batches), H units head-minor.
// s_img lists the biased images first (nb of them), then the unbiased ones.
struct FwdUnit {
  int b, h, tile;
};
// Walks a CTA's contiguous unit range in that order; divisions only in the constructor.
struct FwdWalk {
  int B, H, nb, np, ng;
  const int* img;
  int tile, gi, j;    // row tile, group inside the tile (pair groups first, then solo groups), position in the group
  __host__ __device__ __forceinline__ FwdWalk(int u, int B_, int H_, int nb_, const int* img_) : B(B_), H(H_), nb(nb_), img(img_) {
    const int nu = B - nb;
    np = nb < nu ? nb : nu;
    ng = B - np;
    const int per_tile = B * H;
    tile = u / per_tile;
    int q = u - tile * per_tile;
    if (q < np * 2 * H) {
      gi = q / (2 * H);
      j = q - gi * 2 * H;
    } else {
      q -= np * 2 * H;
      const int solo = q / H;
      gi = np + solo;
      j = q - solo * H;
    }
  }
  __host__ __device__ __forceinline__ void next() {
    const int gsize = gi < np ? 2 * H : H;
    if (++j == gsize) {
      j = 0;
      if (++gi == ng) { gi = 0; ++tile; }
    }
  }
  __host__ __device__ __forceinline__ FwdUnit get() const {
    FwdUnit r;
    r.tile = tile;
    if (gi < np) {
      r.h = j >> 1;
      const int unb = ((j ^ (j >> 1)) & 1) ^ 1;          // 1 = the unbiased image's unit
      r.b = unb ? img[nb + gi] : img[gi];
    } else {
      r.h = j;
      r.b = (2 * nb > B) ? img[gi] : img[nb + gi];       // the biased or the unbiased image without a partner
    }
    return r;
  }
};
__device__ __forceinline__ void cta_range(int units, int& u0, int& u1) {
  u0 = (int)((long long)blockIdx.x * units / gridDim.x);
  u1 = (int)((long long)(blockIdx.x + 1) * units / gridDim.x);
}
template <typename E>
__device__ __forceinline__ int image_widx(const XattnParams<E>& p, int b) {
  if (p.wmap == nullptr) return -1;
  return p.wmap_index ? p.wmap_index[b] : b;
}

// ---------------------------------------------------------------------------------------------------------
// forward kernel
// ---------------------------------------------------------------------------------------------------------
template <int D, int KC, typename E>
__global__ void __launch_bounds__(kThreads, 1) xattn_fwd_kernel(const TcParams<E> tp) {
  using C = core::Tile<D>;
  using CF = Cfg<D, KC>;
  const XattnParams<E>& p = tp.x;
  extern __shared__ __align__(128) unsigned char smem[];
  const uint32_t smem0 = ptx::smem_u32(smem);
  __shared__ int s_img[kMaxBatch];
  __shared__ int s_widx[kMaxBatch];
  __shared__ float s_coef[kMaxBatch];
  __shared__ int s_nb;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 0) {
    // stable partition of the images by "has a weight map"
    int nb_total = 0;
    for (int base = 0; base < p.B; base += 32) {
      const int b = base + lane;
      nb_total += __popc(__ballot_sync(0xffffffffu, b < p.B && image_widx(p, b) >= 0));
    }
    int cb = 0, cu = 0;
    const unsigned lt = (1u << lane) - 1u;
    for (int base = 0; base < p.B; base += 32) {
      const int b = base + lane;
      const bool valid = b < p.B, bi = valid && image_widx(p, b) >= 0;
      const unsigned mb = __ballot_sync(0xffffffffu, bi), mu = __ballot_sync(0xffffffffu, valid && !bi);
      if (bi) s_img[cb + __popc(mb & lt)] = b;
      else if (valid) s_img[nb_total + cu + __popc(mu & lt)] = b;
      cb += __popc(mb);
      cu += __popc(mu);
    }
    if (lane == 0) s_nb = nb_total;
  }
  for (int b = threadIdx.x; b < p.B; b += kThreads) {
    const int wi = image_widx(p, b);
    s_widx[b] = wi;
    s_coef[b] = wi >= 0 ? image_g(p, b) * __ldg(p.stats + b) : 0.f;
  }
  __syncthreads();
  int u0, u1;
  cta_range(tp.units, u0, u1);
  const int n_it = u1 - u0;
  if (n_it <= 0) return;
  const float sl2 = p.scale * 1.4426950408889634f;
  FwdWalk w(u0, p.B, p.H, s_nb, s_img);
  FwdUnit nxt = w.get();
  core::load_operands<D, KC>(smem0, p, nxt.b, nxt.h, nxt.tile, true);
  ptx::cp_async_commit();
  for (int it = 0; it < n_it; ++it) {
    const FwdUnit f = nxt;
    if constexpr (CF::NST == 2) {
      if (it + 1 < n_it) {
        w.next();
        nxt = w.get();
        core::load_operands<D, KC>(smem0 + ((it + 1) & 1) * CF::STAGE, p, nxt.b, nxt.h, nxt.tile, true);
        ptx::cp_async_commit();
        ptx::cp_async_wait<1>();
      } else {
        ptx::cp_async_wait<0>();
      }
    } else {                                       // one stage: refilled once the previous unit is done with it
      if (it > 0) {
        core::load_operands<D, KC>(smem0, p, f.b, f.h, f.tile, true);
        ptx::cp_async_commit();
      }
      ptx::cp_async_wait<0>();
      if (it + 1 < n_it) { w.next(); nxt = w.get(); }
    }
    __syncthreads();
    const uint32_t st = smem0 + (CF::NST == 2 ? (it & 1) : 0) * CF::STAGE;
    const uint32_t qs = st + (uint32_t)(warp * 16 * C::LD) * 2u;
    const int row0 = f.tile * kBM + warp * 16;
    const int widx = s_widx[f.b];
    const int kv = core::chunk_keys<KC>(p.T);
    float o[C::NT][4], m0, m1, l0, l1;
    core::warp_online_begin<D>(o, m0, m1, l0, l1);
#pragma unroll 1
    for (int c = 0; c < KC; ++c) {
      float s[10][4];
      core::warp_qk<D, E>(qs, st + C::QBYTES + c * C::KBYTES, lane, s);
      if (widx >= 0) {
        const float x = s_coef[f.b];
        const float* wm = p.wmap + (int64_t)widx * p.wmap_bs + c * core::kChunk;   // chunk c, slot t = column 77 c + t
#pragma unroll
        for (int j = 0; j < 10; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int t = core::tok(j, e, lane), r = row0 + (lane >> 2) + (e >> 1) * 8;
            if (t < kv && r < p.N) s[j][e] = fmaf(x, __ldg(wm + (int64_t)r * p.T + t), s[j][e]);
          }
      }
      core::warp_online_chunk<D, E>(s, kv, sl2, st + C::QBYTES + (KC + c) * C::KBYTES, lane, o, m0, m1, l0, l1);
    }
    core::warp_online_end<D>(o, l0, l1);
    core::warp_store<D>(o, smem + (st - smem0) + warp * 16 * C::LD * 2, lane, p.out + (int64_t)f.b * p.o_bs + f.h * D, p.o_rs, row0, p.N);
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------------------
// statistics kernel: per-image max / (sum, sumsq) of E(S) over all heads, rows and tokens
// ---------------------------------------------------------------------------------------------------------
template <int D, int KC, typename E>
__global__ void __launch_bounds__(kThreads, 1) xattn_stats_kernel(const TcParams<E> tp) {
  using C = core::Tile<D>;
  using CF = Cfg<D, KC>;
  const XattnParams<E>& p = tp.x;
  extern __shared__ __align__(128) unsigned char smem[];
  const uint32_t smem0 = ptx::smem_u32(smem);
  __shared__ StatPartial s_part[core::kWarps][kMaxLocal];     // [warp][local image]
  __shared__ unsigned char s_skip[kMaxBatch];
  __shared__ bool s_ismax[kMaxBatch];                           // statistic kind per image
  __shared__ int is_last;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int u0, u1;
  cta_range(tp.units, u0, u1);
  const int n_it = u1 - u0;
  const int upi = tp.tiles * p.H;                               // units per image
  const int b_first = n_it > 0 ? u0 / upi : 0;
  for (int b = threadIdx.x; b < p.B; b += kThreads) {
    s_skip[b] = (p.wmap_index != nullptr && p.wmap_index[b] < 0) ? 1 : 0;
    s_ismax[b] = s_skip[b] ? true : image_is_max(p, b);        // skipped images: their kind is never read
  }
  if (threadIdx.x < core::kWarps * kMaxLocal) {
    StatPartial sp;
    sp.vmax = -INFINITY; sp.sum = 0.0; sp.sumsq = 0.0; sp.pad = 0.0;
    s_part[threadIdx.x / kMaxLocal][threadIdx.x % kMaxLocal] = sp;
  }
  __syncthreads();
  auto skip = [&](int b) { return s_skip[b] != 0; };
  {
    float vmax = -INFINITY;
    double dsum = 0.0, dsq = 0.0;
    int cur_b = -1;
    auto flush = [&]() {
      if (cur_b < 0) return;
      double m = vmax, a = dsum, q = dsq;
      core::warp_reduce_stat(m, a, q);
      if (lane == 0) {
        StatPartial sp;
        sp.vmax = m; sp.sum = a; sp.sumsq = q; sp.pad = 1.0;
        s_part[warp][cur_b - b_first] = sp;
      }
      vmax = -INFINITY; dsum = 0.0; dsq = 0.0;
    };
    // the units of images with a map, in order; `nxt` runs one unit ahead (its copies overlap this unit's MMAs)
    UnitIter nxt(u0, tp.tiles, p.H);
    int it_n = 0;
    auto advance = [&]() { while (it_n < n_it && skip(nxt.b)) { nxt.next(); ++it_n; } };
    advance();
    if (it_n < n_it) {
      core::load_operands<D, KC>(smem0, p, nxt.b, nxt.h, nxt.tile, false);
      ptx::cp_async_commit();
    }
    for (int k = 0; it_n < n_it; ++k) {
      const int b = nxt.b, h = nxt.h, tile = nxt.tile;
      if (CF::NST == 1 && k > 0) {                  // one stage: refilled here
        core::load_operands<D, KC>(smem0, p, b, h, tile, false);
        ptx::cp_async_commit();
      }
      nxt.next();
      ++it_n;
      advance();
      if (CF::NST == 2 && it_n < n_it) {
        core::load_operands<D, KC>(smem0 + ((k + 1) & 1) * CF::STAGE, p, nxt.b, nxt.h, nxt.tile, false);
        ptx::cp_async_commit();
        ptx::cp_async_wait<1>();
      } else {
        ptx::cp_async_wait<0>();
      }
      __syncthreads();
      if (b != cur_b) { flush(); cur_b = b; }
      const bool is_max = s_ismax[b];
      const uint32_t st = smem0 + (CF::NST == 2 ? (k & 1) : 0) * CF::STAGE;
      float sum = 0.f, sumsq = 0.f;
#pragma unroll 1
      for (int c = 0; c < KC; ++c) {                // the real tokens of every chunk
        float s[10][4];
        core::warp_qk<D, E>(st + (uint32_t)(warp * 16 * C::LD) * 2u, st + C::QBYTES + c * C::KBYTES, lane, s);
        core::warp_stat<E>(s, core::chunk_keys<KC>(p.T), p.N - tile * kBM - warp * 16, lane, is_max, vmax, sum, sumsq);
      }
      dsum += (double)sum;
      dsq += (double)sumsq;
      __syncthreads();
    }
    flush();
  }
  // ---- per-CTA partials (fixed warp order), then the last CTA to arrive finalises every image ----
  __syncthreads();
  const int G = gridDim.x;
  if (threadIdx.x < kMaxLocal && n_it > 0) {
    const int b = b_first + threadIdx.x;
    if (b < p.B && (int64_t)b * upi < u1 && !skip(b)) {
      StatPartial sp = s_part[0][threadIdx.x];
      for (int w = 1; w < core::kWarps; ++w) {
        sp.vmax = fmax(sp.vmax, s_part[w][threadIdx.x].vmax);
        sp.sum += s_part[w][threadIdx.x].sum;
        sp.sumsq += s_part[w][threadIdx.x].sumsq;
      }
      p.partials[(int64_t)b * G + blockIdx.x] = sp;
    }
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned prev = atomicAdd(p.counters, 1u);
    is_last = (prev == (unsigned)G - 1u) ? 1 : 0;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  // warp w finalises images w, w+8, ...: lanes stride over the CTAs whose unit range intersects the image
  for (int b = warp; b < p.B; b += core::kWarps) {
    if (skip(b)) {
      if (lane == 0) p.stats_out[b] = 0.f;
      continue;
    }
    const long long lo = (long long)b * upi, hi = lo + upi;
    double m = -INFINITY, a = 0.0, q = 0.0;
    for (int c = lane; c < G; c += 32) {
      const long long c0 = (long long)c * tp.units / G, c1 = (long long)(c + 1) * tp.units / G;
      if (c1 > c0 && c0 < hi && c1 > lo) {
        const StatPartial* pp = p.partials + (int64_t)b * G + c;
        m = fmax(m, __ldcg(&pp->vmax));
        a += __ldcg(&pp->sum);
        q += __ldcg(&pp->sumsq);
      }
    }
    core::warp_reduce_stat(m, a, q);
    if (lane == 0) p.stats_out[b] = core::stat_value(p, s_ismax[b], m, a, q, p.T);
  }
  if (threadIdx.x == 0) p.counters[0] = 0u;
}

// ---------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------
// Host replay of the forward kernel's unit schedule (test infrastructure): the same FwdWalk / cta_range code, executed
// on the CPU.  out[u] = {cta, it, b, h, tile} for every unit in launch order of each CTA.
inline int fwd_schedule_host(int B, int H, int tiles, int grid, const int* wmap_index, int* out) {
  if (B <= 0 || B > kMaxBatch || H <= 0 || tiles <= 0 || grid <= 0) return -1;
  int img[kMaxBatch];
  const int nb = partition_images(B, wmap_index, img);
  const long long units = (long long)B * H * tiles;
  int row = 0;
  for (int cta = 0; cta < grid; ++cta) {
    const int u0 = (int)((long long)cta * units / grid), u1 = (int)((long long)(cta + 1) * units / grid);
    const int n_it = u1 - u0;
    if (n_it == 0) continue;
    FwdWalk w(u0, B, H, nb, img);
    for (int it = 0; it < n_it; ++it, w.next()) {
      const FwdUnit f = w.get();
      int* o = out + 5 * (row++);
      o[0] = cta; o[1] = it; o[2] = f.b; o[3] = f.h; o[4] = f.tile;
    }
  }
  return row;
}

// One persistent launch of either kernel of the pair: a CTA per SM, or per unit when there are fewer units.
template <auto Kernel, int D, int KC, typename E>
cudaError_t launch(const XattnParams<E>& x, cudaStream_t s) {
  TcParams<E> tp;
  tp.x = x;
  tp.tiles = ceil_div(x.N, kBM);
  tp.units = x.B * tp.tiles * x.H;
  const cudaError_t e = allow_dynamic_smem<Kernel>(Cfg<D, KC>::SMEM);
  if (e != cudaSuccess) return e;
  const int grid = tp.units < num_sms() ? tp.units : num_sms();
  Kernel<<<grid, kThreads, Cfg<D, KC>::SMEM, s>>>(tp);
  return cudaGetLastError();
}
template <int D, int KC, typename E>
cudaError_t launch_fwd(const XattnParams<E>& x, cudaStream_t s) { return launch<xattn_fwd_kernel<D, KC, E>, D, KC>(x, s); }
template <int D, int KC, typename E>
cudaError_t launch_stats(const XattnParams<E>& x, cudaStream_t s) { return launch<xattn_stats_kernel<D, KC, E>, D, KC>(x, s); }

}  // namespace tc
}  // namespace pww
