// Paint-with-Words cross-attention on Hopper tensor cores (sm_90a), keys T <= 80: the two-launch pair that takes the
// reference's dense [N, T] fp32 weight map (maps with more than 10 distinct columns cannot be packed for the one-launch
// kernel of xattn_fused2.cuh).
//
// Fused region of the reference's inj_forward (paint_with_words.py:87-118), per image b / head h / 128-row tile:
//     statistics kernel:  per-image max / (sum, sumsq) of fp16(Q_h K_h^T) over all heads, rows and tokens
//     forward kernel:     S = Q_h K_h^T;  P = softmax(scale * (S + g * M_b * w[b]));  O = P V_h
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

template <int D>
struct Cfg {
  using T_ = core::Tile<D>;
  static constexpr uint32_t STAGE = T_::QBYTES + 2 * T_::KBYTES;   // Q | K | V of one unit
  static constexpr uint32_t SMEM = 2 * STAGE;
  static_assert(SMEM <= 232448 - 8192, "shared memory budget (dynamic + static tables)");
};

struct TcParams {
  XattnParams x;
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
// Forward-kernel unit order.  Units are tile-major; inside a row tile the images are visited in GROUPS that share one
// [128 x T] mask tile:
//   * pair group: one biased image A (has a weight map) and one unbiased image U (classifier-free guidance puts as many
//     of each in the batch).  2H units, head h = j/2, in the order  U A | A U | U A | ...  so that (1) biased and
//     unbiased units alternate at the finest grain -- every CTA's contiguous range gets the same mix, whatever the image
//     order in the batch -- (2) A's mask tile is reused by all H heads (it stays in L2), and (3) the group ends with its
//     mask no longer needed.
//   * solo group: an image without a partner (all-biased or all-unbiased batches), H units head-minor.
// s_img lists the biased images first (nb of them), then the unbiased ones.
struct FwdUnit {
  int b, h, tile;
  int j, gsize;       // position inside the group, units in the group
  int jl;             // last position whose unit reads the mask (gsize-1 when the group has no mask)
  int mask_b;         // image whose mask tile the group uses, -1 = none
};
// Walks a CTA's contiguous unit range in that order; divisions only in the constructor.
struct FwdWalk {
  int B, H, nb, np, ng, jl_pair;
  const int* img;
  int tile, gi, j;    // row tile, group inside the tile (pair groups first, then solo groups), position in the group
  __host__ __device__ __forceinline__ FwdWalk(int u, int B_, int H_, int nb_, const int* img_) : B(B_), H(H_), nb(nb_), img(img_) {
    const int nu = B - nb;
    np = nb < nu ? nb : nu;
    ng = B - np;
    const int jlast = 2 * H - 1;
    jl_pair = ((((jlast ^ (jlast >> 1)) & 1) ^ 1) == 0) ? jlast : jlast - 1;
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
    r.j = j;
    if (gi < np) {
      r.gsize = 2 * H;
      r.h = j >> 1;
      const int unb = ((j ^ (j >> 1)) & 1) ^ 1;          // 1 = the unbiased image's unit
      r.b = unb ? img[nb + gi] : img[gi];
      r.mask_b = img[gi];
      r.jl = jl_pair;
    } else {
      r.gsize = H;
      r.h = j;
      r.jl = H - 1;
      if (2 * nb > B) { r.b = img[gi]; r.mask_b = r.b; }          // biased image without a partner
      else { r.b = img[nb + gi]; r.mask_b = -1; }                 // unbiased image without a partner
    }
    return r;
  }
};
// Position (inside its group) of the last unit of the CTA's range that reads the group's mask tile: the last
// mask-reading unit if the CTA's range [it - j_lo .., it + rest] contains it, else the last unit of the group in range.
__host__ __device__ __forceinline__ int mask_release_pos(const FwdUnit& f, int it, int n_it) {
  const int j_lo = f.j > it ? f.j - it : 0;
  int j_hi = f.j + (n_it - 1 - it);
  if (j_hi > f.gsize - 1) j_hi = f.gsize - 1;
  return (f.jl >= j_lo && f.jl <= j_hi) ? f.jl : j_hi;
}
// First unit of a mask group inside a CTA's range.
__host__ __device__ __forceinline__ bool mask_group_starts_here(const FwdUnit& f, int it) { return f.j == 0 || it == 0; }
__device__ __forceinline__ void cta_range(int units, int& u0, int& u1) {
  u0 = (int)((long long)blockIdx.x * units / gridDim.x);
  u1 = (int)((long long)(blockIdx.x + 1) * units / gridDim.x);
}
__device__ __forceinline__ int image_widx(const XattnParams& p, int b) {
  if (p.wmap == nullptr) return -1;
  return p.wmap_index ? p.wmap_index[b] : b;
}

// Copies of one unit's operands into a stage: Q rows of the tile, K (and V) rows of the head.
template <int D>
__device__ __forceinline__ void load_unit(uint32_t st, const XattnParams& p, int b, int h, int tile, bool with_v) {
  using C = core::Tile<D>;
  const int rows = p.N - tile * kBM;
  core::load_rows<D>(st, p.q + (int64_t)b * p.q_bs + (int64_t)tile * kBM * p.q_rs + h * D, p.q_rs, kBM, rows < kBM ? rows : kBM);
  core::load_rows<D>(st + C::QBYTES, p.k + (int64_t)b * p.k_bs + h * D, p.k_rs, kTP, p.T);
  if (with_v) core::load_rows<D>(st + C::QBYTES + C::KBYTES, p.v + (int64_t)b * p.k_bs + h * D, p.k_rs, kTP, p.T);
  ptx::cp_async_commit();
}

// ---------------------------------------------------------------------------------------------------------
// forward kernel
// ---------------------------------------------------------------------------------------------------------
template <int D>
__global__ void __launch_bounds__(kThreads, 1) xattn_fwd_kernel(const TcParams tp) {
  using C = core::Tile<D>;
  const XattnParams& p = tp.x;
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
    s_coef[b] = wi >= 0 ? __ldg(p.g_sigma) * __ldg(p.stats + b) : 0.f;
  }
  __syncthreads();
  int u0, u1;
  cta_range(tp.units, u0, u1);
  const int n_it = u1 - u0;
  if (n_it <= 0) return;
  const float sl2 = p.scale * 1.4426950408889634f;
  FwdWalk w(u0, p.B, p.H, s_nb, s_img);
  FwdUnit nxt = w.get();
  load_unit<D>(smem0, p, nxt.b, nxt.h, nxt.tile, true);
  for (int it = 0; it < n_it; ++it) {
    const FwdUnit f = nxt;
    if (it + 1 < n_it) {
      w.next();
      nxt = w.get();
      load_unit<D>(smem0 + ((it + 1) & 1) * Cfg<D>::STAGE, p, nxt.b, nxt.h, nxt.tile, true);
      ptx::cp_async_wait<1>();
    } else {
      ptx::cp_async_wait<0>();
    }
    __syncthreads();
    const uint32_t st = smem0 + (it & 1) * Cfg<D>::STAGE;
    const uint32_t qs = st + (uint32_t)(warp * 16 * C::LD) * 2u;
    float s[10][4];
    core::warp_qk<D>(qs, st + C::QBYTES, lane, s);
    const int row0 = f.tile * kBM + warp * 16;
    const int widx = s_widx[f.b];
    if (widx >= 0) {
      const float x = s_coef[f.b];
      const float* wm = p.wmap + (int64_t)widx * p.wmap_bs;
#pragma unroll
      for (int j = 0; j < 10; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int t = core::tok(j, e, lane), r = row0 + (lane >> 2) + (e >> 1) * 8;
          if (t < p.T && r < p.N) s[j][e] = fmaf(x, __ldg(wm + (int64_t)r * p.T + t), s[j][e]);
        }
    }
    float o[C::NT][4];
    core::warp_softmax_pv<D>(s, p.T, sl2, st + C::QBYTES + C::KBYTES, lane, o);
    core::warp_store<D>(o, smem + (it & 1) * Cfg<D>::STAGE + warp * 16 * C::LD * 2, lane,
                        p.out + (int64_t)f.b * p.o_bs + f.h * D, p.o_rs, row0, p.N);
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------------------
// statistics kernel: per-image max / (sum, sumsq) of fp16(S) over all heads, rows and tokens
// ---------------------------------------------------------------------------------------------------------
template <int D>
__global__ void __launch_bounds__(kThreads, 1) xattn_stats_kernel(const TcParams tp) {
  using C = core::Tile<D>;
  const XattnParams& p = tp.x;
  extern __shared__ __align__(128) unsigned char smem[];
  const uint32_t smem0 = ptx::smem_u32(smem);
  __shared__ StatPartial s_part[core::kWarps][kMaxLocal];     // [warp][local image]
  __shared__ unsigned char s_skip[kMaxBatch];
  __shared__ int is_last;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int u0, u1;
  cta_range(tp.units, u0, u1);
  const int n_it = u1 - u0;
  const int upi = tp.tiles * p.H;                               // units per image
  const int b_first = n_it > 0 ? u0 / upi : 0;
  for (int b = threadIdx.x; b < p.B; b += kThreads) s_skip[b] = (p.wmap_index != nullptr && p.wmap_index[b] < 0) ? 1 : 0;
  if (threadIdx.x < core::kWarps * kMaxLocal) {
    StatPartial sp;
    sp.vmax = -INFINITY; sp.sum = 0.0; sp.sumsq = 0.0; sp.pad = 0.0;
    s_part[threadIdx.x / kMaxLocal][threadIdx.x % kMaxLocal] = sp;
  }
  __syncthreads();
  auto skip = [&](int b) { return s_skip[b] != 0; };
  const bool is_max = p.stat == PWW_STAT_MAX;
  {
    float vmax = -INFINITY;
    double dsum = 0.0, dsq = 0.0;
    int cur_b = -1;
    auto flush = [&]() {
      if (cur_b < 0) return;
      double m = vmax, a = dsum, q = dsq;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
        a += __shfl_xor_sync(0xffffffffu, a, o);
        q += __shfl_xor_sync(0xffffffffu, q, o);
      }
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
    if (it_n < n_it) load_unit<D>(smem0, p, nxt.b, nxt.h, nxt.tile, false);
    for (int k = 0; it_n < n_it; ++k) {
      const int b = nxt.b, tile = nxt.tile;
      nxt.next();
      ++it_n;
      advance();
      if (it_n < n_it) {
        load_unit<D>(smem0 + ((k + 1) & 1) * Cfg<D>::STAGE, p, nxt.b, nxt.h, nxt.tile, false);
        ptx::cp_async_wait<1>();
      } else {
        ptx::cp_async_wait<0>();
      }
      __syncthreads();
      if (b != cur_b) { flush(); cur_b = b; }
      const uint32_t st = smem0 + (k & 1) * Cfg<D>::STAGE;
      float s[10][4];
      core::warp_qk<D>(st + (uint32_t)(warp * 16 * C::LD) * 2u, st + C::QBYTES, lane, s);
      float sum = 0.f, sumsq = 0.f;
      core::warp_stat(s, p.T, p.N - tile * kBM - warp * 16, lane, is_max, vmax, sum, sumsq);
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
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
      a += __shfl_xor_sync(0xffffffffu, a, o);
      q += __shfl_xor_sync(0xffffffffu, q, o);
    }
    if (lane == 0) {
      const double cnt = (double)p.H * (double)p.N * (double)p.T;
      double r;
      if (is_max) {
        r = m;
      } else {
        const double var = (q - a * a / cnt) / (cnt - 1.0);
        r = sqrt(var > 0.0 ? var : 0.0);
      }
      p.stats_out[b] = round_to_f16((float)r);
    }
  }
  if (threadIdx.x == 0) p.counters[0] = 0u;
}

// ---------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------
// Diagnostics of the last host-side failure in the launchers (read by pww_abi.cu into pww_last_cuda_error()).
inline char* tc_error_buf() {
  static thread_local char buf[256] = "";
  return buf;
}

// Per-device host state: the current device decides (the Python shim makes the tensors' device current).
constexpr int kMaxDevices = 64;
inline int cur_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return (dev >= 0 && dev < kMaxDevices) ? dev : 0;
}
inline int num_sms() {
  static int n[kMaxDevices] = {0};
  const int dev = cur_device();
  if (!n[dev]) cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev);
  return n[dev];
}

inline int stats_grid(int units) { return units < num_sms() ? units : num_sms(); }

// Host replay of the forward kernel's unit schedule (test infrastructure): the same FwdWalk / cta_range /
// mask_release_pos / mask_group_starts_here code, executed on the CPU.  out[u] = {cta, it, b, h, tile, group_id, mask_b,
// flags} for every unit in launch order of each CTA; flags bit 0 = last unit of the group in the CTA's range that reads
// the mask tile, bit 1 = first unit of a mask group in the CTA's range.
inline int fwd_schedule_host(int B, int H, int tiles, int grid, const int* wmap_index, int* out) {
  if (B <= 0 || B > kMaxBatch || H <= 0 || tiles <= 0 || grid <= 0) return -1;
  int img[kMaxBatch];
  int nb = 0;
  for (int b = 0; b < B; ++b) if (wmap_index[b] >= 0) img[nb++] = b;
  int nu = 0;
  for (int b = 0; b < B; ++b) if (wmap_index[b] < 0) img[nb + nu++] = b;
  const long long units = (long long)B * H * tiles;
  int row = 0;
  for (int cta = 0; cta < grid; ++cta) {
    const int u0 = (int)((long long)cta * units / grid), u1 = (int)((long long)(cta + 1) * units / grid);
    const int n_it = u1 - u0;
    if (n_it == 0) continue;
    FwdWalk w(u0, B, H, nb, img);
    int grp = -1;
    for (int it = 0; it < n_it; ++it, w.next()) {
      const FwdUnit f = w.get();
      if (f.j == 0 || it == 0) ++grp;
      int* o = out + 8 * (row++);
      o[0] = cta; o[1] = it; o[2] = f.b; o[3] = f.h; o[4] = f.tile; o[5] = grp; o[6] = f.mask_b;
      o[7] = ((f.j == mask_release_pos(f, it, n_it)) ? 1 : 0) | (mask_group_starts_here(f, it) ? 2 : 0);
    }
  }
  return row;
}

template <int D>
cudaError_t set_smem(const void* fn, uint32_t bytes, bool (&done)[kMaxDevices]) {
  if (done[cur_device()]) return cudaSuccess;
  cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e == cudaSuccess) done[cur_device()] = true;
  return e;
}

template <int D>
cudaError_t launch_fwd(const XattnParams& x, cudaStream_t s) {
  TcParams tp;
  tp.x = x;
  tp.tiles = ceil_div(x.N, kBM);
  tp.units = x.B * tp.tiles * x.H;
  static bool attr_set[kMaxDevices] = {false};
  cudaError_t e = set_smem<D>((const void*)xattn_fwd_kernel<D>, Cfg<D>::SMEM, attr_set);
  if (e != cudaSuccess) return e;
  const int grid = tp.units < num_sms() ? tp.units : num_sms();
  xattn_fwd_kernel<D><<<grid, kThreads, Cfg<D>::SMEM, s>>>(tp);
  return cudaGetLastError();
}

template <int D>
cudaError_t launch_stats(const XattnParams& x, cudaStream_t s) {
  TcParams tp;
  tp.x = x;
  tp.tiles = ceil_div(x.N, kBM);
  tp.units = x.B * tp.tiles * x.H;
  static bool attr_set[kMaxDevices] = {false};
  cudaError_t e = set_smem<D>((const void*)xattn_stats_kernel<D>, Cfg<D>::SMEM, attr_set);
  if (e != cudaSuccess) return e;
  xattn_stats_kernel<D><<<stats_grid(tp.units), kThreads, Cfg<D>::SMEM, s>>>(tp);
  return cudaGetLastError();
}

// partial slots the stats kernel writes per image
inline int stats_slots() { return num_sms(); }

}  // namespace tc
}  // namespace pww
