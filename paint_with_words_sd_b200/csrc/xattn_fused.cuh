// Shared pieces of the one-launch Paint-with-Words cross-attention kernel (csrc/xattn_fused2.cuh): constants, launch
// parameters, the unit order (FxWalk: which (image, row tile, head group) a CTA's contiguous range covers and in which order),
// the grid-barrier membership test and the host-side knobs.
//
// Packed weight map (SURVEY 8f-4).  The reference's dense [N, 77] fp32 map has at most a handful of distinct non-zero
// columns (one per painted region, paint_with_words.py:255-272), so it is stored as a column dictionary:
//     W[n, t] = Mu[n, cidx[t]]      Mu [N, R] fp32 (R <= 10 distinct columns), cidx [77] (-1 = zero column)
// and Mu is split into fp16 hi/lo halves:  mpack[n] = [ hi(Mu[n,0..9]) | lo(Mu[n,0..9]) | hi(Mu[n,0..9]) | 0 0 ]  (32 fp16,
// 64 bytes per row instead of 308).  The kernel rebuilds W[n, t] = hi + lo in fp32 (exact to 2^-22 relative) from the row
// tile's 8 KB of packed map in shared memory and adds x * W to the fp32 scores, x = g(sigma) * statistic.
//
// Unit order.  `img` lists the biased images first, then the unbiased ones; pair groups (a biased image with an unbiased
// one: classifier-free guidance supplies both) come first, tile-major, biased unit before unbiased, then the solo groups of
// the images without a partner.  A CTA takes a contiguous range of this order, so it gets the same number of biased and
// unbiased units (+-1) whatever the image order of the batch, and its unbiased units' softmax overlaps the grid barrier.
#pragma once
#include "mma_sm90.cuh"
#include "pww_common.cuh"
#include "xattn_tc.cuh"   // num_sms, tc_error_buf

namespace pww {
namespace fx {

constexpr int kBM = 128;          // query rows per tile
constexpr int kTP = 80;           // padded key count
constexpr int kMaxBatch = 32;     // images per launch (the C ABI splits larger batches)
constexpr int kMaxLocal = 4;      // biased images one CTA's unit range may touch (checked on the host)
constexpr int kMW = 32;           // packed-map columns per row (64 bytes)
constexpr int kRC = 10;           // dictionary capacity (distinct non-zero columns)

struct FxParams {
  XattnParams x;            // q/k/v/out, strides, wmap_index, g_sigma, scale, stat, stats_out, counters, partials
  const int8_t* cidx;       // [Bw, 80] dictionary column per token, -1 = none
  const void* mpack;        // [Bw, N, 32] fp16 packed maps (see above)
  int64_t mpack_bs;         // elements
  int tiles, units;
  int grid;                 // CTAs (== gridDim.x): partial slots per image
  int hg;                   // head groups per row tile (grouped-head kernel, xattn_fused2.cuh)
  unsigned* jobs_dump;      // debug only: [grid][2 + 2 * 512] = njobs, nstat, job table of every CTA (grouped-head kernel)
};
// ------------------------------------------------------------------------------------------------------------------
// unit order (shared by the kernel and the host replay)
// ------------------------------------------------------------------------------------------------------------------
// `img` lists the biased images first (nb of them), then the unbiased ones.  Groups: np = min(nb, nu) PAIR groups (biased
// image img[g] + unbiased image img[nb + g], tiles * 2H units: tile-major, then head, biased unit before unbiased), then
// the SOLO groups of the images without a partner (tiles * H units).  A CTA takes a contiguous range of this order, so it
// gets the same number of biased and unbiased units (+-1) whatever the image order of the batch, and stays inside one or
// two images.
struct FxUnit {
  int b, h, tile, biased, gi;
};
struct FxWalk {
  int B, H, tiles, nb, np;
  const int* img;
  int gi, tile, j;
  __host__ __device__ __forceinline__ FxWalk() {}
  __host__ __device__ __forceinline__ FxWalk(int u, int B_, int H_, int tiles_, int nb_, const int* img_)
      : B(B_), H(H_), tiles(tiles_), nb(nb_), img(img_) {
    const int nu = B - nb;
    np = nb < nu ? nb : nu;
    const int per_pair = tiles * 2 * H;
    if (u < np * per_pair) {
      gi = u / per_pair;
      const int r = u - gi * per_pair;
      tile = r / (2 * H);
      j = r - tile * 2 * H;
    } else {
      u -= np * per_pair;
      const int per_solo = tiles * H;
      const int s = u / per_solo;
      gi = np + s;
      const int r = u - s * per_solo;
      tile = r / H;
      j = r - tile * H;
    }
  }
  __host__ __device__ __forceinline__ void next() {
    const int gsize = gi < np ? 2 * H : H;
    if (++j == gsize) {
      j = 0;
      if (++tile == tiles) { tile = 0; ++gi; }
    }
  }
  __host__ __device__ __forceinline__ FxUnit get() const {
    FxUnit r;
    r.tile = tile;
    r.gi = gi;
    if (gi < np) {
      r.h = j >> 1;
      r.biased = (j & 1) ^ 1;
      r.b = r.biased ? img[gi] : img[nb + gi];
    } else {
      r.h = j;
      r.biased = (2 * nb > B) ? 1 : 0;
      r.b = r.biased ? img[gi] : img[nb + gi];
    }
    return r;
  }
};
// 32-bit arithmetic on purpose: a 64-bit division is ~100 SASS instructions and this is inlined at every membership test
// (it was 28 % of the grouped-head kernel's code); the host checks units * grid < 2^32 (fused_units_ok).
__host__ __device__ __forceinline__ void fx_range(int cta, int grid, int units, int& u0, int& u1) {
  u0 = (int)((unsigned)cta * (unsigned)units / (unsigned)grid);
  u1 = (int)((unsigned)(cta + 1) * (unsigned)units / (unsigned)grid);
}
inline bool fused_units_ok(long long units, int grid) { return units > 0 && units * (long long)(grid + 1) < (1ll << 32); }
// Does CTA `cta` own at least one unit of the BIASED image at list position `pos` (== its group index)?
__host__ __device__ __forceinline__ bool fx_cta_has_image(int cta, int grid, int units, int pos, int H, int tiles, int np) {
  int lo, hi;
  fx_range(cta, grid, units, lo, hi);
  const int per_pair = tiles * 2 * H, per_solo = tiles * H;
  const bool pair = pos < np;
  const int base = pair ? pos * per_pair : np * per_pair + (pos - np) * per_solo;
  const int len = pair ? per_pair : per_solo;
  const int a = lo > base ? lo : base, b = hi < base + len ? hi : base + len;
  if (a >= b) return false;
  if (!pair) return true;
  return (b - a >= 2) || (((a - base) & 1) == 0);        // biased units sit at even offsets of a pair group
}

// ------------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------------
inline unsigned*& debug_jobs_dump() {   // test infrastructure: device buffer the grouped-head kernel copies its job tables to
  static unsigned* p = nullptr;
  return p;
}
inline int& debug_grid() {          // test infrastructure: cap the persistent grid (0 = number of SMs)
  static int g = 0;
  return g;
}
inline int fused_grid(int units) {
  int g = tc::num_sms();
  if (debug_grid() > 0 && debug_grid() < g) g = debug_grid();
  return units < g ? units : g;
}
// A CTA range may touch at most kMaxLocal biased images (partial slots in shared memory).
inline bool fused_range_ok(int B, int H, int tiles, int grid) {
  const long long units = (long long)B * H * tiles;
  const long long per_cta = (units + grid - 1) / grid;
  return per_cta <= (long long)(kMaxLocal - 1) * tiles * H;
}
inline size_t fused_workspace_bytes() {
  return 512 + (size_t)kMaxBatch * 2048 * sizeof(StatPartial) / 8;   // counters | per-image maxima | [32][256] partial slots
}

inline int fused_cta_has_image_host(int cta, int grid, int B, int H, int tiles, const int* wmap_index, int b) {
  int nb = 0, pos = -1;
  for (int i = 0; i < B; ++i)
    if (wmap_index[i] >= 0) { if (i == b) pos = nb; ++nb; }
  if (pos < 0) return 0;
  const int nu = B - nb, np = nb < nu ? nb : nu;
  return fx_cta_has_image(cta, grid, B * H * tiles, pos, H, tiles, np) ? 1 : 0;
}

}  // namespace fx
}  // namespace pww
