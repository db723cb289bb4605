// Paint-with-Words cross-attention in ONE launch (statistic + bias + softmax + P.V) on Hopper tensor cores, keys T <= 80
// or 2 / 3 CLIP chunks of 77 (T = 154, 231).
//
// The per-image statistic (max or std of Q K^T over all heads, rows and tokens) is a grid-wide dependency of every
// biased score, so the kernel is a persistent cooperative launch (one CTA per SM, all co-resident) that runs three passes
// over its contiguous range of work units:
//     1. statistic jobs of the units of biased images: S = Q K^T, folded into per-warp partials, then published to the
//        image's word in the workspace (max: one atomic max of an order-preserving key; std: a partial slot per CTA,
//        summed by the waiters in CTA order -- deterministic for a given grid);
//     2. softmax jobs of the unbiased units: they need no statistic and overlap the other CTAs' statistic pass;
//     3. grid barrier (per biased image, only the CTAs that publish for it), then the softmax jobs of the biased units
//        with the bias x * W, x = g(sigma) * E(statistic), W rebuilt from the packed map (below).  E, the element type
//        of q / k / v / out, is fp16 or bf16; the packed map is fp16 whatever E is.
// The statistic kind and g(sigma) are per image when the launch carries per-image arrays (XattnParams::stat_kind,
// g_stride = 1), else one kind and one g(sigma) for every image; each CTA keeps the kind of its local biased images in
// shared memory, so the statistic jobs, the publish step and the finalise step branch per image.
// Work unit = (image, 128-row tile, group of G heads); a unit expands into one job per head.  Each job is computed by the
// 8 warps of the CTA with the warp-level MMA tiles of xattn_core.cuh; the cp.async copies of job i + 1 (Q rows, K, V
// and, for biased softmax jobs, the row tile's packed map) are in flight while job i is computed.
//
// Key chunks (KC = 1, 2 or 3): a stage holds one 80-row K and V tile per chunk; a job loops over the chunks (statistic:
// S of every chunk; softmax: per-chunk bias and the streaming softmax of xattn_core.cuh).  Where two such stages do not
// fit in shared memory (head dim 80 at 3 chunks, head dim 160 at 2 and 3) the kernel runs on one stage and the copies of
// job i + 1 start once job i is done.  The unit and job order do not depend on KC.
//
// Packed weight map (SURVEY 8f-4).  The reference's dense [N, 77] fp32 map has at most a handful of distinct non-zero
// columns (one per painted region, paint_with_words.py:255-272), so it is stored as a column dictionary:
//     W[n, t] = Mu[n, cidx[t]]      Mu [N, R] fp32 (R <= 10 distinct columns), cidx [77] (-1 = zero column)
// and Mu is split into fp16 hi/lo halves:  mpack[n] = [ hi(Mu[n,0..9]) | lo(Mu[n,0..9]) | hi(Mu[n,0..9]) | 0 0 ]  (32 fp16,
// 64 bytes per row instead of 308).  The kernel rebuilds W[n, t] = hi + lo in fp32 (exact to 2^-22 relative) from the row
// tile's 8 KB of packed map in shared memory and adds x * W to the fp32 scores.
//
// Attention recording (REC = true, FxRecord): the softmax jobs of the recorded images also add each query row's softmax
// mass per region slot (16 slots, a token -> slot row per image) into a caller-owned fp32 accumulator, computed from the
// same packed P as P.V (xattn_core.cuh: warp_region_chunk / warp_region_add).  The plain instances (REC = false) are
// the kernel without it: every recording instruction is behind `if constexpr`.
//
// Region prompts (RGN = true, FxRegion, KC = 2, 3): one softmax per key chunk, mixed per query row by fp32 chunk
// weights (xattn_core.cuh: warp_weighted_chunk); the chunks no row of a tile weighs are not copied, and a biased
// image's statistic jobs skip the chunks outside its statistic mask.  Every region instruction is behind
// `if constexpr` as well.
#pragma once
#include <algorithm>
#include <type_traits>
#include <vector>

#include "mma_sm90.cuh"
#include "pww_common.cuh"
#include "xattn_core.cuh"

namespace pww {
namespace fx {

constexpr int kMaxBatch = 32;     // images per launch (the C ABI splits larger batches)
constexpr int kMaxLocal = 4;      // biased images one CTA's unit range may touch (checked on the host)
constexpr int kMW = 32;           // packed-map columns per row (64 bytes)
constexpr int kRC = 10;           // dictionary capacity (distinct non-zero columns)

template <typename E>
struct FxParams {
  XattnParams<E> x;            // q/k/v/out, strides, wmap_index, g_sigma, scale, stat, stats_out, counters, partials
  const int8_t* cidx;       // [Bw, 80 k] dictionary column per token (k key chunks; token 77 c + j at 80 c + j), -1 = none
  const void* mpack;        // [Bw, N, 32] fp16 packed maps (see above)
  int64_t mpack_bs;         // elements
  int tiles, units;
  int grid;                 // CTAs (== gridDim.x): partial slots per image
  int hg;                   // head groups per row tile
  unsigned* jobs_dump;      // debug only: [grid][2 + 2 * 512] = njobs, nstat, job table of every CTA
};

// Attention recording (the REC instances): image b with rec_index[b] >= 0 adds, for every head h and query row n, the
// softmax mass of each region slot r < 16,  mass[n, r] = sum_{t : ridx[t] = r} P[n, t] / sum_t P[n, t],  into
// rec_acc[rec_index[b], h, n, r].  Biased and unbiased images alike; the plain instances never see these fields.
struct FxRecord {
  const int8_t* ridx;       // [Br, 80 k] region slot per token (the cidx column layout), -1 = no region
  const int32_t* rec_index; // [B] record of image b, -1 = not recorded
  float* rec_acc;           // [Br, H, N, 16] fp32, accumulated into
  int64_t rec_bs;           // elements between records (>= H * N * 16)
};
template <typename E>
struct FxRecParams : FxParams<E> {
  FxRecord rec;
};
// Region prompts (the RGN instances, KC = 2, 3): chunk c of image b's context gets its own softmax over its 77 keys,
// and query row n takes  out(n) = sum_c w_c(n) softmax_c(..) V_c  (xattn_core.cuh: warp_weighted_chunk).  The weights
// of image b are row rw_index[b] (row b when rw_index is NULL) of rw; an image with index -1 takes (1, 0, ..) on every
// row.  The K / V of a chunk that no row of a softmax job's tile weighs are neither copied nor multiplied.  The weight
// row is independent of the bias: an unbiased image with a row runs the same mixed softmax with no bias, and a biased
// image with -1 takes its first chunk alone with the bias.  A biased image's statistic covers the chunks of its mask
// stat_chunks[b] (chunk 0 always; the other chunks' K is not even copied for it): its max, or its std over the
// H * N * 77 * popcount(mask) scores; with stat_chunks NULL every chunk, all H * N * 77 KC scores.
struct FxRegion {
  const float* rw;              // [Bw, N, KC] fp32 chunk weights
  int64_t rw_bs;                // elements between weight rows (>= N * KC)
  const int32_t* rw_index;      // [B] weight row of image b, -1 = none; NULL = row b
  const int32_t* stat_chunks;   // [B] bit c = chunk c is in image b's statistic; NULL = every chunk
};
template <typename E>
struct FxRgnParams : FxParams<E> {
  FxRegion rg;
};
template <typename E, bool REC, bool RGN = false>
using FxArgs = std::conditional_t<RGN, FxRgnParams<E>, std::conditional_t<REC, FxRecParams<E>, FxParams<E>>>;

template <int D, int KC = 1>
struct Cfg2 {
  // heads per unit (the granularity of a CTA's range): 2 at head dims 40 and 64, one head at 80 and 160
  static constexpr int G = (D == 40 || D == 64) ? 2 : 1;
  using T_ = core::Tile<D>;
  static constexpr uint32_t MBYTES = core::kBM * kMW * 2;              // packed-map rows of the row tile
  static constexpr uint32_t OFF_M = T_::QBYTES + 2 * KC * T_::KBYTES;
  static constexpr uint32_t STAGE = OFF_M + MBYTES;                    // Q | K chunks | V chunks | map of one job
  static constexpr int NST = (2 * STAGE + 8192 <= 232448) ? 2 : 1;     // stages (see the header)
  static constexpr uint32_t SMEM = NST * STAGE;
  static_assert(SMEM + 8192 <= 232448, "shared memory budget (dynamic + ~7 KB of static tables incl. the 4 KB job table)");
  // region instances: [2][kWarps] per-warp chunk bits and [2] chunk masks of the jobs in flight, after the stages
  static constexpr uint32_t SMEM_RGN = SMEM + 128;
  static_assert(SMEM_RGN + 8192 <= 232448, "shared memory budget of the region instances");
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
// job lists (shared by the kernel and the host replay)
// ------------------------------------------------------------------------------------------------------------------
// Units are walked with FxWalk, "heads" being head GROUPS (hg = ceil(H / G) of them); a unit expands into one job per
// head of its group.  A CTA runs three passes over its contiguous unit range: statistic jobs of the biased units,
// softmax jobs of the unbiased units, softmax jobs of the biased units.
struct Fx2Job {
  int b, h, tile, biased;
  int kind;     // 0 = stat, 1 = main
  int i;        // job index
  int li;       // local index of the biased image inside this CTA's range (biased jobs)
};
struct Fx2Jobs {
  FxWalk w;
  int u0, n_units, B, H, HG, G, tiles, nb;
  const int* img;
  int it, phase, i, li, lastb;
  FxUnit cur;
  int cur_li, hl, nh;
  bool have;
  __host__ __device__ __forceinline__ Fx2Jobs(int u0_, int n_units_, int B_, int H_, int G_, int tiles_, int nb_,
                                              const int* img_)
      : u0(u0_), n_units(n_units_), B(B_), H(H_), G(G_), tiles(tiles_), nb(nb_), img(img_) {
    HG = (H + G - 1) / G;
    phase = nb > 0 ? 0 : 1;
    i = 0;
    rewind();
  }
  __host__ __device__ __forceinline__ void rewind() {
    w = FxWalk(u0, B, HG, tiles, nb, img);
    it = 0; li = -1; lastb = -1; have = false;
  }
  __host__ __device__ __forceinline__ bool next(Fx2Job& jb) {
    for (;;) {
      if (have) {
        jb.b = cur.b; jb.h = cur.h * G + hl; jb.tile = cur.tile; jb.biased = cur.biased;
        jb.kind = phase == 0 ? 0 : 1;
        jb.i = i++;
        jb.li = cur.biased ? cur_li : -1;
        if (++hl == nh) have = false;
        return true;
      }
      while (it < n_units) {
        const FxUnit u = w.get();
        w.next();
        ++it;
        if (u.biased && u.b != lastb) { ++li; lastb = u.b; }
        const bool want = (phase == 1) ? !u.biased : (u.biased != 0);
        if (!want) continue;
        cur = u; cur_li = li;
        hl = 0;
        nh = H - u.h * G < G ? H - u.h * G : G;
        have = true;
        break;
      }
      if (have) continue;
      if (phase == 2) return false;
      ++phase;
      rewind();
    }
  }
};

// ------------------------------------------------------------------------------------------------------------------
// the kernel
// ------------------------------------------------------------------------------------------------------------------
// Job table.  One warp builds the CTA's job list in shared memory during the prologue (parallel over the units of the
// range: ballots and warp scans, no sequential walk); the whole CTA then walks it.
//   s_jobs[i].x = b | h << 8 | tile << 16          s_jobs[i].y = flags, see the JF_* masks
constexpr int kMaxUnits = 64;        // units per CTA (host-checked: the C ABI splits larger batches)
constexpr int kMaxJobs = 512;        // kMaxUnits * G heads * 2 passes
constexpr uint32_t JF_MAIN = 1u, JF_BIASED = 2u;   // | li << 4 (2 bits)

// Order-preserving map float -> unsigned (0 is below every real number: a zero-filled workspace reads as -infinity).
__device__ __forceinline__ unsigned f32_key(float f) {
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_f32(unsigned k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// REC = true: the recording instance (FxRecord above); RGN = true: the region-prompt instance (FxRegion above).  Their
// extra work is behind `if constexpr`, so the plain instances are the kernel without it.
template <int D, int KC, typename E, bool REC = false, bool RGN = false>
__global__ void __launch_bounds__(core::kThreads, 1) xattn_fused2_kernel(const FxArgs<E, REC, RGN> fp) {
  static_assert(!(REC && RGN), "attention recording has no region-prompt instance");
  static_assert(!RGN || KC > 1, "region prompts need 2 or 3 key chunks");
  using C = core::Tile<D>;
  using CF = Cfg2<D, KC>;
  constexpr int CW = core::kTP * KC;                    // cidx columns: token 77 c + j of chunk c at column 80 c + j
  const XattnParams<E>& p = fp.x;
  extern __shared__ __align__(128) unsigned char smem[];
  const uint32_t smem0 = ptx::smem_u32(smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int T = p.T;
  int u0, u1;
  fx_range(blockIdx.x, gridDim.x, fp.units, u0, u1);
  const int n_it = u1 - u0;
  const int HG = fp.hg;

  __shared__ int s_widx[kMaxBatch];
  __shared__ int s_img[kMaxBatch];                // biased images first, then unbiased
  __shared__ int s_nb, s_njobs, s_nstat, s_nl;
  __shared__ int s_lb[kMaxLocal], s_lp[kMaxLocal];   // image / group position of the CTA's local biased images
  __shared__ float s_coef[kMaxLocal];             // g(sigma) * statistic of the CTA's local biased images
  __shared__ bool s_ismax[kMaxLocal];             // statistic kind of the CTA's local biased images
  __shared__ StatPartial s_part[core::kWarps][kMaxLocal];   // [warp][local biased image]
  __shared__ uint2 s_jobs[kMaxJobs];
  __shared__ uint4 s_unit[kMaxUnits];              // job-table build scratch: one entry per unit of the range
  __shared__ int s_expect[kMaxLocal];              // CTAs that publish a partial for each local biased image
  __shared__ signed char s_cidx[kMaxLocal][CW];    // token -> dictionary column of the CTA's local biased images

  if (warp == 0) {
    // ---- stable partition of the images by "has a weight map" ----
    {
      const int b = lane;
      const int wi = (b < p.B && p.wmap != nullptr) ? (p.wmap_index ? p.wmap_index[b] : b) : -1;   // wmap == NULL: no maps at all
      const bool valid = b < p.B, bi = valid && wi >= 0;
      const unsigned mb = __ballot_sync(0xffffffffu, bi), mu = __ballot_sync(0xffffffffu, valid && !bi);
      const unsigned lt = (1u << lane) - 1u;
      const int nbt = __popc(mb);
      if (bi) s_img[__popc(mb & lt)] = b;
      else if (valid) s_img[nbt + __popc(mu & lt)] = b;
      if (valid) s_widx[b] = wi;
      if (lane == 0) s_nb = nbt;
    }
    __syncwarp();
    // ---- job table: pass 1 gives every unit its place in the three lists, pass 2 expands units into head jobs ----
    const int nbi = s_nb;
    const unsigned lt = (1u << lane) - 1u;
    int c_sj = 0, c_uj = 0, c_li = -1, c_lastb = -1;
    for (int base = 0; base < n_it; base += 32) {
      const int ul = base + lane;
      const bool valid = ul < n_it;
      FxUnit u;
      u.b = 0; u.h = 0; u.tile = 0; u.biased = 0; u.gi = 0;
      if (valid) u = FxWalk(u0 + ul, p.B, HG, fp.tiles, nbi, s_img).get();
      const bool isb = valid && u.biased, isu = valid && !u.biased;
      const unsigned mb = __ballot_sync(0xffffffffu, isb);
      const unsigned prev = mb & lt;
      const int pl = prev ? 31 - __clz(prev) : 0;
      int bprev = __shfl_sync(0xffffffffu, u.b, pl);
      if (!prev) bprev = c_lastb;
      const bool newimg = isb && u.b != bprev;
      const unsigned mn = __ballot_sync(0xffffffffu, newimg);
      const int li = c_li + __popc(mn & (lt | (1u << lane)));
      const int nh = valid ? ((p.H - u.h * CF::G) < CF::G ? (p.H - u.h * CF::G) : CF::G) : 0;
      int sb = isb ? nh : 0, su = isu ? nh : 0;            // inclusive warp scans of the head counts
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int tb = __shfl_up_sync(0xffffffffu, sb, o), tu = __shfl_up_sync(0xffffffffu, su, o);
        if (lane >= o) { sb += tb; su += tu; }
      }
      const int joff = isb ? c_sj + sb - nh : c_uj + su - nh;
      if (valid) s_unit[ul] = make_uint4((unsigned)u.b | ((unsigned)u.h << 8) | ((unsigned)u.tile << 16),
                                         (unsigned)u.biased | ((unsigned)(li < 0 ? 0 : li) << 4) | ((unsigned)nh << 8),
                                         (unsigned)joff, 0u);
      if (newimg && li < kMaxLocal) { s_lb[li] = u.b; s_lp[li] = u.gi; }
      c_sj += __shfl_sync(0xffffffffu, sb, 31);
      c_uj += __shfl_sync(0xffffffffu, su, 31);
      c_li += __popc(mn);
      if (mb) c_lastb = __shfl_sync(0xffffffffu, u.b, 31 - __clz(mb));
    }
    __syncwarp();
    const int ns = c_sj, nuj = c_uj;
    for (int ul = lane; ul < n_it; ul += 32) {
      const uint4 r = s_unit[ul];
      const unsigned bi = r.y & 1u, li = (r.y >> 4) & 3u, nh = (r.y >> 8) & 0xffu, hg = (r.x >> 8) & 0xffu;
      const unsigned base_x = (r.x & 0xffu) | (r.x & 0xffff0000u);
      for (unsigned hl = 0; hl < nh; ++hl) {
        const unsigned x = base_x | ((hg * CF::G + hl) << 8);
        const unsigned fl = li << 4;
        if (bi) {
          s_jobs[r.z + hl] = make_uint2(x, fl | JF_BIASED);
          s_jobs[ns + nuj + r.z + hl] = make_uint2(x, fl | JF_BIASED | JF_MAIN);
        } else {
          s_jobs[ns + r.z + hl] = make_uint2(x, fl | JF_MAIN);
        }
      }
    }
    if (lane == 0) { s_njobs = 2 * ns + nuj; s_nstat = ns; s_nl = c_li + 1; }
  }
  for (int i = threadIdx.x; i < core::kWarps * kMaxLocal; i += blockDim.x) {
    StatPartial sp;
    sp.vmax = -INFINITY; sp.sum = 0.0; sp.sumsq = 0.0; sp.pad = 0.0;
    s_part[i / kMaxLocal][i % kMaxLocal] = sp;
  }
  __syncthreads();
  const int nb = s_nb;
  const int njobs = s_njobs, ns = s_nstat, nl = s_nl;
  if (fp.jobs_dump != nullptr) {                              // debug: the job table as built on the device
    unsigned* d = fp.jobs_dump + (size_t)blockIdx.x * (2 + 2 * kMaxJobs);
    if (threadIdx.x == 0) { d[0] = (unsigned)njobs; d[1] = (unsigned)ns; }
#pragma unroll 1
    for (int i = threadIdx.x; i < njobs; i += blockDim.x) { d[2 + 2 * i] = s_jobs[i].x; d[3 + 2 * i] = s_jobs[i].y; }
  }
  const int nu_img = p.B - nb;
  const int np = nb < nu_img ? nb : nu_img;
  const int nuj = njobs - 2 * ns;                             // softmax jobs of unbiased units

  if (blockIdx.x == 0 && p.stats_out != nullptr)            // images without a weight map report statistic 0
#pragma unroll 1
    for (int b = threadIdx.x; b < p.B; b += blockDim.x)
      if (s_widx[b] < 0) p.stats_out[b] = 0.f;
  if (warp == 1) {
    // how many CTAs publish a partial for each of my local biased images, and which statistic each one takes
#pragma unroll 1
    for (int l = 0; l < nl && l < kMaxLocal; ++l) {
      int e = 0;
      const int pos = s_lp[l];
#pragma unroll 1
      for (int c = lane; c < (int)gridDim.x; c += 32) e += fx_cta_has_image(c, gridDim.x, fp.units, pos, HG, fp.tiles, np) ? 1 : 0;
      e = __reduce_add_sync(0xffffffffu, e);
      if (lane == 0) { s_expect[l] = e; s_ismax[l] = image_is_max(p, s_lb[l]); }
    }
  } else if (warp == 2) {
    for (int idx = lane; idx < nl * CW && idx < kMaxLocal * CW; idx += 32) {
      const int l = idx / CW, t = idx - l * CW;
      const bool real = t % core::kTP < core::chunk_keys<KC>(T);
      s_cidx[l][t] = real ? fp.cidx[(int64_t)s_widx[s_lb[l]] * CW + t] : (signed char)-1;
    }
  }

  // the copies of job i into stage i % 2 (stage 0 when there is one)
  auto stage = [&](int i) { return (uint32_t)(CF::NST == 2 ? (i & 1) : 0) * CF::STAGE; };
  // RGN: the chunks some row of softmax job i's tile weighs (bit c = chunk c), also left for the job in the mask word
  // of slot i & 1.  Consecutive jobs of one (image, tile) -- the heads of a unit -- reuse the last scan.
  struct RegionScan { unsigned key = ~0u, bits = 0u; };
  struct NoScan {};
  [[maybe_unused]] std::conditional_t<RGN, RegionScan, NoScan> rgs;
  [[maybe_unused]] auto region_chunks = [&](int i, int b, int tile) -> unsigned {
    if constexpr (!RGN) return 0u;
    else {
    unsigned* words = reinterpret_cast<unsigned*>(smem + CF::SMEM);
    const unsigned key = (unsigned)b | ((unsigned)tile << 8);
    if (key != rgs.key) {                           // CTA-uniform: every thread walks the same job list
      const int ri = fp.rg.rw_index != nullptr ? __ldg(fp.rg.rw_index + b) : b;
      unsigned bits = 1u;                           // no weights: chunk 0 alone
      if (ri >= 0) {
        const int rows = p.N - tile * core::kBM < core::kBM ? p.N - tile * core::kBM : core::kBM;
        const float* wt = fp.rg.rw + (int64_t)ri * fp.rg.rw_bs + (int64_t)tile * core::kBM * KC;
        bits = 0u;
        for (int idx = threadIdx.x; idx < rows * KC; idx += blockDim.x)
          if (__ldg(wt + idx) != 0.f) bits |= 1u << (idx % KC);
        bits = __reduce_or_sync(0xffffffffu, bits);
        if (lane == 0) words[(i & 1) * core::kWarps + warp] = bits;
        __syncthreads();
        bits = 0u;
#pragma unroll
        for (int w = 0; w < core::kWarps; ++w) bits |= words[(i & 1) * core::kWarps + w];
      }
      rgs.key = key;
      rgs.bits = bits;
    }
    if (threadIdx.x == 0) words[2 * core::kWarps + (i & 1)] = rgs.bits;
    return rgs.bits;
    }
  };
  // RGN: the chunks of image b's statistic (bit c = chunk c; chunk 0 always)
  [[maybe_unused]] auto stat_chunks = [&](int b) -> unsigned {
    constexpr unsigned all = (1u << KC) - 1u;
    if constexpr (!RGN) return all;
    else return fp.rg.stat_chunks != nullptr ? ((unsigned)__ldg(fp.rg.stat_chunks + b) | 1u) & all : all;
  };
  auto issue = [&](int i) {
    const uint2 r = s_jobs[i];
    const int b = r.x & 0xff, h = (r.x >> 8) & 0xff, tile = r.x >> 16;
    const bool is_main = (r.y & JF_MAIN) != 0, biased = (r.y & JF_BIASED) != 0;
    const uint32_t st = smem0 + stage(i);
    if constexpr (RGN) {
      if (is_main) core::load_operands_of<D, KC>(st, p, b, h, tile, region_chunks(i, b, tile), true);
      else core::load_operands_of<D, KC>(st, p, b, h, tile, stat_chunks(b), false);
    } else {
      core::load_operands<D, KC>(st, p, b, h, tile, is_main);
    }
    if (is_main && biased) {
      const int rows = p.N - tile * core::kBM;
      const __half* mp = reinterpret_cast<const __half*>(fp.mpack) + (int64_t)s_widx[b] * fp.mpack_bs + (int64_t)tile * core::kBM * kMW;
      for (int idx = threadIdx.x; idx < core::kBM * (kMW / 8); idx += blockDim.x) {
        const int rr = idx >> 2, c = idx & 3;
        const bool ok = rr < rows;
        ptx::cp_async16(st + CF::OFF_M + (uint32_t)(rr * kMW + c * 8) * 2u, ok ? (const void*)(mp + rr * kMW + c * 8) : fp.mpack,
                        ok ? 16u : 0u);
      }
    }
    ptx::cp_async_commit();
  };

  const float sl2 = p.scale * 1.4426950408889634f;
  const unsigned long long* sync_words = reinterpret_cast<const unsigned long long*>(p.counters + 64);
  float vmax = -INFINITY;                          // this thread's statistic partial of local image cur_li
  double dsum = 0.0, dsq = 0.0;
  int cur_li = -1;
  auto flush = [&]() {
    if (cur_li < 0) return;
    double m = vmax, a = dsum, q = dsq;
    core::warp_reduce_stat(m, a, q);
    if (lane == 0 && cur_li < kMaxLocal) {
      StatPartial sp;
      sp.vmax = m; sp.sum = a; sp.sumsq = q; sp.pad = 1.0;
      s_part[warp][cur_li] = sp;
    }
    vmax = -INFINITY; dsum = 0.0; dsq = 0.0;
  };

  if (njobs > 0) issue(0);
#pragma unroll 1
  for (int i = 0; i < njobs; ++i) {
    if constexpr (CF::NST == 2) {
      if (i + 1 < njobs) {
        issue(i + 1);
        ptx::cp_async_wait<1>();
      } else {
        ptx::cp_async_wait<0>();
      }
    } else {                                        // one stage: job i - 1 is done with it (barrier at the loop's end)
      if (i > 0) issue(i);
      ptx::cp_async_wait<0>();
    }
    __syncthreads();
    if (i == ns && ns > 0 && warp == 0) {
      // ---- publish the CTA's statistic partials: the 8 warps' partials in a fixed order, folded into the image's word ----
      for (int l = 0; l < nl && l < kMaxLocal; ++l) {
        if (!s_ismax[l]) continue;                                 // warp-uniform: one kind per image
        const unsigned k = __reduce_max_sync(0xffffffffu, lane < core::kWarps ? f32_key((float)s_part[lane][l].vmax) : 0u);
        if (lane == 0) {
          unsigned* word = p.counters + 64 + 2 * s_lb[l];          // {max key, count}, see ld_acquire_gpu_u64
          asm volatile("red.relaxed.gpu.global.max.u32 [%0], %1;" ::"l"(word), "r"(k) : "memory");
          // release: the maximum above is visible to whoever acquires the new count
          asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(word + 1) : "memory");
        }
      }
      if (lane < nl && lane < kMaxLocal && !s_ismax[lane]) {       // std images: one lane per local image
        const int lbv = s_lb[lane];
        StatPartial sp = s_part[0][lane];
#pragma unroll 1
        for (int w2 = 1; w2 < core::kWarps; ++w2) {
          sp.sum += s_part[w2][lane].sum;
          sp.sumsq += s_part[w2][lane].sumsq;
        }
        p.partials[(int64_t)lbv * gridDim.x + blockIdx.x] = sp;
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(p.counters + 64 + 2 * lbv + 1) : "memory");
      }
      __syncwarp();
    }
    if (i == ns + nuj && ns > 0) {
      if (warp == 0) {
        // ---- grid barrier: every CTA owning units of my biased images has published its partial ----
        const int G = (int)gridDim.x;
#pragma unroll 1
        for (int l = 0; l < nl && l < kMaxLocal; ++l) {
          const int bl = s_lb[l], pos = s_lp[l];
          const unsigned expect = (unsigned)s_expect[l];
          unsigned long long word = 0;
          if (lane == 0) {
            const long long t0 = clock64();
            while ((unsigned)((word = ptx::ld_acquire_gpu_u64(sync_words + bl)) >> 32) < expect) {
              if (clock64() - t0 > 20000000000LL) {
                printf("pww: grid barrier timeout block %d image %d have %u want %u\n", blockIdx.x, bl,
                       (unsigned)(word >> 32), expect);
                __trap();
              }
            }
          }
          __syncwarp();
          const bool is_max = s_ismax[l];
          double m = -INFINITY, a = 0.0, q = 0.0;
          if (is_max) {
            // the maximum is order independent: every publisher folded its partial into the word with an atomic max
            m = (double)key_f32((unsigned)__shfl_sync(0xffffffffu, (unsigned)word, 0));
          } else {
            (void)ptx::ld_acquire_gpu_u64(sync_words + bl);      // every lane orders its partial loads behind the count
            for (int c = lane; c < G; c += 32)
              if (fx_cta_has_image(c, G, fp.units, pos, HG, fp.tiles, np)) {
                const StatPartial* pp = p.partials + (int64_t)bl * G + c;
                a += __ldcg(&pp->sum);
                q += __ldcg(&pp->sumsq);
              }
            core::warp_reduce_stat(m, a, q);
          }
          if (lane == 0) {
            const int keys = RGN ? core::kChunk * __popc(stat_chunks(bl)) : p.T;
            const float stv = core::stat_value(p, is_max, m, a, q, keys);
            s_coef[l] = (p.g_sigma != nullptr ? image_g(p, bl) : 0.f) * stv;
            if (p.stats_out != nullptr) p.stats_out[bl] = stv;   // every CTA of the image writes the same value
          }
        }
        __syncwarp();
      }
      __syncthreads();
    }
    // ---- the job ----
    const uint2 r = s_jobs[i];
    const int b = r.x & 0xff, h = (r.x >> 8) & 0xff, tile = r.x >> 16;
    const bool is_main = (r.y & JF_MAIN) != 0, biased = (r.y & JF_BIASED) != 0;
    const int li = (r.y >> 4) & 3;
    const uint32_t st = smem0 + stage(i);
    const uint32_t qs = st + (uint32_t)(warp * 16 * C::LD) * 2u;
    const int row0 = tile * core::kBM + warp * 16;
    const int kv = core::chunk_keys<KC>(T);
    if (!is_main) {
      if (li != cur_li) { flush(); cur_li = li; }
      float sum = 0.f, sumsq = 0.f;
      [[maybe_unused]] const unsigned sc = stat_chunks(b);
#pragma unroll 1
      for (int c = 0; c < KC; ++c) {                // the real tokens of every chunk (RGN: of the image's statistic)
        if constexpr (RGN) {
          if (!((sc >> c) & 1u)) continue;
        }
        float s[10][4];
        core::warp_qk<D, E>(qs, st + C::QBYTES + c * C::KBYTES, lane, s);
        core::warp_stat<E>(s, kv, p.N - row0, lane, s_ismax[li], vmax, sum, sumsq);
      }
      dsum += (double)sum;
      dsq += (double)sumsq;
      if (i == ns - 1) flush();
    } else if constexpr (RGN) {
      const float x = biased ? s_coef[li] : 0.f;
      const __half* mrow = reinterpret_cast<const __half*>(smem + stage(i) + CF::OFF_M) + (warp * 16 + (lane >> 2)) * kMW;
      const unsigned cm = reinterpret_cast<const unsigned*>(smem + CF::SMEM)[2 * core::kWarps + (i & 1)];
      const int ri = fp.rg.rw_index != nullptr ? __ldg(fp.rg.rw_index + b) : b;
      const int ra = row0 + (lane >> 2), rb = ra + 8;          // this thread's two query rows
      const float* wr = fp.rg.rw + (int64_t)(ri < 0 ? 0 : ri) * fp.rg.rw_bs;
      float o[C::NT][4];
#pragma unroll
      for (int j = 0; j < C::NT; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
#pragma unroll 1
      for (int c = 0; c < KC; ++c) {
        if (!((cm >> c) & 1u)) continue;                       // no row of the tile weighs chunk c: not even copied
        float w0 = c == 0 ? 1.f : 0.f, w1 = w0;
        if (ri >= 0) {
          w0 = ra < p.N ? __ldg(wr + (int64_t)ra * KC + c) : 0.f;
          w1 = rb < p.N ? __ldg(wr + (int64_t)rb * KC + c) : 0.f;
        }
        if (!__any_sync(0xffffffffu, w0 != 0.f || w1 != 0.f)) continue;   // nor of this warp's 16 rows
        float s[10][4];
        core::warp_qk<D, E>(qs, st + C::QBYTES + c * C::KBYTES, lane, s);
        if (biased) {
          const signed char* ci = s_cidx[li] + c * core::kTP;
#pragma unroll
          for (int j = 0; j < 10; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const int cc = ci[core::tok(j, e, lane)];
              if (cc >= 0) {
                const __half* mr = mrow + (e >> 1) * 8 * kMW;
                s[j][e] = fmaf(x, __half2float(mr[cc]) + __half2float(mr[kRC + cc]), s[j][e]);
              }
            }
        }
        core::warp_weighted_chunk<D, E>(s, kv, sl2, st + C::QBYTES + (KC + c) * C::KBYTES, lane, w0, w1, o);
      }
      core::warp_store<D>(o, smem + stage(i) + warp * 16 * C::LD * 2, lane, p.out + (int64_t)b * p.o_bs + h * D, p.o_rs,
                          row0, p.N);
    } else {
      const float x = biased ? s_coef[li] : 0.f;
      const __half* mrow = reinterpret_cast<const __half*>(smem + stage(i) + CF::OFF_M) + (warp * 16 + (lane >> 2)) * kMW;
      float o[C::NT][4], m0, m1, l0, l1;
      core::warp_online_begin<D>(o, m0, m1, l0, l1);
      [[maybe_unused]] float rm[2][4] = {};                          // REC: region mass of the warp's rows
      [[maybe_unused]] int ri = -1;
      [[maybe_unused]] const int8_t* rrow = nullptr;                // REC: the image's token -> region row, or none
      if constexpr (REC) {
        ri = __ldg(fp.rec.rec_index + b);
        if (ri >= 0) rrow = fp.rec.ridx + (int64_t)ri * CW;
      }
#pragma unroll 1
      for (int c = 0; c < KC; ++c) {
        float s[10][4];
        core::warp_qk<D, E>(qs, st + C::QBYTES + c * C::KBYTES, lane, s);
        if (biased) {
          const signed char* ci = s_cidx[li] + c * core::kTP;
#pragma unroll
          for (int j = 0; j < 10; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const int cc = ci[core::tok(j, e, lane)];
              if (cc >= 0) {
                const __half* mr = mrow + (e >> 1) * 8 * kMW;
                s[j][e] = fmaf(x, __half2float(mr[cc]) + __half2float(mr[kRC + cc]), s[j][e]);
              }
            }
        }
        if constexpr (REC) {
          core::warp_online_chunk<D, E>(s, kv, sl2, st + C::QBYTES + (KC + c) * C::KBYTES, lane, o, m0, m1, l0, l1,
                                        [&](const auto& pa, float a0, float a1) {
                                          if (rrow != nullptr) core::warp_region_chunk<E>(pa, a0, a1, rrow + c * core::kTP, lane, rm);
                                        });
        } else {
          core::warp_online_chunk<D, E>(s, kv, sl2, st + C::QBYTES + (KC + c) * C::KBYTES, lane, o, m0, m1, l0, l1);
        }
      }
      if constexpr (REC) {
        if (rrow != nullptr)
          core::warp_region_add(rm, l0, l1, fp.rec.rec_acc + (int64_t)ri * fp.rec.rec_bs + (int64_t)h * p.N * core::kRegions,
                                row0, p.N, lane);
      }
      core::warp_online_end<D>(o, l0, l1);
      core::warp_store<D>(o, smem + stage(i) + warp * 16 * C::LD * 2, lane, p.out + (int64_t)b * p.o_bs + h * D, p.o_rs,
                          row0, p.N);
    }
    __syncthreads();
  }
  // the last CTA to leave resets the arrival counters for the next launch (every waiter has passed its barrier)
  __syncthreads();
  if (threadIdx.x == 0 && nb > 0) {
    __threadfence();
    const unsigned prev = atomicAdd(p.counters + kMaxBatch, 1u);
    if (prev == gridDim.x - 1u) {
#pragma unroll 1
      for (int b = 0; b < kMaxBatch + 1; ++b) p.counters[b] = 0u;
#pragma unroll 1
      for (int b = 0; b < 2 * kMaxBatch; ++b) p.counters[64 + b] = 0u;      // sync words: maximum back to "-infinity", count 0
      __threadfence();
    }
  }
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
  int g = num_sms();
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
  std::vector<int> img(B > 0 ? B : 0);
  const int nb = partition_images(B, wmap_index, img.data());
  const int pos = (int)(std::find(img.begin(), img.begin() + nb, b) - img.begin());   // b's place among the biased images
  if (pos == nb) return 0;
  const int nu = B - nb, np = nb < nu ? nb : nu;
  return fx_cta_has_image(cta, grid, B * H * tiles, pos, H, tiles, np) ? 1 : 0;
}

// A launch fits when every CTA's unit range touches at most kMaxLocal biased images and holds at most kMaxUnits units
// (job table in shared memory); the C ABI halves the images per launch until it does.
inline bool fused2_fits(int B, int hg, int tiles, int grid) {
  const long long units = (long long)B * hg * tiles;
  return fused_range_ok(B, hg, tiles, grid) && fused_units_ok(units, grid) && (units + grid - 1) / grid + 1 <= kMaxUnits;
}

template <int D, int KC, typename E, bool REC, bool RGN = false>
cudaError_t launch_fused2_instance(const FxArgs<E, REC, RGN>& fp, cudaStream_t s) {
  using CF = Cfg2<D, KC>;
  constexpr uint32_t smem_bytes = RGN ? CF::SMEM_RGN : CF::SMEM;
  const cudaError_t e = allow_dynamic_smem<xattn_fused2_kernel<D, KC, E, REC, RGN>>(smem_bytes);
  if (e != cudaSuccess) return e;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(fp.grid);
  cfg.blockDim = dim3(core::kThreads);
  cfg.dynamicSmemBytes = smem_bytes;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;     // all CTAs co-resident: the in-kernel grid barrier cannot deadlock
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, xattn_fused2_kernel<D, KC, E, REC, RGN>, fp);
}

// rec == NULL: the plain instance; else the recording instance with *rec (rec_index starting at this launch's image 0).
// rg != NULL: the region-prompt instance with *rg (KC = 2, 3 only; rec must be NULL).
template <int D, int KC, typename E>
cudaError_t launch_fused2(const XattnParams<E>& x, const void* mpack, int64_t mpack_bs, const int8_t* cidx, cudaStream_t s,
                          const FxRecord* rec = nullptr, const FxRegion* rg = nullptr) {
  using CF = Cfg2<D, KC>;
  FxParams<E> fp;
  memset(&fp, 0, sizeof(fp));
  fp.x = x;
  fp.cidx = cidx;
  fp.mpack = mpack;
  fp.mpack_bs = mpack_bs;
  fp.tiles = ceil_div(x.N, core::kBM);
  fp.hg = ceil_div(x.H, CF::G);
  fp.units = x.B * fp.tiles * fp.hg;
  fp.grid = fused_grid(fp.units);
  fp.jobs_dump = debug_jobs_dump();
  if (!fused2_fits(x.B, fp.hg, fp.tiles, fp.grid)) return cudaErrorInvalidConfiguration;
  if (rg != nullptr) {
    if constexpr (KC > 1) {
      if (rec != nullptr) return cudaErrorInvalidValue;
      FxRgnParams<E> gp;
      memset(&gp, 0, sizeof(gp));
      static_cast<FxParams<E>&>(gp) = fp;
      gp.rg = *rg;
      return launch_fused2_instance<D, KC, E, false, true>(gp, s);
    }
    return cudaErrorInvalidValue;
  }
  if (rec == nullptr) return launch_fused2_instance<D, KC, E, false>(fp, s);
  FxRecParams<E> rp;
  memset(&rp, 0, sizeof(rp));
  static_cast<FxParams<E>&>(rp) = fp;
  rp.rec = *rec;
  return launch_fused2_instance<D, KC, E, true>(rp, s);
}

// Host replay of the job lists (test infrastructure): out[job] = {cta, i, kind, b, h, tile, biased, li} for every job of
// every CTA; returns the number of jobs written.
inline int fused2_schedule_host(int B, int H, int G, int tiles, int grid, const int* wmap_index, int* out, int max_jobs) {
  if (B <= 0 || B > kMaxBatch || H <= 0 || G <= 0 || tiles <= 0 || grid <= 0) return -1;
  int img[kMaxBatch];
  const int nb = partition_images(B, wmap_index, img);
  const int hg = (H + G - 1) / G;
  const int units = B * hg * tiles;
  int row = 0;
  for (int cta = 0; cta < grid; ++cta) {
    int u0, u1;
    fx_range(cta, grid, units, u0, u1);
    Fx2Jobs jobs(u0, u1 - u0, B, H, G, tiles, nb, img);
    Fx2Job jb;
    while (jobs.next(jb)) {
      if (row >= max_jobs) return -2;
      int* o = out + 8 * (row++);
      o[0] = cta; o[1] = jb.i; o[2] = jb.kind; o[3] = jb.b; o[4] = jb.h; o[5] = jb.tile; o[6] = jb.biased; o[7] = jb.li;
    }
  }
  return row;
}

}  // namespace fx
}  // namespace pww
