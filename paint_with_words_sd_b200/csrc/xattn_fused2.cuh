// Paint-with-Words cross-attention in ONE launch (statistic + bias + softmax + P.V) on Hopper tensor cores, keys T <= 80.
//
// The per-image statistic (max or std of Q K^T over all heads, rows and tokens) is a grid-wide dependency of every
// biased score, so the kernel is a persistent cooperative launch (one CTA per SM, all co-resident) that runs three passes
// over its contiguous range of work units:
//     1. statistic jobs of the units of biased images: S = Q K^T, folded into per-warp partials, then published to the
//        image's word in the workspace (max: one atomic max of an order-preserving key; std: a partial slot per CTA,
//        summed by the waiters in CTA order -- deterministic for a given grid);
//     2. softmax jobs of the unbiased units: they need no statistic and overlap the other CTAs' statistic pass;
//     3. grid barrier (per biased image, only the CTAs that publish for it), then the softmax jobs of the biased units
//        with the bias x * W, x = g(sigma) * fp16(statistic), W rebuilt from the packed map (xattn_fused.cuh).
// Work unit = (image, 128-row tile, group of G heads); a unit expands into one job per head.  Each job is computed by the
// 8 warps of the CTA with the warp-level MMA tiles of xattn_core.cuh; the cp.async copies of job i + 1 (Q rows, K, V
// and, for biased softmax jobs, the row tile's packed map) are in flight while job i is computed.
#pragma once
#include "mma_sm90.cuh"
#include "pww_common.cuh"
#include "xattn_core.cuh"
#include "xattn_tc.cuh"      // num_sms, cur_device, tc_error_buf
#include "xattn_fused.cuh"   // FxWalk, fx_range, fx_cta_has_image, debug knobs

namespace pww {
namespace fx2 {
using namespace fx;   // unit walk, helpers and constants shared with the host replay

template <int D>
struct Cfg2 {
  // heads per unit (the granularity of a CTA's range): 2 at head dims 40 and 64, one head at 80 and 160
  static constexpr int G = (D == 40 || D == 64) ? 2 : 1;
  using T_ = core::Tile<D>;
  static constexpr uint32_t MBYTES = kBM * kMW * 2;                    // packed-map rows of the row tile
  static constexpr uint32_t OFF_M = T_::QBYTES + 2 * T_::KBYTES;
  static constexpr uint32_t STAGE = OFF_M + MBYTES;                    // Q | K | V | map of one job
  static constexpr uint32_t SMEM = 2 * STAGE;
  static_assert(SMEM + 8192 <= 232448, "shared memory budget (dynamic + ~7 KB of static tables incl. the 4 KB job table)");
};

// ------------------------------------------------------------------------------------------------------------------
// job lists (shared by the kernel and the host replay)
// ------------------------------------------------------------------------------------------------------------------
// ------------------------------------------------------------------------------------------------------------------
// job lists (shared by the kernel and the host replay)
// ------------------------------------------------------------------------------------------------------------------
// Units are walked with the per-head kernel's FxWalk, "heads" being head GROUPS (hg = ceil(H / G) of them); a unit
// expands into one job per head of its group.  A CTA runs three passes over its contiguous unit range, as in the
// per-head kernel: statistic jobs of the biased units, softmax jobs of the unbiased units, softmax jobs of the biased
// units.  `up` numbers the unit passes in processing order (Q ring), `ul` is the unit's position in the CTA's range.
struct Fx2Job {
  int b, h, tile, biased, gi;
  int kind;     // 0 = stat, 1 = main
  int i;        // job index (score slot = i % NS, softmax group = i % 2, K stage = i % NK)
  int m;        // main-job index (V stage = m % NV), -1 for stat jobs
  int li;       // local index of the biased image inside this CTA's range (biased jobs)
  int up, ul;   // unit pass / local unit
  int first, last;   // first / last job of its unit pass
};
struct Fx2Jobs {
  FxWalk w;
  int u0, n_units, B, H, HG, G, tiles, nb;
  const int* img;
  int it, phase, i, m, li, lastb, up;
  FxUnit cur;
  int cur_ul, cur_up, cur_li, hl, nh;
  bool have;
  __host__ __device__ __forceinline__ Fx2Jobs(int u0_, int n_units_, int B_, int H_, int G_, int tiles_, int nb_,
                                              const int* img_)
      : u0(u0_), n_units(n_units_), B(B_), H(H_), G(G_), tiles(tiles_), nb(nb_), img(img_) {
    HG = (H + G - 1) / G;
    phase = nb > 0 ? 0 : 1;
    i = 0; m = 0; up = 0;
    rewind();
  }
  __host__ __device__ __forceinline__ void rewind() {
    w = FxWalk(u0, B, HG, tiles, nb, img);
    it = 0; li = -1; lastb = -1; have = false;
  }
  __host__ __device__ __forceinline__ bool next(Fx2Job& jb) {
    for (;;) {
      if (have) {
        jb.b = cur.b; jb.h = cur.h * G + hl; jb.tile = cur.tile; jb.biased = cur.biased; jb.gi = cur.gi;
        jb.kind = phase == 0 ? 0 : 1;
        jb.i = i++;
        jb.m = phase == 0 ? -1 : m++;
        jb.li = cur.biased ? cur_li : -1;
        jb.up = cur_up; jb.ul = cur_ul;
        jb.first = hl == 0; jb.last = hl == nh - 1;
        if (++hl == nh) have = false;
        return true;
      }
      while (it < n_units) {
        const FxUnit u = w.get();
        w.next();
        const int ul = it++;
        if (u.biased && u.b != lastb) { ++li; lastb = u.b; }
        const bool want = (phase == 1) ? !u.biased : (u.biased != 0);
        if (!want) continue;
        cur = u; cur_ul = ul; cur_li = li; cur_up = up++;
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
constexpr uint32_t JF_MAIN = 1u, JF_BIASED = 2u, JF_FIRST = 4u, JF_LAST = 8u;   // | li << 4 (2 bits) | ul << 8 (8 bits)

// Order-preserving map float -> unsigned (0 is below every real number: a zero-filled workspace reads as -infinity).
__device__ __forceinline__ unsigned f32_key(float f) {
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_f32(unsigned k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

template <int D>
__global__ void __launch_bounds__(core::kThreads, 1) xattn_fused2_kernel(const FxParams fp) {
  using C = core::Tile<D>;
  using CF = Cfg2<D>;
  const XattnParams& p = fp.x;
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
  __shared__ StatPartial s_part[core::kWarps][kMaxLocal];   // [warp][local biased image]
  __shared__ uint2 s_jobs[kMaxJobs];
  __shared__ uint4 s_unit[kMaxUnits];              // job-table build scratch: one entry per unit of the range
  __shared__ int s_expect[kMaxLocal];              // CTAs that publish a partial for each local biased image
  __shared__ signed char s_cidx[kMaxLocal][kTP];   // token -> dictionary column of the CTA's local biased images

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
        const unsigned fl = (hl == 0 ? JF_FIRST : 0u) | (hl == nh - 1 ? JF_LAST : 0u) | (li << 4) | ((unsigned)(ul & 0xff) << 8);
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
    // how many CTAs publish a partial for each of my local biased images
#pragma unroll 1
    for (int l = 0; l < nl && l < kMaxLocal; ++l) {
      int e = 0;
      const int pos = s_lp[l];
#pragma unroll 1
      for (int c = lane; c < (int)gridDim.x; c += 32) e += fx_cta_has_image(c, gridDim.x, fp.units, pos, HG, fp.tiles, np) ? 1 : 0;
      e = __reduce_add_sync(0xffffffffu, e);
      if (lane == 0) s_expect[l] = e;
    }
  } else if (warp == 2) {
    for (int idx = lane; idx < nl * kTP && idx < kMaxLocal * kTP; idx += 32) {
      const int l = idx / kTP, t = idx - l * kTP;
      s_cidx[l][t] = (t < T) ? fp.cidx[(int64_t)s_widx[s_lb[l]] * kTP + t] : (signed char)-1;
    }
  }

  // the copies of job i into stage i % 2
  auto issue = [&](int i) {
    const uint2 r = s_jobs[i];
    const int b = r.x & 0xff, h = (r.x >> 8) & 0xff, tile = r.x >> 16;
    const bool is_main = (r.y & JF_MAIN) != 0, biased = (r.y & JF_BIASED) != 0;
    const uint32_t st = smem0 + (i & 1) * CF::STAGE;
    const int rows = p.N - tile * kBM < kBM ? p.N - tile * kBM : kBM;
    core::load_rows<D>(st, p.q + (int64_t)b * p.q_bs + (int64_t)tile * kBM * p.q_rs + h * D, p.q_rs, kBM, rows);
    core::load_rows<D>(st + C::QBYTES, p.k + (int64_t)b * p.k_bs + h * D, p.k_rs, kTP, T);
    if (is_main) core::load_rows<D>(st + C::QBYTES + C::KBYTES, p.v + (int64_t)b * p.k_bs + h * D, p.k_rs, kTP, T);
    if (is_main && biased) {
      const __half* mp = reinterpret_cast<const __half*>(fp.mpack) + (int64_t)s_widx[b] * fp.mpack_bs + (int64_t)tile * kBM * kMW;
      for (int idx = threadIdx.x; idx < kBM * (kMW / 8); idx += blockDim.x) {
        const int rr = idx >> 2, c = idx & 3;
        const bool ok = rr < rows;
        ptx::cp_async16(st + CF::OFF_M + (uint32_t)(rr * kMW + c * 8) * 2u, ok ? (const void*)(mp + rr * kMW + c * 8) : fp.mpack,
                        ok ? 16u : 0u);
      }
    }
    ptx::cp_async_commit();
  };

  const float sl2 = p.scale * 1.4426950408889634f;
  const bool is_max = p.stat == PWW_STAT_MAX;
  const float gsig = (nb > 0 && p.g_sigma != nullptr) ? __ldg(p.g_sigma) : 0.f;
  const unsigned long long* sync_words = reinterpret_cast<const unsigned long long*>(p.counters + 64);
  float vmax = -INFINITY;                          // this thread's statistic partial of local image cur_li
  double dsum = 0.0, dsq = 0.0;
  int cur_li = -1;
  auto flush = [&]() {
    if (cur_li < 0) return;
    double m = vmax, a = dsum, q = dsq;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
      a += __shfl_xor_sync(0xffffffffu, a, o);
      q += __shfl_xor_sync(0xffffffffu, q, o);
    }
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
    if (i + 1 < njobs) {
      issue(i + 1);
      ptx::cp_async_wait<1>();
    } else {
      ptx::cp_async_wait<0>();
    }
    __syncthreads();
    if (i == ns && ns > 0 && warp == 0) {
      // ---- publish the CTA's statistic partials: the 8 warps' partials in a fixed order, folded into the image's word ----
      if (is_max) {
        for (int l = 0; l < nl && l < kMaxLocal; ++l) {
          const unsigned k = __reduce_max_sync(0xffffffffu, lane < core::kWarps ? f32_key((float)s_part[lane][l].vmax) : 0u);
          if (lane == 0) {
            unsigned* word = p.counters + 64 + 2 * s_lb[l];        // {max key, count}, see ld_acquire_gpu_u64
            asm volatile("red.relaxed.gpu.global.max.u32 [%0], %1;" ::"l"(word), "r"(k) : "memory");
            // release: the maximum above is visible to whoever acquires the new count
            asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(word + 1) : "memory");
          }
        }
      } else if (lane < nl && lane < kMaxLocal) {
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
#pragma unroll 1
            for (int o = 16; o > 0; o >>= 1) {
              a += __shfl_xor_sync(0xffffffffu, a, o);
              q += __shfl_xor_sync(0xffffffffu, q, o);
            }
          }
          if (lane == 0) {
            const double cnt = (double)p.H * (double)p.N * (double)p.T;
            double rr;
            if (is_max) {
              rr = m;
            } else {
              const double var = (q - a * a / cnt) / (cnt - 1.0);
              rr = sqrt(var > 0.0 ? var : 0.0);
            }
            const float st16 = round_to_f16((float)rr);         // qk.max() / qk.std() return fp16 in the reference
            s_coef[l] = gsig * st16;
            if (p.stats_out != nullptr) p.stats_out[bl] = st16;   // every CTA of the image writes the same value
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
    const uint32_t st = smem0 + (i & 1) * CF::STAGE;
    const int row0 = tile * kBM + warp * 16;
    float s[10][4];
    core::warp_qk<D>(st + (uint32_t)(warp * 16 * C::LD) * 2u, st + C::QBYTES, lane, s);
    if (!is_main) {
      if (li != cur_li) { flush(); cur_li = li; }
      float sum = 0.f, sumsq = 0.f;
      core::warp_stat(s, T, p.N - row0, lane, is_max, vmax, sum, sumsq);
      dsum += (double)sum;
      dsq += (double)sumsq;
      if (i == ns - 1) flush();
    } else {
      if (biased) {
        const float x = s_coef[li];
        const signed char* ci = s_cidx[li];
        const __half* mrow = reinterpret_cast<const __half*>(smem + (i & 1) * CF::STAGE + CF::OFF_M) + (warp * 16 + (lane >> 2)) * kMW;
#pragma unroll
        for (int j = 0; j < 10; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int c = ci[core::tok(j, e, lane)];
            if (c >= 0) {
              const __half* mr = mrow + (e >> 1) * 8 * kMW;
              s[j][e] = fmaf(x, __half2float(mr[c]) + __half2float(mr[kRC + c]), s[j][e]);
            }
          }
      }
      float o[C::NT][4];
      core::warp_softmax_pv<D>(s, T, sl2, st + C::QBYTES + C::KBYTES, lane, o);
      core::warp_store<D>(o, smem + (i & 1) * CF::STAGE + warp * 16 * C::LD * 2, lane, p.out + (int64_t)b * p.o_bs + h * D,
                          p.o_rs, row0, p.N);
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
// A launch fits when every CTA's unit range touches at most kMaxLocal biased images and holds at most kMaxUnits units
// (job table in shared memory); the C ABI halves the images per launch until it does.
inline bool fused2_fits(int B, int hg, int tiles, int grid) {
  const long long units = (long long)B * hg * tiles;
  return fused_range_ok(B, hg, tiles, grid) && fused_units_ok(units, grid) && (units + grid - 1) / grid + 1 <= kMaxUnits;
}

template <int D>
cudaError_t launch_fused2(const XattnParams& x, const void* mpack, int64_t mpack_bs, const int8_t* cidx, cudaStream_t s) {
  using CF = Cfg2<D>;
  FxParams fp;
  memset(&fp, 0, sizeof(fp));
  fp.x = x;
  fp.cidx = cidx;
  fp.mpack = mpack;
  fp.mpack_bs = mpack_bs;
  fp.tiles = ceil_div(x.N, kBM);
  fp.hg = ceil_div(x.H, CF::G);
  fp.units = x.B * fp.tiles * fp.hg;
  fp.grid = fused_grid(fp.units);
  fp.jobs_dump = debug_jobs_dump();
  if (!fused2_fits(x.B, fp.hg, fp.tiles, fp.grid)) return cudaErrorInvalidConfiguration;
  static bool attr_set[tc::kMaxDevices] = {false};
  if (!attr_set[tc::cur_device()]) {
    cudaError_t e = cudaFuncSetAttribute(xattn_fused2_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, CF::SMEM);
    if (e != cudaSuccess) return e;
    attr_set[tc::cur_device()] = true;
  }
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(fp.grid);
  cfg.blockDim = dim3(core::kThreads);
  cfg.dynamicSmemBytes = CF::SMEM;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;     // all CTAs co-resident: the in-kernel grid barrier cannot deadlock
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, xattn_fused2_kernel<D>, fp);
}

// Host replay of the job lists (test infrastructure): out[job] = {cta, i, kind, m, b, h, tile, biased, li, gi, up, ul,
// first, last} for every job of every CTA; returns the number of jobs written.
inline int fused2_schedule_host(int B, int H, int G, int tiles, int grid, const int* wmap_index, int* out, int max_jobs) {
  if (B <= 0 || B > kMaxBatch || H <= 0 || G <= 0 || tiles <= 0 || grid <= 0) return -1;
  int img[kMaxBatch];
  int nb = 0;
  for (int b = 0; b < B; ++b) if (wmap_index[b] >= 0) img[nb++] = b;
  int nu = 0;
  for (int b = 0; b < B; ++b) if (wmap_index[b] < 0) img[nb + nu++] = b;
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
      int* o = out + 14 * (row++);
      o[0] = cta; o[1] = jb.i; o[2] = jb.kind; o[3] = jb.m; o[4] = jb.b; o[5] = jb.h; o[6] = jb.tile; o[7] = jb.biased;
      o[8] = jb.li; o[9] = jb.gi; o[10] = jb.up; o[11] = jb.ul; o[12] = jb.first; o[13] = jb.last;
    }
  }
  return row;
}

}  // namespace fx2
}  // namespace pww
