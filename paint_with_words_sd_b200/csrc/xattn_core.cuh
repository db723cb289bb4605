// Warp-level building blocks of the attention kernels on Hopper tensor cores.
//
// A CTA of 8 warps works on one [128-row x head] tile at a time; warp w owns query rows [16 w, 16 w + 16).  Operands are
// staged in shared memory by 16-byte cp.async copies (rows of LD = DP + 8 halfs: the 16-byte pad makes every ldmatrix
// phase hit 8 distinct bank groups), read into registers with ldmatrix and multiplied with mma.m16n8k16 (fp16 in, fp32
// accumulate).  Cross-attention (keys T <= 80):
//     S = Q K^T   16 x 80 per warp, DP / 16 k-steps      accumulators: 10 n-tiles x 4 fp32 per thread
//     P = 2^(log2e * scale * (S + bias - rowmax))        in registers; packed to fp16 it is the A operand of
//     O = P V     16 x D per warp, 5 k-steps over the 80 padded keys, V fragments by ldmatrix.trans
// and O is divided by the row sum of the fp16 P that was multiplied.  Padding (d >= D, token >= T, row >= N) is zero-filled
// by the copies; padded tokens are masked to -inf before the softmax.
#pragma once
#include "mma_sm90.cuh"
#include "pww_common.cuh"

namespace pww {
namespace core {

constexpr int kBM = 128;       // query rows per tile
constexpr int kTP = 80;        // padded key count
constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;

template <int D>
struct Tile {
  static_assert(D == 40 || D == 64 || D == 80 || D == 160, "head dims of SD1.5 (40 / 80 / 160) and SD2.x (64)");
  static constexpr int DP = (D + 15) / 16 * 16;    // k extent of Q K^T
  static constexpr int LD = DP + 8;                // shared-memory row stride in halfs
  static constexpr int KS = DP / 16;
  static constexpr int NT = D / 8;                 // n-tiles of P V
  static constexpr uint32_t QBYTES = kBM * LD * 2;
  static constexpr uint32_t KBYTES = kTP * LD * 2;
};

// Block-cooperative copy of rows [0, nrows) of a [rows x D] fp16 head slice (row stride rs elements) into shared rows of
// LD halfs.  Rows >= valid and columns D .. DP-1 are zero-filled.
template <int D>
__device__ __forceinline__ void load_rows(uint32_t dst, const __half* src, int64_t rs, int nrows, int valid) {
  using C = Tile<D>;
  constexpr int CH = C::DP / 8, DCH = D / 8;
  for (int idx = threadIdx.x; idx < nrows * CH; idx += blockDim.x) {
    const int r = idx / CH, c = idx - r * CH;
    const bool ok = r < valid && c < DCH;
    ptx::cp_async16(dst + (uint32_t)(r * C::LD + c * 8) * 2u, ok ? (const void*)(src + (int64_t)r * rs + c * 8) : (const void*)src,
                    ok ? 16u : 0u);
  }
}

// S (16 x 80) of the warp's rows: qs = shared address of the warp's first Q row, ks = the K tile.
template <int D>
__device__ __forceinline__ void warp_qk(uint32_t qs, uint32_t ks, int lane, float (&s)[10][4]) {
  using C = Tile<D>;
#pragma unroll
  for (int j = 0; j < 10; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
  for (int kk = 0; kk < C::KS; ++kk) {
    uint32_t a[4];
    ptx::ldsm_x4(qs + (uint32_t)((lane & 15) * C::LD + kk * 16 + (lane >> 4) * 8) * 2u, a[0], a[1], a[2], a[3]);
#pragma unroll
    for (int jp = 0; jp < 5; ++jp) {
      const int t = 16 * jp + (lane & 7) + ((lane >> 4) << 3), d = kk * 16 + ((lane >> 3) & 1) * 8;
      uint32_t b0, b1, b2, b3;
      ptx::ldsm_x4(ks + (uint32_t)(t * C::LD + d) * 2u, b0, b1, b2, b3);
      ptx::mma16816(s[2 * jp], a, b0, b1);
      ptx::mma16816(s[2 * jp + 1], a, b2, b3);
    }
  }
}

// Token of accumulator element e of n-tile j for this lane; the row is lane / 4 (+ 8 for e >= 2).
__device__ __forceinline__ int tok(int j, int e, int lane) { return 8 * j + 2 * (lane & 3) + (e & 1); }

// Softmax of the warp's 16 rows over the T real tokens (s already holds S + bias) followed by O = P V, normalised.
template <int D>
__device__ __forceinline__ void warp_softmax_pv(float (&s)[10][4], int T, float sl2, uint32_t vs, int lane,
                                                float (&o)[Tile<D>::NT][4]) {
  using C = Tile<D>;
  float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
  for (int j = 0; j < 10; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (tok(j, e, lane) >= T) s[j][e] = -INFINITY;
      if (e < 2) m0 = fmaxf(m0, s[j][e]); else m1 = fmaxf(m1, s[j][e]);
    }
  m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1));
  m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
  m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1));
  m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
  const float n0 = -m0 * sl2, n1 = -m1 * sl2;
  uint32_t pa[5][4];
  float l0 = 0.f, l1 = 0.f;
#pragma unroll
  for (int j = 0; j < 10; ++j) {
    const uint32_t p01 = ptx::pack_h2(ptx::ex2(fmaf(s[j][0], sl2, n0)), ptx::ex2(fmaf(s[j][1], sl2, n0)));
    const uint32_t p23 = ptx::pack_h2(ptx::ex2(fmaf(s[j][2], sl2, n1)), ptx::ex2(fmaf(s[j][3], sl2, n1)));
    const float2 f01 = ptx::unpack_h2(p01), f23 = ptx::unpack_h2(p23);    // sum exactly what the MMA multiplies
    l0 += f01.x + f01.y;
    l1 += f23.x + f23.y;
    pa[j >> 1][(j & 1) * 2] = p01;
    pa[j >> 1][(j & 1) * 2 + 1] = p23;
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
#pragma unroll
  for (int j = 0; j < C::NT; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
#pragma unroll
  for (int kk = 0; kk < 5; ++kk) {
    const int t = 16 * kk + (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
    for (int jp = 0; jp < C::NT / 2; ++jp) {
      uint32_t b0, b1, b2, b3;
      ptx::ldsm_x4_t(vs + (uint32_t)(t * C::LD + 16 * jp + (lane >> 4) * 8) * 2u, b0, b1, b2, b3);
      ptx::mma16816(o[2 * jp], pa[kk], b0, b1);
      ptx::mma16816(o[2 * jp + 1], pa[kk], b2, b3);
    }
    if constexpr (C::NT & 1) {
      uint32_t b0, b1;
      ptx::ldsm_x2_t(vs + (uint32_t)(t * C::LD + 8 * (C::NT - 1)) * 2u, b0, b1);
      ptx::mma16816(o[C::NT - 1], pa[kk], b0, b1);
    }
  }
  const float i0 = 1.f / l0, i1 = 1.f / l1;
#pragma unroll
  for (int j = 0; j < C::NT; ++j) {
    o[j][0] *= i0; o[j][1] *= i0; o[j][2] *= i1; o[j][3] *= i1;
  }
}

// Normalised O of the warp's 16 rows -> fp16 in global memory: staged over the warp's own Q rows in shared memory (dead
// once S exists), then written as whole 16-byte pieces of each row.  Rows >= N are dropped.
template <int D>
__device__ __forceinline__ void warp_store(const float (&o)[Tile<D>::NT][4], unsigned char* stage, int lane, __half* out,
                                           int64_t o_rs, int row0, int N) {
  using C = Tile<D>;
  __syncwarp();
  const int g = lane >> 2, q = lane & 3;
#pragma unroll
  for (int j = 0; j < C::NT; ++j) {
    *reinterpret_cast<uint32_t*>(stage + (g * C::LD + 8 * j + 2 * q) * 2) = ptx::pack_h2(o[j][0], o[j][1]);
    *reinterpret_cast<uint32_t*>(stage + ((g + 8) * C::LD + 8 * j + 2 * q) * 2) = ptx::pack_h2(o[j][2], o[j][3]);
  }
  __syncwarp();
  for (int idx = lane; idx < 16 * C::NT; idx += 32) {
    const int r = idx / C::NT, c = idx - r * C::NT;
    if (row0 + r < N)
      *reinterpret_cast<uint4*>(out + (int64_t)(row0 + r) * o_rs + c * 8) =
          *reinterpret_cast<const uint4*>(stage + (r * C::LD + c * 8) * 2);
  }
  __syncwarp();
}

// Statistic partials of S over the warp's valid elements (row < N, token < T): running max of S (rounding to fp16 is
// monotonic, so the maximum is rounded once at the end) or sum / sum of squares of fp16(S).
__device__ __forceinline__ void warp_stat(const float (&s)[10][4], int T, int rows_left, int lane, bool is_max, float& vmax,
                                          float& sum, float& sumsq) {
  const int g = lane >> 2;
#pragma unroll
  for (int j = 0; j < 10; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const bool ok = tok(j, e, lane) < T && (g + (e >> 1) * 8) < rows_left;
      if (is_max) {
        if (ok) vmax = fmaxf(vmax, s[j][e]);
      } else if (ok) {
        const float h = round_to_f16(s[j][e]);
        sum += h;
        sumsq = fmaf(h, h, sumsq);
      }
    }
}

}  // namespace core
}  // namespace pww
