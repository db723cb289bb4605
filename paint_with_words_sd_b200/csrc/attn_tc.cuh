// Self-attention (context=None in the reference's inj_forward, paint_with_words.py:71-72, 87-118) as a flash attention
// forward on Hopper tensor cores: softmax(scale * Q_h K_h^T) V_h with keys = the image's own N pixels.
//
// One CTA = (image, head, 128 query rows); warp w owns rows [16 w, 16 w + 16) and keeps its Q fragments in registers.
// Key tiles of BN = 64 rows of K and V stream through a two-stage cp.async ring in shared memory (the copies of tile j + 1
// are in flight while tile j is computed):
//     S = Q K_j^T     mma.m16n8k16, 8 n-tiles per warp, fp32 accumulators in registers
//     online softmax: running row max m and row sum l; O and l are rescaled by 2^(m_old - m_new) when the max moves
//     O += P V_j      P packed to fp16 straight from the S accumulators (the C layout of two n-tiles is the A layout of one
//                     k-step), V fragments by ldmatrix.trans
// Padding (d >= D, key >= N, row >= N) is zero-filled by the copies; padded keys of the last tile are masked to -inf.
#pragma once
#include "mma_sm90.cuh"
#include "pww_common.cuh"
#include "xattn_core.cuh"
#include "xattn_tc.cuh"   // num_sms, cur_device

namespace pww {
namespace fa {

constexpr int kThreads = core::kThreads;
constexpr int kBM = core::kBM;
constexpr int kBN = 64;                                    // keys per tile

template <int D>
struct Cfg {
  using T_ = core::Tile<D>;
  static constexpr uint32_t KVBYTES = kBN * T_::LD * 2;
  static constexpr uint32_t OFF_KV = T_::QBYTES;
  static constexpr uint32_t SMEM = T_::QBYTES + 2 * 2 * KVBYTES;   // Q | 2 x (K | V)
  static_assert(SMEM <= 232448, "shared memory budget");
};

struct Params {
  const __half* q;
  const __half* k;
  const __half* v;
  __half* out;
  int B, H, N;
  int64_t bs, rs;          // q/k/v element strides (batch, row)
  int64_t o_bs, o_rs;
  float scale;
};

template <int D>
__global__ void __launch_bounds__(kThreads) attn_fwd_kernel(const Params p) {
  using C = core::Tile<D>;
  using CF = Cfg<D>;
  extern __shared__ __align__(128) unsigned char smem[];
  const uint32_t smem0 = ptx::smem_u32(smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qtiles = (p.N + kBM - 1) / kBM;
  const int bh = blockIdx.x / qtiles, qt = blockIdx.x - bh * qtiles;
  const int b = bh / p.H, h = bh - b * p.H;
  const int row_base = qt * kBM;
  const __half* qb = p.q + (int64_t)b * p.bs + h * D;
  const __half* kb = p.k + (int64_t)b * p.bs + h * D;
  const __half* vb = p.v + (int64_t)b * p.bs + h * D;
  const int ntiles = (p.N + kBN - 1) / kBN;
  auto issue_kv = [&](int j) {
    const uint32_t st = smem0 + CF::OFF_KV + (j & 1) * 2 * CF::KVBYTES;
    const int rows = p.N - j * kBN < kBN ? p.N - j * kBN : kBN;
    core::load_rows<D>(st, kb + (int64_t)j * kBN * p.rs, p.rs, kBN, rows);
    core::load_rows<D>(st + CF::KVBYTES, vb + (int64_t)j * kBN * p.rs, p.rs, kBN, rows);
    ptx::cp_async_commit();
  };
  {
    const int rows = p.N - row_base < kBM ? p.N - row_base : kBM;
    core::load_rows<D>(smem0, qb + (int64_t)row_base * p.rs, p.rs, kBM, rows);
  }
  issue_kv(0);                                     // one group: Q and the first key tile
  uint32_t qa[C::KS][4];
  float o[C::NT][4];
#pragma unroll
  for (int j = 0; j < C::NT; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  const float sl2 = p.scale * 1.4426950408889634f;
  const uint32_t qs = smem0 + (uint32_t)(warp * 16 * C::LD) * 2u;
#pragma unroll 1
  for (int jt = 0; jt < ntiles; ++jt) {
    if (jt + 1 < ntiles) {
      issue_kv(jt + 1);
      ptx::cp_async_wait<1>();
    } else {
      ptx::cp_async_wait<0>();
    }
    __syncthreads();
    if (jt == 0) {
#pragma unroll
      for (int kk = 0; kk < C::KS; ++kk)
        ptx::ldsm_x4(qs + (uint32_t)((lane & 15) * C::LD + kk * 16 + (lane >> 4) * 8) * 2u, qa[kk][0], qa[kk][1], qa[kk][2], qa[kk][3]);
    }
    const uint32_t ks = smem0 + CF::OFF_KV + (jt & 1) * 2 * CF::KVBYTES, vs = ks + CF::KVBYTES;
    float s[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < C::KS; ++kk) {
#pragma unroll
      for (int jp = 0; jp < 4; ++jp) {
        const int t = 16 * jp + (lane & 7) + ((lane >> 4) << 3), d = kk * 16 + ((lane >> 3) & 1) * 8;
        uint32_t b0, b1, b2, b3;
        ptx::ldsm_x4(ks + (uint32_t)(t * C::LD + d) * 2u, b0, b1, b2, b3);
        ptx::mma16816(s[2 * jp], qa[kk], b0, b1);
        ptx::mma16816(s[2 * jp + 1], qa[kk], b2, b3);
      }
    }
    const int valid = p.N - jt * kBN;              // keys of this tile that exist
    float t0 = -INFINITY, t1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (core::tok(j, e, lane) >= valid) s[j][e] = -INFINITY;
        if (e < 2) t0 = fmaxf(t0, s[j][e]); else t1 = fmaxf(t1, s[j][e]);
      }
    t0 = fmaxf(t0, __shfl_xor_sync(0xffffffffu, t0, 1));
    t0 = fmaxf(t0, __shfl_xor_sync(0xffffffffu, t0, 2));
    t1 = fmaxf(t1, __shfl_xor_sync(0xffffffffu, t1, 1));
    t1 = fmaxf(t1, __shfl_xor_sync(0xffffffffu, t1, 2));
    const float mn0 = fmaxf(m0, t0), mn1 = fmaxf(m1, t1);
    const float a0 = ptx::ex2((m0 - mn0) * sl2), a1 = ptx::ex2((m1 - mn1) * sl2);   // 0 on the first tile (m = -inf)
    m0 = mn0; m1 = mn1;
    const float n0 = -mn0 * sl2, n1 = -mn1 * sl2;
    uint32_t pa[4][4];
    float r0 = 0.f, r1 = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t p01 = ptx::pack_h2(ptx::ex2(fmaf(s[j][0], sl2, n0)), ptx::ex2(fmaf(s[j][1], sl2, n0)));
      const uint32_t p23 = ptx::pack_h2(ptx::ex2(fmaf(s[j][2], sl2, n1)), ptx::ex2(fmaf(s[j][3], sl2, n1)));
      const float2 f01 = ptx::unpack_h2(p01), f23 = ptx::unpack_h2(p23);
      r0 += f01.x + f01.y;
      r1 += f23.x + f23.y;
      pa[j >> 1][(j & 1) * 2] = p01;
      pa[j >> 1][(j & 1) * 2 + 1] = p23;
    }
    l0 = l0 * a0 + r0;                             // per-thread partial row sums; reduced over the quad at the end
    l1 = l1 * a1 + r1;
#pragma unroll
    for (int j = 0; j < C::NT; ++j) {
      o[j][0] *= a0; o[j][1] *= a0; o[j][2] *= a1; o[j][3] *= a1;
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
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
    __syncthreads();                               // stage jt & 1 is refilled by the copies issued next iteration
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.f / l0, i1 = 1.f / l1;
#pragma unroll
  for (int j = 0; j < C::NT; ++j) {
    o[j][0] *= i0; o[j][1] *= i0; o[j][2] *= i1; o[j][3] *= i1;
  }
  core::warp_store<D>(o, smem + warp * 16 * C::LD * 2, lane, p.out + (int64_t)b * p.o_bs + h * D, p.o_rs,
                      row_base + warp * 16, p.N);
}

template <int D>
cudaError_t launch(const void* q, const void* k, const void* v, void* out, int B, int H, int N, int64_t bs, int64_t rs,
                   int64_t o_bs, int64_t o_rs, float scale, cudaStream_t s) {
  using CF = Cfg<D>;
  Params p;
  p.q = (const __half*)q; p.k = (const __half*)k; p.v = (const __half*)v; p.out = (__half*)out;
  p.B = B; p.H = H; p.N = N; p.bs = bs; p.rs = rs; p.o_bs = o_bs; p.o_rs = o_rs; p.scale = scale;
  static bool attr_set[tc::kMaxDevices] = {false};
  if (!attr_set[tc::cur_device()]) {
    cudaError_t e = cudaFuncSetAttribute(attn_fwd_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, CF::SMEM);
    if (e != cudaSuccess) return e;
    attr_set[tc::cur_device()] = true;
  }
  const long long grid = (long long)B * H * ((N + kBM - 1) / kBM);
  if (grid > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
  attn_fwd_kernel<D><<<(unsigned)grid, kThreads, CF::SMEM, s>>>(p);
  return cudaGetLastError();
}

}  // namespace fa
}  // namespace pww
