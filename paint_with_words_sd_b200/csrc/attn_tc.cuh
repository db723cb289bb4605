// Self-attention (context=None in the reference's inj_forward, paint_with_words.py:71-72, 87-118) as a flash attention
// forward on Hopper tensor cores: softmax(scale * Q_h K_h^T) V_h with keys = the image's own N pixels.
//
// One CTA = (image, head, 128 query rows); warp w owns rows [16 w, 16 w + 16) and keeps its Q fragments in registers.
// Key tiles of BN = 64 rows of K and V stream through a two-stage cp.async ring in shared memory (the copies of tile j + 1
// are in flight while tile j is computed):
//     S = Q K_j^T     mma.m16n8k16, 8 n-tiles per warp, fp32 accumulators in registers
//     online softmax: running row max m and row sum l; O and l are rescaled by 2^(m_old - m_new) when the max moves
//     O += P V_j      P packed to E (fp16 or bf16, the element type of q / k / v / out) straight from the S accumulators (the C layout of two n-tiles is the A layout of one
//                     k-step), V fragments by ldmatrix.trans
// The softmax and P V are the cross-attention kernels' block (core::warp_online_*, xattn_core.cuh) at 8 n-tiles per tile.
// Padding (d >= D, key >= N, row >= N) is zero-filled by the copies; padded keys of the last tile are masked to -inf.
#pragma once
#include "mma_sm90.cuh"
#include "pww_common.cuh"
#include "xattn_core.cuh"

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

template <typename E>
struct Params {
  const E* q;
  const E* k;
  const E* v;
  E* out;
  int B, H, N;
  int64_t bs, rs;          // q/k/v element strides (batch, row)
  int64_t o_bs, o_rs;
  float scale;
};

// Minimum CTAs per SM of the launch bound (0 = none).  Unbounded, ptxas fits the bf16 head-dim-80 instance into 128
// registers (two CTAs per SM) and spills 24 bytes; its fp16 twin takes 137 registers, one CTA per SM.  A bound of one
// CTA gives the bf16 instance that same occupancy without spills.  Every other instance keeps the unbounded choice.
template <int D, typename E>
constexpr int kMinBlocks = (D == 80 && std::is_same_v<E, __nv_bfloat16>) ? 1 : 0;

template <int D, typename E>
__global__ void __launch_bounds__(kThreads, kMinBlocks<D, E>) attn_fwd_kernel(const Params<E> p) {
  using C = core::Tile<D>;
  using CF = Cfg<D>;
  extern __shared__ __align__(128) unsigned char smem[];
  const uint32_t smem0 = ptx::smem_u32(smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qtiles = (p.N + kBM - 1) / kBM;
  const int bh = blockIdx.x / qtiles, qt = blockIdx.x - bh * qtiles;
  const int b = bh / p.H, h = bh - b * p.H;
  const int row_base = qt * kBM;
  const E* qb = p.q + (int64_t)b * p.bs + h * D;
  const E* kb = p.k + (int64_t)b * p.bs + h * D;
  const E* vb = p.v + (int64_t)b * p.bs + h * D;
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
  float o[C::NT][4], m0, m1, l0, l1;
  core::warp_online_begin<D>(o, m0, m1, l0, l1);
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
    float s[kBN / 8][4];
#pragma unroll
    for (int j = 0; j < kBN / 8; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < C::KS; ++kk) {
#pragma unroll
      for (int jp = 0; jp < kBN / 16; ++jp) {
        const int t = 16 * jp + (lane & 7) + ((lane >> 4) << 3), d = kk * 16 + ((lane >> 3) & 1) * 8;
        uint32_t b0, b1, b2, b3;
        ptx::ldsm_x4(ks + (uint32_t)(t * C::LD + d) * 2u, b0, b1, b2, b3);
        ptx::mma16816<E>(s[2 * jp], qa[kk], b0, b1);
        ptx::mma16816<E>(s[2 * jp + 1], qa[kk], b2, b3);
      }
    }
    core::warp_online_chunk<D, E>(s, p.N - jt * kBN, sl2, vs, lane, o, m0, m1, l0, l1);
    __syncthreads();                               // stage jt & 1 is refilled by the copies issued next iteration
  }
  core::warp_online_end<D>(o, l0, l1);
  core::warp_store<D>(o, smem + warp * 16 * C::LD * 2, lane, p.out + (int64_t)b * p.o_bs + h * D, p.o_rs,
                      row_base + warp * 16, p.N);
}

template <int D, typename E>
cudaError_t launch(const void* q, const void* k, const void* v, void* out, int B, int H, int N, int64_t bs, int64_t rs,
                   int64_t o_bs, int64_t o_rs, float scale, cudaStream_t s) {
  using CF = Cfg<D>;
  Params<E> p;
  p.q = (const E*)q; p.k = (const E*)k; p.v = (const E*)v; p.out = (E*)out;
  p.B = B; p.H = H; p.N = N; p.bs = bs; p.rs = rs; p.o_bs = o_bs; p.o_rs = o_rs; p.scale = scale;
  const cudaError_t e = allow_dynamic_smem<attn_fwd_kernel<D, E>>(CF::SMEM);
  if (e != cudaSuccess) return e;
  const long long grid = (long long)B * H * ((N + kBM - 1) / kBM);
  if (grid > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
  attn_fwd_kernel<D, E><<<(unsigned)grid, kThreads, CF::SMEM, s>>>(p);
  return cudaGetLastError();
}

}  // namespace fa
}  // namespace pww
