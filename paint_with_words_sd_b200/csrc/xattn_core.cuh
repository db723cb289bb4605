// Warp-level building blocks of the attention kernels on Hopper tensor cores.
//
// A CTA of 8 warps works on one [128-row x head] tile at a time; warp w owns query rows [16 w, 16 w + 16).  Operands are
// staged in shared memory by 16-byte cp.async copies (rows of LD = DP + 8 elements: the 16-byte pad makes every ldmatrix
// phase hit 8 distinct bank groups), read into registers with ldmatrix and multiplied with mma.m16n8k16 (E in, fp32
// accumulate).  E, the element type of q / k / v / out, is fp16 (__half) or bf16 (__nv_bfloat16); both are 2-byte types,
// so only the MMA, the packing of P and O and the rounding of the statistic depend on it.  Cross-attention, per chunk
// of at most 80 keys (the softmax streams over 1, 2 or 3 chunks, below):
//     S = Q K^T   16 x 80 per warp, DP / 16 k-steps      accumulators: 10 n-tiles x 4 fp32 per thread
//     P = 2^(log2e * scale * (S + bias - rowmax))        in registers; packed to E it is the A operand of
//     O = P V     16 x D per warp, 5 k-steps over the 80 padded keys, V fragments by ldmatrix.trans
// and O is divided by the row sum of the E-rounded P that was multiplied.  Padding (d >= D, token >= T, row >= N) is zero-filled
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
  static constexpr int LD = DP + 8;                // shared-memory row stride in (2-byte) elements
  static constexpr int KS = DP / 16;
  static constexpr int NT = D / 8;                 // n-tiles of P V
  static constexpr uint32_t QBYTES = kBM * LD * 2;
  static constexpr uint32_t KBYTES = kTP * LD * 2;
};

// Block-cooperative copy of rows [0, nrows) of a [rows x D] head slice (row stride rs elements) into shared rows of
// LD elements.  Rows >= valid and columns D .. DP-1 are zero-filled.
template <int D, typename E>
__device__ __forceinline__ void load_rows(uint32_t dst, const E* src, int64_t rs, int nrows, int valid) {
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
template <int D, typename E>
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
      ptx::mma16816<E>(s[2 * jp], a, b0, b1);
      ptx::mma16816<E>(s[2 * jp + 1], a, b2, b3);
    }
  }
}

// Token of accumulator element e of n-tile j for this lane; the row is lane / 4 (+ 8 for e >= 2).
__device__ __forceinline__ int tok(int j, int e, int lane) { return 8 * j + 2 * (lane & 3) + (e & 1); }

// Normalised O of the warp's 16 rows -> E in global memory: staged over the warp's own Q rows in shared memory (dead
// once S exists), then written as whole 16-byte pieces of each row.  Rows >= N are dropped.
template <int D, typename E>
__device__ __forceinline__ void warp_store(const float (&o)[Tile<D>::NT][4], unsigned char* stage, int lane, E* out,
                                           int64_t o_rs, int row0, int N) {
  using C = Tile<D>;
  __syncwarp();
  const int g = lane >> 2, q = lane & 3;
#pragma unroll
  for (int j = 0; j < C::NT; ++j) {
    *reinterpret_cast<uint32_t*>(stage + (g * C::LD + 8 * j + 2 * q) * 2) = ptx::pack2<E>(o[j][0], o[j][1]);
    *reinterpret_cast<uint32_t*>(stage + ((g + 8) * C::LD + 8 * j + 2 * q) * 2) = ptx::pack2<E>(o[j][2], o[j][3]);
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

// ---- key chunks: T <= 80 is one chunk of T keys; T = 154, 231 are 2 / 3 CLIP chunks of 77 ----
// Chunk c (keys 77 c .. 77 c + kv - 1) is staged as its own 80-row K / V tile, rows kv .. 79 zero-filled and masked to
// -inf, so warp_qk runs unchanged on every chunk.  The softmax streams over the chunks (running row max and sum, O
// rescaled when the max moves; attn_tc.cuh streams its 64-key tiles through the same block); P is packed to E and the row
// sum is the sum of the E-rounded P values that were multiplied, rescaled in fp32.  The first chunk's rescale factor is ex2(-inf * scale) = 0 (scale > 0), so a
// single chunk gives exactly the one-pass softmax.
constexpr int kChunk = 77;      // keys per CLIP chunk
constexpr int kMaxChunks = 3;
__host__ __device__ __forceinline__ constexpr int chunks_of(int T) { return T <= kTP ? 1 : T / kChunk; }
// T <= 80 (one tile) or a whole number of chunks, at most kMaxChunks.
__host__ __device__ __forceinline__ constexpr bool supported_keys(int T) {
  return T <= kTP || T == 2 * kChunk || T == kMaxChunks * kChunk;
}
// Real keys of every chunk of a KC-chunk instance.
template <int KC>
__host__ __device__ __forceinline__ constexpr int chunk_keys(int T) { return KC == 1 ? T : kChunk; }

// Copies of one job's operands into a stage: Q rows of the tile, then K (and V) rows of head h, one 80-row tile per
// chunk with chunk_keys<KC>(T) real rows.  The caller commits the group.
template <int D, int KC, typename E>
__device__ __forceinline__ void load_operands(uint32_t st, const XattnParams<E>& p, int b, int h, int tile, bool with_v) {
  using C = Tile<D>;
  const int rows = p.N - tile * kBM;
  load_rows<D>(st, p.q + (int64_t)b * p.q_bs + (int64_t)tile * kBM * p.q_rs + h * D, p.q_rs, kBM, rows < kBM ? rows : kBM);
  const int kv = chunk_keys<KC>(p.T);
#pragma unroll 1
  for (int c = 0; c < KC; ++c) {
    const int64_t off = (int64_t)b * p.k_bs + (int64_t)c * kChunk * p.k_rs + h * D;
    load_rows<D>(st + C::QBYTES + c * C::KBYTES, p.k + off, p.k_rs, kTP, kv);
    if (with_v) load_rows<D>(st + C::QBYTES + (KC + c) * C::KBYTES, p.v + off, p.k_rs, kTP, kv);
  }
}
// The same copies with K (and V) of the chunks in `chunks` (bit c = chunk c) only: a region-prompt softmax job skips
// the chunks no row of its tile weighs, and a statistic job the chunks outside its image's statistic.
template <int D, int KC, typename E>
__device__ __forceinline__ void load_operands_of(uint32_t st, const XattnParams<E>& p, int b, int h, int tile,
                                                 unsigned chunks, bool with_v) {
  using C = Tile<D>;
  const int rows = p.N - tile * kBM;
  load_rows<D>(st, p.q + (int64_t)b * p.q_bs + (int64_t)tile * kBM * p.q_rs + h * D, p.q_rs, kBM, rows < kBM ? rows : kBM);
#pragma unroll 1
  for (int c = 0; c < KC; ++c) {
    if (!((chunks >> c) & 1u)) continue;
    const int64_t off = (int64_t)b * p.k_bs + (int64_t)c * kChunk * p.k_rs + h * D;
    load_rows<D>(st + C::QBYTES + c * C::KBYTES, p.k + off, p.k_rs, kTP, kChunk);
    if (with_v) load_rows<D>(st + C::QBYTES + (KC + c) * C::KBYTES, p.v + off, p.k_rs, kTP, kChunk);
  }
}

template <int D>
__device__ __forceinline__ void warp_online_begin(float (&o)[Tile<D>::NT][4], float& m0, float& m1, float& l0, float& l1) {
#pragma unroll
  for (int j = 0; j < Tile<D>::NT; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
  m0 = m1 = -INFINITY;
  l0 = l1 = 0.f;
}

// What warp_online_chunk hands its hook after P V: the packed P fragments (the A operands) and the rescale factors of
// the rows' running max.  The default hook does nothing and compiles to nothing.
struct NoPHook {
  template <int NK>
  __device__ __forceinline__ void operator()(const uint32_t (&)[NK][4], float, float) const {}
};

// O += P V for the packed P of one key tile (NK k-steps of 16 keys); vs is the tile's V in shared memory.
template <int D, typename E, int NK>
__device__ __forceinline__ void warp_pv(const uint32_t (&pa)[NK][4], uint32_t vs, int lane, float (&o)[Tile<D>::NT][4]) {
  using C = Tile<D>;
#pragma unroll
  for (int kk = 0; kk < NK; ++kk) {
    const int t = 16 * kk + (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
    for (int jp = 0; jp < C::NT / 2; ++jp) {
      uint32_t b0, b1, b2, b3;
      ptx::ldsm_x4_t(vs + (uint32_t)(t * C::LD + 16 * jp + (lane >> 4) * 8) * 2u, b0, b1, b2, b3);
      ptx::mma16816<E>(o[2 * jp], pa[kk], b0, b1);
      ptx::mma16816<E>(o[2 * jp + 1], pa[kk], b2, b3);
    }
    if constexpr (C::NT & 1) {
      uint32_t b0, b1;
      ptx::ldsm_x2_t(vs + (uint32_t)(t * C::LD + 8 * (C::NT - 1)) * 2u, b0, b1);
      ptx::mma16816<E>(o[C::NT - 1], pa[kk], b0, b1);
    }
  }
}

// One key tile of NJ n-tiles (10: a cross-attention chunk of 80 padded keys; 8: a self-attention tile of 64): s holds
// S (+ bias) of the tile, of which the first kv keys are real; vs is its V tile.  l0 / l1 are per-thread partial row sums.
template <int D, typename E, int NJ, typename Hook = NoPHook>
__device__ __forceinline__ void warp_online_chunk(float (&s)[NJ][4], int kv, float sl2, uint32_t vs, int lane,
                                                  float (&o)[Tile<D>::NT][4], float& m0, float& m1, float& l0, float& l1,
                                                  const Hook& hook = Hook{}) {
  static_assert(NJ % 2 == 0, "P V takes two n-tiles of P per k-step");
  using C = Tile<D>;
  float t0 = -INFINITY, t1 = -INFINITY;
#pragma unroll
  for (int j = 0; j < NJ; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (tok(j, e, lane) >= kv) s[j][e] = -INFINITY;
      if (e < 2) t0 = fmaxf(t0, s[j][e]); else t1 = fmaxf(t1, s[j][e]);
    }
  t0 = fmaxf(t0, __shfl_xor_sync(0xffffffffu, t0, 1));
  t0 = fmaxf(t0, __shfl_xor_sync(0xffffffffu, t0, 2));
  t1 = fmaxf(t1, __shfl_xor_sync(0xffffffffu, t1, 1));
  t1 = fmaxf(t1, __shfl_xor_sync(0xffffffffu, t1, 2));
  const float mn0 = fmaxf(m0, t0), mn1 = fmaxf(m1, t1);
  const float a0 = ptx::ex2((m0 - mn0) * sl2), a1 = ptx::ex2((m1 - mn1) * sl2);   // 0 on the first chunk (m = -inf)
  m0 = mn0; m1 = mn1;
  const float n0 = -mn0 * sl2, n1 = -mn1 * sl2;
  uint32_t pa[NJ / 2][4];
  float r0 = 0.f, r1 = 0.f;
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const uint32_t p01 = ptx::pack2<E>(ptx::ex2(fmaf(s[j][0], sl2, n0)), ptx::ex2(fmaf(s[j][1], sl2, n0)));
    const uint32_t p23 = ptx::pack2<E>(ptx::ex2(fmaf(s[j][2], sl2, n1)), ptx::ex2(fmaf(s[j][3], sl2, n1)));
    const float2 f01 = ptx::unpack2<E>(p01), f23 = ptx::unpack2<E>(p23);    // sum exactly what the MMA multiplies
    r0 += f01.x + f01.y;
    r1 += f23.x + f23.y;
    pa[j >> 1][(j & 1) * 2] = p01;
    pa[j >> 1][(j & 1) * 2 + 1] = p23;
  }
  l0 = l0 * a0 + r0;
  l1 = l1 * a1 + r1;
#pragma unroll
  for (int j = 0; j < C::NT; ++j) {
    o[j][0] *= a0; o[j][1] *= a0; o[j][2] *= a1; o[j][3] *= a1;
  }
  warp_pv<D, E>(pa, vs, lane, o);
  hook(pa, a0, a1);
}

// ---- region prompts (the RGN instances of the one-launch kernel) ----
// Chunk c of a job gets a softmax of its own, mixed per query row by the row's chunk weight w_c:
//     O += E(p * (w_c / l_c)) V_c,   p = 2^(log2e * scale * (S + bias - rowmax_c)) in fp32,  l_c = fp32 sum of those p
// A chunk is one 80-key tile, so its row max and sum are complete before its P V: there is no rescale across chunks
// and no division at the end.  A row with w_c = 0 multiplies exact zeros (l_c >= 1: the row max contributes 2^0).
template <int D, typename E>
__device__ __forceinline__ void warp_weighted_chunk(float (&s)[10][4], int kv, float sl2, uint32_t vs, int lane,
                                                    float w0, float w1, float (&o)[Tile<D>::NT][4]) {
  float t0 = -INFINITY, t1 = -INFINITY;
#pragma unroll
  for (int j = 0; j < 10; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      if (tok(j, e, lane) >= kv) s[j][e] = -INFINITY;
      if (e < 2) t0 = fmaxf(t0, s[j][e]); else t1 = fmaxf(t1, s[j][e]);
    }
  t0 = fmaxf(t0, __shfl_xor_sync(0xffffffffu, t0, 1));
  t0 = fmaxf(t0, __shfl_xor_sync(0xffffffffu, t0, 2));
  t1 = fmaxf(t1, __shfl_xor_sync(0xffffffffu, t1, 1));
  t1 = fmaxf(t1, __shfl_xor_sync(0xffffffffu, t1, 2));
  const float n0 = -t0 * sl2, n1 = -t1 * sl2;
  float r0 = 0.f, r1 = 0.f;
#pragma unroll
  for (int j = 0; j < 10; ++j) {
    s[j][0] = ptx::ex2(fmaf(s[j][0], sl2, n0)); s[j][1] = ptx::ex2(fmaf(s[j][1], sl2, n0));
    s[j][2] = ptx::ex2(fmaf(s[j][2], sl2, n1)); s[j][3] = ptx::ex2(fmaf(s[j][3], sl2, n1));
    r0 += s[j][0] + s[j][1];
    r1 += s[j][2] + s[j][3];
  }
  r0 += __shfl_xor_sync(0xffffffffu, r0, 1);
  r0 += __shfl_xor_sync(0xffffffffu, r0, 2);
  r1 += __shfl_xor_sync(0xffffffffu, r1, 1);
  r1 += __shfl_xor_sync(0xffffffffu, r1, 2);
  const float f0 = w0 / r0, f1 = w1 / r1;
  uint32_t pa[5][4];
#pragma unroll
  for (int j = 0; j < 10; ++j) {
    pa[j >> 1][(j & 1) * 2] = ptx::pack2<E>(s[j][0] * f0, s[j][1] * f0);
    pa[j >> 1][(j & 1) * 2 + 1] = ptx::pack2<E>(s[j][2] * f1, s[j][3] * f1);
  }
  warp_pv<D, E>(pa, vs, lane, o);
}

// Divides O by the row sums (reduced over the quad) once every chunk has been accumulated.
template <int D>
__device__ __forceinline__ void warp_online_end(float (&o)[Tile<D>::NT][4], float l0, float l1) {
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.f / l0, i1 = 1.f / l1;
#pragma unroll
  for (int j = 0; j < Tile<D>::NT; ++j) {
    o[j][0] *= i0; o[j][1] *= i0; o[j][2] *= i1; o[j][3] *= i1;
  }
}

// ---- per-region softmax mass (the recording instance of the cross-attention kernel) ----
// The 16 region slots are two more 8-column "V" tiles: R[t, r] = (ridx[t] == r), a 0/1 matrix built in registers, so
// mass[n, r] = sum_t P[n, t] R[t, r] is two MMAs per k-step of P V with the same packed P, rescaled like O when the row
// max moves and divided by the same row sum at the end.  rm[2][4] holds the [16 rows x 16 slots] C fragments.
constexpr int kRegions = 16;

// After chunk c's P V: rescale rm by the chunk's factors a0 / a1 and add P R; rt = the chunk's 80 ridx entries.
template <typename E, int NK>
__device__ __forceinline__ void warp_region_chunk(const uint32_t (&pa)[NK][4], float a0, float a1, const int8_t* rt,
                                                  int lane, float (&rm)[2][4]) {
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    rm[j][0] *= a0; rm[j][1] *= a0; rm[j][2] *= a1; rm[j][3] *= a1;
  }
  const int r = lane >> 2;
#pragma unroll
  for (int kk = 0; kk < NK; ++kk) {
    // B fragment of m16n8k16: tokens 16 kk + 2 (lane & 3) + {0, 1} (b0) and + 8 (b1), column lane / 4 of the tile
    const int t = 16 * kk + 2 * (lane & 3);
    const int i0 = __ldg(rt + t), i1 = __ldg(rt + t + 1), i2 = __ldg(rt + t + 8), i3 = __ldg(rt + t + 9);
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int slot = r + 8 * j;
      const uint32_t b0 = ptx::pack2<E>(i0 == slot ? 1.f : 0.f, i1 == slot ? 1.f : 0.f);
      const uint32_t b1 = ptx::pack2<E>(i2 == slot ? 1.f : 0.f, i3 == slot ? 1.f : 0.f);
      ptx::mma16816<E>(rm[j], pa[kk], b0, b1);
    }
  }
}

// Normalises rm by the row sums (the quad reduction of warp_online_end) and adds it to acc, the fp32 [N, 16] mass of
// this (record, head): plain read-add-write, rows >= N dropped.  One job owns each (image, head, row) of a launch.
__device__ __forceinline__ void warp_region_add(const float (&rm)[2][4], float l0, float l1, float* acc, int row0, int N,
                                                int lane) {
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float inv[2] = {1.f / l0, 1.f / l1};
  const int g = lane >> 2, q = lane & 3;
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    const int row = row0 + g + 8 * hf;
    if (row >= N) continue;
    float* a = acc + (int64_t)row * kRegions + 2 * q;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      a[8 * j] += rm[j][2 * hf] * inv[hf];
      a[8 * j + 1] += rm[j][2 * hf + 1] * inv[hf];
    }
  }
}

// Statistic partials of S over the warp's valid elements (row < N, token < T): running max of S (rounding to E is
// monotonic, so the maximum is rounded once at the end) or sum / sum of squares of E(S).
template <typename E>
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
        const float h = round_to<E>(s[j][e]);
        sum += h;
        sumsq = fmaf(h, h, sumsq);
      }
    }
}

// Warp reduction of a (max, sum, sumsq) partial: every lane ends with the warp's total.
__device__ __forceinline__ void warp_reduce_stat(double& m, double& a, double& q) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    a += __shfl_xor_sync(0xffffffffu, a, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
}

// The statistic of an image from its totals over its H * N * keys scores (keys = T, or 77 per chunk of a region-prompt
// image's statistic): the maximum, or the unbiased standard deviation (variance clamped at 0), rounded to E as
// qk.max() / qk.std() return it in the reference's op sequence under an E autocast.
template <typename E>
__device__ __forceinline__ float stat_value(const XattnParams<E>& p, bool is_max, double m, double a, double q, int keys) {
  const double cnt = (double)p.H * (double)p.N * (double)keys;
  double r;
  if (is_max) {
    r = m;
  } else {
    const double var = (q - a * a / cnt) / (cnt - 1.0);
    r = sqrt(var > 0.0 ? var : 0.0);
  }
  return round_to<E>((float)r);
}

}  // namespace core
}  // namespace pww
