// extern "C" entry points of libpww_b200.so (declared in include/pww_b200.h).
#include <stdio.h>
#include <string.h>

#include "pww_common.cuh"
#include "xattn_tc.cuh"
#include "xattn_fused2.cuh"
#include "attn_tc.cuh"
#include "unet_ops.cuh"
#include "sampler_step.cuh"
#include "sampler_rescale.cuh"
#include "sampler_window.cuh"
#include "control_inject.cuh"
#include "control_combine.cuh"
#include "adapter_residual.cuh"
#include <stdlib.h>
#include <algorithm>
#include <type_traits>

namespace {

thread_local char g_last_cuda_error[640] = "";

int cuda_fail(cudaError_t e);

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

bool supported_head_dim(int D) { return D == 40 || D == 64 || D == 80 || D == 160; }

int check_common(const void* q, const void* k, int B, int H, int N, int T, int D, int64_t q_bs, int64_t q_rs,
                 int64_t k_bs, int64_t k_rs) {
  if (!q || !k || B <= 0 || H <= 0 || N <= 0 || T <= 0 || D <= 0) return PWW_ERR_BAD_ARG;
  if (!aligned16(q) || !aligned16(k)) return PWW_ERR_BAD_ARG;
  if ((q_bs | q_rs | k_bs | k_rs) & 7) return PWW_ERR_BAD_ARG;  // 16-byte vector access on rows
  if (q_rs < (int64_t)H * D || k_rs < (int64_t)H * D) return PWW_ERR_BAD_ARG;
  if (!supported_head_dim(D) || !pww::core::supported_keys(T)) return PWW_ERR_UNSUPPORTED;
  return PWW_OK;
}

// Kernel instance for a (head dim, key chunk count) pair: f(Shape<D, KC>{}) with KC = 1 for T <= 80, else T / 77.
template <int D_, int KC_>
struct Shape {
  static constexpr int D = D_, KC = KC_;
};
template <int D, typename F>
cudaError_t with_chunks(int T, F&& f) {
  switch (pww::core::chunks_of(T)) {
    case 1: return f(Shape<D, 1>{});
    case 2: return f(Shape<D, 2>{});
    case 3: return f(Shape<D, 3>{});
  }
  return cudaErrorInvalidValue;
}
template <typename F>
cudaError_t with_shape(int D, int T, F&& f) {
  switch (D) {
    case 40: return with_chunks<40>(T, f);
    case 64: return with_chunks<64>(T, f);
    case 80: return with_chunks<80>(T, f);
    case 160: return with_chunks<160>(T, f);
  }
  return cudaErrorInvalidValue;
}

// f(std::integral_constant<int, v>{}) for lo <= v <= hi.
template <int lo, int hi, typename F>
void with_int(int v, F&& f) {
  if constexpr (lo < hi)
    if (v != lo) return with_int<lo + 1, hi>(v, f);
  f(std::integral_constant<int, lo>{});
}

size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// f(T{}) for the element type T of a PWW_DTYPE_* code the caller has checked: fp16, bf16, else fp32.
template <typename F>
cudaError_t with_dtype(int dtype, F&& f) {
  if (dtype == PWW_DTYPE_F16) return f(__half{});
  if (dtype == PWW_DTYPE_BF16) return f(__nv_bfloat16{});
  return f(float{});
}

// The pww_sampler_update* entry points' shared part: the argument checks (every PWW_ERR_BAD_ARG before the dtype's
// PWW_ERR_UNSUPPORTED, and none of them a CUDA call), the UpdateArgs and the layout.  PX = 4 needs h w % 4 == 0 and
// 16-byte aligned latents, history and noise, and `px4_extra` (the caller's own inputs read 4 pixels at a time).
int update_setup(const void* eps, int eps_dtype, int64_t e_sn, int64_t e_sc, int64_t e_sh, int64_t e_sw,
                 float* latents, float* history, int history_len, const float* noise, const float* guidance,
                 const float* beta, const float* form, int m, int height, int width, bool px4_extra,
                 pww::smp::UpdateArgs& a, bool& px4, bool& cl) {
  if (!eps || !latents || !history || !guidance || !beta || !form) return PWW_ERR_BAD_ARG;
  if (m <= 0 || height <= 0 || width <= 0 || history_len < 1 || history_len > 4) return PWW_ERR_BAD_ARG;
  if (eps_dtype != PWW_DTYPE_F32 && eps_dtype != PWW_DTYPE_F16 && eps_dtype != PWW_DTYPE_BF16) return PWW_ERR_UNSUPPORTED;
  a.eps = eps; a.e_sn = e_sn; a.e_sc = e_sc; a.e_sh = e_sh; a.e_sw = e_sw;
  a.lat = latents; a.hist = history; a.noise = noise; a.gscale = guidance; a.beta = beta; a.form = form;
  a.m = m; a.h = height; a.w = width; a.nh = history_len;
  const int64_t hw = (int64_t)height * width;
  const size_t es = eps_dtype == PWW_DTYPE_F32 ? 4 : 2;
  px4 = (hw % 4) == 0 && aligned16(latents) && aligned16(history) && (!noise || aligned16(noise)) && px4_extra;
  // channels-last packed rows: pixel p's 4 channels at 4p (8 bytes per pixel in fp16 / bf16, 16 in fp32)
  const size_t need = px4 ? 16 : 4 * es;
  cl = e_sc == 1 && e_sw == 4 && e_sh == 4 * (int64_t)width && (reinterpret_cast<uintptr_t>(eps) % need) == 0 &&
       ((size_t)e_sn * es) % need == 0;
  return PWW_OK;
}

// Partial slots the statistics workspace reserves per image: one per CTA of the persistent grid, a device-independent
// upper bound so that the size can be computed without a GPU.
constexpr int kStatSlotsPerImage = 2048;

int cuda_fail(cudaError_t e) {
  snprintf(g_last_cuda_error, sizeof(g_last_cuda_error), "%s: %s ", cudaGetErrorName(e), cudaGetErrorString(e));
  return PWW_ERR_CUDA;
}

// The XattnParams fields every cross-attention launch takes from its arguments; the others start at zero.
template <typename E>
pww::XattnParams<E> xattn_params(const void* q, const void* k, const void* v, void* out, int B, int H, int N, int T, int D,
                                 int64_t q_bs, int64_t q_rs, int64_t k_bs, int64_t k_rs, int64_t o_bs, int64_t o_rs) {
  pww::XattnParams<E> p;
  memset(&p, 0, sizeof(p));
  p.q = (const E*)q; p.k = (const E*)k; p.v = (const E*)v; p.out = (E*)out;
  p.B = B; p.H = H; p.N = N; p.T = T; p.D = D;
  p.q_bs = q_bs; p.q_rs = q_rs; p.k_bs = k_bs; p.k_rs = k_rs; p.o_bs = o_bs; p.o_rs = o_rs;
  return p;
}

// p restricted to images [b0, b0 + n): every per-image pointer that is set starts at image b0.  The workspace
// (counters, partials) is shared by the launches, and the weight maps are reached through wmap_index; a caller that maps
// image b to map b without an index offsets its maps itself.
template <typename E>
pww::XattnParams<E> images(const pww::XattnParams<E>& p, int b0, int n) {
  pww::XattnParams<E> c = p;
  c.B = n;
  c.q += (int64_t)b0 * p.q_bs;
  c.k += (int64_t)b0 * p.k_bs;
  if (c.v) c.v += (int64_t)b0 * p.k_bs;
  if (c.out) c.out += (int64_t)b0 * p.o_bs;
  if (c.wmap_index) c.wmap_index += b0;
  if (c.stat_kind) c.stat_kind += b0;
  if (c.stats) c.stats += b0;
  if (c.stats_out) c.stats_out += b0;
  if (c.g_sigma) c.g_sigma += (int64_t)b0 * p.g_stride;
  return c;
}

}  // namespace

extern "C" {

int pww_version(void) { return 300; }  // 0.3.0: per-image statistic kind and G(sigma) (the _multi entry points)

const char* pww_status_str(int status) {
  switch (status) {
    case PWW_OK: return "ok";
    case PWW_ERR_BAD_ARG: return "bad argument (null/misaligned pointer, non-positive size or stride not a multiple of 8)";
    case PWW_ERR_UNSUPPORTED: return "unsupported shape or dtype (head dim must be 40/64/80/160, T <= 80, 154 or 231)";
    case PWW_ERR_CUDA: return "CUDA error (see pww_last_cuda_error)";
    case PWW_ERR_WORKSPACE: return "workspace too small (see pww_xattn_workspace_bytes)";
    default: return "unknown status";
  }
}

const char* pww_last_cuda_error(void) { return g_last_cuda_error; }

int pww_device_supported(void) {
  int dev = 0, major = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return cuda_fail(e);
  e = cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  if (e != cudaSuccess) return cuda_fail(e);
  return major == 9 ? 1 : 0;
}

size_t pww_xattn_workspace_bytes(int B, int H, int N, int T, int D) {
  (void)T; (void)D;
  if (B <= 0 || H <= 0 || N <= 0) return 0;
  return align_up((size_t)B * sizeof(unsigned int), 256) +
         (size_t)B * kStatSlotsPerImage * sizeof(pww::StatPartial);
}

}  // extern "C"

namespace {

// The statistics launches of pww_xattn_stats_{f16,bf16} (kinds == NULL: `stat` for every image) and of
// pww_xattn_stats_multi_{f16,bf16} (per_image: kinds[b] for image b); E = __half or __nv_bfloat16.
template <typename E>
int xattn_stats(const void* q, const void* k, int B, int H, int N, int T, int D, int64_t q_batch_stride,
                int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride, int stat, const int32_t* kinds,
                bool per_image, const int32_t* wmap_index, float* stats, void* workspace, size_t workspace_bytes,
                void* stream) {
  int rc = check_common(q, k, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride, k_row_stride);
  if (rc) return rc;
  if (!stats || !workspace) return PWW_ERR_BAD_ARG;
  if (per_image ? !kinds : (stat != PWW_STAT_MAX && stat != PWW_STAT_STD)) return PWW_ERR_BAD_ARG;
  if (workspace_bytes < pww_xattn_workspace_bytes(B, H, N, T, D)) return PWW_ERR_WORKSPACE;
  if (pww::num_sms() > kStatSlotsPerImage) return PWW_ERR_WORKSPACE;
  pww::XattnParams<E> p = xattn_params<E>(q, k, nullptr, nullptr, B, H, N, T, D, q_batch_stride, q_row_stride,
                                          k_batch_stride, k_row_stride, 0, 0);
  p.wmap_index = wmap_index; p.stat = stat; p.stat_kind = per_image ? kinds : nullptr; p.stats_out = stats;
  p.counters = (unsigned int*)workspace;
  p.partials = (pww::StatPartial*)((char*)workspace + align_up((size_t)B * sizeof(unsigned int), 256));
  for (int b0 = 0; b0 < B; b0 += pww::tc::kMaxBatch) {
    const pww::XattnParams<E> c = images(p, b0, std::min(B - b0, pww::tc::kMaxBatch));
    const cudaError_t e =
        with_shape(D, T, [&](auto k) { return pww::tc::launch_stats<k.D, k.KC>(c, (cudaStream_t)stream); });
    if (e != cudaSuccess) return cuda_fail(e);
  }
  return PWW_OK;
}

// The forward launches of pww_xattn_fwd_{f16,bf16} (g_stride 0: g_sigma[0] for every image) and of
// pww_xattn_fwd_multi_{f16,bf16} (g_stride 1: g_sigma[b] for image b).
template <typename E>
int xattn_fwd(const void* q, const void* k, const void* v, void* out, int B, int H, int N, int T, int D,
              int64_t q_batch_stride, int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride,
              int64_t o_batch_stride, int64_t o_row_stride, const float* wmap, int64_t wmap_batch_stride,
              const int32_t* wmap_index, const float* stats, const float* g_sigma, int64_t g_stride, float scale,
              void* stream) {
  int rc = check_common(q, k, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride, k_row_stride);
  if (rc) return rc;
  if (!v || !out || !aligned16(v) || !aligned16(out)) return PWW_ERR_BAD_ARG;
  if ((o_batch_stride | o_row_stride) & 7 || o_row_stride < (int64_t)H * D) return PWW_ERR_BAD_ARG;
  if (wmap && (!stats || !g_sigma)) return PWW_ERR_BAD_ARG;
  pww::XattnParams<E> p = xattn_params<E>(q, k, v, out, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride,
                                          k_row_stride, o_batch_stride, o_row_stride);
  p.wmap = wmap; p.wmap_bs = wmap_batch_stride; p.wmap_index = wmap ? wmap_index : nullptr;
  p.stats = stats; p.g_sigma = g_sigma; p.g_stride = g_stride; p.scale = scale;
  for (int b0 = 0; b0 < B; b0 += pww::tc::kMaxBatch) {
    pww::XattnParams<E> c = images(p, b0, std::min(B - b0, pww::tc::kMaxBatch));
    if (wmap && !wmap_index) c.wmap += (int64_t)b0 * wmap_batch_stride;   // identity mapping: image b uses map b
    const cudaError_t e =
        with_shape(D, T, [&](auto k) { return pww::tc::launch_fwd<k.D, k.KC>(c, (cudaStream_t)stream); });
    if (e != cudaSuccess) return cuda_fail(e);
  }
  return PWW_OK;
}

// The one launch of pww_xattn_fused_{f16,bf16} (one `stat` and g_sigma[0] for every image) and of
// pww_xattn_fused_multi_{f16,bf16} (per_image: kinds[b] and g_sigma[b] for image b).  mpack is fp16 for both E.
template <typename E>
int xattn_fused(const void* q, const void* k, const void* v, void* out, int B, int H, int N, int T, int D,
                int64_t q_batch_stride, int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride,
                int64_t o_batch_stride, int64_t o_row_stride, const void* mpack, int64_t mpack_batch_stride, int Bw,
                const int8_t* cidx, const int32_t* wmap_index, int stat, const int32_t* kinds, bool per_image,
                const float* g_sigma, float scale, float* stats, void* workspace, size_t workspace_bytes,
                void* stream, const pww::fx::FxRecord* rec = nullptr, const pww::fx::FxRegion* rg = nullptr) {
  int rc = check_common(q, k, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride, k_row_stride);
  if (rc) return rc;
  if (rg) {
    if (pww::core::chunks_of(T) < 2) return PWW_ERR_UNSUPPORTED;       // region prompts: T = 154, 231
    if (!rg->rw || (reinterpret_cast<uintptr_t>(rg->rw) & 3u) ||
        rg->rw_bs < (int64_t)N * pww::core::chunks_of(T))
      return PWW_ERR_BAD_ARG;
  }
  if (!v || !out || !aligned16(v) || !aligned16(out)) return PWW_ERR_BAD_ARG;
  if ((o_batch_stride | o_row_stride) & 7 || o_row_stride < (int64_t)H * D || o_batch_stride <= 0) return PWW_ERR_BAD_ARG;
  if (rec && (!rec->ridx || !rec->rec_index || !rec->rec_acc || !aligned16(rec->rec_acc) ||
              rec->rec_bs < (int64_t)H * N * pww::core::kRegions))
    return PWW_ERR_BAD_ARG;
  if (mpack) {
    if (!cidx || !g_sigma || !workspace || Bw <= 0 || !aligned16(mpack)) return PWW_ERR_BAD_ARG;
    if ((mpack_batch_stride & 7) || mpack_batch_stride < (int64_t)N * pww::fx::kMW) return PWW_ERR_BAD_ARG;
    if (per_image ? !kinds : (stat != PWW_STAT_MAX && stat != PWW_STAT_STD)) return PWW_ERR_BAD_ARG;
    if (workspace_bytes < pww_xattn_fused_workspace_bytes()) return PWW_ERR_WORKSPACE;
  }
  pww::XattnParams<E> p = xattn_params<E>(q, k, v, out, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride,
                                          k_row_stride, o_batch_stride, o_row_stride);
  p.g_sigma = g_sigma; p.g_stride = per_image ? 1 : 0; p.scale = scale; p.stat = stat;
  p.stat_kind = per_image ? kinds : nullptr; p.stats_out = stats;
  // image b is biased iff it has a packed map: with mpack == NULL the kernel takes every index as -1
  p.wmap_index = mpack ? wmap_index : nullptr;
  p.counters = (unsigned int*)workspace;
  p.partials = workspace ? (pww::StatPartial*)((char*)workspace + 512) : nullptr;   // header: counters @0, per-image maxima @256
  // images per launch: halved until every CTA's job table holds at most 64 units
  int chunk = pww::fx::kMaxBatch;
  const int tiles = pww::ceil_div(N, pww::core::kBM);
  const int hg = pww::ceil_div(H, D == 40 ? pww::fx::Cfg2<40>::G : (D == 64 ? pww::fx::Cfg2<64>::G : 1));
  while (chunk > 1) {
    const int cb = B < chunk ? B : chunk;
    if (pww::fx::fused2_fits(cb, hg, tiles, pww::fx::fused_grid(cb * hg * tiles))) break;
    chunk >>= 1;
  }
  for (int b0 = 0; b0 < B; b0 += chunk) {
    pww::XattnParams<E> c = images(p, b0, std::min(B - b0, chunk));
    const void* mp = mpack;
    const int8_t* ci = cidx;
    if (mpack && !wmap_index) {                                    // identity mapping: image b uses map b
      mp = (const __half*)mpack + (int64_t)b0 * mpack_batch_stride;
      ci = cidx + (int64_t)b0 * pww::core::kTP * pww::core::chunks_of(T);   // [Bw, 80 k]
    }
    c.wmap = (const float*)mp;                                     // non-null marks "maps present" for the kernel
    pww::fx::FxRecord r;
    if (rec) {                                                     // records are reached through rec_index
      r = *rec;
      r.rec_index += b0;
    }
    pww::fx::FxRegion g;
    if (rg) {                                                      // weights through rw_index, else row b
      g = *rg;
      if (g.rw_index) g.rw_index += b0;
      else g.rw += (int64_t)b0 * g.rw_bs;
      if (g.stat_chunks) g.stat_chunks += b0;
    }
    const cudaError_t e = with_shape(D, T, [&](auto k) {
      return pww::fx::launch_fused2<k.D, k.KC>(c, mp, mpack_batch_stride, ci, (cudaStream_t)stream, rec ? &r : nullptr,
                                               rg ? &g : nullptr);
    });
    if (e == cudaErrorInvalidConfiguration) return PWW_ERR_UNSUPPORTED;
    if (e != cudaSuccess) return cuda_fail(e);
  }
  return PWW_OK;
}

template <typename E>
int groupnorm_nhwc(const void* x, const void* add, int64_t add_batch_stride, const void* gamma, const void* beta, void* y,
                   int B, int HW, int C, int G, float eps, int silu, void* workspace, size_t workspace_bytes,
                   void* stream) {
  if (!x || !gamma || !beta || !y || !workspace || B <= 0 || HW <= 0 || C <= 0 || G <= 0) return PWW_ERR_BAD_ARG;
  if (!aligned16(x) || !aligned16(y) || !aligned16(gamma) || !aligned16(beta) || (add && !aligned16(add)))
    return PWW_ERR_BAD_ARG;
  if ((C & 7) || (C % G) || G > 64 || (C >> 3) > 1024) return PWW_ERR_UNSUPPORTED;
  if (add && ((add_batch_stride & 7) || add_batch_stride < C)) return PWW_ERR_BAD_ARG;
  if (workspace_bytes < pww_groupnorm_workspace_bytes(B, HW, G)) return PWW_ERR_WORKSPACE;
  const pww::uops::GnSplit sp = pww::uops::gn_split(HW, C, G);
  pww::uops::GnParams<E> p;
  p.x = (const E*)x; p.add = (const E*)add; p.add_bs = add_batch_stride; p.gamma = (const E*)gamma; p.beta = (const E*)beta;
  p.y = (E*)y;
  p.partial = (float2*)workspace;
  p.HW = HW; p.C = C; p.G = G; p.eps = eps; p.silu = silu;
  p.sv = sp.sv; p.chunks = sp.chunks; p.rows_per_chunk = sp.rows_per_chunk;
  cudaStream_t s = (cudaStream_t)stream;
  // 64 group shifts + per-thread channel sums: 16 KB up to 256-vector slices, 64 KB at most (C = 8192, one group)
  const size_t smem1 = (64 + (size_t)2 * sp.rpp * sp.sv * 8) * sizeof(float);
  if (smem1 > 48 * 1024) {
    const cudaError_t e = pww::allow_dynamic_smem<pww::uops::gn_stats_kernel<E>>(64 * 1024 + 256);
    if (e != cudaSuccess) return cuda_fail(e);
  }
  pww::uops::gn_stats_kernel<E><<<dim3(sp.chunks, sp.slices, B), sp.threads, smem1, s>>>(p);
  // rows per thread: 4, or fewer until the apply grid has two blocks per SM (the split of the apply pass does not
  // change any result, so it may depend on B)
  int rows = 4;
  while (rows > 1 && (long long)B * sp.slices * pww::ceil_div(HW, sp.rpp * rows) < 2 * pww::num_sms()) rows >>= 1;
  // Programmatic dependent launch: the apply grid starts while the stats grid runs and waits (griddepcontrol.wait)
  // only before it reads the partials
  cudaLaunchAttribute pdl;
  pdl.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  pdl.val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(pww::ceil_div(HW, sp.rpp * rows), sp.slices, B);
  cfg.blockDim = dim3(sp.threads);
  cfg.stream = s;
  cfg.attrs = &pdl;
  cfg.numAttrs = 1;
  cudaError_t e = cudaLaunchKernelEx(&cfg, pww::uops::gn_apply_kernel<E>, p, sp.rpp * rows);
  if (e == cudaSuccess) e = cudaGetLastError();
  return e == cudaSuccess ? PWW_OK : cuda_fail(e);
}

template <typename E>
int geglu(const void* in, void* out, int64_t M, int I, void* stream) {
  if (!in || !out || M <= 0 || I <= 0 || !aligned16(in) || !aligned16(out)) return PWW_ERR_BAD_ARG;
  if (I & 7) return PWW_ERR_UNSUPPORTED;
  const long long total = (long long)M * (I >> 3);
  long long blocks = (total + 255) / 256;
  const long long cap = (long long)pww::num_sms() * 16;
  if (blocks > cap) blocks = cap;
  pww::uops::geglu_kernel<E><<<(int)blocks, 256, 0, (cudaStream_t)stream>>>((const E*)in, (E*)out, M, I);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? PWW_OK : cuda_fail(e);
}

template <typename E>
int add_layernorm(const void* x, const void* res, const void* gamma, const void* beta, void* sum_out, void* y, int64_t M,
                  int C, float eps, void* stream) {
  if (!x || !gamma || !beta || !y || M <= 0 || C <= 0) return PWW_ERR_BAD_ARG;
  if (!aligned16(x) || !aligned16(y) || !aligned16(gamma) || !aligned16(beta) || (res && !aligned16(res)) ||
      (sum_out && !aligned16(sum_out)))
    return PWW_ERR_BAD_ARG;
  if ((C & 7) || C > 2048) return PWW_ERR_UNSUPPORTED;
  const int warps = 8;
  const unsigned grid = (unsigned)((M + warps - 1) / warps);
  // 16-byte vectors per lane: 1 .. 8 for C <= 2048
  with_int<1, 8>(((C >> 3) + 31) / 32, [&](auto vpl) {
    pww::uops::add_layernorm_kernel<E, vpl><<<grid, warps * 32, 0, (cudaStream_t)stream>>>(
        (const E*)x, (const E*)res, (const E*)gamma, (const E*)beta, (E*)sum_out, (E*)y, M, C, eps);
  });
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? PWW_OK : cuda_fail(e);
}

template <typename E>
int resnet_residual(const void* a, const void* h, const float* bias, void* out, int64_t rows, int C, void* stream) {
  if (!a || !h || !bias || !out || rows <= 0 || C <= 0 || (C & 7)) return PWW_ERR_BAD_ARG;
  if (!aligned16(a) || !aligned16(h) || !aligned16(bias) || !aligned16(out)) return PWW_ERR_BAD_ARG;
  const long long total = (long long)rows * (C >> 3);
  long long blocks = (total + 255) / 256;
  const long long cap = (long long)pww::num_sms() * 16;
  if (blocks > cap) blocks = cap;
  pww::uops::resnet_residual_kernel<E><<<(int)blocks, 256, 0, (cudaStream_t)stream>>>(
      (const E*)a, (const E*)h, bias, (E*)out, total, C >> 3);
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? PWW_OK : cuda_fail(e);
}

template <typename E>
int adapter_residual(const void* a, const void* b, const float* bias, const void* feat, void* out, int rows,
                     int64_t pixels, int C, int feat_rows, void* stream) {
  if (!a || !b || !out || rows <= 0 || pixels <= 0 || C <= 0 || (C & 7)) return PWW_ERR_BAD_ARG;
  if (feat_rows < 0 || feat_rows > rows || (feat_rows > 0 && !feat)) return PWW_ERR_BAD_ARG;
  if (!aligned16(a) || !aligned16(b) || !aligned16(out) || (bias && !aligned16(bias)) || (feat && !aligned16(feat)))
    return PWW_ERR_BAD_ARG;
  const long long per_row = (long long)pixels * (C >> 3);
  const cudaError_t e = pww::adp::launch<E>(a, b, bias, feat, out, (long long)rows * per_row,
                                            (long long)feat_rows * per_row, C >> 3, (long long)pww::num_sms() * 16,
                                            (cudaStream_t)stream);
  return e == cudaSuccess ? PWW_OK : cuda_fail(e);
}

template <typename E>
int attn_fwd(const void* q,const void* k, const void* v, void* out, int B, int H, int N, int D, int64_t qkv_batch_stride,
             int64_t qkv_row_stride, int64_t o_batch_stride, int64_t o_row_stride, float scale, void* stream) {
  if (!q || !k || !v || !out || B <= 0 || H <= 0 || N <= 0 || D <= 0) return PWW_ERR_BAD_ARG;
  if (!aligned16(q) || !aligned16(k) || !aligned16(v) || !aligned16(out)) return PWW_ERR_BAD_ARG;
  if ((qkv_batch_stride | qkv_row_stride | o_batch_stride | o_row_stride) & 7) return PWW_ERR_BAD_ARG;
  if (qkv_row_stride < (int64_t)H * D || o_row_stride < (int64_t)H * D) return PWW_ERR_BAD_ARG;
  if (!supported_head_dim(D)) return PWW_ERR_UNSUPPORTED;
  // self-attention has no key chunks: T = 1 picks the one-chunk shape of the head dim
  const cudaError_t e = with_shape(D, 1, [&](auto sh) {
    return pww::fa::launch<sh.D, E>(q, k, v, out, B, H, N, qkv_batch_stride, qkv_row_stride, o_batch_stride,
                                    o_row_stride, scale, (cudaStream_t)stream);
  });
  return e == cudaSuccess ? PWW_OK : cuda_fail(e);
}

template <typename E>
int control_inject(int n, void* const* dst, const void* const* res, const int64_t* elems_per_image, int rows,
                   const float* scales, void* stream) {
  if (n < 1 || n > pww::ctl::kMaxLevels || rows < 1 || !dst || !res || !elems_per_image) return PWW_ERR_BAD_ARG;
  pww::ctl::InjectArgs a;
  a.off[0] = 0;
  for (int k = 0; k < n; ++k) {
    const int64_t e = elems_per_image[k];
    if (e <= 0 || (e % pww::ctl::kVec) != 0) return PWW_ERR_BAD_ARG;
    if (!dst[k] || !res[k] || !aligned16(dst[k]) || !aligned16(res[k])) return PWW_ERR_BAD_ARG;
    a.dst[k] = dst[k];
    a.res[k] = res[k];
    a.vec_per_image[k] = e / pww::ctl::kVec;
    a.off[k + 1] = a.off[k] + (int64_t)rows * a.vec_per_image[k];
  }
  for (int k = n; k < pww::ctl::kMaxLevels; ++k) {
    a.dst[k] = nullptr;
    a.res[k] = nullptr;
    a.vec_per_image[k] = 0;
    a.off[k + 1] = a.off[n];
  }
  a.scales = scales;
  a.n = n;
  a.rows = rows;
  const cudaError_t e = pww::ctl::launch_inject<E>(a, (int64_t)pww::num_sms() * 8, (cudaStream_t)stream);
  return e == cudaSuccess ? PWW_OK : cuda_fail(e);
}

template <typename E>
int control_combine(int units, int n, void* const* out, const void* const* res, const int64_t* elems_per_image,
                    int rows, const float* scales, void* stream) {
  if (units < 1 || units > pww::ctl::kMaxUnits || n < 1 || n > pww::ctl::kMaxLevels || rows < 1 || !out || !res ||
      !elems_per_image || !scales)
    return PWW_ERR_BAD_ARG;
  pww::ctl::CombineArgs a = {};
  for (int k = 0; k < n; ++k) {
    const int64_t e = elems_per_image[k];
    if (e <= 0 || (e % pww::ctl::kVec) != 0) return PWW_ERR_BAD_ARG;
    if (!out[k] || !aligned16(out[k])) return PWW_ERR_BAD_ARG;
    a.out[k] = out[k];
    a.vec_per_image[k] = e / pww::ctl::kVec;
    a.off[k + 1] = a.off[k] + (int64_t)rows * a.vec_per_image[k];
  }
  for (int i = 0; i < units * n; ++i) {
    if (!res[i] || !aligned16(res[i])) return PWW_ERR_BAD_ARG;
    a.res[i] = res[i];
  }
  for (int k = n; k < pww::ctl::kMaxLevels; ++k) a.off[k + 1] = a.off[n];
  a.scales = scales;
  a.units = units;
  a.n = n;
  a.rows = rows;
  const cudaError_t e = pww::ctl::launch_combine<E>(a, (int64_t)pww::num_sms() * 8, (cudaStream_t)stream);
  return e == cudaSuccess ? PWW_OK : cuda_fail(e);
}

}  // namespace

extern "C" {

// Every _f16 / _bf16 pair below is one templated body above, instantiated for __half / __nv_bfloat16.
int pww_xattn_stats_f16(const void* q, const void* k, int B, int H, int N, int T, int D, int64_t q_batch_stride,
    int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride, int stat, const int32_t* wmap_index,
    float* stats, void* workspace, size_t workspace_bytes, void* stream) {
  return xattn_stats<__half>(
      q, k, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride, k_row_stride, stat, nullptr, false,
      wmap_index, stats, workspace, workspace_bytes, stream);
}
int pww_xattn_stats_bf16(const void* q, const void* k, int B, int H, int N, int T, int D, int64_t q_batch_stride,
    int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride, int stat, const int32_t* wmap_index,
    float* stats, void* workspace, size_t workspace_bytes, void* stream) {
  return xattn_stats<__nv_bfloat16>(
      q, k, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride, k_row_stride, stat, nullptr, false,
      wmap_index, stats, workspace, workspace_bytes, stream);
}

int pww_xattn_stats_multi_f16(const void* q, const void* k, int B, int H, int N, int T, int D, int64_t q_batch_stride,
    int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride, const int32_t* stat, const int32_t* wmap_index,
    float* stats, void* workspace, size_t workspace_bytes, void* stream) {
  return xattn_stats<__half>(
      q, k, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride, k_row_stride, PWW_STAT_MAX, stat, true,
      wmap_index, stats, workspace, workspace_bytes, stream);
}
int pww_xattn_stats_multi_bf16(const void* q, const void* k, int B, int H, int N, int T, int D, int64_t q_batch_stride,
    int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride, const int32_t* stat, const int32_t* wmap_index,
    float* stats, void* workspace, size_t workspace_bytes, void* stream) {
  return xattn_stats<__nv_bfloat16>(
      q, k, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride, k_row_stride, PWW_STAT_MAX, stat, true,
      wmap_index, stats, workspace, workspace_bytes, stream);
}

int pww_xattn_fwd_f16(const void* q, const void* k, const void* v, void* out, int B, int H, int N, int T, int D,
    int64_t q_batch_stride, int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride, int64_t o_batch_stride,
    int64_t o_row_stride, const float* wmap, int64_t wmap_batch_stride, const int32_t* wmap_index, const float* stats,
    const float* g_sigma, float scale, void* stream) {
  return xattn_fwd<__half>(q, k, v, out, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride, k_row_stride,
      o_batch_stride, o_row_stride, wmap, wmap_batch_stride, wmap_index, stats, g_sigma, 0, scale, stream);
}
int pww_xattn_fwd_bf16(const void* q, const void* k, const void* v, void* out, int B, int H, int N, int T, int D,
    int64_t q_batch_stride, int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride, int64_t o_batch_stride,
    int64_t o_row_stride, const float* wmap, int64_t wmap_batch_stride, const int32_t* wmap_index, const float* stats,
    const float* g_sigma, float scale, void* stream) {
  return xattn_fwd<__nv_bfloat16>(
      q, k, v, out, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride, k_row_stride,
      o_batch_stride, o_row_stride, wmap, wmap_batch_stride, wmap_index, stats, g_sigma, 0, scale, stream);
}

int pww_xattn_fwd_multi_f16(const void* q, const void* k, const void* v, void* out, int B, int H, int N, int T, int D,
    int64_t q_batch_stride, int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride, int64_t o_batch_stride,
    int64_t o_row_stride, const float* wmap, int64_t wmap_batch_stride, const int32_t* wmap_index, const float* stats,
    const float* g_sigma, float scale, void* stream) {
  return xattn_fwd<__half>(q, k, v, out, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride, k_row_stride,
      o_batch_stride, o_row_stride, wmap, wmap_batch_stride, wmap_index, stats, g_sigma, 1, scale, stream);
}
int pww_xattn_fwd_multi_bf16(const void* q, const void* k, const void* v, void* out, int B, int H, int N, int T, int D,
    int64_t q_batch_stride, int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride, int64_t o_batch_stride,
    int64_t o_row_stride, const float* wmap, int64_t wmap_batch_stride, const int32_t* wmap_index, const float* stats,
    const float* g_sigma, float scale, void* stream) {
  return xattn_fwd<__nv_bfloat16>(
      q, k, v, out, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride, k_row_stride,
      o_batch_stride, o_row_stride, wmap, wmap_batch_stride, wmap_index, stats, g_sigma, 1, scale, stream);
}

size_t pww_xattn_fused_workspace_bytes(void) { return pww::fx::fused_workspace_bytes(); }

int pww_xattn_fused_f16(const void* q, const void* k, const void* v, void* out, int B, int H, int N, int T, int D,
    int64_t q_batch_stride, int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride, int64_t o_batch_stride,
    int64_t o_row_stride, const void* mpack, int64_t mpack_batch_stride, int Bw, const int8_t* cidx,
    const int32_t* wmap_index, int stat, const float* g_sigma, float scale, float* stats, void* workspace,
    size_t workspace_bytes, void* stream) {
  return xattn_fused<__half>(q, k, v, out, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride, k_row_stride,
      o_batch_stride, o_row_stride, mpack, mpack_batch_stride, Bw, cidx, wmap_index, stat, nullptr, false,
      g_sigma, scale, stats, workspace, workspace_bytes, stream);
}
int pww_xattn_fused_bf16(const void* q, const void* k, const void* v, void* out, int B, int H, int N, int T, int D,
    int64_t q_batch_stride, int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride, int64_t o_batch_stride,
    int64_t o_row_stride, const void* mpack, int64_t mpack_batch_stride, int Bw, const int8_t* cidx,
    const int32_t* wmap_index, int stat, const float* g_sigma, float scale, float* stats, void* workspace,
    size_t workspace_bytes, void* stream) {
  return xattn_fused<__nv_bfloat16>(
      q, k, v, out, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride, k_row_stride,
      o_batch_stride, o_row_stride, mpack, mpack_batch_stride, Bw, cidx, wmap_index, stat, nullptr, false,
      g_sigma, scale, stats, workspace, workspace_bytes, stream);
}

int pww_xattn_fused_multi_f16(const void* q, const void* k, const void* v, void* out, int B, int H, int N, int T, int D,
    int64_t q_batch_stride, int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride, int64_t o_batch_stride,
    int64_t o_row_stride, const void* mpack, int64_t mpack_batch_stride, int Bw, const int8_t* cidx,
    const int32_t* wmap_index, const int32_t* stat, const float* g_sigma, float scale, float* stats, void* workspace,
    size_t workspace_bytes, void* stream) {
  return xattn_fused<__half>(q, k, v, out, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride, k_row_stride,
      o_batch_stride, o_row_stride, mpack, mpack_batch_stride, Bw, cidx, wmap_index, PWW_STAT_MAX, stat, true,
      g_sigma, scale, stats, workspace, workspace_bytes, stream);
}
int pww_xattn_fused_multi_bf16(const void* q, const void* k, const void* v, void* out, int B, int H, int N, int T, int D,
    int64_t q_batch_stride, int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride, int64_t o_batch_stride,
    int64_t o_row_stride, const void* mpack, int64_t mpack_batch_stride, int Bw, const int8_t* cidx,
    const int32_t* wmap_index, const int32_t* stat, const float* g_sigma, float scale, float* stats, void* workspace,
    size_t workspace_bytes, void* stream) {
  return xattn_fused<__nv_bfloat16>(
      q, k, v, out, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride, k_row_stride,
      o_batch_stride, o_row_stride, mpack, mpack_batch_stride, Bw, cidx, wmap_index, PWW_STAT_MAX, stat, true,
      g_sigma, scale, stats, workspace, workspace_bytes, stream);
}

int pww_xattn_fused_rec_f16(const void* q, const void* k, const void* v, void* out, int B, int H, int N, int T, int D,
    int64_t q_batch_stride, int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride, int64_t o_batch_stride,
    int64_t o_row_stride, const void* mpack, int64_t mpack_batch_stride, int Bw, const int8_t* cidx,
    const int32_t* wmap_index, const int32_t* stat, const float* g_sigma, float scale, float* stats, void* workspace,
    size_t workspace_bytes, void* stream, const int8_t* ridx, const int32_t* rec_index, float* rec_acc,
    int64_t rec_batch_stride) {
  const pww::fx::FxRecord rec = {ridx, rec_index, rec_acc, rec_batch_stride};
  return xattn_fused<__half>(q, k, v, out, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride, k_row_stride,
      o_batch_stride, o_row_stride, mpack, mpack_batch_stride, Bw, cidx, wmap_index, PWW_STAT_MAX, stat, true,
      g_sigma, scale, stats, workspace, workspace_bytes, stream, &rec);
}
int pww_xattn_fused_rec_bf16(const void* q, const void* k, const void* v, void* out, int B, int H, int N, int T, int D,
    int64_t q_batch_stride, int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride, int64_t o_batch_stride,
    int64_t o_row_stride, const void* mpack, int64_t mpack_batch_stride, int Bw, const int8_t* cidx,
    const int32_t* wmap_index, const int32_t* stat, const float* g_sigma, float scale, float* stats, void* workspace,
    size_t workspace_bytes, void* stream, const int8_t* ridx, const int32_t* rec_index, float* rec_acc,
    int64_t rec_batch_stride) {
  const pww::fx::FxRecord rec = {ridx, rec_index, rec_acc, rec_batch_stride};
  return xattn_fused<__nv_bfloat16>(
      q, k, v, out, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride, k_row_stride,
      o_batch_stride, o_row_stride, mpack, mpack_batch_stride, Bw, cidx, wmap_index, PWW_STAT_MAX, stat, true,
      g_sigma, scale, stats, workspace, workspace_bytes, stream, &rec);
}

int pww_xattn_fused_region_f16(const void* q, const void* k, const void* v, void* out, int B, int H, int N, int T,
    int D, int64_t q_batch_stride, int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride,
    int64_t o_batch_stride, int64_t o_row_stride, const void* mpack, int64_t mpack_batch_stride, int Bw,
    const int8_t* cidx, const int32_t* wmap_index, int stat, const float* g_sigma, float scale, float* stats,
    void* workspace, size_t workspace_bytes, void* stream, const float* region_weights, int64_t region_batch_stride) {
  const pww::fx::FxRegion rg = {region_weights, region_batch_stride, wmap_index};
  return xattn_fused<__half>(q, k, v, out, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride, k_row_stride,
      o_batch_stride, o_row_stride, mpack, mpack_batch_stride, Bw, cidx, wmap_index, stat, nullptr, false,
      g_sigma, scale, stats, workspace, workspace_bytes, stream, nullptr, &rg);
}
int pww_xattn_fused_region_bf16(const void* q, const void* k, const void* v, void* out, int B, int H, int N, int T,
    int D, int64_t q_batch_stride, int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride,
    int64_t o_batch_stride, int64_t o_row_stride, const void* mpack, int64_t mpack_batch_stride, int Bw,
    const int8_t* cidx, const int32_t* wmap_index, int stat, const float* g_sigma, float scale, float* stats,
    void* workspace, size_t workspace_bytes, void* stream, const float* region_weights, int64_t region_batch_stride) {
  const pww::fx::FxRegion rg = {region_weights, region_batch_stride, wmap_index};
  return xattn_fused<__nv_bfloat16>(q, k, v, out, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride,
      k_row_stride, o_batch_stride, o_row_stride, mpack, mpack_batch_stride, Bw, cidx, wmap_index, stat, nullptr, false,
      g_sigma, scale, stats, workspace, workspace_bytes, stream, nullptr, &rg);
}
int pww_xattn_fused_region_multi_f16(const void* q, const void* k, const void* v, void* out, int B, int H, int N,
    int T, int D, int64_t q_batch_stride, int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride,
    int64_t o_batch_stride, int64_t o_row_stride, const void* mpack, int64_t mpack_batch_stride, int Bw,
    const int8_t* cidx, const int32_t* wmap_index, const int32_t* stat, const float* g_sigma, float scale, float* stats,
    void* workspace, size_t workspace_bytes, void* stream, const float* region_weights, int64_t region_batch_stride) {
  const pww::fx::FxRegion rg = {region_weights, region_batch_stride, wmap_index};
  return xattn_fused<__half>(q, k, v, out, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride, k_row_stride,
      o_batch_stride, o_row_stride, mpack, mpack_batch_stride, Bw, cidx, wmap_index, PWW_STAT_MAX, stat, true,
      g_sigma, scale, stats, workspace, workspace_bytes, stream, nullptr, &rg);
}
int pww_xattn_fused_region_multi_bf16(const void* q, const void* k, const void* v, void* out, int B, int H, int N,
    int T, int D, int64_t q_batch_stride, int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride,
    int64_t o_batch_stride, int64_t o_row_stride, const void* mpack, int64_t mpack_batch_stride, int Bw,
    const int8_t* cidx, const int32_t* wmap_index, const int32_t* stat, const float* g_sigma, float scale, float* stats,
    void* workspace, size_t workspace_bytes, void* stream, const float* region_weights, int64_t region_batch_stride) {
  const pww::fx::FxRegion rg = {region_weights, region_batch_stride, wmap_index};
  return xattn_fused<__nv_bfloat16>(q, k, v, out, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride,
      k_row_stride, o_batch_stride, o_row_stride, mpack, mpack_batch_stride, Bw, cidx, wmap_index, PWW_STAT_MAX, stat,
      true, g_sigma, scale, stats, workspace, workspace_bytes, stream, nullptr, &rg);
}

int pww_xattn_fused_region_rows_f16(const void* q, const void* k, const void* v, void* out, int B, int H, int N, int T,
    int D, int64_t q_batch_stride, int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride,
    int64_t o_batch_stride, int64_t o_row_stride, const void* mpack, int64_t mpack_batch_stride, int Bw,
    const int8_t* cidx, const int32_t* wmap_index, int stat, const float* g_sigma, float scale, float* stats,
    void* workspace, size_t workspace_bytes, void* stream, const float* region_weights, int64_t region_batch_stride,
    const int32_t* region_index, const int32_t* stat_chunks) {
  const pww::fx::FxRegion rg = {region_weights, region_batch_stride, region_index, stat_chunks};
  return xattn_fused<__half>(q, k, v, out, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride, k_row_stride,
      o_batch_stride, o_row_stride, mpack, mpack_batch_stride, Bw, cidx, wmap_index, stat, nullptr, false,
      g_sigma, scale, stats, workspace, workspace_bytes, stream, nullptr, &rg);
}
int pww_xattn_fused_region_rows_bf16(const void* q, const void* k, const void* v, void* out, int B, int H, int N,
    int T, int D, int64_t q_batch_stride, int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride,
    int64_t o_batch_stride, int64_t o_row_stride, const void* mpack, int64_t mpack_batch_stride, int Bw,
    const int8_t* cidx, const int32_t* wmap_index, int stat, const float* g_sigma, float scale, float* stats,
    void* workspace, size_t workspace_bytes, void* stream, const float* region_weights, int64_t region_batch_stride,
    const int32_t* region_index, const int32_t* stat_chunks) {
  const pww::fx::FxRegion rg = {region_weights, region_batch_stride, region_index, stat_chunks};
  return xattn_fused<__nv_bfloat16>(q, k, v, out, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride,
      k_row_stride, o_batch_stride, o_row_stride, mpack, mpack_batch_stride, Bw, cidx, wmap_index, stat, nullptr, false,
      g_sigma, scale, stats, workspace, workspace_bytes, stream, nullptr, &rg);
}
int pww_xattn_fused_region_rows_multi_f16(const void* q, const void* k, const void* v, void* out, int B, int H, int N,
    int T, int D, int64_t q_batch_stride, int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride,
    int64_t o_batch_stride, int64_t o_row_stride, const void* mpack, int64_t mpack_batch_stride, int Bw,
    const int8_t* cidx, const int32_t* wmap_index, const int32_t* stat, const float* g_sigma, float scale, float* stats,
    void* workspace, size_t workspace_bytes, void* stream, const float* region_weights, int64_t region_batch_stride,
    const int32_t* region_index, const int32_t* stat_chunks) {
  const pww::fx::FxRegion rg = {region_weights, region_batch_stride, region_index, stat_chunks};
  return xattn_fused<__half>(q, k, v, out, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride, k_row_stride,
      o_batch_stride, o_row_stride, mpack, mpack_batch_stride, Bw, cidx, wmap_index, PWW_STAT_MAX, stat, true,
      g_sigma, scale, stats, workspace, workspace_bytes, stream, nullptr, &rg);
}
int pww_xattn_fused_region_rows_multi_bf16(const void* q, const void* k, const void* v, void* out, int B, int H, int N,
    int T, int D, int64_t q_batch_stride, int64_t q_row_stride, int64_t k_batch_stride, int64_t k_row_stride,
    int64_t o_batch_stride, int64_t o_row_stride, const void* mpack, int64_t mpack_batch_stride, int Bw,
    const int8_t* cidx, const int32_t* wmap_index, const int32_t* stat, const float* g_sigma, float scale, float* stats,
    void* workspace, size_t workspace_bytes, void* stream, const float* region_weights, int64_t region_batch_stride,
    const int32_t* region_index, const int32_t* stat_chunks) {
  const pww::fx::FxRegion rg = {region_weights, region_batch_stride, region_index, stat_chunks};
  return xattn_fused<__nv_bfloat16>(q, k, v, out, B, H, N, T, D, q_batch_stride, q_row_stride, k_batch_stride,
      k_row_stride, o_batch_stride, o_row_stride, mpack, mpack_batch_stride, Bw, cidx, wmap_index, PWW_STAT_MAX, stat,
      true, g_sigma, scale, stats, workspace, workspace_bytes, stream, nullptr, &rg);
}

int pww_attn_fwd_f16(const void* q, const void* k, const void* v, void* out, int B, int H, int N, int D,
    int64_t qkv_batch_stride, int64_t qkv_row_stride, int64_t o_batch_stride, int64_t o_row_stride, float scale,
    void* stream) {
  return attn_fwd<__half>(
      q, k, v, out, B, H, N, D, qkv_batch_stride, qkv_row_stride, o_batch_stride, o_row_stride, scale, stream);
}
int pww_attn_fwd_bf16(const void* q, const void* k, const void* v, void* out, int B, int H, int N, int D,
    int64_t qkv_batch_stride, int64_t qkv_row_stride, int64_t o_batch_stride, int64_t o_row_stride, float scale,
    void* stream) {
  return attn_fwd<__nv_bfloat16>(
      q, k, v, out, B, H, N, D, qkv_batch_stride, qkv_row_stride, o_batch_stride, o_row_stride, scale, stream);
}

size_t pww_groupnorm_workspace_bytes(int B, int HW, int G) {
  if (B <= 0 || HW <= 0 || G <= 0) return 0;
  // gn_split never makes more than min(HW, kGnMaxChunks) row chunks, whatever C is
  const size_t chunks = (size_t)std::min(HW, pww::uops::kGnMaxChunks);
  return align_up((size_t)B * G * chunks * sizeof(float2), 256);
}

int pww_groupnorm_nhwc_f16(const void* x, const void* add, int64_t add_batch_stride, const void* gamma,
    const void* beta, void* y, int B, int HW, int C, int G, float eps, int silu, void* workspace, size_t workspace_bytes,
    void* stream) {
  return groupnorm_nhwc<__half>(
      x, add, add_batch_stride, gamma, beta, y, B, HW, C, G, eps, silu, workspace, workspace_bytes,
      stream);
}
int pww_groupnorm_nhwc_bf16(const void* x, const void* add, int64_t add_batch_stride, const void* gamma,
    const void* beta, void* y, int B, int HW, int C, int G, float eps, int silu, void* workspace, size_t workspace_bytes,
    void* stream) {
  return groupnorm_nhwc<__nv_bfloat16>(
      x, add, add_batch_stride, gamma, beta, y, B, HW, C, G, eps, silu, workspace, workspace_bytes,
      stream);
}

int pww_geglu_f16(const void* in, void* out, int64_t M, int I, void* stream) {
  return geglu<__half>(in, out, M, I, stream);
}
int pww_geglu_bf16(const void* in, void* out, int64_t M, int I, void* stream) {
  return geglu<__nv_bfloat16>(in, out, M, I, stream);
}

int pww_add_layernorm_f16(const void* x, const void* res, const void* gamma, const void* beta, void* sum_out, void* y,
    int64_t M, int C, float eps, void* stream) {
  return add_layernorm<__half>(x, res, gamma, beta, sum_out, y, M, C, eps, stream);
}
int pww_add_layernorm_bf16(const void* x, const void* res, const void* gamma, const void* beta, void* sum_out, void* y,
    int64_t M, int C, float eps, void* stream) {
  return add_layernorm<__nv_bfloat16>(x, res, gamma, beta, sum_out, y, M, C, eps, stream);
}

int pww_resnet_residual_f16(const void* a, const void* h, const float* bias, void* out, int64_t rows, int C,
                            void* stream) {
  return resnet_residual<__half>(a, h, bias, out, rows, C, stream);
}
int pww_resnet_residual_bf16(const void* a, const void* h, const float* bias, void* out, int64_t rows, int C,
                             void* stream) {
  return resnet_residual<__nv_bfloat16>(a, h, bias, out, rows, C, stream);
}

int pww_adapter_residual_f16(const void* a, const void* b, const float* bias, const void* feat, void* out, int rows,
                             int64_t pixels, int C, int feat_rows, void* stream) {
  return adapter_residual<__half>(a, b, bias, feat, out, rows, pixels, C, feat_rows, stream);
}
int pww_adapter_residual_bf16(const void* a, const void* b, const float* bias, const void* feat, void* out, int rows,
                              int64_t pixels, int C, int feat_rows, void* stream) {
  return adapter_residual<__nv_bfloat16>(a, b, bias, feat, out, rows, pixels, C, feat_rows, stream);
}

int pww_sampler_input(const float* latents, const float* scale, const float* extra, void* out, int out_dtype, int m,
                      int channels, int height, int width, void* stream) {
  if (!latents || !scale || !out || m <= 0 || height <= 0 || width <= 0) return PWW_ERR_BAD_ARG;
  if (channels != 4 && channels != 9) return PWW_ERR_BAD_ARG;
  if ((channels == 9) != (extra != nullptr)) return PWW_ERR_BAD_ARG;
  if (out_dtype != PWW_DTYPE_F32 && out_dtype != PWW_DTYPE_F16 && out_dtype != PWW_DTYPE_BF16) return PWW_ERR_UNSUPPORTED;
  pww::smp::InputArgs a;
  a.lat = latents; a.scale = scale; a.extra = extra; a.out = out; a.m = m; a.C = channels; a.hw = height * width;
  const bool px4 = (a.hw % 4) == 0 && aligned16(latents) && (!extra || aligned16(extra)) && aligned16(out);
  const cudaError_t e = with_dtype(out_dtype, [&](auto t) {
    return pww::smp::launch_input<decltype(t)>(a, px4, (cudaStream_t)stream);
  });
  return e == cudaSuccess ? PWW_OK : cuda_fail(e);
}

int pww_sampler_update(const void* eps, int eps_dtype, int64_t eps_batch_stride, int64_t eps_channel_stride,
                       int64_t eps_row_stride, int64_t eps_col_stride, float* latents, float* history, int history_len,
                       const float* noise, const float* guidance, const float* beta, const float* form, int m,
                       int height, int width, void* stream) {
  pww::smp::UpdateArgs a;
  bool px4, cl;
  const int st = update_setup(eps, eps_dtype, eps_batch_stride, eps_channel_stride, eps_row_stride, eps_col_stride,
                              latents, history, history_len, noise, guidance, beta, form, m, height, width, true, a,
                              px4, cl);
  if (st != PWW_OK) return st;
  const cudaError_t e = with_dtype(eps_dtype, [&](auto t) {
    return pww::smp::launch_update<decltype(t), false>(a, pww::smp::BlendArgs{}, px4, cl, (cudaStream_t)stream);
  });
  return e == cudaSuccess ? PWW_OK : cuda_fail(e);
}

int pww_sampler_update_rescale(const void* eps, int eps_dtype, int64_t eps_batch_stride, int64_t eps_channel_stride,
                               int64_t eps_row_stride, int64_t eps_col_stride, float* latents, float* history,
                               int history_len, const float* noise, const float* guidance, const float* beta,
                               const float* form, const float* rescale, float* stats_out, int m, int height, int width,
                               void* stream) {
  if (!rescale) return PWW_ERR_BAD_ARG;
  pww::smp::UpdateArgs a;
  bool px4, cl;
  const int st = update_setup(eps, eps_dtype, eps_batch_stride, eps_channel_stride, eps_row_stride, eps_col_stride,
                              latents, history, history_len, noise, guidance, beta, form, m, height, width, true, a,
                              px4, cl);
  if (st != PWW_OK) return st;
  pww::smp::RescaleArgs r;
  r.phi = rescale; r.stats = stats_out;
  const cudaError_t e = with_dtype(eps_dtype, [&](auto t) {
    return pww::smp::launch_update_rescale<decltype(t), false>(a, r, pww::smp::BlendArgs{}, px4, cl,
                                                               (cudaStream_t)stream);
  });
  return e == cudaSuccess ? PWW_OK : cuda_fail(e);
}

int pww_sampler_update_masked(const void* eps, int eps_dtype, int64_t eps_batch_stride, int64_t eps_channel_stride,
                              int64_t eps_row_stride, int64_t eps_col_stride, float* latents, float* history,
                              int history_len, const float* noise, const float* guidance, const float* beta,
                              const float* form, const float* rescale, float* stats_out, const float* init_latents,
                              const float* init_noise, const float* mask, const float* sigma_next, int m, int height,
                              int width, void* stream) {
  if (!init_latents || !init_noise || !mask || !sigma_next || (stats_out && !rescale)) return PWW_ERR_BAD_ARG;
  pww::smp::UpdateArgs a;
  bool px4, cl;
  // the blend inputs are read 4 pixels at a time too
  const bool blend16 = aligned16(init_latents) && aligned16(init_noise) && aligned16(mask);
  const int st = update_setup(eps, eps_dtype, eps_batch_stride, eps_channel_stride, eps_row_stride, eps_col_stride,
                              latents, history, history_len, noise, guidance, beta, form, m, height, width, blend16, a,
                              px4, cl);
  if (st != PWW_OK) return st;
  pww::smp::BlendArgs bl;
  bl.init = init_latents; bl.noise0 = init_noise; bl.mask = mask; bl.sigma_next = sigma_next;
  pww::smp::RescaleArgs r;
  r.phi = rescale; r.stats = stats_out;
  const cudaError_t e = with_dtype(eps_dtype, [&](auto t) {
    using T = decltype(t);
    return rescale ? pww::smp::launch_update_rescale<T, true>(a, r, bl, px4, cl, (cudaStream_t)stream)
                   : pww::smp::launch_update<T, true>(a, bl, px4, cl, (cudaStream_t)stream);
  });
  return e == cudaSuccess ? PWW_OK : cuda_fail(e);
}

int pww_window_input(const float* latents, const float* scale, const int* row_starts, int n_rows,
                     const int* col_starts, int n_cols, int first_view, int n_views, int window, void* out,
                     int out_dtype, int height, int width, void* stream) {
  if (!latents || !scale || !row_starts || !col_starts || !out) return PWW_ERR_BAD_ARG;
  if (height <= 0 || width <= 0 || window <= 0 || window > height || window > width) return PWW_ERR_BAD_ARG;
  if (n_rows <= 0 || n_cols <= 0 || n_views <= 0 || first_view < 0 ||
      (int64_t)first_view + n_views > (int64_t)n_rows * n_cols)
    return PWW_ERR_BAD_ARG;
  if (out_dtype != PWW_DTYPE_F32 && out_dtype != PWW_DTYPE_F16 && out_dtype != PWW_DTYPE_BF16) return PWW_ERR_UNSUPPORTED;
  pww::smp::WindowInputArgs a;
  a.lat = latents; a.scale = scale; a.rows = row_starts; a.cols = col_starts; a.out = out;
  a.n_cols = n_cols; a.first = first_view; a.n = n_views; a.window = window; a.H = height; a.W = width;
  const bool px4 = (window % 4) == 0 && aligned16(out);
  const cudaError_t e = with_dtype(out_dtype, [&](auto t) {
    return pww::smp::launch_window_input<decltype(t)>(a, px4, (cudaStream_t)stream);
  });
  return e == cudaSuccess ? PWW_OK : cuda_fail(e);
}

int pww_window_update(const void* const* eps, int n_chunks, int views_per_chunk, int eps_dtype,
                      int64_t eps_batch_stride, int64_t eps_channel_stride, int64_t eps_row_stride,
                      int64_t eps_col_stride, const int* row_starts, int n_rows, const int* col_starts, int n_cols,
                      int window, float* latents, float* history, int history_len, const float* noise,
                      const float* guidance, const float* beta, const float* form, int height, int width,
                      void* stream) {
  if (!eps || !row_starts || !col_starts || !latents || !history || !guidance || !beta || !form) return PWW_ERR_BAD_ARG;
  if (height <= 0 || width <= 0 || window <= 0 || window > height || window > width) return PWW_ERR_BAD_ARG;
  if (history_len < 1 || history_len > 4 || n_rows <= 0 || n_cols <= 0 || views_per_chunk <= 0) return PWW_ERR_BAD_ARG;
  if (n_chunks < 1 || n_chunks > pww::smp::kMaxWindowChunks) return PWW_ERR_BAD_ARG;
  const int64_t views = (int64_t)n_rows * n_cols;
  if ((views + views_per_chunk - 1) / views_per_chunk != n_chunks) return PWW_ERR_BAD_ARG;
  if (eps_dtype != PWW_DTYPE_F32 && eps_dtype != PWW_DTYPE_F16 && eps_dtype != PWW_DTYPE_BF16) return PWW_ERR_UNSUPPORTED;
  const size_t es = eps_dtype == PWW_DTYPE_F32 ? 4 : 2;
  // window outputs are read one pixel (4 channels) at a time: channels-last packed rows take one 8- or 16-byte access
  const size_t need = 4 * es;
  bool cl = eps_channel_stride == 1 && eps_col_stride == 4 && eps_row_stride == 4 * (int64_t)window &&
            ((size_t)eps_batch_stride * es) % need == 0;
  pww::smp::WindowOutputs t;
  for (int k = 0; k < n_chunks; ++k) {
    if (!eps[k]) return PWW_ERR_BAD_ARG;
    t.eps[k] = eps[k];
    cl = cl && (reinterpret_cast<uintptr_t>(eps[k]) % need) == 0;
  }
  pww::smp::UpdateArgs a{};
  a.lat = latents; a.hist = history; a.noise = noise; a.gscale = guidance; a.beta = beta; a.form = form;
  a.m = 1; a.h = height; a.w = width; a.nh = history_len;
  pww::smp::WindowArgs v;
  v.rows = row_starts; v.cols = col_starts; v.n_rows = n_rows; v.n_cols = n_cols; v.window = window;
  v.per_chunk = views_per_chunk; v.views = (int)views;
  v.e_sn = eps_batch_stride; v.e_sc = eps_channel_stride; v.e_sh = eps_row_stride; v.e_sw = eps_col_stride;
  const bool px4 = (width % 4) == 0 && aligned16(latents) && aligned16(history) && (!noise || aligned16(noise));
  const cudaError_t e = with_dtype(eps_dtype, [&](auto et) {
    return pww::smp::launch_window_update<decltype(et)>(a, v, t, px4, cl, (cudaStream_t)stream);
  });
  return e == cudaSuccess ? PWW_OK : cuda_fail(e);
}

int pww_control_inject_f16(int n, void* const* dst, const void* const* res, const int64_t* elems_per_image, int rows,
                           const float* scales, void* stream) {
  return control_inject<__half>(n, dst, res, elems_per_image, rows, scales, stream);
}
int pww_control_inject_bf16(int n, void* const* dst, const void* const* res, const int64_t* elems_per_image, int rows,
                            const float* scales, void* stream) {
  return control_inject<__nv_bfloat16>(n, dst, res, elems_per_image, rows, scales, stream);
}

int pww_control_combine_f16(int units, int n, void* const* out, const void* const* res,
                            const int64_t* elems_per_image, int rows, const float* scales, void* stream) {
  return control_combine<__half>(units, n, out, res, elems_per_image, rows, scales, stream);
}
int pww_control_combine_bf16(int units, int n, void* const* out, const void* const* res,
                             const int64_t* elems_per_image, int rows, const float* scales, void* stream) {
  return control_combine<__nv_bfloat16>(units, n, out, res, elems_per_image, rows, scales, stream);
}

// Test infrastructure (not declared in the public header): replay the forward kernel's unit schedule on the host.
// wmap_index and out are HOST pointers; out receives 5 int32 per unit (see fwd_schedule_host); returns the number of
// units written or a negative value for bad arguments.  No GPU needed.
int pww_debug_fwd_schedule(int B, int H, int tiles, int grid, const int* wmap_index, int* out) {
  if (!wmap_index || !out) return PWW_ERR_BAD_ARG;
  return pww::tc::fwd_schedule_host(B, H, tiles, grid, wmap_index, out);
}

// Test infrastructure (not declared in the public header): cap the persistent grid of the fused kernel (0 = all SMs) so
// small shapes exercise long job lists; does CTA `cta` contribute a partial to image b's statistic (H = head GROUPS)?
int pww_debug_set_fused_grid(int grid) {
  pww::fx::debug_grid() = grid < 0 ? 0 : grid;
  return PWW_OK;
}
// Host replay of the grouped-head kernel's job lists (8 int32 per job, see fused2_schedule_host).
int pww_debug_fused2_schedule(int B, int H, int G, int tiles, int grid, const int* wmap_index, int* out, int max_jobs) {
  if (!wmap_index || !out) return PWW_ERR_BAD_ARG;
  return pww::fx::fused2_schedule_host(B, H, G, tiles, grid, wmap_index, out, max_jobs);
}
// Heads per unit of the grouped-head kernel at head dim 40 (a build-time constant).
int pww_debug_fused2_heads_per_unit(void) { return pww::fx::Cfg2<40>::G; }
// Test infrastructure: device buffer of grid * (2 + 1024) uint32 the grouped-head kernel copies every CTA's job table to.
int pww_debug_set_fused_jobs_dump(void* device_buffer) {
  pww::fx::debug_jobs_dump() = (unsigned*)device_buffer;
  return PWW_OK;
}
int pww_debug_fused_cta_has_image(int cta, int grid, int B, int H, int tiles, const int* wmap_index, int b) {
  if (!wmap_index) return PWW_ERR_BAD_ARG;
  return pww::fx::fused_cta_has_image_host(cta, grid, B, H, tiles, wmap_index, b);
}

}  // extern "C"
