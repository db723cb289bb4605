"""Per-element error bounds for the native UNet ops of `csrc/unet_ops.cuh` (GroupNorm[+add][+SiLU], GEGLU, residual
add + LayerNorm), the fp64 references they are measured against, and the shapes they are checked at.

Each kernel loads E (fp16 or bf16), does its arithmetic in fp32 and rounds to E once, so an element may differ from
the fp64 result on the same E inputs by one rounding to E plus the fp32 error of the kernel's formula:

    |got - ref| <= ulp_E(ref) + K * terms,      ulp_E(r) = 2^(floor(log2 max(|r|, tiny_E)) - p)

with p = 10 (fp16) or 7 (bf16) and tiny_E the type's smallest normal.  One ulp_E(ref) covers the final rounding (half
an ulp, or a quarter of one when the fp32 value lies across a binade edge) with half an ulp to spare.  `terms` is a
per-element magnitude built from the formula: every fp32 operation of the kernel errs by at most u = 2^-24 of its
result, and the terms list the magnitudes those results take, so that the fp32 error is at most (a small count of
ulps) x terms.  K = 2^-18 = 64 u for every kernel.  The reductions are the longest chains, and their error is taken
with the usual sqrt-of-depth growth of independent roundings (a chain of d fp32 adds errs by about sqrt(d) u, and by
d u only under adversarial rounding); the depths are listed per kernel below.

GroupNorm (`gn_stats_kernel` + `gn_apply_kernel`).  With sc = rstd * gamma, sh = beta + ((add - shift) - E[d]) * sc,
the kernel computes y = fma(x, sc, sh), then y / (1 + exp(-y)) with __expf / __fdividef.
  * rstd: the sums are taken about the group's first element (shift) and var = E[d^2] - E[d]^2.  Each sum is a chain
    of a thread's rows (gn_split: <= 36), the strided shared-memory values of a warp (<= 30) and 5 shuffles, the
    chunk partials of a lane (<= 2) and 5 shuffles: depth <= 55 at the shapes below, 204 for one 6144-channel group,
    so <= 15 u of relative error in each sum; the subtraction adds a few u while the shift lies within a few standard
    deviations of the mean, and rsqrtf 2 ulps.  Together <= ~25 u relative in sc, which reaches y through |x * sc|
    and |(add - mean) * sc|.
  * mean = shift + E[d] is never rounded as such: E[d] errs by <= 15 u of mean|x + add - shift|, which reaches y as
    mad * |sc| with mad that mean absolute deviation from the shift (a per-group term; zero for a constant group,
    about |gamma| otherwise).  A mean rounded to fp32 would err by u |mean| instead, which no term here covers where
    |add| >> std: with add ~ 0.5 and std 1e-4, rstd ~ 1 / sqrt(eps) turns it into 19 fp16 ulps of y.
  * the shift x[0] + add[0] and add - shift are exact in fp32 (sums of two E values within 13 binades of each other
    in fp16, 16 in bf16), and (add - shift) - E[d] rounds once,
    so sh errs by <= 3 u of |(add - mean) * sc| + |beta|; the fma: one rounding of y.
  The fma cancels where y ~ 0 (x * sc ~ -sh): the error there is absolute, set by |x * sc|, not by |y|.  With mean
  50 the products are ~50 while y ~ 1, so the absolute term is what lets a correct kernel through.
  SiLU: silu' <= 1.1 carries the pre-activation error over scaled by 1.1; __expf errs by <= 2 + 1.16 |y| ulps and
  __fdividef by 2, so SiLU adds <= ~21 u of |silu(y)| <= |y| <= terms for |y| <= 16 (the elements here; beyond that
  silu(y) is y or below E's range).
      terms = |x * sc| + |(add - mean) * sc| + |beta| + mad * |sc|     (x 1.1 with SiLU)
GEGLU (`geglu_kernel`): out = a * 0.5 g (1 + erff(g / sqrt 2)), torch's eager exact-erf GELU in fp32.  erff errs by
  <= 2 ulps of |erf| <= 1; the products by one rounding each.  For g below about -4, 1 + erff cancels in fp32: the
  error of 1 + erff is absolute, <= 2.5 u, so the GELU errs by <= 1.3 u |g| and at g = -5 that is 4 % of gelu(g); for
  g <= -6 the kernel returns (-)0.  This is the formula's property, shared with torch's eager GELU (which the fast
  route must match), not a fault; the absolute term covers it.
      terms = |a| (|g| + 1)
add + LayerNorm (`add_layernorm_kernel`): s = E(x + res) (bit-exact, checked separately), then two passes over s in
  fp32: mean (per-lane chains of <= 8 VPL <= 64 adds, then 5 shuffles: ~9 u of mean|s|), sum of (s - mean)^2 (same
  depth: ~9 u relative), rsqrtf (2 ulps), then (s - mean) * rstd * gamma + beta (three roundings).  The mean's error
  is per row and absolute, so it enters through mean|s| * rstd * |gamma|; the rest is relative to the normalised
  value, or to beta.
      terms = |(s - mu) * rstd * gamma| + |beta| + mean|s| * rstd * |gamma|

`tests/test_unet_ops_bound.py` runs float32 emulations of the three kernels through these bounds on the CPU (they must
pass) together with plausible wrong kernels (they must fail); `tests/test_unet_ops_bound_gpu.py` runs the kernels.
"""
from __future__ import annotations

import math

import torch

K_GN = 2.0 ** -18
K_GEGLU = 2.0 ** -18
K_LN = 2.0 ** -18

_P = {torch.float16: 10, torch.bfloat16: 7}
_TINY = {torch.float16: 2.0 ** -14, torch.bfloat16: 2.0 ** -126}
# |r| at and above which rounding to E gives inf: the largest finite value plus half its ulp
_OVERFLOW = {torch.float16: 65504.0 + 16.0, torch.bfloat16: (2.0 - 2.0 ** -7) * 2.0 ** 127 + 2.0 ** 119}

# GroupNorm shapes (HW, C, G, B).  SD1.5 and SD2.1 share the UNet's channel widths and 32 groups, so one list per
# resolution covers both: every ResNet / transformer / conv_norm_out GroupNorm of a 512 px (64x64 latent) and a 768 px
# (96x96 latent) image, cond + uncond.
SD_512 = [(4096, 320, 32, 2), (4096, 640, 32, 2), (4096, 960, 32, 2),
          (1024, 320, 32, 2), (1024, 640, 32, 2), (1024, 960, 32, 2), (1024, 1280, 32, 2), (1024, 1920, 32, 2),
          (256, 640, 32, 2), (256, 1280, 32, 2), (256, 1920, 32, 2), (256, 2560, 32, 2),
          (64, 1280, 32, 2), (64, 2560, 32, 2)]
SD_768 = [(9216, 320, 32, 2), (9216, 640, 32, 2), (9216, 960, 32, 2),
          (2304, 320, 32, 2), (2304, 640, 32, 2), (2304, 960, 32, 2), (2304, 1280, 32, 2), (2304, 1920, 32, 2),
          (576, 640, 32, 2), (576, 1280, 32, 2), (576, 1920, 32, 2), (576, 2560, 32, 2),
          (144, 1280, 32, 2), (144, 2560, 32, 2)]
GN_TINY = [(256, 160, 8, 2), (64, 480, 8, 2), (16, 960, 8, 2), (4, 640, 8, 2)]
GN_RAGGED = [(1, 320, 32, 2), (49, 640, 32, 2), (1089, 960, 32, 2)]
GN_BATCH = [(1024, 640, 32, 1), (576, 960, 32, 3), (256, 1280, 32, 16), (64, 2560, 32, 16)]
# 3 channels per group, one channel per group (G = 64), and wide channel slices up to one 6144-channel group
GN_ODD = [(100, 96, 32, 2), (33, 64, 64, 3), (300, 6144, 32, 1), (16, 6144, 1, 1)]
GN_SHAPES = SD_512 + SD_768 + GN_TINY + GN_RAGGED + GN_BATCH + GN_ODD
GN_VARIANTS = [(True, True), (True, False), (False, False)]   # (silu, with add)
GN_VARIANT_IDS = ["silu_add", "silu", "plain"]

GEGLU_I = [8, 1280, 2560, 5120]
GEGLU_M = [1, 3, 77, 2 * 4096, 2 * 9216]
# one C per vectors-per-lane instance 1..8 of add_layernorm_kernel (ceil(C / 8 / 32))
LN_C = [8, 320, 640, 1024, 1280, 1408, 1792, 2048]
LN_M = [1, 7, 8, 2 * 4096]

DTYPES = [torch.float16, torch.bfloat16]
DTYPE_IDS = ["fp16", "bf16"]


def ulp_E(r: torch.Tensor, dtype) -> torch.Tensor:
    """2^(floor(log2 max(|r|, tiny_E)) - p): the spacing of E at r (fp64)."""
    a = r.double().abs().clamp_min(_TINY[dtype])
    _, e = torch.frexp(a)                      # a = m 2^e, m in [0.5, 1): floor(log2 a) = e - 1
    return torch.ldexp(torch.ones_like(a), (e - 1 - _P[dtype]).to(a.dtype))


def check_within(got: torch.Tensor, ref64: torch.Tensor, fp32_terms: torch.Tensor, dtype, K: float,
                 name: str = "") -> float:
    """Per element |got - ref| <= ulp_E(ref) + K * fp32_terms; got may be ±inf only where ref rounds to that inf
    within the allowance.  Tensors are [B, rows, C] (image, row, channel) or [rows, C].  Raises AssertionError naming
    the worst failing element; returns the largest |got - ref| / allowance."""
    assert got.dtype == dtype, (got.dtype, dtype)
    assert got.shape == ref64.shape == fp32_terms.shape, (got.shape, ref64.shape, fp32_terms.shape)
    g, r = got.double(), ref64.double()
    allow = ulp_E(r, dtype) + K * fp32_terms.double()
    finite = torch.isfinite(g)
    err = torch.where(finite, (g - r).abs(), torch.full_like(g, math.inf))
    inf_ok = torch.isinf(g) & (torch.sign(g) == torch.sign(r)) & (r.abs() + allow >= _OVERFLOW[dtype])
    ratio = torch.where(inf_ok, torch.zeros_like(g), err / allow)   # NaN got -> inf ratio
    bad = ~(ratio <= 1.0)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    if bool(bad.any()):
        flat = int(torch.argmax(torch.where(bad, ratio, torch.full_like(ratio, -1.0)).flatten()))
        C = got.shape[-1]
        rows = got.shape[-2] if got.dim() >= 2 else 1
        b, row, c = flat // (rows * C), (flat // C) % rows, flat % C
        raise AssertionError(
            f"{name}: {int(bad.sum())} of {got.numel()} elements outside |got - ref| <= ulp_E(ref) + K * terms "
            f"(K = 2^{math.log2(K):.0f}); worst at (image {b}, row {row}, channel {c}): got {float(g.flatten()[flat])!r} "
            f"ref {float(r.flatten()[flat])!r} ulp_E {float(ulp_E(r.flatten()[flat], dtype))!r} "
            f"allowance {float(allow.flatten()[flat])!r} ({float(ratio.flatten()[flat]):.3g}x)")
    return worst


# ---- fp64 references -------------------------------------------------------------------------------------------------
def gn_reference(x, gamma, beta, G, eps, add=None, silu=False):
    """x: [B, HW, C] in E, add: [B, C] in E or None, gamma / beta: [C] in E.  (ref, terms), both fp64 [B, HW, C]."""
    B, HW, C = x.shape
    cg = C // G
    xd = x.double()
    ad = add.double()[:, None, :] if add is not None else torch.zeros(B, 1, C, dtype=torch.float64, device=x.device)
    gd, bd = gamma.double(), beta.double()
    grp = (xd + ad).reshape(B, HW, G, cg)
    mean = grp.mean(dim=(1, 3), keepdim=True)
    var = (grp - mean).pow(2).mean(dim=(1, 3), keepdim=True)
    mad = (grp - grp[:, :1, :, :1]).abs().mean(dim=(1, 3), keepdim=True)

    def per_channel(t):
        return t.expand(B, 1, G, cg).reshape(B, 1, C)
    mean, rstd, mad = per_channel(mean), per_channel((var + eps).rsqrt()), per_channel(mad)
    sc = rstd * gd
    y = (xd + ad - mean) * sc + bd
    terms = (xd * sc).abs() + ((ad - mean) * sc).abs() + bd.abs() + mad * sc.abs()
    if silu:
        y = y * torch.sigmoid(y)
        terms = 1.1 * terms
    return y, terms


def geglu_reference(h):
    """h: [M, 2I] in E.  (ref, terms) fp64 [M, I]; gelu via erfc, accurate where 1 + erf cancels."""
    I = h.shape[-1] // 2
    a, g = h[..., :I].double(), h[..., I:].double()
    gelu = 0.5 * g * torch.special.erfc(-g / math.sqrt(2.0))
    return a * gelu, a.abs() * (g.abs() + 1.0)


def ln_reference(s, gamma, beta, eps):
    """s: [M, C] in E (the rounded residual sum).  (ref, terms) fp64 [M, C]."""
    sd, gd, bd = s.double(), gamma.double(), beta.double()
    mu = sd.mean(-1, keepdim=True)
    rstd = ((sd - mu).pow(2).mean(-1, keepdim=True) + eps).rsqrt()
    n = (sd - mu) * rstd * gd
    return n + bd, n.abs() + bd.abs() + sd.abs().mean(-1, keepdim=True) * rstd * gd.abs()


# ---- inputs ----------------------------------------------------------------------------------------------------------
def _gen(device, seed):
    return torch.Generator(device=device).manual_seed(seed)


def gn_inputs(HW, C, G, B, dtype, with_add, seed, device="cpu", offset=0.3, scale=1.5):
    """(x [B, HW, C], gamma, beta, add [B, C] or None), all in E: activations ~ N(offset, scale^2)."""
    g = _gen(device, seed)
    x = (torch.randn(B, HW, C, generator=g, device=device) * scale + offset).to(dtype)
    gamma = (torch.randn(C, generator=g, device=device) * 0.5 + 1.0).to(dtype)
    beta = (torch.randn(C, generator=g, device=device) * 0.2).to(dtype)
    add = (torch.randn(B, C, generator=g, device=device) * 0.5).to(dtype) if with_add else None
    return x, gamma, beta, add


def geglu_inputs(M, I, dtype, seed, device="cpu"):
    """[M, 2I] in E: values ~ N(0, 4), gates uniform over [-10, 10] (the cancellation region included)."""
    g = _gen(device, seed)
    a = torch.randn(M, I, generator=g, device=device) * 2.0
    gate = torch.rand(M, I, generator=g, device=device) * 20.0 - 10.0
    return torch.cat([a, gate], -1).to(dtype)


def ln_inputs(M, C, dtype, seed, device="cpu", mean=0.0, std=2.0):
    """(x, res, gamma, beta) in E: x ~ N(mean, std^2), res ~ N(0, std^2)."""
    g = _gen(device, seed)
    x = (torch.randn(M, C, generator=g, device=device) * std + mean).to(dtype)
    res = (torch.randn(M, C, generator=g, device=device) * std).to(dtype)
    gamma = (torch.randn(C, generator=g, device=device) * 0.5 + 1.0).to(dtype)
    beta = (torch.randn(C, generator=g, device=device) * 0.2).to(dtype)
    return x, res, gamma, beta


def gn_case_inputs(HW, C, G, B, dtype, with_add, kind, seed, device="cpu"):
    """Inputs of one GroupNorm case: N(0.3, 1.5^2) activations, mean 50 (1000 in fp16 with kind "mean1000"), std 1e-4
    about 0 (far below sqrt(eps): eps sets rstd), or groups in which x + add is constant (variance 0)."""
    if kind in ("mean50", "mean1000"):
        return gn_inputs(HW, C, G, B, dtype, with_add, seed, device, offset=float(kind[4:]), scale=1.0)
    if kind == "std1e-4":
        return gn_inputs(HW, C, G, B, dtype, with_add, seed, device, offset=0.0, scale=1e-4)
    x, gamma, beta, add = gn_inputs(HW, C, G, B, dtype, with_add, seed, device)
    if kind == "const":
        # every other group constant over its rows and channels: x the image's group value minus add
        cg = C // G
        g = torch.Generator(device=device).manual_seed(seed + 1)
        val = (torch.randn(B, G, generator=g, device=device) * 2.0).to(dtype)
        a = add if add is not None else torch.zeros(B, C, dtype=dtype, device=device)
        a = a.reshape(B, G, cg)
        a[:, :, :] = a[:, :, :1]                                  # add constant within each group
        const = (val[:, :, None] - a.float()).to(dtype).reshape(B, 1, C)
        on = (torch.arange(C, device=device) // cg) % 2 == 0
        x[:, :, on] = const[:, :, on].expand(B, HW, int(on.sum()))
        add = a.reshape(B, C) if add is not None else None
    return x, gamma, beta, add
