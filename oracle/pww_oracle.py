"""CPU restatement of the Paint-with-Words hot path -- the parity ORACLE.

TEST INFRASTRUCTURE.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import this file, and only as the checker (or as the timed CPU baseline).  The product package
`paint_with_words_sd_b200` never imports it and has no CPU fallback.

Every function restates one reference function (file:line relative to the reference checkout's root) in plain
torch-CPU / numpy.  Pinning: the reference ships NO tests or golden vectors for this path (SURVEY.md
section 4), so the restatement is pinned against outputs of the reference's own functions executed in
the build container through `oracle/ref_loader.py`; `tests/golden/make_golden.py` generated the
committed fixtures in tests/golden/*.npz and `tests/test_oracle_golden.py` checks this file against
them (bit-exact for the integer/mask steps, 1e-6 relative for fp32 attention).

Reference semantics that are easy to get wrong and are restated faithfully here:
  * scores are UNSCALED when the statistic is taken and when the bias is added; `scale` multiplies
    (scores + bias) afterwards                                   (paint_with_words.py:87,112)
  * qk.max() / qk.std() span ALL heads and all pixels of the image: one scalar per call (pww.py:106)
  * std is the unbiased (Bessel) estimator, torch.Tensor.std default
  * the uncond branch and tensor/None contexts add exactly 0.0    (pww.py:107-110, 493)
"""
from __future__ import annotations

import math
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F


# --------------------------------------------------------------------------------------------
# integer / index helpers
# --------------------------------------------------------------------------------------------
def always_round(x: float) -> int:
    """Round-half-up for even integer parts, Python round() (banker's) otherwise.
    Restates paint_with_words.py:18-26 (the odd branch really is `round`, so 33.5 -> 34, 31.5 -> 32)."""
    ix = int(x)
    if ix % 2 == 0:
        return ix if x < ix + 0.5 else ix + 1
    return round(x)


def img_importance_flatten(img: torch.Tensor, w: int, h: int) -> torch.Tensor:
    """Bilinear, align_corners=True resize of a [H,W] fp32 map to (w,h).  paint_with_words.py:38-45.

    Bit-exactness note: this is the same ATen CPU call the reference makes.  A hand-rolled numpy
    bilinear differs from ATen by 1 ulp on O(100) pixels (FMA contraction inside ATen's vectorised
    kernel), so the oracle -- like the product's host-side builder -- keeps the ATen call and the
    golden fixtures pin its output."""
    return F.interpolate(img.unsqueeze(0).unsqueeze(1), size=(w, h), mode="bilinear",
                         align_corners=True).squeeze()


def parse_color_key(color) -> Tuple[int, int, int]:
    """'#rrggbb' -> (r,g,b); tuples pass through.  paint_with_words.py:228-230."""
    if isinstance(color, str):
        return (int(color[1:3], 16), int(color[3:5], 16), int(color[5:7], 16))
    return tuple(int(c) for c in color)


def image_context_separator(img_rgb: Optional[np.ndarray], color_context: Dict, tokenizer):
    """paint_with_words.py:207-244.  `img_rgb` is uint8 [H,W,3] (np.array of the PIL image) or None.
    Returns (list of (label_token_ids, strength_mask[H,W] fp32), w, h) with (w,h) in PIL order."""
    ret = []
    if img_rgb is not None:
        h, w = img_rgb.shape[:2]
        for color, v in color_context.items():
            parts = v.split(",")
            strength = float(parts[-1])
            label = ",".join(parts[:-1])
            ids = tokenizer(label, max_length=tokenizer.model_max_length, truncation=True)["input_ids"][1:-1]
            rgb = parse_color_key(color)
            where = (img_rgb == np.array(rgb, dtype=img_rgb.dtype)).all(axis=-1)  # exact integer match
            ret.append((list(ids), torch.tensor(where, dtype=torch.float32) * strength))
    else:
        w, h = 512, 512
    if len(ret) == 0:
        ret.append(([-1], torch.zeros((w, h), dtype=torch.float32)))
    return ret, w, h


def tokens_img_attention_weight(separated, token_ids: Sequence[int], ratio: int = 8,
                                original_shape: bool = False) -> torch.Tensor:
    """paint_with_words.py:247-276.  `token_ids` is the 77-id prompt sequence.
    For every start index where the label's ids occur in the prompt, ADD the region mask (bilinearly
    resized to always_round(H/ratio) x always_round(W/ratio)) to those columns."""
    token_lis = list(token_ids)
    w, h = separated[0][1].shape  # reference naming: first dim called w
    w_r, h_r = always_round(w / ratio), always_round(h / ratio)
    ret = torch.zeros((w_r * h_r, len(token_lis)), dtype=torch.float32)
    for label_ids, mask in separated:
        L = len(label_ids)
        for idx in range(len(token_lis)):
            if token_lis[idx: idx + L] == label_ids:
                ret[:, idx: idx + L] += img_importance_flatten(mask, w_r, h_r).reshape(-1, 1).repeat(1, L)
    if original_shape:
        ret = ret.reshape((w_r, h_r, len(token_lis)))
    return ret


def extract_seed_and_sigma_from_context(color_context: Dict, ignore_seed: int = -1):
    """paint_with_words.py:279-297.  Mutates and returns `color_context` like the reference."""
    extra_seeds, extra_sigmas = {}, {}
    for i, (k, ctx) in enumerate(color_context.items()):
        parts = ctx.split(",")
        if len(parts) > 2:
            try:
                seed = int(parts[-2])
                sigma = float(parts[-1])
                parts = parts[:-2]
                extra_sigmas[i] = sigma
            except ValueError:
                seed = int(parts[-1])
                parts = parts[:-1]
            if seed != ignore_seed:
                extra_seeds[i] = seed
        color_context[k] = ",".join(parts)
    return color_context, extra_seeds, extra_sigmas


def get_binary_mask(separated, extra_seeds: Dict[int, int], dtype, size):
    """paint_with_words.py:300-304 (bilinear, align_corners=False default)."""
    masks = [(separated[k][1] > 0).type(dtype) for k in extra_seeds.keys()]
    return [F.interpolate(m.unsqueeze(0).unsqueeze(1), size=size, mode="bilinear") for m in masks]


def gaussian_blur_39(img: torch.Tensor, sigma: float) -> torch.Tensor:
    """torchvision GaussianBlur(kernel_size=39, sigma) on a [H,W] map: separable, reflect padding.
    Restates what paint_with_words.py:307-312 calls (torchvision is third-party; algorithm restated)."""
    ks = 39
    half = (ks - 1) * 0.5
    x = torch.linspace(-half, half, steps=ks, dtype=torch.float32)
    pdf = torch.exp(-0.5 * (x / sigma).pow(2))
    k1 = pdf / pdf.sum()
    k2 = torch.mm(k1[:, None], k1[None, :])
    pad = ks // 2
    t = F.pad(img[None, None], [pad, pad, pad, pad], mode="reflect")
    return F.conv2d(t, k2[None, None])[0, 0]


def regional_seed_latents(latent_size, seed: int, extra_seeds: Dict[int, int], separated) -> torch.Tensor:
    """paint_with_words.py:445-455: base latents from `seed`, regions re-seeded and mixed by mask."""
    latents = torch.randn(latent_size, generator=torch.manual_seed(seed))
    if len(extra_seeds) > 0:
        multi = [torch.randn(latent_size, generator=torch.manual_seed(s)) for s in extra_seeds.values()]
        masks = get_binary_mask(separated, extra_seeds, dtype=latents[0].dtype, size=latent_size[-2:])
        fg = (sum(masks) > 0).squeeze()
        summed = sum(l * m for l, m in zip(multi, masks))
        latents[:, :, fg] = summed[:, :, fg]
    return latents


# --------------------------------------------------------------------------------------------
# the hot function
# --------------------------------------------------------------------------------------------
def default_weight_function(w, sigma, qk):
    """paint_with_words.py:402-405."""
    return 0.1 * w * math.log(sigma + 1) * qk.max()


def _h2b(x: torch.Tensor, heads: int) -> torch.Tensor:
    b, n, c = x.shape
    return x.reshape(b, n, heads, c // heads).permute(0, 2, 1, 3).reshape(b * heads, n, c // heads)


def _b2h(x: torch.Tensor, heads: int) -> torch.Tensor:
    bh, n, d = x.shape
    return x.reshape(bh // heads, heads, n, d).permute(0, 2, 1, 3).reshape(bh // heads, n, heads * d)


def attention_core(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int, scale: float,
                   bias_fn: Optional[Callable[[torch.Tensor], object]] = None,
                   emulate_fp16: bool = False, emulate_dtype: Optional[torch.dtype] = None) -> torch.Tensor:
    """Everything between to_q/to_k/to_v and to_out for ONE image (B=1 as in the reference).

    q [1,N,C], k/v [1,T,C].  Restates paint_with_words.py:83-118:
        S = Q_h K_h^T (unscaled) ; S' = (S + bias_fn(S)) * scale ; P = softmax(S') ; O = P V_h.
    `bias_fn(S[h,N,T])` returns the additive term (a [N,T] tensor or 0.0).
    emulate_dtype=torch.float16 (or emulate_fp16=True) reproduces the rounding points of the reference's CUDA-autocast
    path on fp32 hardware: inputs/S/P/O rounded to fp16 where eager fp16 autocast rounds them (SURVEY 8a-1);
    emulate_dtype=torch.bfloat16 rounds at the same points to bf16, as an eager bf16 autocast does."""
    em = _emulated_dtype(emulate_fp16, emulate_dtype)

    def rnd(t):
        return t.to(em).to(torch.float32) if em is not None else t
    q, k, v = rnd(q.float()), rnd(k.float()), rnd(v.float())
    qh, kh, vh = _h2b(q, heads), _h2b(k, heads), _h2b(v, heads)
    s = rnd(torch.matmul(qh, kh.transpose(-1, -2)))
    bias = bias_fn(s.to(em) if em is not None else s) if bias_fn is not None else 0.0
    if isinstance(bias, torch.Tensor):
        bias = bias.float()
        s = (s + bias) * scale
    else:
        s = rnd((s + bias) * scale)   # half + python float stays half under autocast
    p = rnd(s.softmax(dim=-1))
    o = rnd(torch.matmul(p, vh))
    return _b2h(o, heads)


def _emulated_dtype(emulate_fp16: bool, emulate_dtype: Optional[torch.dtype]) -> Optional[torch.dtype]:
    if emulate_dtype not in (None, torch.float16, torch.bfloat16):
        raise ValueError(f"emulate_dtype must be None, torch.float16 or torch.bfloat16, got {emulate_dtype}")
    if emulate_fp16 and emulate_dtype not in (None, torch.float16):
        raise ValueError(f"emulate_fp16=True contradicts emulate_dtype={emulate_dtype}")
    return torch.float16 if emulate_fp16 else emulate_dtype


def inj_forward(attn, hidden_states, context=None, mask=None, emulate_fp16: bool = False,
                emulate_dtype: Optional[torch.dtype] = None):
    """Restates paint_with_words.py:60-125 for a module with the diffusers-0.10 CrossAttention contract
    (to_q/to_k/to_v/to_out, heads, scale).  fp32 unless emulate_fp16 / emulate_dtype (see attention_core)."""
    is_dict = True
    if context is not None:
        if isinstance(context, dict):
            ctx = context["CONTEXT_TENSOR"]
        else:
            ctx, is_dict = context, False
    else:
        ctx = hidden_states
    q = attn.to_q(hidden_states)
    k = attn.to_k(ctx)
    v = attn.to_v(ctx)
    n = q.shape[1]
    bias_fn = None
    if context is not None and is_dict:
        f = context["WEIGHT_FUNCTION"]
        try:
            w = context[f"CROSS_ATTENTION_WEIGHT_{n}"]
        except KeyError:
            w = context["CROSS_ATTENTION_WEIGHT_ORIG"]
            if not isinstance(w, int):
                w = orig_map_fallback(w, n)
            else:
                w = 0
        sigma = context["SIGMA"]
        bias_fn = lambda s: f(w, sigma, s)  # noqa: E731
    outs = []
    for b in range(q.shape[0]):            # reference is B=1; per-image stat scope for B>1
        outs.append(attention_core(q[b:b + 1], k[b:b + 1], v[b:b + 1], attn.heads, attn.scale,
                                   bias_fn, emulate_fp16, emulate_dtype))
    o = torch.cat(outs, 0)
    o = attn.to_out[0](o.to(hidden_states.dtype))
    return attn.to_out[1](o)


def orig_map_fallback(w_orig: torch.Tensor, n: int) -> torch.Tensor:
    """paint_with_words.py:97-101: rebuild an [n,77] map from the [H,W,77] ORIG map."""
    img_h, img_w, nc = w_orig.shape
    ratio = math.sqrt(img_h * img_w / n)
    w = F.interpolate(w_orig.permute(2, 0, 1).unsqueeze(0), scale_factor=1 / ratio, mode="bilinear",
                      align_corners=True)
    return F.interpolate(w.reshape(1, nc, -1), size=(n,), mode="nearest").permute(2, 1, 0).squeeze()


# --------------------------------------------------------------------------------------------
# numpy float64 form of the fused region (second, independent statement used for tolerances)
# --------------------------------------------------------------------------------------------
def attention_core_f64(q: np.ndarray, k: np.ndarray, v: np.ndarray, heads: int, scale: float,
                       w: Optional[np.ndarray], coef_g: float, stat: str) -> np.ndarray:
    """q [N,C], k/v [T,C] -> [N,C] in float64.  bias = coef_g * stat(S) * w (SURVEY 8a spec)."""
    n, c = q.shape
    d = c // heads
    qh = q.astype(np.float64).reshape(n, heads, d).transpose(1, 0, 2)
    kh = k.astype(np.float64).reshape(-1, heads, d).transpose(1, 0, 2)
    vh = v.astype(np.float64).reshape(-1, heads, d).transpose(1, 0, 2)
    s = qh @ kh.transpose(0, 2, 1)
    if w is not None:
        m = s.max() if stat == "max" else s.std(ddof=1)
        s = s + coef_g * m * w.astype(np.float64)[None]
    s = s * scale
    s = s - s.max(-1, keepdims=True)
    p = np.exp(s)
    p /= p.sum(-1, keepdims=True)
    return (p @ vh).transpose(1, 0, 2).reshape(n, c)
