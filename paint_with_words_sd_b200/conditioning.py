"""Host-side conditioning builder: color map + color_context + prompt -> per-resolution weight maps
and the two context dicts that travel through the UNet as `encoder_hidden_states`.

Mirrors the reference interface (same function names, argument meaning, return structure and
warnings) for paint_with_words.py:18-45 and 207-388 so that the parity tests read like calls to the
reference.  This is one-time, per-image host work (SURVEY.md 8a rows a-3..a-6); the bilinear
downsample stays the same ATen CPU call the reference makes, which is what keeps the mask
index/downsample step bit-exact.  Differences that do not change results:
  * each region mask is resized once per ratio and reused for every matching token span (the
    reference re-runs F.interpolate per span);
  * the 80 MB `[H,W,77]` ORIG map is kept on the host and only expanded if a UNet level asks for a
    size that has no precomputed key (see `attention.resolve_weight_map`), instead of being uploaded
    and re-interpolated at every attention call (paint_with_words.py:97-101, 343-345).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

RATIOS = (8, 16, 32, 64)


def always_round(x: float) -> int:
    """paint_with_words.py:18-26 -- half-up when int(x) is even, Python round() when odd."""
    whole = int(x)
    if whole % 2:
        return round(x)
    return whole + (0 if x < whole + 0.5 else 1)


def _img_importance_flatten(img: torch.Tensor, w: int, h: int) -> torch.Tensor:
    """paint_with_words.py:38-45 (bilinear, align_corners=True, CPU fp32)."""
    return F.interpolate(img[None, None], size=(w, h), mode="bilinear", align_corners=True).squeeze()


def _rgb_of(color) -> Tuple[int, int, int]:
    if isinstance(color, str):  # "#rrggbb" keys, paint_with_words.py:228-230
        return int(color[1:3], 16), int(color[3:5], 16), int(color[5:7], 16)
    return color


def _image_context_seperator(img, color_context: dict, _tokenizer):
    """paint_with_words.py:207-244.  -> ([(label_token_ids, strength_mask[H,W])...], w, h)."""
    regions: List[Tuple[List[int], torch.Tensor]] = []
    if img is None:
        w, h = 512, 512
    else:
        w, h = img.size
        pixels = np.array(img)
        for color, spec in color_context.items():
            label, _, strength = spec.rpartition(",")
            strength = float(strength)
            ids = _tokenizer(label, max_length=_tokenizer.model_max_length, truncation=True)["input_ids"][1:-1]
            rgb = _rgb_of(color)
            hit = (pixels == rgb).all(axis=-1)        # exact integer colour match
            if not hit.any():
                print(f"Warning : not a single color {rgb} not found in image")
            regions.append((list(ids), torch.from_numpy(hit).to(torch.float32) * strength))
    if not regions:
        regions.append(([-1], torch.zeros((w, h), dtype=torch.float32)))
    return regions, w, h


def _match_positions(token_lis: List[int], label: List[int]) -> List[int]:
    n = len(label)
    return [i for i in range(len(token_lis)) if token_lis[i:i + n] == label]


def _tokens_img_attention_weight(img_context_seperated, tokenized_texts, ratio: int = 8,
                                 original_shape: bool = False) -> torch.Tensor:
    """paint_with_words.py:247-276.  [H_r*W_r, 77] fp32 (or [H_r, W_r, 77])."""
    token_lis = tokenized_texts["input_ids"][0].tolist()
    dim0, dim1 = img_context_seperated[0][1].shape
    r0, r1 = always_round(dim0 / ratio), always_round(dim1 / ratio)
    out = torch.zeros((r0 * r1, len(token_lis)), dtype=torch.float32)
    for label, mask in img_context_seperated:
        starts = _match_positions(token_lis, label)
        if not starts:
            print(f"Warning ratio {ratio} : tokens {label} not found in text")
            continue
        column = _img_importance_flatten(mask, r0, r1).reshape(-1, 1)
        for s in starts:                      # overlapping / repeated labels accumulate (+=)
            out[:, s:s + len(label)] += column
    return out.reshape(r0, r1, len(token_lis)) if original_shape else out


def _tokens_img_attention_factors(img_context_seperated, tokenized_texts, ratio: int = 8):
    """The same weight map as `_tokens_img_attention_weight`, kept in the factored form it is built from:
    W[n, t] = sum_r M[n, r] * C[t, r] with M [N, R] fp32 (column r = region r's resized strength mask,
    paint_with_words.py:269-272) and C [T, R] fp32 (how many matched label spans of region r cover token t,
    paint_with_words.py:259-268; 0/1 unless labels repeat or overlap).  Regions whose label is not in the prompt are
    dropped exactly like the reference drops them.  R is the number of painted regions (5 in the reference's examples),
    so (M, C) is N*R + 77*R numbers instead of N*77 -- the packed mask format of SURVEY 8f-4: the bias
    g*M_b*W = (g*M_b*M) C^T is a dictionary lookup per token instead of a dense [N, 77] fp32 map read per query row.
    Not consumed by a kernel yet (DESIGN.md 8)."""
    token_lis = tokenized_texts["input_ids"][0].tolist()
    dim0, dim1 = img_context_seperated[0][1].shape
    r0, r1 = always_round(dim0 / ratio), always_round(dim1 / ratio)
    cols, counts = [], []
    for label, mask in img_context_seperated:
        starts = _match_positions(token_lis, label)
        if not starts:
            continue
        cnt = torch.zeros(len(token_lis), dtype=torch.float32)
        for s in starts:
            cnt[s:s + len(label)] += 1.0
        cols.append(_img_importance_flatten(mask, r0, r1).reshape(-1))
        counts.append(cnt)
    if not cols:
        return torch.zeros((r0 * r1, 0), dtype=torch.float32), torch.zeros((len(token_lis), 0), dtype=torch.float32)
    return torch.stack(cols, dim=1), torch.stack(counts, dim=1)


PACK_COLS = 32          # fp16 columns per pixel of the packed map (csrc/xattn_fused.cuh: kMW)
PACK_CAPACITY = 10      # distinct non-zero columns a packed map can hold (kRC)
PACK_TOKENS = 80        # padded token count of the column index (kTP)


def pack_weight_map(w: torch.Tensor):
    """Packed form of dense weight maps (SURVEY 8f-4), the input of `pww_xattn_fused_f16`.

    The reference's `[N, 77]` fp32 map (paint_with_words.py:255-272) is a sum of per-region columns: every token of a
    region's label gets the SAME resized strength mask, so the map has only a handful of distinct non-zero columns
    (one per region; one more per token that two regions share).  It is stored as a column dictionary

        w[n, t] == Mu[n, cidx[t]]        Mu [N, R] fp32 (R <= 10), cidx[t] = -1 for an all-zero column

    with Mu split into fp16 halves hi = fp16(Mu), lo = fp16(Mu - hi) so that hi + lo reproduces Mu to 2^-22:
        mpack [Bw, N, 32] fp16 = [ hi(0..9) | lo(0..9) | hi(0..9) | 0 0 ],   cidx [Bw, 80] int8.
    Works on CPU or CUDA tensors (torch ops only; the map builder is host-side set-up work, as in the reference).
    Returns None when a map has more than PACK_CAPACITY distinct non-zero columns or values outside fp16 range --
    such maps take the dense two-launch path."""
    if w.dim() == 2:
        w = w.unsqueeze(0)
    bw, n, t = w.shape
    if t > PACK_TOKENS:
        return None
    w = w.to(torch.float32)
    mpack = torch.zeros((bw, n, PACK_COLS), dtype=torch.float16, device=w.device)
    cidx = torch.full((bw, PACK_TOKENS), -1, dtype=torch.int8, device=w.device)
    for i in range(bw):
        cols = torch.nonzero((w[i] != 0).any(dim=0)).flatten()
        if cols.numel() == 0:
            continue
        uniq, inv = torch.unique(w[i][:, cols].t().contiguous(), dim=0, return_inverse=True)   # rows = distinct columns
        r = uniq.shape[0]
        if r > PACK_CAPACITY or not torch.isfinite(uniq).all() or float(uniq.abs().max()) > 6.0e4:
            return None
        hi = uniq.to(torch.float16)
        lo = (uniq - hi.to(torch.float32)).to(torch.float16)
        mpack[i, :, 0:r] = hi.t()
        mpack[i, :, PACK_CAPACITY:PACK_CAPACITY + r] = lo.t()
        mpack[i, :, 2 * PACK_CAPACITY:2 * PACK_CAPACITY + r] = hi.t()
        cidx[i, cols] = inv.to(torch.int8)
    return mpack, cidx


def unpack_weight_map(mpack: torch.Tensor, cidx: torch.Tensor, tokens: int = 77) -> torch.Tensor:
    """Inverse of `pack_weight_map` (tests / documentation): dense [Bw, N, tokens] fp32 with hi + lo per entry."""
    bw, n, _ = mpack.shape
    mu = mpack[..., :PACK_CAPACITY].to(torch.float32) + mpack[..., PACK_CAPACITY:2 * PACK_CAPACITY].to(torch.float32)
    out = torch.zeros((bw, n, tokens), dtype=torch.float32, device=mpack.device)
    for i in range(bw):
        idx = cidx[i, :tokens].to(torch.int64)
        sel = idx >= 0
        out[i][:, sel] = mu[i][:, idx[sel]]
    return out


def packed_key(n: int) -> str:
    return f"CROSS_ATTENTION_PACKED_{n}"


def _extract_seed_and_sigma_from_context(color_context: dict, ignore_seed: int = -1):
    """paint_with_words.py:279-297: "label,strength[,seed[,blur_sigma]]".  Mutates `color_context`."""
    extra_seeds: Dict[int, int] = {}
    extra_sigmas: Dict[int, float] = {}
    for i, key in enumerate(list(color_context.keys())):
        fields = color_context[key].split(",")
        if len(fields) > 2:
            try:
                seed, sigma = int(fields[-2]), float(fields[-1])
                fields = fields[:-2]
                extra_sigmas[i] = sigma
            except ValueError:
                seed = int(fields[-1])
                fields = fields[:-1]
            if seed != ignore_seed:
                extra_seeds[i] = seed
        color_context[key] = ",".join(fields)
    return color_context, extra_seeds, extra_sigmas


def _get_binary_mask(seperated_word_contexts, extra_seeds, dtype, size):
    """paint_with_words.py:300-304."""
    return [F.interpolate((seperated_word_contexts[k][1] > 0).type(dtype)[None, None], size=size, mode="bilinear")
            for k in extra_seeds.keys()]


def _gaussian_kernel1d(ks: int, sigma: float) -> torch.Tensor:
    half = (ks - 1) * 0.5
    x = torch.linspace(-half, half, steps=ks)
    pdf = torch.exp(-0.5 * (x / sigma).pow(2))
    return pdf / pdf.sum()


def _blur_image_mask(seperated_word_contexts, extra_sigmas):
    """paint_with_words.py:307-312: GaussianBlur(39, sigma) of the full-resolution strength masks
    (separable kernel, reflect padding -- the torchvision algorithm, restated so torchvision is not a
    dependency of the product)."""
    for k, sigma in extra_sigmas.items():
        ids, mask = seperated_word_contexts[k]
        k1 = _gaussian_kernel1d(39, sigma)
        k2 = torch.mm(k1[:, None], k1[None, :])
        padded = F.pad(mask[None, None], [19, 19, 19, 19], mode="reflect")
        seperated_word_contexts[k] = (ids, F.conv2d(padded, k2[None, None])[0, 0])
    return seperated_word_contexts


def weight_key(n: int) -> str:
    return f"CROSS_ATTENTION_WEIGHT_{n}"


def _encode_text_color_inputs(text_encoder, tokenizer, device, color_map_image, color_context,
                              input_prompt, unconditional_input_prompt, use_blur: bool = True):
    """paint_with_words.py:315-388 (and the pipeline-class copy 561-627, which ignores blur sigmas:
    pass use_blur=False for that behaviour).  Returns
    (extra_seeds, seperated_word_contexts, encoder_hidden_states, uncond_encoder_hidden_states)."""
    text_input = tokenizer([input_prompt], padding="max_length", max_length=tokenizer.model_max_length,
                           truncation=True, return_tensors="pt")
    color_context, extra_seeds, extra_sigmas = _extract_seed_and_sigma_from_context(color_context)
    seperated_word_contexts, width, height = _image_context_seperator(color_map_image, color_context, tokenizer)
    if use_blur and len(extra_sigmas) > 0:
        print("Use extra sigma to smooth mask", extra_sigmas)
        seperated_word_contexts = _blur_image_mask(seperated_word_contexts, extra_sigmas)

    cond = {"CONTEXT_TENSOR": None}
    uncond = {"CONTEXT_TENSOR": None}
    # ratio 1 keeps [H,W,77] and stays on the host (see module docstring)
    cond["CROSS_ATTENTION_WEIGHT_ORIG"] = _tokens_img_attention_weight(
        seperated_word_contexts, text_input, ratio=1, original_shape=True)
    uncond["CROSS_ATTENTION_WEIGHT_ORIG"] = 0
    for r in RATIOS:
        key = weight_key(always_round(height / r) * always_round(width / r))
        cond[key] = _tokens_img_attention_weight(seperated_word_contexts, text_input, ratio=r).to(device)
        uncond[key] = 0

    cond["CONTEXT_TENSOR"] = text_encoder(text_input.input_ids.to(device))[0]
    uncond_input = tokenizer([unconditional_input_prompt], padding="max_length",
                             max_length=text_input.input_ids.shape[-1], return_tensors="pt")
    uncond["CONTEXT_TENSOR"] = text_encoder(uncond_input.input_ids.to(device))[0]
    return extra_seeds, seperated_word_contexts, cond, uncond


def expand_orig_weight_map(w_orig: torch.Tensor, n: int) -> torch.Tensor:
    """paint_with_words.py:97-101: the KeyError path -- derive an [n,77] map from the [H,W,77] ORIG map
    with the same two interpolate calls, once per n instead of once per attention call."""
    img_h, img_w, nc = w_orig.shape
    ratio = math.sqrt(img_h * img_w / n)
    w = F.interpolate(w_orig.permute(2, 0, 1).unsqueeze(0), scale_factor=1 / ratio, mode="bilinear",
                      align_corners=True)
    return F.interpolate(w.reshape(1, nc, -1), size=(n,), mode="nearest").permute(2, 1, 0).squeeze().contiguous()
