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
from typing import Dict, List, Optional, Sequence, Tuple

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


def _token_region_counts(img_context_seperated, token_lis: List[int]) -> List[Optional[torch.Tensor]]:
    """Per region (in order): fp32 [T] counts of the matched spans of its label covering each token -- the columns
    `_tokens_img_attention_weight` adds the region's mask into -- or None when the label is not in the prompt."""
    out: List[Optional[torch.Tensor]] = []
    for label, _ in img_context_seperated:
        starts = _match_positions(token_lis, label)
        if not starts:
            out.append(None)
            continue
        cnt = torch.zeros(len(token_lis), dtype=torch.float32)
        for s in starts:
            cnt[s:s + len(label)] += 1.0
        out.append(cnt)
    return out


MAX_RECORDED_REGIONS = 16    # region slots of the attention recording (csrc/xattn_core.cuh: kRegions)
REGION_INDEX_KEY = "REGION_TOKEN_INDEX"   # cond-dict key of `region_token_index`'s row
REGION_COUNT_KEY = "REGION_COUNT"         # cond-dict key of the number of regions (the row's slots 0 .. count - 1)


def region_token_index(img_context_seperated, tokenized_texts) -> torch.Tensor:
    """Token -> region row of one image for attention recording (`pww_xattn_fused_rec_f16`): int8 [80 k] in the packed
    map's column layout (k key chunks; token 77 c + j at column 80 c + j, `_cidx_columns`), entry = the index in
    `color_context` order of the region whose label covers the token, -1 for tokens of no region.

    A token belongs to region r when a matched span of r's label covers it: exactly the token columns the reference's
    `_tokens_img_attention_weight` adds r's mask into (the incidence of `_tokens_img_attention_factors`).  A token
    covered by the labels of several regions goes to the FIRST of them in `color_context` order.  A region whose label
    is not in the prompt gets no tokens.  A long prompt (k = 2, 3) maps its concatenated ids.  More than 16 regions
    raises ValueError."""
    if len(img_context_seperated) > MAX_RECORDED_REGIONS:
        raise ValueError(f"attention recording takes at most {MAX_RECORDED_REGIONS} regions, got "
                         f"{len(img_context_seperated)}")
    token_lis = tokenized_texts["input_ids"][0].tolist()
    t = len(token_lis)
    k = key_chunks(t)
    if k == 0:
        raise ValueError(f"no attention kernel for a context of {t} tokens")
    owner = torch.full((t,), -1, dtype=torch.int8)
    for r, cnt in enumerate(_token_region_counts(img_context_seperated, token_lis)):
        if cnt is not None:
            owner[(cnt > 0) & (owner < 0)] = r
    row = torch.full((PACK_TOKENS * k,), -1, dtype=torch.int8)
    row[_cidx_columns(t)] = owner
    return row


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
    for (label, mask), cnt in zip(img_context_seperated, _token_region_counts(img_context_seperated, token_lis)):
        if cnt is None:
            continue
        cols.append(_img_importance_flatten(mask, r0, r1).reshape(-1))
        counts.append(cnt)
    if not cols:
        return torch.zeros((r0 * r1, 0), dtype=torch.float32), torch.zeros((len(token_lis), 0), dtype=torch.float32)
    return torch.stack(cols, dim=1), torch.stack(counts, dim=1)


PACK_COLS = 32          # fp16 columns per pixel of the packed map (csrc/xattn_fused2.cuh: kMW)
PACK_CAPACITY = 10      # distinct non-zero columns a packed map can hold (kRC)
PACK_TOKENS = 80        # padded token count of the column index (kTP), per key chunk
CHUNK_TOKENS = 77       # one CLIP window: [BOS] + up to 75 prompt tokens + [EOS] (+ padding)
MAX_PROMPT_CHUNKS = 3   # longest context the attention kernels take: T = 231


def key_chunks(t: int) -> int:
    """Key chunks of a context of t tokens as the attention kernels stage it: 1 for t <= 80, k for t = 77 k (k = 2, 3),
    0 for any other length (no kernel)."""
    if t <= PACK_TOKENS:
        return 1
    k, r = divmod(t, CHUNK_TOKENS)
    return k if r == 0 and 2 <= k <= MAX_PROMPT_CHUNKS else 0


def _cidx_columns(t: int) -> torch.Tensor:
    """Column of token j in the packed column index: j itself for t <= 80; for a chunked context token 77 c + i sits at
    column 80 c + i (columns 80 c + 77 .. 80 c + 79 stay -1)."""
    j = torch.arange(t)
    return j if t <= PACK_TOKENS else j // CHUNK_TOKENS * PACK_TOKENS + j % CHUNK_TOKENS


def pack_weight_map(w: torch.Tensor):
    """Packed form of dense weight maps (SURVEY 8f-4), the input of `pww_xattn_fused_f16`.

    The reference's `[N, 77]` fp32 map (paint_with_words.py:255-272) is a sum of per-region columns: every token of a
    region's label gets the SAME resized strength mask, so the map has only a handful of distinct non-zero columns
    (one per region; one more per token that two regions share).  It is stored as a column dictionary

        w[n, t] == Mu[n, cidx[t]]        Mu [N, R] fp32 (R <= 10), cidx[t] = -1 for an all-zero column

    with Mu split into fp16 halves hi = fp16(Mu), lo = fp16(Mu - hi) so that hi + lo reproduces Mu to 2^-22:
        mpack [Bw, N, 32] fp16 = [ hi(0..9) | lo(0..9) | hi(0..9) | 0 0 ],   cidx [Bw, 80 k] int8.
    k is the number of key chunks: 1 for T <= 80; for a long context of k CLIP chunks (T = 154, 231) token 77 c + j is
    at column 80 c + j and the three padding columns of each chunk are -1.
    Works on CPU or CUDA tensors (torch ops only; the map builder is host-side set-up work, as in the reference).
    Returns None when a map has more than PACK_CAPACITY distinct non-zero columns, values outside fp16 range or a
    token count without a kernel -- such maps take the dense two-launch path."""
    if w.dim() == 2:
        w = w.unsqueeze(0)
    bw, n, t = w.shape
    k = key_chunks(t)
    if k == 0:
        return None
    w = w.to(torch.float32)
    mpack = torch.zeros((bw, n, PACK_COLS), dtype=torch.float16, device=w.device)
    cidx = torch.full((bw, PACK_TOKENS * k), -1, dtype=torch.int8, device=w.device)
    col = _cidx_columns(t).to(w.device)
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
        cidx[i, col[cols]] = inv.to(torch.int8)
    return mpack, cidx


def unpack_weight_map(mpack: torch.Tensor, cidx: torch.Tensor, tokens: int = 77) -> torch.Tensor:
    """Inverse of `pack_weight_map` (tests / documentation): dense [Bw, N, tokens] fp32 with hi + lo per entry."""
    bw, n, _ = mpack.shape
    mu = mpack[..., :PACK_CAPACITY].to(torch.float32) + mpack[..., PACK_CAPACITY:2 * PACK_CAPACITY].to(torch.float32)
    out = torch.zeros((bw, n, tokens), dtype=torch.float32, device=mpack.device)
    col = _cidx_columns(tokens).to(cidx.device)
    for i in range(bw):
        idx = cidx[i, col].to(torch.int64)
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


def _special_ids(tokenizer, length: int) -> Tuple[int, int, int]:
    """(BOS, EOS, padding id) as the tokenizer lays out one padded window."""
    row = list(tokenizer([""], padding="max_length", max_length=length)["input_ids"][0])
    return row[0], row[1], row[-1]


def _prompt_windows(ids: List[int], labels: List[List[int]], max_chunks: int, width: int) -> List[List[int]]:
    """Split prompt token ids (without BOS / EOS) into at most `max_chunks` windows of at most `width` tokens.  A window
    never ends inside a span where a region label matches: it ends before the span instead, so every label that fits is
    matched inside one chunk.  Tokens past the last window are dropped (truncation, as with one window)."""
    spans = [(s, s + len(lab)) for lab in labels if lab for s in _match_positions(ids, lab)]
    windows: List[List[int]] = []
    pos = 0
    while pos < len(ids) and len(windows) < max_chunks:
        end = min(pos + width, len(ids))
        if end < len(ids):
            cut = end
            while True:
                inside = [a for a, b in spans if a < cut < b]
                if not inside:
                    break
                cut = min(inside)
            if cut > pos:                  # overlapping spans longer than a window: keep the plain cut
                end = cut
        windows.append(ids[pos:end])
        pos = end
    return windows


def _chunked_ids(tokenizer, windows: List[List[int]], chunks: int) -> torch.Tensor:
    """[1, 77 * chunks] ids: each window as [BOS] + window + [EOS] padded to one 77-token chunk, then empty chunks."""
    length = tokenizer.model_max_length
    bos, eos, pad = _special_ids(tokenizer, length)
    rows = []
    for c in range(chunks):
        win = windows[c] if c < len(windows) else []
        rows += [bos] + list(win) + [eos] + [pad] * (length - 2 - len(win))
    return torch.tensor([rows], dtype=torch.long)


def _encode_chunked(text_encoder, ids: torch.Tensor, device) -> torch.Tensor:
    """Each 77-token chunk through the text encoder on its own, concatenated along tokens (the A1111 / compel layout)."""
    length = CHUNK_TOKENS
    return torch.cat([text_encoder(ids[:, c:c + length].to(device))[0] for c in range(0, ids.shape[1], length)], 1)


def chunk_prompt(tokenizer, prompt: str, labels: Sequence[str] = (), max_prompt_chunks: int = 1) -> torch.Tensor:
    """Token ids [1, 77 k] of `prompt` in k <= `max_prompt_chunks` CLIP windows of up to 75 tokens (k = 1: the
    tokenizer's own padded, truncated window).  `labels` are the region labels: no window ends inside one of their
    matches.  A label longer than one window raises ValueError."""
    if not 1 <= max_prompt_chunks <= MAX_PROMPT_CHUNKS:
        raise ValueError(f"max_prompt_chunks must be 1 .. {MAX_PROMPT_CHUNKS}, got {max_prompt_chunks}")
    length = tokenizer.model_max_length
    if max_prompt_chunks == 1:
        return tokenizer([prompt], padding="max_length", max_length=length, truncation=True,
                         return_tensors="pt")["input_ids"]
    width = length - 2
    ids = list(tokenizer(prompt)["input_ids"])[1:-1]
    lab_ids = []
    for label in labels:
        li = list(tokenizer(label)["input_ids"])[1:-1]
        if len(li) > width:
            raise ValueError(f"region label {label!r} is {len(li)} tokens long; a label must fit one {width}-token window")
        lab_ids.append(li)
    windows = _prompt_windows(ids, lab_ids, max_prompt_chunks, width)
    return _chunked_ids(tokenizer, windows, max(1, len(windows)))


MAX_REGION_PROMPTS = 2          # 1 + 2 chunks of 77: the longest context the attention kernels take (T = 231)
REGION_SIDE = 64                # colour-map sides must be multiples of this: every UNet level then has its weights


def region_key(n: int) -> str:
    """Dict key of the region-prompt chunk weights of the level with n query rows: fp32 [n, 1 + R] on the device."""
    return f"REGION_WEIGHTS_{n}"


def check_region_prompts(region_prompts, region_base_ratio: float, max_prompt_chunks: int = 1) -> None:
    """The ValueErrors of region prompts that do not need the tokenizer or the colour map."""
    if not isinstance(region_prompts, dict) or not 1 <= len(region_prompts) <= MAX_REGION_PROMPTS:
        n = len(region_prompts) if isinstance(region_prompts, dict) else region_prompts
        raise ValueError(f"region_prompts takes 1 .. {MAX_REGION_PROMPTS} colour -> sentence entries, got {n}")
    if max_prompt_chunks > 1:
        raise ValueError("region prompts and max_prompt_chunks > 1 do not combine: the base prompt is one 77-token chunk")
    if not 0.0 <= float(region_base_ratio) <= 1.0:
        raise ValueError(f"region_base_ratio must be in [0, 1], got {region_base_ratio}")


def region_chunk_ids(tokenizer, input_prompt: str, region_prompts: dict, base_name: str = "input_prompt",
                     sentence_name: str = "region prompt") -> torch.Tensor:
    """[1, 77 (1 + R)] ids: the base prompt, then each region's sentence in dict order, each as [BOS] + tokens + [EOS]
    + padding in a chunk of its own.  A prompt longer than 75 tokens raises ValueError (naming it `base_name` or
    `sentence_name` and its colour)."""
    width = tokenizer.model_max_length - 2
    windows = []
    for what, text in [(base_name, input_prompt)] + [(f"{sentence_name} {k!r}", v) for k, v in region_prompts.items()]:
        ids = list(tokenizer(text)["input_ids"])[1:-1]
        if len(ids) > width:
            raise ValueError(f"{what} is {len(ids)} tokens long; with region prompts every prompt must fit one "
                             f"{width}-token window")
        windows.append(ids)
    return _chunked_ids(tokenizer, windows, len(windows))


def region_chunk_weights(color_map_image, region_prompts: dict, region_base_ratio: float, ratio: int,
                         layout: Optional[Sequence] = None) -> torch.Tensor:
    """fp32 [N, 1 + R] chunk weights of the level with latent ratio `ratio` (CPU):
        w_c = (1 - beta) * f_c   (c >= 1),   w_0 = 1 - sum_{c >= 1} w_c
    with f_c the binary mask of region c's colour resized as the weight maps are (`_img_importance_flatten` to
    always_round(side / ratio)).  A colour absent from the map gives f_c = 0.  `layout` (default: region_prompts'
    colours) is the colour of every chunk c >= 1; a colour of it that region_prompts lacks gets f_c = 0 too."""
    pixels = np.array(color_map_image)
    dim0, dim1 = pixels.shape[:2]
    r0, r1 = always_round(dim0 / ratio), always_round(dim1 / ratio)
    beta = float(region_base_ratio)
    mine = {tuple(_rgb_of(c)) for c in region_prompts}
    cols = []
    for color in (region_prompts if layout is None else layout):
        if tuple(_rgb_of(color)) not in mine:
            cols.append(torch.zeros(r0 * r1, dtype=torch.float32))
            continue
        hit = torch.from_numpy((pixels == _rgb_of(color)).all(axis=-1)).to(torch.float32)
        cols.append((1.0 - beta) * _img_importance_flatten(hit, r0, r1).reshape(-1))
    w = torch.stack(cols, 1)
    return torch.cat([1.0 - w.sum(1, keepdim=True), w], 1).contiguous()


REGION_SENTENCES_KEY = "REGION_SENTENCE_CHUNKS"   # dict key: bit c = chunk c holds a sentence of this side (int)
REGION_ROWS_KEY = "REGION_ROWS"                   # batched-dict key: int32 [B] weight row of every image, -1 = none
STAT_CHUNKS_KEY = "REGION_STAT_CHUNKS"            # batched-dict key: int32 [B] chunks of every image's statistic


def region_layout(region_prompts: Optional[dict], negative_region_prompts: Optional[dict]) -> list:
    """The colour of every chunk c >= 1 of a context with region or negative region prompts: region_prompts' colours
    in dict order, then negative_region_prompts' colours that region_prompts lacks, in dict order (one colour in two
    key forms, "#ff0000" and (255, 0, 0), is one colour)."""
    layout, seen = [], set()
    for prompts in (region_prompts or {}, negative_region_prompts or {}):
        for color in prompts:
            if tuple(_rgb_of(color)) not in seen:
                seen.add(tuple(_rgb_of(color)))
                layout.append(color)
    return layout


def _side_sentences(layout: Sequence, prompts: Optional[dict], base: str) -> Tuple[dict, int]:
    """One side's sentence for every chunk c >= 1 of `layout` (its own, else `base` again) and the bit mask of the
    chunks that hold its own sentences."""
    own = {tuple(_rgb_of(c)): text for c, text in (prompts or {}).items()}
    texts, bits = {}, 0
    for c, color in enumerate(layout, start=1):
        text = own.get(tuple(_rgb_of(color)))
        texts[color] = base if text is None else text
        bits |= 0 if text is None else 1 << c
    return texts, bits


def check_negative_region_prompts(region_prompts, negative_region_prompts, region_base_ratio: float,
                                  max_prompt_chunks: int = 1) -> None:
    """The ValueErrors of negative region prompts that need neither a model nor the colour map (region_prompts may be
    None)."""
    if region_prompts is not None:
        check_region_prompts(region_prompts, region_base_ratio, max_prompt_chunks)
    if not isinstance(negative_region_prompts, dict) or not negative_region_prompts:
        n = len(negative_region_prompts) if isinstance(negative_region_prompts, dict) else negative_region_prompts
        raise ValueError(f"negative_region_prompts takes 1 .. {MAX_REGION_PROMPTS} colour -> sentence entries, got {n}")
    n = len(region_layout(region_prompts, negative_region_prompts))
    if n > MAX_REGION_PROMPTS:
        raise ValueError(f"region_prompts and negative_region_prompts name {n} colours in all; at most "
                         f"{MAX_REGION_PROMPTS} (1 .. {MAX_REGION_PROMPTS} extra 77-token chunks)")
    if max_prompt_chunks > 1:
        raise ValueError("negative region prompts and max_prompt_chunks > 1 do not combine: the base prompts are one "
                         "77-token chunk")
    if not 0.0 <= float(region_base_ratio) <= 1.0:
        raise ValueError(f"region_base_ratio must be in [0, 1], got {region_base_ratio}")


def _encode_text_color_inputs(text_encoder, tokenizer, device, color_map_image, color_context,
                              input_prompt, unconditional_input_prompt, use_blur: bool = True,
                              max_prompt_chunks: int = 1, region_prompts: Optional[dict] = None,
                              region_base_ratio: float = 0.2, negative_region_prompts: Optional[dict] = None):
    """paint_with_words.py:315-388 (and the pipeline-class copy 561-627, which ignores blur sigmas:
    pass use_blur=False for that behaviour).  Returns
    (extra_seeds, seperated_word_contexts, encoder_hidden_states, uncond_encoder_hidden_states).

    `max_prompt_chunks` > 1 lets a prompt longer than 75 tokens fill up to that many 77-token CLIP chunks (T = 77 k,
    see `chunk_prompt`); the uncond prompt is encoded to the same number of chunks, each chunk by the text encoder on its
    own.  A prompt that fits one chunk gives the same dicts as max_prompt_chunks=1 (the reference's behaviour).

    `region_prompts` ({colour: sentence}, 1 or 2 entries, colours of `color_map_image` in `color_context`'s key forms)
    gives every painted region a sentence of its own: the context is 1 + R chunks (the base prompt, then the sentences
    in dict order), and both dicts get `region_key(N)` chunk weights per level (`region_chunk_weights`; the uncond
    dict's are (1, 0, ..) on every row).  `region_base_ratio` is the base prompt's share beta inside a region.

    `negative_region_prompts` ({colour: sentence}) does the same on the uncond side.  The chunks c >= 1 are the colours
    of `region_layout` (at most 2 in all); a side without a sentence for colour c holds its own base prompt again in
    chunk c, with weight 0.  The uncond prompt is then one 75-token chunk, and the uncond dict's weights are
    `region_chunk_weights` over the negative colours.  Both dicts carry REGION_SENTENCES_KEY, the bit mask of the
    chunks holding their own sentences (0 for a side without any), whenever they carry region weights."""
    if not 1 <= max_prompt_chunks <= MAX_PROMPT_CHUNKS:
        raise ValueError(f"max_prompt_chunks must be 1 .. {MAX_PROMPT_CHUNKS}, got {max_prompt_chunks}")
    if negative_region_prompts is not None:
        check_negative_region_prompts(region_prompts, negative_region_prompts, region_base_ratio, max_prompt_chunks)
    elif region_prompts is not None:
        check_region_prompts(region_prompts, region_base_ratio, max_prompt_chunks)
    sided = region_prompts is not None or negative_region_prompts is not None
    if sided:
        if color_map_image is None:
            raise ValueError("region prompts need a color_map_image")
        if color_map_image.size[0] % REGION_SIDE or color_map_image.size[1] % REGION_SIDE:
            raise ValueError(f"region prompts need colour-map sides that are multiples of {REGION_SIDE}, got "
                             f"{color_map_image.size}")
    text_input = tokenizer([input_prompt], padding="max_length", max_length=tokenizer.model_max_length,
                           truncation=True, return_tensors="pt")
    color_context, extra_seeds, extra_sigmas = _extract_seed_and_sigma_from_context(color_context)
    chunks = 1
    layout = region_layout(region_prompts, negative_region_prompts)
    un_ids = None
    if sided:
        texts, cond_bits = _side_sentences(layout, region_prompts, input_prompt)
        text_input = {"input_ids": region_chunk_ids(tokenizer, input_prompt, texts)}
        chunks = 1 + len(layout)
        un_texts, un_bits = _side_sentences(layout, negative_region_prompts, unconditional_input_prompt)
        if negative_region_prompts is not None:
            un_ids = region_chunk_ids(tokenizer, unconditional_input_prompt, un_texts, "unconditional_input_prompt",
                                      "negative region prompt")
    elif max_prompt_chunks > 1:
        labels = [spec.rpartition(",")[0] for spec in color_context.values()] if color_map_image is not None else []
        ids = chunk_prompt(tokenizer, input_prompt, labels, max_prompt_chunks)
        chunks = ids.shape[1] // CHUNK_TOKENS
        if chunks > 1:
            text_input = {"input_ids": ids}
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
    # the token -> region row of attention recording (PwWSampler(record_attention=True)); None: too many regions to record
    cond[REGION_INDEX_KEY] = (region_token_index(seperated_word_contexts, text_input)
                              if len(seperated_word_contexts) <= MAX_RECORDED_REGIONS else None)
    cond[REGION_COUNT_KEY] = len(seperated_word_contexts)
    if sided:
        for r in RATIOS:
            w = region_chunk_weights(color_map_image, region_prompts or {}, region_base_ratio, r, layout)
            n = w.shape[0]
            cond[region_key(n)] = w.to(device)
            if negative_region_prompts is None:
                plain = torch.zeros_like(w)
                plain[:, 0] = 1.0
                uncond[region_key(n)] = plain.to(device)
            else:
                uncond[region_key(n)] = region_chunk_weights(color_map_image, negative_region_prompts,
                                                             region_base_ratio, r, layout).to(device)
        cond[REGION_SENTENCES_KEY] = cond_bits
        uncond[REGION_SENTENCES_KEY] = un_bits

    if chunks > 1:
        cond["CONTEXT_TENSOR"] = _encode_chunked(text_encoder, text_input["input_ids"], device)
        if un_ids is None:
            width = tokenizer.model_max_length - 2
            un_tokens = list(tokenizer(unconditional_input_prompt)["input_ids"])[1:-1]
            un_ids = _chunked_ids(tokenizer, _prompt_windows(un_tokens, [], chunks, width), chunks)
        uncond["CONTEXT_TENSOR"] = _encode_chunked(text_encoder, un_ids, device)
        return extra_seeds, seperated_word_contexts, cond, uncond
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
