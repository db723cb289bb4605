"""CPU restatement of the per-region cross-attention maps -- TEST INFRASTRUCTURE.

The definition `PwWSampler(record_attention=True).attention_maps()` implements, restated in fp32 on the CPU over the
reference loop of `oracle/loop.py`: at every step, every cross-attention call of the COND forward contributes, per
region r, the softmax mass its pixels give to the tokens of r's label,

    mass[h, n, r] = sum_{t in tokens(r)} P[h, n, t] / sum_t P[h, n, t]      (P: `pww_oracle.attention_core`'s softmax)

averaged over heads, reshaped to the call's (h_r, w_r) grid, upsampled bilinearly (align_corners=False) to the latent
grid, and averaged over every recorded (step, call).  tokens(r) are the tokens a matched span of r's label covers (the
columns the reference's `_tokens_img_attention_weight` writes r's mask into); a token of several regions belongs to the
first.  The existing oracle functions are used as they are: the recording wraps `pww_oracle.inj_forward`.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

from . import pww_oracle
from .loop import reference_denoise_loop


def token_regions(label_ids: Sequence[Sequence[int]], token_ids: Sequence[int]) -> List[int]:
    """Region of every token (-1 = none): first region, in order, with a label span covering the token."""
    tok = list(token_ids)
    owner = [-1] * len(tok)
    for r, lab in enumerate(label_ids):
        n = len(lab)
        for s in range(len(tok)):
            if n and tok[s:s + n] == list(lab):
                for t in range(s, s + n):
                    if owner[t] < 0:
                        owner[t] = r
    return owner


def _level_grids(h: int, w: int) -> Dict[int, Tuple[int, int]]:
    """N -> (h_r, w_r) of the weight-map builder at ratios 8, 16, 32, 64 for a latent grid of h x w (image 8h x 8w)."""
    grids = {}
    for r in (8, 16, 32, 64):
        hr, wr = pww_oracle.always_round(8 * h / r), pww_oracle.always_round(8 * w / r)
        grids[hr * wr] = (hr, wr)
    return grids


@torch.no_grad()
def reference_attention_maps(unet, scheduler, cond: dict, uncond: dict, latents: torch.Tensor,
                             weight_function: Callable, owner: Sequence[int], regions: int,
                             guidance_scale: float = 7.5, timesteps=None,
                             extra_input: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """(final latents, maps fp32 [regions, h, w]) of the reference loop over `unet`, whose CrossAttention class is
    patched here for the duration of the call.  owner[t] = region of token t (`token_regions`)."""
    h, w = latents.shape[-2:]
    grids = _level_grids(h, w)
    owner_t = torch.tensor(list(owner), dtype=torch.long)
    total = torch.zeros((regions, h, w), dtype=torch.float32)
    calls = [0]

    def fwd(attn, hidden_states, context=None, mask=None):
        if context is cond:
            q = attn.to_q(hidden_states).float()
            ctx = context["CONTEXT_TENSOR"].float()
            k, v = attn.to_k(ctx).float(), attn.to_v(ctx).float()
            n = q.shape[1]
            wmap = context.get(f"CROSS_ATTENTION_WEIGHT_{n}")
            if wmap is None:
                raise KeyError(f"no weight map for N = {n}")
            f, sigma = context["WEIGHT_FUNCTION"], context["SIGMA"]
            heads, scale = attn.heads, attn.scale
            qh, kh = pww_oracle._h2b(q, heads), pww_oracle._h2b(k, heads)
            s = torch.matmul(qh, kh.transpose(-1, -2))
            bias = f(wmap, sigma, s)
            p = (((s + bias.float()) if isinstance(bias, torch.Tensor) else (s + bias)) * scale).softmax(dim=-1)
            mass = torch.zeros(p.shape[:2] + (regions,), dtype=torch.float32)
            for r in range(regions):
                sel = owner_t == r
                if sel.any():
                    mass[..., r] = p[..., sel].sum(-1) / p.sum(-1)
            hr, wr = grids[n]
            grid = mass.mean(0).reshape(hr, wr, regions).permute(2, 0, 1)[None]
            total.add_(F.interpolate(grid, size=(h, w), mode="bilinear", align_corners=False)[0])
            calls[0] += 1
        return pww_oracle.inj_forward(attn, hidden_states, context, mask)

    classes = {m.__class__ for m in unet.modules() if m.__class__.__name__ == "CrossAttention"}
    saved = {c: c.__dict__.get("__call__") for c in classes}
    try:
        for c in classes:
            c.__call__ = fwd
        out = reference_denoise_loop(unet, scheduler, cond, uncond, latents, weight_function, guidance_scale,
                                     timesteps=timesteps, extra_input=extra_input)
    finally:
        for c, orig in saved.items():
            if orig is None:
                delattr(c, "__call__")
            else:
                c.__call__ = orig
    return out, total / max(1, calls[0])
