"""Region prompts on the CPU in fp32 -- TEST INFRASTRUCTURE.

A restatement of the region-prompt attention (DESIGN.md section 1, Region prompts) and the patch that puts it into a
UNet for `oracle.loop`'s control flow.  For one image, head h and query row n of a context of K chunks of 77 keys:

    out(n) = sum_c w_c(n) * softmax_c(scale * (S_c(n) + bias_c(n))) V_c

softmax_c runs over the 77 keys of chunk c alone; the bias is the reference's weight function applied to the whole
[H, N, 77 K] score tensor, so its statistic is the one over every chunk.  A context without weights takes
(1, 0, ..): the first chunk alone.
"""
from __future__ import annotations

from typing import Callable, Optional

import torch

from . import loop as oracle_loop
from . import pww_oracle

CHUNK = 77


def region_attention_core(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int, scale: float,
                          weights: Optional[torch.Tensor], bias_fn: Optional[Callable] = None,
                          dtype: torch.dtype = torch.float32) -> torch.Tensor:
    """q [1, N, C], k / v [1, 77 K, C], weights [N, K] (None: (1, 0, ..)) -> [1, N, C] in `dtype` (fp32 or fp64)."""
    q, k, v = q.to(dtype), k.to(dtype), v.to(dtype)
    n, t = q.shape[1], k.shape[1]
    kc = t // CHUNK
    if kc * CHUNK != t:
        raise ValueError(f"region prompts need whole 77-key chunks, got T = {t}")
    if weights is None:
        weights = torch.zeros(n, kc, dtype=dtype)
        weights[:, 0] = 1.0
    weights = weights.to(dtype)
    qh, kh, vh = pww_oracle._h2b(q, heads), pww_oracle._h2b(k, heads), pww_oracle._h2b(v, heads)
    s = torch.matmul(qh, kh.transpose(-1, -2))
    if bias_fn is not None:
        bias = bias_fn(s)
        s = s + (bias.to(dtype) if isinstance(bias, torch.Tensor) else bias)
    s = s * scale
    out = torch.zeros_like(qh[..., :1].expand(-1, -1, vh.shape[-1])).clone()
    for c in range(kc):
        sl = slice(c * CHUNK, (c + 1) * CHUNK)
        p = s[..., sl].softmax(dim=-1)
        out = out + weights[:, c].reshape(1, n, 1) * torch.matmul(p, vh[:, sl])
    return pww_oracle._b2h(out, heads)


def region_inj_forward(attn, hidden_states, context=None, mask=None):
    """`pww_oracle.inj_forward` with region prompts: a dict context with `REGION_WEIGHTS_{N}` ([N, K] or [B, N, K])
    takes `region_attention_core`; anything else the oracle's plain path."""
    n = hidden_states.shape[1]
    if not isinstance(context, dict) or f"REGION_WEIGHTS_{n}" not in context:
        return pww_oracle.inj_forward(attn, hidden_states, context, mask)
    ctx = context["CONTEXT_TENSOR"]
    q, k, v = attn.to_q(hidden_states), attn.to_k(ctx), attn.to_v(ctx)
    w = context[f"CROSS_ATTENTION_WEIGHT_{n}"]
    f, sigma = context["WEIGHT_FUNCTION"], context["SIGMA"]
    weights = context[f"REGION_WEIGHTS_{n}"].float().cpu()
    outs = []
    for b in range(q.shape[0]):
        wb = weights[b] if weights.dim() == 3 else weights
        outs.append(region_attention_core(q[b:b + 1], k[b:b + 1], v[b:b + 1], attn.heads, attn.scale, wb,
                                          lambda s: f(w, sigma, s)))
    o = attn.to_out[0](torch.cat(outs, 0).to(hidden_states.dtype))
    return attn.to_out[1](o)


def patch_with_region_oracle(unet) -> int:
    """Class-level `__call__` patch installing `region_inj_forward` (undo it by deleting the class's `__call__`)."""
    n = 0
    for m in unet.modules():
        if m.__class__.__name__ == "CrossAttention":
            m.__class__.__call__ = region_inj_forward
            n += 1
    return n


@torch.no_grad()
def reference_region_loop(unet, scheduler, cond: dict, uncond: dict, latents: torch.Tensor,
                          weight_function: Callable, guidance_scale: float = 7.5, timesteps=None) -> torch.Tensor:
    """`oracle.loop.reference_denoise_loop` over a UNet patched with `region_inj_forward` (the caller patches)."""
    return oracle_loop.reference_denoise_loop(unet, scheduler, cond, uncond, latents, weight_function,
                                              guidance_scale, timesteps=timesteps)
