"""Negative region prompts on the CPU in fp32 -- TEST INFRASTRUCTURE.

`oracle.region_prompt` with the statistic rule of negative region prompts (DESIGN.md section 1, Negative region
prompts): a biased image's max / std covers chunk 0 and the chunks of its own sentences alone (the bit mask
REGION_SENTENCE_CHUNKS of its dict), not the chunks that only the other side's sentences fill.  The uncond dict carries
the negative sentences' chunk weights as its own REGION_WEIGHTS_{N}, so `oracle.loop`'s two batch-1 forwards per step
(cond dict, then uncond dict) need nothing else: the loops of `oracle.region_prompt`, `oracle.loop` and
`oracle.controlnet_loop` run unchanged over a UNet patched here.
"""
from __future__ import annotations

from typing import Callable, List

from . import region_prompt as RO

CHUNK = RO.CHUNK
SENTENCES_KEY = "REGION_SENTENCE_CHUNKS"


def stat_columns(mask: int, t: int) -> List[int]:
    """The key columns of chunk 0 and of the chunks c with bit c of `mask` set, in a context of T = t keys."""
    return [c * CHUNK + j for c in range(t // CHUNK) if c == 0 or (mask >> c) & 1 for j in range(CHUNK)]


def masked_weight_function(f: Callable, mask: int, t: int) -> Callable:
    """The weight function `f` with its statistic taken over the score columns of `stat_columns(mask, t)` alone."""
    cols = stat_columns(mask, t)
    return lambda w, sigma, qk: f(w, sigma, qk[..., cols])


def negative_region_inj_forward(attn, hidden_states, context=None, mask=None):
    """`region_prompt.region_inj_forward` whose bias statistic covers chunk 0 and the dict's own sentence chunks."""
    if isinstance(context, dict) and context.get(SENTENCES_KEY) is not None:
        t = context["CONTEXT_TENSOR"].shape[1]
        context = dict(context, WEIGHT_FUNCTION=masked_weight_function(context["WEIGHT_FUNCTION"],
                                                                       int(context[SENTENCES_KEY]), t))
    return RO.region_inj_forward(attn, hidden_states, context, mask)


def patch_with_negative_region_oracle(unet) -> int:
    """Class-level `__call__` patch installing `negative_region_inj_forward` (undo it by deleting the class's
    `__call__`)."""
    n = 0
    for m in unet.modules():
        if m.__class__.__name__ == "CrossAttention":
            m.__class__.__call__ = negative_region_inj_forward
            n += 1
    return n
