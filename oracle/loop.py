"""CPU restatement of the reference denoising loop (paint_with_words.py:471-506) -- TEST INFRASTRUCTURE.

Two batch-1 UNet forwards per step (cond dict, then uncond dict with the zero weight function), CFG
combine, LMS step -- exactly the reference's control flow -- over any UNet with the diffusers-0.10
contract whose attention modules are patched with `oracle.pww_oracle.inj_forward`.  Used (a) as the
loop-level parity oracle for `PwWSampler`, (b) as the timed CPU baseline in bench.py
(`cpu_baseline`, `--impl reference`).
"""
from __future__ import annotations

from typing import Callable, Optional

import torch

from . import pww_oracle


def patch_with_oracle(unet, emulate_fp16: bool = False, emulate_dtype: Optional[torch.dtype] = None) -> int:
    """Class-level `__call__` patch as at paint_with_words.py:193-195, installing the oracle's inj_forward
    (`emulate_fp16` / `emulate_dtype`: the rounding points of an eager fp16 / bf16 autocast, see attention_core)."""
    pww_oracle._emulated_dtype(emulate_fp16, emulate_dtype)

    def fwd(self, hidden_states, context=None, mask=None):
        return pww_oracle.inj_forward(self, hidden_states, context, mask, emulate_fp16=emulate_fp16,
                                      emulate_dtype=emulate_dtype)
    n = 0
    for m in unet.modules():
        if m.__class__.__name__ == "CrossAttention":
            m.__class__.__call__ = fwd
            n += 1
    return n


@torch.no_grad()
def reference_denoise_loop(unet, scheduler, cond: dict, uncond: dict, latents: torch.Tensor,
                           weight_function: Callable, guidance_scale: float = 7.5, timesteps=None,
                           extra_input: Optional[torch.Tensor] = None, max_steps: Optional[int] = None,
                           on_step: Optional[Callable[[int], None]] = None) -> torch.Tensor:
    timesteps = scheduler.timesteps if timesteps is None else timesteps
    for i, t in enumerate(timesteps):
        if max_steps is not None and i >= max_steps:
            break
        step_index = (scheduler.timesteps == t).nonzero().item()
        sigma = scheduler.sigmas[step_index]
        x = scheduler.scale_model_input(latents, t)
        if extra_input is not None:
            x = torch.cat([x, extra_input], dim=1)
        cond.update({"SIGMA": sigma, "WEIGHT_FUNCTION": weight_function})
        eps_text = unet(x, t, encoder_hidden_states=cond).sample
        uncond.update({"SIGMA": sigma, "WEIGHT_FUNCTION": lambda w, sigma, qk: 0.0})
        eps_uncond = unet(x, t, encoder_hidden_states=uncond).sample
        noise_pred = eps_uncond + guidance_scale * (eps_text - eps_uncond)
        latents = scheduler.step(noise_pred, t, latents).prev_sample
        if on_step is not None:
            on_step(i)
    return latents
