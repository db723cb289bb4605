"""CPU reference loop with guidance rescale and any prediction type -- TEST INFRASTRUCTURE.

`oracle.loop.reference_denoise_loop`'s control flow (two batch-1 UNet forwards per step, CFG), then diffusers'
`rescale_noise_cfg` (Lin et al. 2023, "Common Diffusion Noise Schedules and Sample Steps are Flawed", section 3.4)
restated in torch fp32, then the host `scheduler.step`, which reads the model output as the scheduler's
`prediction_type` says.  With guidance_rescale = 0 it is `reference_denoise_loop`, as diffusers skips the rescale then.
"""
from __future__ import annotations

from typing import Callable, Optional

import torch


def rescale_noise_cfg(noise_cfg: torch.Tensor, noise_pred_text: torch.Tensor, guidance_rescale: float) -> torch.Tensor:
    """diffusers' rescale_noise_cfg: the guided output rescaled to the cond output's std (unbiased, per image), then
    mixed with the unrescaled one by guidance_rescale."""
    dims = list(range(1, noise_pred_text.ndim))
    std_text = noise_pred_text.std(dim=dims, keepdim=True)
    std_cfg = noise_cfg.std(dim=dims, keepdim=True)
    noise_pred_rescaled = noise_cfg * (std_text / std_cfg)
    return guidance_rescale * noise_pred_rescaled + (1 - guidance_rescale) * noise_cfg


@torch.no_grad()
def reference_rescale_loop(unet, scheduler, cond: dict, uncond: dict, latents: torch.Tensor,
                           weight_function: Callable, guidance_scale: float = 7.5, guidance_rescale: float = 0.0,
                           timesteps=None, extra_input: Optional[torch.Tensor] = None) -> torch.Tensor:
    timesteps = scheduler.timesteps if timesteps is None else timesteps
    for t in timesteps:
        step_index = (scheduler.timesteps == t).nonzero().item()
        sigma = scheduler.sigmas[step_index]
        x = scheduler.scale_model_input(latents, t)
        if extra_input is not None:
            x = torch.cat([x, extra_input], dim=1)
        cond.update({"SIGMA": sigma, "WEIGHT_FUNCTION": weight_function})
        out_text = unet(x, t, encoder_hidden_states=cond).sample
        uncond.update({"SIGMA": sigma, "WEIGHT_FUNCTION": lambda w, sigma, qk: 0.0})
        out_uncond = unet(x, t, encoder_hidden_states=uncond).sample
        noise_pred = out_uncond + guidance_scale * (out_text - out_uncond)
        if guidance_rescale > 0.0:
            noise_pred = rescale_noise_cfg(noise_pred.float(), out_text.float(), guidance_rescale)
        latents = scheduler.step(noise_pred, t, latents).prev_sample
    return latents
