"""CPU reference loop for masked img2img (latent-blend inpainting with any model) -- TEST INFRASTRUCTURE.

`oracle.rescale_loop.reference_rescale_loop`'s control flow (two batch-1 UNet forwards per step, CFG, optional
guidance rescale, the host `scheduler.step`), then after every step the area outside the mask is put back on the init
latents' noise path at the next step's sigma:

    latents = M * latents + (1 - M) * scheduler.add_noise(init, z, [t'])

t' is the next timestep of the schedule, sigma' = scheduler.sigmas[step_index + 1].  After the last step there is no
t' and sigma' = 0, so the noised init is init + z * 0, add_noise's arithmetic with that sigma.  This is the loop of
diffusers' legacy inpaint pipeline with one deliberate difference: that pipeline noises the init latents to the
current step's t, which leaves sigma_last of noise in the kept area; here they end as `init` exactly.
"""
from __future__ import annotations

from typing import Callable, Optional

import torch

from .rescale_loop import rescale_noise_cfg


def noised_init(scheduler, init: torch.Tensor, noise: torch.Tensor, step_index: int) -> torch.Tensor:
    """The init latents noised to sigma' = sigmas[step_index + 1]: `scheduler.add_noise` at the next timestep, or
    init + noise * 0 after the last one."""
    if step_index + 1 < len(scheduler.timesteps):
        return scheduler.add_noise(init, noise, scheduler.timesteps[step_index + 1:step_index + 2])
    return init + noise * scheduler.sigmas[step_index + 1].to(init.dtype)


@torch.no_grad()
def reference_mask_blend_loop(unet, scheduler, cond: dict, uncond: dict, latents: torch.Tensor,
                              weight_function: Callable, init: torch.Tensor, noise: torch.Tensor, mask: torch.Tensor,
                              guidance_scale: float = 7.5, guidance_rescale: float = 0.0, timesteps=None,
                              extra_input: Optional[torch.Tensor] = None) -> torch.Tensor:
    """`latents` are the start latents (init + sigma_0 noise for img2img); `mask` [1, 1, h, w], 1 = repaint."""
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
        latents = mask * latents + (1 - mask) * noised_init(scheduler, init, noise, step_index)
    return latents
