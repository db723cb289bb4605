"""CPU restatement of the PwW + ControlNet denoising loop (pww_controlnet/scripts/hook_pww.py) -- TEST INFRASTRUCTURE.

`reference_controlnet_loop` is `oracle.loop.reference_denoise_loop` with the extension's ControlNet semantics added:
fp32 on the CPU, two batch-1 UNet forwards per step, attention patched with `oracle.loop.patch_with_oracle` (the
ControlNet's attention modules are the same class, so the patch covers them), residuals scaled and added in the UNet's
torch (slow) path.  The loop-level parity oracle for `PwWSampler(controlnet=...)`.
"""
from __future__ import annotations

from typing import Callable, Optional

import torch


@torch.no_grad()
def reference_controlnet_loop(unet, controlnet, scheduler, cond: dict, uncond: dict, latents: torch.Tensor,
                              weight_function: Callable, control_image: torch.Tensor, guidance_scale: float = 7.5,
                              conditioning_scale: float = 1.0, guess_mode: bool = False,
                              control_guidance_start: float = 0.0, control_guidance_end: float = 1.0, timesteps=None,
                              extra_input: Optional[torch.Tensor] = None) -> torch.Tensor:
    """At step i of n with start <= i/n <= end (hook_pww.py:23-26) the ControlNet runs on the 4 latent channels of the
    UNet input (:113-119), with the same timestep, the hint image (`control_image` [1,3,H,W] in [0,1], embedded anew
    every step as the extension does) and the PLAIN text context (the PwW dict is built only afterwards, :144-149):
    once on the cond context and, unless in guess mode, once on the uncond context.  Residual k (0..12) is multiplied
    by the weight, times 0.825 ** (12 - k) in guess mode (:123-136), and the UNet adds it to skip k / the mid output
    (:166-175).  In guess mode only the cond forward gets residuals (`cfg_based_adder`, :39-53)."""
    timesteps = scheduler.timesteps if timesteps is None else timesteps
    n = len(timesteps)
    scales = [conditioning_scale * (0.825 ** float(12 - k)) if guess_mode else conditioning_scale for k in range(13)]

    def control(x, t, ctx):
        down, mid = controlnet(x[:, :4], t, encoder_hidden_states=ctx, controlnet_cond=control_image,
                               return_dict=False)
        res = [r * s for r, s in zip(list(down) + [mid], scales)]
        return {"down_block_additional_residuals": res[:-1], "mid_block_additional_residual": res[-1]}

    for i, t in enumerate(timesteps):
        step_index = (scheduler.timesteps == t).nonzero().item()
        sigma = scheduler.sigmas[step_index]
        x = scheduler.scale_model_input(latents, t)
        if extra_input is not None:
            x = torch.cat([x, extra_input], dim=1)
        active = control_guidance_start <= i / n <= control_guidance_end
        res_c = control(x, t, cond["CONTEXT_TENSOR"]) if active else {}
        res_u = control(x, t, uncond["CONTEXT_TENSOR"]) if active and not guess_mode else {}
        cond.update({"SIGMA": sigma, "WEIGHT_FUNCTION": weight_function})
        eps_text = unet(x, t, encoder_hidden_states=cond, **res_c).sample
        uncond.update({"SIGMA": sigma, "WEIGHT_FUNCTION": lambda w, sigma, qk: 0.0})
        eps_uncond = unet(x, t, encoder_hidden_states=uncond, **res_u).sample
        noise_pred = eps_uncond + guidance_scale * (eps_text - eps_uncond)
        latents = scheduler.step(noise_pred, t, latents).prev_sample
    return latents
