"""CPU restatement of the PwW + Multi-ControlNet denoising loop (pww_controlnet/scripts/hook_pww.py:100-139) -- TEST
INFRASTRUCTURE.

`reference_multi_controlnet_loop` is `oracle.controlnet_loop.reference_controlnet_loop` with several control units:
fp32 on the CPU, two batch-1 UNet forwards per step, attention patched with `oracle.loop.patch_with_oracle`, the summed
residuals added in the UNet's torch (slow) path.  The loop-level parity oracle for `PwWSampler(controlnet=[...])`.
"""
from __future__ import annotations

from typing import Callable, Optional, Sequence

import torch


@torch.no_grad()
def reference_multi_controlnet_loop(unet, controlnets: Sequence, scheduler, cond: dict, uncond: dict,
                                    latents: torch.Tensor, weight_function: Callable,
                                    control_images: Sequence[torch.Tensor], guidance_scale: float = 7.5,
                                    conditioning_scales: Sequence[float] = None, guess_modes: Sequence[bool] = None,
                                    control_guidance_starts: Sequence[float] = None,
                                    control_guidance_ends: Sequence[float] = None, timesteps=None,
                                    extra_input: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Unit u (ControlNet `controlnets[u]`, hint `control_images[u]` [1,3,H,W] in [0,1], weight, guess mode, window)
    is active at step i of n iff start_u <= i/n <= end_u (hook_pww.py:23-26).  Each active unit runs on the 4 latent
    channels of the UNet input with the plain text context, once on the cond context and, unless ANY unit is in guess
    mode (`self.guess_mode = any(...)`, :199), once on the uncond context.  Its residual k is multiplied by its weight,
    times 0.825 ** (12 - k) if the unit itself is in guess mode (:123-132), and added to a per-level total in unit order
    (`total_control[idx] += item`, :136-139).  The UNet adds the totals to its skips / mid output; with guess-mode
    routing the uncond forward gets none (`cfg_based_adder`, :39-53)."""
    U = len(controlnets)
    timesteps = scheduler.timesteps if timesteps is None else timesteps
    n = len(timesteps)
    weights = [1.0] * U if conditioning_scales is None else list(conditioning_scales)
    guesses = [False] * U if guess_modes is None else list(guess_modes)
    starts = [0.0] * U if control_guidance_starts is None else list(control_guidance_starts)
    ends = [1.0] * U if control_guidance_ends is None else list(control_guidance_ends)
    routed = any(guesses)
    scales = [[w * (0.825 ** float(12 - k)) if g else w for k in range(13)] for w, g in zip(weights, guesses)]

    def control(x, t, ctx, active):
        total = None
        for u in range(U):
            if not active[u]:
                continue
            down, mid = controlnets[u](x[:, :4], t, encoder_hidden_states=ctx, controlnet_cond=control_images[u],
                                       return_dict=False)
            res = [r * s for r, s in zip(list(down) + [mid], scales[u])]
            total = res if total is None else [a + r for a, r in zip(total, res)]
        if total is None:
            return {}
        return {"down_block_additional_residuals": total[:-1], "mid_block_additional_residual": total[-1]}

    for i, t in enumerate(timesteps):
        step_index = (scheduler.timesteps == t).nonzero().item()
        sigma = scheduler.sigmas[step_index]
        x = scheduler.scale_model_input(latents, t)
        if extra_input is not None:
            x = torch.cat([x, extra_input], dim=1)
        active = [s <= i / n <= e for s, e in zip(starts, ends)]
        res_c = control(x, t, cond["CONTEXT_TENSOR"], active)
        res_u = {} if routed else control(x, t, uncond["CONTEXT_TENSOR"], active)
        cond.update({"SIGMA": sigma, "WEIGHT_FUNCTION": weight_function})
        eps_text = unet(x, t, encoder_hidden_states=cond, **res_c).sample
        uncond.update({"SIGMA": sigma, "WEIGHT_FUNCTION": lambda w, sigma, qk: 0.0})
        eps_uncond = unet(x, t, encoder_hidden_states=uncond, **res_u).sample
        noise_pred = eps_uncond + guidance_scale * (eps_text - eps_uncond)
        latents = scheduler.step(noise_pred, t, latents).prev_sample
    return latents
