"""CPU restatement of the PwW loop with T2I-Adapter and ControlNet units (pww_controlnet/scripts/hook_pww.py:23-179,
adapter.py:94-107) -- TEST INFRASTRUCTURE.

`reference_adapter_loop` is `oracle.multi_controlnet_loop.reference_multi_controlnet_loop` with units that are either
ControlNets or adapters: fp32 on the CPU, two batch-1 UNet forwards per step, attention patched with
`oracle.loop.patch_with_oracle`, the adapter features and ControlNet residuals added in the UNet's torch (slow) path.
The loop-level parity oracle for `PwWSampler(controlnet=[...])` with adapters among the units.
"""
from __future__ import annotations

from typing import Callable, Optional, Sequence

import torch
import torch.nn.functional as F

GUESS_SCALES = (0.25, 0.62, 0.825, 1.0)     # hook_pww.py:130, as the per-level product it stands for


@torch.no_grad()
def reference_adapter_loop(unet, units: Sequence, is_adapter: Sequence[bool], scheduler, cond: dict, uncond: dict,
                           latents: torch.Tensor, weight_function: Callable, control_images: Sequence[torch.Tensor],
                           guidance_scale: float = 7.5, conditioning_scales: Sequence[float] = None,
                           guess_modes: Sequence[bool] = None, control_guidance_starts: Sequence[float] = None,
                           control_guidance_ends: Sequence[float] = None, timesteps=None,
                           extra_input: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Unit u (model `units[u]`, an adapter iff `is_adapter[u]`, hint `control_images[u]` [1,3,H,W] in [0,1], weight,
    guess mode, window) is active at step i of n iff start_u <= i/n <= end_u (hook_pww.py:23-26).

    An adapter runs once, on its hint alone (PlugableAdapter caches `self.control`), giving 4 batch-1 features.  At
    each step an active adapter's feature l is multiplied by its weight, times GUESS_SCALES[l] if the unit is in guess
    mode, and added to `total_adapter[l]` in unit order (:123-139); the UNet adds total_adapter[l] to the output of
    encoder level l's last layer (:156-163), resized (nearest) to it where the sizes differ (:55-61), so the skip
    carries it.  ControlNet units are as in the multi-ControlNet oracle.  If ANY unit is in guess mode, the uncond
    forward gets neither features nor residuals (`cfg_based_adder`, :39-53)."""
    U = len(units)
    timesteps = scheduler.timesteps if timesteps is None else timesteps
    n = len(timesteps)
    weights = [1.0] * U if conditioning_scales is None else list(conditioning_scales)
    guesses = [False] * U if guess_modes is None else list(guess_modes)
    starts = [0.0] * U if control_guidance_starts is None else list(control_guidance_starts)
    ends = [1.0] * U if control_guidance_ends is None else list(control_guidance_ends)
    routed = any(guesses)
    scales = []
    for w, g, ad in zip(weights, guesses, is_adapter):
        if ad:
            scales.append([w * s for s in GUESS_SCALES] if g else [w] * 4)
        else:
            scales.append([w * (0.825 ** float(12 - k)) if g else w for k in range(13)])
    # the adapter picks the hint's first channel itself when it takes one (adapter.py:101-104)
    features = {u: units[u](control_images[u]) for u in range(U) if is_adapter[u]}

    # the UNet's encoder level sizes: its downsamplers are 3x3 convs with stride 2 and padding 1
    h, w = latents.shape[-2:]
    sizes = [(h, w)]
    for _ in range(3):
        h, w = (h + 2 - 3) // 2 + 1, (w + 2 - 3) // 2 + 1
        sizes.append((h, w))

    def control(x, t, ctx, active):
        total_control, total_adapter = None, None
        for u in range(U):
            if not active[u]:
                continue
            if is_adapter[u]:
                res = [f * s for f, s in zip(features[u], scales[u])]
                total_adapter = res if total_adapter is None else [a + r for a, r in zip(total_adapter, res)]
                continue
            down, mid = units[u](x[:, :4], t, encoder_hidden_states=ctx, controlnet_cond=control_images[u],
                                 return_dict=False)
            res = [r * s for r, s in zip(list(down) + [mid], scales[u])]
            total_control = res if total_control is None else [a + r for a, r in zip(total_control, res)]
        kw = {}
        if total_control is not None:
            kw.update(down_block_additional_residuals=total_control[:-1], mid_block_additional_residual=total_control[-1])
        if total_adapter is not None:
            kw["down_intrablock_additional_residuals"] = [
                f if tuple(f.shape[-2:]) == s else F.interpolate(f, size=s, mode="nearest")
                for f, s in zip(total_adapter, sizes)]
        return kw

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
