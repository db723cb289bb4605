"""CPU restatement of diffusers' MultiDiffusion loop (`StableDiffusionPanoramaPipeline`) over paint-with-words
windows -- TEST INFRASTRUCTURE.

`reference_panorama_loop`: per step and window, in window order, `oracle.loop.reference_denoise_loop`'s control flow
on the window's crop (two batch-1 UNet forwards with the window's cond and uncond dicts, CFG), then `scheduler.step`
with that window's own copy of the scheduler state (diffusers keeps one deep copy per view), added into `value`;
after every window, latents = value / count.  Euler ancestral's step noise is the window's crop of one canvas-sized
draw (diffusers draws it per window).  Circular windows read columns (c0 + x) mod W.

`canvas_step_loop`: the same guided outputs averaged per canvas value first (summed in window order from the first
value, divided by the count), then ONE canvas-level `scheduler.step`: the order `PanoramaSampler` computes in.  Every
step form is linear in (x, output, history) with coefficients shared by all windows, so the two loops agree in exact
arithmetic.
"""
from __future__ import annotations

import copy
from typing import Callable, List, Optional, Sequence, Tuple

import torch


def windows_of(views: Tuple[Sequence[int], Sequence[int]], window: int, width: int) -> List[Tuple[int, torch.Tensor]]:
    """(row start, canvas column indices) of every window, in window order."""
    return [(int(r0), torch.arange(int(c0), int(c0) + window) % width) for r0 in views[0] for c0 in views[1]]


def _guided(unet, cond: dict, uncond: dict, x, t, sigma, weight_function: Callable, guidance_scale: float):
    cond.update({"SIGMA": sigma, "WEIGHT_FUNCTION": weight_function})
    eps_text = unet(x, t, encoder_hidden_states=cond).sample
    uncond.update({"SIGMA": sigma, "WEIGHT_FUNCTION": lambda w, sigma, qk: 0.0})
    eps_uncond = unet(x, t, encoder_hidden_states=uncond).sample
    return eps_uncond + guidance_scale * (eps_text - eps_uncond)


def _noise_kw(noise: Optional[torch.Tensor], i: int, r0: Optional[int] = None, cols=None, window: int = 0) -> dict:
    if noise is None:
        return {}
    z = noise[i]
    return {"noise": z if r0 is None else z[:, :, r0:r0 + window][..., cols]}


@torch.no_grad()
def reference_panorama_loop(unet, scheduler, conds: Sequence[dict], unconds: Sequence[dict], latents: torch.Tensor,
                            views, window: int, weight_function: Callable, guidance_scale: float = 7.5,
                            timesteps=None, noise: Optional[torch.Tensor] = None) -> torch.Tensor:
    """diffusers' order: step every window with its own scheduler state, then average the stepped windows.  `noise`
    [n, 1, 4, H, W]: Euler ancestral's canvas noise of each step (None for the other samplers)."""
    timesteps = scheduler.timesteps if timesteps is None else timesteps
    wins = windows_of(views, window, latents.shape[-1])
    states = [copy.deepcopy(scheduler) for _ in wins]
    for i, t in enumerate(timesteps):
        step_index = (scheduler.timesteps == t).nonzero().item()
        sigma = scheduler.sigmas[step_index]
        value, count = torch.zeros_like(latents), torch.zeros_like(latents)
        for v, (r0, cols) in enumerate(wins):
            crop = latents[:, :, r0:r0 + window][..., cols]
            x = scheduler.scale_model_input(crop, t)
            noise_pred = _guided(unet, conds[v], unconds[v], x, t, sigma, weight_function, guidance_scale)
            out = states[v].step(noise_pred, t, crop, **_noise_kw(noise, i, r0, cols, window)).prev_sample
            value[:, :, r0:r0 + window, cols] += out
            count[:, :, r0:r0 + window, cols] += 1
        latents = value / count
    return latents


@torch.no_grad()
def canvas_step_loop(unet, scheduler, conds: Sequence[dict], unconds: Sequence[dict], latents: torch.Tensor,
                     views, window: int, weight_function: Callable, guidance_scale: float = 7.5, timesteps=None,
                     noise: Optional[torch.Tensor] = None) -> torch.Tensor:
    """PanoramaSampler's order: average the windows' guided outputs, then one canvas step."""
    timesteps = scheduler.timesteps if timesteps is None else timesteps
    wins = windows_of(views, window, latents.shape[-1])
    canvas = copy.deepcopy(scheduler)
    for i, t in enumerate(timesteps):
        step_index = (scheduler.timesteps == t).nonzero().item()
        sigma = scheduler.sigmas[step_index]
        total = torch.zeros_like(latents)
        count = torch.zeros_like(latents)
        for v, (r0, cols) in enumerate(wins):
            x = scheduler.scale_model_input(latents[:, :, r0:r0 + window][..., cols], t)
            g = _guided(unet, conds[v], unconds[v], x, t, sigma, weight_function, guidance_scale)
            seen = count[:, :, r0:r0 + window, cols] > 0
            total[:, :, r0:r0 + window, cols] = torch.where(seen, total[:, :, r0:r0 + window, cols] + g, g)
            count[:, :, r0:r0 + window, cols] += 1
        latents = canvas.step(total / count, t, latents, **_noise_kw(noise, i)).prev_sample
    return latents
